// wgmma flash attention for the ViT (SigLIP so400m: 16 heads x head_dim 72, N = 729 keys, non-causal)
//   HF modeling_siglip.py:229-249,293-306 (softmax(q k^T * d^-1/2) v), reference call site v1/modeling_detikzify.py:63-72.
//
// One CTA = 128 queries of one (image, head); 288 threads, warp-specialised like gemm_tc.cu:
//   warp 8      TMA producer : Q once, then per 128-key block K (rank-3 map over the qkv matrix viewed as
//                              [token][3*heads][72]: the 64..127 half of the padded head_dim lies past extent 72 and is
//                              ZERO filled by TMA) and V^T (from the per-layer transposed copy, keys contiguous) into a
//                              2-stage ring
//   warps 0-7   two consumer warpgroups, 64 queries each: S = Q K^T (m64n128, K = 80: 5 wgmma from shared-memory
//                              descriptors) into registers; online softmax on the accumulator layout (a row lives in the
//                              four lanes of a quad: two shuffles per reduction); P as bf16 straight into the register
//                              A operand of PV = P V (m64n80, K = 128: 8 wgmma, B = V^T tile), accumulated on top of the
//                              rescaled fp32 output registers.
// Keys past the image's 729 (rows of the next image / zero padding of V^T) are masked to -inf before the softmax.
// The CROSS instantiation is the TikZero adapter's cross-attention (reference model/adapter/modeling_adapter.py:38-120): the
// queries come from a [B*N, heads*72] matrix, the keys of image b are the first klen[b] rows of its Tk caption rows of a
// [B*Tk, 2*heads*72] K | V matrix; keys at or past klen[b] are masked exactly like the padding keys above.
// All mbarrier waits are bounded (trap instead of hanging the GPU).
#include <cuda.h>

#include "common.cuh"
#include "launch.h"
#include "wgmma.cuh"

namespace dtk {
namespace {

constexpr int AQ = 128, AK = 128, DH = 72, DP = 80;       // queries / keys per block, head_dim, padded to the mma K step
constexpr int ATC_THREADS = 288;
constexpr int QB = AQ * 128;                                // one [128 rows x 64 cols] bf16 SWIZZLE_128B block = 16 KB
constexpr int VB = DP * 128;                                // one [80 rows x 64 keys] block = 10 KB
constexpr int KV_STAGE = 2 * QB + 2 * VB;                   // K (2 blocks) + V^T (2 blocks)
constexpr int ATC_SMEM = 2 * QB /*Q*/ + 2 * KV_STAGE + 1024 + 256;

struct AttnTcArgs {
  bf16* o;                   // [B*N, D] bf16, head h at columns h*72
  int64_t o_rs;              // row stride (elements)
  int B, heads, N;           // tokens per image
  float scale_log2;          // scale * log2(e)
  int kv_rows;               // CROSS: caption rows per image in the K map
  int klen[XATTN_MAX_B];     // CROSS: valid keys of image b
};

template <bool CROSS>
__global__ void __launch_bounds__(ATC_THREADS, 1) attn_tc_kernel(const __grid_constant__ CUtensorMap mapQ,
                                                                 const __grid_constant__ CUtensorMap mapK,
                                                                 const __grid_constant__ CUtensorMap mapVT, const AttnTcArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sQ = sbase, sKV = sQ + 2 * QB;
  const uint32_t bars = sKV + 2 * KV_STAGE;
  // barriers: q_full, kv_full[2], kv_empty[2]
  const uint32_t q_full = bars, kv_full0 = bars + 8, kv_empty0 = bars + 24;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int qt = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * AQ;
  const int nk = CROSS ? p.klen[b] : p.N;                   // keys of this image
  const int krow0 = CROSS ? b * p.kv_rows : b * p.N;        // its first key row in the K map
  const int khead = CROSS ? head : p.heads + head;          // K column block
  const int nblk = (nk + AK - 1) / AK;

  if (threadIdx.x == 0) {
    mbar_init(q_full, 1);
    for (int s = 0; s < 2; ++s) { mbar_init(kv_full0 + 8 * s, 1); mbar_init(kv_empty0 + 8 * s, 8); }   // empty: one arrive per consumer warp
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == 8) {
    // ===== TMA producer
    if (lane == 0) {
      const int row0 = b * p.N;
      mbar_expect_tx(q_full, 2 * QB);
      tma_load_3d(sQ, &mapQ, 0, head, row0 + q0, q_full);                  // d 0..63
      tma_load_3d(sQ + QB, &mapQ, 64, head, row0 + q0, q_full);            // d 64..127 (>= 72: zero fill)
      for (int j = 0; j < nblk; ++j) {
        const int s = j & 1, use = j >> 1;
        if (use > 0) mbar_wait(kv_empty0 + 8 * s, (use - 1) & 1);
        const uint32_t sk = sKV + s * KV_STAGE, sv = sk + 2 * QB;
        mbar_expect_tx(kv_full0 + 8 * s, KV_STAGE);
        tma_load_3d(sk, &mapK, 0, khead, krow0 + j * AK, kv_full0 + 8 * s);
        tma_load_3d(sk + QB, &mapK, 64, khead, krow0 + j * AK, kv_full0 + 8 * s);
        tma_load_2d(sv, &mapVT, j * AK, (b * p.heads + head) * DP, kv_full0 + 8 * s);
        tma_load_2d(sv + VB, &mapVT, j * AK + 64, (b * p.heads + head) * DP, kv_full0 + 8 * s);
      }
    }
    return;
  }
  // ===== consumer warpgroup wg: this thread holds query rows q0 + 64 wg + 16 (warp % 4) + g and + 8 (accumulator layout in wgmma.cuh)
  const int wg = warp >> 2, g = lane >> 2, c = lane & 3;
  const uint32_t sQw = sQ + wg * (64 * 128);
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f}, o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;
  mbar_wait(q_full, 0);
  for (int j = 0; j < nblk; ++j) {
    const int s = j & 1, use = j >> 1;
    mbar_wait(kv_full0 + 8 * s, use & 1);
    const uint32_t sk = sKV + s * KV_STAGE, sv = sk + 2 * QB;
    // S = Q K^T over head_dim 80 = 4 k-steps of block 0 + 1 k-step of block 1
    float sc[AK / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_m64n128k16_ss(sc, wgmma_desc(sQw + k * 32), wgmma_desc(sk + k * 32), k != 0);
    wgmma_m64n128k16_ss(sc, wgmma_desc(sQw + QB), wgmma_desc(sk + QB), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_fence(sc);
    const int kvalid = min(AK, nk - j * AK);            // keys of this block that belong to the image
    float alpha[2], m_new[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {   // h = 0: row g, h = 1: row g + 8
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < AK / 8; ++jj) {
        const int col = 8 * jj + 2 * c;
        if (col < kvalid) mx = fmaxf(mx, sc[4 * jj + 2 * h]);
        if (col + 1 < kvalid) mx = fmaxf(mx, sc[4 * jj + 2 * h + 1]);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      m_new[h] = fmaxf(m_run[h], mx * p.scale_log2);
      alpha[h] = exp2f(m_run[h] - m_new[h]);             // first block: exp2(-inf) = 0
      m_run[h] = m_new[h];
    }
    // p = exp2(s * scale - m) as bf16 in the A-fragment layout of the 8 k-steps (16 keys each) of PV
    uint32_t pa[AK / 16][4];
    float ps[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < AK / 8; ++jj) {
      const int col = 8 * jj + 2 * c;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float p0 = (col < kvalid) ? exp2f(sc[4 * jj + 2 * h] * p.scale_log2 - m_new[h]) : 0.f;
        const float p1 = (col + 1 < kvalid) ? exp2f(sc[4 * jj + 2 * h + 1] * p.scale_log2 - m_new[h]) : 0.f;
        // the denominator uses the bf16-rounded probabilities the tensor core multiplies with
        const __nv_bfloat162 pb = __floats2bfloat162_rn(p0, p1);
        ps[h] += __low2float(pb) + __high2float(pb);
        pa[jj >> 1][(jj & 1) * 2 + h] = *reinterpret_cast<const uint32_t*>(&pb);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + ps[h];   // per-thread partial of the row sum (reduced over the quad at the end)
#pragma unroll
    for (int i = 0; i < DP / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    // O += P V over the 128 keys of the block (2 V^T blocks of 4 k-steps)
    wgmma_acc_fence(o);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k) wgmma_m64n80k16_rs(o, pa[k], wgmma_desc(sv + (k >> 2) * VB + (k & 3) * 32), 1);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_acc_fence(o);
    if (lane == 0) mbar_arrive(kv_empty0 + 8 * s);          // K / V^T stage free once this warp's MMAs have read it
  }
  // normalise + store the 72 bf16 of the two rows
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const int q = q0 + wg * 64 + (warp & 3) * 16 + g + 8 * h;
    if (q < p.N) {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      bf16* dst = p.o + (int64_t)(b * p.N + q) * p.o_rs + head * DH;
#pragma unroll
      for (int jj = 0; jj < DH / 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj + 2 * c) = pack_bf16x2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
    }
  }
}

// V^T copy of one layer: qkv [B*N, 3*D] (v at column 2*D + h*72 + d) -> vT [(b*heads + h)*80 + d, NP] with keys contiguous,
// zero for d >= 72 and keys >= N. 32 x 32 shared-memory transpose tiles; grid (NP / 32, 3 (d tiles of 32: 96 >= 80), B*heads).
__global__ void __launch_bounds__(256) transpose_v_kernel(const bf16* __restrict__ qkv, int B, int heads, int N, int D, int NP,
                                                          bf16* __restrict__ vT) {
  __shared__ bf16 tile[32][33];
  const int bh = blockIdx.z, b = bh / heads, h = bh % heads;
  const int k0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;   // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int key = k0 + i, d = d0 + tx;
    bf16 v = __float2bfloat16_rn(0.f);
    if (key < N && d < DH) v = qkv[(int64_t)(b * N + key) * (3 * D) + 2 * D + h * DH + d];
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int d = d0 + i, key = k0 + tx;
    if (d < DP && key < NP) vT[((int64_t)bh * DP + d) * NP + key] = tile[tx][i];
  }
}

// V^T copy of the caption values: kv [B*Tk, 2*D] (v at column D + h*72 + d) -> vT [(b*heads + h)*80 + d, NP], zero for d >= 72
// and for keys >= klen[b] (padded caption rows never reach the PV product). Same tiling as transpose_v_kernel.
__global__ void __launch_bounds__(256) transpose_xv_kernel(const bf16* __restrict__ kv, int heads, int Tk, int D, int NP,
                                                           const AttnTcArgs p, bf16* __restrict__ vT) {
  __shared__ bf16 tile[32][33];
  const int bh = blockIdx.z, b = bh / heads, h = bh % heads;
  const int k0 = blockIdx.x * 32, d0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int nk = p.klen[b];
  for (int i = ty; i < 32; i += 8) {
    const int key = k0 + i, d = d0 + tx;
    bf16 v = __float2bfloat16_rn(0.f);
    if (key < nk && d < DH) v = kv[(int64_t)(b * Tk + key) * (2 * D) + D + h * DH + d];
    tile[i][tx] = v;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int d = d0 + i, key = k0 + tx;
    if (d < DP && key < NP) vT[((int64_t)bh * DP + d) * NP + key] = tile[tx][i];
  }
}

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn a_encode_fn() {
  static EncodeFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = (EncodeFn)f;
  }
  return fn;
}

// rank-3 view [rows][cols / 72][72] of a bf16 matrix with row stride ld: box 64 (d) x 1 (head) x 128 (rows), 128-byte swizzle,
// zero fill past d = 72
bool map_heads(EncodeFn fn, CUtensorMap* map, const bf16* ptr, int64_t rows, int col_heads, int64_t ld) {
  cuuint64_t dims[3] = {(cuuint64_t)DH, (cuuint64_t)col_heads, (cuuint64_t)rows};
  cuuint64_t strides[2] = {(cuuint64_t)DH * 2, (cuuint64_t)ld * 2};
  cuuint32_t box[3] = {64, 1, (cuuint32_t)AQ};
  cuuint32_t estr[3] = {1, 1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// V^T [rows, NP]: box 64 keys x 80 rows
bool map_vt(EncodeFn fn, CUtensorMap* map, const bf16* vT, int64_t rows, int NP) {
  cuuint64_t dims[2] = {(cuuint64_t)NP, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)NP * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)DP};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)vT, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <bool CROSS>
cudaError_t set_smem_attr() {
  static bool attr_done[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    e = cudaFuncSetAttribute(attn_tc_kernel<CROSS>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATC_SMEM);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  return cudaSuccess;
}

}  // namespace

bool attn_tc_supported() { return a_encode_fn() != nullptr; }
int attn_tc_vt_cols(int N) { return (N + AK - 1) / AK * AK; }   // keys padded to whole blocks

// qkv bf16 [B*N, 3*D] with D = heads * 72; vT scratch bf16 [B*heads*80, attn_tc_vt_cols(N)]; o bf16 [B*N, D]
cudaError_t launch_attn_tc(const bf16* qkv, bf16* vT, bf16* o, int B, int heads, int N, float scale, cudaStream_t s, uint64_t* counter) {
  EncodeFn fn = a_encode_fn();
  if (!fn) return cudaErrorNotSupported;
  const int D = heads * DH, NP = attn_tc_vt_cols(N);
  CUtensorMap mapQK, mapVT;
  // qkv viewed as [token][3*heads][72]
  if (!map_heads(fn, &mapQK, qkv, (int64_t)B * N, 3 * heads, 3 * D) || !map_vt(fn, &mapVT, vT, (int64_t)B * heads * DP, NP))
    return cudaErrorInvalidValue;
  cudaError_t e = set_smem_attr<false>();
  if (e != cudaSuccess) return e;
  transpose_v_kernel<<<dim3(NP / 32, 3, B * heads), 256, 0, s>>>(qkv, B, heads, N, D, NP, vT);
  AttnTcArgs a{};
  a.o = o; a.o_rs = D; a.B = B; a.heads = heads; a.N = N; a.scale_log2 = scale * 1.4426950408889634f;
  attn_tc_kernel<false><<<dim3((N + AQ - 1) / AQ, heads, B), ATC_THREADS, ATC_SMEM, s>>>(mapQK, mapQK, mapVT, a);
  if (counter) *counter += 2;
  return cudaGetLastError();
}

cudaError_t launch_xattn_tc(const bf16* q, const bf16* kv, const int* klen_host, int Tk, bf16* vT, bf16* o, int B, int heads,
                            int N, float scale, cudaStream_t s, uint64_t* counter) {
  EncodeFn fn = a_encode_fn();
  if (!fn) return cudaErrorNotSupported;
  if (B <= 0 || B > XATTN_MAX_B || Tk <= 0 || N <= 0 || heads <= 0) return cudaErrorInvalidValue;
  AttnTcArgs a{};
  for (int b = 0; b < B; ++b) {
    if (klen_host[b] < 1 || klen_host[b] > Tk) return cudaErrorInvalidValue;
    a.klen[b] = klen_host[b];
  }
  const int D = heads * DH, NP = attn_tc_vt_cols(Tk);
  CUtensorMap mapQ, mapK, mapVT;
  if (!map_heads(fn, &mapQ, q, (int64_t)B * N, heads, D) || !map_heads(fn, &mapK, kv, (int64_t)B * Tk, 2 * heads, 2 * D) ||
      !map_vt(fn, &mapVT, vT, (int64_t)B * heads * DP, NP))
    return cudaErrorInvalidValue;
  cudaError_t e = set_smem_attr<true>();
  if (e != cudaSuccess) return e;
  a.o = o; a.o_rs = D; a.B = B; a.heads = heads; a.N = N; a.scale_log2 = scale * 1.4426950408889634f; a.kv_rows = Tk;
  transpose_xv_kernel<<<dim3(NP / 32, 3, B * heads), 256, 0, s>>>(kv, heads, Tk, D, NP, a, vT);
  attn_tc_kernel<true><<<dim3((N + AQ - 1) / AQ, heads, B), ATC_THREADS, ATC_SMEM, s>>>(mapQ, mapK, mapVT, a);
  if (counter) *counter += 2;
  return cudaGetLastError();
}

}  // namespace dtk
