// Dense GEMM  C[M,N] = A[M,K] * W[N,K]^T  (bf16 operands, fp32 accumulate) with fused epilogues.
//
// Bring-up / small-M tensor path: mma.sync m16n8k16 fed by a 4-stage cp.async ring, 128x128x32
// tiles, XOR-swizzled shared memory read with ldmatrix. It serves every dense contraction of the
// path (ViT patch-embed / qkv / out / fc1 / fc2, projector, LLaMA prefill qkv / o / gate-up / down)
// so the whole engine is correct end to end; the wgmma/TMA kernel in gemm_tc.cu takes over the
// large-M shapes (see DESIGN.md "GEMM").
//
// Replaces (reference has no native code; these are the library calls it dispatches to):
//   nn.Linear in HF SiglipEncoderLayer / SiglipMLP (modeling_siglip.py:269-327),
//   mm_projector (detikzify/model/v1/modeling_detikzify.py:163),
//   LlamaAttention / LlamaMLP projections (modeling_llama.py:176-184,238-249).
#include "common.cuh"
#include "launch.h"

namespace dtk {

namespace {

constexpr int BM = 128, BN = 128, BK = 32, STAGES = 4, THREADS = 256;
constexpr int TILE_BYTES = BM * BK * 2;  // 8 KB per operand per stage

// 64-byte rows (4 x 16 B chunks); chunk index XOR-swizzled with (row >> 1) & 3 so that the 8 rows
// of one ldmatrix 8x8 tile hit 8 distinct 16-byte bank groups.
DTK_DEV uint32_t swz(int row, int chunk) { return (uint32_t)(row * 64 + ((chunk ^ ((row >> 1) & 3)) << 4)); }

DTK_DEV const bf16* a_row_ptr(const GemmArgs& p, int m) {
  if (p.a_rows_per_batch > 0) {
    int b = m / p.a_rows_per_batch, r = m - b * p.a_rows_per_batch;
    return p.A + (int64_t)b * p.a_batch_stride + (int64_t)r * p.lda;
  }
  return p.A + (int64_t)m * p.lda;
}

DTK_DEV void load_tiles(const GemmArgs& p, uint32_t sA, uint32_t sB, int m0, int n0, int k0, int tid) {
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int c = tid + i * THREADS;  // 0..511
    int row = c >> 2, kc = c & 3;
    int k = k0 + kc * 8;
    {
      int m = m0 + row;
      bool ok = (m < p.M) && (k < p.K);
      const bf16* src = ok ? a_row_ptr(p, m) + k : p.A;
      cp_async16(sA + swz(row, kc), src, ok ? 16 : 0);
    }
    {
      int n = n0 + row;
      bool ok = (n < p.N) && (k < p.K);
      const bf16* src = ok ? p.W + (int64_t)n * p.ldw + k : p.W;
      cp_async16(sB + swz(row, kc), src, ok ? 16 : 0);
    }
  }
}

__global__ void __launch_bounds__(THREADS) gemm_bf16_tn_kernel(const GemmArgs p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps, warp tile 64 x 32
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int KT = (p.K + BK - 1) / BK;

  float acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KT) load_tiles(p, sbase + s * 2 * TILE_BYTES, sbase + s * 2 * TILE_BYTES + TILE_BYTES, m0, n0, s * BK, tid);
    cp_async_commit();
  }

  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nk = kt + STAGES - 1;
      if (nk < KT) {
        int s = nk % STAGES;
        load_tiles(p, sbase + s * 2 * TILE_BYTES, sbase + s * 2 * TILE_BYTES + TILE_BYTES, m0, n0, nk * BK, tid);
      }
      cp_async_commit();
    }
    const uint32_t sA = sbase + (kt % STAGES) * 2 * TILE_BYTES;
    const uint32_t sB = sA + TILE_BYTES;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      uint32_t af[4][4];
#pragma unroll
      for (int mi = 0; mi < 4; ++mi) {
        int row = wm * 64 + mi * 16 + (lane & 15);
        int kc = ks * 2 + (lane >> 4);
        ldmatrix_x4(af[mi][0], af[mi][1], af[mi][2], af[mi][3], sA + swz(row, kc));
      }
      uint32_t bfr[4][2];
#pragma unroll
      for (int nj = 0; nj < 2; ++nj) {
        int row = wn * 32 + nj * 16 + ((lane >> 4) << 3) + (lane & 7);
        int kc = ks * 2 + ((lane >> 3) & 1);
        ldmatrix_x4(bfr[2 * nj][0], bfr[2 * nj][1], bfr[2 * nj + 1][0], bfr[2 * nj + 1][1], sB + swz(row, kc));
      }
#pragma unroll
      for (int mi = 0; mi < 4; ++mi)
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) mma_bf16_16816(acc[mi][ni], af[mi], bfr[ni][0], bfr[ni][1]);
    }
  }
  cp_async_wait<0>();

  // ---- epilogue
  const int g = lane >> 2, tq = lane & 3;
#pragma unroll
  for (int mi = 0; mi < 4; ++mi) {
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int m = m0 + wm * 64 + mi * 16 + g + half * 8;
      if (m >= p.M) continue;
#pragma unroll
      for (int ni = 0; ni < 4; ++ni) {
        const int n = n0 + wn * 32 + ni * 8 + tq * 2;
        if (n >= p.N) continue;
        float v0 = acc[mi][ni][half * 2 + 0], v1 = acc[mi][ni][half * 2 + 1];
        if (p.bias) {
          float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.bias + n));
          v0 += b.x; v1 += b.y;
        }
        if (p.act == ACT_GELU_TANH) { v0 = gelu_tanh(v0); v1 = gelu_tanh(v1); }
        else if (p.act == ACT_GELU_ERF) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
        if (p.glu) {
          float r = silu(v0) * v1;
          int64_t o = (int64_t)m * p.ldo + (n >> 1);
          if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(r);
          else p.out_f32[o] = r;
          continue;
        }
        if (p.gate) {
          const float gs = 1.f / (1.f + expf(-__bfloat162float(*p.gate)));
          v0 *= gs; v1 *= gs;
        }
        if (p.rowbias) {
          float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.rowbias + (int64_t)(m % p.rowbias_mod) * p.N + n));
          v0 += b.x; v1 += b.y;
        }
        if (p.resid) {
          float2 r = *reinterpret_cast<const float2*>(p.resid + (int64_t)m * p.ldr + n);
          v0 += r.x; v1 += r.y;
        }
        int64_t o = (int64_t)m * p.ldo + n;
        if (p.out_bf16) *reinterpret_cast<uint32_t*>(p.out_bf16 + o) = pack_bf16x2(v0, v1);
        else *reinterpret_cast<float2*>(p.out_f32 + o) = make_float2(v0, v1);
      }
    }
  }
}

}  // namespace

static int g_gemm_impl = 2;  // 0 = mma.sync everywhere, 1 = wgmma one-tile-per-CTA 128 x 128 kernel, 2 (default) = persistent 128 x 256 wgmma kernel (dtk_set_option "gemm_impl")
void set_gemm_impl(int impl) { g_gemm_impl = impl; }
int get_gemm_impl() { return g_gemm_impl; }

cudaError_t launch_gemm(const GemmArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.gate && a.glu) return cudaErrorInvalidValue;   // the GLU epilogue has no gate
  // large-M dense contractions go to the wgmma kernel; tiny M (pool head, M = B) stays on mma.sync
  // (M < 4: pool-head probes and other tiny products stay on mma.sync; 4 <= M < 64 takes the swapped-operand wgmma tile)
  if (g_gemm_impl >= 1 && a.M >= 4 && gemm_tc_supported(a)) return launch_gemm_tc(a, s, counter);
  return launch_gemm_mma(a, s, counter);
}

cudaError_t launch_gemm_mma(const GemmArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaSuccess;
  if ((a.K & 7) || (a.N & 1) || (a.lda & 7) || (a.ldw & 7)) return cudaErrorInvalidValue;
  static bool attr_done[64] = {};            // per device
  const int smem = STAGES * 2 * TILE_BYTES;  // 64 KB
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    e = cudaFuncSetAttribute(gemm_bf16_tn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  dim3 grid((a.N + BN - 1) / BN, (a.M + BM - 1) / BM);
  gemm_bf16_tn_kernel<<<grid, THREADS, smem, s>>>(a);
  if (counter) ++*counter;
  return cudaGetLastError();
}

}  // namespace dtk
