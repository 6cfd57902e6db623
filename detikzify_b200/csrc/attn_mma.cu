// Flash attention (online softmax, fp32 statistics) on mma.sync tiles.
//   * ViT self-attention: 16 heads x head_dim 72 (zero-padded to 80 in shared memory for the
//     QK^T contraction), N = 729 keys, non-causal  — HF modeling_siglip.py:229-249,293-306.
//   * LLaMA prefill: head_dim 128 or 64 (TinyLlama), causal over cached positions — HF modeling_llama.py:199-222;
//     non-causal partials of the shared prefix of a batched decode step.
//   * TikZero caption encoder (Llama-3.2-1B): head_dim 64, causal.
// One CTA = 64 queries of one (batch, head); 4 warps x 16 query rows; K/V streamed in 64-key tiles
// through a 2-stage cp.async ring. P is re-used straight from the score accumulators as the
// A-operand of the PV product.
#include "common.cuh"
#include "launch.h"

namespace dtk {
namespace {

constexpr int BQ = 64, BKV = 64, ATHREADS = 128;

template <int D, int DP>
struct AttnSmem {
  static constexpr int DPS = DP + 8;  // row stride (elements): (DPS*2) % 128 == 16 (mod 32) -> conflict-free ldmatrix
  static constexpr int TILE = BQ * DPS * 2;  // bytes
  static constexpr int BYTES = 5 * TILE;     // Q + 2 x (K, V)
};

// rows below split_row come from base2 (shared KV prefix held by another slot), the others from base
template <int D, int DP>
DTK_DEV void load_rows(uint32_t sdst, const bf16* base, int64_t row_stride, int row0, int nrows_valid, int tid,
                       const bf16* base2 = nullptr, int split_row = 0) {
  constexpr int DPS = AttnSmem<D, DP>::DPS;
  constexpr int CH = D / 8;
  for (int c = tid; c < BQ * CH; c += ATHREADS) {
    int r = c / CH, kc = c - r * CH;
    bool ok = (row0 + r) < nrows_valid;
    const bf16* rb = (row0 + r) < split_row ? base2 : base;
    const bf16* src = ok ? rb + (int64_t)(row0 + r) * row_stride + kc * 8 : base;
    cp_async16(sdst + (uint32_t)(r * DPS + kc * 8) * 2, src, ok ? 16 : 0);
  }
}

template <int D, int DP, bool CAUSAL, bool PARTIAL>
__global__ void __launch_bounds__(ATHREADS) flash_attn_kernel(const AttnArgs p) {
  using S = AttnSmem<D, DP>;
  constexpr int DPS = S::DPS;
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sQ = smem_u32(smem);
  const uint32_t sK0 = sQ + S::TILE, sV0 = sK0 + 2 * S::TILE;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // PARTIAL: one query tile (Tq <= 64 rows = the rollouts of a batched decode step), blockIdx.x = key-tile range
  const int qt = PARTIAL ? 0 : blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int kvh = head / p.kv_group;
  const bf16* qb = p.q + (int64_t)b * p.q_bs + (int64_t)head * p.q_hs;
  const bf16* kb = p.k + (int64_t)b * p.k_bs + (int64_t)kvh * p.k_hs;
  const bf16* vb = p.v + (int64_t)b * p.v_bs + (int64_t)kvh * p.v_hs;
  const bf16* kb2 = p.split_row > 0 ? p.k2 + (int64_t)b * p.k_bs + (int64_t)kvh * p.k_hs : kb;
  const bf16* vb2 = p.split_row > 0 ? p.v2 + (int64_t)b * p.v_bs + (int64_t)kvh * p.v_hs : vb;
  const int q0 = qt * BQ;

  // zero the padding columns [D, DP) of Q and K tiles once (cp.async never touches them)
  if (DP > D) {
    for (int r = tid; r < BQ; r += ATHREADS) {
      *reinterpret_cast<uint4*>(smem + (size_t)(r * DPS + D) * 2) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(smem + S::TILE + (size_t)(r * DPS + D) * 2) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(smem + 2 * S::TILE + (size_t)(r * DPS + D) * 2) = make_uint4(0, 0, 0, 0);
    }
  }

  int tk = p.Tk;
  if (CAUSAL) {
    int last = p.q_pos0 + min(q0 + BQ, p.Tq);  // one past the last visible key for this query tile
    tk = min(tk, last);
  }
  const int jt0 = PARTIAL ? (int)blockIdx.x * p.part_tiles : 0;
  const int ntiles = PARTIAL ? min((tk + BKV - 1) / BKV, jt0 + p.part_tiles) : (tk + BKV - 1) / BKV;

  load_rows<D, DP>(sQ, qb, p.q_rs, q0, p.Tq, tid);
  load_rows<D, DP>(sK0 + (jt0 & 1) * S::TILE, kb, p.k_rs, jt0 * BKV, tk, tid, kb2, p.split_row);
  load_rows<D, DP>(sV0 + (jt0 & 1) * S::TILE, vb, p.v_rs, jt0 * BKV, tk, tid, vb2, p.split_row);
  cp_async_commit();

  float o[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[i][e] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  uint32_t qf[DP / 16][4];
  const float sl2 = p.scale * 1.4426950408889634f;
  const int g = lane >> 2, tq4 = lane & 3;

  for (int j = jt0; j < ntiles; ++j) {
    const int st = j & 1;
    if (j + 1 < ntiles) {
      load_rows<D, DP>(sK0 + (st ^ 1) * S::TILE, kb, p.k_rs, (j + 1) * BKV, tk, tid, kb2, p.split_row);
      load_rows<D, DP>(sV0 + (st ^ 1) * S::TILE, vb, p.v_rs, (j + 1) * BKV, tk, tid, vb2, p.split_row);
    }
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (j == jt0) {
#pragma unroll
      for (int kk = 0; kk < DP / 16; ++kk) {
        int row = warp * 16 + (lane & 15);
        int col = kk * 16 + ((lane >> 4) << 3);
        ldmatrix_x4(qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], sQ + (uint32_t)(row * DPS + col) * 2);
      }
    }
    const uint32_t sK = sK0 + st * S::TILE, sV = sV0 + st * S::TILE;

    float sc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) sc[i][e] = 0.f;
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
#pragma unroll
      for (int nj = 0; nj < 4; ++nj) {
        int row = nj * 16 + ((lane >> 4) << 3) + (lane & 7);
        int col = kk * 16 + (((lane >> 3) & 1) << 3);
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(b0, b1, b2, b3, sK + (uint32_t)(row * DPS + col) * 2);
        mma_bf16_16816(sc[2 * nj], qf[kk], b0, b1);
        mma_bf16_16816(sc[2 * nj + 1], qf[kk], b2, b3);
      }
    }

    // ---- mask + online softmax (rows g and g+8 of this warp's 16-row slab)
    const int qrow0 = q0 + warp * 16 + g;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        int key = j * BKV + ni * 8 + tq4 * 2 + (e & 1);
        int qrow = qrow0 + ((e >> 1) << 3);
        bool ok = key < p.Tk && (!CAUSAL || key <= p.q_pos0 + qrow);
        float v = ok ? sc[ni][e] : -INFINITY;
        sc[ni][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    }
    float alpha[2], muse[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      float mn = fmaxf(m_run[h], mx[h]);
      muse[h] = (mn == -INFINITY) ? 0.f : mn;
      alpha[h] = exp2f((m_run[h] - muse[h]) * sl2);
      m_run[h] = mn;
      l_run[h] *= alpha[h];
    }
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float pv = exp2f((sc[ni][e] - muse[e >> 1]) * sl2);
        sc[ni][e] = pv;
        l_run[e >> 1] += pv;
      }
    }
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o[i][0] *= alpha[0]; o[i][1] *= alpha[0];
      o[i][2] *= alpha[1]; o[i][3] *= alpha[1];
    }

    // ---- O += P * V
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_bf16x2(sc[2 * kk][0], sc[2 * kk][1]);
      a[1] = pack_bf16x2(sc[2 * kk][2], sc[2 * kk][3]);
      a[2] = pack_bf16x2(sc[2 * kk + 1][0], sc[2 * kk + 1][1]);
      a[3] = pack_bf16x2(sc[2 * kk + 1][2], sc[2 * kk + 1][3]);
      const int krow = kk * 16 + (((lane >> 3) & 1) << 3) + (lane & 7);
#pragma unroll
      for (int nd = 0; nd < (D / 8) / 2; ++nd) {
        int col = (nd * 2 + (lane >> 4)) * 8;
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4_trans(b0, b1, b2, b3, sV + (uint32_t)(krow * DPS + col) * 2);
        mma_bf16_16816(o[2 * nd], a, b0, b1);
        mma_bf16_16816(o[2 * nd + 1], a, b2, b3);
      }
      if ((D / 8) & 1) {
        int col = (D / 8 - 1) * 8;
        int r = kk * 16 + (lane & 15);
        uint32_t b0, b1;
        ldmatrix_x2_trans(b0, b1, sV + (uint32_t)(r * DPS + col) * 2);
        mma_bf16_16816(o[D / 8 - 1], a, b0, b1);
      }
    }
    __syncthreads();
  }
  cp_async_wait<0>();

  // ---- normalise + store
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
    l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
  }
  if (PARTIAL) {
    // flash state of this key range, in the convention of decode_attn_kernel's partials (merged there)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int qrow = warp * 16 + g + h * 8;
      if (qrow >= p.Tq) continue;
      const int64_t pi = ((int64_t)qrow * p.heads + head) * p.part_np + p.part_idx0 + blockIdx.x;
      if (tq4 == 0) {
        p.part_ml[pi * 2] = m_run[h] == -INFINITY ? -INFINITY : m_run[h] * sl2;
        p.part_ml[pi * 2 + 1] = l_run[h];
      }
#pragma unroll
      for (int i = 0; i < D / 8; ++i)
        *reinterpret_cast<float2*>(p.part_o + pi * D + i * 8 + tq4 * 2) = make_float2(o[i][h * 2], o[i][h * 2 + 1]);
    }
    return;
  }
  bf16* ob = p.o + (int64_t)b * p.o_bs + (int64_t)head * p.o_hs;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    int qrow = q0 + warp * 16 + g + h * 8;
    if (qrow >= p.Tq) continue;
    float inv = l_run[h] > 0.f ? 1.f / l_run[h] : 0.f;
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      int col = i * 8 + tq4 * 2;
      *reinterpret_cast<uint32_t*>(ob + (int64_t)qrow * p.o_rs + col) =
          pack_bf16x2(o[i][h * 2] * inv, o[i][h * 2 + 1] * inv);
    }
  }
}

template <int D, int DP, bool CAUSAL, bool PARTIAL>
cudaError_t launch_t(const AttnArgs& a, cudaStream_t s) {
  const int smem = AttnSmem<D, DP>::BYTES;
  // the attribute is per device; set once per device (not per launch: launches may be captured into a CUDA graph)
  static bool attr_done[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    e = cudaFuncSetAttribute(flash_attn_kernel<D, DP, CAUSAL, PARTIAL>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  dim3 grid(PARTIAL ? (((a.Tk + BKV - 1) / BKV + a.part_tiles - 1) / a.part_tiles) : (a.Tq + BQ - 1) / BQ, a.heads, a.B);
  flash_attn_kernel<D, DP, CAUSAL, PARTIAL><<<grid, ATHREADS, smem, s>>>(a);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_flash_attn(const AttnArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.Tq <= 0 || a.B <= 0) return cudaSuccess;
  if (a.part_o) {   // shared-prefix partials of a batched decode step
    if ((a.head_dim != 128 && a.head_dim != 64) || a.causal || a.Tq > BQ || a.B != 1 || a.part_tiles <= 0 || a.Tk <= 0 || !a.part_ml)
      return cudaErrorInvalidValue;
    if (counter) ++*counter;
    return a.head_dim == 128 ? launch_t<128, 128, false, true>(a, s) : launch_t<64, 64, false, true>(a, s);
  }
  if (counter) ++*counter;
  if (a.head_dim == 72) return a.causal ? launch_t<72, 80, true, false>(a, s) : launch_t<72, 80, false, false>(a, s);
  if (a.head_dim == 128) return a.causal ? launch_t<128, 128, true, false>(a, s) : launch_t<128, 128, false, false>(a, s);
  if (a.head_dim == 64 && a.causal) return launch_t<64, 64, true, false>(a, s);   // caption encoder, head_dim-64 decoders (prefill)
  return cudaErrorInvalidValue;
}

}  // namespace dtk
