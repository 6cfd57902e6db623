// wgmma GEMM  C[M,N] = A[M,K] * W[N,K]^T  (bf16 operands, fp32 accumulate in registers) — the Hopper tensor path for the
// dense contractions of the ViT (qkv / out / fc1+GELU / fc2, patch embed) and the LLaMA prefill (qkv, o, gate/up with
// SiLU*mul, down), with the same fused epilogues as gemm_mma.cu (bias, GELU, position rows, residual, GLU).
//
// Dense kernel (M >= 64): 128 x BN output tiles, 384 threads, warp-specialised:
//   warp 8      TMA producer : cp.async.bulk.tensor.2d (SWIZZLE_128B boxes of 128 / BN rows x 64 k) for A and W into a
//                              4-stage shared-memory ring, mbarrier complete_tx; runs ahead across tile boundaries
//   warps 0-7   two consumer warpgroups: warpgroup g owns rows 64 g .. 64 g + 63 of the tile and issues
//                              wgmma.mma_async m64nBNk16 from shared-memory descriptors into BN / 2 accumulator registers
//                              per thread; one k-block stays in flight while the previous ring slot is released;
//                              epilogue math in registers, stored straight from the accumulator layout
// setmaxnreg moves registers from the producer warpgroup to the consumers (the 64 x 256 accumulator alone is 128 registers).
// Out-of-range rows / the K tail are zero-filled by TMA. All mbarrier waits are bounded (trap instead of hanging the GPU).
#include <cuda.h>

#include "common.cuh"
#include "fp8.cuh"
#include "launch.h"
#include "wgmma.cuh"

namespace dtk {
namespace {

constexpr int TBM = 128, TBK = 64;
constexpr int A_BYTES = TBM * TBK * 2;                                // 16 KB
constexpr int DSTAGES = 4;
constexpr int DTHREADS = 384;                                         // two consumer warpgroups + the producer's warpgroup

template <int BN>
struct DenseCfg {
  static constexpr int STAGE_BYTES = A_BYTES + BN * TBK * 2;
  static constexpr int SMEM = DSTAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
};
static_assert(DenseCfg<256>::SMEM <= 232448, "dense GEMM shared memory");

DTK_DEV void wgmma_tile(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n128k16_ss(d, a, b, acc); }
DTK_DEV void wgmma_tile(float (&d)[128], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n256k16_ss(d, a, b, acc); }
DTK_DEV void wgmma_tile(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n32k16_ss(d, a, b, acc); }
DTK_DEV void wgmma_tile(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) { wgmma_m64n64k16_ss(d, a, b, acc); }
DTK_DEV void wgmma_tile_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t acc) { wgmma_m64n32k16_rs(d, a, b, acc); }
DTK_DEV void wgmma_tile_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t acc) { wgmma_m64n64k16_rs(d, a, b, acc); }

// 0.5 x (1 + tanh(u)) = x * sigmoid(2u): two MUFU ops instead of the libm tanhf (error ~1e-7 relative, far below bf16 output rounding)
DTK_DEV float gelu_tanh_fast(float x) {
  const float u = 0.7978845608028654f * (x + 0.044715f * x * x * x);
  return __fdividef(x, 1.f + __expf(-2.f * u));
}

// epilogue of the two adjacent columns (n, n + 1) of row m
DTK_DEV void dense_store(const GemmArgs& p, int m, int n, float v0, float v1) {
  if (p.bias) {
    const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.bias + n));
    v0 += b.x; v1 += b.y;
  }
  if (p.act == ACT_GELU_TANH) { v0 = gelu_tanh_fast(v0); v1 = gelu_tanh_fast(v1); }
  else if (p.act == ACT_GELU_ERF) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
  if (p.glu) {
    const float rr = silu(v0) * v1;
    const int64_t o = (int64_t)m * p.ldo + (n >> 1);
    if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(rr);
    else p.out_f32[o] = rr;
    return;
  }
  if (p.gate) {
    const float gs = 1.f / (1.f + expf(-__bfloat162float(*p.gate)));
    v0 *= gs; v1 *= gs;
  }
  if (p.rowbias) {
    const float2 b = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(p.rowbias + (int64_t)(m % p.rowbias_mod) * p.N + n));
    v0 += b.x; v1 += b.y;
  }
  if (p.resid) {
    const float2 rs = *reinterpret_cast<const float2*>(p.resid + (int64_t)m * p.ldr + n);
    v0 += rs.x; v1 += rs.y;
  }
  const int64_t o = (int64_t)m * p.ldo + n;
  if (p.out_bf16) *reinterpret_cast<uint32_t*>(p.out_bf16 + o) = pack_bf16x2(v0, v1);
  else *reinterpret_cast<float2*>(p.out_f32 + o) = make_float2(v0, v1);
}

// log-softmax epilogue of the lm_head (LSE instantiation, BN = 256): this thread holds rows r0 (i = 0) and r0 + 8 (i = 1)
// at columns n0 + 8 j + 2 c + {0, 1}. Per row: {max, sum exp} over the valid columns (n < N; the TMA zero fill past V
// stays out), reduced in the thread, then over the quad's 4 lanes by shuffle; lane c = 0 writes the tile's partial.
template <int BN>
DTK_DEV void lse_epilogue(const GemmLseArgs& p, const float (&acc)[BN / 2], int r0, int n0, int c) {
  const int NT = (p.N + BN - 1) / BN, tj = n0 / BN;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = r0 + 8 * i;
    float mx = -INFINITY, sum = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      if (n0 + 8 * j + 2 * c < p.N) mx = fmaxf(mx, fmaxf(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]));
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      if (n0 + 8 * j + 2 * c < p.N) sum += __expf(acc[4 * j + 2 * i] - mx) + __expf(acc[4 * j + 2 * i + 1] - mx);
#pragma unroll
    for (int o = 1; o < 4; o <<= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o), os = __shfl_xor_sync(0xffffffffu, sum, o);
      lse_combine(mx, sum, om, os);
    }
    if (m >= p.M) continue;
    if (c == 0) p.part[(int64_t)m * NT + tj] = make_float2(mx, sum);
    const int64_t t = p.targets[m] - n0;
    if (t >= 0 && t < BN && n0 + t < p.N && ((t & 7) >> 1) == c) {   // the target column is one of this thread's
      const int jt = (int)(t >> 3);
      float v = 0.f;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
        if (j == jt) v = (t & 1) ? acc[4 * j + 2 * i + 1] : acc[4 * j + 2 * i];
      p.tgt[m] = v;
    }
    if (p.out_f32) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * c;
        if (n < p.N) *reinterpret_cast<float2*>(p.out_f32 + (int64_t)m * p.ldo + n) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      }
    }
  }
}

template <bool LSE> struct DenseArgs { using type = GemmArgs; };
template <> struct DenseArgs<true> { using type = GemmLseArgs; };

// CTAs walk the output tiles (m fastest: concurrent CTAs share a BN-row band of W) with stride gridDim.x.
// LSE = true: the lm_head's log-softmax epilogue instead of the generic one.
template <int BN, bool LSE = false>
__global__ void __launch_bounds__(DTHREADS, 1) gemm_tc_kernel(const __grid_constant__ CUtensorMap mapA,
                                                              const __grid_constant__ CUtensorMap mapB,
                                                              const typename DenseArgs<LSE>::type p) {
  constexpr int STAGE_BYTES = DenseCfg<BN>::STAGE_BYTES;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;      // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t full0 = sbase + DSTAGES * STAGE_BYTES, empty0 = full0 + 8 * DSTAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int KT = (p.K + TBK - 1) / TBK;
  const int MT = (p.M + TBM - 1) / TBM, NT = (p.N + BN - 1) / BN;
  const int tiles = MT * NT;

  if (threadIdx.x == 0) {
    for (int s = 0; s < DSTAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }   // empty: one arrive per consumer warp
    mbar_init_fence();
  }
  __syncthreads();

  if (warp >= 8) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n");
    if (warp == 8 && lane == 0) {
      uint32_t it = 0;   // k-blocks issued so far (ring position across tiles)
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int m0 = (tile % MT) * TBM, n0 = (tile / MT) * BN;
        for (int kt = 0; kt < KT; ++kt, ++it) {
          const uint32_t s = it % DSTAGES, use = it / DSTAGES;
          if (use > 0) mbar_wait(empty0 + 8 * s, (use - 1) & 1);
          const uint32_t sa = sbase + s * STAGE_BYTES, sb = sa + A_BYTES;
          mbar_expect_tx(full0 + 8 * s, STAGE_BYTES);
          tma_load_2d(sa, &mapA, kt * TBK, m0, full0 + 8 * s);
          tma_load_2d(sb, &mapB, kt * TBK, n0, full0 + 8 * s);
        }
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n");
  const int wg = warp >> 2;
  const int g = lane >> 2, c = lane & 3;
  uint32_t it = 0;
  for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int m0 = (tile % MT) * TBM, n0 = (tile / MT) * BN;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    for (int kt = 0; kt < KT; ++kt, ++it) {
      const uint32_t s = it % DSTAGES, use = it / DSTAGES;
      mbar_wait(full0 + 8 * s, use & 1);
      const uint32_t sa = sbase + s * STAGE_BYTES + wg * (64 * 128), sb = sbase + s * STAGE_BYTES + A_BYTES;
      wgmma_acc_fence(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TBK / 16; ++k) wgmma_tile(acc, wgmma_desc(sa + k * 32), wgmma_desc(sb + k * 32), (kt | k) != 0);
      wgmma_commit();
      if (kt > 0) {   // the previous k-block has been read: its ring slot goes back to the producer
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty0 + 8 * ((it - 1) % DSTAGES));
      }
    }
    wgmma_wait<0>();
    wgmma_acc_fence(acc);
    if (lane == 0) mbar_arrive(empty0 + 8 * ((it - 1) % DSTAGES));

    const int r0 = m0 + wg * 64 + (warp & 3) * 16 + g;
    if constexpr (LSE) {
      lse_epilogue<BN>(p, acc, r0, n0, c);
    } else {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int n = n0 + 8 * j + 2 * c;
        if (n >= p.N) break;   // N is even: the pair (n, n + 1) is inside or outside together
        if (r0 < p.M) dense_store(p, r0, n, acc[4 * j], acc[4 * j + 1]);
        if (r0 + 8 < p.M) dense_store(p, r0 + 8, n, acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
  }
}

// ---- thread-block cluster helpers (split-K reduce of the batched-decode tile)
DTK_DEV uint32_t cluster_ctarank() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r)); return r; }
DTK_DEV void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
DTK_DEV uint32_t dsmem_addr(uint32_t local_addr, uint32_t rank) {   // same offset in the shared memory of CTA `rank`
  uint32_t ra;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(ra) : "r"(local_addr), "r"(rank));
  return ra;
}
DTK_DEV float ld_dsmem(uint32_t cluster_addr) {
  float v;
  asm volatile("ld.shared::cluster.f32 %0, [%1];\n" : "=f"(v) : "r"(cluster_addr) : "memory");
  return v;
}

// ---- swapped-operand tile for the batched decode step (M = rollouts < 64): out[b, n] = sum_k X[b, k] W[n, k].
// The weight rows are the wgmma M dimension (128 rows of W per CTA, K-major, straight from the arena; warpgroup g takes rows
// 64 g .. 64 g + 63) and the few batch rows are the N dimension (NB = 32 or 64 columns): per 64-wide k-block a CTA moves
// 16 KB of weights (bytes that must come from HBM once per step anyway) and only NB x 128 B of activations (L2 resident).
// The accumulator comes out transposed (row = output feature n, column = batch row b).
// Epilogue: bias, residual, SwiGLU (gate_i / up_i are adjacent ROWS of W = lanes 4 apart: one shuffle), fp32 or bf16 out.
//
// Split-K over a thread-block cluster: a decode GEMM has only N / 128 weight tiles (32 for a 4096-wide projection), far fewer
// than 2 x 132 CTA slots, and a CTA's bytes in flight are bounded by its ring. `nsplit` CTAs of one cluster share a tile, each
// streams a contiguous K range into its own accumulator, ranks > 0 park their fp32 partial tile in their shared memory
// and rank 0 adds them IN RANK ORDER through distributed shared memory (deterministic) and runs the epilogue. No workspace in
// HBM, no atomics. Two CTAs per SM (5-stage rings) keep ~200 KB of weights in flight per SM.
//
// F8 = true: the weights are FP8 decode tiles (GemmF8; mapW unused). The CTA's 128 rows are the 8 row groups
// 8 (blockIdx / nsplit) .. + 7, warp q's 16 accumulator rows = group q in the tiles' row permutation (tile_row). A 64-wide
// k-block kb of one group is 1 KB of contiguous codes ([kstep pair 2][lane 32][16 B] at byte (kb % 4) KB of 256-k tile
// kb / 4): the producer bulk-copies one per group that exists, each lane loads its 2 x 16 B, rebuilds the bf16 bits of
// code x 2^k_r for rows g and g + 8 (fp8.cuh) and issues the wgmma with A from registers. Same k-blocks, split-K cuts,
// k16 order and rank-order reduction as the bf16 tile, so a matrix holding exactly those values gives the same bits.
// A stage carries half the weight bytes, so the ring is deeper (TSTAGES as deep as two CTAs per SM allow).
constexpr int STHREADS = 288;   // two consumer warpgroups + the producer warp
template <int NB, int TSTAGES, bool F8 = false>
__global__ void __launch_bounds__(STHREADS, 2) gemm_tc_swap_kernel(const __grid_constant__ CUtensorMap mapW,
                                                                  const __grid_constant__ CUtensorMap mapX, const GemmArgs p,
                                                                  const int nsplit, const GemmF8 f8) {
  constexpr int W_BYTES = F8 ? TBM * TBK : A_BYTES;   // e4m3 codes or bf16 weights of one k-block
  constexpr int X_BYTES = NB * TBK * 2;
  constexpr int STAGE_BYTES = W_BYTES + X_BYTES;
  constexpr int NACC = NB / 2;
  static_assert(NACC * 256 * 4 <= TSTAGES * STAGE_BYTES, "the partial tile is parked in the drained ring");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full0 = sbase + TSTAGES * STAGE_BYTES, empty0 = full0 + 8 * TSTAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = nsplit > 1 ? cluster_ctarank() : 0u;
  const int n0 = (blockIdx.x / nsplit) * TBM;
  const int KTall = (p.K + TBK - 1) / TBK;
  const int kt0 = (int)((int64_t)KTall * rank / nsplit), KT = (int)((int64_t)KTall * (rank + 1) / nsplit) - kt0;   // this CTA's k-blocks

  if (threadIdx.x == 0) {
    for (int s = 0; s < TSTAGES; ++s) { mbar_init(full0 + 8 * s, 1); mbar_init(empty0 + 8 * s, 8); }
    mbar_init_fence();
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      if constexpr (F8) {
        const int g0 = n0 / 16, ng = min(8, f8.groups - g0);   // groups past the matrix's last are neither copied nor stored
        const int64_t gstride = (int64_t)f8.tpg * MEGA_F8_TILE_BYTES;
        const uint8_t* src0 = f8.tiles + g0 * gstride;
        for (int kt = 0; kt < KT; ++kt) {
          const int s = kt % TSTAGES, use = kt / TSTAGES, kb = kt0 + kt;
          if (use > 0) mbar_wait(empty0 + 8 * s, (use - 1) & 1);
          const uint32_t sw = sbase + s * STAGE_BYTES, sx = sw + W_BYTES;
          mbar_expect_tx(full0 + 8 * s, ng * 1024 + X_BYTES);
          const uint8_t* src = src0 + (int64_t)(kb >> 2) * MEGA_F8_TILE_BYTES + (kb & 3) * 1024;
          for (int q = 0; q < ng; ++q) bulk_load(sw + q * 1024, src + q * gstride, 1024, full0 + 8 * s);
          tma_load_2d(sx, &mapX, kb * TBK, 0, full0 + 8 * s);
        }
      } else {
        for (int kt = 0; kt < KT; ++kt) {
          const int s = kt % TSTAGES, use = kt / TSTAGES;
          if (use > 0) mbar_wait(empty0 + 8 * s, (use - 1) & 1);
          const uint32_t sw = sbase + s * STAGE_BYTES, sx = sw + A_BYTES;
          mbar_expect_tx(full0 + 8 * s, STAGE_BYTES);
          tma_load_2d(sw, &mapW, (kt0 + kt) * TBK, n0, full0 + 8 * s);
          tma_load_2d(sx, &mapX, (kt0 + kt) * TBK, 0, full0 + 8 * s);
        }
      }
    }
  } else {
    const int wg = warp >> 2;
    const int g = lane >> 2, c = lane & 3;
    float acc[NACC];
#pragma unroll
    for (int i = 0; i < NACC; ++i) acc[i] = 0.f;
    float s0 = 0.f, s1 = 0.f;   // F8: row scales 2^k_r of this thread's rows g and g + 8
    if constexpr (F8) {
      const int gi = n0 / 16 + warp;
      if (gi < f8.groups) { s0 = pow2f(f8.exps[gi * 16 + g]); s1 = pow2f(f8.exps[gi * 16 + g + 8]); }
    }
    for (int kt = 0; kt < KT; ++kt) {
      const int s = kt % TSTAGES, use = kt / TSTAGES;
      mbar_wait(full0 + 8 * s, use & 1);
      if constexpr (F8) {
        const uint32_t sw = sbase + s * STAGE_BYTES + warp * 1024 + lane * 16, sx = sbase + s * STAGE_BYTES + W_BYTES;
        uint4 q[2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
          asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(q[h].x), "=r"(q[h].y), "=r"(q[h].z), "=r"(q[h].w) : "r"(sw + h * 512));
        // k-step 2 h + u: word 2 u = fragments 0 | 1 (rows g | g + 8, k 2c), word 2 u + 1 = fragments 2 | 3 (k 8 + 2c)
        // A operands are read asynchronously: the previous k-block's wgmma must be done with its registers before they are
        // rebuilt (the bf16 tile keeps one k-block in flight; here it overlaps only the wait and the shared loads)
        if (kt > 0) {
          wgmma_wait<0>();
          if (lane == 0) mbar_arrive(empty0 + 8 * ((kt - 1) % TSTAGES));
        }
        uint32_t a[4][4];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint32_t w[4] = {q[h].x, q[h].y, q[h].z, q[h].w};
#pragma unroll
          for (int u = 0; u < 2; ++u) {
            a[2 * h + u][0] = e4m3x2_to_bf16x2(w[2 * u], s0);
            a[2 * h + u][1] = e4m3x2_to_bf16x2(w[2 * u] >> 16, s1);
            a[2 * h + u][2] = e4m3x2_to_bf16x2(w[2 * u + 1], s0);
            a[2 * h + u][3] = e4m3x2_to_bf16x2(w[2 * u + 1] >> 16, s1);
          }
        }
        wgmma_acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TBK / 16; ++k) wgmma_tile_rs(acc, a[k], wgmma_desc(sx + k * 32), (kt | k) != 0);
      } else {
        const uint32_t sw = sbase + s * STAGE_BYTES + wg * (64 * 128), sx = sbase + s * STAGE_BYTES + A_BYTES;
        wgmma_acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TBK / 16; ++k) wgmma_tile(acc, wgmma_desc(sw + k * 32), wgmma_desc(sx + k * 32), (kt | k) != 0);
      }
      wgmma_commit();
      if (!F8 && kt > 0) {
        wgmma_wait<1>();
        if (lane == 0) mbar_arrive(empty0 + 8 * ((kt - 1) % TSTAGES));
      }
    }
    wgmma_wait<0>();
    wgmma_acc_fence(acc);
    // partial tiles of ranks > 0: register i of consumer thread t at word i * 256 + t of the drained ring (both warpgroups
    // have finished reading it: named barrier over the 256 consumer threads); rank 0's thread t reads the same words
    const uint32_t pword = sbase + threadIdx.x * 4;
    if (rank != 0) {
      asm volatile("bar.sync 1, 256;\n" ::: "memory");
#pragma unroll
      for (int i = 0; i < NACC; ++i) asm volatile("st.shared.f32 [%0], %1;\n" ::"r"(pword + i * 1024), "f"(acc[i]) : "memory");
    }
    if (nsplit > 1) cluster_sync_all();   // partials of every rank are visible to rank 0
    if (rank == 0) {
      // partial sums of the other ranks, K ranges in order
#pragma unroll 1
      for (uint32_t q = 1; q < (uint32_t)nsplit; ++q) {
        const uint32_t rword = dsmem_addr(pword, q);
        float t[NACC];
#pragma unroll
        for (int i = 0; i < NACC; ++i) t[i] = ld_dsmem(rword + i * 1024);
#pragma unroll
        for (int i = 0; i < NACC; ++i) acc[i] += t[i];
      }
      if constexpr (F8) {
        // rows g and g + 8 of group gi = output features tile_row(...): TILE_ROPE stores q / k / v in natural order, and in
        // TILE_GLU they are (gate_i, up_i) of i = 8 gi + g, both in this thread (no shuffle)
        const int gi = n0 / 16 + warp;
        if (gi < f8.groups) {
          const int nr[2] = {tile_row(f8.mode, f8.hd, gi, g), tile_row(f8.mode, f8.hd, gi, g + 8)};
#pragma unroll
          for (int i = 0; i < NACC; ++i)
            if (p.bias && nr[(i >> 1) & 1] < p.N) acc[i] += __bfloat162float(p.bias[nr[(i >> 1) & 1]]);
#pragma unroll
          for (int i = 0; i < NACC; ++i) {
            const int j = i >> 2, n = nr[(i >> 1) & 1], b = 8 * j + 2 * c + (i & 1);
            float v = acc[i];
            if (p.glu) {
              if (!(i & 2) && n < p.N && b < p.M) {
                const float rr = silu(v) * acc[i | 2];
                const int64_t o = (int64_t)b * p.ldo + gi * 8 + g;
                if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(rr);
                else p.out_f32[o] = rr;
              }
              continue;
            }
            if (n < p.N && b < p.M) {
              if (p.gate) v *= 1.f / (1.f + expf(-__bfloat162float(*p.gate)));
              if (p.resid) v += p.resid[(int64_t)b * p.ldr + n];
              const int64_t o = (int64_t)b * p.ldo + n;
              if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(v);
              else p.out_f32[o] = v;
            }
          }
        }
      } else {
        // rows = output features n (g and g + 8 of this warp's 16), columns = batch rows b
        const int nA = n0 + wg * 64 + (warp & 3) * 16 + g;
#pragma unroll
        for (int i = 0; i < NACC; ++i) {
          const int j = i >> 2, n = nA + ((i & 2) ? 8 : 0), b = 8 * j + 2 * c + (i & 1);
          float v = acc[i];
          if (p.bias && n < p.N) v += __bfloat162float(p.bias[n]);
          if (p.glu) {
            const float other = __shfl_xor_sync(0xffffffffu, v, 4);   // rows (gate, up) = lanes g, g + 1
            if (!(g & 1) && n < p.N && b < p.M) {
              const float rr = silu(v) * other;
              const int64_t o = (int64_t)b * p.ldo + (n >> 1);
              if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(rr);
              else p.out_f32[o] = rr;
            }
            continue;
          }
          if (n < p.N && b < p.M) {
            if (p.gate) v *= 1.f / (1.f + expf(-__bfloat162float(*p.gate)));
            if (p.resid) v += p.resid[(int64_t)b * p.ldr + n];
            const int64_t o = (int64_t)b * p.ldo + n;
            if (p.out_bf16) p.out_bf16[o] = __float2bfloat16_rn(v);
            else p.out_f32[o] = v;
          }
        }
      }
    }
  }
  if (warp == 8 && nsplit > 1) cluster_sync_all();   // the producer warp takes part in both cluster barriers
  if (nsplit > 1) cluster_sync_all();   // rank 0 has read every partial: the other CTAs' shared memory may go away
}

// ---- tensor maps (driver entry point resolved at run time: no link-time dependency on libcuda)
typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeFn encode_fn() {
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

// 2-D bf16 row-major [rows, cols] (row stride ld elements), box 64 cols x box_rows rows, 128-byte swizzle, zero OOB fill
bool make_map(CUtensorMap* map, const bf16* ptr, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  EncodeFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {(cuuint32_t)TBK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

bool gemm_tc_supported(const GemmArgs& a) {
  if (a.a_rows_per_batch > 0) return false;                       // batched A addressing: mma.sync path
  if ((a.K & 7) || (a.N & 1) || (a.lda & 7) || (a.ldw & 7)) return false;
  if (((uintptr_t)a.A & 15) || ((uintptr_t)a.W & 15)) return false;
  // the dense epilogue stores column pairs (float2 / packed bf16x2) and reads the residual as float2
  if (!a.glu && ((a.ldo & 1) || ((uintptr_t)a.out_f32 & 7) || ((uintptr_t)a.out_bf16 & 3))) return false;
  if (a.resid && ((a.ldr & 1) || ((uintptr_t)a.resid & 7))) return false;
  return encode_fn() != nullptr;
}

// persistent = one CTA per SM walks the tiles; otherwise one CTA per tile
template <int BN, bool LSE = false>
static cudaError_t launch_tc_dense(const typename DenseArgs<LSE>::type& a, bool persistent, cudaStream_t s, uint64_t* counter) {
  CUtensorMap mapA, mapB;
  if (!make_map(&mapA, a.A, a.M, a.K, a.lda, TBM) || !make_map(&mapB, a.W, a.N, a.K, a.ldw, BN)) return cudaErrorInvalidValue;
  constexpr int smem = DenseCfg<BN>::SMEM;
  // the attribute is per device; set once per device (not per launch: launches may be captured into a CUDA graph)
  static bool attr_done[64] = {};
  static int sms[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  if (!attr_done[dev]) {
    e = cudaFuncSetAttribute(gemm_tc_kernel<BN, LSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    e = cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) return e;
    attr_done[dev] = true;
  }
  const int tiles = ((a.M + TBM - 1) / TBM) * ((a.N + BN - 1) / BN);
  gemm_tc_kernel<BN, LSE><<<persistent && tiles > sms[dev] ? sms[dev] : tiles, DTHREADS, smem, s>>>(mapA, mapB, a);
  if (counter) ++*counter;
  return cudaGetLastError();
}

static int g_swap_split = 0;   // dev switch (dtk_set_option "gemm_swap_split"): 0 = heuristic, 1..8 = forced split-K factor
void set_gemm_swap_split(int v) { g_swap_split = v; }

// F8: the weights come from w (mapW is not used); the same grid and split-K factor as the bf16 tile of the same N and K
template <int NB, int TSTAGES, bool F8 = false>
static cudaError_t launch_tc_swap(const GemmArgs& a, cudaStream_t s, uint64_t* counter, const GemmF8& w = GemmF8{}) {
  CUtensorMap mapW{}, mapX;
  if ((!F8 && !make_map(&mapW, a.W, a.N, a.K, a.ldw, TBM)) || !make_map(&mapX, a.A, a.M, a.K, a.lda, NB)) return cudaErrorInvalidValue;
  constexpr int smem = TSTAGES * ((F8 ? TBM * TBK : A_BYTES) + NB * TBK * 2) + 1024 + 256;
  static bool attr_done[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= 64 || !attr_done[dev]) {
    e = cudaFuncSetAttribute(gemm_tc_swap_kernel<NB, TSTAGES, F8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    if (dev >= 0 && dev < 64) attr_done[dev] = true;
  }
  // split-K factor: GEMMs with about one weight tile per SM or more are not split (splitting them only adds the
  // reduction). Projections with few tiles (N = 4096: 32) get the smallest factor that reaches ~100 CTAs, at least 8
  // k-blocks per rank.
  const int tiles = (a.N + TBM - 1) / TBM, KT = (a.K + TBK - 1) / TBK;
  int nsplit = 1;
  if (g_swap_split == 0) {
    while (nsplit < 8 && tiles * nsplit < 100 && KT / (nsplit + 1) >= 8) ++nsplit;
  } else {
    nsplit = g_swap_split;
    while (nsplit > 1 && KT / nsplit < 1) --nsplit;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(tiles * nsplit));
  cfg.blockDim = dim3(STHREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)nsplit;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  e = cudaLaunchKernelEx(&cfg, gemm_tc_swap_kernel<NB, TSTAGES, F8>, mapW, mapX, a, nsplit, w);
  if (counter) ++*counter;
  return e;
}

cudaError_t launch_gemm_tc(const GemmArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaSuccess;
  if (a.M < 64 && a.act == ACT_NONE && !a.rowbias) {   // batched decode: weights are the M side
    return a.M <= 32 ? launch_tc_swap<32, 5>(a, s, counter) : launch_tc_swap<64, 4>(a, s, counter);
  }
  // M < 64 with an activation or row bias (pool-head fc1 at M = images per batch) also lands here: the swapped tile has
  // no such epilogue, so these few small products run on a 128-row tile that is mostly TMA zero fill
  if (get_gemm_impl() == 2) return launch_tc_dense<256>(a, true, s, counter);   // persistent 128 x 256
  return launch_tc_dense<128>(a, false, s, counter);
}

cudaError_t launch_gemm_swap_f8(const GemmArgs& a, const GemmF8& w, cudaStream_t s, uint64_t* counter) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaSuccess;
  if (a.M >= 64 || a.act != ACT_NONE || a.rowbias || !w.tiles || !w.exps || (a.glu != 0) != (w.mode == TILE_GLU) ||
      (int64_t)w.groups * 16 < a.N || (int64_t)w.tpg * 256 < a.K || !gemm_tc_supported(a))
    return cudaErrorInvalidValue;
  if (w.mode == TILE_ROPE && ((w.hd != 64 && w.hd != 128) || a.N % w.hd)) return cudaErrorInvalidValue;
  // 9 / 6 stages: the deepest rings of 8 KB weight blocks that still fit two CTAs per SM
  return a.M <= 32 ? launch_tc_swap<32, 9, true>(a, s, counter, w) : launch_tc_swap<64, 6, true>(a, s, counter, w);
}

cudaError_t launch_gemm_lse(const GemmLseArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.M <= 0 || a.N <= 0 || a.K <= 0) return cudaSuccess;
  if (!a.targets || !a.part || !a.tgt || a.bias || a.rowbias || a.resid || a.act != ACT_NONE || a.glu || a.gate || a.out_bf16 ||
      (a.out_f32 && a.ldo != a.N) || !gemm_tc_supported(a))
    return cudaErrorInvalidValue;
  // every M runs on the dense tile (a small M is mostly TMA zero fill): the swapped and mma.sync tiles have no such epilogue
  return launch_tc_dense<LSE_TILE, true>(a, true, s, counter);
}

}  // namespace dtk
