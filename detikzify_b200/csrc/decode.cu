// Single-token decode kernels (HBM-bound): fused RMSNorm + GEMV with RoPE/KV-write, SiLU*mul and
// residual epilogues; split-K decode attention over the slot KV cache.
//
// Replaces, per decoded token and layer (HF modeling_llama.py:303-333 eager path, ~35-40 launches):
//   RMSNorm :53-67, q/k/v/o_proj GEMV-shaped GEMMs :238-249, RoPE :124-168, DynamicCache.update
//   (torch.cat per step, cache_utils.py:119-120), 1xT SDPA :199-222, SwiGLU MLP :176-184.
#include "common.cuh"
#include "launch.h"

namespace dtk {
namespace {

constexpr int GEMV_THREADS = 256;
constexpr int GEMV_UNROLL = 4;

// block-wide sum for 256 threads
DTK_DEV float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < GEMV_THREADS / 32; ++i) t += red[i];
  __syncthreads();
  return t;
}

// One warp computes TWO output rows (r0, r1) per work item so that RoPE pairs (i, i+HD/2) and SwiGLU
// pairs (gate_i, up_i: interleaved rows 2i, 2i+1) are finished inside one warp. Weights stream with
// 128-bit no-allocate loads (8 in flight per lane); x lives in shared memory as fp32, split into
// lo/hi float4 planes so that LDS.128 is conflict-free. HD (head_dim) matters in GEMV_QKV mode only.
template <int MODE, int HD = 128>
__global__ void __launch_bounds__(GEMV_THREADS) gemv_kernel(const GemvArgs p) {
  extern __shared__ __align__(16) float xs[];  // [2][K/8] float4 planes
  __shared__ float red[GEMV_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.y;
  const int K = p.K, KC = K >> 3;
  float4* xlo = reinterpret_cast<float4*>(xs);
  float4* xhi = xlo + KC;
  const float* x = p.x + (int64_t)b * p.x_stride;

  float ss = 0.f;
  for (int c = tid; c < KC; c += GEMV_THREADS) {
    float4 a = *reinterpret_cast<const float4*>(x + c * 8);
    float4 d = *reinterpret_cast<const float4*>(x + c * 8 + 4);
    ss += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w + d.x * d.x + d.y * d.y + d.z * d.z + d.w * d.w;
    xlo[c] = a;
    xhi[c] = d;
  }
  if (p.norm_w) {
    const float r = rsqrtf(block_sum_256(ss, red) / K + p.eps);
    for (int c = tid; c < KC; c += GEMV_THREADS) {
      float w[8];
      unpack8(*reinterpret_cast<const uint4*>(p.norm_w + c * 8), w);
      float4 a = xlo[c], d = xhi[c];
      xlo[c] = make_float4(a.x * r * w[0], a.y * r * w[1], a.z * r * w[2], a.w * r * w[3]);
      xhi[c] = make_float4(d.x * r * w[4], d.y * r * w[5], d.z * r * w[6], d.w * r * w[7]);
    }
  }
  __syncthreads();

  const int n_items = p.N >> 1;
  for (int item = blockIdx.x * (GEMV_THREADS / 32) + warp; item < n_items; item += gridDim.x * (GEMV_THREADS / 32)) {
    int r0, r1;
    constexpr int HSH = HD == 128 ? 7 : 6;   // log2(HD): signed division by shifts (item, r0 >= 0)
    if (MODE == GEMV_QKV) { r0 = (item >> (HSH - 1)) * HD + (item & (HD / 2 - 1)); r1 = r0 + HD / 2; }
    else { r0 = item * 2; r1 = r0 + 1; }
    const uint4* w0 = reinterpret_cast<const uint4*>(p.W + (int64_t)r0 * K);
    const uint4* w1 = reinterpret_cast<const uint4*>(p.W + (int64_t)r1 * K);
    float a0 = 0.f, a1 = 0.f;
    for (int c0 = lane; c0 < KC; c0 += 32 * GEMV_UNROLL) {
      uint4 v0[GEMV_UNROLL], v1[GEMV_UNROLL];
#pragma unroll
      for (int u = 0; u < GEMV_UNROLL; ++u) {
        int c = c0 + u * 32;
        if (c < KC) { v0[u] = ldg_stream(w0 + c); v1[u] = ldg_stream(w1 + c); }
        else { v0[u] = make_uint4(0, 0, 0, 0); v1[u] = make_uint4(0, 0, 0, 0); }
      }
#pragma unroll
      for (int u = 0; u < GEMV_UNROLL; ++u) {
        int c = c0 + u * 32;
        if (c < KC) {
          float4 xl = xlo[c], xh = xhi[c];
          float f0[8], f1[8];
          unpack8(v0[u], f0);
          unpack8(v1[u], f1);
          a0 += f0[0] * xl.x + f0[1] * xl.y + f0[2] * xl.z + f0[3] * xl.w + f0[4] * xh.x + f0[5] * xh.y + f0[6] * xh.z + f0[7] * xh.w;
          a1 += f1[0] * xl.x + f1[1] * xl.y + f1[2] * xl.z + f1[3] * xl.w + f1[4] * xh.x + f1[5] * xh.y + f1[6] * xh.z + f1[7] * xh.w;
        }
      }
    }
    a0 = warp_sum(a0);
    a1 = warp_sum(a1);
    if (lane == 0) {
      if (MODE == GEMV_STORE) {
        float* o = p.out + (int64_t)b * p.out_stride;
        o[r0] = a0; o[r1] = a1;
      } else if (MODE == GEMV_ADD) {
        float* o = p.out + (int64_t)b * p.out_stride;
        o[r0] += a0; o[r1] += a1;
      } else if (MODE == GEMV_GLU) {
        p.out[(int64_t)b * p.out_stride + item] = silu(a0) * a1;
      } else {  // GEMV_QKV: rotate-half RoPE on q/k, write k/v straight into the slot cache (not for a retired row)
        const int pos = p.pos[b], slot = p.slots[b];
        const int i = r0 & (HD - 1);  // < HD / 2
        if (r0 >= p.q_dim && p.active && !p.active[b]) {
        } else if (r0 < p.q_dim + p.kv_dim) {
          const float2 cs = *reinterpret_cast<const float2*>(p.rope_cs + ((int64_t)pos * (HD / 2) + i) * 2);
          const float y0 = a0 * cs.x - a1 * cs.y, y1 = a1 * cs.x + a0 * cs.y;
          if (r0 < p.q_dim) {
            float* o = p.out + (int64_t)b * p.out_stride;
            o[r0] = y0; o[r1] = y1;
          } else {
            const int kh = (r0 - p.q_dim) >> HSH;
            bf16* d = p.kv_base + (int64_t)slot * p.kv_slot_stride + ((int64_t)kh * p.max_len + pos) * HD;
            d[i] = __float2bfloat16_rn(y0);
            d[i + HD / 2] = __float2bfloat16_rn(y1);
          }
        } else {
          const int kh = (r0 - p.q_dim - p.kv_dim) >> HSH;
          bf16* d = p.kv_base + (int64_t)slot * p.kv_slot_stride + p.kv_v_offset + ((int64_t)kh * p.max_len + pos) * HD;
          d[i] = __float2bfloat16_rn(a0);
          d[i + HD / 2] = __float2bfloat16_rn(a1);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(128) embed_tokens_kernel(const int* __restrict__ tok32,
                                                           const int64_t* __restrict__ tok64,
                                                           const bf16* __restrict__ embed, int H, int vocab,
                                                           float* __restrict__ x) {
  const int b = blockIdx.x;
  int64_t id = tok32 ? (int64_t)tok32[b] : tok64[b];
  if (id < 0 || id >= vocab) id = 0;
  for (int i = threadIdx.x * 8; i < H; i += 128 * 8) {
    float f[8];
    unpack8(*reinterpret_cast<const uint4*>(embed + id * H + i), f);
    *reinterpret_cast<float4*>(x + (int64_t)b * H + i) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(x + (int64_t)b * H + i + 4) = make_float4(f[4], f[5], f[6], f[7]);
  }
}

// ---- split-K single-query attention. grid (heads, nsplit, B), 128 threads. A group of HD/8 lanes owns one
//      key at a time: HD/8 lanes x 16 B = one K (or V) row per load instruction, fully coalesced (a half-warp
//      at head_dim 128, a quarter-warp at 64); 4 keys in flight per group. Partials (m, l, o[HD]) are merged by
//      the last CTA of each (sequence, head) — no second launch.
constexpr int DA_THREADS = 128, DA_UNROLL = 4;

template <int HD>
__global__ void __launch_bounds__(DA_THREADS) decode_attn_kernel(const DecodeAttnArgs p) {
  constexpr int LPK = HD / 8;                 // lanes per key
  constexpr int NGRP = DA_THREADS / LPK;      // key groups per CTA
  __shared__ float sm_m[NGRP], sm_l[NGRP];
  __shared__ float sm_o[NGRP][HD];
  __shared__ int sm_last;
  const int head = blockIdx.x, split = blockIdx.y, b = blockIdx.z;
  const int tid = threadIdx.x, hw = tid / LPK, l16 = tid & (LPK - 1);
  const int T = p.pos[b] + 1, slot = p.slots[b];
  const int kvh = head / p.kv_group;
  // a retired row of a generation loop reads no keys (its slot may already belong to another sequence); its CTAs still
  // take part in the counters protocol and its output is zero
  const bool live = !p.active || p.active[b];
  int chunk = (T - p.key_begin + p.nsplit - 1) / p.nsplit;   // key_begin > 0: the shared prefix was reduced by the prefix kernel
  chunk = (chunk + 7) & ~7;
  const int j0 = p.key_begin + split * chunk, j1 = live ? min(T, j0 + chunk) : j0;
  const bf16* kb = p.kv_base + (int64_t)slot * p.kv_slot_stride + (int64_t)kvh * p.max_len * HD;
  const bf16* vb = kb + p.kv_v_offset;
  // shared prefix: positions below shlen live in another slot (one copy for all rollouts of a figure)
  const int shlen = p.share_len ? p.share_len[b] : 0;
  const bf16* kb2 = shlen > 0 ? p.kv_base + (int64_t)p.share_slot[b] * p.kv_slot_stride + (int64_t)kvh * p.max_len * HD : kb;
  const bf16* vb2 = kb2 + p.kv_v_offset;
  const float sl2 = p.scale * 1.4426950408889634f;

  float q[8];
  {
    const float* qp = p.q + (int64_t)b * p.q_stride + head * HD + l16 * 8;
    float4 a = *reinterpret_cast<const float4*>(qp), d = *reinterpret_cast<const float4*>(qp + 4);
    q[0] = a.x * sl2; q[1] = a.y * sl2; q[2] = a.z * sl2; q[3] = a.w * sl2;
    q[4] = d.x * sl2; q[5] = d.y * sl2; q[6] = d.z * sl2; q[7] = d.w * sl2;
  }
  float m = -INFINITY, l = 0.f, o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;

  for (int jb = j0; jb < j1; jb += NGRP * DA_UNROLL) {
    uint4 kr[DA_UNROLL], vr[DA_UNROLL];
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      int j = jb + u * NGRP + hw;
      if (j < j1) {
        kr[u] = *reinterpret_cast<const uint4*>((j < shlen ? kb2 : kb) + (int64_t)j * HD + l16 * 8);
        vr[u] = *reinterpret_cast<const uint4*>((j < shlen ? vb2 : vb) + (int64_t)j * HD + l16 * 8);
      } else {
        kr[u] = make_uint4(0, 0, 0, 0);
        vr[u] = make_uint4(0, 0, 0, 0);
      }
    }
#pragma unroll
    for (int u = 0; u < DA_UNROLL; ++u) {
      int j = jb + u * NGRP + hw;
      float kf[8];
      unpack8(kr[u], kf);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += q[i] * kf[i];
#pragma unroll
      for (int st = LPK / 2; st > 0; st >>= 1) s += __shfl_xor_sync(0xffffffffu, s, st);
      if (j < j1) {  // uniform within the key group
        float mn = fmaxf(m, s);
        float alpha = exp2f(m - mn), pj = exp2f(s - mn);
        float vf[8];
        unpack8(vr[u], vf);
        l = l * alpha + pj;
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = o[i] * alpha + pj * vf[i];
        m = mn;
      }
    }
  }
  // ---- merge the NGRP key-group states of this CTA
  if (l16 == 0) { sm_m[hw] = m; sm_l[hw] = l; }
#pragma unroll
  for (int i = 0; i < 8; ++i) sm_o[hw][l16 * 8 + i] = o[i];
  __syncthreads();
  if (HD == DA_THREADS || tid < HD) {
    const int d = tid;
    float M = -INFINITY;
#pragma unroll
    for (int h = 0; h < NGRP; ++h) M = fmaxf(M, sm_m[h]);
    float L = 0.f, O = 0.f;
#pragma unroll
    for (int h = 0; h < NGRP; ++h) {
      float w = (sm_m[h] == -INFINITY) ? 0.f : exp2f(sm_m[h] - M);
      L += sm_l[h] * w;
      O += sm_o[h][d] * w;
    }
    const int64_t pi = ((int64_t)(b * p.heads + head) * p.np + split);
    p.part_o[pi * HD + d] = O;
    if (d == 0) { p.part_ml[pi * 2] = M; p.part_ml[pi * 2 + 1] = L; }
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    unsigned prev = atomicAdd(&p.counters[b * p.heads + head], 1u);
    sm_last = (prev == (unsigned)p.nsplit - 1u);
  }
  __syncthreads();
  if (sm_last && (HD == DA_THREADS || tid < HD)) {
    __threadfence();
    const int d = tid;
    const int64_t base = (int64_t)(b * p.heads + head) * p.np;
    float M = -INFINITY;
    for (int s = 0; s < p.np; ++s) M = fmaxf(M, __ldcg(p.part_ml + (base + s) * 2));
    float L = 0.f, O = 0.f;
    for (int s = 0; s < p.np; ++s) {
      float ms = __ldcg(p.part_ml + (base + s) * 2);
      float w = (ms == -INFINITY) ? 0.f : exp2f(ms - M);
      L += __ldcg(p.part_ml + (base + s) * 2 + 1) * w;
      O += __ldcg(p.part_o + (base + s) * HD + d) * w;
    }
    const float res = live ? O / L : 0.f;
    p.out[(int64_t)b * p.out_stride + head * HD + d] = res;
    if (p.out_bf16) p.out_bf16[(int64_t)b * p.out_stride + head * HD + d] = __float2bfloat16_rn(res);
    if (tid == 0) p.counters[b * p.heads + head] = 0u;
  }
}

}  // namespace

cudaError_t launch_gemv(const GemvArgs& a, cudaStream_t s, uint64_t* counter) {
  if ((a.K & 7) || (a.N & 1) || a.B <= 0) return cudaErrorInvalidValue;
  if (a.mode == GEMV_QKV && ((a.head_dim != 64 && a.head_dim != 128) || ((a.q_dim | a.kv_dim) % a.head_dim))) return cudaErrorInvalidValue;
  const int smem = a.K * (int)sizeof(float);
  const int items = a.N / 2;
  int gx = (items + 7) / 8;
  if (gx > 264) gx = 264;  // 2 CTAs per SM x 132 SMs; warps loop over the remaining items
  dim3 grid(gx, a.B);
  cudaError_t e = cudaSuccess;
#define DTK_GEMV_CASE(M, ...)                                                                                   \
  {                                                                                                             \
    if (smem > 48 * 1024) e = cudaFuncSetAttribute(gemv_kernel<M, ##__VA_ARGS__>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem); \
    if (e != cudaSuccess) return e;                                                                             \
    gemv_kernel<M, ##__VA_ARGS__><<<grid, GEMV_THREADS, smem, s>>>(a);                                          \
  }
  switch (a.mode) {
    case GEMV_STORE: DTK_GEMV_CASE(GEMV_STORE) break;
    case GEMV_ADD: DTK_GEMV_CASE(GEMV_ADD) break;
    case GEMV_GLU: DTK_GEMV_CASE(GEMV_GLU) break;
    case GEMV_QKV:
      if (a.head_dim == 128) DTK_GEMV_CASE(GEMV_QKV, 128) else DTK_GEMV_CASE(GEMV_QKV, 64)
      break;
    default: return cudaErrorInvalidValue;
  }
#undef DTK_GEMV_CASE
  if (counter) ++*counter;
  return cudaGetLastError();
}

cudaError_t launch_embed_tokens(const int* tok32, const int64_t* tok64, int B, const bf16* embed, int H, int vocab,
                                float* x, cudaStream_t s, uint64_t* counter) {
  embed_tokens_kernel<<<B, 128, 0, s>>>(tok32, tok64, embed, H, vocab, x);
  if (counter) ++*counter;
  return cudaGetLastError();
}

cudaError_t launch_decode_attn(const DecodeAttnArgs& a0, cudaStream_t s, uint64_t* counter) {
  DecodeAttnArgs a = a0;
  if (a.np < a.nsplit) a.np = a.nsplit;   // plain mode: np left at 0
  dim3 grid(a.heads, a.nsplit, a.B);
  if (a.head_dim == 128) decode_attn_kernel<128><<<grid, DA_THREADS, 0, s>>>(a);
  else if (a.head_dim == 64) decode_attn_kernel<64><<<grid, DA_THREADS, 0, s>>>(a);
  else return cudaErrorInvalidValue;
  if (counter) ++*counter;
  return cudaGetLastError();
}

}  // namespace dtk
