// Row-wise and elementwise kernels of the prefill / ViT paths (all HBM-bound, 128-bit accesses).
#include "common.cuh"
#include "launch.h"

namespace dtk {
namespace {

// ---- LayerNorm (HF modeling_siglip.py:333-362 nn.LayerNorm, eps 1e-6): warp per row, fp32 stats,
//      two-pass variance (row stays L1-resident).
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const bf16* __restrict__ w,
                                                        const bf16* __restrict__ b, float eps, int M, int D,
                                                        bf16* __restrict__ out_bf16, float* __restrict__ out_f32) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (int64_t)row * D;
  float s = 0.f;
  for (int i = lane * 4; i < D; i += 128) {
    float4 v = *reinterpret_cast<const float4*>(xr + i);
    s += v.x + v.y + v.z + v.w;
  }
  const float mean = warp_sum(s) / D;
  float q = 0.f;
  for (int i = lane * 4; i < D; i += 128) {
    float4 v = *reinterpret_cast<const float4*>(xr + i);
    float a = v.x - mean, bb = v.y - mean, c = v.z - mean, d = v.w - mean;
    q += a * a + bb * bb + c * c + d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) / D + eps);
  for (int i = lane * 4; i < D; i += 128) {
    float4 v = *reinterpret_cast<const float4*>(xr + i);
    float2 w0 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i));
    float2 w1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i + 2));
    float2 b0 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i));
    float2 b1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i + 2));
    float y0 = (v.x - mean) * rstd * w0.x + b0.x, y1 = (v.y - mean) * rstd * w0.y + b0.y;
    float y2 = (v.z - mean) * rstd * w1.x + b1.x, y3 = (v.w - mean) * rstd * w1.y + b1.y;
    if (out_bf16) {
      uint2 pk = make_uint2(pack_bf16x2(y0, y1), pack_bf16x2(y2, y3));
      *reinterpret_cast<uint2*>(out_bf16 + (int64_t)row * D + i) = pk;
    }
    if (out_f32) *reinterpret_cast<float4*>(out_f32 + (int64_t)row * D + i) = make_float4(y0, y1, y2, y3);
  }
}

// Same LayerNorm with the row held in registers (D <= 128 * R): one warp per row, all loads of the row in flight at once,
// one pass over memory instead of three dependent ones (the ViT rows are 1152 wide: R = 9).
template <int R>
__global__ void __launch_bounds__(256) layernorm_reg_kernel(const float* __restrict__ x, const bf16* __restrict__ w,
                                                            const bf16* __restrict__ b, float eps, int M, int D,
                                                            bf16* __restrict__ out_bf16, float* __restrict__ out_f32) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* xr = x + (int64_t)row * D;
  float4 v[R];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const int i = (j * 32 + lane) * 4;
    v[j] = i < D ? *reinterpret_cast<const float4*>(xr + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int j = 0; j < R; ++j) s += v[j].x + v[j].y + v[j].z + v[j].w;
  const float mean = warp_sum(s) / D;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    if ((j * 32 + lane) * 4 < D) {
      const float a = v[j].x - mean, bb = v[j].y - mean, c = v[j].z - mean, d = v[j].w - mean;
      q += a * a + bb * bb + c * c + d * d;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / D + eps);
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const int i = (j * 32 + lane) * 4;
    if (i >= D) continue;
    float2 w0 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i));
    float2 w1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i + 2));
    float2 b0 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i));
    float2 b1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i + 2));
    float y0 = (v[j].x - mean) * rstd * w0.x + b0.x, y1 = (v[j].y - mean) * rstd * w0.y + b0.y;
    float y2 = (v[j].z - mean) * rstd * w1.x + b1.x, y3 = (v[j].w - mean) * rstd * w1.y + b1.y;
    if (out_bf16) {
      uint2 pk = make_uint2(pack_bf16x2(y0, y1), pack_bf16x2(y2, y3));
      *reinterpret_cast<uint2*>(out_bf16 + (int64_t)row * D + i) = pk;
    }
    if (out_f32) *reinterpret_cast<float4*>(out_f32 + (int64_t)row * D + i) = make_float4(y0, y1, y2, y3);
  }
}

// ---- RMSNorm (HF modeling_llama.py:53-67): fp32 x * rsqrt(mean(x^2)+eps) * w
// One CTA per row: the row stays in registers between the two passes (D <= 4 * 8 * blockDim), every thread has all its
// loads in flight at once. (One warp per row means 64 dependent load rounds for a 4096-wide row.)
template <int THREADS>
__global__ void __launch_bounds__(THREADS) rmsnorm_kernel(const float* __restrict__ x, int64_t ldx,
                                                          const bf16* __restrict__ w, float eps, int M, int D,
                                                          bf16* __restrict__ out) {
  constexpr int R = 8;
  __shared__ float red[THREADS / 32];
  const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const float* xr = x + (int64_t)row * ldx;
  float4 v[R];
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const int i = (j * THREADS + tid) * 4;
    v[j] = i < D ? *reinterpret_cast<const float4*>(xr + i) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
#pragma unroll
  for (int j = 0; j < R; ++j) q += v[j].x * v[j].x + v[j].y * v[j].y + v[j].z * v[j].z + v[j].w * v[j].w;
  for (int i = (R * THREADS + tid) * 4; i < D; i += THREADS * 4) {   // D beyond the register-resident part (not hit by any preset)
    const float4 t = *reinterpret_cast<const float4*>(xr + i);
    q += t.x * t.x + t.y * t.y + t.z * t.z + t.w * t.w;
  }
  q = warp_sum(q);
  if (lane == 0) red[tid >> 5] = q;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int j = 0; j < THREADS / 32; ++j) tot += red[j];
  const float r = rsqrtf(tot / D + eps);
  auto emit = [&](const float4& t, int i) {
    float2 w0 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i));
    float2 w1 = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i + 2));
    uint2 pk = make_uint2(pack_bf16x2(t.x * r * w0.x, t.y * r * w0.y), pack_bf16x2(t.z * r * w1.x, t.w * r * w1.y));
    *reinterpret_cast<uint2*>(out + (int64_t)row * D + i) = pk;
  };
#pragma unroll
  for (int j = 0; j < R; ++j) {
    const int i = (j * THREADS + tid) * 4;
    if (i < D) emit(v[j], i);
  }
  for (int i = (R * THREADS + tid) * 4; i < D; i += THREADS * 4) emit(*reinterpret_cast<const float4*>(xr + i), i);
}

// ---- patch extraction for the 14x14/s14 conv-as-GEMM (HF modeling_siglip.py:124-130): one warp per
//      patch row; column order (c, py, px) == flattened conv weight [D, 3, P, P]; zero K-padding.
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ pix, int B, int S, int P, int KP,
                                                     bf16* __restrict__ out) {
  const int G = S / P, N = G * G;
  const int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= (int64_t)B * N) return;
  const int b = (int)(row / N), pi = (int)(row % N), gy = pi / G, gx = pi % G;
  const int Kreal = 3 * P * P;
  for (int k = lane; k < KP; k += 32) {
    float v = 0.f;
    if (k < Kreal) {
      int c = k / (P * P), r = k % (P * P), py = r / P, px = r % P;
      v = pix[(((int64_t)b * 3 + c) * S + gy * P + py) * S + gx * P + px];
    }
    out[row * KP + k] = __float2bfloat16_rn(v);
  }
}

__global__ void __launch_bounds__(256) cast_kernel(const float* __restrict__ in, bf16* __restrict__ out, int64_t n) {
  int64_t i = ((int64_t)blockIdx.x * 256 + threadIdx.x) * 4;
  if (i + 3 < n) {
    float4 v = *reinterpret_cast<const float4*>(in + i);
    *reinterpret_cast<uint2*>(out + i) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
  } else {
    for (; i < n; ++i) out[i] = __float2bfloat16_rn(in[i]);
  }
}

// ---- embedding gather + image-feature splice (detikzify/model/v1/modeling_detikzify.py:157-189):
//      rows whose id is the patch token take the projector output instead of the table row.
__global__ void __launch_bounds__(128) embed_splice_kernel(const int64_t* __restrict__ ids, int T, int start_pos,
                                                           const bf16* __restrict__ embed, int H, int vocab,
                                                           int image_token, const float* __restrict__ img,
                                                           int img_start, int n_img, float* __restrict__ x) {
  const int t = blockIdx.x;
  if (t >= T) return;
  int64_t id = ids[t];
  const int ipos = start_pos + t - img_start;
  const bool is_img = (img != nullptr) && (id == image_token) && ipos >= 0 && ipos < n_img;
  if (id < 0 || id >= vocab) id = 0;  // validated on the host; never fault
  for (int i = threadIdx.x * 8; i < H; i += 128 * 8) {
    float f[8];
    if (is_img) {
      float4 a = *reinterpret_cast<const float4*>(img + (int64_t)ipos * H + i);
      float4 b = *reinterpret_cast<const float4*>(img + (int64_t)ipos * H + i + 4);
      f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
    } else {
      unpack8(*reinterpret_cast<const uint4*>(embed + id * H + i), f);
    }
    *reinterpret_cast<float4*>(x + (int64_t)t * H + i) = make_float4(f[0], f[1], f[2], f[3]);
    *reinterpret_cast<float4*>(x + (int64_t)t * H + i + 4) = make_float4(f[4], f[5], f[6], f[7]);
  }
}

// ---- prefill RoPE + KV-cache write (HF modeling_llama.py:124-168 rotate-half; cache append :269-270).
//      grid (T, heads + 2*kv_heads); HD/2 threads: thread i handles the pair (i, i+HD/2).
template <int HD>
__global__ void __launch_bounds__(HD / 2) rope_kv_prefill_kernel(const float* __restrict__ qkv, int T, int start_pos,
                                                                 int heads, int kv_heads,
                                                                 const float* __restrict__ rope_cs,
                                                                 bf16* __restrict__ q_out, bf16* __restrict__ kcache,
                                                                 bf16* __restrict__ vcache, int max_len) {
  constexpr int HALF = HD / 2;
  const int t = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
  const int qd = heads * HD, kd = kv_heads * HD;
  const int pos = start_pos + t;
  const float* src = qkv + (int64_t)t * (qd + 2 * kd) + hh * HD;
  const float a = src[i], b = src[i + HALF];
  const float2 cs = *reinterpret_cast<const float2*>(rope_cs + ((int64_t)pos * HALF + i) * 2);
  if (hh < heads) {
    bf16* d = q_out + (int64_t)t * qd + hh * HD;
    d[i] = __float2bfloat16_rn(a * cs.x - b * cs.y);
    d[i + HALF] = __float2bfloat16_rn(b * cs.x + a * cs.y);
  } else if (hh < heads + kv_heads) {
    bf16* d = kcache + ((int64_t)(hh - heads) * max_len + pos) * HD;
    d[i] = __float2bfloat16_rn(a * cs.x - b * cs.y);
    d[i + HALF] = __float2bfloat16_rn(b * cs.x + a * cs.y);
  } else {
    bf16* d = vcache + ((int64_t)(hh - heads - kv_heads) * max_len + pos) * HD;
    d[i] = __float2bfloat16_rn(a);
    d[i + HALF] = __float2bfloat16_rn(b);
  }
}

// ---- head_dim 64 RoPE of the caption encoder (rotate-half, HF modeling_llama.py), no cache: grid (T, heads + 2*kv_heads),
//      32 threads: thread i handles the pair (i, i+32).
__global__ void __launch_bounds__(32) rope_qkv64_kernel(const float* __restrict__ qkv, int heads, int kv_heads,
                                                        const float* __restrict__ rope_cs, bf16* __restrict__ q,
                                                        bf16* __restrict__ k, bf16* __restrict__ v) {
  const int t = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
  const int row = (heads + 2 * kv_heads) * 64;
  const float* src = qkv + (int64_t)t * row + hh * 64;
  const float a = src[i], b = src[i + 32];
  const float2 cs = *reinterpret_cast<const float2*>(rope_cs + ((int64_t)t * 32 + i) * 2);
  bf16* d;
  if (hh < heads) d = q + (int64_t)t * heads * 64 + hh * 64;
  else if (hh < heads + kv_heads) d = k + (int64_t)t * kv_heads * 64 + (hh - heads) * 64;
  else {
    d = v + (int64_t)t * kv_heads * 64 + (hh - heads - kv_heads) * 64;
    d[i] = __float2bfloat16_rn(a);
    d[i + 32] = __float2bfloat16_rn(b);
    return;
  }
  d[i] = __float2bfloat16_rn(a * cs.x - b * cs.y);
  d[i + 32] = __float2bfloat16_rn(b * cs.x + a * cs.y);
}

// ---- per-head LayerNorm (q_norm / k_norm of the TikZero cross-attention: nn.LayerNorm(head_dim) after the head split).
//      One warp per (row, head); hd even and <= 128: lane j holds the pairs j and j + 32; fp32 two-pass statistics.
__global__ void __launch_bounds__(256) head_layernorm_kernel(const bf16* in, int64_t ld_in, const bf16* __restrict__ w,
                                                             const bf16* __restrict__ b, float eps, int M, int heads, int hd,
                                                             bf16* out, int64_t ld_out) {
  const int64_t item = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (item >= (int64_t)M * heads) return;
  const int64_t row = item / heads;
  const int h = (int)(item % heads);
  const bf16* src = in + row * ld_in + h * hd;
  float2 x[2];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = 2 * (lane + 32 * j);
    x[j] = i < hd ? unpack_bf16x2(*reinterpret_cast<const uint32_t*>(src + i)) : make_float2(0.f, 0.f);
    s += x[j].x + x[j].y;
  }
  const float mean = warp_sum(s) / hd;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    if (2 * (lane + 32 * j) < hd) {
      const float a = x[j].x - mean, c = x[j].y - mean;
      q += a * a + c * c;
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / hd + eps);
  bf16* dst = out + row * ld_out + h * hd;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int i = 2 * (lane + 32 * j);
    if (i >= hd) continue;
    const float2 ww = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(w + i));
    const float2 bb = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(b + i));
    *reinterpret_cast<uint32_t*>(dst + i) =
        pack_bf16x2((x[j].x - mean) * rstd * ww.x + bb.x, (x[j].y - mean) * rstd * ww.y + bb.y);
  }
}

__global__ void __launch_bounds__(256) cast_bf16_f32_kernel(const bf16* __restrict__ in, float* __restrict__ out, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(in[i]);
}

// ---- batched-decode RoPE + KV-cache append: row b belongs to sequence slots[b] at position pos[b]
//      (HF modeling_llama.py:124-168; DynamicCache.update). grid (B, heads + 2*kv_heads); 64 threads.
template <int HD>
__global__ void __launch_bounds__(HD / 2) rope_kv_decode_kernel(const float* __restrict__ qkv, const int* __restrict__ slots,
                                                                const int* __restrict__ posv, const int* __restrict__ active,
                                                                int heads, int kv_heads,
                                                                const float* __restrict__ rope_cs, float* __restrict__ q_out,
                                                                bf16* __restrict__ kv_base, int64_t kv_slot_stride,
                                                                int64_t kv_v_offset, int max_len, bf16* __restrict__ q_bf16) {
  constexpr int HALF = HD / 2;
  const int b = blockIdx.x, hh = blockIdx.y, i = threadIdx.x;
  const int qd = heads * HD, kd = kv_heads * HD;
  const int pos = posv[b];
  const float* src = qkv + (int64_t)b * (qd + 2 * kd) + hh * HD;
  const float a = src[i], c = src[i + HALF];
  const float2 cs = *reinterpret_cast<const float2*>(rope_cs + ((int64_t)pos * HALF + i) * 2);
  if (hh < heads) {
    float* d = q_out + (int64_t)b * qd + hh * HD;
    const float y0 = a * cs.x - c * cs.y, y1 = c * cs.x + a * cs.y;
    d[i] = y0;
    d[i + HALF] = y1;
    if (q_bf16) {   // operand of the shared-prefix attention (tensor cores)
      bf16* d16 = q_bf16 + (int64_t)b * qd + hh * HD;
      d16[i] = __float2bfloat16_rn(y0);
      d16[i + HALF] = __float2bfloat16_rn(y1);
    }
  } else if (active && !active[b]) {
    // a retired row of a generation loop: its slot may already belong to another sequence
  } else if (hh < heads + kv_heads) {
    bf16* d = kv_base + (int64_t)slots[b] * kv_slot_stride + ((int64_t)(hh - heads) * max_len + pos) * HD;
    d[i] = __float2bfloat16_rn(a * cs.x - c * cs.y);
    d[i + HALF] = __float2bfloat16_rn(c * cs.x + a * cs.y);
  } else {
    bf16* d = kv_base + (int64_t)slots[b] * kv_slot_stride + kv_v_offset + ((int64_t)(hh - heads - kv_heads) * max_len + pos) * HD;
    d[i] = __float2bfloat16_rn(a);
    d[i + HALF] = __float2bfloat16_rn(c);
  }
}

// ---- SigLIP attention-pool head, single probe query over N tokens (HF modeling_siglip.py:628-654,
//      nn.MultiheadAttention with a learned probe). grid (heads, B), 128 threads; head_dim 72.
__global__ void __launch_bounds__(128) pool_attn_kernel(const float* __restrict__ q, const bf16* __restrict__ kv,
                                                        int N, int D, int heads, float scale,
                                                        bf16* __restrict__ out) {
  extern __shared__ float sm[];  // scores [N] + reduce scratch
  const int h = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
  const int hd = D / heads;
  float* sc = sm;
  __shared__ float red[4];
  const float* qh = q + h * hd;
  float lmax = -INFINITY;
  for (int j = tid; j < N; j += 128) {
    const bf16* kr = kv + ((int64_t)b * N + j) * 2 * D + h * hd;
    float s = 0.f;
    for (int i = 0; i < hd; i += 2) {
      float2 kk = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(kr + i));
      s += qh[i] * kk.x + qh[i + 1] * kk.y;
    }
    s *= scale;
    sc[j] = s;
    lmax = fmaxf(lmax, s);
  }
  lmax = warp_max(lmax);
  if ((tid & 31) == 0) red[tid >> 5] = lmax;
  __syncthreads();
  const float mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float lsum = 0.f;
  for (int j = tid; j < N; j += 128) {
    float e = __expf(sc[j] - mx);
    sc[j] = e;
    lsum += e;
  }
  lsum = warp_sum(lsum);
  if ((tid & 31) == 0) red[tid >> 5] = lsum;
  __syncthreads();
  const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
  if (tid < hd) {
    float acc = 0.f;
    for (int j = 0; j < N; ++j)
      acc += sc[j] * __bfloat162float(kv[((int64_t)b * N + j) * 2 * D + D + h * hd + tid]);
    out[(int64_t)b * D + h * hd + tid] = __float2bfloat16_rn(acc * inv);
  }
}

// lm_head log-softmax merge: one warp per row; lane l folds the tile partials l, l + 32, ... in order, then a fixed
// xor tree combines the lanes (deterministic)
__global__ void __launch_bounds__(256) lse_merge_kernel(const float2* __restrict__ part, const float* __restrict__ tgt,
                                                        const int64_t* __restrict__ targets, int M, int N, int NT,
                                                        float* __restrict__ logprob, float* __restrict__ lse) {
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  float mx = -INFINITY, s = 0.f;
  for (int j = lane; j < NT; j += 32) {
    const float2 q = part[(int64_t)m * NT + j];
    lse_combine(mx, s, q.x, q.y);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    lse_combine(mx, s, om, os);
  }
  if (lane == 0) {
    const float l = mx + logf(s);
    const int64_t t = targets[m];
    logprob[m] = (t >= 0 && t < N) ? tgt[m] - l : 0.f;
    if (lse) lse[m] = l;
  }
}

}  // namespace

cudaError_t launch_lse_merge(const float2* part, const float* tgt, const int64_t* targets, int M, int N, float* logprob,
                             float* lse, cudaStream_t s, uint64_t* counter) {
  if (M <= 0) return cudaSuccess;
  lse_merge_kernel<<<(M + 7) / 8, 256, 0, s>>>(part, tgt, targets, M, N, (N + LSE_TILE - 1) / LSE_TILE, logprob, lse);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_layernorm(const float* x, const bf16* w, const bf16* b, float eps, int M, int D, bf16* out_bf16,
                             float* out_f32, cudaStream_t s, uint64_t* counter) {
  if (D & 3) return cudaErrorInvalidValue;
  if (D <= 128 * 3) layernorm_reg_kernel<3><<<(M + 7) / 8, 256, 0, s>>>(x, w, b, eps, M, D, out_bf16, out_f32);
  else if (D <= 128 * 9) layernorm_reg_kernel<9><<<(M + 7) / 8, 256, 0, s>>>(x, w, b, eps, M, D, out_bf16, out_f32);
  else layernorm_kernel<<<(M + 7) / 8, 256, 0, s>>>(x, w, b, eps, M, D, out_bf16, out_f32);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_rmsnorm(const float* x, int64_t ldx, const bf16* w, float eps, int M, int D, bf16* out,
                           cudaStream_t s, uint64_t* counter) {
  if (D & 3) return cudaErrorInvalidValue;
  if (D <= 1024) rmsnorm_kernel<32><<<M, 32, 0, s>>>(x, ldx, w, eps, M, D, out);
  else if (D <= 4096) rmsnorm_kernel<128><<<M, 128, 0, s>>>(x, ldx, w, eps, M, D, out);
  else rmsnorm_kernel<256><<<M, 256, 0, s>>>(x, ldx, w, eps, M, D, out);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_im2col(const float* pixels, int B, int S, int P, int KP, bf16* out, cudaStream_t s,
                          uint64_t* counter) {
  int64_t rows = (int64_t)B * (S / P) * (S / P);
  im2col_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, s>>>(pixels, B, S, P, KP, out);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_cast_f32_bf16(const float* in, bf16* out, int64_t n, cudaStream_t s, uint64_t* counter) {
  int64_t blocks = (n + 1023) / 1024;
  cast_kernel<<<(unsigned)blocks, 256, 0, s>>>(in, out, n);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_embed_splice(const int64_t* ids, int T, int start_pos, const bf16* embed, int H, int vocab,
                                int image_token, const float* img, int img_start, int n_img, float* x,
                                cudaStream_t s, uint64_t* counter) {
  if (H & 7) return cudaErrorInvalidValue;
  embed_splice_kernel<<<T, 128, 0, s>>>(ids, T, start_pos, embed, H, vocab, image_token, img, img_start, n_img, x);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_rope_kv_prefill(const float* qkv, int T, int start_pos, int heads, int kv_heads,
                                   const float* rope_cs, bf16* q_out, bf16* kcache, bf16* vcache, int max_len, int hd,
                                   cudaStream_t s, uint64_t* counter) {
  dim3 grid(T, heads + 2 * kv_heads);
  if (hd == 128) rope_kv_prefill_kernel<128><<<grid, 64, 0, s>>>(qkv, T, start_pos, heads, kv_heads, rope_cs, q_out, kcache, vcache, max_len);
  else if (hd == 64) rope_kv_prefill_kernel<64><<<grid, 32, 0, s>>>(qkv, T, start_pos, heads, kv_heads, rope_cs, q_out, kcache, vcache, max_len);
  else return cudaErrorInvalidValue;
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_rope_qkv64(const float* qkv, int T, int heads, int kv_heads, const float* rope_cs, bf16* q, bf16* k, bf16* v,
                              cudaStream_t s, uint64_t* counter) {
  rope_qkv64_kernel<<<dim3(T, heads + 2 * kv_heads), 32, 0, s>>>(qkv, heads, kv_heads, rope_cs, q, k, v);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_head_layernorm(const bf16* in, int64_t ld_in, const bf16* w, const bf16* b, float eps, int M, int heads,
                                  int hd, bf16* out, int64_t ld_out, cudaStream_t s, uint64_t* counter) {
  if ((hd & 1) || hd > 128 || (ld_in & 1) || (ld_out & 1)) return cudaErrorInvalidValue;
  const int64_t items = (int64_t)M * heads;
  head_layernorm_kernel<<<(unsigned)((items + 7) / 8), 256, 0, s>>>(in, ld_in, w, b, eps, M, heads, hd, out, ld_out);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_cast_bf16_f32(const bf16* in, float* out, int64_t n, cudaStream_t s, uint64_t* counter) {
  cast_bf16_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(in, out, n);
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_rope_kv_decode(const float* qkv, int B, const int* slots, const int* pos, const int* active, int heads, int kv_heads,
                                  const float* rope_cs, float* q_out, bf16* kv_base, int64_t kv_slot_stride,
                                  int64_t kv_v_offset, int max_len, int hd, cudaStream_t s, uint64_t* counter, bf16* q_bf16) {
  dim3 grid(B, heads + 2 * kv_heads);
  if (hd == 128)
    rope_kv_decode_kernel<128><<<grid, 64, 0, s>>>(qkv, slots, pos, active, heads, kv_heads, rope_cs, q_out, kv_base, kv_slot_stride,
                                                   kv_v_offset, max_len, q_bf16);
  else if (hd == 64)
    rope_kv_decode_kernel<64><<<grid, 32, 0, s>>>(qkv, slots, pos, active, heads, kv_heads, rope_cs, q_out, kv_base, kv_slot_stride,
                                                  kv_v_offset, max_len, q_bf16);
  else return cudaErrorInvalidValue;
  if (counter) ++*counter;
  return cudaGetLastError();
}
cudaError_t launch_pool_attn(const float* q, const bf16* kv, int B, int N, int D, int heads, float scale, bf16* out,
                             cudaStream_t s, uint64_t* counter) {
  if (D / heads > 128) return cudaErrorInvalidValue;
  dim3 grid(heads, B);
  pool_attn_kernel<<<grid, 128, N * sizeof(float), s>>>(q, kv, N, D, heads, scale, out);
  if (counter) ++*counter;
  return cudaGetLastError();
}

}  // namespace dtk
