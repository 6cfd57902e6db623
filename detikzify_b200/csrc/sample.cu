// Fused sampler: one CTA per sequence over the fp32 logits row.
//
// Replaces the HF logits-processor chain + softmax + multinomial the reference drives through
// model.generate() (detikzify/infer/generate.py:218-227; HF generation/utils.py:2762-2793,
// logits_process.py NoBadWords / SuppressTokensAtBegin / Temperature / TopK / TopP(:521-528)):
//   mask bad word -> mask EOS on the first new token -> /T -> top-k -> softmax -> top-p ->
//   renormalise -> inverse-CDF draw (Philox counter RNG), or argmax when not sampling.
// The full-vocabulary sort of HF's TopP warper is replaced by a bit-wise threshold search on the
// float pattern of the probabilities (31 block reductions): tokens with ascending-cumulative mass
// <= 1 - top_p are removed, exactly HF's rule (ties are kept or dropped together).
// The PROC instantiations (dtk_processors) add HF's other processors in HF's order:
//   repetition penalty -> no-repeat n-gram -> bad words -> min length / min new tokens -> suppress tokens ->
//   begin-suppress tokens -> /T -> top-k -> softmax -> top-p -> min-p -> renormalise -> draw;
// the instantiations without them compile to the same code as before.
#include "common.cuh"
#include "launch.h"

namespace dtk {
namespace {

constexpr int ST = 1024;

struct RedScratch {
  float f[32];
  int i[32];
};

DTK_DEV float block_sum(float v, RedScratch& r) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) r.f[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = (threadIdx.x < 32) ? r.f[threadIdx.x] : 0.f;
  if (threadIdx.x < 32) {
    t = warp_sum(t);
    if (threadIdx.x == 0) r.f[0] = t;
  }
  __syncthreads();
  t = r.f[0];
  __syncthreads();
  return t;
}
DTK_DEV int block_sum_int(int v, RedScratch& r) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) r.i[threadIdx.x >> 5] = v;
  __syncthreads();
  int t = (threadIdx.x < 32) ? r.i[threadIdx.x] : 0;
  if (threadIdx.x < 32) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) r.i[0] = t;
  }
  __syncthreads();
  t = r.i[0];
  __syncthreads();
  return t;
}
// (max value, lowest index attaining it)
DTK_DEV void block_argmax(float& v, int& idx, RedScratch& r) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, idx, o);
    if (ov > v || (ov == v && oi < idx)) { v = ov; idx = oi; }
  }
  if ((threadIdx.x & 31) == 0) { r.f[threadIdx.x >> 5] = v; r.i[threadIdx.x >> 5] = idx; }
  __syncthreads();
  if (threadIdx.x < 32) {
    float tv = r.f[threadIdx.x];
    int ti = r.i[threadIdx.x];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, tv, o);
      int oi = __shfl_xor_sync(0xffffffffu, ti, o);
      if (ov > tv || (ov == tv && oi < ti)) { tv = ov; ti = oi; }
    }
    if (threadIdx.x == 0) { r.f[0] = tv; r.i[0] = ti; }
  }
  __syncthreads();
  v = r.f[0];
  idx = r.i[0];
  __syncthreads();
}

// order-preserving map float -> uint32
DTK_DEV uint32_t fkey(float f) {
  uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Philox4x32-10, returns one uniform in [0,1)
DTK_DEV float philox_uniform(uint64_t seed, uint32_t c0, uint32_t c1) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t x0 = c0, x1 = c1, x2 = 0x243F6A88u, x3 = 0x85A308D3u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(0xD2511F53u, x0), lo0 = 0xD2511F53u * x0;
    uint32_t hi1 = __umulhi(0xCD9E8D57u, x2), lo1 = 0xCD9E8D57u * x2;
    uint32_t n0 = hi1 ^ x1 ^ k0, n1 = lo1, n2 = hi0 ^ x3 ^ k1, n3 = lo0;
    x0 = n0; x1 = n1; x2 = n2; x3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return (float)(x0 >> 8) * (1.0f / 16777216.0f);
}

// the uniform of row b: counter step + loop step on stream seq_id, from the loop's per-row arrays when it has them
DTK_DEV float draw_uniform(const SampleArgs& p, const int b, const SampleSeq& sq) {
  const uint32_t gstep = p.gen_step ? (uint32_t)*p.gen_step : 0u;
  const uint32_t step = p.row_step ? p.row_step[b] : sq.step, sid = p.row_step ? p.row_seq[b] : sq.seq_id;
  return philox_uniform(p.seed_dev ? *p.seed_dev : p.seed, step + gstep, sid);
}

// ---- HF logits processors (sampler instantiations with PROC = true only): the ban and repetition-penalty bitmasks of row
// b, built from its token history h[0, L) and the call's tables in shared memory (2 x 4096 words, so V <= 131072).
// HF generation/logits_process.py: RepetitionPenalty (every distinct id of input_ids), NoRepeatNGram
// (_calc_banned_ngram_tokens), NoBadWords (SequenceBias with -inf: length-1 entries always, a longer entry when the history
// ends with its prefix, skipped when longer than the history), MinLength / MinNewTokensLength (EOS), SuppressTokens,
// SuppressTokensAtBegin (first new token: the suppress flag).
DTK_DEV void set_bit(uint32_t* m, int id, int V) {
  if ((unsigned)id < (unsigned)V) atomicOr(m + (id >> 5), 1u << (id & 31));
}
DTK_DEV bool get_bit(const uint32_t* m, int id) { return (m[id >> 5] >> (id & 31)) & 1u; }

DTK_DEV void build_proc_masks(const SampleProc& q, int b, int suppress, int V, uint32_t* ban, uint32_t* pen) {
  const int tid = threadIdx.x, nw = (V + 31) >> 5;
  for (int i = tid; i < nw; i += ST) { ban[i] = 0u; pen[i] = 0u; }
  __syncthreads();
  const SampleProcTable& t = *q.tab;
  const int L = q.hist_len[b];
  const int* h = q.hist + (int64_t)b * q.hist_stride;
  if (t.penalty != 1.f)
    for (int i = tid; i < L; i += ST) set_bit(pen, h[i], V);
  for (int i = tid; i < t.n_ban; i += ST) set_bit(ban, t.ids[i], V);
  if (suppress)
    for (int i = tid; i < t.n_begin; i += ST) set_bit(ban, t.ids[t.n_ban + i], V);
  if (tid == 0 && L < t.eos_until[b]) set_bit(ban, t.eos, V);
  const int n = t.ngram;
  if (n > 0 && L + 1 >= n) {   // every n-gram h[j, j + n) whose first n - 1 ids equal the last n - 1 ids bans h[j + n - 1]
    const int* tail = h + (L - n + 1);
    for (int j = tid; j <= L - n; j += ST) {
      bool eq = true;
      for (int k = 0; k < n - 1 && eq; ++k) eq = h[j + k] == tail[k];
      if (eq) set_bit(ban, h[j + n - 1], V);
    }
  }
  const int* off = t.ids + t.n_ban + t.n_begin;
  const int* wid = off + t.n_words + 1;
  for (int e = tid; e < t.n_words; e += ST) {
    const int o0 = off[e], len = off[e + 1] - o0;
    if (len > L) continue;
    bool eq = true;
    for (int k = 0; k < len - 1 && eq; ++k) eq = h[L - len + 1 + k] == wid[o0 + k];
    if (eq) set_bit(ban, wid[o0 + len - 1], V);
  }
  __syncthreads();
}

// repetition penalty in fp32 on the raw logit, then the bans (before the division by T)
DTK_DEV float apply_proc(float x, int i, float penalty, const uint32_t* ban, const uint32_t* pen) {
  if (get_bit(pen, i)) x = x < 0.f ? __fmul_rn(x, penalty) : __fdiv_rn(x, penalty);
  return get_bit(ban, i) ? -INFINITY : x;
}

// the generation loop appends the drawn token to the row's history, clamped at the row's end as gen_pos is at max_pos
DTK_DEV void append_hist(const SampleProc& q, int b, int token) {
  const int L = q.hist_len[b];
  if (L < q.hist_stride) q.hist[(int64_t)b * q.hist_stride + L] = token;
  q.hist_len[b] = min(L + 1, q.hist_stride);
}

// one row's token (every thread returns it) from logits lg with row b's state: scratch row, suppress flag, history and RNG
// stream and counter (read at the draw: the loop's step counter advances only after every row of the step has arrived)
template <bool PROC>
DTK_DEV int sample_generic_body(const SampleArgs& p, const SampleProc& q, const int b, const float* lg) {
  __shared__ RedScratch red;
  __shared__ float sm_scan[32];
  __shared__ int sm_choice;
  const int tid = threadIdx.x, V = p.V;
  float* w = p.scratch + (int64_t)b * V;
  const SampleSeq sq = p.seq[b];
  const bool sampling = p.do_sample && p.temperature > 0.f;
  const float T = sampling ? p.temperature : 1.f;
  uint32_t *ban = nullptr, *pen = nullptr;
  float penalty = 1.f, min_p = 0.f;
  if constexpr (PROC) {
    __shared__ uint32_t proc_masks[2 * (kProcMaxVocab / 32)];
    ban = proc_masks;
    pen = proc_masks + ((V + 31) >> 5);
    build_proc_masks(q, b, sq.suppress, V, ban, pen);
    penalty = q.tab->penalty;
    min_p = q.tab->min_p;
  }

  // 1. masks + temperature, running (max, argmax)
  float mx = -INFINITY;
  int amx = 0x7fffffff;
  for (int i = tid; i < V; i += ST) {
    float v = lg[i];
    if constexpr (PROC) v = apply_proc(v, i, penalty, ban, pen);
    if (i == p.bad_token || (sq.suppress && i == p.bs_token)) v = -INFINITY;
    v = v / T;
    w[i] = v;
    if (v > mx) { mx = v; amx = i; }
  }
  block_argmax(mx, amx, red);
  int token = amx;

  if (sampling) {
    // 2. top-k: keep scores >= k-th largest (HF TopKLogitsWarper: remove scores < kth)
    if (p.top_k > 0 && p.top_k < V) {
      uint32_t thr = 0;
      for (int bit = 31; bit >= 0; --bit) {
        uint32_t cand = thr | (1u << bit);
        int cnt = 0;
        for (int i = tid; i < V; i += ST) cnt += (fkey(w[i]) >= cand);
        cnt = block_sum_int(cnt, red);
        if (cnt >= p.top_k) thr = cand;
      }
      for (int i = tid; i < V; i += ST)
        if (fkey(w[i]) < thr) w[i] = -INFINITY;
      __syncthreads();
    }
    // 3. softmax
    float z = 0.f;
    for (int i = tid; i < V; i += ST) {
      float e = __expf(w[i] - mx);
      w[i] = e;
      z += e;
    }
    z = block_sum(z, red);
    const float invz = 1.f / z;
    for (int i = tid; i < V; i += ST) w[i] *= invz;
    __syncthreads();
    // 4. top-p: remove tokens whose ascending cumulative mass is <= 1 - top_p
    float theta = -1.f;  // tokens with prob <= theta are removed
    if (p.top_p < 1.f) {
      const float limit = p.top_p_limit;
      uint32_t tb = 0;
      for (int bit = 30; bit >= 0; --bit) {
        uint32_t cand = tb | (1u << bit);
        float cf = __uint_as_float(cand);
        float sacc = 0.f;
        for (int i = tid; i < V; i += ST) {
          float pv = w[i];
          sacc += (pv <= cf) ? pv : 0.f;
        }
        sacc = block_sum(sacc, red);
        if (sacc <= limit) tb = cand;
      }
      theta = __uint_as_float(tb);
      const float pmax = invz;  // exp(0) / z
      if (theta >= pmax) theta = nextafterf(pmax, 0.f);  // min_tokens_to_keep = 1
    }
    // 5. renormalise over the nucleus (min-p: also drop p < min_p * p_max; p_max = invz is always kept)
    float z2 = 0.f;
    if constexpr (PROC) {
      const float mthr = min_p * invz;
      for (int i = tid; i < V; i += ST) {
        float pv = w[i];
        if (pv <= theta || pv < mthr) { pv = 0.f; w[i] = 0.f; }
        z2 += pv;
      }
    } else {
      for (int i = tid; i < V; i += ST) {
        float pv = w[i];
        if (pv <= theta) { pv = 0.f; w[i] = 0.f; }
        z2 += pv;
      }
    }
    z2 = block_sum(z2, red);
    const float invz2 = 1.f / z2;
    for (int i = tid; i < V; i += ST) w[i] *= invz2;
    __syncthreads();
    // 6. inverse-CDF draw in index order
    const float u = draw_uniform(p, b, sq);
    const int per = (V + ST - 1) / ST;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    float loc = 0.f;
    for (int i = i0; i < i1; ++i) loc += w[i];
    // exclusive block scan of loc
    float inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_up_sync(0xffffffffu, inc, o);
      if ((tid & 31) >= o) inc += t;
    }
    if ((tid & 31) == 31) sm_scan[tid >> 5] = inc;
    if (tid == 0) sm_choice = -1;
    __syncthreads();
    if (tid < 32) {
      float v = sm_scan[tid], t2 = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, t2, o);
        if (tid >= o) t2 += t;
      }
      sm_scan[tid] = t2 - v;  // exclusive warp offsets
    }
    __syncthreads();
    const float excl = sm_scan[tid >> 5] + inc - loc;
    if (loc > 0.f && u >= excl && u < excl + loc) {
      float c = excl;
      int pick = -1;
      for (int i = i0; i < i1; ++i) {
        float pv = w[i];
        if (pv > 0.f) {
          pick = i;
          c += pv;
          if (u < c) break;
        }
      }
      if (pick >= 0) atomicMax(&sm_choice, pick);
    }
    __syncthreads();
    if (sm_choice >= 0) token = sm_choice;  // else: rounding left u beyond the total mass -> argmax
  } else if (p.want_probs) {
    // greedy: probability vector = softmax of the masked logits (for parity inspection only)
    float z = 0.f;
    for (int i = tid; i < V; i += ST) {
      float e = __expf(w[i] - mx);
      w[i] = e;
      z += e;
    }
    z = block_sum(z, red);
    const float invz = 1.f / z;
    for (int i = tid; i < V; i += ST) w[i] *= invz;
  }
  return token;
}

// thread 0 of row b's CTA, after the draw: the output id and the generation-loop state. A retired row (token -1, the ring's
// sentinel) publishes only its stamped ring entry and its arrival, so the host and the step counter see every row every step
template <bool PROC>
DTK_DEV void finish_row(const SampleArgs& p, const SampleProc& q, const int b, const int token) {
  if (p.out_ids) p.out_ids[b] = token;
  if (p.gen_tok) {
    const unsigned long long gstep = *p.gen_step;   // unchanged until this row has arrived below
    if (token >= 0) {
      p.gen_tok[b] = token;
      p.gen_pos[b] = min(p.gen_pos[b] + 1, p.max_pos);
      if constexpr (PROC) append_hist(q, b, token);
    }
    // ONE 8-byte store to the mapped pinned ring carries the token and its step stamp, so no ordering between two
    // host-visible stores (and no system-scope fence, a PCIe round trip) is needed; the host polls the entry itself
    const unsigned long long entry = ((gstep + 1ull) << 32) | (unsigned long long)(unsigned)token;
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(p.host_ring + (gstep % (unsigned long long)p.ring) * p.B + b), "l"(entry) : "memory");
    unsigned prev = atomicAdd(p.done_counter, 1u);
    if (prev == (unsigned)p.B - 1u) {   // last sequence of this step: advance the device-side step counter
      *p.done_counter = 0u;
      *p.gen_step = gstep + 1ull;
    }
  }
}

template <bool PROC>
DTK_DEV int sample_body(const SampleArgs& p, const SampleProc& q, int b, const float* lg);

// one CTA per row: the sampler of dtk_sample and of every generation-loop step
template <bool REG, bool PROC>
DTK_DEV void sample_row(const SampleArgs& p, const SampleProc& q) {
  const int b = blockIdx.x;
  if (p.active && !p.active[b]) {
    if (threadIdx.x == 0) finish_row<PROC>(p, q, b, -1);
    return;
  }
  const float* lg = p.logits + (int64_t)b * p.V;
  int token;
  if constexpr (REG) token = sample_body<PROC>(p, q, b, lg);
  else token = sample_generic_body<PROC>(p, q, b, lg);
  if (threadIdx.x == 0) finish_row<PROC>(p, q, b, token);
}


// ---- register-resident path (V <= ST * VPT): every thread keeps its VPT strided entries i = tid + j * ST in
// registers, so the 31 + 31 threshold-search passes of top-k / top-p touch no memory at all; block reductions use one
// __syncthreads per pass (double-buffered partials, every warp re-reduces the 32 warp partials with the same butterfly,
// so all threads get the bit-identical sum). Per-thread accumulation order and reduction tree are the same as in
// sample_generic_kernel: both kernels produce identical tokens and probability vectors.
constexpr int VPT = 32;

struct Red2 {
  float f[2][32];
  int i[2][32];
};
DTK_DEV float allreduce_sum(float v, Red2& r, int& ph) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) r.f[ph][threadIdx.x >> 5] = v;
  __syncthreads();
  const float t = warp_sum(r.f[ph][threadIdx.x & 31]);
  ph ^= 1;
  return t;
}
DTK_DEV int allreduce_sum_int(int v, Red2& r, int& ph) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) r.i[ph][threadIdx.x >> 5] = v;
  __syncthreads();
  int t = r.i[ph][threadIdx.x & 31];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
  ph ^= 1;
  return t;
}

template <bool PROC>
DTK_DEV int sample_body(const SampleArgs& p, const SampleProc& q, const int b, const float* lg) {
  __shared__ RedScratch red;
  __shared__ Red2 red2;
  __shared__ float sm_scan[32];
  __shared__ int sm_choice;
  const int tid = threadIdx.x, V = p.V;
  float* w = p.scratch + (int64_t)b * V;
  const SampleSeq sq = p.seq[b];
  const bool sampling = p.do_sample && p.temperature > 0.f;
  const float T = sampling ? p.temperature : 1.f;
  int ph = 0;
  uint32_t *ban = nullptr, *pen = nullptr;
  float penalty = 1.f, min_p = 0.f;
  if constexpr (PROC) {
    __shared__ uint32_t proc_masks[2 * (kProcMaxVocab / 32)];
    ban = proc_masks;
    pen = proc_masks + ((V + 31) >> 5);
    build_proc_masks(q, b, sq.suppress, V, ban, pen);
    penalty = q.tab->penalty;
    min_p = q.tab->min_p;
  }

  // 1. masks + temperature, running (max, argmax); entries beyond V are -inf (probability 0 everywhere below)
  float v[VPT];
  float mx = -INFINITY;
  int amx = 0x7fffffff;
#pragma unroll
  for (int j = 0; j < VPT; ++j) {
    const int i = tid + j * ST;
    float x = -INFINITY;
    if (i < V) {
      x = __ldcg(lg + i);
      if constexpr (PROC) x = apply_proc(x, i, penalty, ban, pen);
      if (i == p.bad_token || (sq.suppress && i == p.bs_token)) x = -INFINITY;
      x = x / T;
      if (x > mx) { mx = x; amx = i; }
    }
    v[j] = x;
  }
  block_argmax(mx, amx, red);
  int token = amx;

  if (sampling) {
    // 2. top-k: keep scores >= k-th largest
    if (p.top_k > 0 && p.top_k < V) {
      uint32_t thr = 0;
      for (int bit = 31; bit >= 0; --bit) {
        const uint32_t cand = thr | (1u << bit);
        int cnt = 0;
#pragma unroll
        for (int j = 0; j < VPT; ++j) cnt += (tid + j * ST < V) && (fkey(v[j]) >= cand);
        cnt = allreduce_sum_int(cnt, red2, ph);
        if (cnt >= p.top_k) thr = cand;
      }
#pragma unroll
      for (int j = 0; j < VPT; ++j)
        if (fkey(v[j]) < thr) v[j] = -INFINITY;
    }
    // 3. softmax
    float z = 0.f;
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
      const float e = (tid + j * ST < V) ? __expf(v[j] - mx) : 0.f;
      v[j] = e;
      if (tid + j * ST < V) z += e;
    }
    z = allreduce_sum(z, red2, ph);
    const float invz = 1.f / z;
#pragma unroll
    for (int j = 0; j < VPT; ++j) v[j] *= invz;
    // 4. top-p: remove tokens whose ascending cumulative mass is <= 1 - top_p
    float theta = -1.f;
    if (p.top_p < 1.f) {
      const float limit = p.top_p_limit;
      uint32_t tb = 0;
      for (int bit = 30; bit >= 0; --bit) {
        const uint32_t cand = tb | (1u << bit);
        const float cf = __uint_as_float(cand);
        float sacc = 0.f;
#pragma unroll
        for (int j = 0; j < VPT; ++j)
          if (tid + j * ST < V) sacc += (v[j] <= cf) ? v[j] : 0.f;
        sacc = allreduce_sum(sacc, red2, ph);
        if (sacc <= limit) tb = cand;
      }
      theta = __uint_as_float(tb);
      const float pmax = invz;
      if (theta >= pmax) theta = nextafterf(pmax, 0.f);  // min_tokens_to_keep = 1
    }
    // 5. renormalise over the nucleus; the final probability vector goes to the scratch row
    float z2 = 0.f;
    if constexpr (PROC) {   // min-p: also drop p < min_p * p_max (p_max = invz is always kept)
      const float mthr = min_p * invz;
#pragma unroll
      for (int j = 0; j < VPT; ++j) {
        if (v[j] <= theta || v[j] < mthr) v[j] = 0.f;
        if (tid + j * ST < V) z2 += v[j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < VPT; ++j) {
        if (v[j] <= theta) v[j] = 0.f;
        if (tid + j * ST < V) z2 += v[j];
      }
    }
    z2 = allreduce_sum(z2, red2, ph);
    const float invz2 = 1.f / z2;
#pragma unroll
    for (int j = 0; j < VPT; ++j)
      if (tid + j * ST < V) w[tid + j * ST] = v[j] * invz2;
    __syncthreads();
    // 6. inverse-CDF draw in index order (blocked ranges, read back from the scratch row)
    const float u = draw_uniform(p, b, sq);
    const int per = (V + ST - 1) / ST;
    const int i0 = tid * per, i1 = min(V, i0 + per);
    float loc = 0.f;
    for (int i = i0; i < i1; ++i) loc += w[i];
    float inc = loc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      float t = __shfl_up_sync(0xffffffffu, inc, o);
      if ((tid & 31) >= o) inc += t;
    }
    if ((tid & 31) == 31) sm_scan[tid >> 5] = inc;
    if (tid == 0) sm_choice = -1;
    __syncthreads();
    if (tid < 32) {
      float sv = sm_scan[tid], t2 = sv;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        float t = __shfl_up_sync(0xffffffffu, t2, o);
        if (tid >= o) t2 += t;
      }
      sm_scan[tid] = t2 - sv;
    }
    __syncthreads();
    const float excl = sm_scan[tid >> 5] + inc - loc;
    if (loc > 0.f && u >= excl && u < excl + loc) {
      float c = excl;
      int pick = -1;
      for (int i = i0; i < i1; ++i) {
        float pv = w[i];
        if (pv > 0.f) {
          pick = i;
          c += pv;
          if (u < c) break;
        }
      }
      if (pick >= 0) atomicMax(&sm_choice, pick);
    }
    __syncthreads();
    if (sm_choice >= 0) token = sm_choice;
  } else if (p.want_probs) {
    // greedy: probability vector = softmax of the masked logits (parity inspection only; skipped in the decode loop)
    float z = 0.f;
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
      const float e = (tid + j * ST < V) ? __expf(v[j] - mx) : 0.f;
      v[j] = e;
      if (tid + j * ST < V) z += e;
    }
    z = allreduce_sum(z, red2, ph);
    const float invz = 1.f / z;
#pragma unroll
    for (int j = 0; j < VPT; ++j)
      if (tid + j * ST < V) w[tid + j * ST] = v[j] * invz;
  }
  return token;
}

__global__ void __launch_bounds__(ST) sample_generic_kernel(const SampleArgs p) { sample_row<false, false>(p, SampleProc{}); }
__global__ void __launch_bounds__(ST) sample_generic_proc_kernel(const SampleArgs p, const SampleProc q) {
  sample_row<false, true>(p, q);
}
__global__ void __launch_bounds__(ST) sample_kernel(const SampleArgs p) { sample_row<true, false>(p, SampleProc{}); }
__global__ void __launch_bounds__(ST) sample_proc_kernel(const SampleArgs p, const SampleProc q) { sample_row<true, true>(p, q); }

// admission of a sequence into row m.row of a running generation loop (launch_sample_admit)
template <bool REG, bool PROC>
__global__ void __launch_bounds__(ST) sample_admit_kernel(const SampleArgs p, const SampleProc q, const SampleAdmit m) {
  const int r = m.row;
  if constexpr (PROC) {   // the row's history (prompt) was copied in before this launch; its length and min-length here
    if (threadIdx.x == 0) { q.hist_len[r] = m.hist_len; m.tab->eos_until[r] = m.eos_min; }
    __syncthreads();
  }
  int token;   // counter p.seq[r].step (0) on stream p.seq[r].seq_id: p carries no loop state
  if constexpr (REG) token = sample_body<PROC>(p, q, r, m.logits);
  else token = sample_generic_body<PROC>(p, q, r, m.logits);
  if (threadIdx.x == 0) {
    const unsigned long long gstep = *m.gen_step;   // the loop step that decodes the first token draws counter 1
    m.slots[r] = m.slot; m.posv[r] = m.pos; m.tok[r] = token;
    m.share_slots[r] = m.share_slot; m.share_lens[r] = m.share_len;
    m.row_step[r] = 1u - (uint32_t)gstep; m.row_seq[r] = m.seq_id;
    if constexpr (PROC) append_hist(q, r, token);
    m.active[r] = 1;
    const unsigned long long entry = ((unsigned long long)m.stamp << 32) | (unsigned long long)(unsigned)token;
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(m.mailbox + r), "l"(entry) : "memory");
  }
}

}  // namespace

static int g_sample_impl = 0;  // 0 = register-resident kernel when the vocabulary fits, 1 = always the generic kernel (tests)
void set_sample_impl(int impl) { g_sample_impl = impl; }
int get_sample_impl() { return g_sample_impl; }

cudaError_t launch_sample(const SampleArgs& a, cudaStream_t s, uint64_t* counter) {
  if (a.B <= 0 || a.B > 64) return cudaErrorInvalidValue;
  if (g_sample_impl == 0 && a.V <= ST * VPT) sample_kernel<<<a.B, ST, 0, s>>>(a);
  else sample_generic_kernel<<<a.B, ST, 0, s>>>(a);
  if (counter) ++*counter;
  return cudaGetLastError();
}

cudaError_t launch_sample_admit(const SampleArgs& a, const SampleProc* q, const SampleAdmit& m, cudaStream_t s,
                                uint64_t* counter) {
  if (m.row < 0 || m.row >= 64 || (q && (a.V > kProcMaxVocab || !q->tab || !q->hist || !q->hist_len || !m.tab)))
    return cudaErrorInvalidValue;
  const bool reg = g_sample_impl == 0 && a.V <= ST * VPT;
  if (q) {
    if (reg) sample_admit_kernel<true, true><<<1, ST, 0, s>>>(a, *q, m);
    else sample_admit_kernel<false, true><<<1, ST, 0, s>>>(a, *q, m);
  } else {
    if (reg) sample_admit_kernel<true, false><<<1, ST, 0, s>>>(a, SampleProc{}, m);
    else sample_admit_kernel<false, false><<<1, ST, 0, s>>>(a, SampleProc{}, m);
  }
  if (counter) ++*counter;
  return cudaGetLastError();
}

cudaError_t launch_sample_proc(const SampleArgs& a, const SampleProc& q, cudaStream_t s, uint64_t* counter) {
  if (a.B <= 0 || a.B > 64 || a.V > kProcMaxVocab || !q.tab || !q.hist || !q.hist_len) return cudaErrorInvalidValue;
  if (g_sample_impl == 0 && a.V <= ST * VPT) sample_proc_kernel<<<a.B, ST, 0, s>>>(a, q);
  else sample_generic_proc_kernel<<<a.B, ST, 0, s>>>(a, q);
  if (counter) ++*counter;
  return cudaGetLastError();
}

}  // namespace dtk
