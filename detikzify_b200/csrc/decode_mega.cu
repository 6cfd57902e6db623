// Persistent weight-streaming decode kernel: ONE cooperative launch per generated token.
//
// Why: batch-1 decode streams every decoder weight once per token (2.56 GB for ds-1.3b) through ~120
// dependent GEMV-sized steps of a few microseconds each. Launched as separate kernels (even from a
// CUDA graph) the HBM pipe drains at every step boundary and the chain is launch/ramp bound.
// Here the weight stream is decoupled from the dependency chain:
//
//   * grid = one CTA per SM, resident for the whole token (cooperative launch);
//   * 4 PRODUCER warps per CTA (one issuing lane each, registers handed back with setmaxnreg.dec) walk the
//     CTA's statically known list of weight tiles AND cached key/value items for ALL layers and phases and stream
//     them with 1-D TMA bulk copies (cp.async.bulk + mbarrier complete_tx) into a ~190 KB shared-memory ring of
//     8 KB slots, never waiting for activations — neither weights nor the cache depend on this token — so HBM
//     stays busy across phase boundaries;
//   * 8 CONSUMER warps (setmaxnreg.inc: the kernel calls no function, or ptxas would ignore setmaxnreg) take
//     tiles in order. A tile is 16 output rows x 256 k, pre-arranged in HBM (launch_retile, once at load) so that
//     it lands in shared memory exactly in ldmatrix.x4 order; the dot products run on the tensor pipe (mma.sync
//     m16n8k16, fp32 accumulate) with the activation vector split into bf16 hi + lo parts (x = hi + lo to 2^-17)
//     that occupy alternating columns of the B operand: one HMMA per k-step, fp32-grade GEMV; the ring slot is
//     handed back as soon as its shared-memory reads are issued;
//   * rows are grouped so that one thread's two accumulator rows (g, g+8) are a RoPE pair (i, i+HD/2) or a
//     SwiGLU pair (gate_i, up_i): RMSNorm scale, RoPE + KV-cache write, SiLU*mul and residual add are all fused
//     into the group epilogue; partial sums of a group's k-tiles are combined in a fixed order (deterministic);
//     the epilogues of a phase run in PARALLEL behind a CTA barrier (warp w takes groups w, w + 8, ...), not on whichever
//     warp finishes a group last;
//   * values that cross CTAs travel as 8-byte TAGGED words {fp32, phase tag} (see below): no grid-wide barrier or
//     counter anywhere, readers poll the words they need;
//   * the input vector of a phase is staged per 256-element SLICE by the warp whose tile needs it (stage_slice):
//     one coalesced L2 round trip per warp, no CTA-wide two-pass staging; phases end with a CTA barrier only;
//   * a phase's 16-row groups are cut into equal blocks over as many CTAs as needed (the participating set
//     rotates from phase to phase), so participants finish together and idle CTAs' producers run ahead.
//
// Per layer: P1 qkv(+RMSNorm, RoPE, KV write) | P2 split-KV attention (the CTA's share of the cached keys/values
// arrives through the ring; a fixed owner CTA per head merges the partials) | P3 o-proj + residual | P4 gate/up +
// SiLU*mul (+RMSNorm) | P5 down + residual; finally lm_head (+final RMSNorm, + greedy argmax and token publication
// in the kernel tail). DESIGN.md section 4 describes the design.
//
// Replaces the per-token HF eager path (modeling_llama.py:303-333, ~900 launches per token).
#include "common.cuh"
#include "fp8.cuh"
#include "launch.h"

namespace dtk {
namespace {

constexpr int NCW = 8;                       // consumer warps
constexpr int NPW = 4;                       // producer warps (one issuing lane each)
constexpr int MEGA_THREADS = (NCW + NPW) * 32;
constexpr int CONSUMER_THREADS = NCW * 32;
static_assert(NCW % NPW == 0, "slot ownership: NPW must divide NCW");
constexpr int TILE_BYTES = 8192;             // ring slot = one weight tile = one 16-key K+V attention item
constexpr int KV_V_OFF = 4096;               // byte offset of the V rows in an attention item (K rows at 0; 16 x HD x 2 B each)
constexpr int NT = 104;                      // per-tile partial-sum entries (>= max tiles/group + tiles in flight)
constexpr int NS = 72;                       // 256-column slices of a staged input vector (>= max tiles per group)
constexpr int NG = 48;                       // per-group arrival counters / prefetched residual rows (>= groups in flight)
constexpr long long SPIN_CYCLES = 4000000000ll;  // bounded waits (~2 s): trap instead of hanging the GPU

// ------------------------------------------------------------------ mbarrier / bulk-copy PTX
DTK_DEV void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
DTK_DEV void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
DTK_DEV void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
DTK_DEV uint32_t mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}\n"
      : "=r"(done)
      : "r"(bar), "r"(parity)
      : "memory");
  return done;
}
// slow path of a wait: bounded spin, trap instead of hanging the GPU
DTK_DEV void mbar_wait_slow(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  long long t0 = 0;
  while (!mbar_try(bar, parity)) {
    if ((++spins & 1023u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > SPIN_CYCLES) __trap();
    }
  }
}
DTK_DEV void mbar_wait(uint32_t bar, uint32_t parity) {
  if (!mbar_try(bar, parity)) mbar_wait_slow(bar, parity);
}
DTK_DEV void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// the same copy with an L2 cache policy (createpolicy) attached
DTK_DEV void bulk_g2s_hint(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;\n" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar), "l"(pol)
               : "memory");
}
DTK_DEV uint64_t policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
  return pol;
}
DTK_DEV void consumer_sync() { asm volatile("bar.sync 1, %0;\n" ::"n"(CONSUMER_THREADS) : "memory"); }

// ------------------------------------------------------------------ tagged activation words
// Every activation value that crosses CTAs (residual stream, q, the new key/value row, attention partials and output,
// the SwiGLU vector) travels as ONE 8-byte word {fp32 value, 32-bit phase tag}: aligned 8-byte accesses are single-copy
// atomic, so a reader that sees the expected tag also sees the value written with it — no release fence on the
// producer side and no acquire on the consumer side. Writers use st.relaxed.gpu.
// Readers first try a WEAK coalesced load (ld.cg: may be served by the SM's own L2 partition) and only re-read with
// ld.relaxed.gpu the words whose tag is still old — a stale copy is harmless because it carries a stale tag.
// The grid-wide counter below is therefore only a HINT that says when reading is worthwhile; correctness rests on the
// tags. A buffer is overwritten one layer later, after a chain of data dependencies that runs through every CTA which
// read it (write-after-read safe).
typedef unsigned long long u64;
DTK_DEV void st_tag(u64* p, float v, uint32_t tag) {
  const u64 w = ((u64)tag << 32) | (u64)__float_as_uint(v);
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;\n" ::"l"(p), "l"(w) : "memory");
}
DTK_DEV ulonglong2 ld_strong2(const u64* p) {
  ulonglong2 r;
  asm volatile("ld.relaxed.gpu.global.v2.u64 {%0, %1}, [%2];\n" : "=l"(r.x), "=l"(r.y) : "l"(p) : "memory");
  return r;
}
DTK_DEV ulonglong2 ld_weak2(const u64* p) {
  ulonglong2 r;
  asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];\n" : "=l"(r.x), "=l"(r.y) : "l"(p) : "memory");
  return r;
}
DTK_DEV u64 ld_strong1(const u64* p) {
  u64 r;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];\n" : "=l"(r) : "l"(p) : "memory");
  return r;
}
DTK_DEV u64 ld_weak1(const u64* p) {
  u64 r;
  asm volatile("ld.global.cg.u64 %0, [%1];\n" : "=l"(r) : "l"(p) : "memory");
  return r;
}
DTK_DEV bool tag_ok(u64 w, uint32_t tag) { return (uint32_t)(w >> 32) == tag; }
DTK_DEV float tag_val(u64 w) { return __uint_as_float((uint32_t)w); }
struct Spin {   // bounded polling with a short back-off: trap instead of hanging the GPU
  uint32_t n = 0;
  long long t0 = 0;
  DTK_DEV void tick() {
    __nanosleep(32);   // short back-off between polls of the same word (not re-tuned on the H100)
    if ((++n & 255u) == 0) {
      const long long now = clock64();
      if (t0 == 0) t0 = now;
      else if (now - t0 > SPIN_CYCLES) __trap();
    }
  }
};
// make a (weakly loaded) pair valid: re-read with coherent loads until both tags match (slow path out of line)
DTK_DEV u64 poll1(const u64* p, uint32_t tag) {
  Spin sp;
  for (;;) {
    const u64 w = ld_strong1(p);
    if (tag_ok(w, tag)) return w;
    sp.tick();
  }
}
DTK_DEV float settle1(u64 w, const u64* p, uint32_t tag, bool nowait) {
  if (!tag_ok(w, tag) && !nowait) w = poll1(p, tag);
  return tag_val(w);
}

// N tagged pairs per thread: weak loads first, then every pair whose tag is still old is re-read coherently, all of them per
// round (one L2 round trip per round however many are late)
template <int N>
DTK_DEV void ld_pairs(const u64* const (&ptr)[N], const bool (&on)[N], uint32_t tag, bool nowait, float2 (&out)[N]) {
  ulonglong2 w[N];
#pragma unroll
  for (int u = 0; u < N; ++u)
    if (on[u]) w[u] = ld_weak2(ptr[u]);
  Spin sp;
  for (;;) {
    bool bad[N], any = false;
#pragma unroll
    for (int u = 0; u < N; ++u) {
      bad[u] = on[u] && !(tag_ok(w[u].x, tag) && tag_ok(w[u].y, tag));
      any = any || bad[u];
    }
    if (!any || nowait) break;
    sp.tick();
#pragma unroll
    for (int u = 0; u < N; ++u)
      if (bad[u]) w[u] = ld_strong2(ptr[u]);
  }
#pragma unroll
  for (int u = 0; u < N; ++u) out[u] = on[u] ? make_float2(tag_val(w[u].x), tag_val(w[u].y)) : make_float2(0.f, 0.f);
}

// ------------------------------------------------------------------ work description
enum { PH_QKV = 0, PH_ATTN = 1, PH_O = 2, PH_GU = 3, PH_DOWN = 4, PH_LM = 5 };

// attention split: CTA c handles head c % heads, key range index c / heads (cph ranges per head)
struct AttnSplit {
  int active, head, j0, j1, last;  // keys [j0, j1) among the OLD keys [0, pos); `last` also takes key `pos`
  int cph;                         // CTAs per head
  int n_items;                     // 16-key ring items (K rows + V rows of 16 consecutive positions)
};
DTK_DEV AttnSplit attn_split(const MegaArgs& p, int c, int G, int pos) {
  AttnSplit a;
  int cph = G / p.heads;
  if (cph < 1) cph = 1;            // (heads > G is rejected on the host)
  if (cph > 16) cph = 16;
  a.cph = cph;
  a.active = c < cph * p.heads;
  a.head = c % p.heads;
  const int r = c / p.heads;
  int per = (pos + cph - 1) / cph;
  per = (per + 15) & ~15;
  a.j0 = min(pos, r * per);
  a.j1 = min(pos, a.j0 + per);
  a.last = a.active && (r == cph - 1);
  a.n_items = a.active ? (a.j1 - a.j0 + 15) / 16 : 0;
  return a;
}

// The B operand of mma.m16n8k16 for a GEMV: the input vector lives in shared memory as
// entry [kstep S][t] (uint4) = { hi(x[16S+2t], x[16S+2t+1]), hi(x[16S+2t+8], +9), lo(..2t..), lo(..2t+8..) }
// where hi = bf16(x), lo = bf16(x - hi). All 8 columns of B are the same vector, so every lane of a quad column reads
// entry t = lane & 3. Entries for k >= K (padding up to the 256-column tile) are zero.
//
// DATAFLOW STAGING: a tile (group, ks) needs only the 256-element SLICE ks of the vector, so the warp that owns
// the tile stages that slice itself, when it gets there — ONE warp: 4 tagged pairs per lane in one coalesced L2 round trip,
// re-read coherently until their tags match, converted in registers (the two halves of a B entry meet through one shuffle)
// and written straight to the entries. No CTA-wide barrier in front of a phase: a warp starts multiplying as soon as ITS
// slice has arrived, and when the slowest producer CTA of the previous phase finally publishes its rows, one warp per CTA
// has a few tiles left instead of every warp a whole phase. With norm_w the staged slice is x * w (RMSNorm gain) WITHOUT the
// 1/rms factor (the GEMV is linear: the epilogue scales by r); the slice's sum of squares goes to slice_ss[ks], and
// r = rsqrt(sum over slices / K + eps) is formed by the epilogue warp (same order in every CTA: identical r everywhere).
// The vector buffer is single: a slice may only be overwritten when every warp of the CTA is past the previous weight
// phase (phase_done counts warps x phases); the L2 round trip comes first, so that wait is normally free.
// Inlined (one call site): ptxas ignores setmaxnreg in a kernel that calls functions (C7507).
DTK_DEV void stage_slice(const u64* src, uint32_t in_tag, bool nowait, const bf16* src_bf16, int K, int ks,
                                         const bf16* norm_w, uint4* xb, float* slice_ss, volatile uint32_t* slice_tag,
                                         uint32_t my_tag) {
  const int lane = threadIdx.x & 31;
  const int npair = K >> 1;
  float2 v[4];
  uint32_t gw[4];
  bool on[4];
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int pi = ks * 128 + u * 32 + lane;
    on[u] = pi < npair;
    gw[u] = (norm_w && on[u]) ? *reinterpret_cast<const uint32_t*>(norm_w + 2 * pi) : 0u;
  }
  if (src) {
    ulonglong2 w[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (on[u]) w[u] = ld_weak2(src + 2 * (ks * 128 + u * 32 + lane));
    Spin sp;
    for (;;) {
      bool bad[4], any = false;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        bad[u] = on[u] && !(tag_ok(w[u].x, in_tag) && tag_ok(w[u].y, in_tag));
        any = any || bad[u];
      }
      if (!any || nowait) break;
      sp.tick();
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (bad[u]) w[u] = ld_strong2(src + 2 * (ks * 128 + u * 32 + lane));
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) v[u] = on[u] ? make_float2(tag_val(w[u].x), tag_val(w[u].y)) : make_float2(0.f, 0.f);
  } else {
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      v[u] = make_float2(0.f, 0.f);
      if (on[u]) {
        const uint32_t e = *reinterpret_cast<const uint32_t*>(src_bf16 + 2 * (ks * 128 + u * 32 + lane));
        v[u] = make_float2(__uint_as_float(e << 16), __uint_as_float(e & 0xffff0000u));
      }
    }
  }
  float ss = 0.f;
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    float a = v[u].x, b = v[u].y;
    if (norm_w) {
      ss += a * a + b * b;
      a *= __uint_as_float(gw[u] << 16);
      b *= __uint_as_float(gw[u] & 0xffff0000u);
    }
    const float ah = __bfloat162float(__float2bfloat16_rn(a)), bh = __bfloat162float(__float2bfloat16_rn(b));
    const uint32_t hi = pack_bf16x2(ah, bh), lo = pack_bf16x2(a - ah, b - bh);
    const uint32_t hi2 = __shfl_xor_sync(0xffffffffu, hi, 4), lo2 = __shfl_xor_sync(0xffffffffu, lo, 4);
    if (!(lane & 4)) xb[(size_t)(ks * 16 + u * 4 + (lane >> 3)) * 4 + (lane & 3)] = make_uint4(hi, hi2, lo, lo2);
  }
  if (norm_w) {
    ss = warp_sum(ss);
    if (lane == 0) slice_ss[ks] = ss;
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence_block();
    slice_tag[ks] = my_tag;
  }
  __syncwarp();
}
// r = rsqrt(mean(x^2) + eps) from the slices' sums of squares (fixed order: identical in every warp and CTA)
DTK_DEV float slices_rn(const float* slice_ss, int nslice, int K, float eps) {
  const int lane = threadIdx.x & 31;
  float t = 0.f;
  for (int i = lane; i < nslice; i += 32) t += *reinterpret_cast<const volatile float*>(slice_ss + i);
  t = warp_sum(t);
  return rsqrtf(t / K + eps);
}

// DBG = true: dev instrumentation (phase stamps, per-tile trace, timing-experiment flags) compiled in.
// HD = decoder head_dim (64 or 128): the RoPE row pairing of the qkv epilogue, the KV item rows, the attention lanes per key
// and the partial/merge scratch.
// Both roles run ONE rolled loop over the 5 L + 1 phases of the token (qkv | attention | o | gate/up | down per layer,
// then lm_head) with a single copy of the tile code and a run-time phase switch in the epilogue: the per-token
// instruction footprint of a warp stays inside the SM's 32 KB instruction cache (the fully specialised version was
// ~160 KB, re-fetched from L2 every layer: the first tiles of every phase ran 3-6x slower than the steady state).
// FMT = tile format of the weight stream. 0: bf16 tiles. 1 (F8): the four layer matrices stream as e4m3 tiles (MegaF8); the
// consumers turn each A fragment into the bf16 bits of code x 2^k_r and run the same mma sequence, so the logits equal those of
// the bf16 kernel on the dequantised weights. 2 (PK): every matrix, lm_head included, streams as packed tiles (MegaPack, 13
// bits per weight); the consumers rebuild the exact bf16 bits of the A fragments in registers: the same logits as format 0.
template <bool DBG, int HD, int FMT>
__global__ void __launch_bounds__(MEGA_THREADS, 1) decode_mega_kernel(const MegaArgs p) {
  constexpr bool F8 = FMT == 1, PK = FMT == 2;
  constexpr int HALF = HD / 2;
  constexpr int LPK = HD / 8;                // attention: lanes per key (8 bf16 each)
  constexpr int NGRP = 32 / LPK;             // key groups per warp
  constexpr int NST = NCW * NGRP;            // online-softmax states per CTA
  constexpr int PS = HD + 4;                 // per-CTA partial record: o[HD], m, l (padded)
  constexpr int PPL = HD / 64;               // (q, k, v) pairs per lane when warp 0 fetches a head's vectors
  constexpr int HSH = HD == 128 ? 7 : 6;     // log2(HD): divisions of non-negative ints as shifts
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int c = blockIdx.x, G = gridDim.x;
  const int nslots = p.nslots;
  uint8_t* ring = smem;
  float* actf = reinterpret_cast<float*>(smem + (size_t)nslots * TILE_BYTES);
  uint4* xb = reinterpret_cast<uint4*>(actf);
  uint64_t* bars = reinterpret_cast<uint64_t*>(actf + p.act_floats);
  float* red = reinterpret_cast<float*>(bars + 2 * nslots);  // 16 floats
  float* rope_s = red + 16;                                   // [HD/2][2] cos/sin of this position
  float* tpart = rope_s + 128;                                // [NT][16] per-tile partial sums
  int* gcnt = reinterpret_cast<int*>(tpart + NT * 16);        // [NG] (unused since the epilogues run behind a barrier; keeps the layout)
  float* rbuf = reinterpret_cast<float*>(gcnt + NG);          // [NG][16] residuals prefetched at a group's first tile
  float* qkn = rbuf + NG * 16;                                // [3][HD] q | new key | new value of the CTA's head
  float* slice_ss = qkn + 384;                                // [NS] sum of squares of each staged slice (normed phases)
  uint32_t* slice_tag = reinterpret_cast<uint32_t*>(slice_ss + NS);   // [NS] phase tag of the data a slice holds
  const uint32_t full0 = smem_u32(bars), empty0 = smem_u32(bars + nslots);
  const uint32_t ring_u32 = smem_u32(ring);

  if (tid == 0) {
    for (int s = 0; s < nslots; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
  }
  const int pos = p.pos[0], slot = p.slots[0];
  int tok = p.tok[0];
  if (tok < 0 || tok >= p.V) tok = 0;
  const int qd = p.heads * HD, kd = p.kv_heads * HD;
  if (tid < NS) slice_tag[tid] = (uint32_t)p.bar_base[1];   // the epoch: never a phase tag of this launch
  if (tid < HD) rope_s[tid] = p.rope_cs[(int64_t)pos * HD + tid];
  __syncthreads();
  const AttnSplit as = attn_split(p, c, G, pos);
  const int kvh = as.head / (p.heads / p.kv_heads);
  const bf16* kv_slot = p.kv + (int64_t)slot * p.kv_slot_stride;
  // shared KV prefix: positions [0, shlen) (a multiple of 16, so a 16-position ring item never straddles) live in another slot
  const int shlen = p.share_len[0];
  const bf16* kv_share = p.kv + (int64_t)p.share_slot[0] * p.kv_slot_stride;
  const int nphase = 5 * p.L + 1;

  // ---- item ownership. The CTA's local TILE sequence (all phases, in order) is dealt to agents by index:
  // local tile n -> ring slot n % nslots, producer warp n % NPW, consumer warp n % NCW (nslots is a multiple of
  // both, so a slot always has the same producer and the same consumer -> mbarrier parity waits never alias).
  struct Walk {
    uint32_t nb = 0;     // local tiles before the current phase
    uint32_t gb = 0;     // local groups before the current phase
    uint32_t rot = 0;    // rotation of the participating CTA set
  };
  // A weight phase with `groups` 16-row groups is cut into equal blocks of per = ceil(groups / G) groups; only
  // ceil(groups / per) CTAs take part (same amount of work each, so they finish together), the others idle for that
  // phase. The participating set rotates from phase to phase.
  // (per / nact come from the host and every modulo below is a conditional subtraction: no division on the per-phase path)
  auto phase_span = [&](const Walk& w, const MegaMat& m, int& g0, int& cnt, int& nact) {
    nact = m.nact;
    int ci = c + G - (int)w.rot;   // rot < G
    if (ci >= G) ci -= G;
    g0 = ci * m.per;
    cnt = (ci < nact) ? min(m.per, m.groups - g0) : 0;
  };
  // phase it -> (layer, kind, matrix index into p.mat)
  auto mat_of = [](int ph) { return ph == PH_QKV ? 0 : ph == PH_O ? 1 : ph == PH_GU ? 2 : ph == PH_DOWN ? 3 : 4; };

  if (warp >= NCW) {
    // =============================================================== PRODUCERS
    asm volatile("setmaxnreg.dec.sync.aligned.u32 56;\n");
    const uint32_t pw = (uint32_t)(warp - NCW);
    if (lane == 0) {
      // Weight tiles are read once per token and the stream (2.5 GB for ds-1.3b) is ~50x the L2: their lines are marked
      // evict_first, so the L2 drops them before lines that are read again within the token (the tagged activation words
      // every CTA polls). 3-4 % faster decode on the H100 (DESIGN.md section 9); the same policy on the key/value items was
      // slower. (mega_variant bit 0: plain copies, for A/B runs.)
      const bool evf = !(p.variant & 1);
      const uint64_t pol = policy_evict_first();
      Walk w;
      uint32_t sl = pw, use = 0;   // ring slot / use count of this lane's next tile: its tiles are n = pw, pw + NPW, ... across ALL phases
      long long* tr = nullptr;   // dev trace: row (local tile index within the traced layer), column 0 = issue clock
      uint32_t tr_nb0 = 0;
      int l = 0, ph = 0;
      for (int it = 0; it < nphase; ++it) {
        if (it == nphase - 1) { ph = PH_LM; l = 0; }
        if (DBG && ph == 0) {
          tr = (p.dbg2 && l == p.dbg_layer && it != nphase - 1) ? p.dbg2 + (int64_t)c * MEGA_DBG2_ROWS * 4 : nullptr;
          if (tr) tr_nb0 = w.nb;
        }
        // this phase's local tile list: weight tiles of the CTA's row groups, or (attention) the CTA's share of the
        // cached keys / values of the layer: item i = positions [j0 + 16 i, +16) of the CTA's kv head, K rows at slot
        // offset 0 and V rows at KV_V_OFF (rows of one head are contiguous in the cache). Neither depends on this token, so
        // both stream ahead of the dependency chain and the phases read shared memory only.
        const bool attn = ph == PH_ATTN;
        const MegaMat& m = p.mat[mat_of(ph)];
        int g0 = 0, cnt = 0, nact = 0;
        if (!attn) phase_span(w, m, g0, cnt, nact);
        const int tpg = attn ? 1 : m.tpg;
        const int ntiles = attn ? as.n_items : cnt * tpg;
        const int64_t kvo = (int64_t)l * p.kv_layer_stride + (int64_t)kvh * p.max_len * HD;
        const bf16* base = attn ? kv_slot + kvo
                                : m.base + (int64_t)l * m.layer_stride + (int64_t)g0 * tpg * MEGA_TILE_ELEMS;
        // own tiles j = j0, j0 + NPW, ...
        uint32_t j = (pw + NPW - (w.nb & (NPW - 1))) & (NPW - 1);
        MegaF8 f8{};
        uint32_t jk = 0, jks = j;   // F8: tile j = group jk of the CTA's block, k-tile jks
        if (F8) {
          if (!attn && ph != PH_LM) f8 = p.f8[mat_of(ph)];
          while (jks >= (uint32_t)tpg) { jks -= tpg; ++jk; }
        }
        if ((int)j < ntiles) {
          for (; (int)j < ntiles; j += NPW) {
            if (use > 0) mbar_wait(empty0 + 8 * sl, (use - 1) & 1);
            const uint32_t dst = ring_u32 + sl * TILE_BYTES, fb = full0 + 8 * sl;
            if (attn) {
              const int key0 = as.j0 + (int)j * 16;
              const uint32_t bytes = (uint32_t)min(16, p.max_len - key0) * (uint32_t)(HD * 2);
              const bf16* kb = (key0 < shlen ? kv_share + kvo : base) + (int64_t)key0 * HD;
              mbar_expect_tx(fb, 2 * bytes);
              bulk_g2s(dst, kb, bytes, fb);
              bulk_g2s(dst + KV_V_OFF, kb + p.kv_v_offset, bytes, fb);
            } else if (F8 && ph != PH_LM) {
              // e4m3 codes of the tile, then the row exponents of its group right behind them
              mbar_expect_tx(fb, MEGA_F8_TILE_BYTES + 16);
              const uint8_t* src = f8.tiles + (int64_t)l * f8.layer_stride + ((int64_t)g0 * tpg + j) * MEGA_F8_TILE_BYTES;
              if (evf) bulk_g2s_hint(dst, src, MEGA_F8_TILE_BYTES, fb, pol);
              else bulk_g2s(dst, src, MEGA_F8_TILE_BYTES, fb);
              bulk_g2s(dst + MEGA_F8_TILE_BYTES, f8.exps + (int64_t)l * f8.exp_stride + (int64_t)(g0 + (int)jk) * 16, 16, fb);
            } else if (PK) {
              const MegaPack& pk = p.pk[mat_of(ph)];
              const uint8_t* src = pk.tiles + (int64_t)l * pk.layer_stride + ((int64_t)g0 * tpg + j) * MEGA_PK_TILE_BYTES;
              mbar_expect_tx(fb, MEGA_PK_TILE_BYTES);
              if (evf) bulk_g2s_hint(dst, src, MEGA_PK_TILE_BYTES, fb, pol);
              else bulk_g2s(dst, src, MEGA_PK_TILE_BYTES, fb);
            } else {
              mbar_expect_tx(fb, TILE_BYTES);
              if (evf) bulk_g2s_hint(dst, base + (int64_t)j * MEGA_TILE_ELEMS, TILE_BYTES, fb, pol);
              else bulk_g2s(dst, base + (int64_t)j * MEGA_TILE_ELEMS, TILE_BYTES, fb);
            }
            if (DBG && tr) {
              const uint32_t row = w.nb + j - tr_nb0;
              if (row < 160u) tr[row * 4] = clock64();
            }
            sl += NPW;
            if (sl >= (uint32_t)nslots) { sl -= nslots; ++use; }
            if (F8) {
              jks += NPW;
              while (jks >= (uint32_t)tpg) { jks -= tpg; ++jk; }
            }
          }
        }
        w.nb += ntiles;
        if (!attn) {
          w.gb += cnt;
          w.rot += (uint32_t)nact;
          if (w.rot >= (uint32_t)G) w.rot -= G;
        }
        if (++ph == 5) { ph = 0; ++l; }
      }
    }
    return;
  }

  // ================================================================= CONSUMERS
  asm volatile("setmaxnreg.inc.sync.aligned.u32 224;\n");
  const int dflags = DBG ? p.dbg_flags : 0;
  const bool nowait = (dflags & 2) != 0;
  const int stage_pass = (p.variant & 2) ? 0 : 1;   // weight tiles: stage the input slice before (0) or after (1) reading the tile
  unsigned long long bar_target = p.bar_base[0];   // arrivals counted before this launch
  const uint32_t epoch = (uint32_t)p.bar_base[1];  // tag of phase it = epoch + it + 1
  Walk w;
  uint32_t sl = (uint32_t)warp, use = 0;   // ring slot / use count of this warp's next tile or item: n = warp, warp + NCW, ... across ALL phases
  uint32_t cur_slot = 0;
  auto release = [&]() {   // hand the ring slot back: every lane's shared-memory reads of it are issued, the arrive is ordered after them
    __syncwarp();
    if (lane == 0) mbar_arrive(empty0 + 8 * cur_slot);
  };
  // optional phase timestamps (globaltimer ns, comparable across SMs): [CTA][phase][4] = {start, staged, items done, barrier done}
  long long* dbg = (DBG && p.dbg) ? p.dbg + (int64_t)c * nphase * 4 : nullptr;
  long long* ctr = nullptr;   // dev trace of one layer (see MegaArgs::dbg2)
  uint32_t ctr_nb0 = 0;
  int it = 0, l = 0, ph = 0;
  auto stamp = [&](int k) {
    if (!DBG) return;
    if (dbg && tid == 0) {
      unsigned long long t;
      asm volatile("mov.u64 %0, %%globaltimer;\n" : "=l"(t));
      dbg[it * 4 + k] = (long long)t;
    }
    if (ctr && tid == 0 && ph < 5) ctr[(160 + ph) * 4 + k] = clock64();
  };

  // tagged cross-CTA vectors (MegaArgs::tg): residual stream after attention (xa) / after the MLP (xb), q, the new
  // key and value rows, merged attention output, SwiGLU vector, per-CTA attention partials
  u64* const t_xa = p.tg;
  u64* const t_xb = t_xa + p.tg_H;
  u64* const t_q = t_xb + p.tg_H;
  u64* const t_kn = t_q + qd;
  u64* const t_vn = t_kn + kd;
  u64* const t_att = t_vn + kd;
  u64* const t_h = t_att + qd;
  u64* const t_part = t_h + p.tg_I;

  float best_v = -INFINITY;   // greedy tail: this thread's best (logit, index) over the lm_head rows it finished
  int best_i = 0x7fffffff;
  for (it = 0; it < nphase; ++it) {
    if (it == nphase - 1) { ph = PH_LM; l = 0; }
    const uint32_t tag = epoch + (uint32_t)it + 1u;   // tags of this phase's outputs; its inputs carry tag - 1
    if (DBG && ph == 0) {
      ctr = (p.dbg2 && l == p.dbg_layer && it != nphase - 1) ? p.dbg2 + (int64_t)c * MEGA_DBG2_ROWS * 4 : nullptr;
      ctr_nb0 = w.nb;
    }
    stamp(0);
    if (ph == PH_ATTN) {
      // ---------------- attention over this CTA's key range of its head. No grid-wide wait in front of it: the cached
      // keys/values arrive through the ring, and q / the new key and value are polled (by one warp) as tagged words of
      // this head only.
      if (as.active) {
        const int hw = lane >> (HSH - 3), l16 = lane & (LPK - 1);   // key group of the lane, lane inside the group
        if (warp == 0) {   // one warp fetches q (and, in the head's last key range, the new key / value row): HD/2 pairs each
          // head_dim^-1/2 * log2(e)
          const float sl2 = (HD == 128 ? 0.08838834764831845f : 0.125f) * 1.4426950408889634f;
          float2* q2 = reinterpret_cast<float2*>(qkn);
          const bool lastr = as.last != 0;
          const u64* ptr[3 * PPL];
          bool on[3 * PPL];
#pragma unroll
          for (int u = 0; u < PPL; ++u) {
            ptr[u] = t_q + as.head * HD + 2 * (lane + 32 * u);
            ptr[PPL + u] = t_kn + kvh * HD + 2 * (lane + 32 * u);
            ptr[2 * PPL + u] = t_vn + kvh * HD + 2 * (lane + 32 * u);
            on[u] = true;
            on[PPL + u] = lastr;
            on[2 * PPL + u] = lastr;
          }
          float2 v[3 * PPL];
          ld_pairs<3 * PPL>(ptr, on, tag - 1, nowait, v);
#pragma unroll
          for (int u = 0; u < PPL; ++u) {
            q2[lane + 32 * u] = make_float2(v[u].x * sl2, v[u].y * sl2);
            if (lastr) { q2[HALF + lane + 32 * u] = v[PPL + u]; q2[HD + lane + 32 * u] = v[2 * PPL + u]; }
          }
        }
        consumer_sync();   // q is staged; every warp is past its last qkv tile (the merge scratch below aliases the staged vector)
        stamp(1);
        float q[8];
        {
          const float4 a = *reinterpret_cast<const float4*>(qkn + l16 * 8), b = *reinterpret_cast<const float4*>(qkn + l16 * 8 + 4);
          q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
        }
        float m = -INFINITY, lsum = 0.f, o[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) o[i] = 0.f;
        // online softmax over FOUR keys at a time (per key group): the four dot products and their shuffle reductions are
        // independent chains, one rescale per batch instead of one per key
        auto keys4 = [&](const uint4 (&kr)[4], const uint4 (&vr)[4], const bool (&valid)[4]) {
          float s2[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            float kf[8];
            unpack8(kr[u], kf);
            float d = 0.f;
#pragma unroll
            for (int i = 0; i < 8; ++i) d += q[i] * kf[i];
            s2[u] = d;
          }
#pragma unroll
          for (int st = LPK / 2; st > 0; st >>= 1)
#pragma unroll
            for (int u = 0; u < 4; ++u) s2[u] += __shfl_xor_sync(0xffffffffu, s2[u], st);
          float mx = m;
#pragma unroll
          for (int u = 0; u < 4; ++u) { s2[u] = valid[u] ? s2[u] : -INFINITY; mx = fmaxf(mx, s2[u]); }
          if (mx == -INFINITY) return;           // nothing valid so far
          const float alpha = exp2f(m - mx);      // m = -inf -> 0
          float pj[4], ps = 0.f;
#pragma unroll
          for (int u = 0; u < 4; ++u) { pj[u] = exp2f(s2[u] - mx); ps += pj[u]; }
          lsum = lsum * alpha + ps;
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] *= alpha;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (valid[u]) {   // (positions past the range may hold uninitialised cache memory: 0 * NaN must not reach o)
              float vf[8];
              unpack8(vr[u], vf);
#pragma unroll
              for (int i = 0; i < 8; ++i) o[i] += pj[u] * vf[i];
            }
          }
          m = mx;
        };
        // ring items: 16 positions each; key group hw takes positions hw, hw + NGRP, ... of the item (16 / NGRP / 4 batches of 4)
        {
          uint32_t j = ((uint32_t)warp + NCW - (w.nb & (NCW - 1))) & (NCW - 1);
          if ((int)j < as.n_items) {
            for (; (int)j < as.n_items; j += NCW) {
              long long* trow = nullptr;
              if (DBG && ctr) {
                const uint32_t row = w.nb + j - ctr_nb0;
                if (row < 160u) trow = ctr + row * 4;
              }
              if (DBG && trow && lane == 0) trow[3] = clock64();
              mbar_wait(full0 + 8 * sl, use & 1);
              if (DBG && trow && lane == 0) trow[1] = clock64();
              cur_slot = sl;
              const uint32_t base = ring_u32 + sl * TILE_BYTES + l16 * 16;
              const int key0 = as.j0 + (int)j * 16;
              constexpr int KPG = 16 / NGRP;   // positions of the item per key group
              uint4 kr[KPG / 4][4], vr[KPG / 4][4];
#pragma unroll
              for (int u = 0; u < KPG; ++u) {
                const uint32_t a = base + (uint32_t)(u * NGRP + hw) * (uint32_t)(HD * 2);
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(kr[u >> 2][u & 3].x), "=r"(kr[u >> 2][u & 3].y), "=r"(kr[u >> 2][u & 3].z), "=r"(kr[u >> 2][u & 3].w) : "r"(a));
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(vr[u >> 2][u & 3].x), "=r"(vr[u >> 2][u & 3].y), "=r"(vr[u >> 2][u & 3].z), "=r"(vr[u >> 2][u & 3].w) : "r"(a + (uint32_t)KV_V_OFF));
              }
              release();
#pragma unroll
              for (int h = 0; h < KPG / 4; ++h) {
                const bool valid[4] = {key0 + (h * 4 + 0) * NGRP + hw < as.j1, key0 + (h * 4 + 1) * NGRP + hw < as.j1,
                                       key0 + (h * 4 + 2) * NGRP + hw < as.j1, key0 + (h * 4 + 3) * NGRP + hw < as.j1};
                keys4(kr[h], vr[h], valid);
              }
              if (DBG && trow && lane == 0) trow[2] = clock64();
              sl += NCW;
              if (sl >= (uint32_t)nslots) { sl -= nslots; ++use; }
            }
          }
          w.nb += as.n_items;
        }
        if (as.last && warp == 0 && hw == 0) {   // the key / value of the token being decoded (published by the qkv phase of this launch)
          float d = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) d += q[i] * qkn[HD + l16 * 8 + i];
#pragma unroll
          for (int st = LPK / 2; st > 0; st >>= 1) d += __shfl_xor_sync((1u << LPK) - 1u, d, st);
          const float mx = fmaxf(m, d), alpha = exp2f(m - mx), pj = exp2f(d - mx);
          lsum = lsum * alpha + pj;
#pragma unroll
          for (int i = 0; i < 8; ++i) o[i] = o[i] * alpha + pj * qkn[2 * HD + l16 * 8 + i];
          m = mx;
        }
        // merge the NST key-group states -> one partial per CTA
        float* sm_m = actf;              // [NST]
        float* sm_l = actf + NST;        // [NST]
        float* sm_o = actf + 2 * NST;    // [NST][HD]
        const int hidx = warp * NGRP + hw;
        if (l16 == 0) { sm_m[hidx] = m; sm_l[hidx] = lsum; }
#pragma unroll
        for (int i = 0; i < 8; ++i) sm_o[hidx * HD + l16 * 8 + i] = o[i];
        consumer_sync();
        const bool owner = c < p.heads;   // the CTA of the head's first key range folds the head's partials
        float* mg = sm_o + NST * HD;      // [cph][PS] (owner only)
        if (tid < HD) {
          float M = -INFINITY;
#pragma unroll
          for (int h = 0; h < NST; ++h) M = fmaxf(M, sm_m[h]);
          float Lt = 0.f, O = 0.f;
#pragma unroll
          for (int h = 0; h < NST; ++h) {
            const float wgt = (sm_m[h] == -INFINITY) ? 0.f : exp2f(sm_m[h] - M);
            Lt += sm_l[h] * wgt;
            O += sm_o[h * HD + tid] * wgt;
          }
          if (owner) {
            mg[tid] = O;
            if (tid == 0) { mg[HD] = M; mg[HD + 1] = Lt; }
          } else {
            u64* pp = t_part + (int64_t)c * PS;
            st_tag(pp + tid, O, tag);
            if (tid == 0) { st_tag(pp + HD, M, tag); st_tag(pp + HD + 1, Lt, tag); }
          }
        }
        if (owner) {
          // fixed owner instead of "last CTA to arrive": no atomic round trip on the critical path; the partials are tagged,
          // the owner polls them (coalesced, with back-off) as soon as its own share is done
          constexpr int PW = HD + 2;   // words of a partial record
          const int nw = (as.cph - 1) * PW;
          for (int i0 = 0; i0 < nw; i0 += 2 * CONSUMER_THREADS) {
            u64 wv2[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int i = i0 + u * CONSUMER_THREADS + tid;
              if (i < nw) wv2[u] = ld_weak1(t_part + (int64_t)((i / PW + 1) * p.heads + as.head) * PS + (i % PW));
            }
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              const int i = i0 + u * CONSUMER_THREADS + tid;
              if (i < nw) mg[(i / PW + 1) * PS + (i % PW)] = settle1(wv2[u], t_part + (int64_t)((i / PW + 1) * p.heads + as.head) * PS + (i % PW), tag, nowait);
            }
          }
          consumer_sync();
          if (tid < HD) {
            float M = -INFINITY;
            for (int r = 0; r < as.cph; ++r) M = fmaxf(M, mg[r * PS + HD]);
            float Lt = 0.f, O = 0.f;
#pragma unroll 1
            for (int r = 0; r < as.cph; ++r) {
              const float mr = mg[r * PS + HD];
              const float wgt = (mr == -INFINITY) ? 0.f : exp2f(mr - M);
              Lt += mg[r * PS + HD + 1] * wgt;
              O += mg[r * PS + tid] * wgt;
            }
            st_tag(t_att + as.head * HD + tid, O / Lt, tag);
          }
        }
      } else {
        stamp(1);
      }
      stamp(2);
    } else {
      // ---------------- weight phase: multiply the CTA's row groups (each warp stages the input slices of its own tiles), fused epilogue
      const MegaMat& m = p.mat[mat_of(ph)];
      int g0, cnt, nact;
      phase_span(w, m, g0, cnt, nact);
      const int tpg = m.tpg;
      const int64_t no = (int64_t)l * p.norm_stride;
      const u64* src = ph == PH_QKV ? (l == 0 ? nullptr : t_xb) : ph == PH_O ? t_att : ph == PH_GU ? t_xa : ph == PH_DOWN ? t_h : t_xb;
      const int K = ph == PH_O ? qd : ph == PH_DOWN ? p.I : p.H;
      const bf16* nw = ph == PH_QKV ? p.norm1_0 + no : ph == PH_GU ? p.norm2_0 + no : ph == PH_LM ? p.final_norm : nullptr;
      float rn = 0.f;   // RMSNorm scale of this phase's input: formed by the first epilogue this warp runs (0 = not yet)
      stamp(1);
      const uint32_t nb0 = w.nb, gb0 = w.gb;
      // residual source of the O / DOWN epilogues: the row's previous value in the other residual buffer
      const u64* res_src = (ph == PH_O) ? t_xb : t_xa;
      const uint32_t res_tag = (ph == PH_O) ? tag - 3 : tag - 2;   // O: x after the previous layer's MLP; DOWN: this layer's xa
      const int ntiles = cnt * tpg;
      uint32_t j = ((uint32_t)warp + NCW - (nb0 & (NCW - 1))) & (NCW - 1);
      // The warps walk their tiles in ROUNDS (tile j + 8 r in round r) and meet every sync_every rounds: a ring slot belongs
      // to one consumer warp, so nothing else stops a warp from running many groups ahead of another one, and a warp that
      // gets NT tiles ahead would overwrite its own partial sums of a group whose epilogue has not run yet (seen at the
      // v2-8b shape: 880 lm_head tiles per CTA, scattered wrong logits). The interval is as long as the windows allow:
      // drift (interval rounds) + one group + the round in flight <= NT partial sums, groups in flight <= NG / 2.
      // (QKV -> attention has no barrier in between, but the attention phase writes no partial sums.)
      const int rounds = (ntiles + NCW - 1) / NCW;
      const int sync_every = max(1, min((NT - tpg - 2 * NCW) / NCW, NG * tpg / (2 * NCW)));
      int since_sync = 0;
      // ---- group epilogues. They do NOT run inside the tile loop: with "the warp that finishes a group's last tile runs its
      // epilogue" the warp that is last in one round starts its next tile late, is last again, and ends up with ALL epilogues of
      // the phase in series. The
      // tiles only leave their partial sums in shared memory; after a CTA barrier the complete groups are dealt to the warps
      // (warp w: groups k_ep + w, + 8, ...) and run in parallel — no per-tile counter, atomic or fence either. Partials are
      // summed in k order (deterministic).
      uint32_t k_ep = 0;   // groups of this phase whose epilogue has run
      auto run_epilogues = [&](uint32_t k_hi) {
        for (uint32_t ek = k_ep + (uint32_t)warp; ek < k_hi; ek += NCW) {
          const uint32_t egs = (gb0 + ek) % NG;
              const uint32_t n0 = nb0 + ek * tpg;
              float v = 0.f;
              if (lane < 16)
                for (int t = 0; t < tpg; ++t) v += tpart[((n0 + t) % NT) * 16 + lane];
              const float v1 = __shfl_down_sync(0xffffffffu, v, 8);
              if (nw && rn == 0.f) rn = slices_rn(slice_ss, tpg, K, p.eps);   // (every slice of the vector is staged: the group is complete)
              if (lane < 8) {
                const int gi = g0 + (int)ek, r = lane;
                if (ph == PH_QKV) {
                  constexpr int GPH = HALF / 8;                          // 16-row groups per head
                  const int hb = gi >> (HSH - 4), i = ((gi & (GPH - 1)) << 3) + r;   // HD-row head block, index inside the half
                  const int row0 = hb * HD + i;
                  const float a0 = v * rn, a1 = v1 * rn;
                  if (row0 < qd + kd) {
                    const float2 csn = *reinterpret_cast<const float2*>(rope_s + i * 2);
                    const float y0 = a0 * csn.x - a1 * csn.y, y1 = a1 * csn.x + a0 * csn.y;
                    if (row0 < qd) { st_tag(t_q + row0, y0, tag); st_tag(t_q + row0 + HALF, y1, tag); }
                    else {
                      const int kh = (row0 - qd) >> HSH;
                      bf16* dd = p.kv + (int64_t)slot * p.kv_slot_stride + (int64_t)l * p.kv_layer_stride + ((int64_t)kh * p.max_len + pos) * HD;
                      const bf16 z0 = __float2bfloat16_rn(y0), z1 = __float2bfloat16_rn(y1);
                      dd[i] = z0;
                      dd[i + HALF] = z1;
                      st_tag(t_kn + kh * HD + i, __bfloat162float(z0), tag);      // the cache row as this launch's attention reads it
                      st_tag(t_kn + kh * HD + i + HALF, __bfloat162float(z1), tag);
                    }
                  } else {
                    const int kh = (row0 - qd - kd) >> HSH;
                    bf16* dd = p.kv + (int64_t)slot * p.kv_slot_stride + (int64_t)l * p.kv_layer_stride + p.kv_v_offset + ((int64_t)kh * p.max_len + pos) * HD;
                    const bf16 z0 = __float2bfloat16_rn(a0), z1 = __float2bfloat16_rn(a1);
                    dd[i] = z0;
                    dd[i + HALF] = z1;
                    st_tag(t_vn + kh * HD + i, __bfloat162float(z0), tag);
                    st_tag(t_vn + kh * HD + i + HALF, __bfloat162float(z1), tag);
                  }
                } else if (ph == PH_O || ph == PH_DOWN) {
                  u64* dst = (ph == PH_O) ? t_xa : t_xb;
                  const int r0 = gi * 16 + r, r1 = r0 + 8;
                  const float b0 = rbuf[egs * 16 + r], b1 = rbuf[egs * 16 + r + 8];
                  if (r0 < p.H) st_tag(dst + r0, b0 + v, tag);
                  if (r1 < p.H) st_tag(dst + r1, b1 + v1, tag);
                } else if (ph == PH_GU) {
                  const int i = gi * 8 + r;
                  if (i < p.I) st_tag(t_h + i, silu(v * rn) * (v1 * rn), tag);
                } else {
                  const int r0 = gi * 16 + r, r1 = r0 + 8;
                  const float l0 = v * rn, l1 = v1 * rn;
                  if (r0 < p.V) p.logits[r0] = l0;
                  if (r1 < p.V) p.logits[r1] = l1;
                  if (p.fuse_greedy) {   // rows are visited in increasing order per thread: '>' keeps the lowest index on ties
                    if (r0 < p.V && r0 != p.bad_token && l0 > best_v) { best_v = l0; best_i = r0; }
                    if (r1 < p.V && r1 != p.bad_token && l1 > best_v) { best_v = l1; best_i = r1; }
                  }
                }
              }
        }
        k_ep = k_hi;
      };
      {
        uint32_t k = 0, ks = j;
        while (ks >= (uint32_t)tpg) { ks -= tpg; ++k; }
        for (int rd = 0; rd <= rounds; ++rd) {
          // a meeting point: every sync_every rounds (partial-sum window) and once after the last round (rd == rounds). All tiles
          // j < 8 rd are done: the groups they complete get their epilogues (ONE call site: the epilogue code exists once).
          const bool at_end = rd == rounds;
          if (at_end || ++since_sync > sync_every) {
            consumer_sync();
            run_epilogues(at_end ? (uint32_t)cnt : (uint32_t)(NCW * rd) / (uint32_t)tpg);
            since_sync = 1;
          }
          if (at_end) break;
          if ((int)j >= ntiles) { j += NCW; continue; }
          long long* trow = nullptr;
          if (DBG && ctr) {
            const uint32_t row = nb0 + j - ctr_nb0;
            if (row < 160u) trow = ctr + row * 4;
          }
          if (DBG && trow && lane == 0) trow[3] = clock64();
          // ---- one tile = 16 k-steps of mma.m16n8k16. The warp first waits for the tile, reads it and hands the slot back,
          // rebuilds the A fragments of all 16 k-steps in registers (ldmatrix for bf16 tiles; the FP8 or packed conversion),
          // and only then stages the tile's slice of the input vector if it is not staged yet (normally this very warp staged
          // it at its previous tile of the same ks; at the warp's first tile of a phase the staging polls the previous phase's
          // output, the cross-CTA hop). So the slot is free for the producer during the hop and the conversion runs while the
          // warp would otherwise wait for its input: after the hop only the B loads and the mma chain remain.
          // (mega_variant bit 1: stage first, as earlier builds did; the same results, for A/B runs.)
          uint32_t A[16][4];
#pragma unroll 1
          for (int pass = 0; pass < 2; ++pass) {
            if (pass == stage_pass && *reinterpret_cast<volatile uint32_t*>(slice_tag + ks) != tag)
              stage_slice(src, tag - 1, nowait, p.embed + (int64_t)tok * p.H, K, (int)ks, nw, xb, slice_ss, slice_tag, tag);
            if (pass == 1) break;
            mbar_wait(full0 + 8 * sl, use & 1);
            if (DBG && trow && lane == 0) trow[1] = clock64();
            cur_slot = sl;
            const uint32_t tb = ring_u32 + sl * TILE_BYTES;
            if (F8 && ph != PH_LM) {
              // ---- e4m3 tile: [kstep pair][lane][16 B] = this lane's A fragments of two k-steps, converted in registers to the
              // bf16 bits of code x 2^k_r (rows g and g + 8 of the group: one scale each)
              uint4 q[8];
#pragma unroll
              for (int s = 0; s < 8; ++s)
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(q[s].x), "=r"(q[s].y), "=r"(q[s].z), "=r"(q[s].w) : "r"(tb + lane * 16 + s * 512));
              int e0, e1;
              asm volatile("ld.shared.s8 %0, [%1];\n" : "=r"(e0) : "r"(tb + MEGA_F8_TILE_BYTES + (lane >> 2)));
              asm volatile("ld.shared.s8 %0, [%1];\n" : "=r"(e1) : "r"(tb + MEGA_F8_TILE_BYTES + 8 + (lane >> 2)));
              release();
              const float s0 = pow2f(e0), s1 = pow2f(e1);
              if (!(dflags & 1)) {
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                  A[2 * s][0] = e4m3x2_to_bf16x2(q[s].x, s0);
                  A[2 * s][1] = e4m3x2_to_bf16x2(q[s].x >> 16, s1);
                  A[2 * s][2] = e4m3x2_to_bf16x2(q[s].y, s0);
                  A[2 * s][3] = e4m3x2_to_bf16x2(q[s].y >> 16, s1);
                  A[2 * s + 1][0] = e4m3x2_to_bf16x2(q[s].z, s0);
                  A[2 * s + 1][1] = e4m3x2_to_bf16x2(q[s].z >> 16, s1);
                  A[2 * s + 1][2] = e4m3x2_to_bf16x2(q[s].w, s0);
                  A[2 * s + 1][3] = e4m3x2_to_bf16x2(q[s].w >> 16, s1);
                }
              }
            } else if (PK) {
              // ---- packed tile (MegaPack): byte i of word k of kstep pair s is sign | mantissa7 of one value (the e4m3 codes'
              // order: word k = kstep 2 s + (k >> 1), bytes 0-1 in row g, bytes 2-3 in row g + 8); its exponent is the row base
              // plus a 5-bit code (nibble plane + high-bit plane), or in an escape tile the biased exponent itself (side buffer)
              uint4 q[8], nb[4], hb;
#pragma unroll
              for (int s = 0; s < 8; ++s)
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(q[s].x), "=r"(q[s].y), "=r"(q[s].z), "=r"(q[s].w) : "r"(tb + lane * 16 + s * 512));
#pragma unroll
              for (int s = 0; s < 4; ++s)
                asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(nb[s].x), "=r"(nb[s].y), "=r"(nb[s].z), "=r"(nb[s].w) : "r"(tb + MEGA_PK_NIB + lane * 16 + s * 512));
              asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];\n" : "=r"(hb.x), "=r"(hb.y), "=r"(hb.z), "=r"(hb.w) : "r"(tb + MEGA_PK_HB + lane * 16));
              uint32_t r0, r1;
              int ei;
              asm volatile("ld.shared.u8 %0, [%1];\n" : "=r"(r0) : "r"(tb + MEGA_PK_HDR + (lane >> 2)));
              asm volatile("ld.shared.u8 %0, [%1];\n" : "=r"(r1) : "r"(tb + MEGA_PK_HDR + 8 + (lane >> 2)));
              asm volatile("ld.shared.s32 %0, [%1];\n" : "=r"(ei) : "r"(tb + MEGA_PK_HDR + 16));
              release();
              if (!(dflags & 1)) {
                uint32_t ex[8][4];   // the exponent byte of every value, four per word of q
                if (ei < 0) {
                  // code of byte i of word k of kstep pair s: nibble i of nibble word k >> 1 (low / high half by k & 1), bit
                  // 8 i + 4 (s & 1) + k of high-bit word s >> 1. Code <= 31 and base <= 224: one add for the four bytes (no carry)
                  const uint32_t bb = r0 * 0x00000101u + r1 * 0x01010000u;
#pragma unroll
                  for (int s = 0; s < 8; ++s) {
                    const uint32_t n0 = (s & 1) ? nb[s >> 1].z : nb[s >> 1].x, n1 = (s & 1) ? nb[s >> 1].w : nb[s >> 1].y;
                    const uint32_t hw = (s >> 1) == 0 ? hb.x : (s >> 1) == 1 ? hb.y : (s >> 1) == 2 ? hb.z : hb.w;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                      const int t = 4 * (s & 1) + k;   // the code's high bit goes from bit 8 i + t to bit 8 i + 4
                      const uint32_t hs = t >= 4 ? hw >> (t - 4) : hw << (4 - t);
                      ex[s][k] = ((((k >> 1) ? n1 : n0) >> (4 * (k & 1)) & 0x0F0F0F0Fu) | (hs & 0x10101010u)) + bb;
                    }
                  }
                } else {
                  const uint4* ep = reinterpret_cast<const uint4*>(p.pk_esc + (int64_t)ei * MEGA_PK_ESC_BYTES) + lane;
#pragma unroll
                  for (int s = 0; s < 8; ++s) {
                    const uint4 e = __ldg(ep + s * 32);
                    ex[s][0] = e.x; ex[s][1] = e.y; ex[s][2] = e.z; ex[s][3] = e.w;
                  }
                }
                // bf16 value = hi byte (sign | exponent >> 1) : lo byte (exponent bit 0 | mantissa7); two prmt interleave
                // the four values' bytes into the A registers of rows g (bytes 0-1) and g + 8 (bytes 2-3)
#pragma unroll
                for (int s = 0; s < 8; ++s) {
                  const uint32_t w[4] = {q[s].x, q[s].y, q[s].z, q[s].w};
#pragma unroll
                  for (int k = 0; k < 4; ++k) {
                    uint32_t lo, hi;   // bit select (c ? a : b): one lop3 each
                    asm("lop3.b32 %0, %1, %2, 0x7F7F7F7F, 0xE4;\n" : "=r"(lo) : "r"(w[k]), "r"(ex[s][k] << 7));
                    asm("lop3.b32 %0, %1, %2, 0x80808080, 0xE4;\n" : "=r"(hi) : "r"(w[k]), "r"(ex[s][k] >> 1));
                    uint32_t* a = A[2 * s + (k >> 1)] + 2 * (k & 1);
                    asm("prmt.b32 %0, %1, %2, 0x5140;\n" : "=r"(a[0]) : "r"(lo), "r"(hi));
                    asm("prmt.b32 %0, %1, %2, 0x7362;\n" : "=r"(a[1]) : "r"(lo), "r"(hi));
                  }
                }
              }
            } else {
#pragma unroll
              for (int s = 0; s < 16; ++s) ldmatrix_x4(A[s][0], A[s][1], A[s][2], A[s][3], tb + lane * 16 + s * 512);
              release();
            }
          }
          // B operand: even columns of the 16 x 8 B tile carry the hi part of x, odd columns the lo part (column = lane >> 2), so
          // ONE mma per k-step yields W.hi in accumulator column 0 and W.lo in column 1; even k-steps go to acc, odd ones to c1
          float rA0 = 0.f, rA2 = 0.f;
          if (!(dflags & 1)) {
            const uint2* xp = reinterpret_cast<const uint2*>(xb + (size_t)ks * 64 + (lane & 3)) + ((lane >> 2) & 1);
            float acc[4] = {0.f, 0.f, 0.f, 0.f}, c1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int s = 0; s < 16; s += 2) {
              const uint2 b0 = xp[8 * s], b1 = xp[8 * s + 8];
              mma_bf16_16816(acc, A[s], b0.x, b0.y);
              mma_bf16_16816(c1, A[s + 1], b1.x, b1.y);
            }
            // lanes with (lane & 3) == 0 hold columns 0 (hi) and 1 (lo) of rows g (c[0], c[1]) and g + 8 (c[2], c[3])
            rA0 = (acc[0] + c1[0]) + (acc[1] + c1[1]);
            rA2 = (acc[2] + c1[2]) + (acc[3] + c1[3]);
          }
          const uint32_t gsA = (gb0 + k) % NG;
          if ((ph == PH_O || ph == PH_DOWN) && lane < 16 && ks == 0) {
            // residual of row (group, lane), fetched at the group's FIRST tile so that its L2 latency is off the
            // critical path of the group's epilogue (the value was published two or more phases ago)
            const int row = (g0 + (int)k) * 16 + lane;
            float bres = 0.f;
            if (row < p.H)
              bres = (ph == PH_O && l == 0) ? __bfloat162float(p.embed[(int64_t)tok * p.H + row])
                                            : settle1(ld_weak1(res_src + row), res_src + row, res_tag, nowait);
            rbuf[gsA * 16 + lane] = bres;
          }
          if ((lane & 3) == 0) {
            float* tp = tpart + ((nb0 + j) % NT) * 16;
            tp[lane >> 2] = rA0;
            tp[(lane >> 2) + 8] = rA2;
          }
          if (DBG && trow && lane == 0) trow[2] = clock64();
          j += NCW;
          sl += NCW;
          if (sl >= (uint32_t)nslots) { sl -= nslots; ++use; }
          ks += NCW;
          while (ks >= (uint32_t)tpg) { ks -= tpg; ++k; }
        }
      }
      w.nb += ntiles;
      w.gb += cnt;
      w.rot += (uint32_t)nact;
      if (w.rot >= (uint32_t)G) w.rot -= G;
      stamp(2);
    }
    // Phase boundary: a CTA-wide barrier only (none after qkv: the attention phase meets after polling its head's q; none
    // after lm_head). No grid-wide arrival counter: the next phase's warps poll the tagged words of their own slices.
    // The CTA barrier is what allows the single
    // vector buffer (slices are overwritten by the next phase; the attention merge scratch aliases it).
    if (ph != PH_QKV && ph != PH_LM) consumer_sync();
    stamp(3);
    if (++ph == 5) { ph = 0; ++l; }
  }
  if (p.fuse_greedy) {
    // ---- greedy tail (HF argmax after NoBadWords; lowest index wins ties): CTA-local argmax, one 64-bit atomicMax per CTA
    // on {order-preserving logit bits, ~index}; the last CTA to arrive publishes the token exactly as the sampler does
    // (device state of the loop + ONE 8-byte store to the mapped host ring) — no second launch per token.
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best_v, o);
      const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
      if (ov > best_v || (ov == best_v && oi < best_i)) { best_v = ov; best_i = oi; }
    }
    int* red_i = reinterpret_cast<int*>(red + 8);
    consumer_sync();   // every warp has read the final norm's partial sums out of `red`
    if (lane == 0) { red[warp] = best_v; red_i[warp] = best_i; }
    consumer_sync();
    if (tid == 0) {
      for (int wv = 1; wv < NCW; ++wv)
        if (red[wv] > best_v || (red[wv] == best_v && red_i[wv] < best_i)) { best_v = red[wv]; best_i = red_i[wv]; }
      uint32_t u = __float_as_uint(best_v);
      u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
      const unsigned long long key = ((unsigned long long)u << 32) | (unsigned long long)(0xffffffffu - (uint32_t)best_i);
      atomicMax(p.amax, key);
      unsigned long long prev;
      asm volatile("atom.acq_rel.gpu.global.add.u64 %0, [%1], 1;\n" : "=l"(prev) : "l"(p.amax + 1) : "memory");
      if (prev == (unsigned long long)G - 1ull) {
        const unsigned long long best = atomicExch(p.amax, 0ull);
        const int token = (int)(0xffffffffu - (uint32_t)(best & 0xffffffffull));
        const unsigned long long gstep = *p.gen_step;
        p.gen_tok[0] = token;
        p.gen_pos[0] = min(pos + 1, p.max_pos);
        const unsigned long long entry = ((gstep + 1ull) << 32) | (unsigned long long)(unsigned)token;
        asm volatile("st.relaxed.sys.global.u64 [%0], %1;\n" ::"l"(p.host_ring + (gstep % (unsigned long long)p.ring)), "l"(entry) : "memory");
        *p.gen_step = gstep + 1ull;
        p.amax[1] = 0ull;
      }
    }
  }
  // publish the arrival count and the tag epoch for the next launch (stream-ordered): every CTA made 4L arrivals and
  // the launch used tags epoch + 1 .. epoch + 5L + 1
  if (c == 0 && tid == 0 && !(dflags & 2)) {
    p.bar_base[0] = bar_target;
    p.bar_base[1] = (unsigned long long)(uint32_t)(epoch + (uint32_t)nphase);
  }
}

// ------------------------------------------------------------------ one-time weight re-tiling
// dst chunk q (16 B) = tile (group, ks) -> [kstep s][matrix m][row r]: rows-half = m & 1, k-half = m >> 1; rows in the
// order of tile_row (fp8.cuh)
__global__ void __launch_bounds__(256) retile_kernel(const bf16* __restrict__ src, int N, int K, int mode, int hd, int groups,
                                                     int tpg, bf16* __restrict__ dst) {
  const int64_t q = (int64_t)blockIdx.x * 256 + threadIdx.x;
  const int64_t total = (int64_t)groups * tpg * 512;
  if (q >= total) return;
  const int r = (int)(q & 7), m = (int)((q >> 3) & 3), s = (int)((q >> 5) & 15);
  const int64_t tile = q >> 9;
  const int ks = (int)(tile % tpg), gi = (int)(tile / tpg);
  const int ar = (m & 1) * 8 + r;                      // A-operand row 0..15
  const int col = ks * 256 + s * 16 + (m >> 1) * 8;
  const int row = tile_row(mode, hd, gi, ar);
  uint4 v = make_uint4(0, 0, 0, 0);
  if (row < N && col < K) v = *reinterpret_cast<const uint4*>(src + (int64_t)row * K + col);
  *reinterpret_cast<uint4*>(dst + q * 8) = v;
}

// FP8 tiles, step 1: one warp per tile row derives k_r and counts the row's values that are not e4m3 x 2^k_r
__global__ void __launch_bounds__(256) f8_rows_kernel(const bf16* __restrict__ src, int N, int K, int mode, int hd, int groups,
                                                      int8_t* __restrict__ exps, unsigned int* bad) {
  const int tr = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (tr >= groups * 16) return;
  const int row = tile_row(mode, hd, tr >> 4, tr & 15);
  const bf16* w = src + (int64_t)row * K;
  float amax = 0.f;
  if (row < N)
    for (int i = lane; i < K; i += 32) amax = fmaxf(amax, fabsf(__bfloat162float(w[i])));   // (fmaxf drops NaN: checked below)
  amax = warp_max(amax);
  int k = 0;
  if (amax > 0.f && isfinite(amax)) {
    int e;
    const float f = frexpf(amax, &e);   // amax = f 2^e, f in [0.5, 1); 448 = 0.875 2^9: amax <= 448 2^k  <=>  k >= e - 9 (+1 if f > 0.875)
    k = max(e - 9 + (f > 0.875f ? 1 : 0), -117);
  }
  unsigned int nbad = 0;
  if (row < N) {
    const float inv = pow2f(-k);
    for (int i = lane; i < K; i += 32) {
      const float v = __bfloat162float(w[i]) * inv;
      if (!(e4m3x2_to_float2(float2_to_e4m3x2(v, 0.f)).x == v)) ++nbad;   // NaN, inf and values off the e4m3 grid
    }
  }
  nbad = __reduce_add_sync(0xffffffffu, nbad);
  if (lane == 0) {
    exps[tr] = (int8_t)k;
    if (nbad) atomicAdd(bad, nbad);
  }
}
// FP8 tiles, step 2: one thread per 16-byte chunk (tile, kstep pair p, lane) = e4m3 codes of the lane's A fragments
__global__ void __launch_bounds__(256) f8_tile_kernel(const bf16* __restrict__ src, int N, int K, int mode, int hd, int groups,
                                                      int tpg, const int8_t* __restrict__ exps, uint8_t* __restrict__ dst) {
  const int64_t q = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (q >= (int64_t)groups * tpg * 256) return;
  const int lane = (int)(q & 31), p = (int)((q >> 5) & 7);
  const int64_t tile = q >> 8;
  const int ks = (int)(tile % tpg), gi = (int)(tile / tpg);
  uint32_t out[4];
#pragma unroll
  for (int h = 0; h < 4; ++h) {   // word h: k-step 2p + (h >> 1), fragments 2 (h & 1) and 2 (h & 1) + 1
    uint32_t word = 0;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = 2 * (h & 1) + u;                        // fragment: rows-half m & 1, k-half m >> 1
      const int ar = (m & 1) * 8 + (lane >> 2);
      const int row = tile_row(mode, hd, gi, ar);
      const int col = ks * 256 + (2 * p + (h >> 1)) * 16 + (m >> 1) * 8 + 2 * (lane & 3);
      uint32_t codes = 0;
      if (row < N && col < K) {   // K % 8 == 0: col + 1 < K too
        const float inv = pow2f(-exps[gi * 16 + ar]);
        const float2 v = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(src + (int64_t)row * K + col));
        codes = float2_to_e4m3x2(v.x * inv, v.y * inv);
      }
      word |= codes << (16 * u);
    }
    out[h] = word;
  }
  *reinterpret_cast<uint4*>(dst + q * 16) = make_uint4(out[0], out[1], out[2], out[3]);
}

// Packed tiles, pass 1: one CTA per tile, warp w takes tile rows w and w + 8 (8 columns per lane). Row base b_r = max(row max
// exponent - 31, 0) over the row's values inside the matrix; the tile escapes when a value's exponent lies below its row's base.
__global__ void __launch_bounds__(256) pk_scan_kernel(const bf16* __restrict__ src, int N, int K, int mode, int hd, int tpg,
                                                      uint8_t* __restrict__ dst, uint8_t* __restrict__ escape) {
  const int64_t tile = blockIdx.x;
  const int ks = (int)(tile % tpg), gi = (int)(tile / tpg);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t base[2];
  bool esc = false;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = tile_row(mode, hd, gi, warp + 8 * h), col = ks * 256 + lane * 8;
    uint32_t emax = 0, emin = 255;
    if (row < N && col < K) {   // K % 8 == 0: the lane's 8 columns are all inside or all outside
      const uint4 v = *reinterpret_cast<const uint4*>(src + (int64_t)row * K + col);
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t e0 = (u[i] >> 7) & 0xffu, e1 = (u[i] >> 23) & 0xffu;
        emax = max(emax, max(e0, e1));
        emin = min(emin, min(e0, e1));
      }
    }
    emax = __reduce_max_sync(0xffffffffu, emax);
    emin = __reduce_min_sync(0xffffffffu, emin);
    base[h] = emax > 31u ? emax - 31u : 0u;
    esc = esc || emin < base[h];
  }
  esc = __syncthreads_or(esc) != 0;
  uint8_t* hdr = dst + tile * MEGA_PK_TILE_BYTES + MEGA_PK_HDR;
  if (lane == 0) {
    hdr[warp] = esc ? 0 : (uint8_t)base[0];
    hdr[warp + 8] = esc ? 0 : (uint8_t)base[1];
  }
  if (threadIdx.x == 0) escape[tile] = esc ? 1 : 0;
}

// Packed tiles, pass 2: one thread per (tile, lane) writes the lane's bytes of every plane (value order of f8_tile_kernel)
__global__ void __launch_bounds__(256) pk_tile_kernel(const bf16* __restrict__ src, int N, int K, int mode, int hd, int groups,
                                                      int tpg, const int* __restrict__ esc_idx, uint8_t* __restrict__ dst,
                                                      uint8_t* __restrict__ esc) {
  const int64_t q = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (q >= (int64_t)groups * tpg * 32) return;
  const int lane = (int)(q & 31);
  const int64_t tile = q >> 5;
  const int ks = (int)(tile % tpg), gi = (int)(tile / tpg);
  uint8_t* t = dst + tile * MEGA_PK_TILE_BYTES;
  const int ei = esc_idx[tile];
  const uint32_t rb[2] = {t[MEGA_PK_HDR + (lane >> 2)], t[MEGA_PK_HDR + 8 + (lane >> 2)]};
  uint32_t hbw[4] = {0u, 0u, 0u, 0u};
  for (int p = 0; p < 8; ++p) {
    uint32_t bytes[4], ex[4], nib[2] = {0u, 0u};
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // word k: kstep 2p + (k >> 1), fragments 2 (k & 1) and 2 (k & 1) + 1 (bytes 0-1 / 2-3)
      uint32_t bw = 0, xw = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int m = 2 * (k & 1) + (i >> 1);   // fragment: rows-half m & 1, k-half m >> 1
        const int ar = (m & 1) * 8 + (lane >> 2);
        const int row = tile_row(mode, hd, gi, ar);
        const int col = ks * 256 + (2 * p + (k >> 1)) * 16 + (m >> 1) * 8 + 2 * (lane & 3) + (i & 1);
        const bool in = row < N && col < K;
        const uint32_t v = in ? (uint32_t)__bfloat16_as_ushort(src[(int64_t)row * K + col]) : 0u;
        const uint32_t e = (v >> 7) & 0xffu;
        bw |= (((v >> 8) & 0x80u) | (v & 0x7fu)) << (8 * i);
        xw |= e << (8 * i);
        if (ei < 0) {
          const uint32_t c = in ? e - rb[m & 1] : 0u;   // 0..31 outside an escape tile (pass 1)
          nib[k >> 1] |= (c & 15u) << (8 * i + 4 * (k & 1));
          hbw[p >> 1] |= (c >> 4) << (8 * i + 4 * (p & 1) + k);
        }
      }
      bytes[k] = bw;
      ex[k] = xw;
    }
    *reinterpret_cast<uint4*>(t + p * 512 + lane * 16) = make_uint4(bytes[0], bytes[1], bytes[2], bytes[3]);
    *reinterpret_cast<uint2*>(t + MEGA_PK_NIB + (p >> 1) * 512 + lane * 16 + (p & 1) * 8) = make_uint2(nib[0], nib[1]);
    if (ei >= 0)
      *reinterpret_cast<uint4*>(esc + (int64_t)ei * MEGA_PK_ESC_BYTES + p * 512 + lane * 16) = make_uint4(ex[0], ex[1], ex[2], ex[3]);
  }
  *reinterpret_cast<uint4*>(t + MEGA_PK_HB + lane * 16) = make_uint4(hbw[0], hbw[1], hbw[2], hbw[3]);
  if (lane == 0) *reinterpret_cast<uint4*>(t + MEGA_PK_HDR + 16) = make_uint4((uint32_t)ei, 0u, 0u, 0u);
}

}  // namespace

int64_t mega_tiled_elems(int N, int K, int mode, int* groups, int* tpg) {
  int g = (mode == TILE_GLU) ? (N / 2 + 7) / 8 : (N + 15) / 16;
  int t = (K + 255) / 256;
  if (groups) *groups = g;
  if (tpg) *tpg = t;
  return (int64_t)g * t * MEGA_TILE_ELEMS;
}

cudaError_t launch_retile(const bf16* src, int N, int K, int mode, int hd, bf16* dst, cudaStream_t s) {
  if ((K & 7) || (mode == TILE_ROPE && ((hd != 64 && hd != 128) || N % hd))) return cudaErrorInvalidValue;
  int groups, tpg;
  mega_tiled_elems(N, K, mode, &groups, &tpg);
  const int64_t chunks = (int64_t)groups * tpg * 512;
  retile_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, s>>>(src, N, K, mode, hd, groups, tpg, dst);
  return cudaGetLastError();
}

cudaError_t launch_retile_f8(const bf16* src, int N, int K, int mode, int hd, uint8_t* dst, int8_t* exps, unsigned int* bad,
                             cudaStream_t s) {
  if ((K & 7) || (mode == TILE_ROPE && ((hd != 64 && hd != 128) || N % hd))) return cudaErrorInvalidValue;
  int groups, tpg;
  mega_tiled_elems(N, K, mode, &groups, &tpg);
  f8_rows_kernel<<<(unsigned)((groups * 16 + 7) / 8), 256, 0, s>>>(src, N, K, mode, hd, groups, exps, bad);
  const int64_t chunks = (int64_t)groups * tpg * 256;
  f8_tile_kernel<<<(unsigned)((chunks + 255) / 256), 256, 0, s>>>(src, N, K, mode, hd, groups, tpg, exps, dst);
  return cudaGetLastError();
}

cudaError_t launch_pack_scan(const bf16* src, int N, int K, int mode, int hd, uint8_t* dst, uint8_t* escape, cudaStream_t s) {
  if ((K & 7) || (mode == TILE_ROPE && ((hd != 64 && hd != 128) || N % hd))) return cudaErrorInvalidValue;
  int groups, tpg;
  mega_tiled_elems(N, K, mode, &groups, &tpg);
  pk_scan_kernel<<<(unsigned)(groups * tpg), 256, 0, s>>>(src, N, K, mode, hd, tpg, dst, escape);
  return cudaGetLastError();
}

cudaError_t launch_pack_tiles(const bf16* src, int N, int K, int mode, int hd, const int* esc_idx, uint8_t* dst, uint8_t* esc,
                              cudaStream_t s) {
  if ((K & 7) || (mode == TILE_ROPE && ((hd != 64 && hd != 128) || N % hd))) return cudaErrorInvalidValue;
  int groups, tpg;
  mega_tiled_elems(N, K, mode, &groups, &tpg);
  const int64_t threads = (int64_t)groups * tpg * 32;
  pk_tile_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, s>>>(src, N, K, mode, hd, groups, tpg, esc_idx, dst, esc);
  return cudaGetLastError();
}

// fixed-size shared memory after the ring and the activation vector: barriers, red, rope_s, tpart, gcnt, rbuf, qkn, slice
// tables (sized for head_dim 128; head_dim 64 uses a prefix of rope_s and qkn)
int mega_smem_bytes(const MegaArgs& a) {
  return a.nslots * TILE_BYTES + a.act_floats * 4 + 2 * a.nslots * 8 + (16 + 128 + NT * 16) * 4 + NG * 4 + NG * 16 * 4 + 384 * 4 + NS * 8;
}

cudaError_t mega_configure(MegaArgs& a, int H, int I, int heads, int hd, int max_smem_optin, int num_sms, int* grid_out) {
  if (hd != 64 && hd != 128) return cudaErrorInvalidValue;
  a.hd = hd;
  auto pad = [](int k) { return (k + 255) / 256 * 256; };
  int actf = pad(H) > pad(I) ? pad(H) : pad(I);
  if (pad(heads * hd) > actf) actf = pad(heads * hd);
  // attention merge scratch: key-group states (m, l, o) + the head's per-CTA partials (up to 16 records of hd + 4)
  const int nst = NCW * (256 / hd), merge = 2 * nst + nst * hd + 16 * (hd + 4);
  if (actf < merge) actf = merge;
  actf = (actf + 31) & ~31;
  a.act_floats = actf;
  a.tg_H = pad(H);
  a.tg_I = pad(I);
  if ((I + 255) / 256 > NT - 44 || (I + 255) / 256 > NS || (H + 255) / 256 > NS) return cudaErrorInvalidValue;  // partial-sum window must cover a group + tiles in flight; slice table
  const int fixed = actf * 4 + (16 + 128 + NT * 16) * 4 + NG * 4 + NG * 16 * 4 + 384 * 4 + NS * 8 + 64;
  int nslots = (max_smem_optin - fixed) / (TILE_BYTES + 16);
  if (nslots > 32) nslots = 32;
  // every ring slot must always be filled by the same producer warp and drained by the same consumer warp
  // (slot s <-> producer s % NPW, consumer s % NCW): mbarrier parity waits are only alias-free when the
  // successive uses of one barrier are ordered inside one thread.
  nslots &= ~(NCW - 1);
  if (nslots < NCW) return cudaErrorInvalidValue;
  a.nslots = nslots;
  if (heads > num_sms) return cudaErrorInvalidValue;
  *grid_out = num_sms;
  return cudaSuccess;
}

cudaError_t launch_decode_mega(const MegaArgs& a, int grid, cudaStream_t s, uint64_t* counter) {
  const int smem = mega_smem_bytes(a);
  const bool dbgk = a.dbg != nullptr || a.dbg2 != nullptr || a.dbg_flags != 0;
  const void* fn;
  const int fmt = a.pk[0].tiles ? 2 : a.f8[0].tiles ? 1 : 0;
#define DTK_MEGA_FN(hd, f) (dbgk ? (const void*)decode_mega_kernel<true, hd, f> : (const void*)decode_mega_kernel<false, hd, f>)
  if (a.hd == 128) fn = fmt == 0 ? DTK_MEGA_FN(128, 0) : fmt == 1 ? DTK_MEGA_FN(128, 1) : DTK_MEGA_FN(128, 2);
  else if (a.hd == 64) fn = fmt == 0 ? DTK_MEGA_FN(64, 0) : fmt == 1 ? DTK_MEGA_FN(64, 1) : DTK_MEGA_FN(64, 2);
  else return cudaErrorInvalidValue;
#undef DTK_MEGA_FN
  cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) return e;
  void* args[] = {(void*)&a};
  e = cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(MEGA_THREADS), args, (size_t)smem, s);
  if (counter) ++*counter;
  return e;
}

}  // namespace dtk
