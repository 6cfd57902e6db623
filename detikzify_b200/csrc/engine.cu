// C-ABI implementation (see include/detikzify_b200.h). Host-side orchestration only: weight-arena
// layout, KV sequence slots, workspaces, CUDA-graph capture of the decode+sample step and the launch
// sequences for ViT encode / projector / prefill / decode. All arithmetic is in the .cu kernels.
#include <cuda_runtime.h>

#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <thread>
#include <vector>

#include "../../include/detikzify_b200.h"
#include "launch.h"

using namespace dtk;

namespace {

struct WEntry {
  std::string name;
  int rows, cols;
  uint64_t offset, nbytes;
};

inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }
inline int patch_k_padded(const dtk_config& c) { return (int)align_up((uint64_t)3 * c.v_patch * c.v_patch, 64); }
inline int v_tokens(const dtk_config& c) { int g = c.v_image / c.v_patch; return g * g; }
inline int img_tokens(const dtk_config& c) { return v_tokens(c) / c.concat; }

std::vector<WEntry> build_table(const dtk_config& c) {
  std::vector<WEntry> t;
  uint64_t off = 0;
  auto add = [&](const std::string& n, int rows, int cols) {
    WEntry e{n, rows, cols, off, (uint64_t)rows * cols * 2};
    off = align_up(off + e.nbytes, 256);
    t.push_back(e);
  };
  const int H = c.hidden, I = c.inter, V = c.vocab, qd = c.heads * c.head_dim, kd = c.kv_heads * c.head_dim;
  add("dec.embed", V, H);
  for (int l = 0; l < c.layers; ++l) {
    std::string p = "dec.L" + std::to_string(l) + ".";
    add(p + "norm1", 1, H);
    add(p + "wqkv", qd + 2 * kd, H);
    add(p + "wo", H, qd);
    add(p + "norm2", 1, H);
    add(p + "wgu", 2 * I, H);  // interleaved rows: 2i = gate_i, 2i+1 = up_i
    add(p + "wd", H, I);
  }
  add("dec.norm", 1, H);
  add("dec.lm_head", V, H);
  const int D = c.v_hidden, VI = c.v_inter, N = v_tokens(c);
  add("proj.w", H, D * c.concat);
  add("proj.b", 1, H);
  add("vit.patch_w", D, patch_k_padded(c));
  add("vit.patch_b", 1, D);
  add("vit.pos", N, D);
  for (int l = 0; l < c.v_layers; ++l) {
    std::string p = "vit.L" + std::to_string(l) + ".";
    add(p + "ln1_w", 1, D); add(p + "ln1_b", 1, D);
    add(p + "wqkv", 3 * D, D); add(p + "bqkv", 1, 3 * D);
    add(p + "wo", D, D); add(p + "bo", 1, D);
    add(p + "ln2_w", 1, D); add(p + "ln2_b", 1, D);
    add(p + "w1", VI, D); add(p + "b1", 1, VI);
    add(p + "w2", D, VI); add(p + "b2", 1, D);
  }
  add("vit.post_w", 1, D); add("vit.post_b", 1, D);
  add("vit.head.probe", 1, D);
  add("vit.head.wq", D, D); add("vit.head.bq", 1, D);
  add("vit.head.wkv", 2 * D, D); add("vit.head.bkv", 1, 2 * D);
  add("vit.head.wo", D, D); add("vit.head.bo", 1, D);
  add("vit.head.ln_w", 1, D); add("vit.head.ln_b", 1, D);
  add("vit.head.w1", VI, D); add("vit.head.b1", 1, VI);
  add("vit.head.w2", D, VI); add("vit.head.b2", 1, D);
  return t;
}

bool config_ok(const dtk_config& c, std::string& why) {
  auto bad = [&](const char* m) { why = m; return false; };
  if (c.hidden <= 0 || c.inter <= 0 || c.layers <= 0 || c.heads <= 0 || c.kv_heads <= 0 || c.vocab <= 0) return bad("non-positive decoder dims");
  if (c.head_dim != 128 && c.head_dim != 64) return bad("decoder head_dim must be 64 or 128");
  if (c.heads * c.head_dim != c.hidden) return bad("decoder heads * head_dim must equal hidden");
  if (c.heads % c.kv_heads) return bad("heads % kv_heads != 0");
  if ((c.hidden & 7) || (c.inter & 7)) return bad("hidden/inter must be multiples of 8");
  if (c.rope_type != 0 && c.rope_type != 1) return bad("rope_type must be 0 (linear) or 1 (llama3)");
  if (c.rope_type == 1 && (c.rope_low_freq <= 0.f || c.rope_high_freq <= c.rope_low_freq || c.rope_orig_max_pos <= 0)) return bad("bad llama3 rope parameters");
  if (c.max_len <= 0 || c.max_seqs <= 0 || c.max_batch <= 0 || c.max_batch > 64) return bad("bad max_len/max_seqs/max_batch (max_batch <= 64)");
  if (c.v_hidden <= 0 || c.v_heads <= 0 || c.v_hidden % c.v_heads) return bad("bad vision dims");
  if (c.v_hidden / c.v_heads != 72) return bad("vision head_dim must be 72 (SigLIP so400m)");
  if ((c.v_hidden & 7) || (c.v_inter & 7)) return bad("vision dims must be multiples of 8");
  if (c.v_patch <= 0 || c.v_image < c.v_patch) return bad("bad image/patch size");  // conv stride P, no padding: floor(S/P) patches
  if (c.concat <= 0 || img_tokens(c) <= 0) return bad("bad concat");
  return true;
}

// TikZero adapter arena: caption embedder (LlamaModel without lm_head), connector, one cross layer per selected vision layer
// (reference model/adapter/modeling_adapter.py:293-394), dummy image
bool has_cross(const dtk_adapter_config& a, int l) { return (l + 1) % a.cross_every_n == 0; }

std::vector<WEntry> build_adapter_table(const dtk_config& c, const dtk_adapter_config& a) {
  std::vector<WEntry> t;
  uint64_t off = 0;
  auto add = [&](const std::string& n, int rows, int cols) {
    WEntry e{n, rows, cols, off, (uint64_t)rows * cols * 2};
    off = align_up(off + e.nbytes, 256);
    t.push_back(e);
  };
  const int E = a.hidden, I = a.inter, qd = a.heads * 64, kd = a.kv_heads * 64;
  add("emb.embed", a.vocab, E);
  for (int l = 0; l < a.layers; ++l) {
    std::string p = "emb.L" + std::to_string(l) + ".";
    add(p + "norm1", 1, E);
    add(p + "wqkv", qd + 2 * kd, E);
    add(p + "wo", E, qd);
    add(p + "norm2", 1, E);
    add(p + "wgu", 2 * I, E);  // interleaved rows: 2i = gate_i, 2i+1 = up_i
    add(p + "wd", E, I);
  }
  add("emb.norm", 1, E);
  const int D = c.v_hidden, VI = c.v_inter;
  add("ad.connector_w", D, E); add("ad.connector_b", 1, D);
  for (int l = 0; l < c.v_layers; ++l) {
    if (!has_cross(a, l)) continue;
    std::string p = "ad.L" + std::to_string(l) + ".";
    add(p + "ln1_w", 1, D); add(p + "ln1_b", 1, D);
    add(p + "wq", D, D); add(p + "bq", 1, D);
    add(p + "wkv", 2 * D, D); add(p + "bkv", 1, 2 * D);
    add(p + "wo", D, D); add(p + "bo", 1, D);
    add(p + "q_norm_w", 1, 72); add(p + "q_norm_b", 1, 72);
    add(p + "k_norm_w", 1, 72); add(p + "k_norm_b", 1, 72);
    add(p + "ln2_w", 1, D); add(p + "ln2_b", 1, D);
    add(p + "w1", VI, D); add(p + "b1", 1, VI);
    add(p + "w2", D, VI); add(p + "b2", 1, D);
    add(p + "attn_gate", 1, 1); add(p + "mlp_gate", 1, 1);
  }
  add("ad.dummy", 3, c.v_image * c.v_image);
  return t;
}

bool adapter_config_ok(const dtk_config& c, const dtk_adapter_config& a, std::string& why) {
  auto bad = [&](const char* m) { why = m; return false; };
  if (!config_ok(c, why)) return false;
  if (a.hidden <= 0 || a.inter <= 0 || a.layers <= 0 || a.heads <= 0 || a.kv_heads <= 0 || a.vocab <= 0) return bad("non-positive embedder dims");
  if (a.head_dim != 64) return bad("embedder head_dim must be 64");
  if (a.heads % a.kv_heads) return bad("embedder heads % kv_heads != 0");
  if ((a.hidden & 7) || (a.inter & 7)) return bad("embedder hidden/inter must be multiples of 8");
  if (a.rope_type != 0 && a.rope_type != 1) return bad("rope_type must be 0 (linear) or 1 (llama3)");
  if (a.rope_type == 1 && (a.rope_low_freq <= 0.f || a.rope_high_freq <= a.rope_low_freq || a.rope_orig_max_pos <= 0)) return bad("bad llama3 rope parameters");
  if (a.max_text <= 0 || a.max_text > 8192) return bad("max_text must be in 1..8192");
  if (a.cross_every_n <= 0) return bad("cross_every_n must be positive");
  return true;
}

// RoPE cos/sin table [T, hd/2, 2] (HF modeling_llama.py:83-121: inv_freq = theta^(-2i/d) / factor, fp32; angle = pos * inv_freq)
std::vector<float> rope_table(float theta, float factor, int type, float low_freq, float high_freq, int orig_max_pos, int hd, int64_t T) {
  const int half = hd / 2;
  std::vector<float> tab((size_t)T * half * 2);
  for (int i = 0; i < half; ++i) {
    float inv = 1.0f / powf(theta, (float)(2 * i) / (float)hd);
    if (type == 1) {   // llama3 (HF modeling_rope_utils.py _compute_llama3_parameters), fp32 like HF
      const float old_len = (float)orig_max_pos;
      const float low_wl = old_len / low_freq, high_wl = old_len / high_freq;
      const float wl = 2.0f * 3.14159265358979323846f / inv;
      if (wl > low_wl) inv = inv / factor;
      else if (!(wl < high_wl)) {
        const float smooth = (old_len / wl - low_freq) / (high_freq - low_freq);
        inv = (1.0f - smooth) * inv / factor + smooth * inv;
      }
    } else {
      inv = inv / factor;
    }
    for (int64_t p = 0; p < T; ++p) {
      float ang = (float)p * inv;
      tab[((size_t)p * half + i) * 2] = (float)cos((double)ang);
      tab[((size_t)p * half + i) * 2 + 1] = (float)sin((double)ang);
    }
  }
  return tab;
}

}  // namespace

struct dtk_engine {
  dtk_config cfg;
  int device = 0;
  std::string err;
  uint64_t launches = 0;
  const uint8_t* arena = nullptr;
  std::map<std::string, const bf16*> w;

  // KV slots: [slot][layer][2][kv_head][max_len][head_dim] bf16
  bf16* kv = nullptr;
  int64_t kv_layer_stride = 0, kv_v_offset = 0, kv_slot_stride = 0;
  std::vector<char> slot_used;
  // one-level shared KV prefix: positions [0, share_len[s]) of slot s are read from slot share_base[s] (a multiple of 16
  // positions, never written through s); refcnt[b] = sequences borrowing from b, shared_upto[b] = longest prefix lent out
  std::vector<int> share_base, share_len, refcnt, shared_upto;
  float* rope_cs = nullptr;  // [max_len, head_dim/2, 2]

  // prefill workspace (max_len rows)
  float *p_x = nullptr, *p_qkv = nullptr;
  bf16 *p_xn = nullptr, *p_q = nullptr, *p_att = nullptr, *p_h = nullptr;
  // scoring workspace (dtk_score; allocated at the first call): lm_head log-softmax partials [max_len, ceil(V / 256)], targets' logits
  float2* lse_part = nullptr;
  float* lse_tgt = nullptr;
  // decode workspace (max_batch rows)
  float *d_x = nullptr, *d_q = nullptr, *d_att = nullptr, *d_h = nullptr, *d_logits = nullptr, *d_scratch = nullptr;
  float *d_part_o = nullptr, *d_part_ml = nullptr;
  unsigned int* d_counters = nullptr;  // [max_batch*heads] + 1 (sampler done counter)
  int *d_slots = nullptr, *d_pos = nullptr, *d_tok = nullptr, *d_share_slot = nullptr, *d_share_len = nullptr;
  // per-row loop state the batched step and its sampler read: activity (a retired row writes no KV and draws nothing), RNG
  // counter base (a row admitted at step s0 draws counter 1 + step - s0) and RNG stream
  int* d_active = nullptr;
  uint32_t *d_row_step = nullptr, *d_row_seq = nullptr;
  unsigned long long* d_gen = nullptr;  // [0] = step counter
  // ViT workspace (grows with batch)
  int vit_cap = 0;
  float *v_x = nullptr, *v_small_f = nullptr, *v_pq = nullptr;
  bf16 *v_xn = nullptr, *v_qkv = nullptr, *v_att = nullptr, *v_h = nullptr, *v_small_b = nullptr;
  bool pq_ready = false;
  // the ViT forward of a chunk of nb images is captured once per (nb, outputs) into a CUDA graph over engine-owned
  // staging buffers (~250 launches per chunk, each encoding two tensor maps on the host, become one graph launch)
  struct VitGraph { cudaGraphExec_t exec; uint64_t launches; };
  std::map<int, VitGraph> vit_graphs;
  float *v_pix_in = nullptr, *v_tok_out = nullptr, *v_pool_out = nullptr;
  bf16* v_vt = nullptr;      // per-layer V^T copy for the wgmma attention
  int vit_graph = 1;
  int attn_impl = 1;         // ViT attention: 1 = wgmma (attn_tc.cu), 0 = mma.sync flash attention (attn_mma.cu)

  // generation loop
  int gen_B = 0;
  dtk_sampling gen_params{};
  unsigned long long* host_ring = nullptr;   // pinned, mapped: [ring][64] entries ((step + 1) << 32) | token
  unsigned long long* dev_ring = nullptr;     // ... followed by the admission mailbox [64]: (stamp << 32) | first token
  // admissions (dtk_gen_admit): host mirror of d_active, per-row admission stamps, and a pinned staging row per loop row for
  // the admitted history (reused only after the event of the row's previous admission has passed)
  std::vector<char> row_active;
  std::vector<uint32_t> admit_stamp;
  int* h_admit_hist = nullptr;
  std::vector<cudaEvent_t> admit_ev;
  int ring = 256;
  std::map<std::string, cudaGraphExec_t> graphs;
  cudaGraphExec_t gen_graph = nullptr;
  cudaStream_t gen_stream = nullptr;
  cudaStream_t cap_stream = nullptr;  // engine-owned: graph capture never touches the caller's stream
  // persistent decode kernel (B = 1)
  MegaArgs mega{};
  int mega_grid = 0;
  bool mega_ok = false;
  int decode_impl = 1;       // 1 = persistent weight-streaming kernel (default), 0 = per-op kernels / CUDA graph
  int decode_gemm_min_batch = 4;  // B >= this: batched decode runs the dense matrices as tensor-core GEMMs (weights once per step)
  bool gen_mega = false;
  bool gen_fused = false;    // greedy generation on the persistent kernel: argmax + token publication in the kernel tail
  unsigned long long* d_amax = nullptr;
  SampleArgs gen_sample{};
  // HF logits processors (dtk_set_processors): tables and per-row token histories in engine-owned device buffers
  SampleProcTable* d_proc_tab = nullptr;
  int* d_hist = nullptr;                // [max_batch][max_len]
  int* d_hist_len = nullptr;            // [max_batch]
  int proc_B = 0;                       // rows set by the last dtk_set_processors; 0 = processors off
  bool gen_proc = false;                // the generation loop runs the processor instantiation of the sampler
  unsigned long long* d_bar = nullptr;  // [0] counter, [1] epoch base
  unsigned int* d_head_cnt = nullptr;
  bf16* d_tiled = nullptr;             // decode-side re-tiled copy of the four layer matrices (bf16 mode)
  bf16* d_tiled_lm = nullptr;          // ... and of the lm_head (always bf16)
  uint8_t* d_tiled8 = nullptr;         // FP8 mode (option "decode_fp8"): e4m3 tiles, row exponents and check counters
  int decode_fp8 = 0;
  uint8_t* d_tiledpk = nullptr;        // packed mode (option "decode_pack"): packed tiles of the layer matrices and the lm_head
  uint8_t* d_pk_esc = nullptr;         // ... and the exponent planes of the escape tiles
  int decode_pack = 0;
  int64_t pk_escapes = 0;              // escape tiles of the packed weights
  unsigned long long* d_tagged = nullptr;  // {fp32 value, phase tag} cross-CTA activation words of the persistent kernel
  long long* d_dbg = nullptr;           // phase timestamps of the persistent kernel (option mega_debug)
  long long* d_dbg2 = nullptr;          // per-tile clock trace of one layer (option mega_trace_layer)
  int mega_trace_layer = -1;
  int mega_debug = 0;
  int mega_flags = 0;
  int mega_variant = 0;
  int mega_nslots = 0;       // dev option "mega_nslots": cap on the ring depth of the persistent kernel (0 = as configured)
  int fuse_greedy = 1;
  int cascade_attn = 1;      // batched decode: rows that share one prefix reduce it with ONE tensor-core pass (option "cascade_attn")
  int cas_slot = -1, cas_len = 0;   // set per step by dtk_decode / dtk_gen_begin: uniform shared prefix of the current batch
  int prefill_layers = -1;   // dev option "prefill_layers": decoder_stack runs only the first n layers (-1 = all)

  // TikZero adapter (dtk_adapter_attach): borrowed arena, caption-encoder workspace (max_text rows) and the conditioned
  // ViT's caption buffers (one ViT chunk of captions)
  bool has_adapter = false;
  dtk_adapter_config acfg{};
  std::map<std::string, const bf16*> aw;
  float *t_rope = nullptr, *t_x = nullptr, *t_qkv = nullptr;
  bf16 *t_xn = nullptr, *t_q = nullptr, *t_k = nullptr, *t_v = nullptr, *t_att = nullptr, *t_h = nullptr;
  bf16 *x_cond = nullptr, *x_kv = nullptr, *x_vt = nullptr;
};

namespace {

#define DTK_CK(expr)                                                                          \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      eng->err = std::string(#expr) + ": " + cudaGetErrorString(_e);                          \
      return DTK_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

#define DTK_REQUIRE(cond, msg)                                                                \
  do {                                                                                        \
    if (!(cond)) {                                                                            \
      eng->err = std::string("invalid argument: ") + msg;                                     \
      return DTK_ERR_INVALID;                                                                 \
    }                                                                                         \
  } while (0)

template <typename T>
int dev_alloc(dtk_engine* eng, T** p, uint64_t count) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, count * sizeof(T));
  if (e != cudaSuccess) {
    eng->err = std::string("cudaMalloc failed: ") + cudaGetErrorString(e);
    cudaGetLastError();
    return DTK_ERR_OOM;
  }
  *p = (T*)q;
  return DTK_OK;
}
#define DTK_ALLOC(ptr, count)                         \
  do {                                                \
    int _r = dev_alloc(eng, &(ptr), (uint64_t)(count)); \
    if (_r != DTK_OK) return _r;                      \
  } while (0)

const bf16* W(dtk_engine* eng, const std::string& n) { return eng->w.at(n); }
std::string LN(const char* prefix, int l, const char* s) { return std::string(prefix) + std::to_string(l) + "." + s; }

struct StateArgs {
  int n;
  int slots[64], pos[64], share_slot[64], share_len[64];
  long long tok[64];
  uint32_t seq[64];
  int have_tok;   // dtk_gen_begin: also the first tokens, RNG streams seq[i] and counter base 1
};
__global__ void set_state_kernel(StateArgs a, int* slots, int* pos, int* tok, int* share_slot, int* share_len, int* active,
                                 uint32_t* row_step, uint32_t* row_seq) {
  int i = threadIdx.x;
  if (i < a.n) {
    slots[i] = a.slots[i];
    pos[i] = a.pos[i];
    share_slot[i] = a.share_slot[i];
    share_len[i] = a.share_len[i];
    active[i] = 1;
    if (a.have_tok) {
      tok[i] = (int)a.tok[i];
      row_step[i] = 1u;
      row_seq[i] = a.seq[i];
    }
  }
}
// rows of a batched step that all borrow the same prefix [0, len) from the same slot (the rollouts of one figure)
void set_cascade(dtk_engine* eng, const StateArgs& st) {
  eng->cas_slot = -1; eng->cas_len = 0;
  if (!eng->cascade_attn || st.n < 4 || st.n > 64) return;
  const int len = st.share_len[0], base = st.share_slot[0];
  if (len < 64 || base == st.slots[0]) return;
  for (int i = 1; i < st.n; ++i)
    if (st.share_len[i] != len || st.share_slot[i] != base) return;
  eng->cas_slot = base; eng->cas_len = len;
}
__global__ void tok64_to_32_kernel(const int64_t* in, int* out, int n) {
  if ((int)threadIdx.x < n) out[threadIdx.x] = (int)in[threadIdx.x];
}
__global__ void reset_gen_kernel(unsigned long long* gen, unsigned int* done, unsigned long long seed) {
  gen[0] = 0ull;
  gen[1] = seed;   // read by the sampler of the generation loop (not baked into the captured graph)
  *done = 0u;
}

constexpr int VIT_CHUNK = 64;   // images per ViT pass (larger batches are processed in chunks)

// ViT workspace: allocated ONCE, for a full chunk, at the first vision call (no regrowth: a cudaFree inside a stream-ordered
// call would synchronise the device, and captured graphs keep pointing at these buffers)
int ensure_vit_ws(dtk_engine* eng, int /*B*/) {
  if (eng->vit_cap > 0) return DTK_OK;
  const dtk_config& c = eng->cfg;
  const int B = VIT_CHUNK;
  const int64_t rows = (int64_t)B * v_tokens(c);
  DTK_ALLOC(eng->v_x, rows * c.v_hidden);
  DTK_ALLOC(eng->v_xn, rows * c.v_hidden);
  DTK_ALLOC(eng->v_qkv, rows * 3 * c.v_hidden);
  DTK_ALLOC(eng->v_att, rows * c.v_hidden);
  int64_t hcols = c.v_inter > patch_k_padded(c) ? c.v_inter : patch_k_padded(c);
  DTK_ALLOC(eng->v_h, rows * hcols);
  DTK_ALLOC(eng->v_small_f, (int64_t)B * c.v_hidden * 2);
  DTK_ALLOC(eng->v_small_b, (int64_t)B * (c.v_hidden * 2 + c.v_inter));
  DTK_ALLOC(eng->v_pix_in, (int64_t)B * 3 * c.v_image * c.v_image);
  DTK_ALLOC(eng->v_tok_out, rows * c.v_hidden);
  DTK_ALLOC(eng->v_pool_out, (int64_t)B * c.v_hidden);
  DTK_ALLOC(eng->v_vt, (int64_t)B * c.v_heads * 80 * attn_tc_vt_cols(v_tokens(c)));
  eng->vit_cap = B;
  return DTK_OK;
}

// probe query of the attention-pool head: input independent (q = probe Wq^T + bq), computed once per engine
int ensure_probe_query(dtk_engine* eng, cudaStream_t s) {
  if (eng->pq_ready) return DTK_OK;
  const int D = eng->cfg.v_hidden;
  GemmArgs g{};
  g.A = W(eng, "vit.head.probe"); g.lda = D; g.W = W(eng, "vit.head.wq"); g.ldw = D; g.M = 1; g.N = D; g.K = D;
  g.bias = W(eng, "vit.head.bq"); g.out_f32 = eng->v_pq; g.ldo = D;
  DTK_CK(launch_gemm(g, s, &eng->launches));
  eng->pq_ready = true;
  return DTK_OK;
}

// caption conditioning of one ViT chunk: bf16 caption states [B, Tmax, D] (rows >= len[b] of caption b are padding)
struct XCond {
  const bf16* cond;
  const int* len;   // host int[B]
  int Tmax;
};

// TikZero cross layer l on the residual stream v_x (reference modeling_adapter.py:326-352, run as a forward pre-hook of vision
// layer l): x += sigmoid(g_attn) * out_proj(xattn(q_norm(q_proj(LN1 x)), k_norm(k_proj(cond)), v_proj(cond)));
// x += sigmoid(g_mlp) * fc2(act(fc1(LN2 x)))
int cross_layer(dtk_engine* eng, int l, const XCond& xc, int B, cudaStream_t s) {
  const dtk_config& c = eng->cfg;
  const int D = c.v_hidden, VI = c.v_inter, N = v_tokens(c), M = B * N, Mk = B * xc.Tmax;
  const int act = c.v_act == 1 ? ACT_GELU_ERF : ACT_GELU_TANH;
  uint64_t* lc = &eng->launches;
  auto aw = [&](const char* n) { return eng->aw.at(LN("ad.L", l, n)); };
  DTK_CK(launch_layernorm(eng->v_x, aw("ln1_w"), aw("ln1_b"), c.v_eps, M, D, eng->v_xn, nullptr, s, lc));
  bf16* q = eng->v_qkv;   // [M, D]
  {
    GemmArgs g{};
    g.A = eng->v_xn; g.lda = D; g.W = aw("wq"); g.ldw = D; g.M = M; g.N = D; g.K = D;
    g.bias = aw("bq"); g.out_bf16 = q; g.ldo = D;
    DTK_CK(launch_gemm(g, s, lc));
  }
  DTK_CK(launch_head_layernorm(q, D, aw("q_norm_w"), aw("q_norm_b"), c.v_eps, M, c.v_heads, 72, q, D, s, lc));
  {  // K | V of the captions, once per layer for the whole chunk
    GemmArgs g{};
    g.A = xc.cond; g.lda = D; g.W = aw("wkv"); g.ldw = D; g.M = Mk; g.N = 2 * D; g.K = D;
    g.bias = aw("bkv"); g.out_bf16 = eng->x_kv; g.ldo = 2 * D;
    DTK_CK(launch_gemm(g, s, lc));
  }
  DTK_CK(launch_head_layernorm(eng->x_kv, 2 * D, aw("k_norm_w"), aw("k_norm_b"), c.v_eps, Mk, c.v_heads, 72, eng->x_kv, 2 * D, s, lc));
  DTK_CK(launch_xattn_tc(q, eng->x_kv, xc.len, xc.Tmax, eng->x_vt, eng->v_att, B, c.v_heads, N, 1.0f / sqrtf(72.f), s, lc));
  {
    GemmArgs g{};
    g.A = eng->v_att; g.lda = D; g.W = aw("wo"); g.ldw = D; g.M = M; g.N = D; g.K = D;
    g.bias = aw("bo"); g.gate = aw("attn_gate"); g.resid = eng->v_x; g.ldr = D; g.out_f32 = eng->v_x; g.ldo = D;
    DTK_CK(launch_gemm(g, s, lc));
  }
  DTK_CK(launch_layernorm(eng->v_x, aw("ln2_w"), aw("ln2_b"), c.v_eps, M, D, eng->v_xn, nullptr, s, lc));
  {
    GemmArgs g{};
    g.A = eng->v_xn; g.lda = D; g.W = aw("w1"); g.ldw = D; g.M = M; g.N = VI; g.K = D;
    g.bias = aw("b1"); g.act = act; g.out_bf16 = eng->v_h; g.ldo = VI;
    DTK_CK(launch_gemm(g, s, lc));
  }
  {
    GemmArgs g{};
    g.A = eng->v_h; g.lda = VI; g.W = aw("w2"); g.ldw = VI; g.M = M; g.N = D; g.K = VI;
    g.bias = aw("b2"); g.gate = aw("mlp_gate"); g.resid = eng->v_x; g.ldr = D; g.out_f32 = eng->v_x; g.ldo = D;
    DTK_CK(launch_gemm(g, s, lc));
  }
  return DTK_OK;
}

// ViT blocks for B images already resident as fp32 pixels; leaves post-LN tokens (bf16) in v_xn. xc (TikZero) inserts the
// adapter's cross layers before the vision layers that have one.
int vit_forward(dtk_engine* eng, const float* pixels, int B, float* tokens_out, float* pooled_out, cudaStream_t s,
                const XCond* xc = nullptr) {
  const dtk_config& c = eng->cfg;
  const int D = c.v_hidden, VI = c.v_inter, N = v_tokens(c), KP = patch_k_padded(c);
  const int M = B * N;
  const int act = c.v_act == 1 ? ACT_GELU_ERF : ACT_GELU_TANH;
  uint64_t* lc = &eng->launches;
  bf16* col = eng->v_h;  // alias: v_h is free until the first MLP
  DTK_CK(launch_im2col(pixels, B, c.v_image, c.v_patch, KP, col, s, lc));
  {
    GemmArgs g{};
    g.A = col; g.lda = KP; g.W = W(eng, "vit.patch_w"); g.ldw = KP; g.M = M; g.N = D; g.K = KP;
    g.bias = W(eng, "vit.patch_b"); g.rowbias = W(eng, "vit.pos"); g.rowbias_mod = N;
    g.out_f32 = eng->v_x; g.ldo = D;
    DTK_CK(launch_gemm(g, s, lc));
  }
  for (int l = 0; l < c.v_layers; ++l) {
    if (xc && has_cross(eng->acfg, l)) {
      int r = cross_layer(eng, l, *xc, B, s);
      if (r != DTK_OK) return r;
    }
    DTK_CK(launch_layernorm(eng->v_x, W(eng, LN("vit.L", l, "ln1_w")), W(eng, LN("vit.L", l, "ln1_b")), c.v_eps, M, D, eng->v_xn, nullptr, s, lc));
    {
      GemmArgs g{};
      g.A = eng->v_xn; g.lda = D; g.W = W(eng, LN("vit.L", l, "wqkv")); g.ldw = D; g.M = M; g.N = 3 * D; g.K = D;
      g.bias = W(eng, LN("vit.L", l, "bqkv")); g.out_bf16 = eng->v_qkv; g.ldo = 3 * D;
      DTK_CK(launch_gemm(g, s, lc));
    }
    if (eng->attn_impl == 1 && attn_tc_supported()) {
      DTK_CK(launch_attn_tc(eng->v_qkv, eng->v_vt, eng->v_att, B, c.v_heads, N, 1.0f / sqrtf(72.f), s, lc));
    } else {
      AttnArgs a{};
      a.q = eng->v_qkv; a.k = eng->v_qkv + D; a.v = eng->v_qkv + 2 * D; a.o = eng->v_att;
      a.q_bs = a.k_bs = a.v_bs = (int64_t)N * 3 * D; a.q_hs = a.k_hs = a.v_hs = 72; a.q_rs = a.k_rs = a.v_rs = 3 * D;
      a.o_bs = (int64_t)N * D; a.o_hs = 72; a.o_rs = D;
      a.B = B; a.heads = c.v_heads; a.kv_group = 1; a.Tq = N; a.Tk = N; a.q_pos0 = 0; a.causal = 0; a.head_dim = 72;
      a.scale = 1.0f / sqrtf(72.f);
      DTK_CK(launch_flash_attn(a, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->v_att; g.lda = D; g.W = W(eng, LN("vit.L", l, "wo")); g.ldw = D; g.M = M; g.N = D; g.K = D;
      g.bias = W(eng, LN("vit.L", l, "bo")); g.resid = eng->v_x; g.ldr = D; g.out_f32 = eng->v_x; g.ldo = D;
      DTK_CK(launch_gemm(g, s, lc));
    }
    DTK_CK(launch_layernorm(eng->v_x, W(eng, LN("vit.L", l, "ln2_w")), W(eng, LN("vit.L", l, "ln2_b")), c.v_eps, M, D, eng->v_xn, nullptr, s, lc));
    {
      GemmArgs g{};
      g.A = eng->v_xn; g.lda = D; g.W = W(eng, LN("vit.L", l, "w1")); g.ldw = D; g.M = M; g.N = VI; g.K = D;
      g.bias = W(eng, LN("vit.L", l, "b1")); g.act = act; g.out_bf16 = eng->v_h; g.ldo = VI;
      DTK_CK(launch_gemm(g, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->v_h; g.lda = VI; g.W = W(eng, LN("vit.L", l, "w2")); g.ldw = VI; g.M = M; g.N = D; g.K = VI;
      g.bias = W(eng, LN("vit.L", l, "b2")); g.resid = eng->v_x; g.ldr = D; g.out_f32 = eng->v_x; g.ldo = D;
      DTK_CK(launch_gemm(g, s, lc));
    }
  }
  DTK_CK(launch_layernorm(eng->v_x, W(eng, "vit.post_w"), W(eng, "vit.post_b"), c.v_eps, M, D, eng->v_xn, tokens_out, s, lc));

  if (pooled_out) {
    bf16* kvb = eng->v_qkv;  // [M, 2D]
    {
      GemmArgs g{};
      g.A = eng->v_xn; g.lda = D; g.W = W(eng, "vit.head.wkv"); g.ldw = D; g.M = M; g.N = 2 * D; g.K = D;
      g.bias = W(eng, "vit.head.bkv"); g.out_bf16 = kvb; g.ldo = 2 * D;
      DTK_CK(launch_gemm(g, s, lc));
    }
    bf16* pa = eng->v_small_b;               // [B, D] attention output
    bf16* pn = eng->v_small_b + (int64_t)B * D;      // [B, D] LN output
    bf16* ph = eng->v_small_b + (int64_t)B * 2 * D;  // [B, VI]
    float* pr = eng->v_small_f;              // [B, D] residual
    DTK_CK(launch_pool_attn(eng->v_pq, kvb, B, N, D, c.v_heads, 1.0f / sqrtf(72.f), pa, s, lc));
    {
      GemmArgs g{};
      g.A = pa; g.lda = D; g.W = W(eng, "vit.head.wo"); g.ldw = D; g.M = B; g.N = D; g.K = D;
      g.bias = W(eng, "vit.head.bo"); g.out_f32 = pr; g.ldo = D;
      DTK_CK(launch_gemm(g, s, lc));
    }
    DTK_CK(launch_layernorm(pr, W(eng, "vit.head.ln_w"), W(eng, "vit.head.ln_b"), c.v_eps, B, D, pn, nullptr, s, lc));
    {
      GemmArgs g{};
      g.A = pn; g.lda = D; g.W = W(eng, "vit.head.w1"); g.ldw = D; g.M = B; g.N = VI; g.K = D;
      g.bias = W(eng, "vit.head.b1"); g.act = act; g.out_bf16 = ph; g.ldo = VI;
      DTK_CK(launch_gemm(g, s, lc));
    }
    {
      GemmArgs g{};
      g.A = ph; g.lda = VI; g.W = W(eng, "vit.head.w2"); g.ldw = VI; g.M = B; g.N = D; g.K = VI;
      g.bias = W(eng, "vit.head.b2"); g.resid = pr; g.ldr = D; g.out_f32 = pooled_out; g.ldo = D;
      DTK_CK(launch_gemm(g, s, lc));
    }
  }
  return DTK_OK;
}

// concat-3 projector on bf16 tokens [B, N, D] -> fp32 [B, P, H]
int project_bf16(dtk_engine* eng, const bf16* tokens, int B, float* out, cudaStream_t s) {
  const dtk_config& c = eng->cfg;
  const int D = c.v_hidden, N = v_tokens(c), P = img_tokens(c), K = D * c.concat;
  GemmArgs g{};
  g.A = tokens + (int64_t)(N - P * c.concat) * D;  // drop the first patches when N % concat != 0
  g.lda = K; g.a_rows_per_batch = P; g.a_batch_stride = (int64_t)N * D;
  g.W = W(eng, "proj.w"); g.ldw = K; g.M = B * P; g.N = c.hidden; g.K = K;
  g.bias = W(eng, "proj.b"); g.out_f32 = out; g.ldo = c.hidden;
  DTK_CK(launch_gemm(g, s, &eng->launches));
  return DTK_OK;
}

bf16* kv_layer(dtk_engine* eng, int slot, int layer) {
  return eng->kv + (int64_t)slot * eng->kv_slot_stride + (int64_t)layer * eng->kv_layer_stride;
}

// Decode-side tiles of the four layer matrices from the arena: bf16 (MegaMat::base) or FP8 (MegaArgs::f8, which requires
// every row of every layer matrix to be e4m3 x 2^k_r); the lm_head streams as bf16 tiles in both formats (d_tiled_lm, rebuilt
// here after packed mode). The new tiles are built and checked in a buffer of their own; only then are they swapped in and the
// other format's tiles freed, so a failure leaves the engine as it was.
// Frees the decode tiles of the current format (the lm_head's bf16 tiles only in packed mode, where they are not read). Every
// captured graph that bakes in MegaArgs or the FP8 tile pointers goes with them: the batched decode steps and the per-token
// graph of a generation loop (which lives in the same cache).
void drop_decode_tiles(dtk_engine* eng) {
  for (auto& g : eng->graphs) cudaGraphExecDestroy(g.second);
  eng->graphs.clear();
  eng->gen_graph = nullptr;
  cudaFree(eng->d_tiled);
  cudaFree(eng->d_tiled8);
  cudaFree(eng->d_tiledpk);
  cudaFree(eng->d_pk_esc);
  for (int i = 0; i < 4; ++i) eng->mega.mat[i].base = nullptr;
  eng->d_tiled = nullptr;
  eng->d_tiled8 = nullptr;
  eng->d_tiledpk = eng->d_pk_esc = nullptr;
  MegaArgs& m = eng->mega;
  for (int i = 0; i < 5; ++i) m.pk[i] = MegaPack{};
  for (int i = 0; i < 4; ++i) m.f8[i] = MegaF8{};
  m.pk_esc = nullptr;
  eng->decode_fp8 = eng->decode_pack = 0;
  eng->pk_escapes = 0;
}

int mega_pack_tiles(dtk_engine* eng);

int mega_layer_tiles(dtk_engine* eng, bool fp8) {
  static const char* names[4] = {"wqkv", "wo", "wgu", "wd"};
  const dtk_config& c = eng->cfg;
  MegaArgs& m = eng->mega;
  const int hd = c.head_dim, L = c.layers;
  const int64_t esz = fp8 ? 1 : 2;   // bytes per weight of a tile
  int64_t per_layer = 0, off[4], exp_layer = 0, eoff[4];
  for (int i = 0; i < 4; ++i) {
    off[i] = per_layer;
    per_layer += (int64_t)m.mat[i].groups * m.mat[i].tpg * MEGA_TILE_ELEMS * esz;
    eoff[i] = exp_layer;
    exp_layer += (int64_t)m.mat[i].groups * 16;
  }
  const int64_t tiles_bytes = per_layer * L, exp0 = tiles_bytes, bad0 = (exp0 + exp_layer * L + 255) / 256 * 256;
  const int64_t total = fp8 ? bad0 + 4 * (int64_t)L * 4 : tiles_bytes;
  DTK_CK(cudaDeviceSynchronize());   // the arena is written; no launch reads the current tiles any more
  uint8_t* buf = nullptr;
  DTK_ALLOC(buf, total);
  unsigned int* bad = reinterpret_cast<unsigned int*>(buf + bad0);
  cudaError_t e = fp8 ? cudaMemset(bad, 0, 4 * (size_t)L * sizeof(unsigned int)) : cudaSuccess;
  bf16* lm = nullptr;
  if (e == cudaSuccess && !eng->d_tiled_lm) {
    e = cudaMalloc(&lm, (size_t)m.mat[4].groups * m.mat[4].tpg * MEGA_TILE_ELEMS * sizeof(bf16));
    if (e == cudaSuccess) e = launch_retile(W(eng, "dec.lm_head"), c.vocab, c.hidden, TILE_SEQ, hd, lm, 0);
  }
  for (int l = 0; l < L && e == cudaSuccess; ++l)
    for (int i = 0; i < 4 && e == cudaSuccess; ++i) {
      const MegaMat& mm = m.mat[i];
      const bf16* src = W(eng, LN("dec.L", l, names[i]));
      uint8_t* dst = buf + (int64_t)l * per_layer + off[i];
      e = fp8 ? launch_retile_f8(src, mm.N, mm.K, mm.mode, hd, dst, reinterpret_cast<int8_t*>(buf + exp0 + (int64_t)l * exp_layer + eoff[i]),
                                 bad + l * 4 + i, 0)
              : launch_retile(src, mm.N, mm.K, mm.mode, hd, reinterpret_cast<bf16*>(dst), 0);
    }
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  std::vector<unsigned int> nbad(fp8 ? 4 * L : 0);
  if (e == cudaSuccess && fp8) e = cudaMemcpy(nbad.data(), bad, nbad.size() * sizeof(unsigned int), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) {
    cudaFree(buf);
    cudaFree(lm);
    eng->err = std::string("decode tiles: ") + cudaGetErrorString(e);
    return DTK_ERR_CUDA;
  }
  for (size_t k = 0; k < nbad.size(); ++k)
    if (nbad[k]) {
      cudaFree(buf);
      cudaFree(lm);
      eng->err = "invalid argument: decode_fp8: layer " + std::to_string(k / 4) + " " + names[k % 4] + " holds " +
                 std::to_string(nbad[k]) + " values that are not an e4m3 value times a power-of-two row scale (quantize the "
                 "weights first: load(..., quantize=\"fp8\"))";
      return DTK_ERR_INVALID;
    }
  drop_decode_tiles(eng);
  eng->d_tiled = fp8 ? nullptr : reinterpret_cast<bf16*>(buf);
  eng->d_tiled8 = fp8 ? buf : nullptr;
  for (int i = 0; i < 4; ++i) {
    m.mat[i].base = fp8 ? nullptr : reinterpret_cast<const bf16*>(buf + off[i]);
    m.mat[i].layer_stride = fp8 ? 0 : per_layer / 2;
    m.f8[i] = fp8 ? MegaF8{buf + off[i], reinterpret_cast<const int8_t*>(buf + exp0 + eoff[i]), per_layer, exp_layer} : MegaF8{};
  }
  if (lm) eng->d_tiled_lm = lm;
  m.mat[4].base = eng->d_tiled_lm;
  eng->decode_fp8 = fp8 ? 1 : 0;
  return DTK_OK;
}

// Packed decode tiles (MegaArgs::pk) of the four layer matrices and the lm_head from the arena: lossless, any bf16 weights.
// Two passes over every matrix: the first derives the row bases and marks the escape tiles, the host numbers the escape tiles
// in tile order (deterministic side-buffer layout), the second writes the planes. Built in buffers of their own and swapped in
// on success, as mega_layer_tiles.
int mega_pack_tiles(dtk_engine* eng) {
  static const char* names[4] = {"wqkv", "wo", "wgu", "wd"};
  const dtk_config& c = eng->cfg;
  MegaArgs& m = eng->mega;
  const int hd = c.head_dim, L = c.layers;
  int64_t per_layer = 0, toff[4];   // tiles
  for (int i = 0; i < 4; ++i) {
    toff[i] = per_layer;
    per_layer += (int64_t)m.mat[i].groups * m.mat[i].tpg;
  }
  const int64_t lm0 = per_layer * L, ntiles = lm0 + (int64_t)m.mat[4].groups * m.mat[4].tpg;
  DTK_CK(cudaDeviceSynchronize());   // the arena is written; no launch reads the current tiles any more
  uint8_t *buf = nullptr, *flags = nullptr, *esc = nullptr;
  int* idx = nullptr;
  cudaError_t e = cudaMalloc(&buf, (size_t)ntiles * MEGA_PK_TILE_BYTES);
  bool dropped = false;
  if (e == cudaErrorMemoryAllocation) {
    // no room for both tile sets (a 7B model with a large KV cache): the current tiles go first, and bf16 tiles are rebuilt
    // from the arena if packing fails below
    cudaGetLastError();
    drop_decode_tiles(eng);
    cudaFree(eng->d_tiled_lm);
    eng->d_tiled_lm = nullptr;
    dropped = true;
    e = cudaMalloc(&buf, (size_t)ntiles * MEGA_PK_TILE_BYTES);
  }
  if (e == cudaSuccess) e = cudaMalloc(&flags, (size_t)ntiles);
  if (e == cudaSuccess) e = cudaMalloc(&idx, (size_t)ntiles * sizeof(int));
  // every matrix with the index of its first tile
  auto each = [&](auto&& f) {
    for (int l = 0; l < L && e == cudaSuccess; ++l)
      for (int i = 0; i < 4 && e == cudaSuccess; ++i) e = f(W(eng, LN("dec.L", l, names[i])), m.mat[i], l * per_layer + toff[i]);
    if (e == cudaSuccess) e = f(W(eng, "dec.lm_head"), m.mat[4], lm0);
  };
  each([&](const bf16* src, const MegaMat& mm, int64_t t0) {
    return launch_pack_scan(src, mm.N, mm.K, mm.mode, hd, buf + t0 * MEGA_PK_TILE_BYTES, flags + t0, 0);
  });
  std::vector<uint8_t> hflag(e == cudaSuccess ? ntiles : 0);
  std::vector<int> hidx(hflag.size());
  if (e == cudaSuccess) e = cudaMemcpy(hflag.data(), flags, hflag.size(), cudaMemcpyDeviceToHost);
  int64_t nesc = 0;
  for (size_t t = 0; t < hflag.size(); ++t) hidx[t] = hflag[t] ? (int)nesc++ : -1;
  if (e == cudaSuccess) e = cudaMemcpy(idx, hidx.data(), hidx.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nesc) e = cudaMalloc(&esc, (size_t)nesc * MEGA_PK_ESC_BYTES);
  each([&](const bf16* src, const MegaMat& mm, int64_t t0) {
    return launch_pack_tiles(src, mm.N, mm.K, mm.mode, hd, idx + t0, buf + t0 * MEGA_PK_TILE_BYTES, esc, 0);
  });
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  cudaFree(flags);
  cudaFree(idx);
  if (e != cudaSuccess) {
    cudaFree(buf);
    cudaFree(esc);
    cudaGetLastError();
    const std::string msg = std::string("packed decode tiles: ") + cudaGetErrorString(e);
    if (dropped && mega_layer_tiles(eng, false) != DTK_OK) eng->err = msg + "; rebuilding the bf16 tiles failed: " + eng->err;
    else eng->err = msg + (dropped ? " (the engine is back on bf16 tiles)" : "");
    return DTK_ERR_CUDA;
  }
  drop_decode_tiles(eng);
  cudaFree(eng->d_tiled_lm);
  eng->d_tiled_lm = nullptr;
  eng->d_tiledpk = buf;
  eng->d_pk_esc = esc;
  for (int i = 0; i < 5; ++i) {
    m.mat[i].base = nullptr;
    m.mat[i].layer_stride = 0;
    m.pk[i] = MegaPack{buf + (i < 4 ? toff[i] : lm0) * MEGA_PK_TILE_BYTES, i < 4 ? per_layer * MEGA_PK_TILE_BYTES : 0};
  }
  m.pk_esc = esc;
  eng->decode_pack = 1;
  eng->pk_escapes = nesc;
  return DTK_OK;
}

// weight bytes one batch-1 persistent decode token streams: the four layer matrices (bf16, or e4m3 codes plus one exponent
// per row), the lm_head in bf16
// (packed mode: decode_pack_weight_bytes)
uint64_t decode_weight_bytes(const dtk_config& c, bool fp8) {
  const uint64_t H = c.hidden, I = c.inter, V = c.vocab, qd = (uint64_t)c.heads * c.head_dim, kd = (uint64_t)c.kv_heads * c.head_dim;
  const uint64_t layer_w = (uint64_t)c.layers * ((qd + 2 * kd) * H + H * qd + 3 * H * I);
  const uint64_t layer_rows = (uint64_t)c.layers * ((qd + 2 * kd) + H + 2 * I + H);
  return (fp8 ? layer_w + layer_rows : 2 * layer_w) + 2 * V * H;
}

// packed mode: every tile of the layer matrices and the lm_head (planes and header) plus the escape tiles' exponent planes
uint64_t decode_pack_weight_bytes(const dtk_engine* eng) {
  const MegaArgs& m = eng->mega;
  uint64_t layer = 0;
  for (int i = 0; i < 4; ++i) layer += (uint64_t)m.mat[i].groups * m.mat[i].tpg;
  const uint64_t tiles = layer * eng->cfg.layers + (uint64_t)m.mat[4].groups * m.mat[4].tpg;
  return tiles * MEGA_PK_TILE_BYTES + (uint64_t)eng->pk_escapes * MEGA_PK_ESC_BYTES;
}

int nsplit_for(const dtk_config& c, int B) {
  int n = (2 * 132 + c.heads * B - 1) / (c.heads * B);   // two CTAs on each of the H100's 132 SMs
  if (n < 1) n = 1;
  if (n > 16) n = 16;
  return n;
}

// one decode step for the B sequences whose (slot, pos, tok) live in d_slots / d_pos / d_tok (or tok64)
int decode_launches(dtk_engine* eng, int B, const int64_t* tok64, float* logits, cudaStream_t s) {
  const dtk_config& c = eng->cfg;
  const int H = c.hidden, I = c.inter, HD = c.head_dim, qd = c.heads * HD, kd = c.kv_heads * HD;
  const float scale = 1.0f / sqrtf((float)HD);
  uint64_t* lc = &eng->launches;
  if (B == 1 && eng->decode_impl == 1 && eng->mega_ok) {
    if (tok64) {
      tok64_to_32_kernel<<<1, 32, 0, s>>>(tok64, eng->d_tok, 1);
      ++*lc;
      DTK_CK(cudaGetLastError());
    }
    MegaArgs m = eng->mega;
    m.logits = logits;
    m.dbg = eng->mega_debug ? eng->d_dbg : nullptr;
    m.dbg_flags = eng->mega_flags;
    m.variant = eng->mega_variant;
    if (eng->mega_nslots >= 8 && eng->mega_nslots < m.nslots) m.nslots = eng->mega_nslots & ~7;
    m.fuse_greedy = 0;
    if (eng->gen_fused && logits == eng->d_logits) {   // inside the greedy generation loop
      m.fuse_greedy = 1; m.bad_token = eng->gen_sample.bad_token; m.ring = eng->ring; m.max_pos = eng->cfg.max_len - 1;
      m.amax = eng->d_amax; m.gen_tok = eng->d_tok; m.gen_pos = eng->d_pos; m.gen_step = eng->d_gen; m.host_ring = eng->dev_ring;
    }
    m.dbg2 = (eng->mega_debug && eng->mega_trace_layer >= 0) ? eng->d_dbg2 : nullptr;
    m.dbg_layer = eng->mega_trace_layer;
    DTK_CK(launch_decode_mega(m, eng->mega_grid, s, lc));
    return DTK_OK;
  }
  DTK_CK(launch_embed_tokens(tok64 ? nullptr : eng->d_tok, tok64, B, W(eng, "dec.embed"), H, c.vocab, eng->d_x, s, lc));
  int nsplit = nsplit_for(c, B);
  if (eng->decode_gemm_min_batch > 0 && B >= eng->decode_gemm_min_batch && B <= c.max_len) {
    if (eng->cas_len > 0 && eng->cas_slot >= 0 && nsplit > 4) nsplit = 4;   // cascade: the per-row kernel covers the (short) private suffix only; 12+ partial slots stay for the prefix   // (B rows fit the prefill buffers)
    // ---- batched decode (MCTS rollouts / several figures): the B rows go through the dense matrices as ONE GEMM each, so
    // the weights are streamed once per step instead of once per sequence (the GEMV kernels below re-read them B times).
    // Activations are rounded to bf16 GEMM operands exactly as in prefill
    // (fp32 residual stream, fp32 accumulation); RoPE / KV append / attention are per row (slot, position).
    const int qkvd = qd + 2 * kd;
    // decode_fp8: the four layer matrices (mat = 0..3 of layer l) stream from the FP8 decode tiles on the swapped-operand
    // tile, with the result bits of the bf16 arena. B >= 64 runs the dense bf16 tile, and the lm_head stays bf16.
    const bool fp8 = eng->decode_fp8 != 0 && B < 64;
    auto gemm = [&](const bf16* A, int K, const bf16* Wm, int N, const float* resid, int glu, float* o32, bf16* o16, int ldo,
                    int l = 0, int mat = -1) {
      GemmArgs g{};
      g.A = A; g.lda = K; g.W = Wm; g.ldw = K; g.M = B; g.N = N; g.K = K;
      g.resid = resid; g.ldr = ldo; g.glu = glu; g.out_f32 = o32; g.out_bf16 = o16; g.ldo = ldo;
      if (fp8 && mat >= 0) {
        const MegaMat& mm = eng->mega.mat[mat];
        const MegaF8& t = eng->mega.f8[mat];
        const GemmF8 w{t.tiles + l * t.layer_stride, t.exps + l * t.exp_stride, mm.groups, mm.tpg, mm.mode, HD};
        return launch_gemm_swap_f8(g, w, s, lc);
      }
      return launch_gemm(g, s, lc);
    };
    // Shared-prefix ("cascade") attention: when every row borrows the same prefix from one slot (MCTS rollouts of a figure),
    // the prefix keys are reduced ONCE per head by the tensor-core flash kernel with the B query rows as its M dimension
    // (K/V tiles read once instead of B times); the
    // per-row kernel covers the private suffix only and merges both partial sets.
    const bool cas = eng->cas_len > 0 && eng->cas_slot >= 0;
    const int ctiles_all = cas ? (eng->cas_len + 63) / 64 : 0;
    const int cslots = 16 - nsplit;   // partial slots per (row, head) left for the prefix (buffers hold 16)
    const int ctile = cas ? std::max(2, (ctiles_all + cslots - 1) / cslots) : 0;   // 64-key tiles per prefix CTA
    const int csplit = cas ? (ctiles_all + ctile - 1) / ctile : 0;
    for (int l = 0; l < c.layers; ++l) {
      DTK_CK(launch_rmsnorm(eng->d_x, H, W(eng, LN("dec.L", l, "norm1")), c.rms_eps, B, H, eng->p_xn, s, lc));
      DTK_CK(gemm(eng->p_xn, H, W(eng, LN("dec.L", l, "wqkv")), qkvd, nullptr, 0, eng->p_qkv, nullptr, qkvd, l, 0));
      DTK_CK(launch_rope_kv_decode(eng->p_qkv, B, eng->d_slots, eng->d_pos, eng->d_active, c.heads, c.kv_heads, eng->rope_cs, eng->d_q,
                                   kv_layer(eng, 0, l), eng->kv_slot_stride, eng->kv_v_offset, c.max_len, HD, s, lc, cas ? eng->p_q : nullptr));
      if (cas) {
        AttnArgs f{};
        f.q = eng->p_q; f.k = kv_layer(eng, eng->cas_slot, l); f.v = f.k + eng->kv_v_offset;
        f.q_bs = 0; f.q_hs = HD; f.q_rs = qd;
        f.k_bs = 0; f.k_hs = (int64_t)c.max_len * HD; f.k_rs = HD;
        f.v_bs = 0; f.v_hs = (int64_t)c.max_len * HD; f.v_rs = HD;
        f.B = 1; f.heads = c.heads; f.kv_group = c.heads / c.kv_heads; f.Tq = B; f.Tk = eng->cas_len; f.q_pos0 = 0;
        f.causal = 0; f.head_dim = HD; f.scale = scale;
        f.part_o = eng->d_part_o; f.part_ml = eng->d_part_ml; f.part_np = nsplit + csplit; f.part_idx0 = nsplit; f.part_tiles = ctile;
        DTK_CK(launch_flash_attn(f, s, lc));
      }
      {
        DecodeAttnArgs a{};
        a.q = eng->d_q; a.q_stride = qd; a.kv_base = kv_layer(eng, 0, l); a.kv_slot_stride = eng->kv_slot_stride;
        a.kv_v_offset = eng->kv_v_offset; a.slots = eng->d_slots; a.pos = eng->d_pos; a.share_slot = eng->d_share_slot; a.share_len = eng->d_share_len;
        a.B = B; a.heads = c.heads; a.kv_group = c.heads / c.kv_heads; a.max_len = c.max_len; a.nsplit = nsplit;
        a.head_dim = HD; a.scale = scale;
        a.part_o = eng->d_part_o; a.part_ml = eng->d_part_ml; a.counters = eng->d_counters;
        a.out = eng->d_att; a.out_stride = qd; a.out_bf16 = eng->p_att;   // bf16 copy = the o-proj operand (no cast launch)
        a.active = eng->d_active;
        if (cas) { a.key_begin = eng->cas_len; a.np = nsplit + csplit; }
        DTK_CK(launch_decode_attn(a, s, lc));
      }
      DTK_CK(gemm(eng->p_att, qd, W(eng, LN("dec.L", l, "wo")), H, eng->d_x, 0, eng->d_x, nullptr, H, l, 1));
      DTK_CK(launch_rmsnorm(eng->d_x, H, W(eng, LN("dec.L", l, "norm2")), c.rms_eps, B, H, eng->p_xn, s, lc));
      DTK_CK(gemm(eng->p_xn, H, W(eng, LN("dec.L", l, "wgu")), 2 * I, nullptr, 1, nullptr, eng->p_h, I, l, 2));
      DTK_CK(gemm(eng->p_h, I, W(eng, LN("dec.L", l, "wd")), H, eng->d_x, 0, eng->d_x, nullptr, H, l, 3));
    }
    DTK_CK(launch_rmsnorm(eng->d_x, H, W(eng, "dec.norm"), c.rms_eps, B, H, eng->p_xn, s, lc));
    DTK_CK(gemm(eng->p_xn, H, W(eng, "dec.lm_head"), c.vocab, nullptr, 0, logits, nullptr, c.vocab));
    return DTK_OK;
  }
  for (int l = 0; l < c.layers; ++l) {
    {
      GemvArgs g{};
      g.mode = GEMV_QKV; g.W = W(eng, LN("dec.L", l, "wqkv")); g.N = qd + 2 * kd; g.K = H;
      g.x = eng->d_x; g.x_stride = H; g.norm_w = W(eng, LN("dec.L", l, "norm1")); g.eps = c.rms_eps;
      g.out = eng->d_q; g.out_stride = qd; g.B = B;
      g.slots = eng->d_slots; g.pos = eng->d_pos; g.rope_cs = eng->rope_cs;
      g.kv_base = kv_layer(eng, 0, l); g.kv_slot_stride = eng->kv_slot_stride; g.kv_v_offset = eng->kv_v_offset;
      g.q_dim = qd; g.kv_dim = kd; g.max_len = c.max_len; g.head_dim = HD; g.active = eng->d_active;
      DTK_CK(launch_gemv(g, s, lc));
    }
    {
      DecodeAttnArgs a{};
      a.q = eng->d_q; a.q_stride = qd; a.kv_base = kv_layer(eng, 0, l); a.kv_slot_stride = eng->kv_slot_stride;
      a.kv_v_offset = eng->kv_v_offset; a.slots = eng->d_slots; a.pos = eng->d_pos; a.share_slot = eng->d_share_slot; a.share_len = eng->d_share_len;
      a.B = B; a.heads = c.heads; a.kv_group = c.heads / c.kv_heads; a.max_len = c.max_len; a.nsplit = nsplit;
      a.head_dim = HD; a.scale = scale;
      a.part_o = eng->d_part_o; a.part_ml = eng->d_part_ml; a.counters = eng->d_counters;
      a.out = eng->d_att; a.out_stride = qd; a.active = eng->d_active;
      DTK_CK(launch_decode_attn(a, s, lc));
    }
    {
      GemvArgs g{};
      g.mode = GEMV_ADD; g.W = W(eng, LN("dec.L", l, "wo")); g.N = H; g.K = qd;
      g.x = eng->d_att; g.x_stride = qd; g.out = eng->d_x; g.out_stride = H; g.B = B;
      DTK_CK(launch_gemv(g, s, lc));
    }
    {
      GemvArgs g{};
      g.mode = GEMV_GLU; g.W = W(eng, LN("dec.L", l, "wgu")); g.N = 2 * I; g.K = H;
      g.x = eng->d_x; g.x_stride = H; g.norm_w = W(eng, LN("dec.L", l, "norm2")); g.eps = c.rms_eps;
      g.out = eng->d_h; g.out_stride = I; g.B = B;
      DTK_CK(launch_gemv(g, s, lc));
    }
    {
      GemvArgs g{};
      g.mode = GEMV_ADD; g.W = W(eng, LN("dec.L", l, "wd")); g.N = H; g.K = I;
      g.x = eng->d_h; g.x_stride = I; g.out = eng->d_x; g.out_stride = H; g.B = B;
      DTK_CK(launch_gemv(g, s, lc));
    }
  }
  {
    GemvArgs g{};
    g.mode = GEMV_STORE; g.W = W(eng, "dec.lm_head"); g.N = c.vocab; g.K = H;
    g.x = eng->d_x; g.x_stride = H; g.norm_w = W(eng, "dec.norm"); g.eps = c.rms_eps;
    g.out = logits; g.out_stride = c.vocab; g.B = B;
    DTK_CK(launch_gemv(g, s, lc));
  }
  return DTK_OK;
}

// the sampling rules of dtk_sampling, shared by the engine's sampler and the engine-free test hook dtk_dbg_sample
void fill_sample_params(SampleArgs& a, const float* logits, int B, int V, const dtk_sampling& p) {
  std::memset(&a, 0, sizeof(a));
  a.logits = logits; a.B = B; a.V = V;
  a.temperature = (float)p.temperature; a.top_p = (float)p.top_p; a.top_p_limit = (float)(1.0 - p.top_p); a.top_k = p.top_k;
  a.do_sample = (p.do_sample && p.temperature >= 1e-5) ? 1 : 0;
  a.bad_token = p.bad_token; a.bs_token = p.begin_suppress_token; a.seed = p.seed;
}

void fill_sample_args(dtk_engine* eng, SampleArgs& a, const float* logits, int B, const dtk_sampling& p) {
  fill_sample_params(a, logits, B, eng->cfg.vocab, p);
  a.max_pos = eng->cfg.max_len - 1;
  a.scratch = eng->d_scratch;
}

// host image of the processor table for B rows: validates dtk_processors (HF's argument checks) and the histories
bool fill_proc_table(const dtk_processors& p, int B, int V, int max_len, const int32_t* hist_ids, const int32_t* hist_len,
                     const int32_t* eos_min_len, SampleProcTable& t, std::vector<int>& hist, std::string& why) {
  std::memset(&t, 0, sizeof(t));
  if (!(p.repetition_penalty > 0.0) || !std::isfinite(p.repetition_penalty)) { why = "repetition_penalty must be a positive float"; return false; }
  if (p.no_repeat_ngram_size < 0) { why = "no_repeat_ngram_size must be >= 0"; return false; }
  if (!(p.min_p >= 0.0 && p.min_p <= 1.0)) { why = "min_p must lie in [0, 1]"; return false; }
  if (p.n_ban < 0 || p.n_begin < 0 || p.n_words < 0) { why = "negative table size"; return false; }
  if ((p.n_ban && !p.ban_ids) || (p.n_begin && !p.begin_ids) || (p.n_words && (!p.word_ids || !p.word_lens))) { why = "null table"; return false; }
  if (V > kProcMaxVocab) { why = "logits processors need vocab <= " + std::to_string(kProcMaxVocab); return false; }
  auto id_ok = [&](int id) { return id >= 0 && id < V; };
  if (p.eos_token_id != -1 && !id_ok(p.eos_token_id)) { why = "eos_token_id outside [0, vocab)"; return false; }
  int64_t nword_ids = 0;
  for (int e = 0; e < p.n_words; ++e) {
    if (p.word_lens[e] < 2) { why = "bad-word sequences in word_ids must hold >= 2 ids (single ids go to ban_ids)"; return false; }
    nword_ids += p.word_lens[e];
  }
  const int64_t total = (int64_t)p.n_ban + p.n_begin + p.n_words + 1 + nword_ids;
  if (total > kProcMaxIds) { why = "processor tables exceed " + std::to_string(kProcMaxIds) + " ids (ban + begin + bad-word ids + bad-word count + 1)"; return false; }
  t.penalty = (float)p.repetition_penalty; t.min_p = (float)p.min_p; t.ngram = p.no_repeat_ngram_size; t.eos = p.eos_token_id;
  t.n_ban = p.n_ban; t.n_begin = p.n_begin; t.n_words = p.n_words;
  int k = 0;
  for (int i = 0; i < p.n_ban; ++i) { if (!id_ok(p.ban_ids[i])) { why = "ban id outside [0, vocab)"; return false; } t.ids[k++] = p.ban_ids[i]; }
  for (int i = 0; i < p.n_begin; ++i) { if (!id_ok(p.begin_ids[i])) { why = "begin-suppress id outside [0, vocab)"; return false; } t.ids[k++] = p.begin_ids[i]; }
  int o = 0;
  for (int e = 0; e <= p.n_words; ++e) { t.ids[k++] = o; if (e < p.n_words) o += p.word_lens[e]; }
  for (int i = 0; i < nword_ids; ++i) { if (!id_ok(p.word_ids[i])) { why = "bad-word id outside [0, vocab)"; return false; } t.ids[k++] = p.word_ids[i]; }
  hist.assign((size_t)B * max_len, 0);
  int64_t at = 0;
  for (int b = 0; b < B; ++b) {
    const int L = hist_len ? hist_len[b] : 0;
    if (L < 0 || L > max_len) { why = "history length outside [0, max_len]"; return false; }
    for (int i = 0; i < L; ++i) {
      const int id = hist_ids[at + i];
      if (!id_ok(id)) { why = "history id outside [0, vocab)"; return false; }
      hist[(size_t)b * max_len + i] = id;
    }
    at += L;
    t.eos_until[b] = eos_min_len ? eos_min_len[b] : 0;
  }
  return true;
}

SampleProc proc_args(dtk_engine* eng) {
  SampleProc q{};
  q.tab = eng->d_proc_tab; q.hist = eng->d_hist; q.hist_len = eng->d_hist_len; q.hist_stride = eng->cfg.max_len;
  return q;
}

// the generation loop's sampler launch: the processor instantiation while processors are set at dtk_gen_begin
cudaError_t launch_gen_sample(dtk_engine* eng, cudaStream_t s) {
  return eng->gen_proc ? launch_sample_proc(eng->gen_sample, proc_args(eng), s, &eng->launches)
                       : launch_sample(eng->gen_sample, s, &eng->launches);
}

}  // namespace

// ================================================================== C ABI
extern "C" {

int dtk_abi_version(void) { return DTK_ABI_VERSION; }

int dtk_weight_count(const dtk_config* cfg) {
  if (!cfg) return DTK_ERR_INVALID;
  std::string why;
  if (!config_ok(*cfg, why)) return DTK_ERR_INVALID;
  return (int)build_table(*cfg).size();
}

int dtk_weight_get(const dtk_config* cfg, int index, dtk_weight_info* out) {
  if (!cfg || !out) return DTK_ERR_INVALID;
  std::string why;
  if (!config_ok(*cfg, why)) return DTK_ERR_INVALID;
  auto t = build_table(*cfg);
  if (index < 0 || index >= (int)t.size()) return DTK_ERR_INVALID;
  std::memset(out, 0, sizeof(*out));
  std::snprintf(out->name, sizeof(out->name), "%s", t[index].name.c_str());
  out->offset = t[index].offset; out->nbytes = t[index].nbytes; out->rows = t[index].rows; out->cols = t[index].cols;
  return DTK_OK;
}

uint64_t dtk_arena_bytes(const dtk_config* cfg) {
  if (!cfg) return 0;
  std::string why;
  if (!config_ok(*cfg, why)) return 0;
  auto t = build_table(*cfg);
  return align_up(t.back().offset + t.back().nbytes, 256);
}

uint64_t dtk_decode_bytes(const dtk_config* c, int T) {
  if (!c) return 0;
  const uint64_t H = c->hidden, I = c->inter, V = c->vocab, qd = (uint64_t)c->heads * c->head_dim, kd = (uint64_t)c->kv_heads * c->head_dim;
  uint64_t wbytes = 2 * ((uint64_t)c->layers * ((qd + 2 * kd) * H + H * qd + 3 * H * I) + V * H);
  uint64_t kv = 2 * (uint64_t)c->layers * 2 * kd;  // bytes per cached position (K and V, bf16)
  return wbytes + (uint64_t)T * kv;
}

int dtk_create(const dtk_config* cfg, const void* weight_arena, uint64_t arena_bytes, int device, dtk_engine** out) {
  if (!cfg || !weight_arena || !out) return DTK_ERR_INVALID;
  std::string why;
  if (!config_ok(*cfg, why)) return DTK_ERR_INVALID;
  if (arena_bytes < dtk_arena_bytes(cfg)) return DTK_ERR_INVALID;
  dtk_engine* eng = new (std::nothrow) dtk_engine();
  if (!eng) return DTK_ERR_OOM;
  eng->cfg = *cfg;
  eng->device = device;
  *out = eng;  // returned even on failure so the caller can read dtk_last_error, then dtk_destroy
  DTK_CK(cudaSetDevice(device));
  eng->arena = (const uint8_t*)weight_arena;
  for (auto& e : build_table(*cfg)) eng->w[e.name] = (const bf16*)(eng->arena + e.offset);

  const dtk_config& c = eng->cfg;
  const int64_t HD = c.head_dim, H = c.hidden, I = c.inter, V = c.vocab, qd = c.heads * HD, kd = c.kv_heads * HD, T = c.max_len, MB = c.max_batch;
  eng->kv_v_offset = (int64_t)c.kv_heads * c.max_len * HD;
  eng->kv_layer_stride = 2 * eng->kv_v_offset;
  eng->kv_slot_stride = eng->kv_layer_stride * c.layers;
  DTK_ALLOC(eng->kv, eng->kv_slot_stride * c.max_seqs);
  eng->slot_used.assign(c.max_seqs, 0);
  eng->share_base.assign(c.max_seqs, -1);
  eng->share_len.assign(c.max_seqs, 0);
  eng->refcnt.assign(c.max_seqs, 0);
  eng->shared_upto.assign(c.max_seqs, 0);

  {
    std::vector<float> tab = rope_table(c.rope_theta, c.rope_factor, c.rope_type, c.rope_low_freq, c.rope_high_freq,
                                        c.rope_orig_max_pos, (int)HD, T);
    DTK_ALLOC(eng->rope_cs, tab.size());
    DTK_CK(cudaMemcpy(eng->rope_cs, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  DTK_ALLOC(eng->p_x, T * H);
  DTK_ALLOC(eng->p_qkv, T * (qd + 2 * kd));
  DTK_ALLOC(eng->p_xn, T * H);
  DTK_ALLOC(eng->p_q, T * qd);
  DTK_ALLOC(eng->p_att, T * qd);
  DTK_ALLOC(eng->p_h, T * I);
  DTK_ALLOC(eng->d_x, MB * H);
  DTK_ALLOC(eng->d_q, MB * qd);
  DTK_ALLOC(eng->d_att, MB * qd);
  DTK_ALLOC(eng->d_h, MB * I);
  DTK_ALLOC(eng->d_logits, MB * V);
  DTK_ALLOC(eng->d_scratch, MB * V);
  DTK_ALLOC(eng->d_part_o, MB * c.heads * 16 * HD);
  DTK_ALLOC(eng->d_part_ml, MB * c.heads * 16 * 2);
  DTK_ALLOC(eng->d_counters, MB * c.heads + 1);
  DTK_CK(cudaMemset(eng->d_counters, 0, (MB * c.heads + 1) * sizeof(unsigned int)));
  DTK_ALLOC(eng->d_slots, MB);
  DTK_ALLOC(eng->d_pos, MB);
  DTK_ALLOC(eng->d_tok, MB);
  DTK_ALLOC(eng->d_share_slot, MB);
  DTK_ALLOC(eng->d_share_len, MB);
  DTK_ALLOC(eng->d_active, MB);
  DTK_ALLOC(eng->d_row_step, MB);
  DTK_ALLOC(eng->d_row_seq, MB);
  DTK_CK(cudaMemset(eng->d_share_slot, 0, MB * sizeof(int)));
  DTK_CK(cudaMemset(eng->d_share_len, 0, MB * sizeof(int)));
  DTK_ALLOC(eng->d_gen, 2);
  DTK_CK(cudaMemset(eng->d_gen, 0, 2 * sizeof(unsigned long long)));
  DTK_ALLOC(eng->v_pq, c.v_hidden);
  {
    int smem_optin = 0, sms = 0, coop = 0;
    DTK_CK(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    DTK_CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    DTK_CK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, device));
    MegaArgs& m = eng->mega;
    int grid = 0;
    if (coop && mega_configure(m, c.hidden, c.inter, c.heads, c.head_dim, smem_optin, sms, &grid) == cudaSuccess) {
      m.H = c.hidden; m.I = c.inter; m.L = c.layers; m.heads = c.heads; m.kv_heads = c.kv_heads; m.V = c.vocab;
      m.max_len = c.max_len; m.eps = c.rms_eps;
      m.embed = W(eng, "dec.embed"); m.final_norm = W(eng, "dec.norm");
      m.norm1_0 = W(eng, "dec.L0.norm1"); m.norm2_0 = W(eng, "dec.L0.norm2");
      m.norm_stride = c.layers > 1 ? (int64_t)(W(eng, "dec.L1.norm1") - W(eng, "dec.L0.norm1")) : 0;
      // decode-side tiled weight copy (one-time, on device): [layer][qkv | o | gu | down] (mega_layer_tiles), [lm_head]
      const int qkvN = (int)((c.heads + 2 * c.kv_heads) * HD);
      struct Spec { MegaMat* mm; int N, K, mode; } specs[4] = {
          {&m.mat[0], qkvN, c.hidden, TILE_ROPE}, {&m.mat[1], c.hidden, (int)qd, TILE_SEQ},
          {&m.mat[2], 2 * c.inter, c.hidden, TILE_GLU}, {&m.mat[3], c.hidden, c.inter, TILE_SEQ}};
      for (int i = 0; i < 4; ++i) {
        MegaMat& mm = *specs[i].mm;
        mega_tiled_elems(specs[i].N, specs[i].K, specs[i].mode, &mm.groups, &mm.tpg);
        mm.N = specs[i].N; mm.K = specs[i].K; mm.mode = specs[i].mode;
      }
      mega_tiled_elems(c.vocab, c.hidden, TILE_SEQ, &m.mat[4].groups, &m.mat[4].tpg);
      m.mat[4].layer_stride = 0; m.mat[4].N = c.vocab; m.mat[4].K = c.hidden; m.mat[4].mode = TILE_SEQ;
      for (int i = 0; i < 5; ++i) {
        m.mat[i].per = (m.mat[i].groups + grid - 1) / grid;
        m.mat[i].nact = (m.mat[i].groups + m.mat[i].per - 1) / m.mat[i].per;
      }
      {
        const int r = mega_layer_tiles(eng, false);   // bf16 tiles (and the lm_head's)
        if (r != DTK_OK) return r;
      }
      m.tok = eng->d_tok; m.pos = eng->d_pos; m.slots = eng->d_slots; m.share_slot = eng->d_share_slot; m.share_len = eng->d_share_len;
      m.kv = eng->kv; m.kv_slot_stride = eng->kv_slot_stride; m.kv_layer_stride = eng->kv_layer_stride;
      m.kv_v_offset = eng->kv_v_offset; m.rope_cs = eng->rope_cs;
      m.logits = eng->d_logits;
      {
        const int64_t words = 2 * (int64_t)m.tg_H + 2 * qd + 2 * kd + m.tg_I + (int64_t)grid * (HD + 4);
        DTK_ALLOC(eng->d_tagged, words);
        DTK_CK(cudaMemset(eng->d_tagged, 0, (size_t)words * sizeof(unsigned long long)));
        m.tg = eng->d_tagged;
      }
      DTK_ALLOC(eng->d_amax, 2);
      DTK_CK(cudaMemset(eng->d_amax, 0, 2 * sizeof(unsigned long long)));
      DTK_ALLOC(eng->d_bar, 4);
      DTK_CK(cudaMemset(eng->d_bar, 0, 4 * sizeof(unsigned long long)));
      m.bar_count = eng->d_bar; m.bar_base = eng->d_bar + 1;
      DTK_ALLOC(eng->d_head_cnt, c.heads);
      DTK_CK(cudaMemset(eng->d_head_cnt, 0, c.heads * sizeof(unsigned int)));
      m.head_cnt = eng->d_head_cnt;
      DTK_ALLOC(eng->d_dbg, (int64_t)grid * (c.layers * 5 + 1) * 4);
      DTK_CK(cudaMemset(eng->d_dbg, 0, (size_t)grid * (c.layers * 5 + 1) * 4 * sizeof(long long)));
      DTK_ALLOC(eng->d_dbg2, (int64_t)grid * MEGA_DBG2_ROWS * 4);
      DTK_CK(cudaMemset(eng->d_dbg2, 0, (size_t)grid * MEGA_DBG2_ROWS * 4 * sizeof(long long)));
      m.dbg = nullptr; m.dbg2 = nullptr; m.dbg_layer = -1;
      eng->mega_grid = grid;
      eng->mega_ok = true;
    }
  }
  DTK_CK(cudaHostAlloc((void**)&eng->host_ring, (size_t)(eng->ring + 1) * 64 * sizeof(unsigned long long), cudaHostAllocMapped));
  std::memset(eng->host_ring, 0, (size_t)(eng->ring + 1) * 64 * sizeof(unsigned long long));
  DTK_CK(cudaHostGetDevicePointer((void**)&eng->dev_ring, eng->host_ring, 0));
  DTK_CK(cudaDeviceSynchronize());
  return DTK_OK;
}

int dtk_destroy(dtk_engine* eng) {
  if (!eng) return DTK_ERR_INVALID;
  cudaSetDevice(eng->device);
  cudaDeviceSynchronize();
  for (auto& g : eng->graphs) cudaGraphExecDestroy(g.second);
  for (auto& g : eng->vit_graphs) cudaGraphExecDestroy(g.second.exec);
  void* ptrs[] = {eng->v_pix_in, eng->v_tok_out, eng->v_pool_out, eng->v_vt, eng->kv, eng->rope_cs, eng->p_x, eng->p_qkv, eng->p_xn, eng->p_q, eng->p_att, eng->p_h, eng->d_x, eng->d_q,
                  eng->d_att, eng->d_h, eng->d_logits, eng->d_scratch, eng->d_part_o, eng->d_part_ml, eng->d_counters,
                  eng->d_slots, eng->d_pos, eng->d_tok, eng->d_share_slot, eng->d_share_len, eng->d_gen, eng->d_amax, eng->d_bar, eng->d_dbg, eng->d_dbg2, eng->d_head_cnt, eng->d_tiled, eng->d_tiled_lm, eng->d_tiled8, eng->d_tiledpk, eng->d_pk_esc, eng->d_tagged, eng->v_x, eng->v_small_f, eng->v_pq, eng->v_xn,
                  eng->v_qkv, eng->v_att, eng->v_h, eng->v_small_b, eng->lse_part, eng->lse_tgt, eng->d_proc_tab, eng->d_hist,
                  eng->d_hist_len, eng->d_active, eng->d_row_step, eng->d_row_seq};
  for (void* p : ptrs) if (p) cudaFree(p);
  dtk_adapter_detach(eng);
  if (eng->cap_stream) cudaStreamDestroy(eng->cap_stream);
  if (eng->host_ring) cudaFreeHost(eng->host_ring);
  if (eng->h_admit_hist) cudaFreeHost(eng->h_admit_hist);
  for (cudaEvent_t e : eng->admit_ev) cudaEventDestroy(e);
  cudaGetLastError();
  delete eng;
  return DTK_OK;
}

const char* dtk_last_error(const dtk_engine* eng) { return eng ? eng->err.c_str() : "null engine"; }
uint64_t dtk_launch_count(const dtk_engine* eng) { return eng ? eng->launches : 0; }

int dtk_vit_encode(dtk_engine* eng, const float* pixels, int B, float* tokens_out, float* pooled_out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(pixels && B > 0, "pixels/B");
  DTK_CK(cudaSetDevice(eng->device));
  const dtk_config& c = eng->cfg;
  cudaStream_t s = (cudaStream_t)stream;
  int r = ensure_vit_ws(eng, B);
  if (r != DTK_OK) return r;
  if (pooled_out && (r = ensure_probe_query(eng, s)) != DTK_OK) return r;
  const int64_t pix_per = (int64_t)3 * c.v_image * c.v_image, N = v_tokens(c), D = c.v_hidden;
  for (int b0 = 0; b0 < B; b0 += VIT_CHUNK) {
    const int nb = B - b0 < VIT_CHUNK ? B - b0 : VIT_CHUNK;
    float* tok = tokens_out ? tokens_out + b0 * N * D : nullptr;
    float* pool = pooled_out ? pooled_out + (int64_t)b0 * D : nullptr;
    if (!eng->vit_graph) {
      r = vit_forward(eng, pixels + b0 * pix_per, nb, tok, pool, s);
      if (r != DTK_OK) return r;
      continue;
    }
    const int key = nb | (tok ? 1 << 8 : 0) | (pool ? 1 << 9 : 0) | (get_gemm_impl() << 10) | (eng->attn_impl << 12);
    auto it = eng->vit_graphs.find(key);
    if (it == eng->vit_graphs.end()) {
      if (!eng->cap_stream) DTK_CK(cudaStreamCreateWithFlags(&eng->cap_stream, cudaStreamNonBlocking));
      cudaStream_t cs = eng->cap_stream;
      const uint64_t before = eng->launches;
      cudaGraph_t graph = nullptr;
      DTK_CK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
      r = vit_forward(eng, eng->v_pix_in, nb, tok ? eng->v_tok_out : nullptr, pool ? eng->v_pool_out : nullptr, cs);
      cudaError_t ce = cudaStreamEndCapture(cs, &graph);
      const uint64_t n = eng->launches - before;
      eng->launches = before;             // captured launches are counted per replay
      if (r != DTK_OK) { if (graph) cudaGraphDestroy(graph); return r; }
      if (ce != cudaSuccess) { eng->err = std::string("cudaStreamEndCapture (ViT): ") + cudaGetErrorString(ce); return DTK_ERR_CUDA; }
      cudaGraphExec_t exec = nullptr;
      DTK_CK(cudaGraphInstantiate(&exec, graph, 0));
      cudaGraphDestroy(graph);
      it = eng->vit_graphs.emplace(key, dtk_engine::VitGraph{exec, n}).first;
    }
    DTK_CK(cudaMemcpyAsync(eng->v_pix_in, pixels + b0 * pix_per, (size_t)nb * pix_per * sizeof(float), cudaMemcpyDeviceToDevice, s));
    DTK_CK(cudaGraphLaunch(it->second.exec, s));
    eng->launches += it->second.launches;
    if (tok) DTK_CK(cudaMemcpyAsync(tok, eng->v_tok_out, (size_t)nb * N * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (pool) DTK_CK(cudaMemcpyAsync(pool, eng->v_pool_out, (size_t)nb * D * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  return DTK_OK;
}

int dtk_adapter_weight_count(const dtk_config* cfg, const dtk_adapter_config* acfg) {
  if (!cfg || !acfg) return DTK_ERR_INVALID;
  std::string why;
  if (!adapter_config_ok(*cfg, *acfg, why)) return DTK_ERR_INVALID;
  return (int)build_adapter_table(*cfg, *acfg).size();
}

int dtk_adapter_weight_get(const dtk_config* cfg, const dtk_adapter_config* acfg, int index, dtk_weight_info* out) {
  if (!cfg || !acfg || !out) return DTK_ERR_INVALID;
  std::string why;
  if (!adapter_config_ok(*cfg, *acfg, why)) return DTK_ERR_INVALID;
  auto t = build_adapter_table(*cfg, *acfg);
  if (index < 0 || index >= (int)t.size()) return DTK_ERR_INVALID;
  std::memset(out, 0, sizeof(*out));
  std::snprintf(out->name, sizeof(out->name), "%s", t[index].name.c_str());
  out->offset = t[index].offset; out->nbytes = t[index].nbytes; out->rows = t[index].rows; out->cols = t[index].cols;
  return DTK_OK;
}

uint64_t dtk_adapter_arena_bytes(const dtk_config* cfg, const dtk_adapter_config* acfg) {
  if (!cfg || !acfg) return 0;
  std::string why;
  if (!adapter_config_ok(*cfg, *acfg, why)) return 0;
  auto t = build_adapter_table(*cfg, *acfg);
  return align_up(t.back().offset + t.back().nbytes, 256);
}

int dtk_adapter_detach(dtk_engine* eng) {
  if (!eng) return DTK_ERR_INVALID;
  cudaSetDevice(eng->device);
  cudaDeviceSynchronize();   // buffers may still be read by queued work
  void* ptrs[] = {eng->t_rope, eng->t_x, eng->t_qkv, eng->t_xn, eng->t_q, eng->t_k, eng->t_v, eng->t_att, eng->t_h,
                  eng->x_cond, eng->x_kv, eng->x_vt};
  for (void* p : ptrs) if (p) cudaFree(p);
  eng->t_rope = eng->t_x = eng->t_qkv = nullptr;
  eng->t_xn = eng->t_q = eng->t_k = eng->t_v = eng->t_att = eng->t_h = nullptr;
  eng->x_cond = eng->x_kv = eng->x_vt = nullptr;
  eng->aw.clear();
  eng->has_adapter = false;
  return DTK_OK;
}

int dtk_adapter_attach(dtk_engine* eng, const dtk_adapter_config* acfg, const void* arena, uint64_t arena_bytes) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(acfg && arena, "null pointer");
  std::string why;
  if (!adapter_config_ok(eng->cfg, *acfg, why)) { eng->err = "invalid adapter config: " + why; return DTK_ERR_INVALID; }
  DTK_REQUIRE(arena_bytes >= dtk_adapter_arena_bytes(&eng->cfg, acfg), "adapter arena too small");
  dtk_adapter_detach(eng);
  DTK_CK(cudaSetDevice(eng->device));
  eng->acfg = *acfg;
  for (auto& e : build_adapter_table(eng->cfg, *acfg)) eng->aw[e.name] = (const bf16*)((const uint8_t*)arena + e.offset);
  const dtk_adapter_config& a = eng->acfg;
  const dtk_config& c = eng->cfg;
  const int64_t T = a.max_text, E = a.hidden, qd = a.heads * 64, kd = a.kv_heads * 64;
  {
    std::vector<float> tab = rope_table(a.rope_theta, a.rope_factor, a.rope_type, a.rope_low_freq, a.rope_high_freq,
                                        a.rope_orig_max_pos, 64, T);
    DTK_ALLOC(eng->t_rope, tab.size());
    DTK_CK(cudaMemcpy(eng->t_rope, tab.data(), tab.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  DTK_ALLOC(eng->t_x, T * E);
  DTK_ALLOC(eng->t_qkv, T * (qd + 2 * kd));
  DTK_ALLOC(eng->t_xn, T * E);
  DTK_ALLOC(eng->t_q, T * qd);
  DTK_ALLOC(eng->t_k, T * kd);
  DTK_ALLOC(eng->t_v, T * kd);
  DTK_ALLOC(eng->t_att, T * qd);
  DTK_ALLOC(eng->t_h, T * a.inter);
  const int64_t crow = (int64_t)VIT_CHUNK * T;
  DTK_ALLOC(eng->x_cond, crow * c.v_hidden);
  DTK_ALLOC(eng->x_kv, crow * 2 * c.v_hidden);
  DTK_ALLOC(eng->x_vt, (int64_t)VIT_CHUNK * c.v_heads * 80 * attn_tc_vt_cols((int)T));
  eng->has_adapter = true;
  return DTK_OK;
}

int dtk_text_encode(dtk_engine* eng, const int64_t* ids, int T, float* hidden_out, float* cond_out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->has_adapter, "no adapter attached");
  DTK_REQUIRE(ids && cond_out, "null pointer");
  const dtk_adapter_config& a = eng->acfg;
  DTK_REQUIRE(T >= 1 && T <= a.max_text, "T must be in 1..max_text");
  DTK_CK(cudaSetDevice(eng->device));
  cudaStream_t s = (cudaStream_t)stream;
  uint64_t* lc = &eng->launches;
  const int E = a.hidden, I = a.inter, qd = a.heads * 64, kd = a.kv_heads * 64, qkvd = qd + 2 * kd;
  auto aw = [&](const std::string& n) { return eng->aw.at(n); };
  DTK_CK(launch_embed_splice(ids, T, 0, aw("emb.embed"), E, a.vocab, -1, nullptr, 0, 0, eng->t_x, s, lc));
  for (int l = 0; l < a.layers; ++l) {
    DTK_CK(launch_rmsnorm(eng->t_x, E, aw(LN("emb.L", l, "norm1")), a.rms_eps, T, E, eng->t_xn, s, lc));
    {
      GemmArgs g{};
      g.A = eng->t_xn; g.lda = E; g.W = aw(LN("emb.L", l, "wqkv")); g.ldw = E; g.M = T; g.N = qkvd; g.K = E;
      g.out_f32 = eng->t_qkv; g.ldo = qkvd;
      DTK_CK(launch_gemm(g, s, lc));
    }
    DTK_CK(launch_rope_qkv64(eng->t_qkv, T, a.heads, a.kv_heads, eng->t_rope, eng->t_q, eng->t_k, eng->t_v, s, lc));
    {
      AttnArgs f{};
      f.q = eng->t_q; f.k = eng->t_k; f.v = eng->t_v; f.o = eng->t_att;
      f.q_bs = 0; f.q_hs = 64; f.q_rs = qd;
      f.k_bs = 0; f.k_hs = 64; f.k_rs = kd;
      f.v_bs = 0; f.v_hs = 64; f.v_rs = kd;
      f.o_bs = 0; f.o_hs = 64; f.o_rs = qd;
      f.B = 1; f.heads = a.heads; f.kv_group = a.heads / a.kv_heads; f.Tq = T; f.Tk = T; f.q_pos0 = 0;
      f.causal = 1; f.head_dim = 64; f.scale = 0.125f;
      DTK_CK(launch_flash_attn(f, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->t_att; g.lda = qd; g.W = aw(LN("emb.L", l, "wo")); g.ldw = qd; g.M = T; g.N = E; g.K = qd;
      g.resid = eng->t_x; g.ldr = E; g.out_f32 = eng->t_x; g.ldo = E;
      DTK_CK(launch_gemm(g, s, lc));
    }
    DTK_CK(launch_rmsnorm(eng->t_x, E, aw(LN("emb.L", l, "norm2")), a.rms_eps, T, E, eng->t_xn, s, lc));
    {
      GemmArgs g{};
      g.A = eng->t_xn; g.lda = E; g.W = aw(LN("emb.L", l, "wgu")); g.ldw = E; g.M = T; g.N = 2 * I; g.K = E;
      g.glu = 1; g.out_bf16 = eng->t_h; g.ldo = I;
      DTK_CK(launch_gemm(g, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->t_h; g.lda = I; g.W = aw(LN("emb.L", l, "wd")); g.ldw = I; g.M = T; g.N = E; g.K = I;
      g.resid = eng->t_x; g.ldr = E; g.out_f32 = eng->t_x; g.ldo = E;
      DTK_CK(launch_gemm(g, s, lc));
    }
  }
  DTK_CK(launch_rmsnorm(eng->t_x, E, aw("emb.norm"), a.rms_eps, T, E, eng->t_xn, s, lc));
  if (hidden_out) DTK_CK(launch_cast_bf16_f32(eng->t_xn, hidden_out, (int64_t)T * E, s, lc));
  {
    GemmArgs g{};
    g.A = eng->t_xn; g.lda = E; g.W = aw("ad.connector_w"); g.ldw = E; g.M = T; g.N = eng->cfg.v_hidden; g.K = E;
    g.bias = aw("ad.connector_b"); g.out_f32 = cond_out; g.ldo = eng->cfg.v_hidden;
    DTK_CK(launch_gemm(g, s, lc));
  }
  return DTK_OK;
}

int dtk_vit_encode_cond(dtk_engine* eng, const float* pixels, int B, const float* cond, const int* cond_len, int Tmax,
                        float* tokens_out, float* pooled_out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->has_adapter, "no adapter attached");
  DTK_REQUIRE(pixels && cond && cond_len && B > 0, "pixels/cond/cond_len/B");
  DTK_REQUIRE(Tmax >= 1 && Tmax <= eng->acfg.max_text, "Tmax must be in 1..max_text");
  for (int b = 0; b < B; ++b) DTK_REQUIRE(cond_len[b] >= 1 && cond_len[b] <= Tmax, "cond_len[b] must be in 1..Tmax");
  DTK_CK(cudaSetDevice(eng->device));
  const dtk_config& c = eng->cfg;
  cudaStream_t s = (cudaStream_t)stream;
  int r = ensure_vit_ws(eng, B);
  if (r != DTK_OK) return r;
  if (pooled_out && (r = ensure_probe_query(eng, s)) != DTK_OK) return r;
  const int64_t pix_per = (int64_t)3 * c.v_image * c.v_image, N = v_tokens(c), D = c.v_hidden;
  for (int b0 = 0; b0 < B; b0 += VIT_CHUNK) {
    const int nb = B - b0 < VIT_CHUNK ? B - b0 : VIT_CHUNK;
    DTK_CK(launch_cast_f32_bf16(cond + (int64_t)b0 * Tmax * D, eng->x_cond, (int64_t)nb * Tmax * D, s, &eng->launches));
    XCond xc{eng->x_cond, cond_len + b0, Tmax};
    r = vit_forward(eng, pixels + b0 * pix_per, nb, tokens_out ? tokens_out + b0 * N * D : nullptr,
                    pooled_out ? pooled_out + (int64_t)b0 * D : nullptr, s, &xc);
    if (r != DTK_OK) return r;
  }
  return DTK_OK;
}

int dtk_image_preprocess(dtk_engine* eng, const uint8_t* rgb, int h, int w, int S, const int32_t* bounds_h, const int32_t* coef_h,
                         int ksize_h, const int32_t* bounds_v, const int32_t* coef_v, int ksize_v, float rescale,
                         const float* mean3_host, const float* std3_host, uint8_t* tmp, float* out, uint8_t* out_u8, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(rgb && bounds_h && coef_h && bounds_v && coef_v && mean3_host && std3_host && tmp && out, "null pointer");
  DTK_REQUIRE(h > 0 && w > 0 && S > 0 && ksize_h > 0 && ksize_v > 0, "sizes");
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(launch_image_preprocess(rgb, h, w, S, bounds_h, coef_h, ksize_h, bounds_v, coef_v, ksize_v, rescale, mean3_host, std3_host,
                                 tmp, out, out_u8, (cudaStream_t)stream, &eng->launches));
  return DTK_OK;
}

int dtk_project(dtk_engine* eng, const float* tokens, int B, float* out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(tokens && out && B > 0, "tokens/out/B");
  DTK_CK(cudaSetDevice(eng->device));
  const dtk_config& c = eng->cfg;
  const int CH = VIT_CHUNK;
  int r = ensure_vit_ws(eng, B < CH ? B : CH);
  if (r != DTK_OK) return r;
  const int64_t per = (int64_t)v_tokens(c) * c.v_hidden;
  for (int b0 = 0; b0 < B; b0 += CH) {
    int nb = B - b0 < CH ? B - b0 : CH;
    DTK_CK(launch_cast_f32_bf16(tokens + b0 * per, eng->v_xn, nb * per, (cudaStream_t)stream, &eng->launches));
    r = project_bf16(eng, eng->v_xn, nb, out + (int64_t)b0 * img_tokens(c) * c.hidden, (cudaStream_t)stream);
    if (r != DTK_OK) return r;
  }
  return DTK_OK;
}

namespace {
// copy cached positions [p0, p1) of every (layer, K|V, kv head) segment from slot src to slot dst
int copy_kv_range(dtk_engine* eng, int src, int dst, int p0, int p1, cudaStream_t s) {
  if (p1 <= p0) return DTK_OK;
  const dtk_config& c = eng->cfg;
  const int64_t HD = c.head_dim;
  const size_t pitch = (size_t)c.max_len * HD * sizeof(bf16);
  DTK_CK(cudaMemcpy2DAsync(kv_layer(eng, dst, 0) + p0 * HD, pitch, kv_layer(eng, src, 0) + p0 * HD, pitch,
                           (size_t)(p1 - p0) * HD * sizeof(bf16), (size_t)c.layers * 2 * c.kv_heads, cudaMemcpyDeviceToDevice, s));
  return DTK_OK;
}
void drop_share(dtk_engine* eng, int slot) {
  const int b = eng->share_base[slot];
  if (b >= 0) {
    if (--eng->refcnt[b] == 0) eng->shared_upto[b] = 0;
    eng->share_base[slot] = -1;
    eng->share_len[slot] = 0;
  }
}
}  // namespace

int dtk_seq_alloc(dtk_engine* eng, int* slot) {
  if (!eng || !slot) return DTK_ERR_INVALID;
  for (size_t i = 0; i < eng->slot_used.size(); ++i)
    if (!eng->slot_used[i]) {
      eng->slot_used[i] = 1;
      *slot = (int)i;
      return DTK_OK;
    }
  eng->err = "no free KV sequence slot";
  return DTK_ERR_NOSLOT;
}

int dtk_seq_free(dtk_engine* eng, int slot) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(slot >= 0 && slot < (int)eng->slot_used.size() && eng->slot_used[slot], "slot");
  DTK_REQUIRE(eng->refcnt[slot] == 0, "slot still lends a shared prefix to other sequences (free them first)");
  drop_share(eng, slot);
  eng->slot_used[slot] = 0;
  return DTK_OK;
}

int dtk_seq_fork(dtk_engine* eng, int src, int dst, int len, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(src >= 0 && src < c.max_seqs && dst >= 0 && dst < c.max_seqs && src != dst, "slots");
  DTK_REQUIRE(len >= 0 && len <= c.max_len, "len");
  DTK_REQUIRE(eng->refcnt[dst] == 0, "destination lends a shared prefix to other sequences");
  DTK_CK(cudaSetDevice(eng->device));
  drop_share(eng, dst);          // the copy makes dst self-contained
  if (len == 0) return DTK_OK;
  // positions below src's shared length live in its base slot
  const int sl = eng->share_len[src] < len ? eng->share_len[src] : len;
  int r = DTK_OK;
  if (sl > 0) r = copy_kv_range(eng, eng->share_base[src], dst, 0, sl, (cudaStream_t)stream);
  if (r == DTK_OK) r = copy_kv_range(eng, src, dst, sl, len, (cudaStream_t)stream);
  return r;
}

int dtk_seq_share(dtk_engine* eng, int base, int dst, int len, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(base >= 0 && base < c.max_seqs && dst >= 0 && dst < c.max_seqs && base != dst, "slots");
  DTK_REQUIRE(eng->slot_used[base] && eng->slot_used[dst], "slots must be allocated");
  DTK_REQUIRE(len >= 0 && len <= c.max_len, "len");
  DTK_REQUIRE(eng->refcnt[dst] == 0, "destination lends a shared prefix to other sequences");
  DTK_CK(cudaSetDevice(eng->device));
  drop_share(eng, dst);
  if (len == 0) return DTK_OK;
  // one level only: if `base` itself borrows [0, L0) from a root slot, dst borrows that part from the root too
  int root = base, rootlen = len;
  if (eng->share_base[base] >= 0) {
    root = eng->share_base[base];
    rootlen = len < eng->share_len[base] ? len : eng->share_len[base];
  }
  const int s16 = rootlen & ~15;               // the decode kernel streams the cache in 16-position items
  if (s16 > 0) {
    eng->share_base[dst] = root;
    eng->share_len[dst] = s16;
    ++eng->refcnt[root];
    if (eng->shared_upto[root] < s16) eng->shared_upto[root] = s16;
  }
  // the remainder [s16, len) becomes dst's own copy: from the root up to rootlen, from base beyond
  int r = copy_kv_range(eng, root, dst, s16, rootlen, (cudaStream_t)stream);
  if (r == DTK_OK && root != base) r = copy_kv_range(eng, base, dst, rootlen, len, (cudaStream_t)stream);
  return r;
}

namespace {
// embedding splice + every decoder layer over ids[0..T) at positions [start_pos, start_pos + T) of `slot` (KV appended);
// leaves the residual stream in p_x. Shared by dtk_prefill and dtk_score. The dev option "prefill_layers" = n stops the
// stack after layer n (layers >= n write no KV rows).
int decoder_stack(dtk_engine* eng, int slot, const int64_t* ids, int T, int start_pos, const float* img_embeds, int img_start,
                  int n_img, cudaStream_t s) {
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(ids && T > 0, "ids/T");
  DTK_REQUIRE(slot >= 0 && slot < c.max_seqs, "slot");
  DTK_REQUIRE(start_pos >= 0 && start_pos + T <= c.max_len, "start_pos + T exceeds max_len");
  DTK_REQUIRE(start_pos >= eng->share_len[slot], "start_pos lies inside the sequence's shared (read-only) prefix");
  DTK_REQUIRE(start_pos >= eng->shared_upto[slot], "start_pos lies inside a prefix other sequences share from this slot");
  DTK_CK(cudaSetDevice(eng->device));
  uint64_t* lc = &eng->launches;
  const int H = c.hidden, I = c.inter, HD = c.head_dim, qd = c.heads * HD, kd = c.kv_heads * HD;
  DTK_CK(launch_embed_splice(ids, T, start_pos, W(eng, "dec.embed"), H, c.vocab, c.image_token_id, img_embeds, img_start,
                             n_img, eng->p_x, s, lc));
  const int layers = eng->prefill_layers >= 0 ? eng->prefill_layers : c.layers;
  for (int l = 0; l < layers; ++l) {
    DTK_CK(launch_rmsnorm(eng->p_x, H, W(eng, LN("dec.L", l, "norm1")), c.rms_eps, T, H, eng->p_xn, s, lc));
    {
      GemmArgs g{};
      g.A = eng->p_xn; g.lda = H; g.W = W(eng, LN("dec.L", l, "wqkv")); g.ldw = H; g.M = T; g.N = qd + 2 * kd; g.K = H;
      g.out_f32 = eng->p_qkv; g.ldo = qd + 2 * kd;
      DTK_CK(launch_gemm(g, s, lc));
    }
    bf16* kc = kv_layer(eng, slot, l);
    bf16* vc = kc + eng->kv_v_offset;
    DTK_CK(launch_rope_kv_prefill(eng->p_qkv, T, start_pos, c.heads, c.kv_heads, eng->rope_cs, eng->p_q, kc, vc, c.max_len, HD, s, lc));
    {
      AttnArgs a{};
      a.q = eng->p_q; a.k = kc; a.v = vc; a.o = eng->p_att;
      a.q_bs = 0; a.q_hs = HD; a.q_rs = qd;
      a.k_bs = 0; a.k_hs = (int64_t)c.max_len * HD; a.k_rs = HD;
      a.v_bs = 0; a.v_hs = (int64_t)c.max_len * HD; a.v_rs = HD;
      a.o_bs = 0; a.o_hs = HD; a.o_rs = qd;
      a.B = 1; a.heads = c.heads; a.kv_group = c.heads / c.kv_heads; a.Tq = T; a.Tk = start_pos + T; a.q_pos0 = start_pos;
      a.causal = 1; a.head_dim = HD; a.scale = 1.0f / sqrtf((float)HD);
      if (eng->share_len[slot] > 0) {   // keys below the shared length come from the base slot
        a.k2 = kv_layer(eng, eng->share_base[slot], l);
        a.v2 = a.k2 + eng->kv_v_offset;
        a.split_row = eng->share_len[slot];
      }
      DTK_CK(launch_flash_attn(a, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->p_att; g.lda = qd; g.W = W(eng, LN("dec.L", l, "wo")); g.ldw = qd; g.M = T; g.N = H; g.K = qd;
      g.resid = eng->p_x; g.ldr = H; g.out_f32 = eng->p_x; g.ldo = H;
      DTK_CK(launch_gemm(g, s, lc));
    }
    DTK_CK(launch_rmsnorm(eng->p_x, H, W(eng, LN("dec.L", l, "norm2")), c.rms_eps, T, H, eng->p_xn, s, lc));
    {
      GemmArgs g{};
      g.A = eng->p_xn; g.lda = H; g.W = W(eng, LN("dec.L", l, "wgu")); g.ldw = H; g.M = T; g.N = 2 * I; g.K = H;
      g.glu = 1; g.out_bf16 = eng->p_h; g.ldo = I;
      DTK_CK(launch_gemm(g, s, lc));
    }
    {
      GemmArgs g{};
      g.A = eng->p_h; g.lda = I; g.W = W(eng, LN("dec.L", l, "wd")); g.ldw = I; g.M = T; g.N = H; g.K = I;
      g.resid = eng->p_x; g.ldr = H; g.out_f32 = eng->p_x; g.ldo = H;
      DTK_CK(launch_gemm(g, s, lc));
    }
  }
  return DTK_OK;
}
}  // namespace

int dtk_prefill(dtk_engine* eng, int slot, const int64_t* ids, int T, int start_pos, const float* img_embeds,
                int img_start, int n_img, float* last_logits, float* all_logits, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  cudaStream_t s = (cudaStream_t)stream;
  uint64_t* lc = &eng->launches;
  const int H = c.hidden;
  int r = decoder_stack(eng, slot, ids, T, start_pos, img_embeds, img_start, n_img, s);
  if (r != DTK_OK) return r;
  if (last_logits) {  // final RMSNorm + lm_head on the last row only (reference computes all T rows, v1/modeling:251-257)
    GemvArgs g{};
    g.mode = GEMV_STORE; g.W = W(eng, "dec.lm_head"); g.N = c.vocab; g.K = H;
    g.x = eng->p_x + (int64_t)(T - 1) * H; g.x_stride = H; g.norm_w = W(eng, "dec.norm"); g.eps = c.rms_eps;
    g.out = last_logits; g.out_stride = c.vocab; g.B = 1;
    DTK_CK(launch_gemv(g, s, lc));
  }
  if (all_logits) {
    DTK_CK(launch_rmsnorm(eng->p_x, H, W(eng, "dec.norm"), c.rms_eps, T, H, eng->p_xn, s, lc));
    GemmArgs g{};
    g.A = eng->p_xn; g.lda = H; g.W = W(eng, "dec.lm_head"); g.ldw = H; g.M = T; g.N = c.vocab; g.K = H;
    g.out_f32 = all_logits; g.ldo = c.vocab;
    DTK_CK(launch_gemm(g, s, lc));
  }
  return DTK_OK;
}

int dtk_score(dtk_engine* eng, int slot, const int64_t* ids, int T, int start_pos, const float* img_embeds, int img_start,
              int n_img, const int64_t* targets, float* logprob, float* lse, float* all_logits, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(targets && logprob, "targets/logprob");
  cudaStream_t s = (cudaStream_t)stream;
  uint64_t* lc = &eng->launches;
  const int H = c.hidden;
  int r = decoder_stack(eng, slot, ids, T, start_pos, img_embeds, img_start, n_img, s);
  if (r != DTK_OK) return r;
  // first scoring call: partials workspace for max_len rows (engines that never score do not pay it)
  if (!eng->lse_part) DTK_ALLOC(eng->lse_part, (int64_t)c.max_len * ((c.vocab + LSE_TILE - 1) / LSE_TILE));
  if (!eng->lse_tgt) DTK_ALLOC(eng->lse_tgt, c.max_len);
  DTK_CK(launch_rmsnorm(eng->p_x, H, W(eng, "dec.norm"), c.rms_eps, T, H, eng->p_xn, s, lc));
  GemmLseArgs g{};
  g.A = eng->p_xn; g.lda = H; g.W = W(eng, "dec.lm_head"); g.ldw = H; g.M = T; g.N = c.vocab; g.K = H;
  g.out_f32 = all_logits; g.ldo = c.vocab;
  g.targets = targets; g.part = eng->lse_part; g.tgt = eng->lse_tgt;
  DTK_CK(launch_gemm_lse(g, s, lc));
  DTK_CK(launch_lse_merge(eng->lse_part, eng->lse_tgt, targets, T, c.vocab, logprob, lse, s, lc));
  return DTK_OK;
}

// Validates row i of a decode step or loop (slot in range, position below max_len and past every shared prefix: the
// slot's own borrowed one and any it lends) and fills its StateArgs entry, including the prefix it reads through.
static int fill_row(dtk_engine* eng, StateArgs& st, int i, int slot, int position) {
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(slot >= 0 && slot < c.max_seqs, "slot");
  DTK_REQUIRE(position >= 0 && position < c.max_len, "position exceeds max_len");
  DTK_REQUIRE(position >= eng->share_len[slot] && position >= eng->shared_upto[slot],
              "position lies inside a shared prefix (one the slot borrows, or one it lends to other sequences)");
  st.slots[i] = slot;
  st.pos[i] = position;
  st.share_slot[i] = eng->share_base[slot] >= 0 ? eng->share_base[slot] : slot;
  st.share_len[i] = eng->share_len[slot];
  return DTK_OK;
}

int dtk_decode(dtk_engine* eng, const int* slots, const int* positions, const int64_t* ids, int B, float* logits,
               void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(slots && positions && ids && logits, "null pointer");
  DTK_REQUIRE(B > 0 && B <= eng->cfg.max_batch, "B exceeds max_batch");
  StateArgs st{};
  st.n = B;
  for (int i = 0; i < B; ++i)
    if (int r = fill_row(eng, st, i, slots[i], positions[i])) return r;
  DTK_CK(cudaSetDevice(eng->device));
  cudaStream_t s = (cudaStream_t)stream;
  set_state_kernel<<<1, 64, 0, s>>>(st, eng->d_slots, eng->d_pos, eng->d_tok, eng->d_share_slot, eng->d_share_len, eng->d_active,
                                    eng->d_row_step, eng->d_row_seq);
  ++eng->launches;
  DTK_CK(cudaGetLastError());
  set_cascade(eng, st);
  return decode_launches(eng, B, ids, logits, s);
}

int dtk_sample(dtk_engine* eng, const float* logits, int B, const dtk_sampling* params, const int* suppress,
               const uint32_t* steps, const uint32_t* seq_ids, int64_t* out_ids, float* probs_out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(logits && params && B > 0 && B <= eng->cfg.max_batch, "logits/params/B");
  DTK_CK(cudaSetDevice(eng->device));
  SampleArgs a;
  fill_sample_args(eng, a, logits, B, *params);
  if (probs_out) { a.scratch = probs_out; a.want_probs = 1; }
  a.out_ids = out_ids;
  for (int i = 0; i < B; ++i) {
    a.seq[i].suppress = suppress ? suppress[i] : 0;
    a.seq[i].step = steps ? steps[i] : 0;
    a.seq[i].seq_id = seq_ids ? seq_ids[i] : (uint32_t)i;
  }
  if (eng->proc_B > 0) {
    DTK_REQUIRE(B <= eng->proc_B, "B exceeds the rows given to dtk_set_processors");
    DTK_CK(launch_sample_proc(a, proc_args(eng), (cudaStream_t)stream, &eng->launches));
  } else {
    DTK_CK(launch_sample(a, (cudaStream_t)stream, &eng->launches));
  }
  return DTK_OK;
}

int dtk_set_processors(dtk_engine* eng, const dtk_processors* proc, int B, const int32_t* hist_ids, const int32_t* hist_len,
                       const int32_t* eos_min_len, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B == 0, "processors cannot change inside a generation loop");
  if (!proc) { eng->proc_B = 0; return DTK_OK; }
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(B > 0 && B <= c.max_batch && B <= 64, "B outside [1, max_batch]");
  DTK_REQUIRE(hist_len, "null history lengths");
  int64_t n = 0;
  for (int b = 0; b < B; ++b) n += hist_len[b] > 0 ? hist_len[b] : 0;
  DTK_REQUIRE(n == 0 || hist_ids, "null history ids");
  SampleProcTable t;
  std::vector<int> hist;
  std::string why;
  if (!fill_proc_table(*proc, B, c.vocab, c.max_len, hist_ids, hist_len, eos_min_len, t, hist, why)) {
    eng->err = "invalid argument: " + why;
    return DTK_ERR_INVALID;
  }
  DTK_CK(cudaSetDevice(eng->device));
  if (!eng->d_proc_tab) {
    DTK_ALLOC(eng->d_proc_tab, 1);
    DTK_ALLOC(eng->d_hist, (int64_t)c.max_batch * c.max_len);
    DTK_ALLOC(eng->d_hist_len, c.max_batch);
  }
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<int> lens(hist_len, hist_len + B);
  // pageable sources: the copies are staged before the calls return, so the host vectors may go out of scope
  DTK_CK(cudaMemcpyAsync(eng->d_proc_tab, &t, sizeof(t), cudaMemcpyHostToDevice, s));
  DTK_CK(cudaMemcpyAsync(eng->d_hist, hist.data(), hist.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  DTK_CK(cudaMemcpyAsync(eng->d_hist_len, lens.data(), lens.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  DTK_CK(cudaStreamSynchronize(s));
  eng->proc_B = B;
  return DTK_OK;
}

int dtk_gen_begin(dtk_engine* eng, const int* slots, const int* positions, const int64_t* first_ids_host, int B,
                  const dtk_sampling* params, const uint32_t* seq_ids, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(slots && positions && first_ids_host && params, "null pointer");
  DTK_REQUIRE(B > 0 && B <= c.max_batch, "B exceeds max_batch");
  DTK_CK(cudaSetDevice(eng->device));
  cudaStream_t s = (cudaStream_t)stream;
  StateArgs st{};
  st.n = B; st.have_tok = 1;
  for (int i = 0; i < B; ++i) {
    if (int r = fill_row(eng, st, i, slots[i], positions[i])) return r;
    st.tok[i] = first_ids_host[i]; st.seq[i] = seq_ids ? seq_ids[i] : (uint32_t)i;
  }
  set_cascade(eng, st);
  set_state_kernel<<<1, 64, 0, s>>>(st, eng->d_slots, eng->d_pos, eng->d_tok, eng->d_share_slot, eng->d_share_len, eng->d_active,
                                    eng->d_row_step, eng->d_row_seq);
  reset_gen_kernel<<<1, 1, 0, s>>>(eng->d_gen, eng->d_counters + (int64_t)c.max_batch * c.heads, params->seed);
  eng->launches += 2;
  DTK_CK(cudaGetLastError());
  DTK_CK(cudaStreamSynchronize(s));
  std::memset(eng->host_ring, 0, (size_t)(eng->ring + 1) * 64 * sizeof(unsigned long long));  // stamps restart at step 1
  eng->row_active.assign(64, 0);
  std::fill(eng->row_active.begin(), eng->row_active.begin() + B, 1);
  eng->admit_stamp.assign(64, 0u);

  eng->gen_B = B;
  eng->gen_params = *params;
  eng->gen_stream = s;
  {  // sampler arguments of the loop (suppress = 0; RNG counter row_step + step on stream row_seq, set above to 1 and seq_ids)
    SampleArgs& a = eng->gen_sample;
    fill_sample_args(eng, a, eng->d_logits, B, *params);
    a.active = eng->d_active; a.row_step = eng->d_row_step; a.row_seq = eng->d_row_seq;
    a.gen_tok = eng->d_tok; a.gen_pos = eng->d_pos; a.gen_step = eng->d_gen; a.seed_dev = eng->d_gen + 1; a.seed = 0;
    a.host_ring = eng->dev_ring; a.ring = eng->ring;
    a.done_counter = eng->d_counters + (int64_t)c.max_batch * c.heads;
  }
  DTK_REQUIRE(eng->proc_B == 0 || B <= eng->proc_B, "B exceeds the rows given to dtk_set_processors");
  eng->gen_proc = eng->proc_B > 0;
  eng->gen_mega = (B == 1 && eng->decode_impl == 1 && eng->mega_ok);
  // the fused argmax of the persistent kernel knows only the bad token: processors take the token from the sampler
  eng->gen_fused = eng->gen_mega && eng->fuse_greedy && !eng->gen_sample.do_sample && !eng->gen_proc;
  if (eng->gen_mega) {  // one cooperative launch (+ sampler when sampling) per token: no graph needed
    eng->gen_graph = nullptr;
    return DTK_OK;
  }
  // graph key: everything baked into kernel arguments
  char key[256];
  std::snprintf(key, sizeof(key), "B%d|t%.9g|p%.17g|k%d|s%d|b%d|e%d", B, (double)params->temperature,
                (double)params->top_p, params->top_k, params->do_sample, params->bad_token, params->begin_suppress_token);
  std::string skey(key);
  skey += "|g" + std::to_string(eng->decode_gemm_min_batch) + "|i" + std::to_string(get_gemm_impl());
  skey += "|c" + std::to_string(eng->cas_slot) + ":" + std::to_string(eng->cas_len);   // shared-prefix attention bakes slot and length in
  if (eng->gen_proc) skey += "|P";   // processor tables and histories are read from engine buffers at replay
  auto it = eng->graphs.find(skey);
  if (it == eng->graphs.end()) {
    cudaGraph_t graph = nullptr;
    uint64_t before = eng->launches;
    if (!eng->cap_stream) DTK_CK(cudaStreamCreateWithFlags(&eng->cap_stream, cudaStreamNonBlocking));
    cudaStream_t cs = eng->cap_stream;
    DTK_CK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    int r = decode_launches(eng, B, nullptr, eng->d_logits, cs);
    if (r == DTK_OK) {
      cudaError_t e = launch_gen_sample(eng, cs);
      if (e != cudaSuccess) { eng->err = std::string("launch_sample: ") + cudaGetErrorString(e); r = DTK_ERR_CUDA; }
    }
    cudaError_t ce = cudaStreamEndCapture(cs, &graph);
    eng->launches = before;  // captured launches are counted per replay
    if (r != DTK_OK) { if (graph) cudaGraphDestroy(graph); return r; }
    if (ce != cudaSuccess) { eng->err = std::string("cudaStreamEndCapture: ") + cudaGetErrorString(ce); return DTK_ERR_CUDA; }
    cudaGraphExec_t exec = nullptr;
    DTK_CK(cudaGraphInstantiate(&exec, graph, 0));
    cudaGraphDestroy(graph);
    if (eng->graphs.size() >= 64) {  // bound the cache
      for (auto& g : eng->graphs) cudaGraphExecDestroy(g.second);
      eng->graphs.clear();
    }
    it = eng->graphs.emplace(skey, exec).first;
  }
  eng->gen_graph = it->second;
  return DTK_OK;
}

int dtk_gen_step(dtk_engine* eng, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B > 0, "dtk_gen_begin not called");
  if (eng->gen_mega) {
    int r = decode_launches(eng, 1, nullptr, eng->d_logits, (cudaStream_t)stream);
    if (r != DTK_OK) return r;
    if (!eng->gen_fused) DTK_CK(launch_gen_sample(eng, (cudaStream_t)stream));
    return DTK_OK;
  }
  DTK_REQUIRE(eng->gen_graph != nullptr, "dtk_gen_begin not called");
  DTK_CK(cudaGraphLaunch(eng->gen_graph, (cudaStream_t)stream));
  const bool gemm_path = eng->decode_gemm_min_batch > 0 && eng->gen_B >= eng->decode_gemm_min_batch;
  eng->launches += gemm_path ? (uint64_t)eng->cfg.layers * (9 + (eng->cas_len > 0 ? 1 : 0)) + 4 : (uint64_t)eng->cfg.layers * 5 + 3;   // kernels per replay
  return DTK_OK;
}

// Spins until the host-ring entry *e carries the stamp `want` in its upper half (one 8-byte device store) and returns its
// lower half, the token. Every 1024 spins it checks the loop's stream for an error, for running idle without the store,
// and for 60 s gone since t0. With `ring`, a larger stamp means the device overwrote the entry a whole ring ahead.
static int wait_stamped(dtk_engine* eng, volatile const unsigned long long* e, unsigned long long want, bool ring,
                        const char* what, std::chrono::steady_clock::time_point t0, int32_t* token_out) {
  uint64_t spins = 0;
  unsigned long long v;
  while (((v = *e) >> 32) != want) {
    if (ring && (v >> 32) > want) {
      eng->err = "token ring overrun: dtk_gen_wait lagged more than the ring depth behind dtk_gen_step";
      return DTK_ERR_INVALID;
    }
    if ((++spins & 0x3ff) == 0) {
      cudaError_t q = cudaStreamQuery(eng->gen_stream);
      if (q != cudaSuccess && q != cudaErrorNotReady) {
        eng->err = std::string("stream error while waiting for ") + what + ": " + cudaGetErrorString(q);
        return DTK_ERR_CUDA;
      }
      if (q == cudaSuccess && (*e >> 32) != want) {
        eng->err = std::string("stream idle but ") + what + " was never published";
        return DTK_ERR_INVALID;
      }
      if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(60)) {
        eng->err = std::string("timeout waiting for ") + what;
        return DTK_ERR_CUDA;
      }
    }
  }
  *token_out = (int32_t)(uint32_t)(v & 0xffffffffull);
  return DTK_OK;
}

int dtk_gen_wait(dtk_engine* eng, int64_t step, int32_t* tokens_out_host) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B > 0 && step >= 0 && tokens_out_host, "gen state/step/out");
  // every sequence's entry of this step carries the stamp step + 1
  volatile const unsigned long long* row = eng->host_ring + (size_t)(step % eng->ring) * eng->gen_B;
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < eng->gen_B; ++i)
    if (int r = wait_stamped(eng, row + i, (unsigned long long)(step + 1), true, "the generated token", t0,
                             tokens_out_host + i))
      return r;
  return DTK_OK;
}

int dtk_gen_admit(dtk_engine* eng, int row, int slot, int position, const float* logits, uint32_t seq_id,
                  const int32_t* hist_ids, int hist_len, int eos_min_len, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(eng->gen_B > 0, "dtk_gen_begin not called");
  if (eng->gen_mega) {
    eng->err = "unsupported: the batch-1 persistent generation loop takes no admissions";
    return DTK_ERR_UNSUPPORTED;
  }
  DTK_REQUIRE((cudaStream_t)stream == eng->gen_stream, "admissions are enqueued on the loop's stream");
  DTK_REQUIRE(row >= 0 && row < eng->gen_B, "row outside the loop's rows");
  DTK_REQUIRE(!eng->row_active[row], "row is active (dtk_gen_retire it first)");
  DTK_REQUIRE(slot >= 0 && slot < c.max_seqs && eng->slot_used[slot], "slot is not allocated");
  StateArgs st{};
  if (int r = fill_row(eng, st, 0, slot, position)) return r;
  DTK_REQUIRE(logits, "null logits");
  const int share_slot = st.share_slot[0], share_len = st.share_len[0];
  // the shared-prefix attention of this loop's graph reads one baked prefix for every row
  DTK_REQUIRE(eng->cas_len == 0 || (share_slot == eng->cas_slot && share_len == eng->cas_len),
              "the loop runs shared-prefix (cascade) attention over another prefix than the slot borrows");
  if (eng->gen_proc) {
    DTK_REQUIRE(hist_len > 0 && hist_len <= c.max_len && hist_ids, "processors need the row's history (the prompt)");
    for (int i = 0; i < hist_len; ++i) DTK_REQUIRE(hist_ids[i] >= 0 && hist_ids[i] < c.vocab, "history id outside [0, vocab)");
  }
  DTK_CK(cudaSetDevice(eng->device));
  cudaStream_t s = (cudaStream_t)stream;
  SampleArgs a = eng->gen_sample;   // the loop's parameters, without its state: counter 0 on the request's stream
  a.gen_tok = nullptr; a.gen_pos = nullptr; a.gen_step = nullptr; a.host_ring = nullptr; a.done_counter = nullptr;
  a.active = nullptr; a.row_step = nullptr; a.row_seq = nullptr; a.out_ids = nullptr;
  a.seq[row].suppress = 1; a.seq[row].step = 0; a.seq[row].seq_id = seq_id;
  SampleAdmit m{};
  m.logits = logits; m.row = row; m.slot = slot; m.pos = position; m.share_slot = share_slot; m.share_len = share_len;
  m.hist_len = hist_len; m.eos_min = eos_min_len; m.seq_id = seq_id; m.stamp = ++eng->admit_stamp[row];
  m.slots = eng->d_slots; m.posv = eng->d_pos; m.tok = eng->d_tok; m.share_slots = eng->d_share_slot;
  m.share_lens = eng->d_share_len; m.active = eng->d_active; m.row_step = eng->d_row_step; m.row_seq = eng->d_row_seq;
  m.gen_step = eng->d_gen; m.tab = eng->d_proc_tab; m.mailbox = eng->dev_ring + (size_t)eng->ring * 64;
  SampleProc q{};
  if (eng->gen_proc) {
    if (!eng->h_admit_hist) {
      DTK_CK(cudaHostAlloc((void**)&eng->h_admit_hist, (size_t)c.max_batch * c.max_len * sizeof(int), cudaHostAllocDefault));
      eng->admit_ev.assign(c.max_batch, nullptr);
      for (auto& e : eng->admit_ev) DTK_CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    // the row's staging buffer was last read by its previous admission's copy, which ran before that request's first
    // step: in a loop that waits for its steps this event has long passed
    DTK_CK(cudaEventSynchronize(eng->admit_ev[row]));
    int* stage = eng->h_admit_hist + (size_t)row * c.max_len;
    std::memcpy(stage, hist_ids, (size_t)hist_len * sizeof(int));
    DTK_CK(cudaMemcpyAsync(eng->d_hist + (size_t)row * c.max_len, stage, (size_t)hist_len * sizeof(int), cudaMemcpyHostToDevice, s));
    DTK_CK(cudaEventRecord(eng->admit_ev[row], s));
    q = proc_args(eng);
  }
  DTK_CK(launch_sample_admit(a, eng->gen_proc ? &q : nullptr, m, s, &eng->launches));
  eng->row_active[row] = 1;
  return DTK_OK;
}

int dtk_gen_retire(dtk_engine* eng, int row, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B > 0, "dtk_gen_begin not called");
  if (eng->gen_mega) {
    eng->err = "unsupported: the batch-1 persistent generation loop has no row activity";
    return DTK_ERR_UNSUPPORTED;
  }
  DTK_REQUIRE((cudaStream_t)stream == eng->gen_stream, "retirements are enqueued on the loop's stream");
  DTK_REQUIRE(row >= 0 && row < eng->gen_B, "row outside the loop's rows");
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(cudaMemsetAsync(eng->d_active + row, 0, sizeof(int), (cudaStream_t)stream));
  eng->row_active[row] = 0;
  return DTK_OK;
}

int dtk_gen_first(dtk_engine* eng, int row, int32_t* token_out_host) {
  if (!eng) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B > 0 && token_out_host, "gen state/out");
  DTK_REQUIRE(row >= 0 && row < eng->gen_B && eng->admit_stamp[row] > 0, "row was not admitted in this loop");
  return wait_stamped(eng, eng->host_ring + (size_t)eng->ring * 64 + row, eng->admit_stamp[row], false,
                      "an admitted row's first token", std::chrono::steady_clock::now(), token_out_host);
}

int dtk_gen_end(dtk_engine* eng) {
  if (!eng) return DTK_ERR_INVALID;
  if (eng->gen_B > 0) {
    DTK_CK(cudaSetDevice(eng->device));
    DTK_CK(cudaStreamSynchronize(eng->gen_stream));
  }
  eng->gen_graph = nullptr;
  eng->gen_mega = false;
  eng->gen_fused = false;
  eng->gen_proc = false;
  eng->gen_B = 0;
  return DTK_OK;
}

int dtk_set_option(dtk_engine* eng, const char* key, int64_t value) {
  if (!eng || !key) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->gen_B == 0, "options cannot change inside a generation loop");
  if (std::strcmp(key, "decode_impl") == 0) {
    DTK_REQUIRE(value == 0 || value == 1, "decode_impl must be 0 (per-op) or 1 (persistent)");
    eng->decode_impl = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "decode_gemm_min_batch") == 0) {  // 0 = never; default 4
    DTK_REQUIRE(value >= 0 && value <= 64, "decode_gemm_min_batch must be in 0..64");
    eng->decode_gemm_min_batch = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "gemm_impl") == 0) {  // process-wide dev switch: 0 = mma.sync, 1 / 2 = wgmma where supported
    DTK_REQUIRE(value >= 0 && value <= 2, "gemm_impl must be 0..2");
    set_gemm_impl((int)value);
    return DTK_OK;
  }
  if (std::strcmp(key, "cascade_attn") == 0) {  // 1 (default) = shared-prefix attention for batched steps whose rows share one prefix
    eng->cascade_attn = value ? 1 : 0;
    return DTK_OK;
  }
  if (std::strcmp(key, "gemm_swap_split") == 0) {  // process-wide dev switch: split-K factor of the batched-decode GEMM
    DTK_REQUIRE(value >= 0 && value <= 8, "gemm_swap_split must be 0 (heuristic) .. 8");
    set_gemm_swap_split((int)value);
    return DTK_OK;
  }
  if (std::strcmp(key, "sample_impl") == 0) {  // process-wide: 0 = register-resident sampler when V fits, 1 = generic kernel
    DTK_REQUIRE(value == 0 || value == 1, "sample_impl must be 0 or 1");
    set_sample_impl((int)value);
    return DTK_OK;
  }
  if (std::strcmp(key, "mega_flags") == 0) {  // dev only (timing experiments; results are garbage when set)
    eng->mega_flags = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "mega_debug") == 0) {
    eng->mega_debug = value ? 1 : 0;
    return DTK_OK;
  }
  if (std::strcmp(key, "attn_impl") == 0) {  // ViT attention: 1 (default) = wgmma, 0 = mma.sync
    DTK_REQUIRE(value == 0 || value == 1, "attn_impl must be 0 or 1");
    eng->attn_impl = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "fuse_greedy") == 0) {  // 1 (default): greedy generation loops take the argmax in the decode kernel's tail
    eng->fuse_greedy = value ? 1 : 0;
    return DTK_OK;
  }
  if (std::strcmp(key, "vit_graph") == 0) {  // 1 (default) = ViT chunks replayed from CUDA graphs, 0 = direct launches
    eng->vit_graph = value ? 1 : 0;
    return DTK_OK;
  }
  if (std::strcmp(key, "mega_variant") == 0) {  // dev A/B switches of the persistent kernel (results identical)
    eng->mega_variant = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "decode_fp8") == 0) {  // batch-1 persistent decode streams the layer matrices as e4m3 (1) or bf16 (0) tiles
    DTK_REQUIRE(value == 0 || value == 1, "decode_fp8 must be 0 or 1");
    DTK_REQUIRE(eng->mega_ok, "decode_fp8: the persistent decode kernel is unavailable on this device");
    if ((int)value == eng->decode_fp8) return DTK_OK;
    return mega_layer_tiles(eng, value == 1);
  }
  if (std::strcmp(key, "decode_pack") == 0) {  // batch-1 persistent decode streams every matrix as packed 13-bit (1) or bf16 (0) tiles
    DTK_REQUIRE(value == 0 || value == 1, "decode_pack must be 0 or 1");
    DTK_REQUIRE(eng->mega_ok, "decode_pack: the persistent decode kernel is unavailable on this device");
    if ((int)value == eng->decode_pack) return DTK_OK;
    return value == 1 ? mega_pack_tiles(eng) : mega_layer_tiles(eng, false);
  }
  if (std::strcmp(key, "mega_nslots") == 0) {  // dev: smaller ring (8 / 16) for A/B runs of the stream's depth
    eng->mega_nslots = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "mega_trace_layer") == 0) {  // dev: per-tile clock trace of this layer (-1 = off); needs mega_debug
    eng->mega_trace_layer = (int)value;
    return DTK_OK;
  }
  if (std::strcmp(key, "prefill_layers") == 0) {  // dev: prefill / score run only the first n decoder layers (-1 = all)
    DTK_REQUIRE(value >= -1 && value <= eng->cfg.layers, "prefill_layers must be in -1..layers");
    eng->prefill_layers = (int)value;
    return DTK_OK;
  }
  eng->err = std::string("unknown option ") + key;
  return DTK_ERR_INVALID;
}

int dtk_get_option(dtk_engine* eng, const char* key, int64_t* value) {
  if (!eng || !key || !value) return DTK_ERR_INVALID;
  if (std::strcmp(key, "decode_impl") == 0) { *value = eng->decode_impl; return DTK_OK; }
  if (std::strcmp(key, "decode_persistent") == 0) { *value = (eng->decode_impl == 1 && eng->mega_ok) ? 1 : 0; return DTK_OK; }
  if (std::strcmp(key, "gemm_impl") == 0) { *value = get_gemm_impl(); return DTK_OK; }
  if (std::strcmp(key, "decode_gemm_min_batch") == 0) { *value = eng->decode_gemm_min_batch; return DTK_OK; }
  if (std::strcmp(key, "cascade_attn") == 0) { *value = eng->cascade_attn; return DTK_OK; }
  if (std::strcmp(key, "sample_impl") == 0) { *value = get_sample_impl(); return DTK_OK; }
  if (std::strcmp(key, "mega_flags") == 0) { *value = eng->mega_flags; return DTK_OK; }
  if (std::strcmp(key, "mega_debug") == 0) { *value = eng->mega_debug; return DTK_OK; }
  if (std::strcmp(key, "mega_variant") == 0) { *value = eng->mega_variant; return DTK_OK; }
  if (std::strcmp(key, "decode_fp8") == 0) { *value = eng->decode_fp8; return DTK_OK; }
  if (std::strcmp(key, "decode_pack") == 0) { *value = eng->decode_pack; return DTK_OK; }
  if (std::strcmp(key, "decode_pack_escapes") == 0) { *value = eng->pk_escapes; return DTK_OK; }
  if (std::strcmp(key, "prefill_layers") == 0) { *value = eng->prefill_layers; return DTK_OK; }
  if (std::strcmp(key, "decode_weight_bytes") == 0) {
    *value = (int64_t)(eng->decode_pack ? decode_pack_weight_bytes(eng) : decode_weight_bytes(eng->cfg, eng->decode_fp8 != 0));
    return DTK_OK;
  }
  eng->err = std::string("unknown option ") + key;
  return DTK_ERR_INVALID;
}

// ---- kernel-level test hooks ---------------------------------------------------------------
int dtk_dbg_mega_times(dtk_engine* eng, long long* out_host, int max_values) {
  if (!eng || !out_host) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->d_dbg != nullptr, "persistent kernel unavailable");
  const int n = eng->mega_grid * (eng->cfg.layers * 5 + 1) * 4;
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(cudaDeviceSynchronize());
  DTK_CK(cudaMemcpy(out_host, eng->d_dbg, (size_t)(n < max_values ? n : max_values) * sizeof(long long), cudaMemcpyDeviceToHost));
  return n;
}

int dtk_dbg_mega_trace(dtk_engine* eng, long long* out_host, int max_values) {
  if (!eng || !out_host) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->d_dbg2 != nullptr, "persistent kernel unavailable");
  const int n = eng->mega_grid * MEGA_DBG2_ROWS * 4;
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(cudaDeviceSynchronize());
  DTK_CK(cudaMemcpy(out_host, eng->d_dbg2, (size_t)(n < max_values ? n : max_values) * sizeof(long long), cudaMemcpyDeviceToHost));
  return n;
}

int dtk_dbg_pack_bytes(dtk_engine* eng, int64_t offset, int64_t nbytes, void* out_host) {
  if (!eng || !out_host) return DTK_ERR_INVALID;
  DTK_REQUIRE(eng->d_tiledpk != nullptr, "decode_pack is off");
  const int64_t total = (int64_t)(decode_pack_weight_bytes(eng) - (uint64_t)eng->pk_escapes * MEGA_PK_ESC_BYTES);
  DTK_REQUIRE(offset >= 0 && nbytes >= 0 && offset + nbytes <= total, "byte range outside the packed tiles");
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(cudaDeviceSynchronize());
  DTK_CK(cudaMemcpy(out_host, eng->d_tiledpk + offset, (size_t)nbytes, cudaMemcpyDeviceToHost));
  return DTK_OK;
}

int dtk_dbg_kv_read(dtk_engine* eng, int slot, int layer, int pos0, int n, void* k_out, void* v_out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(k_out && v_out, "null pointer");
  DTK_REQUIRE(slot >= 0 && slot < c.max_seqs && eng->slot_used[slot], "slot is not allocated");
  DTK_REQUIRE(layer >= 0 && layer < c.layers, "layer");
  DTK_REQUIRE(pos0 >= 0 && n >= 0 && (int64_t)pos0 + n <= c.max_len, "positions outside [0, max_len)");
  DTK_CK(cudaSetDevice(eng->device));
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t HD = c.head_dim;
  const size_t src_pitch = (size_t)c.max_len * HD * sizeof(bf16), dst_pitch = (size_t)n * HD * sizeof(bf16);
  // positions below the slot's shared length resolve to the lending slot, as the decode attention kernels read them
  const int split = std::min(std::max(eng->share_len[slot], pos0), pos0 + n);
  const int parts[2][3] = {{eng->share_base[slot] >= 0 ? eng->share_base[slot] : slot, pos0, split}, {slot, split, pos0 + n}};
  for (const auto& pt : parts) {
    if (pt[2] <= pt[1]) continue;
    const bf16* k = kv_layer(eng, pt[0], layer) + (int64_t)pt[1] * HD;
    const size_t off = (size_t)(pt[1] - pos0) * HD, width = (size_t)(pt[2] - pt[1]) * HD * sizeof(bf16);
    DTK_CK(cudaMemcpy2DAsync(static_cast<bf16*>(k_out) + off, dst_pitch, k, src_pitch, width, c.kv_heads,
                             cudaMemcpyDeviceToDevice, s));
    DTK_CK(cudaMemcpy2DAsync(static_cast<bf16*>(v_out) + off, dst_pitch, k + eng->kv_v_offset, src_pitch, width, c.kv_heads,
                             cudaMemcpyDeviceToDevice, s));
  }
  return DTK_OK;
}

int dtk_dbg_residual_read(dtk_engine* eng, int row0, int n, float* out, void* stream) {
  if (!eng) return DTK_ERR_INVALID;
  const dtk_config& c = eng->cfg;
  DTK_REQUIRE(out, "null pointer");
  DTK_REQUIRE(row0 >= 0 && n >= 0 && (int64_t)row0 + n <= c.max_len, "rows outside [0, max_len)");
  DTK_CK(cudaSetDevice(eng->device));
  DTK_CK(cudaMemcpyAsync(out, eng->p_x + (int64_t)row0 * c.hidden, (size_t)n * c.hidden * sizeof(float),
                         cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return DTK_OK;
}

int dtk_dbg_gemm_impl(int impl) {
  if (impl >= 0) {
    set_gemm_impl(impl & 0xff);
    set_gemm_swap_split((impl >> 8) & 0xf);   // forced split-K factor of the batched-decode tile (0 = heuristic)
  }
  return get_gemm_impl();
}

int dtk_dbg_sample(const float* logits, int B, int V, const dtk_sampling* params, const int* suppress, const uint32_t* steps,
                   const uint32_t* seq_ids, int impl, int64_t* out_ids, float* probs, void* stream) {
  if (!logits || !params || !out_ids || !probs || B < 1 || B > 64 || V < 1 || (impl != 0 && impl != 1)) return DTK_ERR_INVALID;
  SampleArgs a;
  fill_sample_params(a, logits, B, V, *params);
  a.scratch = probs; a.want_probs = 1;
  a.out_ids = out_ids;
  for (int i = 0; i < B; ++i) {
    a.seq[i].suppress = suppress ? suppress[i] : 0;
    a.seq[i].step = steps ? steps[i] : 0;
    a.seq[i].seq_id = seq_ids ? seq_ids[i] : (uint32_t)i;
  }
  const int prev = get_sample_impl();
  set_sample_impl(impl);
  const cudaError_t e = launch_sample(a, (cudaStream_t)stream, nullptr);
  set_sample_impl(prev);
  return e == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_sample_proc(const float* logits, int B, int V, const dtk_sampling* params, const int* suppress, const uint32_t* steps,
                        const uint32_t* seq_ids, int impl, const dtk_processors* proc, const int32_t* hist_ids,
                        const int32_t* hist_len, const int32_t* eos_min_len, int max_len, int64_t* out_ids, float* probs,
                        void* stream) {
  if (!logits || !params || !proc || !hist_len || !out_ids || !probs || B < 1 || B > 64 || V < 1 || max_len < 1 ||
      (impl != 0 && impl != 1))
    return DTK_ERR_INVALID;
  SampleProcTable t;
  std::vector<int> hist;
  std::string why;
  if (!fill_proc_table(*proc, B, V, max_len, hist_ids, hist_len, eos_min_len, t, hist, why)) return DTK_ERR_INVALID;
  SampleArgs a;
  fill_sample_params(a, logits, B, V, *params);
  a.scratch = probs; a.want_probs = 1;
  a.out_ids = out_ids;
  for (int i = 0; i < B; ++i) {
    a.seq[i].suppress = suppress ? suppress[i] : 0;
    a.seq[i].step = steps ? steps[i] : 0;
    a.seq[i].seq_id = seq_ids ? seq_ids[i] : (uint32_t)i;
  }
  SampleProc q{};
  q.hist_stride = max_len;
  cudaError_t e = cudaMalloc((void**)&q.tab, sizeof(SampleProcTable));
  if (e == cudaSuccess) e = cudaMalloc((void**)&q.hist, hist.size() * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc((void**)&q.hist_len, B * sizeof(int));
  cudaStream_t s = (cudaStream_t)stream;
  if (e == cudaSuccess) e = cudaMemcpyAsync((void*)q.tab, &t, sizeof(t), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(q.hist, hist.data(), hist.size() * sizeof(int), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemcpyAsync(q.hist_len, hist_len, B * sizeof(int), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) {
    const int prev = get_sample_impl();
    set_sample_impl(impl);
    e = launch_sample_proc(a, q, s, nullptr);
    set_sample_impl(prev);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);   // the temporary tables are freed below
  cudaFree((void*)q.tab); cudaFree(q.hist); cudaFree(q.hist_len);
  return e == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_gemm(const void* A, const void* Wm, const void* bias, const float* resid, int M, int N, int K, int act,
                 int glu, float* out_f32, void* out_bf16, void* stream) {
  GemmArgs g{};
  g.A = (const bf16*)A; g.lda = K; g.W = (const bf16*)Wm; g.ldw = K; g.M = M; g.N = N; g.K = K;
  g.bias = (const bf16*)bias; g.resid = resid; g.ldr = glu ? N / 2 : N; g.act = act; g.glu = glu;
  g.out_f32 = out_f32; g.out_bf16 = (bf16*)out_bf16; g.ldo = glu ? N / 2 : N;
  return launch_gemm(g, (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_lm_logprob(const void* A, const void* Wm, int M, int N, int K, const int64_t* targets, float* logprob, float* lse,
                       void* stream) {
  if (!A || !Wm || !targets || !logprob || M <= 0 || N <= 0 || K <= 0) return DTK_ERR_INVALID;
  // grow-only partials workspace of this test hook (per device; calls must not overlap)
  static float2* part[64] = {};
  static float* tgt[64] = {};
  static int64_t cap_rows[64] = {}, cap_part[64] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return DTK_ERR_CUDA;
  const int64_t np = (int64_t)M * ((N + LSE_TILE - 1) / LSE_TILE);
  if (np > cap_part[dev] || M > cap_rows[dev]) {
    cudaDeviceSynchronize();
    cudaFree(part[dev]);
    cudaFree(tgt[dev]);
    part[dev] = nullptr; tgt[dev] = nullptr; cap_part[dev] = cap_rows[dev] = 0;
    if (cudaMalloc(&part[dev], np * sizeof(float2)) != cudaSuccess || cudaMalloc(&tgt[dev], (size_t)M * sizeof(float)) != cudaSuccess)
      return DTK_ERR_OOM;
    cap_part[dev] = np; cap_rows[dev] = M;
  }
  GemmLseArgs g{};
  g.A = (const bf16*)A; g.lda = K; g.W = (const bf16*)Wm; g.ldw = K; g.M = M; g.N = N; g.K = K;
  g.targets = targets; g.part = part[dev]; g.tgt = tgt[dev];
  if (launch_gemm_lse(g, (cudaStream_t)stream, nullptr) != cudaSuccess) return DTK_ERR_CUDA;
  return launch_lse_merge(part[dev], tgt[dev], targets, M, N, logprob, lse, (cudaStream_t)stream, nullptr) == cudaSuccess
             ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_flash_attn(const void* q, const void* k, const void* v, void* o, int B, int heads, int Tq, int Tk,
                       int head_dim, int causal, int q_pos0, float scale, void* stream) {
  AttnArgs a{};
  a.q = (const bf16*)q; a.k = (const bf16*)k; a.v = (const bf16*)v; a.o = (bf16*)o;
  const int64_t rs = (int64_t)heads * head_dim;
  a.q_bs = (int64_t)Tq * rs; a.q_hs = head_dim; a.q_rs = rs;
  a.k_bs = (int64_t)Tk * rs; a.k_hs = head_dim; a.k_rs = rs;
  a.v_bs = (int64_t)Tk * rs; a.v_hs = head_dim; a.v_rs = rs;
  a.o_bs = (int64_t)Tq * rs; a.o_hs = head_dim; a.o_rs = rs;
  a.B = B; a.heads = heads; a.kv_group = 1; a.Tq = Tq; a.Tk = Tk; a.q_pos0 = q_pos0; a.causal = causal;
  a.head_dim = head_dim; a.scale = scale;
  return launch_flash_attn(a, (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_attn_tc(const void* qkv, void* vt_scratch, void* o, int B, int heads, int N, float scale, void* stream) {
  if (!qkv || !vt_scratch || !o || B <= 0 || heads <= 0 || N <= 0) return DTK_ERR_INVALID;
  if (!attn_tc_supported()) return DTK_ERR_UNSUPPORTED;
  return launch_attn_tc((const bf16*)qkv, (bf16*)vt_scratch, (bf16*)o, B, heads, N, scale, (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_xattn_tc(const void* q, const void* kv, const int* klen_host, int Tk, void* vt_scratch, void* o, int B, int heads,
                     int N, float scale, void* stream) {
  if (!q || !kv || !klen_host || !vt_scratch || !o || B <= 0 || B > XATTN_MAX_B || heads <= 0 || N <= 0 || Tk <= 0) return DTK_ERR_INVALID;
  for (int b = 0; b < B; ++b) if (klen_host[b] < 1 || klen_host[b] > Tk) return DTK_ERR_INVALID;
  if (!attn_tc_supported()) return DTK_ERR_UNSUPPORTED;
  return launch_xattn_tc((const bf16*)q, (const bf16*)kv, klen_host, Tk, (bf16*)vt_scratch, (bf16*)o, B, heads, N, scale,
                         (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_head_layernorm(const void* x, const void* w, const void* b, float eps, int M, int heads, int hd, void* out, void* stream) {
  if (!x || !w || !b || !out || M <= 0 || heads <= 0) return DTK_ERR_INVALID;
  const int64_t ld = (int64_t)heads * hd;
  return launch_head_layernorm((const bf16*)x, ld, (const bf16*)w, (const bf16*)b, eps, M, heads, hd, (bf16*)out, ld,
                               (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_gemm_gated(const void* A, const void* Wm, const void* bias, const void* gate, const float* resid, int M, int N, int K,
                       int act, float* out_f32, void* stream) {
  if (!A || !Wm || !gate || !out_f32) return DTK_ERR_INVALID;
  GemmArgs g{};
  g.A = (const bf16*)A; g.lda = K; g.W = (const bf16*)Wm; g.ldw = K; g.M = M; g.N = N; g.K = K;
  g.bias = (const bf16*)bias; g.gate = (const bf16*)gate; g.resid = resid; g.ldr = N; g.act = act;
  g.out_f32 = out_f32; g.ldo = N;
  return launch_gemm(g, (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

int dtk_dbg_gemv(const void* Wm, const float* x, const void* norm_w, float eps, int N, int K, int mode, float* out,
                 void* stream) {
  if (mode < 0 || mode > 2) return DTK_ERR_INVALID;
  GemvArgs g{};
  g.mode = mode; g.W = (const bf16*)Wm; g.N = N; g.K = K; g.x = x; g.x_stride = K; g.norm_w = (const bf16*)norm_w;
  g.eps = eps; g.out = out; g.out_stride = N; g.B = 1;
  return launch_gemv(g, (cudaStream_t)stream, nullptr) == cudaSuccess ? DTK_OK : DTK_ERR_CUDA;
}

}  // extern "C"
