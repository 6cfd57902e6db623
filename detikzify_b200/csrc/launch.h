// Host-side launcher declarations (one per kernel family). Each launcher returns the CUDA error
// of the launch and bumps *counter (kernel launches issued; bench.py's gpu_launches).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

typedef __nv_bfloat16 bf16;

namespace dtk {

// ---------------------------------------------------------------- dense GEMM  C = A * W^T
enum { ACT_NONE = 0, ACT_GELU_TANH = 1, ACT_GELU_ERF = 2 };

struct GemmArgs {
  const bf16* A;              // [M, K] bf16, row stride lda (elements)
  int64_t lda;
  int a_rows_per_batch;       // 0 = plain; else row m lives at A + (m / rpb) * a_batch_stride + (m % rpb) * lda
  int64_t a_batch_stride;
  const bf16* W;              // [N, K] bf16 row-major (K contiguous), row stride ldw
  int64_t ldw;
  int M, N, K;                // K % 8 == 0, N % 2 == 0
  // epilogue: v = acc (+bias[n]) ; v = act(v) ; (+ rowbias[m % rowbias_mod, n]) ; (+ resid[m, n])
  const bf16* bias;           // [N] or null
  const bf16* rowbias;        // [rowbias_mod, N] or null (ViT position embedding)
  int rowbias_mod;
  const float* resid;         // fp32 [M, ldr] or null (may alias out_f32)
  int64_t ldr;
  int act;
  int glu;                    // 1: columns come in (gate, up) pairs -> out[m, n/2] = silu(gate) * up
  float* out_f32;             // exactly one of out_f32 / out_bf16 is non-null
  bf16* out_bf16;
  int64_t ldo;
  // gated residual (TikZero cross layers): v = sigmoid(*gate) * act(acc + bias) before the residual add; null = off
  const bf16* gate;
};
cudaError_t launch_gemm(const GemmArgs& a, cudaStream_t s, uint64_t* counter);   // dispatches wgmma / mma.sync
cudaError_t launch_gemm_mma(const GemmArgs& a, cudaStream_t s, uint64_t* counter);
cudaError_t launch_gemm_tc(const GemmArgs& a, cudaStream_t s, uint64_t* counter);
bool gemm_tc_supported(const GemmArgs& a);
// lm_head GEMM with a log-softmax epilogue (persistent 128 x 256 wgmma kernel, every M): for each row m < M and 256-column
// tile j of C = A W^T, part[m * ceil(N / 256) + j] = {max, sum exp(v - max)} over the tile's columns n < N, and
// tgt[m] = C[m, targets[m]] when targets[m] is in [0, N). C itself is stored only when out_f32 is non-null (ldo = N); the
// other epilogue fields of GemmArgs must be off. Deterministic: no atomics, fixed reduction order.
struct GemmLseArgs : GemmArgs {
  const int64_t* targets;     // [M] (any value; outside [0, N) = no target)
  float2* part;               // [M, ceil(N / 256)]
  float* tgt;                 // [M]
};
constexpr int LSE_TILE = 256;
cudaError_t launch_gemm_lse(const GemmLseArgs& a, cudaStream_t s, uint64_t* counter);
// folds the partials of each row in a fixed order: lse[m] (may be null) = log sum exp C[m, :N],
// logprob[m] = tgt[m] - lse[m] when targets[m] is in [0, N), else 0
cudaError_t launch_lse_merge(const float2* part, const float* tgt, const int64_t* targets, int M, int N, float* logprob,
                             float* lse, cudaStream_t s, uint64_t* counter);
// FP8 weight operand of the batched-decode GEMM: one layer matrix as decode tiles (launch_retile_f8, row order tile_row)
struct GemmF8 {
  const uint8_t* tiles;       // [groups][tpg] e4m3 tiles of MEGA_F8_TILE_BYTES
  const int8_t* exps;         // [groups][16] row exponents k_r
  int groups, tpg, mode, hd;  // MegaMat geometry and row permutation (hd: head_dim of TILE_ROPE)
};
// out = A W~^T on the swapped-operand wgmma tile (4 <= M < 64) with W~ = code x 2^k_r from the tiles: the same result bits as
// launch_gemm on a bf16 W holding W~, with the same split-K cuts (N, K, glu and the epilogue fields as for launch_gemm;
// W / ldw unused; glu requires TILE_GLU tiles). Other M, an activation or a row bias: cudaErrorInvalidValue.
cudaError_t launch_gemm_swap_f8(const GemmArgs& a, const GemmF8& w, cudaStream_t s, uint64_t* counter);
void set_gemm_swap_split(int v);    // dev: 0 (default) = heuristic split-K factor of the swapped tile, 1..8 = forced
void set_gemm_impl(int impl);   // 0 = mma.sync everywhere, 1 = wgmma one 128 x 128 tile per CTA, 2 = persistent 128 x 256 wgmma (process-wide dev switch)
int get_gemm_impl();

// ---------------------------------------------------------------- flash attention (mma.sync)
struct AttnArgs {
  const bf16 *q, *k, *v;
  bf16* o;
  int64_t q_bs, q_hs, q_rs;   // batch / head / row strides in elements
  int64_t k_bs, k_hs, k_rs;
  int64_t v_bs, v_hs, v_rs;
  int64_t o_bs, o_hs, o_rs;
  int B, heads, kv_group;     // kv head = head / kv_group
  int Tq, Tk;
  int q_pos0;                 // causal: query i sits at position q_pos0 + i; key j visible iff j <= pos
  int causal;
  int head_dim;               // 72, 64 or 128
  float scale;
  // shared KV prefix (prefill on a sequence that borrows positions [0, split_row) from another slot): key rows below
  // split_row are read from k2 / v2 (same strides), the rest from k / v. split_row = 0: everything from k / v.
  const bf16 *k2, *v2;
  int split_row;
  // partial mode (shared-prefix attention of a batched decode step; part_o != null): the Tq <= 64 query rows are the
  // rollouts of one figure, blockIdx.x selects a range of part_tiles key tiles, and instead of the normalised output the
  // kernel exports the flash state of that range in the convention of decode_attn_kernel's partials:
  //   part_ml[(row * heads + head) * part_np + part_idx0 + blockIdx.x] = { max score * scale * log2(e), sum exp2 },
  //   part_o[... * head_dim + d] = unnormalised output (head_dim 64 or 128).
  float *part_o, *part_ml;
  int part_np, part_idx0, part_tiles;
};
cudaError_t launch_flash_attn(const AttnArgs& a, cudaStream_t s, uint64_t* counter);

// ---------------------------------------------------------------- ViT attention on wgmma (attn_tc.cu): head_dim 72, non-causal
// qkv bf16 [B*N, 3*heads*72] (q | k | v column blocks); vT: scratch bf16 [B*heads*80, attn_tc_vt_cols(N)]; o bf16 [B*N, heads*72]
bool attn_tc_supported();
int attn_tc_vt_cols(int N);
cudaError_t launch_attn_tc(const bf16* qkv, bf16* vT, bf16* o, int B, int heads, int N, float scale, cudaStream_t s, uint64_t* counter);
// cross-attention of the TikZero adapter on the same wgmma kernel: q bf16 [B*N, heads*72]; kv bf16 [B*Tk, 2*heads*72] (k | v
// column blocks), image b attends to its first klen[b] (1..Tk) caption rows; vT scratch bf16 [B*heads*80, attn_tc_vt_cols(Tk)]
constexpr int XATTN_MAX_B = 64;
cudaError_t launch_xattn_tc(const bf16* q, const bf16* kv, const int* klen_host, int Tk, bf16* vT, bf16* o, int B, int heads,
                            int N, float scale, cudaStream_t s, uint64_t* counter);

// ---------------------------------------------------------------- row-wise / elementwise
// y = LN(x) * w + b  (fp32 stats); x fp32 [M, D]; writes bf16 and/or fp32 outputs
cudaError_t launch_layernorm(const float* x, const bf16* w, const bf16* b, float eps, int M, int D,
                             bf16* out_bf16, float* out_f32, cudaStream_t s, uint64_t* counter);
// y = x * rsqrt(mean(x^2)+eps) * w ; x fp32 [M, D] row stride ldx; out bf16 [M, D]
cudaError_t launch_rmsnorm(const float* x, int64_t ldx, const bf16* w, float eps, int M, int D, bf16* out,
                           cudaStream_t s, uint64_t* counter);
// pixels fp32 [B,3,S,S] -> patches bf16 [B*N, KP] (channel-major (c, py, px) like conv weight; zero pad)
cudaError_t launch_im2col(const float* pixels, int B, int S, int P, int KP, bf16* out, cudaStream_t s,
                          uint64_t* counter);
cudaError_t launch_cast_f32_bf16(const float* in, bf16* out, int64_t n, cudaStream_t s, uint64_t* counter);
// x[t, :] = ids[t] == image_token ? img[(start_pos + t) - img_start, :] : embed[ids[t], :]
cudaError_t launch_embed_splice(const int64_t* ids, int T, int start_pos, const bf16* embed, int H, int vocab,
                                int image_token, const float* img, int img_start, int n_img, float* x,
                                cudaStream_t s, uint64_t* counter);
// decoder RoPE + KV append, head_dim hd in {64, 128}; rope_cs fp32 [max_len, hd/2, 2]; cache rows [kv_head][max_len][hd].
// decode: qkv fp32 [B, qd+2kd] -> roped q fp32 (and optionally bf16) [B, qd]; K/V of row b into slot slots[b] at pos[b]
// unless active[b] == 0 (a retired row of a generation loop, whose slot may already hold another sequence)
cudaError_t launch_rope_kv_decode(const float* qkv, int B, const int* slots, const int* pos, const int* active, int heads, int kv_heads,
                                  const float* rope_cs, float* q_out, bf16* kv_base, int64_t kv_slot_stride,
                                  int64_t kv_v_offset, int max_len, int hd, cudaStream_t s, uint64_t* counter, bf16* q_bf16 = nullptr);
// prefill: qkv fp32 [T, qd+2kd] -> roped q bf16 [T, qd]; K/V bf16 into the cache at positions start_pos+t
cudaError_t launch_rope_kv_prefill(const float* qkv, int T, int start_pos, int heads, int kv_heads,
                                   const float* rope_cs, bf16* q_out, bf16* kcache, bf16* vcache,
                                   int max_len, int hd, cudaStream_t s, uint64_t* counter);
// head_dim 64 prefill without a KV slot (caption encoder): qkv fp32 [T, (heads+2kv_heads)*64] -> roped q bf16 [T, heads*64],
// roped k bf16 [T, kv_heads*64], v bf16 [T, kv_heads*64]; rope_cs fp32 [T, 32, 2]
cudaError_t launch_rope_qkv64(const float* qkv, int T, int heads, int kv_heads, const float* rope_cs, bf16* q, bf16* k, bf16* v,
                              cudaStream_t s, uint64_t* counter);
// per-head LayerNorm (affine over head_dim, fp32 stats): in bf16 [M, heads*hd] row stride ld_in -> out (may alias in), ld_out
cudaError_t launch_head_layernorm(const bf16* in, int64_t ld_in, const bf16* w, const bf16* b, float eps, int M, int heads,
                                  int hd, bf16* out, int64_t ld_out, cudaStream_t s, uint64_t* counter);
cudaError_t launch_cast_bf16_f32(const bf16* in, float* out, int64_t n, cudaStream_t s, uint64_t* counter);

// ---------------------------------------------------------------- decode (batch of single tokens)
enum { GEMV_STORE = 0, GEMV_ADD = 1, GEMV_GLU = 2, GEMV_QKV = 3 };
struct GemvArgs {
  int mode;
  const bf16* W;              // [N, K]
  int N, K;
  const float* x;             // [B, x_stride] fp32
  int64_t x_stride;
  const bf16* norm_w;         // fused RMSNorm on x (null = none)
  float eps;
  float* out;                 // STORE/ADD: [B, out_stride]; GLU: [B, out_stride] (N/2 valid); QKV: q [B, out_stride]
  int64_t out_stride;
  int B;
  // QKV mode
  const int* slots;           // device int[B]
  const int* pos;             // device int[B] : position of the token being processed
  const float* rope_cs;       // fp32 [max_len, head_dim/2, 2] (cos, sin)
  bf16* kv_base;              // cache base of this layer for slot 0: K then V
  int64_t kv_slot_stride;     // elements between slots
  int64_t kv_v_offset;        // elements from K to V of the same layer
  int q_dim, kv_dim, max_len;
  int head_dim;               // 64 or 128
  const int* active;          // device int[B] or null: rows with active[b] == 0 append no K/V
};
cudaError_t launch_gemv(const GemvArgs& a, cudaStream_t s, uint64_t* counter);

// x[b, :] = embed[tok[b], :]  (fp32 out)
cudaError_t launch_embed_tokens(const int* tok32, const int64_t* tok64, int B, const bf16* embed, int H,
                                int vocab, float* x, cudaStream_t s, uint64_t* counter);

struct DecodeAttnArgs {
  const float* q;             // [B, q_dim] fp32 (roped)
  int64_t q_stride;
  const bf16* kv_base;        // layer base for slot 0
  int64_t kv_slot_stride, kv_v_offset;
  const int* slots;           // device int[B]
  const int* pos;             // device int[B]; keys [0, pos] are attended
  const int* share_slot;      // device int[B]: slot that holds positions [0, share_len[b]) of sequence b (shared prefix)
  const int* share_len;       // device int[B]: 0 = nothing shared
  int B, heads, kv_group, max_len, nsplit;
  int head_dim;               // 64 or 128
  float scale;
  float* part_o;              // [B, heads, np, head_dim]
  float* part_ml;             // [B, heads, np, 2]
  unsigned int* counters;     // [B * heads], zero-initialised, self-resetting
  float* out;                 // [B, q_dim] fp32
  int64_t out_stride;
  // shared-prefix ("cascade") mode: keys [0, key_begin) were already reduced by launch_flash_attn in partial mode into the
  // partial slots [nsplit, np); this kernel covers [key_begin, pos] and its merge adds all np partials. 0 / nsplit = off.
  int key_begin, np;
  bf16* out_bf16;             // optional bf16 copy of the output (the o-proj GEMM operand), same layout
  const int* active;          // device int[B] or null: a row with active[b] == 0 reads no keys and gets a zero output
};
cudaError_t launch_decode_attn(const DecodeAttnArgs& a, cudaStream_t s, uint64_t* counter);

struct SampleSeq {
  int suppress;
  uint32_t step;
  uint32_t seq_id;
};
struct SampleArgs {
  const float* logits;        // [B, V]
  int B, V;
  float temperature, top_p;
  float top_p_limit;              // (float)(1.0 - top_p): ascending cumulative mass <= limit is removed
  int top_k, do_sample, bad_token, bs_token;
  uint64_t seed;
  const unsigned long long* seed_dev;   // generation loop: the seed lives in a device word (written by gen_begin) so that a
                                        // captured decode graph does not depend on it; null = use `seed`
  float* scratch;             // [B, V] fp32 work buffer (receives the final probability vector)
  int want_probs;             // greedy only: also write softmax(masked logits) to scratch (sampling always writes it)
  int64_t* out_ids;           // device int64[B] or null
  // generation-loop state (all optional, device): when gen_tok != null the sampler also advances
  // the loop: gen_tok[b] = token, gen_pos[b] += 1, and publishes the token to the pinned host ring.
  int* gen_tok;
  int* gen_pos;
  unsigned long long* gen_step;   // single counter (device); RNG counter + ring row
  unsigned long long* host_ring;  // mapped pinned u64 [ring, B]: ((step + 1) << 32) | token, one store per token
  int ring;
  int max_pos;                    // gen_pos is clamped to this (max_len - 1)
  unsigned int* done_counter;     // device, zero-initialised, self-resetting
  // generation loop with admissions (device [B], all optional): a row with active[b] == 0 draws nothing, publishes the
  // sentinel token -1 with its step stamp and still counts in done_counter (gen_tok, gen_pos and its history stay as they
  // are); with row_step set, row b draws with RNG counter row_step[b] + step on stream row_seq[b] instead of seq[b]
  const int* active;
  const uint32_t* row_step;
  const uint32_t* row_seq;
  SampleSeq seq[64];
};
cudaError_t launch_sample(const SampleArgs& a, cudaStream_t s, uint64_t* counter);
// HF logits processors beyond one bad token and one begin-suppress token (dtk_processors): the tables live in device
// memory, so a captured graph bakes only the pointers. Every CTA builds a ban bitmask and a repetition-penalty bitmask of
// its row in shared memory (2 x 16 KB, so V <= kProcMaxVocab) from the row's token history and the tables.
constexpr int kProcMaxIds = 4096;
constexpr int kProcMaxVocab = 131072;
struct SampleProcTable {
  float penalty;       // repetition penalty (1 = off)
  float min_p;         // 0 = off; applied only when sampling
  int ngram;           // no_repeat_ngram_size (0 = off)
  int eos;             // id banned while a row's history is shorter than eos_until[row] (-1 = none)
  int n_ban, n_begin, n_words, pad;
  int eos_until[64];
  // ban ids [n_ban] | begin-suppress ids [n_begin] | bad-word offsets [n_words + 1] (relative to the word ids) | word ids
  int ids[kProcMaxIds];
};
struct SampleProc {
  const SampleProcTable* tab;   // device
  int* hist;                    // device int32 [B][hist_stride]: each row's prompt + tokens so far
  int* hist_len;                // device int32 [B]; the generation loop appends the drawn token (clamped at hist_stride)
  int hist_stride;
};
cudaError_t launch_sample_proc(const SampleArgs& a, const SampleProc& q, cudaStream_t s, uint64_t* counter);
// admission of a new sequence into row `row` of a running generation loop (one CTA, stream-ordered between two steps): draws
// the row's first token from `logits` with the sampler arguments `a` (the loop's, with a.seq[row] = {suppress 1, step 0,
// seq_id} and no loop state) and, with processors, the row's fresh history (already in q.hist) and eos_min; then writes the
// row's decode state, RNG stream and counter base (1 - current step, so the n-th token after the first draws counter n),
// appends the token to the history, activates the row and publishes (stamp << 32) | token to mailbox[row]
struct SampleAdmit {
  const float* logits;            // [V]
  int row, slot, pos, share_slot, share_len, hist_len, eos_min;
  uint32_t seq_id, stamp;
  int *slots, *posv, *tok, *share_slots, *share_lens, *active;
  uint32_t *row_step, *row_seq;
  const unsigned long long* gen_step;
  SampleProcTable* tab;           // with processors: eos_until[row] = eos_min
  unsigned long long* mailbox;    // mapped pinned [max_batch]
};
cudaError_t launch_sample_admit(const SampleArgs& a, const SampleProc* q, const SampleAdmit& m, cudaStream_t s,
                                uint64_t* counter);
void set_sample_impl(int impl);   // 0 = register-resident kernel when V <= 32768 (default), 1 = generic kernel
int get_sample_impl();

// ---------------------------------------------------------------- persistent decode kernel (B = 1)
// Decode-side weight copy: every matrix is re-tiled once at load into 8 KB tiles of 16 rows x 256 k that a
// single 1-D bulk copy lands in shared memory exactly as ldmatrix.x4 wants them ([kstep 16][matrix 4][row 8][8 bf16]).
// Row groups are permuted so that the two accumulator rows (g, g+8) of one thread are a RoPE pair (i, i+head_dim/2)
// or a SwiGLU pair (gate_i, up_i).
enum { TILE_SEQ = 0, TILE_ROPE = 1, TILE_GLU = 2 };
constexpr int MEGA_TILE_ELEMS = 4096;  // 16 x 256 bf16 = 8 KB
constexpr int MEGA_DBG2_ROWS = 168;     // dev trace: rows 0..159 = local tiles of the traced layer, 160..164 = phase stamps
struct MegaMat {
  const bf16* base;       // tiled copy, layer 0
  int64_t layer_stride;   // elements between layers
  int N, K;               // logical rows / cols of the matrix (GLU: N = 2I interleaved source rows)
  int groups, tpg;        // 16-row groups, 256-column tiles per group
  int per, nact;          // work split over the grid (host-computed: no division in the kernel): per = ceil(groups / grid) groups per participating CTA, nact = ceil(groups / per) participants
  int mode;
};
// FP8 decode tiles (launch_retile_f8): each bf16 row r of a layer matrix is e4m3 code x 2^k_r. A tile holds the codes of
// the same 16 rows x 256 k as the bf16 tile, 4 KB in mma A-fragment order ([kstep pair 8][lane 32][kstep 2][fragment 4]
// [2 codes]: one 16-byte shared load per lane and kstep pair); exps[group][16] holds k_r of the group's tile rows.
constexpr int MEGA_F8_TILE_BYTES = 4096;
struct MegaF8 {
  const uint8_t* tiles;   // layer 0
  const int8_t* exps;     // layer 0
  int64_t layer_stride;   // bytes between layers of tiles
  int64_t exp_stride;     // bytes between layers of exps
};
// Packed decode tiles (launch_pack_scan / launch_pack_tiles): the same bf16 bits in 13 bits per weight, lossless. A tile of
// 16 rows x 256 k is one 6688-byte block:
//   [0, 4096)     sign | mantissa7 of each value, in the FP8 tile's order ([kstep pair 8][lane 32][16 B]);
//   [4096, 6144)  low 4 bits of the exponent codes, [load 4][lane 32][16 B]: load i holds kstep pairs 2i and 2i + 1, 8 B each
//                 (word w of a pair: byte i of words 2w and 2w + 1 of the pair's 16 bytes in its low / high nibble);
//   [6144, 6656)  high bits of the codes, [lane 32][4 words]: word j = kstep pairs 2j, 2j + 1, bit 8 i + 4 (pair & 1) + word;
//   [6656, 6688)  header: the exponent base b_r of each of the 16 tile rows, then the tile's escape entry (int32, -1 if none).
// A value's biased exponent is b_r + code, b_r = max(row max exponent in the tile - 31, 0). A tile in which some value does not
// fit (more than 31 binades below its row's largest value; also a zero or subnormal in a row with b_r > 0) is an ESCAPE tile:
// its codes are zero, b_r = 0, and its full exponent bytes ([kstep pair][lane][16 B], 4096 B) live in a side buffer at entry
// escape * 4096. The K padding of a tile decodes to a finite value that multiplies a zero input.
constexpr int MEGA_PK_TILE_BYTES = 6688;
constexpr int MEGA_PK_NIB = 4096, MEGA_PK_HB = 6144, MEGA_PK_HDR = 6656, MEGA_PK_ESC_BYTES = 4096;
struct MegaPack {
  const uint8_t* tiles;   // layer 0
  int64_t layer_stride;   // bytes between layers
};
struct MegaArgs {
  int H, I, L, heads, kv_heads, V, max_len;
  int hd;                                                     // decoder head_dim, 64 or 128 (mega_configure)
  float eps;
  const bf16 *embed, *final_norm;
  const bf16 *norm1_0, *norm2_0;                               // row-major arena; layer l = ptr + l * norm_stride
  int64_t norm_stride;
  MegaMat mat[5];                                             // qkv, o, gate/up, down (per layer) and lm_head
  const int *tok, *pos, *slots;                               // device state of the sequence being decoded
  const int *share_slot, *share_len;                          // shared KV prefix: positions [0, share_len[0]) live in share_slot[0] (multiple of 16)
  bf16* kv;
  int64_t kv_slot_stride, kv_layer_stride, kv_v_offset;
  const float* rope_cs;
  float* logits;
  // tagged cross-CTA activation words {fp32 value, phase tag} (zero-initialised): xa[tg_H] xb[tg_H] q[heads*hd]
  // knew[kv_heads*hd] vnew[kv_heads*hd] attn[heads*hd] h[tg_I] part[grid][hd+4]
  unsigned long long* tg;
  int tg_H, tg_I;                                             // H and I padded to the 256-column tile (mega_configure)
  unsigned int* head_cnt;                                     // [heads] arrival counters (zero-initialised, self-resetting)
  unsigned long long *bar_count, *bar_base;                   // arrival counter; bar_base[0] = arrivals, [1] = tag epoch of past launches
  int nslots, act_floats;                                     // shared-memory ring geometry (mega_configure)
  // greedy generation loop: argmax of the masked logits in the kernel tail + token publication (replaces the sampler launch)
  int fuse_greedy, bad_token, ring, max_pos;
  unsigned long long* amax;                                   // [0] packed (ordered logit, ~index) max cell, [1] arrival counter; zero-initialised, self-resetting
  int *gen_tok, *gen_pos;
  unsigned long long *gen_step, *host_ring;
  int variant;                                                // dev A/B switches (option "mega_variant"; results identical): bit 0 = weight copies without the evict_first L2 policy, bit 1 = consumers stage a weight tile's input slice before reading the tile (earlier builds' order)
  int dbg_flags;                                              // dev only: 1 = skip tile math, 2 = skip grid barriers, 4/8 = relaxed arrive/poll
  long long* dbg;                                             // optional: [grid][5L+1][4] globaltimer stamps (null = off)
  long long* dbg2;                                            // optional: [grid][MEGA_DBG2_ROWS][4] clock64 per-tile trace of layer dbg_layer
  int dbg_layer;
  // FP8 decoder weights (option "decode_fp8"; null tiles = bf16): e4m3 tiles of the four layer matrices, same order as mat[0..3]
  MegaF8 f8[4];
  // packed decoder weights (option "decode_pack"; null tiles = off): tiles of the four layer matrices and the lm_head, same order
  // as mat[0..4], and the escape tiles' exponent planes
  MegaPack pk[5];
  const uint8_t* pk_esc;
};
int mega_smem_bytes(const MegaArgs& a);
cudaError_t mega_configure(MegaArgs& a, int H, int I, int heads, int hd, int max_smem_optin, int num_sms, int* grid_out);
cudaError_t launch_decode_mega(const MegaArgs& a, int grid, cudaStream_t s, uint64_t* counter);
// one-time re-tiling of a row-major [N, K] (ld = K) matrix into the decode layout (hd: head_dim of TILE_ROPE)
int64_t mega_tiled_elems(int N, int K, int mode, int* groups, int* tpg);
cudaError_t launch_retile(const bf16* src, int N, int K, int mode, int hd, bf16* dst, cudaStream_t s);
// the same matrix into FP8 tiles: derives each row's k_r (the smallest k with max |w| <= 448 * 2^k, at least -117; 0 for a
// row of zeros) into exps and adds to *bad the number of values that are not an e4m3 value times 2^k_r (those tiles are junk)
cudaError_t launch_retile_f8(const bf16* src, int N, int K, int mode, int hd, uint8_t* dst, int8_t* exps, unsigned int* bad,
                             cudaStream_t s);
// the same matrix into packed tiles, in two passes. Scan: writes each tile's row bases into its header and escape[tile] = 1 for
// an escape tile (0 otherwise). Tiles: with esc_idx[tile] = the tile's escape entry or -1, writes the planes, the rest of the
// header and the escape tiles' exponent planes into esc.
cudaError_t launch_pack_scan(const bf16* src, int N, int K, int mode, int hd, uint8_t* dst, uint8_t* escape, cudaStream_t s);
cudaError_t launch_pack_tiles(const bf16* src, int N, int K, int mode, int hd, const int* esc_idx, uint8_t* dst, uint8_t* esc,
                              cudaStream_t s);

// device image preprocessing (Pillow-exact 8-bit bicubic resize + rescale + normalise): rgb uint8 [h, w, 3] -> fp32 [3, S, S]
cudaError_t launch_image_preprocess(const uint8_t* rgb, int h, int w, int S, const int* bounds_h, const int* coef_h, int ksize_h,
                                    const int* bounds_v, const int* coef_v, int ksize_v, float rescale, const float* mean,
                                    const float* std, uint8_t* tmp, float* out, uint8_t* out_u8, cudaStream_t s, uint64_t* counter);

// single-query attention of the SigLIP attention-pool head: q fp32 [heads*72] (shared by all images),
// kv bf16 [B*N, 2*D] -> out bf16 [B, D]
cudaError_t launch_pool_attn(const float* q, const bf16* kv, int B, int N, int D, int heads, float scale,
                             bf16* out, cudaStream_t s, uint64_t* counter);

}  // namespace dtk
