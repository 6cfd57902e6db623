/*
 * detikzify_b200 — C ABI of the H100-native (sm_90a) engine for DeTikZify's image-conditioned
 * autoregressive hot path (SigLIP ViT encode -> concat-3 projector -> LLaMA prefill +
 * KV-cached decode + sampler).
 *
 * The reference (potamides/DeTikZify) is pure Python and has no FFI layer; the seam is the
 * duck-typed HF model object returned by detikzify.model.load() (detikzify/model/__init__.py:28).
 * This header is the boundary inserted *below* that seam (SURVEY.md §8b): every entry point
 * names the reference code it replaces. Conventions:
 *   - every call returns int: 0 = ok, <0 = dtk_status error; no exceptions / abort() cross
 *     the boundary; dtk_last_error() gives the message of the last failing call on that engine;
 *   - all tensor pointers are BORROWED device pointers (row-major, dense) that the caller keeps
 *     alive until the stream has consumed them; the engine owns only KV slots + workspace;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - no global state; one engine per device; calls on one engine must be serialised by the
 *     caller, distinct engines are independent (the 8-GPU figure-sharded case).
 */
#ifndef DETIKZIFY_B200_H
#define DETIKZIFY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DTK_ABI_VERSION 2

#if defined(__GNUC__)
#define DTK_API __attribute__((visibility("default")))
#else
#define DTK_API
#endif

typedef enum dtk_status {
  DTK_OK = 0,
  DTK_ERR_INVALID = -1,   /* bad argument / shape / state */
  DTK_ERR_CUDA = -2,      /* CUDA runtime error (message in dtk_last_error) */
  DTK_ERR_OOM = -3,       /* device allocation failed */
  DTK_ERR_NOSLOT = -4,    /* no free KV sequence slot */
  DTK_ERR_UNSUPPORTED = -5
} dtk_status;

/* Model shape. Mirrors LlamaConfig / timm-SigLIP dims the reference loads
 * (detikzify/model/v1/configuration_detikzify.py:3-13, SURVEY.md Appendix A). */
typedef struct dtk_config {
  /* decoder; head_dim 64 or 128 with heads * head_dim == hidden */
  int32_t hidden, inter, layers, heads, kv_heads, head_dim, vocab, max_len;
  float rms_eps, rope_theta, rope_factor;
  /* RoPE frequency scaling: 0 = linear (inv_freq / rope_factor; DeepSeek-Coder decoders of the v1 checkpoints),
   * 1 = "llama3" (HF modeling_rope_utils._compute_llama3_parameters; LLaMA-3.x decoders of the v2 checkpoints,
   * detikzify/model/configuration_detikzify.py:83-120): wavelengths above rope_orig_max_pos / rope_low_freq are divided by
   * rope_factor, those below rope_orig_max_pos / rope_high_freq are kept, the band in between is interpolated */
  int32_t rope_type;
  float rope_low_freq, rope_high_freq;
  int32_t rope_orig_max_pos;
  /* vision tower */
  int32_t v_hidden, v_inter, v_layers, v_heads, v_image, v_patch;
  int32_t v_act;              /* 0 = gelu_pytorch_tanh, 1 = exact (erf) gelu */
  float v_eps;
  /* glue */
  int32_t concat;             /* patches concatenated per image token (3) */
  int32_t image_token_id, eos_token_id;
  /* engine sizing */
  int32_t max_seqs;           /* KV sequence slots (each max_len positions) */
  int32_t max_batch;          /* max concurrently decoded sequences */
} dtk_config;

typedef struct dtk_weight_info {
  char name[64];
  uint64_t offset;            /* byte offset in the arena (256-B aligned) */
  uint64_t nbytes;
  int32_t rows, cols;         /* bf16 [rows, cols] row-major (cols = 1-D length if rows==1) */
} dtk_weight_info;

/* Sampling controls == the kwargs detikzify/infer/generate.py:218-227,379-387 passes to HF
 * generate (temperature/top_p/top_k/do_sample + bad_words_ids=[[image_token]] +
 * begin_suppress_tokens=[eos]). */
typedef struct dtk_sampling {
  double temperature;         /* < 1e-5 or do_sample==0 -> greedy argmax */
  double top_p;               /* >= 1 -> off (double: HF compares against python 1 - top_p) */
  int32_t top_k;              /* 0 -> off */
  int32_t do_sample;
  int32_t bad_token;          /* always masked (-1 = none) */
  int32_t begin_suppress_token; /* masked when suppress flag set (-1 = none) */
  uint64_t seed;
} dtk_sampling;

/* HF logits processors beyond one bad token and one begin-suppress token (HF generation/utils.py::_get_logits_processor,
 * generation/logits_process.py), applied in HF's order before the temperature: repetition penalty
 * (RepetitionPenaltyLogitsProcessor: x < 0 ? x * p : x / p in fp32 on every distinct id of the row's history), no-repeat
 * n-gram (NoRepeatNGramLogitsProcessor), bad words (NoBadWordsLogitsProcessor: single ids always, a longer sequence bans
 * its last id when the history ends with its other ids and is skipped when it is longer than the history), minimum length
 * (MinLength / MinNewTokensLength: EOS banned while the history is shorter than the row's eos_min_len), suppress tokens
 * (SuppressTokensLogitsProcessor) and begin-suppress tokens (SuppressTokensAtBeginLogitsProcessor: rows whose suppress
 * flag is set); min-p (MinPLogitsWarper) after top-p when sampling. "Banned" = -inf, like dtk_sampling.bad_token.
 * Limits: vocab <= 131072; n_ban + n_begin + n_words + 1 + (ids in word_ids) <= 4096. */
typedef struct dtk_processors {
  double repetition_penalty;  /* 1 -> off; > 0 */
  double min_p;               /* 0 -> off; in [0, 1]; sampling only */
  int32_t no_repeat_ngram_size; /* 0 -> off */
  int32_t eos_token_id;       /* the id eos_min_len bans (-1 = none) */
  const int32_t* ban_ids;     /* [n_ban] host: always banned (bad words of length 1, suppress_tokens) */
  int32_t n_ban;
  const int32_t* begin_ids;   /* [n_begin] host: banned on rows whose suppress flag is set */
  int32_t n_begin;
  const int32_t* word_ids;    /* host: bad-word sequences of length >= 2, concatenated */
  const int32_t* word_lens;   /* [n_words] host: their lengths */
  int32_t n_words;
} dtk_processors;

typedef struct dtk_engine dtk_engine;

DTK_API int dtk_abi_version(void);

/* ---- weights: one contiguous bf16 arena (single ncclBroadcast at load, SURVEY.md §8e) ---- */
DTK_API int dtk_weight_count(const dtk_config* cfg);
DTK_API int dtk_weight_get(const dtk_config* cfg, int index, dtk_weight_info* out);
DTK_API uint64_t dtk_arena_bytes(const dtk_config* cfg);

/* ---- lifecycle. Replaces DetikzifyForCausalLM.from_pretrained + initialize_vision_modules
 *      (detikzify/model/v1/__init__.py:24-56, v1/modeling_detikzify.py:84-117). ------------ */
DTK_API int dtk_create(const dtk_config* cfg, const void* weight_arena, uint64_t arena_bytes,
               int device, dtk_engine** out);
DTK_API int dtk_destroy(dtk_engine* eng);
DTK_API const char* dtk_last_error(const dtk_engine* eng);

/* ---- ViT. Replaces DetikzifyVisionModel.forward / get_intermediate_layers
 *      (v1/modeling_detikzify.py:63-72) == timm forward_features (+ forward_head).
 *      pixels fp32 [B,3,S,S]; tokens_out fp32 [B,N,D] (may be NULL); pooled_out fp32 [B,D]
 *      (may be NULL; attention-pool head, used by SelfSim evaluate/imagesim.py:101-103). ---- */
DTK_API int dtk_vit_encode(dtk_engine* eng, const float* pixels, int B, float* tokens_out,
                   float* pooled_out, void* stream);

/* ---- TikZero text conditioning (reference detikzify/model/adapter: a Llama-3.2-1B caption embedder, a connector E -> D and
 *      one gated cross-attention layer before every cross_every_n-th ViT layer). The adapter weights live in a SECOND
 *      contiguous bf16 arena whose layout the library defines (dtk_adapter_weight_*), attached to an existing engine. ---- */
typedef struct dtk_adapter_config {
  /* caption embedder (LlamaModel; head_dim must be 64) */
  int32_t hidden, inter, layers, heads, kv_heads, head_dim, vocab;
  float rms_eps, rope_theta, rope_factor;
  int32_t rope_type;          /* as dtk_config.rope_type */
  float rope_low_freq, rope_high_freq;
  int32_t rope_orig_max_pos;
  int32_t max_text;           /* longest caption (tokenizer model_max_length, 512) */
  int32_t cross_every_n;      /* cross layer before vision layer l iff (l + 1) % cross_every_n == 0 */
} dtk_adapter_config;

/* weight table of the adapter arena; the vision dims (cross-layer widths, dummy image size) are the engine config's */
DTK_API int dtk_adapter_weight_count(const dtk_config* cfg, const dtk_adapter_config* acfg);
DTK_API int dtk_adapter_weight_get(const dtk_config* cfg, const dtk_adapter_config* acfg, int index, dtk_weight_info* out);
DTK_API uint64_t dtk_adapter_arena_bytes(const dtk_config* cfg, const dtk_adapter_config* acfg);
/* borrow `arena` (device) until dtk_adapter_detach / dtk_destroy; allocates the caption encoder's workspace */
DTK_API int dtk_adapter_attach(dtk_engine* eng, const dtk_adapter_config* acfg, const void* arena, uint64_t arena_bytes);
DTK_API int dtk_adapter_detach(dtk_engine* eng);
/* caption encoder (reference adapter hook: embedding_model(...).last_hidden_state, then adapter.connect): ids device int64
 * [T], 1 <= T <= max_text, one unpadded caption (with right padding and causal attention the valid rows of a padded batch
 * are exactly this). hidden_out (may be NULL): fp32 [T, E] final-RMSNorm states (bf16-rounded, the connector's operand);
 * cond_out: fp32 [T, D] connector output. */
DTK_API int dtk_text_encode(dtk_engine* eng, const int64_t* ids, int T, float* hidden_out, float* cond_out, void* stream);
/* ViT with the cross layers inserted: as dtk_vit_encode, conditioned on cond fp32 [B, Tmax, D] (dtk_text_encode output,
 * caption b valid in rows [0, cond_len[b])); cond_len host int[B], 1 <= cond_len[b] <= Tmax <= max_text. */
DTK_API int dtk_vit_encode_cond(dtk_engine* eng, const float* pixels, int B, const float* cond, const int* cond_len,
                                int Tmax, float* tokens_out, float* pooled_out, void* stream);

/* ---- image preprocessing on the device. Replaces DetikzifyImageProcessor.preprocess for images already uploaded as
 *      uint8 (detikzify/model/v1/processing_detikzify.py:242-251: bicubic resize to SxS, x 1/255, (x - mean) / std, CHW).
 *      rgb: device uint8 [h, w, 3]; the resize is Pillow's 8-bit resampler bit for bit: bounds_* int32 [S][2] = {first
 *      input index, tap count}, coef_* int32 [S][ksize_*] = 22-bit fixed-point taps for the horizontal / vertical pass
 *      (host-computed from (w -> S) and (h -> S), see model/processing.py::pil_resample_coeffs); tmp: device uint8
 *      [h, S, 3] scratch; out: device fp32 [3, S, S]; out_u8 (may be NULL): the resized uint8 image [S, S, 3] (tests). ---- */
DTK_API int dtk_image_preprocess(dtk_engine* eng, const uint8_t* rgb, int h, int w, int S,
                                 const int32_t* bounds_h, const int32_t* coef_h, int ksize_h,
                                 const int32_t* bounds_v, const int32_t* coef_v, int ksize_v,
                                 float rescale, const float* mean3_host, const float* std3_host,
                                 uint8_t* tmp, float* out, uint8_t* out_u8, void* stream);

/* ---- concat-3 + mm_projector (v1/modeling_detikzify.py:132-137,163).
 *      tokens fp32 [B,N,D] -> out fp32 [B,P,H]; the reshape is folded into addressing. ------ */
DTK_API int dtk_project(dtk_engine* eng, const float* tokens, int B, float* out, void* stream);

/* ---- KV sequence slots (replaces DynamicCache, HF cache_utils; SURVEY.md §8f.1). ---------- */
DTK_API int dtk_seq_alloc(dtk_engine* eng, int* slot);
DTK_API int dtk_seq_free(dtk_engine* eng, int slot);
/* copy the first `len` cached positions of src into dst (dst becomes self-contained) */
DTK_API int dtk_seq_fork(dtk_engine* eng, int src_slot, int dst_slot, int len, void* stream);
/* make dst READ the first `len` cached positions from base instead of holding a copy (MCTS rollouts of one figure share the
 * image prefix and the tree path: detikzify/infer/generate.py:246-257,305-313 re-prefills them per rollout). The shared
 * part is reference counted: base cannot be freed, nor rewritten below the shared length, while a borrower exists; dst
 * writes only positions >= len. Whole 16-position blocks are shared, the remainder (< 16 positions) is copied into dst.
 * One level: sharing from a slot that itself borrows resolves to the root slot. */
DTK_API int dtk_seq_share(dtk_engine* eng, int base_slot, int dst_slot, int len, void* stream);

/* ---- prefill. Replaces DetikzifyModel.forward splice + LlamaModel.forward + lm_head for a
 *      prompt (v1/modeling_detikzify.py:144-200,218-257). Processes ids[0..T) as positions
 *      [start_pos, start_pos+T) of `slot` (positions < start_pos must already be cached).
 *      Rows whose id == image_token_id take their embedding from img_embeds (fp32 [P,H],
 *      row = position - img_start) — the count/contiguity validation is the caller's
 *      (Python shim) job. Writes fp32 logits of the LAST position to last_logits [V]
 *      (may be NULL). all_logits (may be NULL): fp32 [T,V] for parity tests. --------------- */
DTK_API int dtk_prefill(dtk_engine* eng, int slot, const int64_t* ids, int T, int start_pos,
                const float* img_embeds, int img_start, int n_img,
                float* last_logits, float* all_logits, void* stream);

/* ---- sequence scoring. Replaces the logits + CrossEntropyLoss tail of DetikzifyForCausalLM.forward(labels=...)
 *      (v1/modeling_detikzify.py:218-270, modeling_detikzify.py:320-376) without materialising [T,V] logits. Prefills
 *      exactly as dtk_prefill (same preconditions, KV writes and shared-prefix rules), then applies the final RMSNorm to
 *      all T rows and runs the lm_head GEMM with a fused log-softmax. targets: device int64 [T], a negative (or >= V)
 *      value means "no target"; logprob: device fp32 [T] = log softmax(logits[t])[targets[t]] (0 without a target);
 *      lse (may be NULL): device fp32 [T] = log sum exp logits[t]; all_logits (may be NULL): fp32 [T,V], the same values
 *      the log-softmax was taken from. Deterministic. The first call allocates max_len * ceil(V/256) * 8 bytes of
 *      workspace. ------------------------------------------------------------------------------------------------- */
DTK_API int dtk_score(dtk_engine* eng, int slot, const int64_t* ids, int T, int start_pos,
                      const float* img_embeds, int img_start, int n_img, const int64_t* targets,
                      float* logprob, float* lse, float* all_logits, void* stream);

/* ---- single-token decode for B sequences (LlamaModel.forward with cache, q_len == 1;
 *      v1/modeling_detikzify.py:285-305). slots: host int[B]; positions host int[B] (the
 *      position the token occupies); ids: device int64[B]; logits: device fp32 [B,V]. ------ */
DTK_API int dtk_decode(dtk_engine* eng, const int* slots, const int* positions, const int64_t* ids,
               int B, float* logits, void* stream);

/* ---- sampler. Replaces HF LogitsProcessorList + softmax + multinomial / argmax
 *      (HF generation/utils.py:2762-2793). logits fp32 [B,V]; suppress: host int[B]
 *      (1 = apply begin_suppress_token, i.e. first new token); steps: host uint32[B] RNG
 *      counters; out_ids device int64[B]; probs_out (may be NULL) fp32 [B,V] receives the
 *      post-processor probability vector (parity tests). ----------------------------------- */
DTK_API int dtk_sample(dtk_engine* eng, const float* logits, int B, const dtk_sampling* params,
               const int* suppress, const uint32_t* steps, const uint32_t* seq_ids,
               int64_t* out_ids, float* probs_out, void* stream);

/* ---- logits processors (dtk_processors) for the following dtk_sample and dtk_gen_begin calls, until a call with
 *      proc == NULL turns them off. Replaces the HF processors listed at dtk_processors for B rows: row b's history is
 *      hist_len[b] ids (prompt + tokens so far, HF's input_ids) taken in order from the concatenated host array hist_ids,
 *      at most max_len each; eos_min_len host int[B] (may be NULL = 0): EOS is banned while the row's history is shorter.
 *      The histories live in the engine; the generation loop appends every token it draws (clamped at max_len), so
 *      before dtk_gen_begin they must end with first_ids. dtk_sample and dtk_gen_begin then take B <= the rows given
 *      here, and greedy batch-1 generation takes its token from the sampler instead of the persistent kernel's fused
 *      argmax. Not allowed inside a generation loop. Synchronises `stream`. ----------------------------------------- */
DTK_API int dtk_set_processors(dtk_engine* eng, const dtk_processors* proc, int B, const int32_t* hist_ids,
                               const int32_t* hist_len, const int32_t* eos_min_len, void* stream);

/* ---- fused generation loop state (device-resident; one graph launch per token).
 *      dtk_gen_begin: bind B slots whose prompts are prefilled to `positions[b]` tokens and
 *      whose first pending token is first_ids[b] (already sampled from the prefill logits).
 *      dtk_gen_step: decode + sample one token for every bound sequence; token b of step s is
 *      written to host_ring (pinned, int32 [ring][B]) at row s % ring. Returns immediately
 *      (asynchronous on `stream`). dtk_gen_wait blocks until step s has landed. ------------- */
DTK_API int dtk_gen_begin(dtk_engine* eng, const int* slots, const int* positions,
                  const int64_t* first_ids_host, int B, const dtk_sampling* params,
                  const uint32_t* seq_ids, void* stream);
DTK_API int dtk_gen_step(dtk_engine* eng, void* stream);
DTK_API int dtk_gen_wait(dtk_engine* eng, int64_t step, int32_t* tokens_out_host /* [B] */);
DTK_API int dtk_gen_end(dtk_engine* eng);

/* ---- continuous batching: change a row's occupant while the loop runs (batched loops, B >= 2 or the per-op B = 1 loop).
 *      dtk_gen_retire: row `row` stops; every step launched after the call leaves its slot untouched (no KV write, no key
 *      read) and publishes the sentinel token -1 for it (dtk_gen_wait still returns every row of every step).
 *      dtk_gen_admit: row `row` (inactive) takes a new sequence whose prompt is prefilled into `slot` up to `position`
 *      (shared-prefix state as the slot has it); `logits` device fp32 [V] are the prompt's last-position logits. The call
 *      enqueues one kernel that draws the first token with the loop's sampling parameters (begin-suppress on, RNG counter 0
 *      on stream seq_id), writes the row's state and activates it; the n-th token after the first draws counter n, so the
 *      sequence draws exactly what a loop of its own would. With processors set the row's history becomes hist_ids[0,
 *      hist_len) (host; it must end with the prompt) plus the first token, and EOS is banned while it is shorter than
 *      eos_min_len; without them both are ignored. DTK_ERR_UNSUPPORTED on the batch-1 persistent loop; DTK_ERR_INVALID for
 *      an active row, an unallocated slot, a position inside a shared prefix, another stream than the loop's, and on a
 *      loop begun with shared-prefix (cascade) attention a slot that does not borrow exactly that loop's prefix.
 *      dtk_gen_first: waits for the admitted row's first token (as dtk_gen_wait waits for a step).
 *      Ordering: every device effect is ordered on the loop's stream behind the steps already launched, so the host may
 *      dtk_seq_free a retired row's slot at once and reuse it (a prefill into it runs after those steps). A step launched
 *      before the retirement decodes the row once more, at positions beyond the end of its sequence. A sequence admitted
 *      when s steps have been launched appears in the ring from step s on. -------------------------------------------- */
DTK_API int dtk_gen_admit(dtk_engine* eng, int row, int slot, int position, const float* logits, uint32_t seq_id,
                          const int32_t* hist_ids, int hist_len, int eos_min_len, void* stream);
DTK_API int dtk_gen_retire(dtk_engine* eng, int row, void* stream);
DTK_API int dtk_gen_first(dtk_engine* eng, int row, int32_t* token_out_host);

/* ---- engine options. "decode_impl": 1 = persistent weight-streaming decode kernel (default for
 *      B = 1), 0 = per-op kernels replayed from a CUDA graph (always used for B > 1). Others (all with
 *      working defaults): "gemm_impl" (see dtk_dbg_gemm_impl), "attn_impl" (ViT attention: 1 = wgmma, 0 =
 *      mma.sync), "cascade_attn" (shared-prefix attention of batched decode), "decode_gemm_min_batch",
 *      "fuse_greedy", "vit_graph", and dev switches "mega_debug", "mega_flags", "mega_trace_layer",
 *      "mega_nslots", "mega_variant". Unknown keys return DTK_ERR_INVALID.
 *      "prefill_layers" (dev switch for layer-by-layer tests): n in 0..layers makes dtk_prefill / dtk_score run only
 *      the first n decoder layers; layers >= n write no KV rows and the logits come from the partial residual stream
 *      (see dtk_dbg_residual_read). -1 (default) = every layer; other values return DTK_ERR_INVALID.
 *      "decode_fp8": 1 = the persistent kernel (B = 1) and the four layer GEMMs of batched steps with
 *      4 <= B < 64 stream the four decoder-layer matrices as e4m3 codes plus one power-of-two exponent per row
 *      (rebuilt from the arena, whose every row must be e4m3 x 2^k; otherwise DTK_ERR_INVALID names the layer
 *      and matrix and nothing changes), 0 (default) = bf16. The logits equal the bf16 kernels' on the same
 *      arena; B = 2, 3, B >= 64 and the lm_head always run bf16.
 *      "decode_pack": 1 = the persistent kernel (B = 1) streams every matrix, lm_head included, as lossless 13-bit
 *      packed tiles (any bf16 weights; the logits equal the bf16 tiles'), 0 (default of dtk_create) = bf16 tiles.
 *      bf16, e4m3 and packed tiles are exclusive: setting one of decode_fp8 / decode_pack to 1 clears the other. */
DTK_API int dtk_set_option(dtk_engine* eng, const char* key, int64_t value);
/*      Read back an option; the extra key "decode_persistent" reports whether B = 1 decode steps
 *      actually run on the persistent kernel (option set AND the device can co-schedule its grid), and
 *      "decode_weight_bytes" the weight bytes one such step streams in the current mode (packed: tiles and escape
 *      planes; otherwise the lm_head in bf16), "decode_pack_escapes" the packed weights' escape tiles. */
DTK_API int dtk_get_option(dtk_engine* eng, const char* key, int64_t* value);

/* ---- introspection for benches: algorithmic HBM bytes of one decode step at context T ----- */
DTK_API uint64_t dtk_decode_bytes(const dtk_config* cfg, int context_len);
/* kernels launched by this engine since creation (bench.py's gpu_launches) */
DTK_API uint64_t dtk_launch_count(const dtk_engine* eng);

/* ---- kernel-level test hooks (used only by tests/: shape sweeps at the real model sizes
 *      without instantiating a model). All pointers are device pointers. --------------------- */
/* phase timestamps of the last persistent-kernel launch (option "mega_debug" = 1):
 * [grid CTAs][5*layers+1 phases][4] globaltimer (ns) stamps; returns the value count */
DTK_API int dtk_dbg_mega_times(dtk_engine* eng, long long* out_host, int max_values);
/* per-tile SM-clock trace of one layer (options "mega_debug" = 1, "mega_trace_layer" = l): [grid CTAs][168 rows][4];
 * rows 0..159 = the CTA's local tiles of that layer {producer issue, bytes landed, tile done, consumer asked},
 * rows 160..164 = the layer's five phases {start, staged, items done, barrier done}; returns the value count */
DTK_API int dtk_dbg_mega_trace(dtk_engine* eng, long long* out_host, int max_values);
/* bytes [offset, offset + nbytes) of the packed decode tiles (option "decode_pack" = 1): [layer][wqkv | wo | wgu | wd tiles],
 * then the lm_head tiles, 6688 bytes per tile (launch.h, MegaPack) */
DTK_API int dtk_dbg_pack_bytes(dtk_engine* eng, int64_t offset, int64_t nbytes, void* out_host);
/* copy (stream-ordered, no engine state changes) the cached bf16 keys and values of positions [pos0, pos0 + n) of one layer
 * of an allocated slot into k_out / v_out, each [kv_heads][n][head_dim]. Positions below the slot's shared length come from
 * the slot that lends them, as decode reads them. DTK_ERR_INVALID: slot not allocated, layer or range outside the cache. */
DTK_API int dtk_dbg_kv_read(dtk_engine* eng, int slot, int layer, int pos0, int n, void* k_out, void* v_out, void* stream);
/* copy (stream-ordered, no engine state changes) rows [row0, row0 + n) of the fp32 residual stream as the last dtk_prefill /
 * dtk_score left it (row t = the t-th prompt position of that call) into out [n][hidden]. The contents are valid only until
 * the next engine call. DTK_ERR_INVALID: null out, rows outside [0, max_len). */
DTK_API int dtk_dbg_residual_read(dtk_engine* eng, int row0, int n, float* out, void* stream);
/* select the dense GEMM implementation used by dtk_dbg_gemm and the engines of this process:
 * 0 = mma.sync, 1 = wgmma one 128 x 128 tile per CTA, 2 (default) = persistent 128 x 256 wgmma kernel,
 * -1 = query only; returns the current setting. Bits 8..11 of a
 * non-negative value force the split-K factor (cluster size 1..8) of the batched-decode tile; 0 = heuristic. */
DTK_API int dtk_dbg_gemm_impl(int impl);
/* C = act(A[M,K] * W[N,K]^T + bias) (+resid); glu: out[m, n/2] = silu(c[m,n]) * c[m,n+1] */
DTK_API int dtk_dbg_gemm(const void* A_bf16, const void* W_bf16, const void* bias_bf16,
                         const float* resid, int M, int N, int K, int act, int glu,
                         float* out_f32, void* out_bf16, void* stream);
/* lm_head log-softmax of dtk_score on its own: logprob[m] = log softmax(A W^T)[m, targets[m]] (0 when the target is outside
 * [0, N)), lse (may be NULL) [M]; A bf16 [M,K], W bf16 [N,K], targets int64 [M]. Keeps a grow-only workspace per device:
 * calls must not overlap. */
DTK_API int dtk_dbg_lm_logprob(const void* A_bf16, const void* W_bf16, int M, int N, int K, const int64_t* targets,
                               float* logprob, float* lse, void* stream);
/* the sampler of dtk_sample without an engine, at any vocabulary size: logits fp32 [B,V], 1 <= B <= 64, V >= 1; suppress,
 * steps, seq_ids host arrays [B] as in dtk_sample (NULL = 0, 0, b); impl 0 = dtk_sample's dispatch (register-resident kernel
 * while V <= 32768), 1 = the generic kernel (the process-wide "sample_impl" setting is restored afterwards); out_ids int64 [B];
 * probs fp32 [B,V] (required) receives the probability vector the token was drawn from (softmax of the masked logits when
 * greedy) */
DTK_API int dtk_dbg_sample(const float* logits, int B, int V, const dtk_sampling* params, const int* suppress,
                           const uint32_t* steps, const uint32_t* seq_ids, int impl, int64_t* out_ids, float* probs,
                           void* stream);
/* dtk_dbg_sample with logits processors (dtk_set_processors' arguments for B rows of at most max_len ids); the engine's
 * processor sampler without an engine; synchronises `stream` */
DTK_API int dtk_dbg_sample_proc(const float* logits, int B, int V, const dtk_sampling* params, const int* suppress,
                                const uint32_t* steps, const uint32_t* seq_ids, int impl, const dtk_processors* proc,
                                const int32_t* hist_ids, const int32_t* hist_len, const int32_t* eos_min_len, int max_len,
                                int64_t* out_ids, float* probs, void* stream);
/* q,k,v,o bf16 [B, T, heads, head_dim]; head_dim in {72,128} */
DTK_API int dtk_dbg_flash_attn(const void* q, const void* k, const void* v, void* o, int B,
                               int heads, int Tq, int Tk, int head_dim, int causal, int q_pos0,
                               float scale, void* stream);
/* ViT attention on wgmma: qkv bf16 [B*N, 3*heads*72] (q | k | v column blocks), vt_scratch bf16 [B*heads*80, ceil(N/128)*128],
 * o bf16 [B*N, heads*72]; non-causal, head_dim 72 */
DTK_API int dtk_dbg_attn_tc(const void* qkv, void* vt_scratch, void* o, int B, int heads, int N, float scale, void* stream);
/* TikZero cross-attention on wgmma: q bf16 [B*N, heads*72], kv bf16 [B*Tk, 2*heads*72] (k | v), image b attends to its
 * first klen_host[b] keys (1..Tk, B <= 64); vt_scratch bf16 [B*heads*80, ceil(Tk/128)*128]; o bf16 [B*N, heads*72] */
DTK_API int dtk_dbg_xattn_tc(const void* q, const void* kv, const int* klen_host, int Tk, void* vt_scratch, void* o, int B,
                             int heads, int N, float scale, void* stream);
/* per-head LayerNorm: x bf16 [M, heads*hd] -> out bf16 (same layout), affine w/b bf16 [hd] */
DTK_API int dtk_dbg_head_layernorm(const void* x, const void* w, const void* b, float eps, int M, int heads, int hd, void* out,
                                   void* stream);
/* gated residual GEMM: out_f32 = resid + sigmoid(gate) * act(A W^T + bias); gate bf16 [1] device */
DTK_API int dtk_dbg_gemm_gated(const void* A_bf16, const void* W_bf16, const void* bias_bf16, const void* gate_bf16,
                               const float* resid, int M, int N, int K, int act, float* out_f32, void* stream);
/* y = W[N,K] * rmsnorm?(x[K]) ; mode 0 store / 1 add / 2 glu (out[N/2]) */
DTK_API int dtk_dbg_gemv(const void* W_bf16, const float* x, const void* norm_w_bf16, float eps,
                         int N, int K, int mode, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DETIKZIFY_B200_H */
