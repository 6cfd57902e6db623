"""
Thin Python wrapper over the C ABI: owns the weight arena tensor and hands raw device pointers of
torch tensors (the only container) to ``libdtk_b200.so``. ctypes releases the GIL for the duration
of every call, so the streamer/consumer thread of the reference's MCTS driver keeps running.
"""
from __future__ import annotations

import ctypes as C
from typing import TYPE_CHECKING, Dict, List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import DtkConfig, DtkProcessors, DtkSampling, DtkWeightInfo
if TYPE_CHECKING:  # avoid a package-level import cycle (model/ imports this module)
    from .model.configuration import DetikzifyConfig

V = "model.vision_model.vision_model."


class EngineError(RuntimeError):
    pass


def to_c_config(cfg: "DetikzifyConfig", max_seqs: int = 4, max_batch: int = 1, max_len: Optional[int] = None) -> DtkConfig:
    vc = cfg.vision_config
    act = {"gelu_pytorch_tanh": 0, "gelu_tanh": 0, "gelu": 1, "gelu_erf": 1}[vc.hidden_act]
    return DtkConfig(
        hidden=cfg.hidden_size, inter=cfg.intermediate_size, layers=cfg.num_hidden_layers,
        heads=cfg.num_attention_heads, kv_heads=cfg.num_key_value_heads, head_dim=cfg.head_dim,
        vocab=cfg.vocab_size, max_len=max_len or cfg.model_max_length,
        rms_eps=cfg.rms_norm_eps, rope_theta=cfg.rope_theta, rope_factor=cfg.rope_factor,
        rope_type={"linear": 0, "llama3": 1}[cfg.rope_type], rope_low_freq=cfg.rope_low_freq_factor,
        rope_high_freq=cfg.rope_high_freq_factor, rope_orig_max_pos=cfg.rope_original_max_position,
        v_hidden=vc.hidden_size, v_inter=vc.intermediate_size, v_layers=vc.num_hidden_layers,
        v_heads=vc.num_attention_heads, v_image=vc.image_size, v_patch=vc.patch_size, v_act=act,
        v_eps=vc.layer_norm_eps, concat=cfg.concat_patches, image_token_id=cfg.image_token_id,
        eos_token_id=cfg.eos_token_id, max_seqs=max_seqs, max_batch=max_batch)


def weight_table(ccfg: DtkConfig) -> List[DtkWeightInfo]:
    lib = _lib.load_library()
    n = lib.dtk_weight_count(C.byref(ccfg))
    if n <= 0:
        raise EngineError("invalid engine configuration (dtk_weight_count)")
    out = []
    for i in range(n):
        info = DtkWeightInfo()
        if lib.dtk_weight_get(C.byref(ccfg), i, C.byref(info)) != 0:
            raise EngineError("dtk_weight_get failed")
        out.append(info)
    return out


def _arena_source(name: str, sd: Dict[str, torch.Tensor], cfg: "DetikzifyConfig", cols: int) -> torch.Tensor:
    """Arena tensor ``name`` as a function of the canonical (HF-named) state dict."""
    parts = name.split(".")
    if name == "dec.embed":
        return sd["model.embed_tokens.weight"]
    if name == "dec.norm":
        return sd["model.norm.weight"]
    if name == "dec.lm_head":
        return sd["lm_head.weight"]
    if name == "proj.w":
        return sd["model.mm_projector.weight"]
    if name == "proj.b":
        b = sd.get("model.mm_projector.bias")
        return b if b is not None else torch.zeros(cfg.hidden_size)
    if parts[0] == "dec":
        p = f"model.layers.{int(parts[1][1:])}."
        k = parts[2]
        if k == "norm1":
            return sd[p + "input_layernorm.weight"]
        if k == "norm2":
            return sd[p + "post_attention_layernorm.weight"]
        if k == "wqkv":
            return torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)
        if k == "wo":
            return sd[p + "self_attn.o_proj.weight"]
        if k == "wgu":  # interleave rows: 2i = gate_i, 2i+1 = up_i (SwiGLU pair lands in one warp / one mma column pair)
            g, u = sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]
            return torch.stack([g, u], dim=1).reshape(-1, g.shape[1])
        if k == "wd":
            return sd[p + "mlp.down_proj.weight"]
    if parts[0] == "vit":
        if name == "vit.patch_w":
            w = sd[V + "embeddings.patch_embedding.weight"]
            w = w.reshape(w.shape[0], -1)
            out = torch.zeros(w.shape[0], cols, dtype=w.dtype)
            out[:, : w.shape[1]] = w
            return out
        if name == "vit.patch_b":
            return sd[V + "embeddings.patch_embedding.bias"]
        if name == "vit.pos":
            return sd[V + "embeddings.position_embedding.weight"]
        if name == "vit.post_w":
            return sd[V + "post_layernorm.weight"]
        if name == "vit.post_b":
            return sd[V + "post_layernorm.bias"]
        if parts[1] == "head":
            h = V + "head."
            D = cfg.vision_config.hidden_size
            k = parts[2]
            table = {
                "probe": lambda: sd[h + "probe"].reshape(-1),
                "wq": lambda: sd[h + "attention.in_proj_weight"][:D],
                "bq": lambda: sd[h + "attention.in_proj_bias"][:D],
                "wkv": lambda: sd[h + "attention.in_proj_weight"][D:],
                "bkv": lambda: sd[h + "attention.in_proj_bias"][D:],
                "wo": lambda: sd[h + "attention.out_proj.weight"],
                "bo": lambda: sd[h + "attention.out_proj.bias"],
                "ln_w": lambda: sd[h + "layernorm.weight"],
                "ln_b": lambda: sd[h + "layernorm.bias"],
                "w1": lambda: sd[h + "mlp.fc1.weight"], "b1": lambda: sd[h + "mlp.fc1.bias"],
                "w2": lambda: sd[h + "mlp.fc2.weight"], "b2": lambda: sd[h + "mlp.fc2.bias"],
            }
            return table[k]()
        p = V + f"encoder.layers.{int(parts[1][1:])}."
        k = parts[2]
        simple = {"ln1_w": "layer_norm1.weight", "ln1_b": "layer_norm1.bias", "ln2_w": "layer_norm2.weight",
                  "ln2_b": "layer_norm2.bias", "wo": "self_attn.out_proj.weight", "bo": "self_attn.out_proj.bias",
                  "w1": "mlp.fc1.weight", "b1": "mlp.fc1.bias", "w2": "mlp.fc2.weight", "b2": "mlp.fc2.bias"}
        if k in simple:
            return sd[p + simple[k]]
        if k == "wqkv":
            return torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)
        if k == "bqkv":
            return torch.cat([sd[p + f"self_attn.{n}_proj.bias"] for n in "qkv"], dim=0)
    raise KeyError(name)


def pack_arena(cfg: "DetikzifyConfig", sd: Dict[str, torch.Tensor], ccfg: Optional[DtkConfig] = None) -> torch.Tensor:
    """Pack the canonical state dict into one contiguous bf16 arena (CPU uint8 tensor)."""
    lib = _lib.load_library()
    ccfg = ccfg or to_c_config(cfg)
    nbytes = lib.dtk_arena_bytes(C.byref(ccfg))
    if nbytes == 0:
        raise EngineError("invalid engine configuration (dtk_arena_bytes)")
    arena = torch.zeros(nbytes // 2, dtype=torch.bfloat16)
    for info in weight_table(ccfg):
        name = info.name.decode()
        src = _arena_source(name, sd, cfg, info.cols).to(torch.bfloat16).reshape(-1)
        if src.numel() != info.rows * info.cols:
            raise EngineError(f"{name}: expected {info.rows}x{info.cols}, got {src.numel()} elements")
        arena[info.offset // 2: info.offset // 2 + src.numel()] = src
    return arena


def random_arena_device(cfg: "DetikzifyConfig", device, seed: int = 0, ccfg: Optional[DtkConfig] = None) -> torch.Tensor:
    """Synthetic weights generated directly in the device arena (benches only: seconds instead of minutes for ds-7b).
    Same distribution as ``weights.random_init`` (matrices/biases N(0, 0.02^2), norm gains 1 + N(0, 0.02^2)) but a
    different random stream — parity tests use the CPU-seeded ``random_init`` + ``pack_arena``, which the oracle shares."""
    lib = _lib.load_library()
    ccfg = ccfg or to_c_config(cfg)
    nbytes = lib.dtk_arena_bytes(C.byref(ccfg))
    if nbytes == 0:
        raise EngineError("invalid engine configuration (dtk_arena_bytes)")
    dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
    g = torch.Generator(device=dev).manual_seed(seed)
    arena = torch.empty(nbytes // 2, dtype=torch.bfloat16, device=dev)
    step = 1 << 28
    for o in range(0, arena.numel(), step):            # chunked: the fp32 temporary stays at 1 GiB
        n = min(step, arena.numel() - o)
        arena[o:o + n] = (torch.randn(n, device=dev, dtype=torch.float32, generator=g) * 0.02).to(torch.bfloat16)
    gains = ("norm1", "norm2", "ln1_w", "ln2_w", "ln_w", "post_w")
    for info in weight_table(ccfg):
        name = info.name.decode()
        if name == "dec.norm" or name.split(".")[-1] in gains:
            sl = arena[info.offset // 2: info.offset // 2 + info.rows * info.cols]
            sl.copy_((sl.float() + 1.0).to(torch.bfloat16))
        elif name == "vit.patch_w":                    # K padding columns (588 -> 640) must be zero
            vc = cfg.vision_config
            k = vc.num_channels * vc.patch_size * vc.patch_size
            arena[info.offset // 2: info.offset // 2 + info.rows * info.cols].view(info.rows, info.cols)[:, k:] = 0
    return arena


def _i32(xs: Sequence[int]):
    xs = [int(x) for x in xs]
    return (C.c_int32 * max(1, len(xs)))(*xs)


def c_processors(repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_p: float = 0.0, eos_token_id: int = -1,
                 ban_ids: Sequence[int] = (), begin_ids: Sequence[int] = (),
                 words: Sequence[Sequence[int]] = ()) -> DtkProcessors:
    """``dtk_processors`` (include/detikzify_b200.h): ``ban_ids`` always banned, ``begin_ids`` banned on rows whose suppress
    flag is set, ``words`` bad-word sequences of two or more ids. The struct keeps its id arrays alive."""
    words = [[int(i) for i in w] for w in words]
    ban_ids, begin_ids = list(ban_ids), list(begin_ids)
    ban, begin = _i32(ban_ids), _i32(begin_ids)
    wid, wlen = _i32([i for w in words for i in w]), _i32([len(w) for w in words])
    p = DtkProcessors(repetition_penalty=float(repetition_penalty), min_p=float(min_p),
                      no_repeat_ngram_size=int(no_repeat_ngram_size), eos_token_id=int(eos_token_id),
                      ban_ids=ban, n_ban=len(ban_ids), begin_ids=begin, n_begin=len(begin_ids),
                      word_ids=wid, word_lens=wlen, n_words=len(words))
    p._arrays = (ban, begin, wid, wlen)
    return p


def c_histories(histories: Sequence[Sequence[int]]):
    """(concatenated ids, lengths) int32 arrays of per-row token histories."""
    flat = [int(i) for h in histories for i in h]
    return _i32(flat), _i32([len(h) for h in histories])


class Engine:
    """One engine per CUDA device. Not thread-safe: one generation thread at a time."""

    def __init__(self, cfg: "DetikzifyConfig", arena: torch.Tensor, device: torch.device | int | str = 0,
                 max_seqs: int = 4, max_batch: int = 1, max_len: Optional[int] = None):
        if not torch.cuda.is_available():
            raise EngineError("detikzify_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.lib = _lib.load_library()
        self.cfg = cfg
        self.device = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if self.device.type != "cuda":
            raise EngineError(f"unsupported device {self.device}")
        self.ccfg = to_c_config(cfg, max_seqs=max_seqs, max_batch=max_batch, max_len=max_len)
        self.max_len, self.max_batch = self.ccfg.max_len, self.ccfg.max_batch
        self.arena = arena.to(self.device, non_blocking=False).contiguous()
        self._h = C.c_void_p()
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        rc = self.lib.dtk_create(C.byref(self.ccfg), C.c_void_p(self.arena.data_ptr()),
                                 C.c_uint64(self.arena.numel() * self.arena.element_size()), idx, C.byref(self._h))
        if rc != 0:
            msg = self.lib.dtk_last_error(self._h).decode() if self._h else "dtk_create failed"
            if self._h:
                self.lib.dtk_destroy(self._h)
                self._h = C.c_void_p()
            raise EngineError(f"dtk_create: {msg} (rc={rc})")
        vc = cfg.vision_config
        self.N, self.D, self.P, self.H, self.Vocab = vc.num_positions, vc.hidden_size, cfg.num_patches, cfg.hidden_size, cfg.vocab_size

    # ------------------------------------------------------------------ plumbing
    def _check(self, rc: int, what: str):
        if rc != 0:
            raise EngineError(f"{what}: {self.lib.dtk_last_error(self._h).decode()} (rc={rc})")

    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    @staticmethod
    def _ptr(t: Optional[torch.Tensor]) -> C.c_void_p:
        return C.c_void_p(0 if t is None else t.data_ptr())

    def close(self):
        if getattr(self, "_h", None):
            self.lib.dtk_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launch_count(self) -> int:
        return int(self.lib.dtk_launch_count(self._h))

    def set_option(self, key: str, value: int):
        self._check(self.lib.dtk_set_option(self._h, key.encode(), int(value)), "dtk_set_option")

    def get_option(self, key: str) -> int:
        v = C.c_int64(0)
        self._check(self.lib.dtk_get_option(self._h, key.encode(), C.byref(v)), "dtk_get_option")
        return int(v.value)

    def decode_bytes(self, context_len: int) -> int:
        """HBM bytes of one batch-1 decode step at ``context_len``: the weight bytes the persistent kernel streams in the
        current mode (option ``decode_weight_bytes``: e4m3 layer matrices with ``decode_fp8``, 13-bit packed tiles with
        ``decode_pack``) plus the cached keys/values."""
        kv = self.lib.dtk_decode_bytes(C.byref(self.ccfg), context_len) - self.lib.dtk_decode_bytes(C.byref(self.ccfg), 0)
        return self.get_option("decode_weight_bytes") + int(kv)

    # ------------------------------------------------------------------ vision
    def vit_encode(self, pixels: torch.Tensor, want_tokens: bool = True, want_pooled: bool = True):
        """pixels fp32 [B,3,S,S] on device -> (tokens fp32 [B,N,D] | None, pooled fp32 [B,D] | None)."""
        pixels = pixels.to(self.device, torch.float32).contiguous()
        B = pixels.shape[0]
        assert pixels.shape[1:] == (3, self.cfg.vision_config.image_size, self.cfg.vision_config.image_size), pixels.shape
        tokens = torch.empty(B, self.N, self.D, device=self.device, dtype=torch.float32) if want_tokens else None
        pooled = torch.empty(B, self.D, device=self.device, dtype=torch.float32) if want_pooled else None
        self._check(self.lib.dtk_vit_encode(self._h, self._ptr(pixels), B, self._ptr(tokens), self._ptr(pooled), self._stream()), "dtk_vit_encode")
        return tokens, pooled

    def image_preprocess(self, rgb: torch.Tensor, size: int, rescale: float, mean, std, out: torch.Tensor,
                         want_uint8: bool = False) -> Optional[torch.Tensor]:
        """rgb uint8 [h, w, 3] on the device -> ``out`` fp32 [3, size, size] (Pillow-exact bicubic resize, rescale, normalise)."""
        from .model.processing import pil_resample_coeffs
        h, w, ch = rgb.shape
        assert ch == 3 and rgb.dtype == torch.uint8 and rgb.is_contiguous()
        bh, chh, kh = pil_resample_coeffs(w, size)
        bv, cvv, kv = pil_resample_coeffs(h, size)
        dev = [t.to(self.device, non_blocking=True) for t in (bh, chh, bv, cvv)]
        tmp = torch.empty(h, size, 3, dtype=torch.uint8, device=self.device)
        u8 = torch.empty(size, size, 3, dtype=torch.uint8, device=self.device) if want_uint8 else None
        m3, s3 = (C.c_float * 3)(*mean), (C.c_float * 3)(*std)
        self._check(self.lib.dtk_image_preprocess(self._h, self._ptr(rgb), h, w, size, self._ptr(dev[0]), self._ptr(dev[1]), kh,
                                                  self._ptr(dev[2]), self._ptr(dev[3]), kv, float(rescale), m3, s3,
                                                  self._ptr(tmp), self._ptr(out), self._ptr(u8), self._stream()), "dtk_image_preprocess")
        return u8

    def project(self, tokens: torch.Tensor) -> torch.Tensor:
        tokens = tokens.to(self.device, torch.float32).contiguous()
        B = tokens.shape[0]
        out = torch.empty(B, self.P, self.H, device=self.device, dtype=torch.float32)
        self._check(self.lib.dtk_project(self._h, self._ptr(tokens), B, self._ptr(out), self._stream()), "dtk_project")
        return out

    def image_embeds(self, pixels: torch.Tensor) -> torch.Tensor:
        tokens, _ = self.vit_encode(pixels, want_pooled=False)
        return self.project(tokens)

    # ------------------------------------------------------------------ TikZero adapter
    def adapter_attach(self, cacfg, arena: torch.Tensor):
        """Attach the adapter arena (bf16, ``adapter_weight_table`` layout); the engine borrows it until detach."""
        self.adapter_arena = arena.to(self.device).contiguous()
        self.cacfg = cacfg
        self._check(self.lib.dtk_adapter_attach(self._h, C.byref(cacfg), self._ptr(self.adapter_arena),
                                                C.c_uint64(self.adapter_arena.numel() * self.adapter_arena.element_size())),
                    "dtk_adapter_attach")

    def adapter_detach(self):
        self._check(self.lib.dtk_adapter_detach(self._h), "dtk_adapter_detach")
        self.adapter_arena = self.cacfg = None

    def text_encode(self, ids: torch.Tensor, want_hidden: bool = False):
        """One unpadded caption, ids int64 [T] -> (hidden fp32 [T,E] | None, caption states fp32 [T,D])."""
        ids = torch.as_tensor(ids).to(self.device, torch.int64).contiguous().view(-1)
        T = ids.numel()
        hidden = torch.empty(T, self.cacfg.hidden, device=self.device, dtype=torch.float32) if want_hidden else None
        cond = torch.empty(T, self.D, device=self.device, dtype=torch.float32)
        self._check(self.lib.dtk_text_encode(self._h, self._ptr(ids), T, self._ptr(hidden), self._ptr(cond), self._stream()),
                    "dtk_text_encode")
        return hidden, cond

    def vit_encode_cond(self, pixels: torch.Tensor, captions: Sequence[torch.Tensor], want_tokens: bool = True,
                        want_pooled: bool = True):
        """ViT with the adapter's cross layers: image b conditioned on caption ids ``captions[b]`` (unpadded int64 [T_b])."""
        pixels = pixels.to(self.device, torch.float32).contiguous()
        B = pixels.shape[0]
        assert len(captions) == B, (len(captions), B)
        lens = [int(c.numel()) for c in captions]
        Tmax = max(lens)
        cond = torch.zeros(B, Tmax, self.D, device=self.device, dtype=torch.float32)
        for b, ids in enumerate(captions):
            cond[b, : lens[b]] = self.text_encode(ids)[1]
        return self.vit_encode_states(pixels, cond, lens, want_tokens, want_pooled)

    def vit_encode_states(self, pixels: torch.Tensor, cond: torch.Tensor, lens: Sequence[int], want_tokens: bool = True,
                          want_pooled: bool = True):
        """pixels fp32 [B,3,S,S], caption states fp32 [B,Tmax,D] (``text_encode`` output, caption b valid in rows < lens[b])."""
        pixels = pixels.to(self.device, torch.float32).contiguous()
        cond = cond.to(self.device, torch.float32).contiguous()
        B, Tmax = pixels.shape[0], cond.shape[1]
        tokens = torch.empty(B, self.N, self.D, device=self.device, dtype=torch.float32) if want_tokens else None
        pooled = torch.empty(B, self.D, device=self.device, dtype=torch.float32) if want_pooled else None
        cl = (C.c_int * B)(*lens)
        self._check(self.lib.dtk_vit_encode_cond(self._h, self._ptr(pixels), B, self._ptr(cond), cl, Tmax, self._ptr(tokens),
                                                 self._ptr(pooled), self._stream()), "dtk_vit_encode_cond")
        return tokens, pooled

    def image_embeds_cond(self, pixels: torch.Tensor, captions: Sequence[torch.Tensor]) -> torch.Tensor:
        tokens, _ = self.vit_encode_cond(pixels, captions, want_pooled=False)
        return self.project(tokens)

    # ------------------------------------------------------------------ KV slots
    def seq_alloc(self) -> int:
        s = C.c_int(-1)
        self._check(self.lib.dtk_seq_alloc(self._h, C.byref(s)), "dtk_seq_alloc")
        return s.value

    def seq_free(self, slot: int):
        self._check(self.lib.dtk_seq_free(self._h, slot), "dtk_seq_free")

    def seq_fork(self, src: int, dst: int, length: int):
        self._check(self.lib.dtk_seq_fork(self._h, src, dst, length, self._stream()), "dtk_seq_fork")

    def seq_share(self, base: int, dst: int, length: int):
        """dst reads cached positions [0, length) from ``base`` (reference counted, no copy of whole 16-position blocks)."""
        self._check(self.lib.dtk_seq_share(self._h, base, dst, length, self._stream()), "dtk_seq_share")

    # ------------------------------------------------------------------ decoder
    def prefill(self, slot: int, ids: torch.Tensor, start_pos: int = 0, img_embeds: Optional[torch.Tensor] = None,
                img_start: int = 0, want_all_logits: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        """ids int64 [T] on device. Returns (last_logits fp32 [V], all_logits fp32 [T,V] | None)."""
        ids = ids.to(self.device, torch.int64).contiguous().view(-1)
        T = ids.numel()
        last = torch.empty(self.Vocab, device=self.device, dtype=torch.float32)
        alll = torch.empty(T, self.Vocab, device=self.device, dtype=torch.float32) if want_all_logits else None
        n_img = 0
        if img_embeds is not None:
            img_embeds = img_embeds.to(self.device, torch.float32).contiguous().view(-1, self.H)
            n_img = img_embeds.shape[0]
        self._check(self.lib.dtk_prefill(self._h, slot, self._ptr(ids), T, start_pos, self._ptr(img_embeds), img_start,
                                         n_img, self._ptr(last), self._ptr(alll), self._stream()), "dtk_prefill")
        return last, alll

    def score(self, slot: int, ids: torch.Tensor, start_pos: int = 0, img_embeds: Optional[torch.Tensor] = None,
              img_start: int = 0, targets: Optional[torch.Tensor] = None, want_all_logits: bool = False, *,
              logits_out: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
        """Prefill ids int64 [T] like ``prefill`` and score every row with the fused lm_head log-softmax. ``targets`` int64 [T]
        (negative = none). Returns (logprob fp32 [T] (0 where there is no target), lse fp32 [T], all_logits fp32 [T,V] | None).
        ``logits_out``: a contiguous fp32 [T,V] device tensor (e.g. rows of a larger batch output) that receives the logits."""
        if targets is None:
            raise ValueError("score() needs targets: int64 [T], negative = no target")
        ids = ids.to(self.device, torch.int64).contiguous().view(-1)
        T = ids.numel()
        targets = targets.to(self.device, torch.int64).contiguous().view(-1)
        if targets.numel() != T:
            raise ValueError(f"targets must hold one entry per id ({targets.numel()} != {T})")
        if logits_out is not None:
            if logits_out.device != self.device or logits_out.dtype != torch.float32 or not logits_out.is_contiguous() \
                    or logits_out.numel() != T * self.Vocab:
                raise ValueError("logits_out must be a contiguous fp32 [T, V] tensor on the engine's device")
        elif want_all_logits:
            logits_out = torch.empty(T, self.Vocab, device=self.device, dtype=torch.float32)
        logprob = torch.empty(T, device=self.device, dtype=torch.float32)
        lse = torch.empty(T, device=self.device, dtype=torch.float32)
        n_img = 0
        if img_embeds is not None:
            img_embeds = img_embeds.to(self.device, torch.float32).contiguous().view(-1, self.H)
            n_img = img_embeds.shape[0]
        self._check(self.lib.dtk_score(self._h, slot, self._ptr(ids), T, start_pos, self._ptr(img_embeds), img_start, n_img,
                                       self._ptr(targets), self._ptr(logprob), self._ptr(lse), self._ptr(logits_out),
                                       self._stream()), "dtk_score")
        return logprob, lse, logits_out

    def decode(self, slots: Sequence[int], positions: Sequence[int], ids: torch.Tensor) -> torch.Tensor:
        B = len(slots)
        ids = ids.to(self.device, torch.int64).contiguous().view(-1)
        assert ids.numel() == B
        logits = torch.empty(B, self.Vocab, device=self.device, dtype=torch.float32)
        cs, cp = (C.c_int * B)(*slots), (C.c_int * B)(*positions)
        self._check(self.lib.dtk_decode(self._h, cs, cp, self._ptr(ids), B, self._ptr(logits), self._stream()), "dtk_decode")
        return logits

    @staticmethod
    def sampling(temperature: float = 1.0, top_p: float = 1.0, top_k: int = 0, do_sample: bool = False,
                 bad_token: int = -1, begin_suppress_token: int = -1, seed: int = 0) -> DtkSampling:
        return DtkSampling(temperature=float(temperature), top_p=float(top_p), top_k=int(top_k or 0),
                           do_sample=int(bool(do_sample)), bad_token=int(bad_token),
                           begin_suppress_token=int(begin_suppress_token), seed=int(seed) & (2**64 - 1))

    def sample(self, logits: torch.Tensor, params: DtkSampling, suppress: Optional[Sequence[int]] = None,
               steps: Optional[Sequence[int]] = None, seq_ids: Optional[Sequence[int]] = None,
               want_probs: bool = False):
        logits = logits.to(self.device, torch.float32).contiguous().view(-1, self.Vocab)
        B = logits.shape[0]
        out = torch.empty(B, device=self.device, dtype=torch.int64)
        probs = torch.empty(B, self.Vocab, device=self.device, dtype=torch.float32) if want_probs else None
        cs = (C.c_int * B)(*(suppress or [0] * B))
        ct = (C.c_uint32 * B)(*(steps or [0] * B))
        ci = (C.c_uint32 * B)(*(seq_ids or list(range(B))))
        self._check(self.lib.dtk_sample(self._h, self._ptr(logits), B, C.byref(params), cs, ct, ci, self._ptr(out),
                                        self._ptr(probs), self._stream()), "dtk_sample")
        return out, probs

    def set_processors(self, proc: Optional[dict], histories: Sequence[Sequence[int]] = (),
                       eos_min_len: Optional[Sequence[int]] = None):
        """HF logits processors for the following ``sample`` / ``gen_begin`` calls (``dtk_set_processors``); ``proc`` holds
        ``c_processors`` keywords, None turns them off. ``histories[b]``: row b's ids so far (prompt + tokens, ending with
        the first pending token before ``gen_begin``); ``eos_min_len[b]``: EOS is banned while the row is shorter."""
        if proc is None:
            self._check(self.lib.dtk_set_processors(self._h, None, 0, None, None, None, self._stream()), "dtk_set_processors")
            return
        B = len(histories)
        cp = c_processors(**proc)
        ids, lens = c_histories(histories)
        eml = _i32(eos_min_len) if eos_min_len is not None else None
        self._check(self.lib.dtk_set_processors(self._h, C.byref(cp), B, ids, lens, eml, self._stream()), "dtk_set_processors")

    # ------------------------------------------------------------------ fused generation loop
    def gen_begin(self, slots: Sequence[int], positions: Sequence[int], first_ids: Sequence[int], params: DtkSampling,
                  seq_ids: Optional[Sequence[int]] = None):
        B = len(slots)
        cs, cp = (C.c_int * B)(*slots), (C.c_int * B)(*positions)
        cf = (C.c_int64 * B)(*first_ids)
        ci = (C.c_uint32 * B)(*(seq_ids or list(range(B))))
        self._gen_B = B
        self._gen_out = (C.c_int32 * B)()
        self._check(self.lib.dtk_gen_begin(self._h, cs, cp, cf, B, C.byref(params), ci, self._stream()), "dtk_gen_begin")

    def gen_step(self):
        self._check(self.lib.dtk_gen_step(self._h, self._stream()), "dtk_gen_step")

    def gen_wait(self, step: int) -> List[int]:
        self._check(self.lib.dtk_gen_wait(self._h, step, self._gen_out), "dtk_gen_wait")
        return list(self._gen_out)

    def gen_admit(self, row: int, slot: int, position: int, logits: torch.Tensor, seq_id: int,
                  history: Optional[Sequence[int]] = None, eos_min_len: int = 0):
        """Put a new sequence into inactive row ``row`` of the running loop (``dtk_gen_admit``): ``slot`` holds its prompt up
        to ``position``, ``logits`` fp32 [V] are the prompt's last-position logits; ``history`` (the prompt) and
        ``eos_min_len`` matter while processors are set. The first token is drawn on the device; ``gen_first`` returns it."""
        logits = logits.to(self.device, torch.float32).contiguous()
        hist = list(history or [])
        self._check(self.lib.dtk_gen_admit(self._h, row, slot, position, self._ptr(logits), C.c_uint32(seq_id), _i32(hist),
                                           len(hist), int(eos_min_len), self._stream()), "dtk_gen_admit")

    def gen_retire(self, row: int):
        self._check(self.lib.dtk_gen_retire(self._h, row, self._stream()), "dtk_gen_retire")

    def gen_first(self, row: int) -> int:
        t = C.c_int32(0)
        self._check(self.lib.dtk_gen_first(self._h, row, C.byref(t)), "dtk_gen_first")
        return t.value

    def gen_end(self):
        self._check(self.lib.dtk_gen_end(self._h), "dtk_gen_end")
