"""
Model object with the reference's duck-typed surface (SURVEY.md §8b), backed by the C-ABI engine.

Replaces detikzify/model/v1/modeling_detikzify.py (DetikzifyVisionModel :49-72, DetikzifyModel
:75-200, DetikzifyForCausalLM :203-305) *and* the HF ``GenerationMixin.generate/_sample`` loop the
reference drives at detikzify/infer/generate.py:218-227. What callers rely on:

  model.generate(input_ids=[1,T0], bad_words_ids=[[id]], begin_suppress_tokens=[id], pixel_values=...,
                 streamer=..., stopping_criteria=[...], temperature, top_p, top_k, max_length,
                 do_sample, **ignored) -> LongTensor [1,T]          (infer/generate.py:218-227)
  model.device / model.dtype / model.name_or_path / model.config.* / model.generation_config
  model.model.vision_model(pixel_values=...) -> .last_hidden_state, .pooler_output
                                                               (evaluate/imagesim.py:87,101-107)

Beyond the reference (results unchanged): the ViT+projector output is cached per pixel tensor and the
KV cache of the working slot is reused across calls for the longest common token prefix, so an MCTS
expansion prefills only the tree-path suffix instead of re-encoding the image and re-prefilling
243 + len(prefix) tokens on every rollout (reference quirk, SURVEY.md Appendix B.5).
"""
from __future__ import annotations

import threading
from contextlib import nullcontext
from types import SimpleNamespace
from typing import Any, Dict, List, Optional, Sequence

import torch

from ..engine import Engine, EngineError, pack_arena
from ..util.generation import StoppingCriteriaList
from .configuration import DetikzifyConfig


class GenerationConfig:
    def __init__(self, **kw):
        self.__dict__.update(kw)

    def to_dict(self) -> Dict[str, Any]:
        return dict(self.__dict__)


class VisionOutput(SimpleNamespace):
    pass


class DetikzifyVisionModel:
    """``model.model.vision_model`` — callable like the reference's wrapper (v1/modeling:63-69)."""

    def __init__(self, owner: "DetikzifyForCausalLM"):
        self._owner = owner
        self.config = owner.config.vision_config

    def __call__(self, pixel_values: Optional[torch.Tensor] = None, adapter_input_ids=None, adapter_attention_mask=None,
                 **_) -> VisionOutput:
        return self.forward(pixel_values, adapter_input_ids, adapter_attention_mask)

    def forward(self, pixel_values: Optional[torch.Tensor] = None, adapter_input_ids=None,
                adapter_attention_mask=None) -> VisionOutput:
        """With ``adapter_input_ids`` (TikZero) the tower runs with the adapter's cross layers, on the clamped dummy input
        when there is no image (reference modeling_adapter.py:473-491, used by SelfSim for the caption side)."""
        o = self._owner
        caps = None
        if adapter_input_ids is not None:
            caps = o._captions(adapter_input_ids, adapter_attention_mask)
            if pixel_values is None:
                pixel_values = o.adapter.dummy_pixels().expand(len(caps), -1, -1, -1)
        with o._lock, o._on_stream():
            if caps is None:
                tokens, pooled = o.engine.vit_encode(pixel_values)
            else:
                tokens, pooled = o.engine.vit_encode_cond(pixel_values, [torch.tensor(c) for c in caps])
            # cast on the engine stream, before the sync: a tensor must not leave the side stream while work on it is pending
            tokens, pooled = tokens.to(o.dtype), pooled.to(o.dtype)
            o._sync()
        return VisionOutput(last_hidden_state=tokens, pooler_output=pooled)

    def get_intermediate_layers(self, pixel_values: torch.Tensor, n=None, norm: bool = True, **_):
        """Only the configuration the reference uses: last layer, final norm applied
        (v1/modeling_detikzify.py:134 with feature_layer=-1)."""
        return [self.forward(pixel_values).last_hidden_state]


class _Inner:
    """``model.model`` namespace (reference: DetikzifyModel)."""

    def __init__(self, owner):
        self.vision_model = DetikzifyVisionModel(owner)


class _KVSlot:
    """One engine KV slot owned by generate(): the token history whose keys/values it holds, and an LRU tick."""
    __slots__ = ("slot", "tokens", "tick")

    def __init__(self, slot: int):
        self.slot, self.tokens, self.tick = slot, [], 0


class DetikzifyForCausalLM:
    def __init__(self, config: DetikzifyConfig, arena: Optional[torch.Tensor] = None, device=0, dtype=torch.bfloat16,
                 max_seqs: int = 2, max_batch: int = 1, max_len: Optional[int] = None, engine=None,
                 prefix_slots: Optional[int] = None):
        self.config = config
        self.dtype = dtype
        self.name_or_path = config.name_or_path
        # ``engine`` injection exists for host-logic tests (a scripted engine on CPU); the product path always
        # builds the CUDA engine and raises if no device / library is available.
        self.engine = engine if engine is not None else Engine(config, arena, device=device, max_seqs=max_seqs,
                                                                max_batch=max_batch, max_len=max_len)
        self.device = self.engine.device
        self.generation_config = GenerationConfig(
            max_length=config.model_max_length, do_sample=False, temperature=1.0, top_p=1.0, top_k=0,
            bos_token_id=config.bos_token_id, eos_token_id=config.eos_token_id, pad_token_id=config.pad_token_id)
        self.model = _Inner(self)
        self._lock = threading.Lock()
        self._stream = torch.cuda.Stream(device=self.device) if self.device.type == "cuda" else None
        # KV prefix cache of generate(): up to ``prefix_slots`` engine slots, each remembering the token history whose KV
        # it holds. An MCTS expansion prefills only what the best-matching slot does not already hold; when the prompt
        # diverges from that slot's content the shared prefix is forked (one device copy) into the least recently used
        # slot, so alternating between branches of the search tree does not thrash a single working slot. The reference
        # recomputes the whole prompt on every rollout; results are unchanged.
        self._kv_max = max(1, prefix_slots if prefix_slots is not None else max_seqs - max_batch)
        self._kv: List[_KVSlot] = [_KVSlot(self.engine.seq_alloc())]
        self._kv_cur = self._kv[0]
        self._tick = 0
        self._img_cache = None                  # (pixel tensor on device, image embeds [P,H], caption ids or None)
        self._call_counter = 0

    # (kept for callers that reset the cache: ``model._slot_tokens = []`` forgets every cached prefix)
    @property
    def _slot_tokens(self) -> List[int]:
        return self._kv_cur.tokens

    @_slot_tokens.setter
    def _slot_tokens(self, value: List[int]):
        if not value:
            for kv in self._kv:
                kv.tokens = []
        else:
            self._kv_cur.tokens = list(value)

    @property
    def _slot(self) -> int:
        return self._kv_cur.slot

    def _pick_slot(self, ids_host: List[int], span_start: int, span_len: int) -> int:
        """Choose the KV slot for this prompt and make it hold the longest reusable prefix; returns its length L
        (tokens [0, L) are valid in ``self._kv_cur``; never splits the image span [span_start, span_start+span_len))."""
        T0 = len(ids_host)

        def lcp(tokens: List[int]) -> int:
            n, lim = 0, min(len(tokens), T0 - 1)
            while n < lim and tokens[n] == ids_host[n]:
                n += 1
            if span_len and n < span_start + span_len:
                n = min(n, span_start)
            return n
        best = max(self._kv, key=lambda kv: (lcp(kv.tokens), kv.tick))
        L = lcp(best.tokens)
        use = best
        if self._kv_max > 1 and L < len(best.tokens):
            # the prompt leaves the slot's content: keep that content for later prompts and continue in another slot
            victim = None
            if len(self._kv) < self._kv_max:
                try:
                    victim = _KVSlot(self.engine.seq_alloc())
                    self._kv.append(victim)
                except Exception:        # the engine has no free slot left (other users): continue in place
                    victim, self._kv_max = None, len(self._kv)
            if victim is None:
                others = [kv for kv in self._kv if kv is not best]
                victim = min(others, key=lambda kv: kv.tick) if others else None
            if victim is not None:
                if L > 0:
                    self.engine.seq_fork(best.slot, victim.slot, L)
                victim.tokens = best.tokens[:L]
                use = victim
        self._tick += 1
        use.tick = self._tick
        self._kv_cur = use
        return L

    def _on_stream(self):
        return torch.cuda.stream(self._stream) if self._stream is not None else nullcontext()

    def _sync(self):
        if self._stream is not None:
            self._stream.synchronize()

    # ---- reference-compat trivia ---------------------------------------------------------------
    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def requires_grad_(self, *_):
        return self

    def get_model(self):
        return self.model

    # ---- image features (cached per pixel tensor and caption) -----------------------------------
    def _image_embeds(self, pixel_values: torch.Tensor, caption: Optional[List[int]] = None) -> torch.Tensor:
        pix = pixel_values.to(self.device, torch.float32, non_blocking=True)
        if pix.dim() == 3:
            pix = pix[None]
        if pix.shape[0] != 1:
            raise ValueError("generate() supports a single image (batch size 1), like the reference's streamers")
        key = tuple(caption) if caption is not None else None
        cached = self._img_cache
        if cached is not None and cached[2] == key and cached[0].shape == pix.shape and torch.equal(cached[0], pix):
            return cached[1]
        emb = (self.engine.image_embeds(pix) if key is None else self.engine.image_embeds_cond(pix, [torch.tensor(key)]))[0]
        self._img_cache = (pix.clone(), emb, key)
        self._slot_tokens = []  # KV of the image prefix is stale for a new image or caption
        return emb

    # ---- TikZero adapter -------------------------------------------------------------------------
    def has_adapter(self) -> bool:
        return hasattr(self, "adapter")

    def unload_cross_attn_adapter(self):
        """Detach the adapter (reference modeling_adapter.py:528-532); image features conditioned on a caption are dropped."""
        with self._lock:
            self.engine.adapter_detach()
            del self.adapter, self.embedding_model
            self._img_cache = None
            self._slot_tokens = []

    def _captions(self, adapter_input_ids, adapter_attention_mask) -> List[List[int]]:
        """Caption ids per row, padding removed (right padding: the valid rows of the causal embedder are the unpadded ones)."""
        if not self.has_adapter():
            raise ValueError("Got `adapter_input_ids` but no adapter is loaded!")
        ids = torch.as_tensor(adapter_input_ids)
        ids = ids[None] if ids.dim() == 1 else ids
        mask = None if adapter_attention_mask is None else torch.as_tensor(adapter_attention_mask).reshape(ids.shape)
        out = []
        for r in range(ids.shape[0]):
            row = ids[r] if mask is None else ids[r][mask[r].bool()]
            if row.numel() == 0:
                raise ValueError("empty caption")
            if row.numel() > self.adapter.config.max_text:
                raise ValueError(f"caption longer than {self.adapter.config.max_text} tokens (truncate it in the processor)")
            out.append(row.tolist())
        return out

    @staticmethod
    def _first(seq, default=-1) -> int:
        try:
            v = seq[0]
            while isinstance(v, (list, tuple)):
                v = v[0]
            return int(v)
        except (TypeError, IndexError):
            return default

    # ---- generate --------------------------------------------------------------------------------
    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor = None, pixel_values: Optional[torch.Tensor] = None,
                 bad_words_ids=None, begin_suppress_tokens=None, streamer=None, stopping_criteria=None,
                 temperature: Optional[float] = None, top_p: Optional[float] = None, top_k: Optional[int] = None,
                 max_length: Optional[int] = None, max_new_tokens: Optional[int] = None,
                 do_sample: Optional[bool] = None, seed: Optional[int] = None, eos_token_id: Optional[int] = None,
                 adapter_input_ids=None, adapter_attention_mask=None, **ignored) -> torch.Tensor:
        cfg, eng = self.config, self.engine
        caption = None
        if adapter_input_ids is not None:
            caps = self._captions(adapter_input_ids, adapter_attention_mask)
            if len(caps) != 1:
                raise ValueError("generate() is batch-1: pass one caption")
            caption = caps[0]
            if pixel_values is None:
                pixel_values = self.adapter.dummy_pixels()
        gc = self.generation_config
        temperature = gc.temperature if temperature is None else temperature
        top_p = gc.top_p if top_p is None else top_p
        top_k = gc.top_k if top_k is None else top_k
        do_sample = gc.do_sample if do_sample is None else do_sample
        eos = cfg.eos_token_id if eos_token_id is None else eos_token_id

        ids2d = input_ids if input_ids.dim() == 2 else input_ids[None]
        if ids2d.shape[0] != 1:
            raise ValueError("generate() is batch-1 (use generate_batch for parallel rollouts)")
        ids_host: List[int] = ids2d[0].tolist()
        T0 = len(ids_host)
        if max_length is None:
            max_length = T0 + max_new_tokens if max_new_tokens is not None else gc.max_length
        max_length = min(int(max_length), eng.max_len)
        criteria = StoppingCriteriaList(stopping_criteria or [])

        with self._lock, self._on_stream():
            # -- splice validation (v1/modeling_detikzify.py:176-184)
            img, img_start = None, 0
            patch = cfg.image_token_id
            n_patch_tokens = ids_host.count(patch)
            if pixel_values is not None and n_patch_tokens > 0:
                if n_patch_tokens != cfg.num_patches:
                    raise ValueError("The number of image patch tokens should be the same as the number of image patches.")
                img_start = ids_host.index(patch)
                if ids_host[img_start: img_start + n_patch_tokens] != [patch] * n_patch_tokens:
                    raise ValueError("The image patch tokens should be consecutive.")
                img = self._image_embeds(pixel_values, caption)
            elif pixel_values is None and n_patch_tokens:
                # patch tokens without an image: their KV comes from plain embeddings. Forget the image identity too, so a
                # later call WITH the same image re-validates nothing against these slots (ADVICE r1)
                self._img_cache = None
                self._slot_tokens = []
            if T0 == 0:
                raise ValueError("empty prompt")
            if streamer is not None:
                streamer.put(ids2d.cpu())
            if T0 >= max_length:
                if streamer is not None:
                    streamer.end()
                return ids2d.to(self.device)

            # -- longest common prefix with the KV already held by one of the cache slots
            L = self._pick_slot(ids_host, img_start, n_patch_tokens if img is not None else 0)
            ids_dev = torch.tensor(ids_host[L:], dtype=torch.int64)
            if self.device.type == "cuda":
                ids_dev = ids_dev.pin_memory().to(self.device, non_blocking=True)
            self._slot_tokens = list(ids_host[:L])     # if the prefill raises, the slot only claims what it held before
            last_logits, _ = eng.prefill(self._slot, ids_dev, L, img, img_start)
            self._slot_tokens = list(ids_host)

            self._call_counter += 1
            params = eng.sampling(
                temperature=temperature, top_p=top_p, top_k=top_k or 0, do_sample=bool(do_sample),
                bad_token=self._first(bad_words_ids), begin_suppress_token=self._first(begin_suppress_tokens),
                seed=(seed if seed is not None else torch.initial_seed() + self._call_counter))
            first, _ = eng.sample(last_logits, params, suppress=[1], steps=[0])
            tok = int(first.item())

            out_buf = torch.empty(1, max_length, dtype=torch.int64)
            out_buf[0, :T0] = ids2d[0].cpu()
            n_new = max_length - T0        # upper bound on new tokens
            new_tokens: List[int] = []
            launched = waited = 0
            started = False
            try:
                while True:
                    new_tokens.append(tok)
                    out_buf[0, T0 + len(new_tokens) - 1] = tok
                    if streamer is not None:
                        streamer.put(out_buf[0, T0 + len(new_tokens) - 1: T0 + len(new_tokens)])
                    cur = out_buf[:, : T0 + len(new_tokens)]
                    if tok == eos or len(new_tokens) >= n_new or criteria(cur, None):
                        break
                    if not started:
                        eng.gen_begin([self._slot], [T0], [tok], params)
                        started = True
                    while launched < waited + 2 and launched < n_new - 1:
                        eng.gen_step()
                        launched += 1
                    tok = eng.gen_wait(waited)[0]
                    waited += 1
            finally:
                if started:
                    eng.gen_end()
                # decode step s wrote KV at T0+s for new_tokens[s]; only tokens the host has seen count
                self._slot_tokens = list(ids_host) + new_tokens[: min(launched, len(new_tokens))]
            # exceptions escape before this point (the caller's error_callback feeds the streamer,
            # detikzify/infer/generate.py:252); the normal path always terminates the stream
            if streamer is not None:
                streamer.end()
            result = out_buf[:, : T0 + len(new_tokens)].to(self.device)
            self._sync()
            return result

    # ---- batched generation (extension; the reference's generate() is batch-1) ---------------------
    @torch.no_grad()
    def generate_batch(self, input_ids: Sequence[torch.Tensor], pixel_values: Optional[torch.Tensor] = None, *,
                       bad_words_ids=None, begin_suppress_tokens=None, temperature: Optional[float] = None,
                       top_p: Optional[float] = None, top_k: Optional[int] = None, max_length: Optional[int] = None,
                       max_new_tokens: Optional[int] = None, do_sample: Optional[bool] = None, seed: Optional[int] = None,
                       eos_token_id: Optional[int] = None, streamers: Optional[Sequence[Any]] = None,
                       stopping_criteria: Optional[Sequence[Any]] = None, share_prefix: bool = True,
                       adapter_input_ids=None, adapter_attention_mask=None, **ignored) -> List[torch.Tensor]:
        """N independent sequences decoded in lock-step: parallel MCTS rollouts of one figure (``pixel_values`` [1,3,S,S]
        shared) or N figures (``pixel_values`` [N,3,S,S]). One batched decode step per token — the decoder weights are
        streamed once per step for all N sequences instead of once per sequence — with the same logits processors and
        per-sequence RNG streams as N separate ``generate()`` calls (sequence i uses RNG stream i of ``seed``).

        Per-sequence host contract, as ``generate()`` has it for one sequence (reference util/generation.py:25-66 is batch-1
        only): ``streamers[i]`` (or None) receives the prompt as ``[1, T0]`` once, every new token as a ``[1]`` tensor and
        ``end()``; ``stopping_criteria[i]`` (a callable or a list of callables ``(input_ids [1,T], scores) -> bool``; one
        shared entry is also accepted) is evaluated after every token of sequence i and stops only that sequence. Every
        sequence also stops at its own EOS / ``max_length``; the loop ends when all have stopped.

        With one shared image the longest common token prefix of the prompts (image span + tree path of an MCTS
        expansion) is prefilled ONCE and lent to every sequence (``dtk_seq_share``: reference counted, read in place);
        each sequence prefills only its own suffix. Returns a list of 1-D id tensors (prompt included).
        N is bounded by the engine's ``max_batch`` and free KV slots (``load(..., max_seqs=, max_batch=)``)."""
        cfg, eng = self.config, self.engine
        gc = self.generation_config
        temperature = gc.temperature if temperature is None else temperature
        top_p = gc.top_p if top_p is None else top_p
        top_k = gc.top_k if top_k is None else top_k
        do_sample = gc.do_sample if do_sample is None else do_sample
        eos = cfg.eos_token_id if eos_token_id is None else eos_token_id
        prompts: List[List[int]] = [(p[0] if p.dim() == 2 else p).tolist() for p in input_ids]
        N = len(prompts)
        if N == 0:
            return []
        captions = None
        if adapter_input_ids is not None:
            captions = self._captions(adapter_input_ids, adapter_attention_mask)
            if len(captions) not in (1, N):
                raise ValueError("adapter_input_ids must hold one caption (shared) or one caption per sequence")
            if pixel_values is None:
                pixel_values = self.adapter.dummy_pixels()
        if any(len(p) == 0 for p in prompts):
            raise ValueError("empty prompt")
        streamers = list(streamers) if streamers is not None else [None] * N
        if len(streamers) != N:
            raise ValueError("streamers must hold one entry (or None) per sequence")
        crits: List[StoppingCriteriaList] = []
        sc = list(stopping_criteria) if stopping_criteria is not None else []
        per_seq = len(sc) == N and N > 1 or (len(sc) == N and all(isinstance(c, (list, tuple)) for c in sc))
        for i in range(N):
            c = sc[i] if per_seq else sc
            crits.append(StoppingCriteriaList(c if isinstance(c, (list, tuple)) else [c]))
        limits = []
        for p in prompts:
            ml = max_length if max_length is not None else (len(p) + max_new_tokens if max_new_tokens is not None else gc.max_length)
            limits.append(min(int(ml), eng.max_len))
        patch = cfg.image_token_id

        def spans(ids_host):
            n = ids_host.count(patch)
            if n == 0:
                return 0, 0
            if n != cfg.num_patches:   # splice validation (v1/modeling_detikzify.py:176-184)
                raise ValueError("The number of image patch tokens should be the same as the number of image patches.")
            st = ids_host.index(patch)
            if ids_host[st: st + n] != [patch] * n:
                raise ValueError("The image patch tokens should be consecutive.")
            return st, n

        with self._lock, self._on_stream():
            imgs = None
            if pixel_values is not None:
                pix = pixel_values.to(self.device, torch.float32)
                if pix.dim() == 3:
                    pix = pix[None]
                if pix.shape[0] not in (1, N):
                    raise ValueError("pixel_values must hold one image (shared) or one image per sequence")
                if captions is None:
                    imgs = eng.image_embeds(pix)
                else:   # one conditioned tower pass per distinct (image, caption) pairing
                    if pix.shape[0] != len(captions):
                        pix = pix.expand(N, *pix.shape[1:]).contiguous()
                        captions = captions * N if len(captions) == 1 else captions
                    imgs = eng.image_embeds_cond(pix, [torch.tensor(c) for c in captions])
            for i, st in enumerate(streamers):
                if st is not None:
                    st.put(torch.tensor([prompts[i]], dtype=torch.int64))
            slots: List[int] = []
            base_slot = None
            try:
                for _ in range(N):
                    slots.append(eng.seq_alloc())
                # longest common prefix of the prompts (never splitting an image span, never a whole prompt)
                lcp = 0
                one_image = imgs is None or imgs.shape[0] == 1
                if share_prefix and N > 1 and one_image:
                    lim = min(len(p) for p in prompts) - 1
                    while lcp < lim and all(p[lcp] == prompts[0][lcp] for p in prompts[1:]):
                        lcp += 1
                    st0, n0 = spans(prompts[0][:]) if imgs is not None else (0, 0)
                    if n0 and st0 < lcp < st0 + n0:
                        lcp = st0
                    if lcp < 16:
                        lcp = 0
                if lcp:
                    try:
                        base_slot = eng.seq_alloc()
                    except Exception:       # no spare slot: every sequence prefills its whole prompt
                        base_slot, lcp = None, 0
                if lcp:
                    st0, n0 = spans(prompts[0]) if imgs is not None else (0, 0)
                    head = torch.tensor(prompts[0][:lcp], dtype=torch.int64)
                    if self.device.type == "cuda":
                        head = head.pin_memory().to(self.device, non_blocking=True)
                    eng.prefill(base_slot, head, 0, imgs[0] if (imgs is not None and n0 and st0 < lcp) else None, st0)
                last = []
                for i, ids_host in enumerate(prompts):
                    img, img_start = None, 0
                    if imgs is not None:
                        img_start, n_patch = spans(ids_host)
                        if n_patch and img_start >= lcp:
                            img = imgs[i if imgs.shape[0] == N else 0]
                    if lcp:
                        eng.seq_share(base_slot, slots[i], lcp)
                    ids_dev = torch.tensor(ids_host[lcp:], dtype=torch.int64)
                    if self.device.type == "cuda":
                        ids_dev = ids_dev.pin_memory().to(self.device, non_blocking=True)
                    lg, _ = eng.prefill(slots[i], ids_dev, lcp, img, img_start)
                    last.append(lg)
                self._call_counter += 1
                params = eng.sampling(
                    temperature=temperature, top_p=top_p, top_k=top_k or 0, do_sample=bool(do_sample),
                    bad_token=self._first(bad_words_ids), begin_suppress_token=self._first(begin_suppress_tokens),
                    seed=(seed if seed is not None else torch.initial_seed() + self._call_counter))
                seq_ids = list(range(N))
                first, _ = eng.sample(torch.stack(last), params, suppress=[1] * N, steps=[0] * N, seq_ids=seq_ids)
                toks = [int(t) for t in first.tolist()]
                outs: List[List[int]] = [list(p) for p in prompts]
                done = [len(p) >= lim for p, lim in zip(prompts, limits)]   # prompt already at max_length: nothing appended

                def accept(i: int, tok: int):
                    outs[i].append(tok)
                    if streamers[i] is not None:
                        streamers[i].put(torch.tensor([tok], dtype=torch.int64))
                    cur = torch.tensor([outs[i]], dtype=torch.int64) if crits[i] else None
                    done[i] = tok == eos or len(outs[i]) >= limits[i] or (bool(crits[i]) and crits[i](cur, None))

                for i in range(N):
                    if not done[i]:
                        accept(i, toks[i])
                max_steps = max(lim - len(p) for p, lim in zip(prompts, limits)) - 1
                if not all(done) and max_steps > 0:
                    eng.gen_begin(slots, [len(p) for p in prompts], toks, params, seq_ids)
                    launched = waited = 0
                    try:
                        while not all(done) and waited < max_steps:
                            while launched < waited + 2 and launched < max_steps:
                                eng.gen_step()
                                launched += 1
                            row = eng.gen_wait(waited)
                            waited += 1
                            for i in range(N):
                                if not done[i]:          # finished sequences keep decoding on the device; the host ignores them
                                    accept(i, int(row[i]))
                    finally:
                        eng.gen_end()
                for st in streamers:
                    if st is not None:
                        st.end()
                result = [torch.tensor(o, dtype=torch.int64, device=self.device) for o in outs]
                self._sync()
                return result
            finally:
                for s in slots:
                    eng.seq_free(s)
                if base_slot is not None:
                    eng.seq_free(base_slot)

    # ---- SelfSim helper: pooled features straight from the engine --------------------------------
    @torch.no_grad()
    def pooled_features(self, pixel_values: torch.Tensor) -> torch.Tensor:
        with self._lock, self._on_stream():
            _, pooled = self.engine.vit_encode(pixel_values, want_tokens=False)
            self._sync()
        return pooled   # fp32, produced and synchronised on the engine stream

    def close(self):
        self.engine.close()
