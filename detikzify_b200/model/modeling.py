"""
Model object with the reference's duck-typed surface (SURVEY.md §8b), backed by the C-ABI engine.

Replaces detikzify/model/v1/modeling_detikzify.py (DetikzifyVisionModel :49-72, DetikzifyModel
:75-200, DetikzifyForCausalLM :203-305) *and* the HF ``GenerationMixin.generate/_sample`` loop the
reference drives at detikzify/infer/generate.py:218-227. What callers rely on:

  model.generate(input_ids=[1,T0], bad_words_ids=[[id]], begin_suppress_tokens=[id], pixel_values=...,
                 streamer=..., stopping_criteria=[...], temperature, top_p, top_k, max_length,
                 do_sample, **ignored) -> LongTensor [1,T]          (infer/generate.py:218-227)
  HF's other logits processors, applied on the device in HF's order (``_processors``): repetition_penalty,
  no_repeat_ngram_size, bad_words_ids (any number of entries of any length), min_length / min_new_tokens,
  suppress_tokens, begin_suppress_tokens (a list), and min_p when sampling. Each falls back to the
  ``generation_config`` attribute of the same name. Beam search, num_return_sequences, sequence_bias,
  typical / epsilon / eta cutoffs and Python logits_processor callables are ignored.
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
from collections import deque
from contextlib import nullcontext
from types import SimpleNamespace
from typing import Any, Dict, Iterator, List, Optional, Sequence, Tuple, Union

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


class CausalLMOutput:
    """``forward()`` result: ``.loss`` (fp32 scalar or None), ``.logits`` (fp32 [B,T,V]), ``.past_key_values`` (always None).
    Like HF's ModelOutput it also indexes by key (``out["logits"]``) and by position over the set fields (``out[0]``)."""

    def __init__(self, loss: Optional[torch.Tensor], logits: torch.Tensor):
        self.loss, self.logits, self.past_key_values = loss, logits, None

    def to_tuple(self) -> tuple:
        return tuple(v for v in (self.loss, self.logits) if v is not None)

    def __getitem__(self, key):
        return getattr(self, key) if isinstance(key, str) else self.to_tuple()[key]

    def __iter__(self):
        return iter(self.to_tuple())

    def __len__(self) -> int:
        return len(self.to_tuple())


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


class _Processors(SimpleNamespace):
    """What a generate call's processor kwargs became: ``bad_token`` / ``bs_token`` for the sampler's single-id fields,
    ``proc`` (``Engine.set_processors`` keywords, None when nothing beyond those two ids is asked for) and ``eos_min``
    (EOS is banned while a sequence is shorter than ``eos_min(prompt_len)``)."""

    def eos_min(self, prompt_len: int) -> int:
        return prompt_len + self.min_new_tokens if self.min_new_tokens is not None else self.min_length


def _id_list(name: str, value, V: int) -> List[int]:
    vals = [value] if isinstance(value, int) else list(value)
    out = []
    for v in vals:
        if isinstance(v, bool) or not isinstance(v, int) or not 0 <= v < V:
            raise ValueError(f"`{name}` must hold token ids in [0, {V}), got {v!r}")
        out.append(int(v))
    return out


def _int_arg(name: str, value) -> Optional[int]:
    if value is None:
        return None
    if isinstance(value, bool) or not isinstance(value, int) or value < 0:
        raise ValueError(f"`{name}` has to be a non-negative integer, but is {value!r}")
    return int(value)


class _KVSlot:
    """One engine KV slot owned by generate(): the token history whose keys/values it holds, and an LRU tick."""
    __slots__ = ("slot", "tokens", "tick")

    def __init__(self, slot: int):
        self.slot, self.tokens, self.tick = slot, [], 0


class _Requests:
    """Per-sequence host state of a generation call: each request's ids (an int64 [1, limit] CPU buffer, allocated when the
    request starts), streamers, stopping criteria and limits, and the rule by which a new token is accepted and a sequence
    stops. Criteria see a [1, T] view of the buffer; streamers get the prompt as [1, T0] and every new token as [1]."""

    def __init__(self, prompts: List[List[int]], streamers, criteria: List[StoppingCriteriaList], limits: List[int], eos: int):
        self.prompts, self.streamers, self.crits, self.limits, self.eos = prompts, streamers, criteria, limits, eos
        self.bufs: List[Optional[torch.Tensor]] = [None] * len(prompts)
        self.lens = [len(p) for p in prompts]
        self.done = [len(p) >= lim for p, lim in zip(prompts, limits)]   # prompt already at max_length: nothing appended

    def start(self, i: int):
        p = self.prompts[i]
        self.bufs[i] = torch.empty(1, max(self.limits[i], len(p)), dtype=torch.int64)
        self.bufs[i][0, : len(p)] = torch.tensor(p, dtype=torch.int64)
        if self.streamers[i] is not None:
            self.streamers[i].put(self.ids(i))

    def ids(self, i: int) -> torch.Tensor:
        return self.bufs[i][:, : self.lens[i]]

    def accept(self, i: int, tok: int):
        n = self.lens[i]
        self.bufs[i][0, n] = tok
        self.lens[i] = n + 1
        if self.streamers[i] is not None:
            self.streamers[i].put(self.bufs[i][0, n: n + 1])
        crit = self.crits[i]
        self.done[i] = tok == self.eos or n + 1 >= self.limits[i] or (bool(crit) and crit(self.ids(i), None))

    def end(self, i: int):
        if self.streamers[i] is not None:
            self.streamers[i].end()


class _DecodeLoop:
    """The host side of one fused generation loop over the requests ``rq``, for ``generate`` (one row), ``generate_batch``
    (N rows) and ``generate_many`` (a queue). ``run(wave, logits)`` draws the first tokens of the requests ``wave``, whose
    prompts ``slots`` hold and end in ``logits``, begins the loop and keeps two steps in flight until every row has stopped.
    With a ``queue`` a stopped row is retired (slot freed, then ``release(i)``), the next request admitted into it
    (``prefill(i, slot)`` -> its logits) and ``run`` yields the requests completed since its last yield; without one,
    finished rows decode on unread. ``per_row_attn`` turns the shared-prefix cascade off while the loop runs. Every exit
    ends the loop and restores the cascade option and processors. ``launched``: steps launched so far."""

    def __init__(self, model: "DetikzifyForCausalLM", rq: _Requests, g: SimpleNamespace, seed: Optional[int],
                 slots: Dict[int, int], queue: Optional[deque] = None, prefill=None, release=None,
                 per_row_attn: bool = False):
        self.model, self.rq, self.g, self.seed, self.slots = model, rq, g, seed, slots
        self.queue, self.prefill, self.release, self.per_row_attn = queue, prefill, release, per_row_attn
        self.launched = 0

    def run(self, wave: List[int], logits: List[torch.Tensor]) -> Iterator[List[int]]:
        eng, rq, procs, queue = self.model.engine, self.rq, self.g.procs, self.queue
        params = self.model._sampling_params(self.g, self.seed)
        rows: List[Optional[int]] = list(wave)   # occupant of each loop row (None = retired)
        s0 = [0] * len(wave)                      # step from which the ring's entry of a row belongs to its occupant
        pending: List[int] = []                   # rows admitted since the last step launch: first token not read yet
        finished: List[int] = []
        begun, cascade = False, None
        try:
            eos_min = [procs.eos_min(len(rq.prompts[i])) for i in wave]
            if procs.proc is not None:
                eng.set_processors(procs.proc, [rq.prompts[i] for i in wave], eos_min)
            first, _ = eng.sample(torch.stack(logits), params, suppress=[1] * len(wave), steps=[0] * len(wave),
                                  seq_ids=wave)
            toks = [int(t) for t in first.tolist()]
            for i, t in zip(wave, toks):
                if not rq.done[i]:
                    rq.accept(i, t)
            # steps the admitted sequences can use at most (a sequence admitted at step s0 takes its last token from step
            # s0 + limit - len(prompt) - 2); no step is launched beyond the longest of them
            cap = max(rq.limits[i] - len(rq.prompts[i]) for i in wave) - 1
            if (not all(rq.done[i] for i in wave) and cap > 0) or queue:
                if procs.proc is not None:   # device histories continue from prompt + first token (at most max_len ids)
                    eng.set_processors(procs.proc, [(rq.prompts[i] + [t])[:eng.max_len] for i, t in zip(wave, toks)],
                                       eos_min)
                if self.per_row_attn:
                    cascade = eng.get_option("cascade_attn")
                    eng.set_option("cascade_attn", 0)
                eng.gen_begin([self.slots[i] for i in wave], [len(rq.prompts[i]) for i in wave], toks, params, wave)
                begun = True
            waited = 0
            while True:
                if queue is not None:
                    for r, i in enumerate(rows):
                        if i is not None and rq.done[i]:
                            if begun:
                                eng.gen_retire(r)
                            rows[r] = None
                            self._stop(i, finished)
                    # admissions into free rows; a prompt already at its limit completes without one
                    for r in range(len(rows)):
                        while rows[r] is None and queue:
                            i = queue[0]
                            if rq.done[i]:
                                queue.popleft()
                                rq.start(i)
                                self._stop(i, finished)
                                continue
                            try:
                                slot = eng.seq_alloc()
                            except Exception:
                                if any(o is not None for o in rows):
                                    break               # wait for a slot to be released
                                raise
                            queue.popleft()
                            self.slots[i] = slot
                            rq.start(i)
                            lg = self.prefill(i, slot)
                            p = rq.prompts[i]
                            eng.gen_admit(r, slot, len(p), lg, i, p if procs.proc is not None else None,
                                          procs.eos_min(len(p)))
                            rows[r], s0[r] = i, self.launched
                            cap = max(cap, self.launched + rq.limits[i] - len(p) - 1)
                            pending.append(r)
                    if finished:
                        out, finished = finished, []
                        yield out
                if all(i is None or rq.done[i] for i in rows):
                    break
                while self.launched < waited + 2 and self.launched < cap:
                    eng.gen_step()
                    self.launched += 1
                for r in pending:                    # the admission kernels ran before the steps just launched
                    rq.accept(rows[r], eng.gen_first(r))
                pending = []
                if not any(i is not None and not rq.done[i] for i in rows):
                    continue
                row = eng.gen_wait(waited)
                for r, i in enumerate(rows):
                    if i is not None and waited >= s0[r] and not rq.done[i]:
                        rq.accept(i, int(row[r]))
                waited += 1
        finally:
            if begun:
                eng.gen_end()
            if cascade is not None:
                eng.set_option("cascade_attn", cascade)
            if procs.proc is not None:
                eng.set_processors(None)
        for i in rows:
            if i is not None:
                rq.end(i)

    def _stop(self, i: int, finished: List[int]):
        """request i is complete: release its slot (and what the caller keeps for it) and queue it for the next yield"""
        if i in self.slots:
            self.model.engine.seq_free(self.slots.pop(i))
        self.release(i)
        self.rq.end(i)
        finished.append(i)


class DetikzifyForCausalLM:
    def __init__(self, config: DetikzifyConfig, arena: Optional[torch.Tensor] = None, device=0, dtype=torch.bfloat16,
                 max_seqs: int = 2, max_batch: int = 1, max_len: Optional[int] = None, engine=None,
                 prefix_slots: Optional[int] = None, decode_pack: bool = False):
        self.config = config
        self.dtype = dtype
        self.name_or_path = config.name_or_path
        # ``engine`` injection exists for host-logic tests (a scripted engine on CPU); the product path always
        # builds the CUDA engine and raises if no device / library is available.
        self.engine = engine if engine is not None else Engine(config, arena, device=device, max_seqs=max_seqs,
                                                                max_batch=max_batch, max_len=max_len)
        self.device = self.engine.device
        # decode_pack: batch-1 decode streams the weights as lossless 13-bit packed tiles (same logits, fewer bytes per token)
        if decode_pack and engine is None and self.engine.get_option("decode_persistent"):
            self.engine.set_option("decode_pack", 1)
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

    def _processors(self, bad_words_ids, begin_suppress_tokens, kw: Dict[str, Any], eos: int, sampling: bool) -> _Processors:
        """The HF logits-processor kwargs of a generate call (HF generation/utils.py::_get_logits_processor), validated as HF
        validates them, each falling back to the ``generation_config`` attribute of the same name. A call that asks for at
        most one bad id and one begin-suppress id keeps the sampler's single-id fields (the reference's own call,
        infer/generate.py:218-227); anything more runs the sampler's processor tables."""
        gc, V = self.generation_config, self.config.vocab_size

        def arg(name, value=None):
            return getattr(gc, name, None) if value is None else value
        penalty = arg("repetition_penalty", kw.get("repetition_penalty"))
        if penalty is not None and (isinstance(penalty, bool) or not isinstance(penalty, (int, float)) or not penalty > 0):
            raise ValueError(f"`repetition_penalty` has to be a strictly positive float, but is {penalty!r}")
        ngram = _int_arg("no_repeat_ngram_size", arg("no_repeat_ngram_size", kw.get("no_repeat_ngram_size"))) or 0
        min_length = _int_arg("min_length", arg("min_length", kw.get("min_length"))) or 0
        min_new = _int_arg("min_new_tokens", arg("min_new_tokens", kw.get("min_new_tokens")))
        min_p = arg("min_p", kw.get("min_p"))
        if min_p is not None and (isinstance(min_p, bool) or not isinstance(min_p, (int, float)) or not 0 <= min_p <= 1):
            raise ValueError(f"`min_p` has to be a float in [0, 1], but is {min_p!r}")
        bad = arg("bad_words_ids", bad_words_ids)
        words: List[List[int]] = []
        if bad is not None:
            if not isinstance(bad, (list, tuple)) or any(not isinstance(w, (list, tuple)) or not w for w in bad):
                raise ValueError(f"`bad_words_ids` has to be a list of non-empty lists of token ids, but is {bad!r}")
            words = [_id_list("bad_words_ids", w, V) for w in bad]
            words = [w for w in words if w != [eos]]          # NoBadWordsLogitsProcessor drops [eos]
        begin = arg("begin_suppress_tokens", begin_suppress_tokens)
        begin = list(dict.fromkeys(_id_list("begin_suppress_tokens", begin, V))) if begin is not None else []
        suppress = arg("suppress_tokens", kw.get("suppress_tokens"))
        suppress = _id_list("suppress_tokens", suppress, V) if suppress is not None else []
        singles = list(dict.fromkeys(w[0] for w in words if len(w) == 1))
        multi = [w for w in words if len(w) > 1]
        out = _Processors(min_length=min_length, min_new_tokens=min_new, bad_token=-1, bs_token=-1, proc=None)
        active = ((penalty is not None and penalty != 1) or ngram > 0 or multi or len(singles) > 1 or suppress
                  or len(begin) > 1 or min_length > 0 or (min_new is not None and min_new > 0)
                  or (sampling and min_p is not None and min_p > 0))
        if not active:
            out.bad_token = singles[0] if singles else -1
            out.bs_token = begin[0] if begin else -1
            return out
        out.proc = dict(repetition_penalty=float(penalty) if penalty is not None else 1.0, no_repeat_ngram_size=ngram,
                        min_p=float(min_p) if (sampling and min_p is not None) else 0.0, eos_token_id=eos,
                        ban_ids=singles + suppress, begin_ids=begin, words=multi)
        return out

    # ---- prompt helpers shared by generate_batch / forward / score ----------------------------------
    def _image_span(self, ids_host: List[int]) -> Tuple[int, int]:
        """(start, count) of the image-token span of a prompt, (0, 0) without one; splice validation as
        v1/modeling_detikzify.py:176-184."""
        patch = self.config.image_token_id
        n = ids_host.count(patch)
        if n == 0:
            return 0, 0
        if n != self.config.num_patches:
            raise ValueError("The number of image patch tokens should be the same as the number of image patches.")
        st = ids_host.index(patch)
        if ids_host[st: st + n] != [patch] * n:
            raise ValueError("The image patch tokens should be consecutive.")
        return st, n

    def _batch_captions(self, adapter_input_ids, adapter_attention_mask, pixel_values, N: int):
        """TikZero captions of an N-sequence call (one shared or one per sequence) and the pixels to condition: a caption
        without an image runs on the adapter's dummy image."""
        captions = None
        if adapter_input_ids is not None:
            captions = self._captions(adapter_input_ids, adapter_attention_mask)
            if len(captions) not in (1, N):
                raise ValueError("adapter_input_ids must hold one caption (shared) or one caption per sequence")
            if pixel_values is None:
                pixel_values = self.adapter.dummy_pixels()
        return captions, pixel_values

    def _batch_image_embeds(self, pixel_values: Optional[torch.Tensor], captions, N: int) -> Optional[torch.Tensor]:
        """Image embeddings [1 | N, P, H] for one shared image or one image per sequence (None without pixels)."""
        if pixel_values is None:
            return None
        eng = self.engine
        pix = pixel_values.to(self.device, torch.float32)
        if pix.dim() == 3:
            pix = pix[None]
        if pix.shape[0] not in (1, N):
            raise ValueError("pixel_values must hold one image (shared) or one image per sequence")
        if captions is None:
            return eng.image_embeds(pix)
        # one conditioned tower pass per distinct (image, caption) pairing
        if pix.shape[0] != len(captions):
            pix = pix.expand(N, *pix.shape[1:]).contiguous()
            captions = captions * N if len(captions) == 1 else captions
        return eng.image_embeds_cond(pix, [torch.tensor(c) for c in captions])

    def _to_device_ids(self, ids_host: List[int]) -> torch.Tensor:
        t = torch.tensor(ids_host, dtype=torch.int64)
        return t.pin_memory().to(self.device, non_blocking=True) if self.device.type == "cuda" else t

    def _scratch_slot(self) -> Tuple[int, bool]:
        """An engine slot for a call that keeps no KV state: a free one (owned: the caller frees it) or, when none is free,
        the least recently used prefix-cache slot of generate(), whose cached content is forgotten (not owned)."""
        try:
            return self.engine.seq_alloc(), True
        except Exception:
            kv = min(self._kv, key=lambda k: k.tick)
            kv.tokens = []
            return kv.slot, False

    # ---- generation: sampling kwargs, shared-prefix prefill, the three entry points ------------------------------
    def _sampling(self, temperature, top_p, top_k, do_sample, eos_token_id, bad_words_ids, begin_suppress_tokens,
                  kw: Dict[str, Any]) -> SimpleNamespace:
        """The sampling and processor kwargs of a generate call, each falling back to ``generation_config``."""
        gc = self.generation_config
        g = SimpleNamespace(temperature=gc.temperature if temperature is None else temperature,
                            top_p=gc.top_p if top_p is None else top_p, top_k=gc.top_k if top_k is None else top_k,
                            do_sample=gc.do_sample if do_sample is None else do_sample,
                            eos=self.config.eos_token_id if eos_token_id is None else eos_token_id)
        g.procs = self._processors(bad_words_ids, begin_suppress_tokens, kw, g.eos,
                                   bool(g.do_sample) and float(g.temperature) >= 1e-5)
        return g

    def _sampling_params(self, g: SimpleNamespace, seed: Optional[int]):
        """The engine's sampling parameters of one call; without ``seed`` every call draws from a new seed."""
        self._call_counter += 1
        return self.engine.sampling(
            temperature=g.temperature, top_p=g.top_p, top_k=g.top_k or 0, do_sample=bool(g.do_sample),
            bad_token=g.procs.bad_token, begin_suppress_token=g.procs.bs_token,
            seed=(seed if seed is not None else torch.initial_seed() + self._call_counter))

    def _base_prefix(self, prompts: List[List[int]], span: Tuple[int, int], image,
                     lim: Optional[int] = None) -> Tuple[Optional[int], int]:
        """Prefill the longest common token prefix of the prompts of one image once into a new base slot: at most ``lim``
        long (default: one short of the shortest prompt), never splitting prompt 0's image span ``span`` (``image()``: its
        embeddings). Returns (base slot, shared length), or (None, 0) below 16 positions (a shorter shared prefix saves
        less than the sharing costs), for a single prompt, or when no slot is free."""
        eng = self.engine
        if len(prompts) < 2:
            return None, 0
        lim = min(len(p) for p in prompts) - 1 if lim is None else lim
        lcp = 0
        while lcp < lim and all(p[lcp] == prompts[0][lcp] for p in prompts[1:]):
            lcp += 1
        st0, n0 = span
        if n0 and st0 < lcp < st0 + n0:
            lcp = st0
        if lcp < 16:
            return None, 0
        try:
            base = eng.seq_alloc()
        except Exception:       # no spare slot: every sequence prefills its whole prompt
            return None, 0
        try:
            eng.prefill(base, self._to_device_ids(prompts[0][:lcp]), 0, image() if n0 and st0 < lcp else None, st0)
        except BaseException:
            eng.seq_free(base)
            raise
        return base, lcp

    def _prefill_row(self, slot: int, prompt: List[int], base: Optional[int], lcp: int, span: Tuple[int, int],
                     image) -> torch.Tensor:
        """``prompt`` into ``slot``, borrowing its first ``lcp`` positions from ``base``; the last position's logits."""
        st, n = span
        img = image() if n and st >= lcp else None
        if lcp:
            self.engine.seq_share(base, slot, lcp)
        lg, _ = self.engine.prefill(slot, self._to_device_ids(prompt[lcp:]), lcp, img, st)
        return lg

    def _requests(self, prompts: List[List[int]], streamers, stopping_criteria, max_length, max_new_tokens,
                  eos: int) -> _Requests:
        """Per-sequence streamers (one entry or None each), stopping criteria (a callable or list per sequence, or one shared
        entry) and ``max_length`` limits of N prompts."""
        N, gc = len(prompts), self.generation_config
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
            limits.append(min(int(ml), self.engine.max_len))
        return _Requests(prompts, streamers, crits, limits, eos)

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor = None, pixel_values: Optional[torch.Tensor] = None,
                 bad_words_ids=None, begin_suppress_tokens=None, streamer=None, stopping_criteria=None,
                 temperature: Optional[float] = None, top_p: Optional[float] = None, top_k: Optional[int] = None,
                 max_length: Optional[int] = None, max_new_tokens: Optional[int] = None,
                 do_sample: Optional[bool] = None, seed: Optional[int] = None, eos_token_id: Optional[int] = None,
                 adapter_input_ids=None, adapter_attention_mask=None, **ignored) -> torch.Tensor:
        cfg = self.config
        caption = None
        if adapter_input_ids is not None:
            caps = self._captions(adapter_input_ids, adapter_attention_mask)
            if len(caps) != 1:
                raise ValueError("generate() is batch-1: pass one caption")
            caption = caps[0]
            if pixel_values is None:
                pixel_values = self.adapter.dummy_pixels()
        g = self._sampling(temperature, top_p, top_k, do_sample, eos_token_id, bad_words_ids, begin_suppress_tokens, ignored)

        ids2d = input_ids if input_ids.dim() == 2 else input_ids[None]
        if ids2d.shape[0] != 1:
            raise ValueError("generate() is batch-1 (use generate_batch for parallel rollouts)")
        ids_host: List[int] = ids2d[0].tolist()
        T0 = len(ids_host)
        rq = self._requests([ids_host], [streamer], stopping_criteria, max_length, max_new_tokens, g.eos)

        with self._lock, self._on_stream():
            # -- splice validation (v1/modeling_detikzify.py:176-184)
            img = None
            img_start, n_patch = self._image_span(ids_host) if pixel_values is not None else (0, 0)
            if n_patch:
                img = self._image_embeds(pixel_values, caption)
            elif pixel_values is None and cfg.image_token_id in ids_host:
                # patch tokens without an image: their KV comes from plain embeddings. Forget the image identity too, so a
                # later call WITH the same image re-validates nothing against these slots (ADVICE r1)
                self._img_cache = None
                self._slot_tokens = []
            if T0 == 0:
                raise ValueError("empty prompt")
            rq.start(0)
            if rq.done[0]:
                rq.end(0)
                return ids2d.to(self.device)

            # -- longest common prefix with the KV already held by one of the cache slots
            L = self._pick_slot(ids_host, img_start, n_patch)
            self._slot_tokens = list(ids_host[:L])     # if the prefill raises, the slot only claims what it held before
            last_logits, _ = self.engine.prefill(self._slot, self._to_device_ids(ids_host[L:]), L, img, img_start)
            self._slot_tokens = list(ids_host)

            loop = _DecodeLoop(self, rq, g, seed, {0: self._slot})
            try:
                list(loop.run([0], [last_logits]))
            finally:
                # decode step s wrote KV at T0+s for new token s; only tokens the host has seen count
                self._slot_tokens = ids_host + rq.ids(0)[0, T0: T0 + loop.launched].tolist()
            result = rq.ids(0).to(self.device)
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
        eng = self.engine
        g = self._sampling(temperature, top_p, top_k, do_sample, eos_token_id, bad_words_ids, begin_suppress_tokens, ignored)
        prompts: List[List[int]] = [(p[0] if p.dim() == 2 else p).tolist() for p in input_ids]
        N = len(prompts)
        if N == 0:
            return []
        captions, pixel_values = self._batch_captions(adapter_input_ids, adapter_attention_mask, pixel_values, N)
        if any(len(p) == 0 for p in prompts):
            raise ValueError("empty prompt")
        rq = self._requests(prompts, streamers, stopping_criteria, max_length, max_new_tokens, g.eos)
        with self._lock, self._on_stream():
            imgs = self._batch_image_embeds(pixel_values, captions, N)
            spans = [self._image_span(p) if imgs is not None else (0, 0) for p in prompts]
            image = [lambda i=i: imgs[i if imgs.shape[0] == N else 0] for i in range(N)]
            slots: Dict[int, int] = {}
            base, lcp = None, 0
            try:
                for i in range(N):
                    rq.start(i)
                for i in range(N):
                    slots[i] = eng.seq_alloc()
                # one shared image: its prompts' longest common prefix is prefilled once (never splitting an image span)
                if share_prefix and (imgs is None or imgs.shape[0] == 1):
                    base, lcp = self._base_prefix(prompts, spans[0], image[0])
                last = [self._prefill_row(slots[i], prompts[i], base, lcp, spans[i], image[i])
                        for i in range(N)]
                list(_DecodeLoop(self, rq, g, seed, slots).run(list(range(N)), last))
                result = [rq.ids(i)[0].to(self.device) for i in range(N)]
                self._sync()
                return result
            finally:
                for s in slots.values():
                    eng.seq_free(s)
                if base is not None:
                    eng.seq_free(base)

    # ---- continuous batching (extension): a stream of requests through one running decode loop ---------
    def generate_many(self, prompts: Sequence[torch.Tensor], pixel_values: Optional[torch.Tensor] = None, *,
                      figure: Optional[Sequence[int]] = None, batch_size: Optional[int] = None, bad_words_ids=None,
                      begin_suppress_tokens=None, temperature: Optional[float] = None, top_p: Optional[float] = None,
                      top_k: Optional[int] = None, max_length: Optional[int] = None, max_new_tokens: Optional[int] = None,
                      do_sample: Optional[bool] = None, seed: Optional[int] = None, eos_token_id: Optional[int] = None,
                      streamers: Optional[Sequence[Any]] = None, stopping_criteria: Optional[Sequence[Any]] = None,
                      adapter_input_ids=None, adapter_attention_mask=None, **ignored) -> Iterator[Tuple[int, torch.Tensor]]:
        """Any number of independent sequences through ONE batched decode loop of at most ``batch_size`` rows (default and
        upper bound: the engine's ``max_batch``; at least 2): when a sequence stops, its row is retired and the next queued
        prompt is admitted into it while the loop runs on, so rows stay busy however much the programs' lengths vary.
        Yields ``(index, ids)`` (ids: CPU int64 [T], prompt included) in completion order.

        ``pixel_values`` [F,3,S,S] holds F figures and ``figure[i]`` names prompt i's (default: all share figure 0 when
        F = 1, prompt i has figure i when F = N). The vision tower runs in batches of figures ahead of admission. Each
        figure's longest common prompt prefix (``generate_batch``'s rule) is prefilled once into a base slot, lent to that
        figure's sequences and freed after its last one stops; the loop uses shared-prefix (cascade) attention only when
        every sequence borrows one prefix (one figure).

        Per-sequence contract as ``generate_batch``: streamers, stopping criteria, EOS, ``max_length`` and RNG stream i of
        ``seed`` for sequence i, so a sequence's tokens do not depend on when it was admitted; with one figure whose prompts
        share the prefix the first ``batch_size`` share (e.g. samples of one prompt), those first ``batch_size`` sequences
        equal ``generate_batch`` of their prompts. The model is busy until the generator is
        exhausted or closed; slots and processors are released on every exit. TikZero captions are not supported."""
        if adapter_input_ids is not None:
            raise ValueError("generate_many() does not take TikZero captions (adapter_input_ids)")
        eng = self.engine
        B = eng.max_batch if batch_size is None else int(batch_size)
        if not 2 <= B <= eng.max_batch:
            raise ValueError(f"batch_size must lie in [2, max_batch = {eng.max_batch}], got {batch_size!r}")
        g = self._sampling(temperature, top_p, top_k, do_sample, eos_token_id, bad_words_ids, begin_suppress_tokens, ignored)
        ids: List[List[int]] = [torch.as_tensor(p).reshape(-1).tolist() for p in prompts]
        N = len(ids)
        if any(len(p) == 0 for p in ids):
            raise ValueError("empty prompt")
        pix = None
        if pixel_values is not None:
            pix = pixel_values if pixel_values.dim() == 4 else pixel_values[None]
        F = pix.shape[0] if pix is not None else 1
        if figure is None:
            if F not in (1, N):
                raise ValueError("pixel_values must hold one figure (shared) or one per prompt, or pass `figure`")
            figure = [0] * N if F == 1 else list(range(N))
        figure = [int(f) for f in figure]
        if len(figure) != N or any(not 0 <= f < F for f in figure):
            raise ValueError(f"figure must hold one index in [0, {F}) per prompt")
        rq = self._requests(ids, streamers, stopping_criteria, max_length, max_new_tokens, g.eos)
        return self._many(ids, pix, figure, B, g, seed, rq)

    def _many(self, prompts: List[List[int]], pix: Optional[torch.Tensor], figure: List[int], B: int, g: SimpleNamespace,
              seed: Optional[int], rq: _Requests) -> Iterator[Tuple[int, torch.Tensor]]:
        eng, N = self.engine, len(prompts)
        spans = [self._image_span(p) if pix is not None else (0, 0) for p in prompts]
        members: Dict[int, List[int]] = {}
        for i, f in enumerate(figure):
            members.setdefault(f, []).append(i)
        left = {f: len(m) for f, m in members.items()}    # sequences of the figure that have not stopped
        bases: Dict[int, Tuple[Optional[int], int]] = {}   # figure -> (base slot, shared length) once its first one is admitted
        embeds: Dict[int, torch.Tensor] = {}
        queue = deque(range(N))
        slot_of: Dict[int, int] = {}

        def figure_embeds(f: int) -> torch.Tensor:
            if f not in embeds:                                # the tower runs for the next figures in queue order
                todo = [f] + [h for h in dict.fromkeys(figure[i] for i in queue) if h != f and h not in embeds]
                todo = todo[:8]
                out = eng.image_embeds(pix[todo].to(self.device, torch.float32))
                for k, h in enumerate(todo):
                    embeds[h] = out[k]
            return embeds[f]

        def prefill(i: int, slot: int) -> torch.Tensor:
            """prompt i into its slot after its figure's shared prefix; the last position's logits"""
            f = figure[i]
            if f not in bases:
                bases[f] = self._base_prefix([prompts[j] for j in members[f]], spans[members[f][0]],
                                             lambda: figure_embeds(f))
            base, lcp = bases[f]
            return self._prefill_row(slot, prompts[i], base, lcp, spans[i], lambda: figure_embeds(f))

        def release(i: int):
            """after the figure's last sequence: its base slot and embeddings"""
            f = figure[i]
            left[f] -= 1
            if left[f] == 0:
                base, _ = bases.pop(f, (None, 0))
                if base is not None:
                    eng.seq_free(base)
                embeds.pop(f, None)

        self._lock.acquire()
        ctx = self._on_stream()
        ctx.__enter__()
        run = None
        try:
            # ---- first wave: exactly generate_batch's calls for the first batch_size prompts
            wave = [queue.popleft() for _ in range(min(B, N))]
            if pix is not None:
                for f in dict.fromkeys(figure[i] for i in wave):
                    figure_embeds(f)
            for i in wave:
                rq.start(i)
            for i in wave:
                slot_of[i] = eng.seq_alloc()
            last = [prefill(i, slot_of[i]) for i in wave]
            # one shared prefix per figure: per-row reads only
            loop = _DecodeLoop(self, rq, g, seed, slot_of, queue, prefill, release, per_row_attn=len(members) > 1)
            run = loop.run(wave, last)
            for done in run:
                ctx.__exit__(None, None, None)
                try:
                    yield from ((i, rq.ids(i)[0].clone()) for i in done)
                finally:
                    ctx = self._on_stream()
                    ctx.__enter__()
        finally:
            try:
                if run is not None:
                    run.close()      # the loop ends before the slots it reads are freed
                for slot in slot_of.values():
                    eng.seq_free(slot)
                for base, _ in bases.values():
                    if base is not None:
                        eng.seq_free(base)
            finally:
                ctx.__exit__(None, None, None)
                self._lock.release()

    # ---- logits, loss and sequence scoring ---------------------------------------------------------
    def __call__(self, *args, **kwargs):
        return self.forward(*args, **kwargs)

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor = None, pixel_values: Optional[torch.Tensor] = None,
                attention_mask: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                adapter_input_ids=None, adapter_attention_mask=None, logits_to_keep=None, return_dict: Optional[bool] = None,
                **ignored) -> Union[CausalLMOutput, tuple]:
        """The reference's ``forward`` (v1/modeling_detikzify.py:218-283, modeling_detikzify.py:320-389): fp32 logits
        [B,T,V] for every position and, with ``labels``, the mean cross-entropy of the shifted labels (``-100`` ignored; v2
        checkpoints with an ``attention_mask`` count only shifted positions whose mask is set). No gradients, no KV state.

        Each row runs unpadded through one engine call that writes its logits into the output and the log-probs of its
        shifted labels (fused lm_head log-softmax, no cross-entropy over the logits). ``attention_mask`` must be one
        contiguous run of ones per row (left or right padding); logits at masked positions are 0, where HF returns
        whatever the padded rows compute. RoPE sees only relative positions, so the logits match HF's up to rounding.
        ``logits_to_keep`` is accepted and ignored, as the reference does; ``use_cache`` is ignored."""
        for key in ("inputs_embeds", "past_key_values"):
            if ignored.get(key) is not None:
                raise ValueError(f"forward() does not take `{key}`: it runs whole sequences from input_ids and keeps no KV cache")
        for key in ("output_attentions", "output_hidden_states"):
            if ignored.get(key):
                raise ValueError(f"forward() does not return {key[len('output_'):]}")
        cfg, eng, V = self.config, self.engine, self.config.vocab_size
        ids = torch.as_tensor(input_ids).cpu()
        ids = ids[None] if ids.dim() == 1 else ids
        B, T = ids.shape
        if T == 0:
            raise ValueError("empty input_ids")
        if T > eng.max_len:
            raise ValueError(f"sequence length {T} exceeds the engine's max_len {eng.max_len}")
        mask = None if attention_mask is None else torch.as_tensor(attention_mask).cpu().reshape(B, T) != 0
        runs = []
        for b in range(B):
            if mask is None:
                runs.append((0, T))
                continue
            on = mask[b].nonzero().view(-1)
            if on.numel() == 0 or int(on[-1]) - int(on[0]) + 1 != on.numel():
                raise ValueError("attention_mask must hold one contiguous run of ones per row (left or right padding)")
            runs.append((int(on[0]), int(on[-1]) + 1))
        # targets of row t: the label of position t + 1 where the reference's loss counts it, else -1
        targets = torch.full((B, T), -1, dtype=torch.int64)
        count = 0
        if labels is not None:
            sh = torch.as_tensor(labels).cpu().reshape(B, T)[:, 1:].to(torch.int64)
            use = sh != -100
            if not cfg.projector_bias and mask is not None:   # v2: attention_mask[:, 1:] != 0 selects the counted positions
                use &= mask[:, 1:]
            if mask is not None and (use & ~mask[:, :-1]).any():
                raise ValueError("a counted label is predicted from a masked position (set it to -100)")
            if (use & ((sh < 0) | (sh >= V))).any():
                raise ValueError(f"labels must be -100 or in [0, {V})")
            targets[:, :-1] = torch.where(use, sh, torch.full_like(sh, -1))
            count = int(use.sum())
        rows = [ids[b, a:e].tolist() for b, (a, e) in enumerate(runs)]
        captions, pixel_values = self._batch_captions(adapter_input_ids, adapter_attention_mask, pixel_values, B)
        spans = [self._image_span(r) if pixel_values is not None else (0, 0) for r in rows]

        with self._lock, self._on_stream():
            imgs = self._batch_image_embeds(pixel_values, captions, B) if any(n for _, n in spans) else None
            logits = torch.zeros(B, T, V, device=self.device, dtype=torch.float32)
            total = torch.zeros((), device=self.device, dtype=torch.float32)
            slot, owned = self._scratch_slot()
            try:
                for b, (a, e) in enumerate(runs):
                    st, n = spans[b]
                    img = imgs[b if imgs.shape[0] == B else 0] if n else None
                    lp, _, _ = eng.score(slot, self._to_device_ids(rows[b]), 0, img, st, targets[b, a:e].to(self.device),
                                         logits_out=logits[b, a:e])
                    if labels is not None:
                        total += lp.sum()
            finally:
                if owned:
                    eng.seq_free(slot)
            loss = -total / count if labels is not None else None   # 0 / 0 = NaN when nothing is counted, as in torch
            self._sync()
        if return_dict is False:
            return (loss, logits) if loss is not None else (logits,)
        return CausalLMOutput(loss, logits)

    @torch.no_grad()
    def score(self, sequences: Sequence[torch.Tensor], pixel_values: Optional[torch.Tensor] = None, *,
              start: Union[int, Sequence[int]] = 1, adapter_input_ids=None, adapter_attention_mask=None) -> List[torch.Tensor]:
        """Log-likelihood of N id sequences (1-D) under the model, e.g. to rank candidate programs for one figure or to
        measure perplexity. Returns one fp32 device tensor per sequence: entry k of sequence i is
        log p(ids_i[start_i + k] | ids_i[:start_i + k]), for 1 <= start_i < len_i (``start``: one int or one per sequence).
        ``pixel_values``: one shared image or one per sequence, as in ``generate_batch``; TikZero captions likewise.

        The longest common prefix of the sequences (at most min(start_i) positions, never splitting an image span, none
        below 16) is prefilled once into a base slot. Sequence i borrows its first s_i = min(lcp, start_i - 1) positions
        from there and runs only ids_i[s_i : len_i - 1] through the fused lm_head log-softmax, so every scored row is
        computed in its own prefill and no [T, V] logits are materialised. When a sequence's scoring starts right after the
        shared prefix (start_i = lcp, e.g. a program right after the image span of a v1 prompt), it recomputes that one
        last shared row. Uses two engine slots for any N.

        Against ``forward()`` of each sequence alone the log-probs agree to about 1e-3 when a sequence's own prefill
        has at least 64 rows. With fewer rows the decoder GEMMs run on the swapped-operand tile, whose bf16 activations
        round differently, and the difference grows to about 1e-2 over 24 layers (random-init ds-1.3b weights)."""
        seqs: List[List[int]] = [torch.as_tensor(q).reshape(-1).tolist() for q in sequences]
        N = len(seqs)
        if N == 0:
            return []
        starts = [int(start)] * N if isinstance(start, int) else [int(x) for x in start]
        if len(starts) != N:
            raise ValueError("start must be one int or one int per sequence")
        for q, st in zip(seqs, starts):
            if not 1 <= st < len(q):
                raise ValueError(f"start must satisfy 1 <= start < len(sequence) (got {st} for length {len(q)})")
            if len(q) > self.engine.max_len:
                raise ValueError(f"sequence length {len(q)} exceeds the engine's max_len {self.engine.max_len}")
        captions, pixel_values = self._batch_captions(adapter_input_ids, adapter_attention_mask, pixel_values, N)
        eng = self.engine
        with self._lock, self._on_stream():
            imgs = self._batch_image_embeds(pixel_values, captions, N)
            spans = [self._image_span(q) if imgs is not None else (0, 0) for q in seqs]
            work, owned = self._scratch_slot()
            base, lcp = None, 0
            try:
                if imgs is None or imgs.shape[0] == 1:
                    base, lcp = self._base_prefix(seqs, spans[0], lambda: imgs[0], lim=min(starts))
                out = []
                for i, q in enumerate(seqs):
                    s0 = min(lcp, starts[i] - 1)              # positions borrowed from the base slot
                    st, n = spans[i]
                    img = imgs[i if imgs.shape[0] == N else 0] if (imgs is not None and n and st + n > s0) else None
                    if s0:
                        eng.seq_share(base, work, s0)
                    # row r sits at position s0 + r and predicts q[s0 + r + 1]; rows before start_i - 1 are not scored
                    skip = starts[i] - 1 - s0
                    tg = [-1] * skip + q[starts[i]:]
                    lp, _, _ = eng.score(work, self._to_device_ids(q[s0:-1]), s0, img, st, self._to_device_ids(tg))
                    out.append(lp[skip:])
                self._sync()
                return out
            finally:
                if owned:
                    eng.seq_free(work)   # also ends its borrowing from the base slot
                if base is not None:
                    eng.seq_free(base)

    # ---- SelfSim helper: pooled features straight from the engine --------------------------------
    @torch.no_grad()
    def pooled_features(self, pixel_values: torch.Tensor) -> torch.Tensor:
        with self._lock, self._on_stream():
            _, pooled = self.engine.vit_encode(pixel_values, want_tokens=False)
            self._sync()
        return pooled   # fp32, produced and synchronised on the engine stream

    def close(self):
        self.engine.close()
