"""
Sampling + MCTS driver with the reference's public surface (detikzify/infer/generate.py):

    DetikzifyPipeline(model, processor, temperature=0.8, top_p=0.95, top_k=0, compile_timeout=60,
                      metric="model"|"fast"|Metric, **gen_kwargs)
        .sample(image, text=None, preprocess=True, **gen_kwargs) -> TikzDocument          (:399-426)
        .simulate(image, text=None, preprocess=True, expansions=None, timeout=None, **kw)
              -> iterator of (score, TikzDocument)                                         (:428-464)
    DetikzifyGenerator(model, processor, image, text, metric, compile_timeout, mcts_timeout,
                       streamer, control, exploration, strict, **gen_kwargs)               (:145-353)

Search semantics kept from the reference: one expansion = one rollout from the chosen node's token
prefix (same image), a tree node per generated source line, sqrt(n) node thinning, failed-rollout memo
keyed by token prefix, error-line based pruning, min-max normalised SelfSim reward, widen nodes.
The rollout runs ``model.generate`` on a worker thread while the caller consumes a TokenStreamer —
the threading contract of SURVEY.md §8b. What is different underneath: ``model.generate`` is the CUDA
engine (image features cached per figure, KV prefix of the working slot reused, persistent decode
kernel), so an expansion prefills only the tree-path suffix.
"""
from __future__ import annotations

import re
from collections import deque
from dataclasses import dataclass
from functools import cached_property
from math import sqrt
from time import time
from types import SimpleNamespace
from typing import Any, Dict, Generator, List, Optional, Set, Tuple, Union

import torch
from PIL import Image

from ..evaluate.imagesim import ImageSim
from ..mcts import MonteCarlo, Node
from ..util import ExplicitAbort, StreamerList, TokenStreamer, cache_cast, expand, load, unwrap_processor as unwrap
from ..util.generation import StoppingCriteriaList
from .tikz import TikzDocument

Numeric = Union[int, float]


def has_adapter(model) -> bool:
    """reference detikzify/model/adapter/__init__.py:6-7: True once ``detikzify_b200.model.adapter.load`` attached the TikZero
    text-conditioning adapter to the model."""
    return hasattr(model, "adapter")


@dataclass(frozen=True)
class NodeState:
    token_ids: torch.Tensor
    num_lines: int = 0

    def __eq__(self, other: Any) -> bool:
        try:
            return self.token_ids.equal(other.token_ids)
        except (AttributeError, TypeError):
            return False

    def __hash__(self):
        return hash(tuple(self.token_ids.tolist()))


class WideNode(Node):
    """Tree node that always carries a "widen" twin child: selecting the twin re-expands the parent
    (progressive widening), reference :49-81."""
    state: NodeState

    def __init__(self, *args, exploration: float = 0.6, is_widen_node: bool = False, **kwargs):
        super().__init__(NodeState(*args, **kwargs))
        self.discovery_factor = exploration
        self.is_widen_node = is_widen_node
        self.update_policy_value(1.0)
        if not is_widen_node:
            self.add_child(WideNode(*args, exploration=exploration, is_widen_node=True, **kwargs))

    def add_child(self, child):
        self.expanded = self.expanded or not child.is_widen_node
        super().add_child(child)

    @property
    def depth(self) -> int:
        d, cur = 0, self
        while cur.parent is not None:
            d, cur = d + 1, cur.parent
        return d

    @property
    def token_ids(self):
        return self.state.token_ids

    @property
    def num_lines(self):
        return self.state.num_lines


class DynMinMaxNorm:
    """Scores are min-max normalised against every score seen so far, lazily (the normalisation of a
    stored value changes as new extremes arrive), reference :84-142."""

    def __init__(self, default_value: Numeric = 0):
        self.scores: Set[Numeric] = set()
        self.default_value = default_value

    def normalize(self, score: Numeric) -> "DynMinMaxNorm.MinMaxScore":
        self.scores.add(score)
        return self.MinMaxScore(score, all_scores=self.scores, default_value=self.default_value)

    __call__ = normalize

    class MinMaxScore:
        def __init__(self, *scores: Numeric, all_scores: Set[Numeric], default_value: Numeric, no_minmax_scores=()):
            self.scores = list(scores)
            self.all_scores = all_scores
            self.default_value = default_value
            self.no_minmax_scores = list(no_minmax_scores)

        @property
        def score(self) -> Numeric:
            lo, hi = min(self.all_scores), max(self.all_scores)
            if hi == lo:
                total = self.default_value
            else:
                total = sum((s - lo) / (hi - lo) for s in self.scores)
            return total + sum(self.no_minmax_scores)

        def __add__(self, other):
            new = self.__class__(*self.scores, all_scores=self.all_scores, default_value=self.default_value,
                                 no_minmax_scores=self.no_minmax_scores)
            if isinstance(other, DynMinMaxNorm.MinMaxScore):
                new.scores.extend(other.scores)
                new.no_minmax_scores.extend(other.no_minmax_scores)
            else:
                new.no_minmax_scores.append(other)
            return new

        def __mul__(self, other):
            return self.score * other

        def __truediv__(self, other):
            return self.score / other

        def __rtruediv__(self, other):
            return other / self.score

        __radd__, __rmul__ = __add__, __mul__


class LineTracker:
    """Per-sequence observer of one rollout, run by ``model.generate_batch`` as that sequence's stopping criterion (called
    with the ids so far after every new token). It cuts the token stream into source lines — one candidate tree node per
    completed line, as the reference's ``rollout`` generator yields them (detikzify/infer/generate.py:246-282) — and stops
    its sequence as soon as the prefix is one that is already known to fail (``failed_rollouts`` memo, :318-323) or the
    shared abort flag is raised. Unlike the reference's streamer + worker-thread construction this needs no thread per
    rollout, which is what lets K rollouts advance in one lock-step batch."""

    def __init__(self, start: NodeState, newlineinfo: Dict[int, Any], failed: Dict[NodeState, List["WideNode"]],
                 control: ExplicitAbort, exploration: float):
        self.prefix: List[int] = start.token_ids.tolist()
        self.device = start.token_ids.device
        self.num_lines, self.continuation = start.num_lines, False
        self.newlineinfo, self.failed, self.control, self.exploration = newlineinfo, failed, control, exploration
        self.line: List[int] = []
        self.nodes: List[WideNode] = []
        self.memo_hit = False

    def _node(self, num_lines: int) -> "WideNode":
        self.prefix.extend(self.line)
        self.line.clear()
        return WideNode(torch.tensor(self.prefix, device=self.device), num_lines, exploration=self.exploration)

    def __call__(self, input_ids, scores=None, **_) -> bool:
        token = int(input_ids[0, -1])
        self.line.append(token)
        info = self.newlineinfo.get(token)
        if info:
            self.num_lines += info.num_lines - self.continuation
            self.continuation = not info.trailing
            cand = self._node(self.num_lines)
            known = self.failed.get(cand.state)
            if known is not None:          # this prefix ran into a compile error before: reuse its continuation
                self.nodes.extend(known)
                self.memo_hit = True
                return True
            self.nodes.append(cand)
        return self.control.should_stop

    def finish(self) -> List["WideNode"]:
        if self.line and not self.memo_hit:   # trailing text without a newline
            self.nodes.append(self._node(self.num_lines - self.continuation))
        return self.nodes


class DetikzifyGenerator:
    """MCTS over TikZ source lines with the reference's search semantics (detikzify/infer/generate.py:145-353) — one
    expansion = one rollout from the chosen node's token prefix, a tree node per generated line, sqrt(n) node thinning,
    failed-rollout memo keyed by token prefix, error-line pruning, min-max normalised SelfSim reward, widen nodes — but
    organised around BATCHED expansions: ``rollouts`` leaves are selected per step (virtual visits keep the selections
    apart), rolled out together by ``model.generate_batch`` (one weight stream per decode step for all of them, the image
    span + common tree path prefilled once and shared), compiled, scored in one ViT batch and back-propagated.
    ``rollouts=1`` reproduces the reference's one-rollout-per-expansion schedule."""

    def __init__(self, model, processor, image: Optional[Image.Image], text: Optional[str] = None, metric=None,
                 compile_timeout: Optional[int] = 60, mcts_timeout: Optional[int] = None, streamer=None,
                 control: Optional[ExplicitAbort] = None, exploration: float = 0.6, strict: bool = False,
                 rollouts: int = 1, **gen_kwargs):
        self.model, self.processor = model, processor
        self.metric, self.image, self.text = metric, image, text
        self.compile_timeout, self.mcts_timeout = compile_timeout, mcts_timeout
        self.streamer, self.exploration, self.strict = streamer, exploration, strict
        self.rollouts = max(1, int(rollouts))
        self.gen_kwargs = gen_kwargs
        self.solution: deque = deque()
        self.failed_rollouts: Dict[NodeState, List[WideNode]] = dict()
        self.norm = DynMinMaxNorm()
        self.control = control or ExplicitAbort()
        enc = processor(images=self.image, text=self.text, text_kwargs={"truncation": True}, return_tensors="pt")
        self.pixel_values = enc.get("pixel_values")       # preprocessed once per figure (the reference re-runs it per rollout)
        # caption of a TikZero adapter (reference infer/generate.py:209-227 forwards the adapter_* keys to every generate call)
        self.adapter_kwargs = {k: enc[k] for k in ("adapter_input_ids", "adapter_attention_mask") if k in enc}
        root_ids = enc.input_ids.to(model.device).squeeze()
        self.montecarlo = MonteCarlo(root_node=WideNode(root_ids, exploration=self.exploration))
        self.montecarlo.child_finder = self.child_finder
        self.decode = cache_cast(lambda token_ids: tuple(token_ids.tolist()))(self.decode)
        self.score = cache_cast(lambda image: image.tobytes())(self.score)

    def __call__(self, *args, **kwargs):
        return self.simulate(*args, **kwargs)

    # ---- public driver --------------------------------------------------------------------------------------------
    def simulate(self, expansions: Optional[Numeric] = 1) -> Generator[Tuple[Numeric, TikzDocument], None, None]:
        """Yield every rollout (successful or not) as (score, document); reference :197-207. ``expansions`` counts
        rollouts; with ``rollouts = K`` they are produced K at a time."""
        start = time()
        remaining = expansions
        while remaining is None or remaining > 0:
            k = self.rollouts if remaining is None else int(min(self.rollouts, remaining))
            self.expand_batch(k)
            while self.solution:
                yield self.solution.popleft()
            if remaining is not None:
                remaining -= k
            if self.mcts_timeout is not None and time() - start > self.mcts_timeout:
                return

    def sample(self):
        return self.decode(self.generate(input_ids=self.montecarlo.root_node.token_ids))

    def generate(self, input_ids: torch.Tensor, streamer=None, **gen_kwargs) -> torch.Tensor:
        """One batch-1 ``model.generate`` call continuing ``input_ids`` (reference :209-227)."""
        streamers = StreamerList(filter(bool, [streamer, self.streamer]))
        numel = input_ids.numel()
        if self._exhausted(input_ids, gen_kwargs):
            streamers.end()
            return input_ids  # never continue past EOS / the length budget
        with torch.inference_mode():
            return self.model.generate(
                input_ids=input_ids.unsqueeze(0),
                bad_words_ids=[[self.model.config.image_token_id]],
                begin_suppress_tokens=[self.model.config.text_config.eos_token_id],
                pixel_values=self.pixel_values,
                streamer=streamers,
                **self.adapter_kwargs,
                **self.gen_kwargs,
                **gen_kwargs,
            ).squeeze()

    def _exhausted(self, input_ids: torch.Tensor, gen_kwargs=None) -> bool:
        max_length = {**self.model.generation_config.to_dict(), **self.gen_kwargs, **(gen_kwargs or {})}["max_length"]
        numel = input_ids.numel()
        return bool((numel and input_ids[-1] == unwrap(self.processor).tokenizer.eos_token_id) or numel >= max_length)

    @cached_property
    def newlineinfo(self):
        """token id -> (number of newlines it contains, ends with newline?)  (reference :229-244)."""
        info = dict()
        for token_id in unwrap(self.processor).tokenizer.vocab.values():
            token = re.sub(r"\r\n|\r", r"\n", self.processor.decode([token_id]))
            if n := token.count("\n"):
                info[token_id] = SimpleNamespace(num_lines=n, trailing=token.endswith("\n"))
        assert info
        return info

    def decode(self, token_ids: torch.Tensor) -> TikzDocument:
        return TikzDocument(
            timeout=self.compile_timeout,
            code=self.processor.decode(token_ids=token_ids[len(self.montecarlo.root_node.token_ids):], skip_special_tokens=True))

    def score(self, image: Image.Image) -> Numeric:
        assert self.metric
        self.metric.update(img1=image, img2=self.image, text2=self.text)
        value = self.metric.compute()
        self.metric.reset()
        return value

    # ---- one batch of expansions ------------------------------------------------------------------------------------
    def _select(self, k: int) -> List[WideNode]:
        """k leaves by repeated tree descent; every pick leaves a virtual visit on its path so that the next descent
        sees a lower exploration bonus there (undone before the real update)."""
        picks: List[WideNode] = []
        for _ in range(k):
            node = self.montecarlo.root_node
            while node.expanded:
                node = node.get_preferred_child(self.montecarlo.root_node)
            picks.append(node)
            cur: Optional[WideNode] = node
            while cur is not None:
                cur.visits += 1
                cur = cur.parent
        for node in picks:
            cur = node
            while cur is not None:
                cur.visits -= 1
                cur = cur.parent
        return picks

    def _rollout_batch(self, starts: List[WideNode]) -> List[List[WideNode]]:
        """Roll out from every start node; returns the candidate nodes (one per completed line) of each rollout."""
        trackers = [LineTracker(n.state, self.newlineinfo, self.failed_rollouts, self.control.reset() if i == 0 else self.control,
                                self.exploration) for i, n in enumerate(starts)]
        live = [i for i, n in enumerate(starts) if not self._exhausted(n.token_ids)]
        if live:
            streamers = [self.streamer if (i == live[0]) else None for i in live]   # an external streamer follows the first rollout
            with torch.inference_mode():
                if len(live) == 1 or not hasattr(self.model, "generate_batch"):
                    for i, st in zip(live, streamers):
                        self.model.generate(
                            input_ids=starts[i].token_ids.unsqueeze(0), pixel_values=self.pixel_values,
                            bad_words_ids=[[self.model.config.image_token_id]],
                            begin_suppress_tokens=[self.model.config.text_config.eos_token_id],
                            streamer=st, stopping_criteria=StoppingCriteriaList([trackers[i]]), **self.adapter_kwargs,
                            **self.gen_kwargs)
                else:
                    self.model.generate_batch(
                        [starts[i].token_ids for i in live], pixel_values=self.pixel_values,
                        bad_words_ids=[[self.model.config.image_token_id]],
                        begin_suppress_tokens=[self.model.config.text_config.eos_token_id],
                        streamers=streamers, stopping_criteria=[[trackers[i]] for i in live], **self.adapter_kwargs,
                        **self.gen_kwargs)
        elif self.streamer is not None:
            self.streamer.end()
        if self.control.should_stop:
            raise InterruptedError
        return [t.finish() for t in trackers]

    def _graft(self, anchor: WideNode, nodes: List[WideNode], tikz: TikzDocument, scorable: bool) -> WideNode:
        """Attach (a thinned subset of) the rollout's nodes below ``anchor``; returns the deepest attached node."""
        keep = round(sqrt(len(nodes)))   # keep O(sqrt n) of the n lines as explicit tree nodes
        if scorable:
            for cand in nodes[:keep]:
                anchor.add_child(cand)
                anchor = cand
            return anchor
        # Failed program: only usable when the error can be located (line 0 = "unknown").
        error_line = min(tikz.errors or [0])
        if error_line:
            for idx, cand in enumerate(nodes):
                closes_line = self.newlineinfo.get(int(cand.token_ids[-1]))
                if cand.num_lines < error_line and idx < keep:
                    anchor.add_child(cand)
                    anchor = cand
                elif cand.num_lines > error_line or (cand.num_lines == error_line and closes_line):
                    self.failed_rollouts[cand.state] = nodes[idx:]
                    break
        return anchor

    def _rewards(self, docs: List[TikzDocument], scorable: List[bool]) -> List[Numeric]:
        """SelfSim rewards of the scorable documents in ONE batched ViT pass when the metric can do that
        (``ImageSim.get_similarities``); compiler-diagnostic reward without a metric (reference :334-339)."""
        if not self.metric:
            return [ok - d.compiled_with_errors for d, ok in zip(docs, scorable)]
        rewards: List[Numeric] = [-1] * len(docs)
        idx = [i for i, ok in enumerate(scorable) if ok]
        if len(idx) > 1 and hasattr(self.metric, "get_similarities"):
            values = self.metric.get_similarities([docs[i].rasterize() for i in idx], self.image,
                                                  **({"text": self.text} if self.text is not None else {}))
            for i, v in zip(idx, values):
                rewards[i] = v
        else:
            for i in idx:
                rewards[i] = self.score(docs[i].rasterize())
        return rewards

    def expand_batch(self, k: int = 1, starts: Optional[List[WideNode]] = None) -> None:
        starts = starts if starts is not None else self._select(k)
        rollouts = self._rollout_batch(starts)
        anchors, tails, docs = [], [], []
        for node, nodes in zip(starts, rollouts):
            if node.is_widen_node:           # the twin stands for "sample another continuation of my parent"
                node.visits += 1
                node, nodes = self.merge(node.parent, nodes)
            anchors.append(node)
            tails.append(nodes)
            docs.append(self.decode((nodes or [node])[-1].token_ids))
        scorable = [bool(d.is_rasterizable and not (self.strict and d.compiled_with_errors)) for d in docs]
        rewards = self._rewards(docs, scorable)
        for node, nodes, tikz, ok, reward in zip(anchors, tails, docs, scorable, rewards):
            if nodes and nodes[0].parent is None and any(ch.state == nodes[0].state for ch in node.children):
                node, nodes = self.merge(node, nodes)     # two rollouts of this batch started with the same line(s)
            node = self._graft(node, nodes, tikz, ok)
            node.update_win_value(self.norm(reward) if ok and self.metric else reward)
            self.solution.append((reward, tikz))
        for node in starts:   # MonteCarlo.expand's bookkeeping (mcts/montecarlo.py): a node with children is inner from now on
            self.montecarlo.stats_expansion_count += 1   # (every real node carries its widen twin, widen nodes stay leaves)
            if node.children:
                node.expanded = True
            else:
                self.montecarlo.stats_failed_expansion_count += 1

    def child_finder(self, node: WideNode, montecarlo: MonteCarlo):
        """``MonteCarlo.expand`` hook (reference :305-343): one sequential expansion of ``node`` (the caller does the
        expansion bookkeeping itself)."""
        count, failed = montecarlo.stats_expansion_count, montecarlo.stats_failed_expansion_count
        was = node.expanded
        self.expand_batch(1, starts=[node])
        montecarlo.stats_expansion_count, montecarlo.stats_failed_expansion_count, node.expanded = count, failed, was

    def merge(self, node: WideNode, nodes_to_merge: List[WideNode]) -> Tuple[WideNode, List[WideNode]]:
        """Walk down existing children that coincide with the head of the new rollout."""
        while nodes_to_merge:
            match = next((ch for ch in node.children if ch.state == nodes_to_merge[0].state), None)
            if match is None:
                break
            node, nodes_to_merge = match, nodes_to_merge[1:]
        return node, nodes_to_merge


class DetikzifyPipeline:
    def __init__(self, model, processor, temperature: float = 0.8, top_p: float = 0.95, top_k: int = 0,
                 compile_timeout: Optional[int] = 60, metric="model", **gen_kwargs):
        self.model, self.processor = model, processor
        if metric == "model":      # SelfSim
            self.metric = ImageSim.from_detikzify(model, processor, sync_on_compute=False)
        elif metric == "fast":     # compiler diagnostics only
            self.metric = None
        else:
            self.metric = metric
        self.gen_kwargs: Dict[str, Any] = dict(
            temperature=temperature, top_p=top_p, top_k=top_k,
            max_length=unwrap(processor).tokenizer.model_max_length, do_sample=True,
            compile_timeout=compile_timeout, **gen_kwargs)

    def load(self, image: Union[Image.Image, str], preprocess: bool = True):
        image = load(image)
        return expand(image, max(image.size), do_trim=True) if preprocess else image

    def check_inputs(self, image, text):
        assert text is None or has_adapter(self.model), "You need to load an adapter for textual inputs!"
        assert image or text, "Either image or text (or both) required!"

    def sample(self, image=None, text: Optional[str] = None, preprocess: bool = True, **gen_kwargs) -> TikzDocument:
        self.check_inputs(image, text)
        generator = DetikzifyGenerator(
            model=self.model, processor=self.processor,
            image=self.load(image, preprocess=preprocess) if image is not None else None, text=text,
            **self.gen_kwargs, **gen_kwargs)
        return generator.sample()

    def simulate(self, image=None, text: Optional[str] = None, preprocess: bool = True,
                 expansions: Optional[Numeric] = None, timeout: Optional[int] = None, **gen_kwargs):
        self.check_inputs(image, text)
        if text is not None and isinstance(self.metric, ImageSim) and self.metric.tokenizer is None:
            raise ValueError("SelfSim with a caption encodes the caption side with the adapted tower: create the pipeline "
                             "after adapter.load(model, processor)")
        generator = DetikzifyGenerator(
            model=self.model, processor=self.processor, metric=self.metric, mcts_timeout=timeout or None,
            image=self.load(image, preprocess=preprocess) if image is not None else None, text=text,
            **self.gen_kwargs, **gen_kwargs)
        yield from generator.simulate(expansions or None)


    def sample_batch(self, images, preprocess: bool = True, samples_per_image: int = 1, **gen_kwargs) -> List[TikzDocument]:
        """Extension (the reference samples one figure at a time): DeTikZify several figures — and/or draw several samples
        per figure — in ONE lock-step batched decode (``model.generate_batch``): the decoder weights are streamed once per
        step for the whole batch. Returns ``len(images) * samples_per_image`` documents, image-major. Needs a model loaded
        with ``max_batch`` / ``max_seqs`` at least that large."""
        if not hasattr(self.model, "generate_batch"):
            raise TypeError("sample_batch needs a detikzify_b200 model (generate_batch)")
        images = [self.load(im, preprocess=preprocess) for im in images]
        kw = {**self.gen_kwargs, **gen_kwargs}
        timeout = kw.pop("compile_timeout", 60)
        prompts, pixels = [], []
        for im in images:
            enc = self.processor(images=im, text=None, return_tensors="pt")
            for _ in range(samples_per_image):
                prompts.append(enc.input_ids[0])
                pixels.append(enc["pixel_values"][0])
        outs = self.model.generate_batch(
            prompts, pixel_values=torch.stack(pixels), bad_words_ids=[[self.model.config.image_token_id]],
            begin_suppress_tokens=[self.model.config.text_config.eos_token_id], **kw)
        docs = []
        for ids, prompt in zip(outs, prompts):
            code = self.processor.decode(token_ids=ids[len(prompt):], skip_special_tokens=True)
            docs.append(TikzDocument(code=code, timeout=timeout))
        return docs

    def sample_many(self, images, samples_per_image: int = 1, batch_size: Optional[int] = None, preprocess: bool = True,
                    **gen_kwargs) -> Generator[Tuple[int, TikzDocument], None, None]:
        """``sample_batch`` for any number of figures and samples through one continuously refilled decode loop
        (``model.generate_batch``'s kwargs and prompts, ``model.generate_many``): at most ``batch_size`` programs are decoded
        at once and a finished one's row takes the next program at once. Each figure's samples share its image prefix.
        Yields ``(index, document)`` in completion order; index ``i`` is sample ``i % samples_per_image`` of figure
        ``i // samples_per_image``, as in ``sample_batch``'s image-major list."""
        if not hasattr(self.model, "generate_many"):
            raise TypeError("sample_many needs a detikzify_b200 model (generate_many)")
        images = [self.load(im, preprocess=preprocess) for im in images]
        kw = {**self.gen_kwargs, **gen_kwargs}
        timeout = kw.pop("compile_timeout", 60)
        prompts, pixels = [], []
        for im in images:
            enc = self.processor(images=im, text=None, return_tensors="pt")
            pixels.append(enc["pixel_values"][0])
            prompts += [enc.input_ids[0]] * samples_per_image
        if not prompts:
            return
        figure = [i // samples_per_image for i in range(len(prompts))]
        for i, ids in self.model.generate_many(
                prompts, pixel_values=torch.stack(pixels), figure=figure, batch_size=batch_size,
                bad_words_ids=[[self.model.config.image_token_id]],
                begin_suppress_tokens=[self.model.config.text_config.eos_token_id], **kw):
            code = self.processor.decode(token_ids=ids[len(prompts[i]):], skip_special_tokens=True)
            yield i, TikzDocument(code=code, timeout=timeout)

    def __call__(self, *args, **kwargs) -> TikzDocument:
        return self.sample(*args, **kwargs)
