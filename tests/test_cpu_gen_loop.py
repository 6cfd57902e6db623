"""The host decode loop behind ``generate``, ``generate_batch`` and ``generate_many``, pinned on CPU: a recording engine logs
every engine call with its arguments and results, interleaved with streamer payloads, stopping-criterion calls and
generator yields, and each case of the matrix must replay ``tests/golden/host_loop_traces.json`` exactly
(regenerate with ``python tests/golden/make_host_loop_traces.py``)."""

import json
from pathlib import Path

import pytest
import torch

from test_cpu_many import KW, ManyEngine, _figure, _lengths_crit

GOLDEN = Path(__file__).resolve().parent / "golden" / "host_loop_traces.json"


def _plain(v):
    if isinstance(v, torch.Tensor):
        return v.tolist()
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, dict):
        return {str(k): _plain(x) for k, x in sorted(v.items())}
    if hasattr(v, "__dict__"):
        return _plain(vars(v))
    return v


class TraceEngine(ManyEngine):
    """ManyEngine that appends every call the model makes (arguments, and what the call returned) to ``trace``, and takes
    ``set_processors``. ``seq_ids=None`` is logged as the ids the engine uses for it, ``range(B)``."""

    def __init__(self, cfg, trace, **kw):
        super().__init__(cfg, **kw)
        self.trace = trace

    def _log(self, *event):
        self.trace.append(_plain(list(event)))

    def seq_alloc(self):
        s = super().seq_alloc()
        self._log("seq_alloc", s)
        return s

    def seq_free(self, s):
        self._log("seq_free", s)
        super().seq_free(s)

    def seq_fork(self, src, dst, length):
        self._log("seq_fork", src, dst, length)
        super().seq_fork(src, dst, length)

    def seq_share(self, base, dst, length):
        self._log("seq_share", base, dst, length)
        super().seq_share(base, dst, length)

    def image_embeds(self, pix):
        self._log("image_embeds", list(pix.shape))
        return super().image_embeds(pix)

    def prefill(self, slot, ids, start_pos=0, img_embeds=None, img_start=0, want_all_logits=False):
        self._log("prefill", slot, ids, start_pos, None if img_embeds is None else list(img_embeds.shape), img_start)
        return super().prefill(slot, ids, start_pos, img_embeds, img_start, want_all_logits)

    def sampling(self, **kw):
        self._log("sampling", kw)
        return super().sampling(**kw)

    def sample(self, logits, params, suppress=None, steps=None, seq_ids=None, want_probs=False):
        out, probs = super().sample(logits, params, suppress, steps, seq_ids, want_probs)
        B = logits.reshape(-1, 2).shape[0]
        self._log("sample", logits.reshape(-1), params, suppress, steps, list(range(B)) if seq_ids is None else seq_ids,
                  want_probs, out)
        return out, probs

    def set_processors(self, proc, histories=(), eos_min_len=None):
        self._log("set_processors", proc, [list(h) for h in histories], eos_min_len)

    def get_option(self, key):
        v = super().get_option(key)
        self._log("get_option", key, v)
        return v

    def set_option(self, key, value):
        self._log("set_option", key, value)
        super().set_option(key, value)

    def gen_begin(self, slots, positions, first_ids, params, seq_ids=None):
        self._log("gen_begin", slots, positions, first_ids, params, list(range(len(slots))) if seq_ids is None else seq_ids)
        super().gen_begin(slots, positions, first_ids, params, seq_ids)

    def gen_step(self):
        self._log("gen_step")
        super().gen_step()

    def gen_wait(self, step):
        row = super().gen_wait(step)
        self._log("gen_wait", step, row)
        return row

    def gen_end(self):
        self._log("gen_end")
        super().gen_end()

    def gen_retire(self, row):
        self._log("gen_retire", row)
        super().gen_retire(row)

    def gen_admit(self, row, slot, position, logits, seq_id, history=None, eos_min_len=0):
        self._log("gen_admit", row, slot, position, logits, seq_id, history, eos_min_len)
        super().gen_admit(row, slot, position, logits, seq_id, history, eos_min_len)

    def gen_first(self, row):
        t = super().gen_first(row)
        self._log("gen_first", row, t)
        return t


class Streamer:
    def __init__(self, trace, i):
        self.trace, self.i = trace, i

    def put(self, value):
        self.trace.append(["put", self.i, list(value.shape), str(value.dtype), value.tolist()])

    def end(self):
        self.trace.append(["end", self.i])


def _crit(trace, i, stop_len=None, raise_len=None):
    """a logged criterion: stops at ``stop_len`` ids, raises at ``raise_len``"""
    def crit(ids, scores):
        trace.append(["crit", i, list(ids.shape), str(ids.dtype), ids[0, -1].item(), ids.sum().item()])
        if raise_len is not None and ids.shape[1] >= raise_len:
            raise RuntimeError("criterion failed")
        return stop_len is not None and ids.shape[1] >= stop_len
    return crit


def _setup(max_batch=4, eos_at=None):
    from detikzify_b200.model import build_processor, preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    torch.manual_seed(0)                                   # seeds derive from torch.initial_seed() + the call counter
    trace = []
    cfg = preset("tiny")
    eng = TraceEngine(cfg, trace, max_batch=max_batch, eos_at=eos_at)
    model = DetikzifyForCausalLM(cfg, engine=eng)
    trace.clear()
    return model, build_processor(cfg), eng, trace


def _prompt(proc, extra=0):
    ids = proc(images=_figure(), text=None, return_tensors="pt").input_ids[0]
    return torch.cat([ids, torch.arange(40, 60), torch.arange(70, 70 + extra)])


PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3)
SAMPLE = dict(do_sample=True, temperature=0.8, top_p=0.9, top_k=7)


def _case_generate(name):
    sampling, procs, stop, eos_at, at_limit, reuse, boom = (
        "sample" in name, "proc" in name, "stop" in name, 45 if "eos" in name else None, "at_limit" in name,
        "reuse" in name, "raise" in name)
    model, proc, eng, trace = _setup(eos_at=eos_at)
    pix = torch.rand(1, 3, 56, 56)
    p = _prompt(proc)
    kw = dict(KW, **(SAMPLE if sampling else {}), **(PROC if procs else {}))
    if at_limit:
        kw["max_length"] = len(p)
    calls = [p] + ([None] if reuse else [])
    for c, prompt in enumerate(calls):
        if prompt is None:                                 # continue from the first call's output: a cached prefix
            prompt = torch.cat([out[0, : len(p) + 6], torch.arange(90, 95)])
        crit = _crit(trace, c, stop_len=len(prompt) + 9 if stop else None, raise_len=len(prompt) + 7 if boom else None)
        try:
            out = model.generate(prompt[None], pix, streamer=Streamer(trace, c), stopping_criteria=[crit], **kw)
            trace.append(["result", list(out.shape), out.tolist()])
        except RuntimeError as e:
            trace.append(["raised", str(e)])
        trace.append(["slot_tokens", list(model._slot_tokens), eng._gen is None, model._lock.locked()])
    return trace


def _case_generate_batch(name):
    N = int(name.split("_N")[1].split("_")[0])
    model, proc, eng, trace = _setup()
    per_image = "per_image" in name
    pix = torch.rand(N if per_image else 1, 3, 56, 56)
    prompts = [_prompt(proc, extra=i) for i in range(N)]
    kw = dict(KW, **(PROC if "proc" in name else {}), **(SAMPLE if "sample" in name else {}))
    streamers = None if "proc" in name else [Streamer(trace, i) for i in range(N)]
    crits = [[_crit(trace, i, stop_len=len(p) + 3 + 4 * i)] for i, p in enumerate(prompts)]
    outs = model.generate_batch(prompts, pix, streamers=streamers, stopping_criteria=crits,
                                share_prefix="noshare" not in name, **kw)
    trace.append(["result", [o.tolist() for o in outs]])
    trace.append(["slots", sorted(eng._slots), eng._gen is None])
    return trace


def _case_generate_many(name):
    N = int(name.split("_N")[1].split("_")[0])
    B = int(name.split("_B")[1].split("_")[0])
    figs = 2 if "figs" in name else 1
    model, proc, eng, trace = _setup(max_batch=4)
    pix = torch.rand(figs, 3, 56, 56)
    prompts = [_prompt(proc, extra=i % 3) for i in range(N)]
    new = [(7 * i + 3) % 17 + 2 for i in range(N)]
    crits = [[_crit(trace, i, stop_len=len(p) + k)] for i, (p, k) in enumerate(zip(prompts, new))]
    kw = dict(KW, **(PROC if "proc" in name else {}), **(SAMPLE if "sample" in name else {}))
    gen = model.generate_many(prompts, pix, figure=[i % figs for i in range(N)], batch_size=B,
                              streamers=[Streamer(trace, i) for i in range(N)], stopping_criteria=crits, **kw)
    for i, ids in gen:
        trace.append(["yield", i, list(ids.shape), str(ids.dtype), ids.tolist()])
        if "close" in name:
            gen.close()
            break
    trace.append(["slots", sorted(eng._slots), eng._gen is None, eng.options, model._lock.locked()])
    return trace


CASES = (
    ["generate_greedy_stop", "generate_greedy_proc_stop", "generate_sample_stop", "generate_sample_proc_stop",
     "generate_greedy_eos", "generate_sample_proc_eos", "generate_greedy_at_limit", "generate_greedy_reuse",
     "generate_sample_proc_reuse", "generate_greedy_proc_raise"]
    + ["generate_batch_N1", "generate_batch_N3", "generate_batch_N4", "generate_batch_N3_noshare",
       "generate_batch_N4_noshare", "generate_batch_N3_per_image", "generate_batch_N4_sample_proc"]
    + ["generate_many_N3_B2", "generate_many_N3_B4", "generate_many_N23_B2", "generate_many_N23_B4",
       "generate_many_N23_B4_figs", "generate_many_N23_B2_figs_sample_proc", "generate_many_N23_B4_close",
       "generate_many_N23_B4_figs_close"])


def run_case(name):
    if name.startswith("generate_many"):
        return _case_generate_many(name)
    if name.startswith("generate_batch"):
        return _case_generate_batch(name)
    return _case_generate(name)


@pytest.fixture(scope="module")
def golden():
    return json.loads(GOLDEN.read_text())


@pytest.mark.parametrize("name", CASES)
def test_trace_matches_golden(name, golden):
    got = json.loads(json.dumps(run_case(name)))
    want = golden[name]
    for k, (a, b) in enumerate(zip(got, want)):
        assert a == b, f"event {k} of {name} differs"
    assert len(got) == len(want)


@pytest.mark.parametrize("kw", [dict(KW), dict(KW, **SAMPLE, **PROC)], ids=["greedy", "sample_proc"])
def test_generate_equals_generate_batch_of_one(kw):
    """``generate(p)`` and ``generate_batch([p])`` make the same engine calls apart from the slot they decode in."""
    traces = []
    for batch in (False, True):
        model, proc, eng, trace = _setup()
        pix = torch.rand(1, 3, 56, 56)
        p = _prompt(proc)
        crit = _lengths_crit([p], [40])[0]
        if batch:
            out = model.generate_batch([p], pix, stopping_criteria=[crit], **kw)[0]
        else:
            out = model.generate(p[None], pix, stopping_criteria=crit, **kw)[0]
            slot = model._slot
        traces.append(([e for e in trace if e[0] not in ("seq_alloc", "seq_free")], out.tolist()))
    (single, out1), (batched, outb) = traces
    batch_slot = next(e[1] for e in batched if e[0] == "prefill")
    for e in batched:
        if e[0] == "prefill":
            e[1] = slot
        if e[0] == "gen_begin":
            e[1] = [slot if s == batch_slot else s for s in e[1]]
    assert len(single) > 80 and single == batched and out1 == outb
