"""Host logic of continuous batching (``generate_many`` / ``sample_many``) on CPU, driven by a scripted engine that also
takes admissions and retirements: completion order, the per-request contract, equality with ``generate_batch`` for the
first wave, slot accounting on every exit path and the refusals."""

import pytest
import torch
from PIL import Image, ImageDraw

from scripted_engine import ScriptedEngine


class ManyEngine(ScriptedEngine):
    """ScriptedEngine with the loop's row activity: a retired row draws nothing (-1 in the ring) and writes no KV; an admitted
    row draws its first token as ``sample`` would and continues from its prompt. Freeing a slot that still lends a prefix
    raises, as the engine does; ``log`` records slot frees next to streamer ends."""

    def __init__(self, cfg, max_batch=4, **kw):
        super().__init__(cfg, **kw)
        self.max_batch, self.lent, self.log = max_batch, {}, []
        self.options = {"cascade_attn": 1}

    def seq_share(self, base, dst, length):
        super().seq_share(base, dst, length)
        self.lent.setdefault(base, set()).add(dst)

    def seq_free(self, s):
        if self.lent.get(s):
            raise RuntimeError(f"slot {s} still lends a prefix to {self.lent[s]}")
        for borrowers in self.lent.values():
            borrowers.discard(s)
        self.lent.pop(s, None)
        self.log.append(("free", s))
        super().seq_free(s)

    def get_option(self, key):
        return self.options[key]

    def set_option(self, key, value):
        assert self._gen is None
        self.options[key] = value

    def gen_begin(self, slots, positions, first_ids, params, seq_ids=None):
        super().gen_begin(slots, positions, first_ids, params, seq_ids)
        self._gen["active"] = [True] * len(slots)
        self._gen["first"] = {}

    def gen_step(self):
        g = self._gen
        row = []
        for b, slot in enumerate(g["slots"]):
            if not g["active"][b]:
                row.append(-1)
                continue
            pos = min(g["pos"][b], self.max_len - 1)
            self._hist[slot] = self._hist.get(slot, [])[:pos] + [g["tok"][b]]
            nxt = self._next(g["tok"][b], pos + 1, g["params"], False)
            g["pos"][b] += 1; g["tok"][b] = nxt
            row.append(nxt)
        g["out"].append(row)
        self.calls.append(("gen_step",))

    def gen_retire(self, row):
        self.calls.append(("gen_retire", row))
        self._gen["active"][row] = False

    def gen_admit(self, row, slot, position, logits, seq_id, history=None, eos_min_len=0):
        g = self._gen
        assert not g["active"][row] and slot in self._slots and position == len(self._hist[slot])
        self.calls.append(("gen_admit", row, slot, position, seq_id))
        first = self._next(int(logits[0]), int(logits[1]), g["params"], True)
        g["slots"][row], g["pos"][row], g["tok"][row], g["active"][row] = slot, position, first, True
        g["first"][row] = first

    def gen_first(self, row):
        return self._gen["first"][row]


def _model(max_batch=4, eos_at=None):
    from detikzify_b200.model import build_processor, preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    cfg = preset("tiny")
    eng = ManyEngine(cfg, max_batch=max_batch, eos_at=eos_at)
    model = DetikzifyForCausalLM(cfg, engine=eng)
    eng.own = set(eng._slots)                   # generate()'s prefix-cache slot
    return model, build_processor(cfg), eng


def _figure(size=90):
    im = Image.new("RGB", (size, size + 20), "white")
    d = ImageDraw.Draw(im)
    d.line((10, 10, size - 10, size - 5), fill="black", width=3)
    return im


def _prompts(proc, n, extra=lambda i: 0):
    ids = proc(images=_figure(), text=None, return_tensors="pt").input_ids[0]
    return [torch.cat([ids, torch.arange(40, 60), torch.arange(70, 70 + extra(i))]) for i in range(n)]


KW = dict(do_sample=False, bad_words_ids=[[5]], max_length=200)


def _lengths_crit(prompts, new):
    """per-request stopping criteria: request i stops after new[i] new tokens"""
    return [[(lambda ids, scores, n=len(p) + k: ids.shape[1] >= n)] for p, k in zip(prompts, new)]


@pytest.mark.parametrize("N", [3, 4, 23])
def test_completion_order_and_results(N):
    model, proc, eng = _model(max_batch=4)
    pix = torch.rand(1, 3, 56, 56)
    prompts = _prompts(proc, N)
    new = [(7 * i + 3) % 17 + 2 for i in range(N)]
    crit = _lengths_crit(prompts, new)
    done_at = {}
    got = []
    for i, ids in model.generate_many(prompts, pix, stopping_criteria=crit, **KW):
        got.append(i)
        done_at[i] = len(eng.calls)
        assert isinstance(ids, torch.Tensor) and ids.dim() == 1
        assert len(ids) == len(prompts[i]) + new[i]
    assert sorted(got) == list(range(N))
    if N <= 4:                               # one wave: shorter programs complete first
        assert got == sorted(range(N), key=lambda i: (new[i], i))
    else:                                    # later requests complete before the long ones of the first wave
        longest = max(range(4), key=lambda i: new[i])
        assert any(got.index(j) < got.index(longest) for j in range(4, N))
    ref = model.generate_batch(prompts, pix, stopping_criteria=crit, **KW) if N <= 4 else None
    if ref is not None:
        outs = dict(model.generate_many(prompts, pix, stopping_criteria=crit, **KW))
        assert [outs[i].tolist() for i in range(N)] == [r.tolist() for r in ref]
    assert eng._slots == eng.own


def test_tokens_do_not_depend_on_the_schedule():
    """Every request's ids equal a lock-step run of it alone: the row it lands in and the step it enters at do not matter."""
    model, proc, eng = _model(max_batch=3)
    pix = torch.rand(1, 3, 56, 56)
    prompts = _prompts(proc, 9, extra=lambda i: i % 3)
    new = [4, 12, 2, 9, 1, 6, 15, 3, 5]
    crit = _lengths_crit(prompts, new)
    outs = dict(model.generate_many(prompts, pix, stopping_criteria=crit, **KW))
    for i, p in enumerate(prompts):
        alone = model.generate_batch([p, p], pix, stopping_criteria=[crit[i], crit[i]], **KW)[0]
        assert outs[i].tolist() == alone.tolist()
    admits = [c for c in eng.calls if c[0] == "gen_admit"]
    assert [c[4] for c in admits] == list(range(3, 9))      # request i draws on RNG stream i
    assert eng._slots == eng.own


def test_first_wave_equals_generate_batch_calls():
    """N <= batch_size: the same engine calls as generate_batch (retirements aside); N > batch_size: the same calls up to
    the loop's start for the first batch_size prompts, and the same ids for them."""
    model, proc, eng = _model(max_batch=4)
    pix = torch.rand(1, 3, 56, 56)
    prompts = _prompts(proc, 4, extra=lambda i: i)
    crit = _lengths_crit(prompts, [5, 9, 2, 7])
    eng.calls.clear()
    ref = model.generate_batch(prompts, pix, stopping_criteria=crit, **KW)
    ref_calls = list(eng.calls)
    eng.calls.clear()
    outs = dict(model.generate_many(prompts, pix, stopping_criteria=crit, **KW))
    assert [c for c in eng.calls if c[0] != "gen_retire"] == ref_calls
    assert [outs[i].tolist() for i in range(4)] == [r.tolist() for r in ref]

    more = prompts + _prompts(proc, 5, extra=lambda i: 3)
    crit_more = crit + _lengths_crit(more[4:], [3, 3, 8, 1, 4])
    eng.calls.clear()
    outs = dict(model.generate_many(more, pix, batch_size=4, stopping_criteria=crit_more, **KW))
    begin = next(k for k, c in enumerate(eng.calls) if c[0] == "gen_begin")
    assert eng.calls[: begin + 1] == ref_calls[: begin + 1]
    assert [outs[i].tolist() for i in range(4)] == [r.tolist() for r in ref]


def test_streamers_stops_eos_and_max_length_are_per_request():
    from detikzify_b200.util import TokenStreamer
    model, proc, eng = _model(max_batch=2, eos_at=45)
    pix = torch.rand(1, 3, 56, 56)
    prompts = _prompts(proc, 5, extra=lambda i: 2 * i)        # lengths 25 + 2i: EOS at position 45 ends each differently
    streamers = [TokenStreamer(skip_prompt=False) for _ in prompts]
    crit = [[], [lambda ids, s: ids.shape[1] >= len(prompts[1]) + 3], [], [], []]
    outs = dict(model.generate_many(prompts, pix, streamers=streamers, stopping_criteria=crit, max_length=len(prompts[0]) + 30,
                                    do_sample=False))
    eos = model.config.eos_token_id
    assert len(outs[1]) == len(prompts[1]) + 3 and outs[1][-1] != eos
    for i in (0, 2, 3, 4):
        o = outs[i].tolist()
        assert o[-1] == eos or len(o) == len(prompts[0]) + 30
        assert eos not in o[len(prompts[i]):-1]
    for i, st in enumerate(streamers):
        assert list(st) == outs[i].tolist()                     # prompt, every token, and end() (the iterator finished)
    short = dict(model.generate_many(prompts[:3], pix, max_length=len(prompts[1]), do_sample=False))
    assert short[0].tolist()[: len(prompts[0])] == prompts[0].tolist() and len(short[0]) == len(prompts[1])
    assert short[1].tolist() == prompts[1].tolist()             # prompt at max_length: nothing appended
    assert len(short[2]) == len(prompts[2])                      # prompt already beyond max_length: returned as it is
    assert eng._slots == eng.own


def test_slots_released_on_every_exit_path():
    model, proc, eng = _model(max_batch=3)
    pix = torch.rand(1, 3, 56, 56)
    prompts = _prompts(proc, 8)
    crit = _lengths_crit(prompts, [6, 2, 9, 4, 7, 3, 5, 8])

    class Boom:
        def __init__(self):
            self.n = 0

        def put(self, value):
            self.n += 1
            if self.n == 3:
                raise RuntimeError("streamer failed")

        def end(self):
            pass

    with pytest.raises(RuntimeError, match="streamer failed"):
        list(model.generate_many(prompts, pix, streamers=[None] * 4 + [Boom()] + [None] * 3, stopping_criteria=crit, **KW))
    assert eng._slots == eng.own and eng._gen is None and not model._lock.locked()
    gen = model.generate_many(prompts, pix, stopping_criteria=crit, **KW)
    next(gen)
    gen.close()                                                  # the consumer abandons the stream
    assert eng._slots == eng.own and eng._gen is None and not model._lock.locked()
    assert dict(model.generate_many(prompts, pix, stopping_criteria=crit, **KW)).keys() == set(range(8))
    assert eng._slots == eng.own


def test_figure_base_lives_until_its_last_request():
    """Two figures, one shared-prefix base each: a base is freed right after its figure's last request finishes, never while
    a row borrows it (the engine refuses that), and the loop runs without the single-prefix cascade."""
    from detikzify_b200.util import TokenStreamer
    model, proc, eng = _model(max_batch=3)
    pix = torch.rand(2, 3, 56, 56)
    prompts = _prompts(proc, 7)
    figure = [0, 1, 0, 1, 1, 0, 1]
    crit = _lengths_crit(prompts, [9, 2, 5, 3, 7, 4, 2])

    class Ends(TokenStreamer):
        def __init__(self, i):
            super().__init__()
            self.i = i

        def end(self):
            eng.log.append(("end", self.i))
            super().end()

    seen = []
    for i, _ in model.generate_many(prompts, pix, figure=figure, stopping_criteria=crit,
                                    streamers=[Ends(i) for i in range(7)], **KW):
        seen.append(i)
        assert eng.options["cascade_attn"] == 0                  # off while the loop runs
    assert eng.options["cascade_attn"] == 1 and eng._slots == eng.own
    shares = [c for c in eng.calls if c[0] == "seq_share"]
    bases = {}
    for c in shares:
        bases.setdefault(c[1], set()).add(c[2])
    assert len(bases) == 2
    embeds = [c for c in eng.calls if c[0] == "image_embeds"]
    assert embeds == [("image_embeds", (2, 3, 56, 56))]         # the tower ran once, for both figures, ahead of admission
    freed = set()
    for b in bases:
        at = eng.log.index(("free", b))
        kind, last = eng.log[at + 1]                             # the base goes right before its last request ends
        assert kind == "end"
        f = figure[last]
        assert all(eng.log.index(("end", i)) <= at + 1 for i in range(7) if figure[i] == f)
        freed.add(f)
    assert freed == {0, 1}


def test_refusals():
    model, proc, eng = _model(max_batch=4)
    prompts = _prompts(proc, 3)
    pix = torch.rand(1, 3, 56, 56)
    for bs in (1, 5):
        with pytest.raises(ValueError):
            model.generate_many(prompts, pix, batch_size=bs)
    with pytest.raises(ValueError):
        model.generate_many(prompts, pix, adapter_input_ids=torch.tensor([[1, 2]]))
    with pytest.raises(ValueError):
        model.generate_many(prompts, torch.rand(2, 3, 56, 56))   # two figures for three prompts, no `figure`
    with pytest.raises(ValueError):
        model.generate_many(prompts, pix, figure=[0, 1, 0])       # figure index out of range
    assert eng._slots == eng.own


def test_pipeline_sample_many(monkeypatch):
    from detikzify_b200.infer import DetikzifyPipeline, TikzDocument
    model, proc, eng = _model(max_batch=4, eos_at=40)
    monkeypatch.setattr(TikzDocument, "backend", staticmethod(lambda code: Image.new("RGB", (8, 8), "white")))
    pipe = DetikzifyPipeline(model, proc, metric="fast")
    docs = list(pipe.sample_many([_figure(), _figure(70), _figure(80)], samples_per_image=3, batch_size=4))
    assert sorted(i for i, _ in docs) == list(range(9))
    assert all(isinstance(d, TikzDocument) and d.code for _, d in docs)
    assert sum(1 for c in eng.calls if c[0] == "gen_begin") == 1 and any(c[0] == "gen_admit" for c in eng.calls)
    assert ("image_embeds", (3, 3, 56, 56)) in eng.calls
    assert eng.last_sampling["do_sample"] and eng._slots == eng.own
