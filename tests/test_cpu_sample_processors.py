"""HF logits processors of the sampler (dtk_processors): the fp64 restatement in tests/processors_oracle.py against the
installed transformers' processors built in HF's order, and the host plumbing of ``generate`` / ``generate_batch``
(kwargs, generation_config fallbacks, validation, the engine calls) with a scripted engine."""
import numpy as np
import pytest
import torch
from transformers.generation.logits_process import (
    LogitsProcessorList, MinLengthLogitsProcessor, MinNewTokensLengthLogitsProcessor, MinPLogitsWarper,
    NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor, RepetitionPenaltyLogitsProcessor,
    SuppressTokensAtBeginLogitsProcessor, SuppressTokensLogitsProcessor, TemperatureLogitsWarper, TopKLogitsWarper,
    TopPLogitsWarper)

import processors_oracle as po
from scripted_engine import ScriptedEngine


def hf_chain(prompt_len, eos, penalty=None, ngram=0, bad=None, min_length=0, min_new=None, suppress=None, begin=None,
             do_sample=False, temperature=1.0, top_k=0, top_p=1.0, min_p=None):
    """The processors HF generation/utils.py::_get_logits_processor builds, in its order."""
    L = LogitsProcessorList()
    if penalty is not None and penalty != 1.0:
        L.append(RepetitionPenaltyLogitsProcessor(penalty=penalty))
    if ngram > 0:
        L.append(NoRepeatNGramLogitsProcessor(ngram))
    if bad is not None:
        L.append(NoBadWordsLogitsProcessor(bad, eos_token_id=eos))
    if min_length > 0:
        L.append(MinLengthLogitsProcessor(min_length, eos, device="cpu"))
    if min_new is not None and min_new > 0:
        L.append(MinNewTokensLengthLogitsProcessor(prompt_len, min_new, eos, device="cpu"))
    if suppress is not None:
        L.append(SuppressTokensLogitsProcessor(suppress, device="cpu"))
    if begin is not None:
        L.append(SuppressTokensAtBeginLogitsProcessor(begin, prompt_len, device="cpu"))
    if do_sample:
        if temperature != 1.0:
            L.append(TemperatureLogitsWarper(temperature))
        if top_k:
            L.append(TopKLogitsWarper(top_k))
        if top_p < 1.0:
            L.append(TopPLogitsWarper(top_p))
        if min_p:
            L.append(MinPLogitsWarper(min_p))
    return L


def oracle_args(prompt_len, eos, V, penalty=None, ngram=0, bad=None, min_length=0, min_new=None, suppress=None, begin=None,
                L=0, B=1):
    """The dtk_processors tables the model builds from the same kwargs (single ids -> ban list, [eos] dropped)."""
    words = [list(w) for w in (bad or []) if list(w) != [eos]]
    ban = [w[0] for w in words if len(w) == 1] + list(suppress or [])
    eml = max(min_length, prompt_len + (min_new or 0))
    return dict(penalty=penalty or 1.0, ngram=ngram, ban_ids=ban, begin_ids=list(begin or []),
                words=[w for w in words if len(w) > 1], eos=eos, eos_min_len=[eml] * B, suppress=L == prompt_len)


CASES = {
    "penalty": dict(penalty=1.3),
    "penalty_below_1": dict(penalty=0.7),
    "ngram3": dict(ngram=3),
    "ngram1": dict(ngram=1),
    "ngram_longer_than_history": dict(ngram=40),
    "bad_words": dict(bad=[[5], [3, 7], [1, 2, 9], [0], [255]]),
    "bad_word_longer_than_history": dict(bad=[list(range(1, 40)), [2, 4]]),
    "bad_eos_filtered": dict(bad=[[8], [4]]),
    "min_length": dict(min_length=30),
    "min_new_tokens": dict(min_new=5),
    "min_length_and_min_new": dict(min_length=20, min_new=2),
    "suppress": dict(suppress=[0, 255, 17]),
    "begin": dict(begin=[8, 3, 0]),
    "all": dict(penalty=1.2, ngram=2, bad=[[5], [3, 7], [0, 255, 6]], min_new=3, suppress=[11], begin=[8, 12]),
}


def _history(rng, B, L, V):
    """Histories with repeats (small alphabet) so that n-grams and bad-word prefixes do match."""
    h = rng.integers(0, 12, size=(B, L))
    h[:, ::7] = rng.integers(0, V, size=h[:, ::7].shape)
    h[0, -1], h[0, -2] = 7, 3          # row 0 ends with [3, 7]
    h[1, -1] = 3                       # row 1 ends with [3]: bans 7 through the bad word [3, 7]
    return h


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("L,prompt_len", [(24, 24), (24, 20), (3, 3)])
def test_processors_equal_hf(name, L, prompt_len):
    V, B, eos = 256, 4, 8
    kw = CASES[name]
    rng = np.random.default_rng(hash((name, L)) % 2**32)
    logits = rng.normal(0, 3, size=(B, V)).astype(np.float32)
    logits[:, :B] = -np.abs(logits[:, :B])          # negative logits on history ids too (penalty multiplies them)
    hist = _history(rng, B, L, V)
    ref = hf_chain(prompt_len, eos, **kw)(torch.tensor(hist), torch.tensor(logits)).numpy()
    got = po.processed_logits(logits, hist, **oracle_args(prompt_len, eos, V, L=L, B=B, **kw))
    assert np.array_equal(np.isinf(ref), np.isinf(got))
    assert np.array_equal(ref[np.isfinite(ref)].astype(np.float64), got[np.isfinite(got)])   # fp32 penalty bit for bit


@pytest.mark.parametrize("mode", ["top_p", "top_k", "min_p", "all"])
def test_chain_with_warpers_equals_hf(mode):
    V, B, eos, L = 1000, 3, 8, 50
    rng = np.random.default_rng(7)
    logits = rng.normal(0, 2, size=(B, V)).astype(np.float32)
    hist = _history(rng, B, L, V)
    warp = dict(top_p=dict(top_p=0.8), top_k=dict(top_k=40), min_p=dict(min_p=0.05),
                all=dict(top_k=200, top_p=0.9, min_p=0.1, temperature=0.7))[mode]
    procs = dict(penalty=1.3, ngram=3, bad=[[5], [3, 7]], suppress=[1])
    scores = hf_chain(40, eos, do_sample=True, **procs, **warp)(torch.tensor(hist), torch.tensor(logits))
    ref = torch.softmax(scores.double(), -1).numpy()
    r = po.processed_probs(logits, hist, temperature=warp.get("temperature", 1.0), top_p=warp.get("top_p", 1.0),
                           top_k=warp.get("top_k", 0), min_p=warp.get("min_p", 0.0),
                           **oracle_args(40, eos, V, L=L, B=B, **procs))
    assert np.array_equal(ref > 0, r["kept"])
    np.testing.assert_allclose(r["probs"], ref, rtol=1e-5, atol=1e-7)


def test_ngram_and_bad_word_edges():
    assert po.banned_ngram_tokens([1, 2, 1, 3, 1], 1) == [1, 2, 1, 3, 1]
    assert po.banned_ngram_tokens([1, 2, 3, 1, 2], 3) == [3]
    assert po.banned_ngram_tokens([1, 2], 3) == []           # L + 1 = n: no complete n-gram yet
    assert po.banned_ngram_tokens([1], 3) == []
    # HF skips a bad word longer than the history, even one whose prefix would fit ([4, 5, 6] after [4, 5])
    s = po.processed_logits(np.zeros((1, 10), np.float32), [[4, 5]], words=[[4, 5, 6], [1, 4, 5, 7], [5, 9]])
    assert np.isinf(s[0]).nonzero()[0].tolist() == [9]
    s = po.processed_logits(np.zeros((1, 10), np.float32), [[3, 4, 5]], words=[[4, 5, 6], [5, 9], [3, 5, 2]])
    assert np.isinf(s[0]).nonzero()[0].tolist() == [6, 9]


# ------------------------------------------------------------------ host plumbing (scripted engine)
class ProcEngine(ScriptedEngine):
    def set_processors(self, proc, histories=(), eos_min_len=None):
        self.calls.append(("set_processors", None if proc is None else dict(proc), [list(h) for h in histories],
                           None if eos_min_len is None else list(eos_min_len)))


def _model(cls=ProcEngine, eos_at=None):
    from detikzify_b200.model import preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    cfg = preset("tiny")
    eng = cls(cfg, eos_at=eos_at)
    return DetikzifyForCausalLM(cfg, engine=eng), eng


def _prompt(cfg, extra=(65, 66)):
    return torch.tensor([[cfg.patch_token_id] * cfg.num_patches + list(extra)])


def test_generate_passes_processors_and_histories():
    model, eng = _model()
    cfg = model.config
    ids = _prompt(cfg)
    T0 = ids.shape[1]
    out = model.generate(input_ids=ids, pixel_values=torch.zeros(1, 3, 56, 56), max_length=T0 + 6,
                         repetition_penalty=1.3, no_repeat_ngram_size=3, bad_words_ids=[[cfg.image_token_id], [65, 66]],
                         min_new_tokens=4, begin_suppress_tokens=[cfg.eos_token_id])[0].tolist()
    sets = [c for c in eng.calls if c[0] == "set_processors"]
    want = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_p=0.0, eos_token_id=cfg.eos_token_id,
                ban_ids=[cfg.image_token_id], begin_ids=[cfg.eos_token_id], words=[[65, 66]])
    assert sets[0] == ("set_processors", want, [ids[0].tolist()], [T0 + 4])
    assert sets[1] == ("set_processors", want, [out[:T0 + 1]], [T0 + 4])
    assert sets[2] == ("set_processors", None, [], None)
    kinds = [c[0] for c in eng.calls]
    assert kinds.index("sample") > kinds.index("set_processors") and kinds[-1] == "set_processors"
    assert kinds.index("gen_begin") == kinds.index("set_processors", kinds.index("sample")) + 1
    assert eng.last_sampling["bad_token"] == -1 and eng.last_sampling["begin_suppress_token"] == -1


def test_generation_config_fallbacks_and_min_length_precedence():
    model, eng = _model()
    cfg = model.config
    ids = _prompt(cfg)
    T0 = ids.shape[1]
    model.generation_config.repetition_penalty = 1.1
    model.generation_config.min_length = T0 + 9
    model.generation_config.suppress_tokens = [3]
    model.generate(input_ids=ids, max_length=T0 + 3, no_repeat_ngram_size=2)
    s = [c for c in eng.calls if c[0] == "set_processors"][0]
    assert s[1]["repetition_penalty"] == 1.1 and s[1]["no_repeat_ngram_size"] == 2 and s[1]["ban_ids"] == [3]
    assert s[3] == [T0 + 9]
    eng.calls.clear()
    model.generate(input_ids=ids, max_length=T0 + 3, min_new_tokens=2)    # min_new_tokens takes precedence (HF)
    assert [c for c in eng.calls if c[0] == "set_processors"][0][3] == [T0 + 2]
    eng.calls.clear()
    model.generate(input_ids=ids, max_length=T0 + 3, min_p=0.2, do_sample=False, repetition_penalty=1.0,
                   min_length=0, suppress_tokens=[])
    assert not [c for c in eng.calls if c[0] == "set_processors"]      # min_p is a warper: off when greedy


@pytest.mark.parametrize("kw", [dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty="x"),
                                dict(no_repeat_ngram_size=-1), dict(no_repeat_ngram_size=1.5), dict(min_length=-2),
                                dict(min_new_tokens=-1), dict(min_p=1.5), dict(min_p=-0.1), dict(bad_words_ids=[[70000]]),
                                dict(bad_words_ids=[[-1]]), dict(bad_words_ids=[[]]), dict(bad_words_ids=[5]),
                                dict(suppress_tokens=[-1]), dict(begin_suppress_tokens=[10**6])])
def test_invalid_arguments_raise(kw):
    model, eng = _model()
    with pytest.raises(ValueError):
        model.generate(input_ids=_prompt(model.config), max_length=40, **kw)
    with pytest.raises(ValueError):
        model.generate_batch([_prompt(model.config)[0]], max_length=40, **kw)


@pytest.mark.parametrize("batch", [False, True])
def test_no_processors_makes_todays_calls(batch):
    """The reference's call (one bad id, one begin-suppress id) and neutral processor kwargs make the same engine calls as
    the scripted engine without a processor entry point."""
    logs = []
    for cls, extra in ((ScriptedEngine, {}), (ProcEngine, dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_p=0.0,
                                                                min_length=0, suppress_tokens=[]))):
        model, eng = _model(cls, eos_at=60)
        cfg = model.config
        kw = dict(bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id], max_length=70, **extra)
        if batch:
            out = model.generate_batch([_prompt(cfg)[0], _prompt(cfg, (67,))[0]], torch.zeros(1, 3, 56, 56), **kw)
        else:
            out = [model.generate(input_ids=_prompt(cfg), pixel_values=torch.zeros(1, 3, 56, 56), **kw)[0]]
        logs.append((eng.calls, eng.last_sampling, [o.tolist() for o in out]))
    assert logs[0] == logs[1]
    assert logs[0][1]["bad_token"] == model.config.image_token_id


def test_eos_bad_word_is_dropped():
    model, eng = _model()
    cfg = model.config
    model.generate(input_ids=_prompt(cfg), max_length=40, bad_words_ids=[[cfg.eos_token_id]])
    assert eng.last_sampling["bad_token"] == -1
    model.generate(input_ids=_prompt(cfg), max_length=40, bad_words_ids=[[cfg.eos_token_id], [4], [5]])
    s = [c for c in eng.calls if c[0] == "set_processors"][0]
    assert s[1]["ban_ids"] == [4, 5]


def test_generate_batch_histories_per_row():
    model, eng = _model()
    cfg = model.config
    prompts = [_prompt(cfg)[0], _prompt(cfg, (67, 68, 69))[0]]
    out = model.generate_batch(prompts, torch.zeros(1, 3, 56, 56), max_new_tokens=5, no_repeat_ngram_size=2,
                               min_new_tokens=3)
    sets = [c for c in eng.calls if c[0] == "set_processors"]
    assert sets[0][2] == [p.tolist() for p in prompts] and sets[0][3] == [len(p) + 3 for p in prompts]
    assert sets[1][2] == [o.tolist()[:len(p) + 1] for o, p in zip(out, prompts)]
    assert sets[-1][1] is None
    kinds = [c[0] for c in eng.calls]
    assert kinds.index("gen_begin") == kinds.index("set_processors", kinds.index("sample")) + 1
