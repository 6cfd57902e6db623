"""The sampler's HF logits processors (dtk_processors) on the GPU: both sampler kernels through the engine-free hook
``dtk_dbg_sample_proc`` against the fp64 restatement in tests/processors_oracle.py, the neutral tables against
``dtk_dbg_sample``, the generation loop against decode + stepwise sampling with a host-kept history, and ``generate`` /
``generate_batch`` with the processor kwargs against HF's ``generate`` on the fp32 oracle."""
import ctypes as C

import numpy as np
import pytest
import torch

import processors_oracle as po
from conftest import engine_for, model_bundle
from oracle import sample_oracle as so

pytestmark = pytest.mark.gpu


def _lib():
    from detikzify_b200 import _lib as L
    return L.load_library()


def _p(t):
    return C.c_void_p(t.data_ptr())


def _params(temperature=1.0, top_p=1.0, top_k=0, do_sample=True, bad_token=-1, bs_token=-1, seed=0):
    from detikzify_b200.engine import Engine
    return Engine.sampling(temperature=temperature, top_p=top_p, top_k=top_k, do_sample=do_sample, bad_token=bad_token,
                           begin_suppress_token=bs_token, seed=seed)


def dbg_proc(logits, params, proc, hist, eos_min, suppress, steps, impl, max_len):
    from detikzify_b200.engine import c_histories, c_processors
    B, V = logits.shape
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    probs = torch.empty(B, V, dtype=torch.float32, device="cuda")
    ids, lens = c_histories(hist)
    rc = _lib().dtk_dbg_sample_proc(_p(logits), B, V, C.byref(params), (C.c_int * B)(*suppress), (C.c_uint32 * B)(*steps),
                                    None, impl, C.byref(c_processors(**proc)), ids, lens, (C.c_int32 * B)(*eos_min),
                                    max_len, _p(out), _p(probs), None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy(), probs.cpu().numpy()


def dbg_plain(logits, params, suppress, steps, impl):
    B, V = logits.shape
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    probs = torch.empty(B, V, dtype=torch.float32, device="cuda")
    rc = _lib().dtk_dbg_sample(_p(logits), B, V, C.byref(params), (C.c_int * B)(*suppress), (C.c_uint32 * B)(*steps), None,
                               impl, _p(out), _p(probs), None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy(), probs.cpu().numpy()


def _case(V, B, rng, max_len=2048):
    """Logits, histories (small alphabet so that n-grams and bad-word prefixes match; one row at max_len) and tables."""
    logits = rng.normal(0, 3, size=(B, V)).astype(np.float32)
    lens = rng.integers(1, max_len + 1, size=B)
    lens[0] = max_len
    lens[-1] = min(lens[-1], 5)
    hist = []
    for L in lens:
        h = rng.integers(0, 16, size=L)
        h[::5] = rng.integers(0, V, size=h[::5].shape)
        hist.append(h.tolist())
    hist[0][-1] = 3
    words = [[3, 7], [1, 2, V - 1], [hist[-1][-1], 9], list(range(10, 40))]
    proc = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_p=0.05, eos_token_id=V - 2, ban_ids=[0, 5, V - 1],
                begin_ids=[V - 3, 11], words=words)
    eos_min = [int(L) + (b % 2) for b, L in enumerate(lens)]
    suppress = [b % 3 == 0 for b in range(B)]
    return logits, hist, proc, eos_min, suppress


def _oracle(logits, hist, proc, eos_min, suppress, **warp):
    return po.processed_probs(logits, hist, penalty=proc["repetition_penalty"], ngram=proc["no_repeat_ngram_size"],
                              ban_ids=proc["ban_ids"], begin_ids=proc["begin_ids"], words=proc["words"],
                              eos=proc["eos_token_id"], eos_min_len=eos_min, suppress=suppress, **warp)


@pytest.mark.parametrize("V", [264, 32256, 32768, 32769, 128256])
def test_processor_sampler_matches_fp64_reference(V):
    rng = np.random.default_rng(V)
    for B, (T, top_p, top_k, min_p) in zip((1, 7, 64), ((0.8, 1.0, 0, 0.05), (1.0, 0.9, 50, 0.02), (0.6, 0.95, 0, 0.2))):
        max_len = 2048 if B < 64 else 300
        logits, hist, proc, eos_min, sup = _case(V, B, rng, max_len)
        proc["min_p"] = min_p
        params = _params(T, top_p, top_k, seed=V * 31 + B)
        steps = [int(x) for x in rng.integers(0, 2**32, size=B)]
        lg = torch.tensor(logits, device="cuda")
        res = {impl: dbg_proc(lg, params, proc, hist, eos_min, sup, steps, impl, max_len) for impl in (0, 1)}
        tok, probs = res[0]
        assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1])   # kernels bit-identical
        r = _oracle(logits, hist, proc, eos_min, sup, temperature=T, top_p=top_p, top_k=top_k, min_p=min_p)
        u = so.uniform(params.seed, steps, list(range(B)))
        checked = 0
        for b in range(B):
            # rows with a token at the top-p / min-p boundary (within the fp32 chain's error) may keep it either way
            edge = np.abs(r["min_p_rel"][b] - min_p) < 1e-5 * max(min_p, 1e-30)
            if r["mass_below"] is not None:
                edge |= np.abs(r["mass_below"][b] - so.top_p_limit(top_p)) < 2e-6
            if edge[r["softmax"][b] > 0].any():
                continue
            assert np.array_equal(probs[b] > 0, r["kept"][b]), b
            np.testing.assert_allclose(probs[b], r["probs"][b], atol=1e-6, rtol=0)
            cdf = np.cumsum(r["probs"][b])
            if np.min(np.abs(cdf[r["kept"][b]] - u[b])) > 4e-6:     # the fp32 prefix sums put u on the same side
                assert tok[b] == so.draw(r["probs"][b:b + 1], u[b])[0], b
            checked += 1
        assert checked >= max(1, B // 2)
        # greedy: lowest index of the maximum of the processed scores
        g = _params(do_sample=False)
        gt, _ = dbg_proc(lg, g, proc, hist, eos_min, sup, steps, 0, max_len)
        s = po.processed_logits(logits, hist, penalty=proc["repetition_penalty"], ngram=proc["no_repeat_ngram_size"],
                                ban_ids=proc["ban_ids"], begin_ids=proc["begin_ids"], words=proc["words"],
                                eos=proc["eos_token_id"], eos_min_len=eos_min, suppress=sup)
        assert np.array_equal(gt, s.argmax(axis=1))


@pytest.mark.parametrize("V", [264, 32256, 128256])
def test_neutral_processors_equal_plain_sampler(V):
    rng = np.random.default_rng(1 + V)
    B = 7
    logits = torch.tensor(rng.normal(0, 3, size=(B, V)).astype(np.float32), device="cuda")
    hist = [rng.integers(0, V, size=40).tolist() for _ in range(B)]
    proc = dict(repetition_penalty=1.0, no_repeat_ngram_size=0, min_p=0.0, eos_token_id=-1)
    sup, steps = [1, 0, 1, 0, 0, 1, 0], list(range(B))
    for params in (_params(0.7, 0.9, 20, bad_token=3, bs_token=5, seed=9), _params(do_sample=False, bad_token=3, bs_token=5)):
        for impl in (0, 1):
            a = dbg_proc(logits, params, proc, hist, [0] * B, sup, steps, impl, 64)
            b = dbg_plain(logits, params, sup, steps, impl)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


# ---------------------------------------------------------------- generation loop
_ENGINES = {}


def _engine(max_len=None):
    key = max_len
    if key not in _ENGINES:
        from detikzify_b200.engine import Engine, pack_arena
        from detikzify_b200.model.configuration import preset
        from detikzify_b200.model.weights import random_init
        cfg = preset("tiny")
        _ENGINES[key] = (cfg, Engine(cfg, pack_arena(cfg, random_init(cfg, seed=0)), device=0, max_seqs=8, max_batch=8,
                                     max_len=max_len))
    return _ENGINES[key]


def _pixels(cfg, seed=1000):
    g = torch.Generator().manual_seed(seed)
    S = cfg.vision_config.image_size
    return torch.rand(1, 3, S, S, generator=g) * 2 - 1


def _prompt(cfg, n_text, seed):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, 12, (n_text,), generator=g)
    return torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), text]).long()


def _loop_vs_stepwise(cfg, eng, B, impl, do_sample, n_text, steps):
    eng.set_option("decode_impl", impl)
    img = eng.image_embeds(_pixels(cfg).cuda())[0]
    prompts = [_prompt(cfg, n_text[i], 4000 + i) for i in range(B)]
    T0 = [p.numel() for p in prompts]
    ml = eng.max_len
    params = eng.sampling(temperature=1.5, top_p=0.98, do_sample=do_sample, seed=(0xC0FFEE << 32) | 77)
    proc = dict(repetition_penalty=1.4, no_repeat_ngram_size=2, min_p=0.01 if do_sample else 0.0,
                eos_token_id=cfg.eos_token_id, ban_ids=[cfg.image_token_id], begin_ids=[cfg.eos_token_id], words=[[3, 4]])
    eos_min = [t + 6 for t in T0]
    seq_ids = list(range(B))
    slots = [eng.seq_alloc() for _ in range(B)]
    try:
        last = torch.stack([eng.prefill(s, p.cuda(), 0, img, 0)[0] for s, p in zip(slots, prompts)])
        hist = [p.tolist() for p in prompts]
        eng.set_processors(proc, hist, eos_min)
        first, _ = eng.sample(last, params, suppress=[1] * B, steps=[0] * B, seq_ids=seq_ids)
        toks = [first.cpu().tolist()]
        for n in range(1, steps + 1):       # host-kept histories, clamped at max_len as the device clamps them
            hist = [(h + [t])[:ml] for h, t in zip(hist, toks[-1])]
            eng.set_processors(proc, hist, eos_min)
            lg = eng.decode(slots, [min(t + n - 1, ml - 1) for t in T0], torch.tensor(toks[-1], device="cuda"))
            nxt, _ = eng.sample(lg, params, suppress=[0] * B, steps=[n] * B, seq_ids=seq_ids)
            toks.append(nxt.cpu().tolist())
        for s, p in zip(slots, prompts):
            eng.prefill(s, p.cuda(), 0, img, 0)
        eng.set_processors(proc, [(p.tolist() + [t])[:ml] for p, t in zip(prompts, toks[0])], eos_min)
        eng.gen_begin(slots, T0, toks[0], params, seq_ids=seq_ids)
        got = [toks[0]]
        eng.gen_step()
        for i in range(steps):
            if i + 1 < steps:
                eng.gen_step()
            got.append(eng.gen_wait(i))
        eng.gen_end()
    finally:
        eng.set_processors(None)
        for s in slots:
            eng.seq_free(s)
        eng.set_option("decode_impl", 1)
    return got, toks


@pytest.mark.parametrize("B,impl,do_sample", [(1, 1, False), (1, 1, True), (1, 0, True), (2, 1, True), (5, 1, False),
                                              (5, 1, True)],
                         ids=["B1-persistent-greedy", "B1-persistent-sample", "B1-graph-sample", "B2", "B5-gemm-greedy",
                              "B5-gemm-sample"])
def test_generation_loop_with_processors_equals_stepwise(B, impl, do_sample):
    cfg, eng = _engine()
    got, toks = _loop_vs_stepwise(cfg, eng, B, impl, do_sample, [5 + 3 * i for i in range(B)], 24)
    assert got == toks
    for b in range(B):        # no repeated 2-gram among the new tokens (the histories hold them)
        seq = [t[b] for t in toks]
        grams = list(zip(seq, seq[1:]))
        assert len(grams) == len(set(grams)), b


def test_finished_rows_stay_inside_their_history():
    """Row 0's prompt nearly fills max_len, so its history reaches the end long before the loop ends and the sampler keeps
    appending to a full row: rows 1 and 2, whose n-gram bans read their own histories right after row 0's, must still draw
    exactly the stepwise tokens."""
    cfg, eng = _engine(max_len=128)
    n0 = 128 - cfg.num_patches - 4
    got, toks = _loop_vs_stepwise(cfg, eng, 3, 1, True, [n0, 6, 9], 30)
    assert [g[1:] for g in got] == [t[1:] for t in toks]


# ---------------------------------------------------------------- end to end against HF generate
def _hf_generate(oracle, ids, pix, max_length, **kw):
    img = oracle.image_embeds(pix)
    embeds = oracle.spliced_embeds(ids, img)
    return oracle.llm.generate(input_ids=ids, inputs_embeds=embeds, max_length=max_length,
                               pad_token_id=oracle.cfg["pad_token_id"], do_sample=False, **kw)[0]


def _check_parity(oracle, got, ref, T0, pix, tol=6e-2):
    """Equal ids wherever the oracle's top-1 margin of the processed scores allows (the rule of the parity tests)."""
    n = min(got.numel(), ref.numel())
    diff = (got[:n] != ref[:n]).nonzero()
    if diff.numel() == 0:
        assert got.numel() == ref.numel()
        return
    t = int(diff[0])
    assert t >= T0
    logits, _ = oracle.forward_logits(ref[None, :t], pix)
    top2 = logits[0, -1].topk(2).values
    assert (top2[0] - top2[1]).item() < tol, (t, top2)


def test_generate_with_processors_matches_hf():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny")
    model = DetikzifyForCausalLM(cfg, engine=engine_for("tiny"))
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=11)
    ids = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.tensor([5, 6, 7, 5, 6])]).long()[None]
    T0 = ids.shape[1]
    a, b = 6, 7
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, bad_words_ids=[[cfg.image_token_id], [a, b]], min_new_tokens=6,
              begin_suppress_tokens=[cfg.eos_token_id])
    got = model.generate(input_ids=ids, pixel_values=pix, max_length=T0 + 40, do_sample=False, **kw)[0].cpu()
    ref = _hf_generate(oracle, ids, pix, T0 + 40, **kw)
    _check_parity(oracle, got, ref, T0, pix)
    new, seq = got[T0:].tolist(), got.tolist()
    for t in range(T0, len(seq)):       # no 3-gram ending in a new token occurred before it (HF input_ids = prompt + new)
        assert tuple(seq[t - 2:t + 1]) not in {tuple(seq[i:i + 3]) for i in range(t - 2)}, t
    assert cfg.eos_token_id not in new[:6]
    assert all(not (seq[t - 1] == a and seq[t] == b) for t in range(T0, len(seq)))


def test_generate_batch_with_processors_shared_prefix():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny")
    model = DetikzifyForCausalLM(cfg, engine=engine_for("tiny", max_seqs=8, max_batch=4), max_seqs=8, max_batch=4)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=12)
    head = [cfg.patch_token_id] * cfg.num_patches + [9, 10, 11, 12, 13, 14, 15, 16]
    prompts = [torch.tensor(head + tail) for tail in ([1, 2], [3], [4, 5, 6])]
    kw = dict(repetition_penalty=1.25, no_repeat_ngram_size=2, bad_words_ids=[[cfg.image_token_id], [1, 2]],
              begin_suppress_tokens=[cfg.eos_token_id], suppress_tokens=[0])
    outs = model.generate_batch(prompts, pix, max_new_tokens=20, do_sample=False, **kw)
    for p, o in zip(prompts, outs):
        ref = _hf_generate(oracle, p[None], pix, p.numel() + 20, **kw)
        _check_parity(oracle, o.cpu(), ref, p.numel(), pix)
        assert 0 not in o[p.numel():].tolist()
