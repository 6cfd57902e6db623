"""
Both sampler kernels (sample.cu: the register-resident kernel for V <= 32768 and the generic kernel) held to the fp64
restatement in oracle/sample_oracle.py through the engine-free hook ``dtk_dbg_sample``, at the vocabulary sizes of the
checkpoints and at the kernels' dispatch edge (32768 is the last V of the register-resident kernel, 32769 the first of the
generic one), and the fused generation loop held to stepwise sampling.

Per draw:
  (a) the kept set equals the reference's. Two exceptions only. One is a token whose ascending mass is within 1e-6 of the
      top-p limit once every probability may carry the relative error of the kernel's fp32 chain (x / T, x - max, the exp2
      argument and exp2 itself: eps_i = 2^-22 (|s_i| + |max| + 2 |s_i - max| + 2) for the score s_i = x_i / T). Near-equal
      probabilities may then sort either way, so the mass at or below the token lies anywhere between the mass strictly below
      p_i (1 - 2 eps_i) and the mass at or below p_i (1 + 2 eps_i). The other is a token whose exp(score - max) is below
      2^-125, which the kernel's fp32 exp flushes to zero. Kept probabilities agree to 1e-6 absolute (against the reference
      renormalised over the kernel's kept set).
  (b) the token is the inverse-CDF draw of the restated uniform, summed in fp64 over the kernel's own returned vector.
      The kernel sums in fp32: a chunk of ceil(V/1024) entries per thread, two 32-wide scans over the chunk sums, then a
      walk through the chunk that holds u. Every boundary it compares u against is therefore off its fp64 value by that
      summation's rounding. delta at a boundary = |that boundary summed in fp32 in the kernel's order (sample_oracle.
      kernel_prefix_sums) - the same boundary in fp64| + 2^-24; a draw whose u lies within delta of a boundary is
      skipped, and fewer than 5 % of the draws at each V may be. Where u is within delta of the vector's total the kernel
      may return its argmax fallback instead.
  (c) both kernels give bit-identical tokens and vectors wherever both can run.
  (d) greedy returns the lowest index among tied maxima of the masked logits.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import sample_oracle as so

pytestmark = pytest.mark.gpu

REG_MAX_V = 32768                  # ST * VPT: the register-resident kernel's largest vocabulary
VOCABS = [264, 32000, 32256, 32767, 32768, 32769, 128256]
GRID = [(t, p, k) for t in (0.3, 0.8, 2.5) for p in (1.0, 0.95, 0.5, 1e-3) for k in (0, 1, 50, "V")]
BATCHES = (64, 7, 1, 7, 1, 7)     # B of successive grid points (the fp64 reference's CPU time grows with the rows)
KINDS = ("gauss", "peaked", "gauss", "flat", "gauss", "tied_max", "five", "bad_at_max", "bs_at_max")
EDGE_TOL = 1e-6                    # ascending mass this close to the top-p limit may fall on either side
VALUE_TOL = 1e-6
UNDERFLOW = 2.0**-125              # exp(score - max) below this may be flushed to zero by the fp32 exp
MARGIN = 2.0**-24                  # added to the per-boundary fp32 summation error
MAX_SKIPPED = 0.05


def _lib():
    from detikzify_b200 import _lib as L
    return L.load_library()


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _params(temperature, top_p, top_k, do_sample=True, bad_token=-1, bs_token=-1, seed=0):
    from detikzify_b200.engine import Engine
    return Engine.sampling(temperature=temperature, top_p=top_p, top_k=top_k, do_sample=do_sample, bad_token=bad_token,
                           begin_suppress_token=bs_token, seed=seed)


def dbg_sample(logits, params, suppress, steps, seq_ids, impl, probs=None):
    """dtk_dbg_sample on a device fp32 [B, V] tensor -> (tokens int64 [B], probability vectors fp32 [B, V]) on the device."""
    B, V = logits.shape
    out = torch.full((B,), -7, dtype=torch.int64, device=logits.device)
    if probs is None:
        probs = torch.full((B, V), float("nan"), device=logits.device)
    rc = _lib().dtk_dbg_sample(_p(logits), B, V, C.byref(params), (C.c_int * B)(*suppress), (C.c_uint32 * B)(*steps),
                               (C.c_uint32 * B)(*seq_ids), impl, _p(out), _p(probs),
                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, rc
    return out, probs


def _impls(V):
    return (0, 1) if V <= REG_MAX_V else (1,)


def make_rows(V, B, rng, kind_offset, bad, bs):
    """fp32 [B, V] logits cycling through the row kinds, and the per-row begin-suppress flags."""
    rows = np.empty((B, V), dtype=np.float32)
    kinds = []
    for r in range(B):
        kind = KINDS[(r + kind_offset) % len(KINDS)]
        kinds.append(kind)
        x = rng.standard_normal(V) * 3
        if kind == "peaked":             # one token at p ~ 0.999 at T = 1
            x = rng.standard_normal(V)
            x[rng.integers(V)] = np.log(999.0) + np.log(np.exp(x).sum())
        elif kind == "flat":
            x = np.full(V, 0.75)
        elif kind == "tied_max":
            i, j = rng.choice(V, 2, replace=False)
            x[[i, j]] = x.max() + 1.0
        elif kind == "five":             # -inf outside five tokens
            keep = rng.choice(V, 5, replace=False)
            y = np.full(V, -np.inf)
            y[keep] = rng.standard_normal(5) * 2
            x = y
        elif kind == "bad_at_max":
            x[bad] = x.max() + 4.0
        elif kind == "bs_at_max":
            x[bs] = x.max() + 4.0
        rows[r] = x
    suppress = [int(r % 3 == 0) for r in range(B)]      # the begin-suppress mask applies on some rows only
    return rows, suppress, kinds


def _top_p_edge(sm, i, s, limit):
    """Whether fp32 rounding may put token i on either side of the top-p limit: sm = the fp64 softmax row (after top-k),
    s = the fp64 scores x / T of the row."""
    m = s[np.isfinite(s)].max()
    eps = 2.0**-22 * (abs(s[i]) + abs(m) + 2 * abs(s[i] - m) + 2)
    ps = np.sort(sm)
    cs = np.concatenate([[0.0], np.cumsum(ps)])
    lo = cs[np.searchsorted(ps, sm[i] * (1 - 2 * eps), side="left")]     # mass strictly below the band
    hi = cs[np.searchsorted(ps, sm[i] * (1 + 2 * eps), side="right")]    # mass at or below the band's top
    return lo - EDGE_TOL <= limit <= hi + EDGE_TOL


def _check_draws(V, ci, T, top_p, top_k, rng, stats):
    B = BATCHES[ci % len(BATCHES)]
    k = V if top_k == "V" else top_k
    bad, bs = int(rng.integers(V)), int(rng.integers(V))
    while bs == bad:
        bs = int(rng.integers(V))
    rows, suppress, kinds = make_rows(V, B, rng, ci, bad, bs)
    seed = (0x9E3779B9 << 32) | (0x7F4A7C15 + 977 * ci)        # both seed words matter
    seq_ids = [int(s) for s in rng.integers(0, 2**32, B)]
    steps = [(2**32 - 1 - r) if r % 2 == 0 else int(rng.integers(0, 2**32)) for r in range(B)]   # the top of the counter range
    params = _params(T, top_p, k, bad_token=bad, bs_token=bs, seed=seed)
    dev = torch.from_numpy(rows).cuda()
    res = [dbg_sample(dev, params, suppress, steps, seq_ids, impl) for impl in _impls(V)]
    toks = res[0][0].cpu().numpy()
    got = res[0][1].cpu().numpy()
    for t2, p2 in res[1:]:      # (c) both kernels, bit for bit
        assert torch.equal(t2, res[0][0]) and torch.equal(p2, res[0][1]), (V, T, top_p, k)

    ref = so.processed_probs(rows, T, top_p, k, bad_token=bad, begin_suppress_token=bs, suppress=np.array(suppress, bool))
    kept_got = got > 0
    # (a) kept set
    mism = ref["kept"] != kept_got
    allowed = ref["kept"] & ~kept_got & (ref["rel"] < UNDERFLOW)
    if top_p < 1:
        for r, i in zip(*np.nonzero(mism & ~allowed)):
            allowed[r, i] = _top_p_edge(ref["softmax"][r], i, rows[r].astype(np.float64) / T, so.top_p_limit(top_p))
    bad_rows = np.flatnonzero((mism & ~allowed).any(axis=1))
    assert bad_rows.size == 0, (V, T, top_p, k, [(int(r), kinds[r], np.flatnonzero(mism[r] & ~allowed[r])[:8].tolist())
                                                  for r in bad_rows[:4]])
    stats["edge"] += int((mism & allowed).any(axis=1).sum())
    # (a) kept values, against the reference renormalised over the kernel's kept set
    alt = np.where(kept_got, ref["softmax"], 0.0)
    alt /= alt.sum(axis=1, keepdims=True)
    err = np.abs(got.astype(np.float64) - alt).max(axis=1)
    assert (err <= VALUE_TOL).all(), (V, T, top_p, k, float(err.max()), kinds[int(err.argmax())])
    stats["max_value_err"] = max(stats["max_value_err"], float(err.max()))
    # (b) the token against the fp64 inverse-CDF draw of the restated uniform over the kernel's vector
    u = so.uniform(seed, steps, seq_ids)
    want = so.draw(got, u)
    argmax = so.greedy(rows, bad, bs, np.array(suppress, bool))
    for r in range(B):
        b64, b32 = so.kernel_prefix_sums(got[r])
        delta = np.abs(b32 - b64) + MARGIN
        stats["draws"] += 1
        stats["max_delta"] = max(stats["max_delta"], float(delta.max()))
        if (np.abs(u[r] - b64) <= delta).any():
            stats["skipped"] += 1
            continue
        ok = {int(want[r])}
        if u[r] >= got[r].astype(np.float64).sum() - delta.max():
            ok.add(int(argmax[r]))             # the kernel's fallback when rounding leaves u beyond the total
        assert int(toks[r]) in ok, (V, T, top_p, k, r, kinds[r], int(toks[r]), ok, float(u[r]))
        assert kept_got[r, toks[r]]


@pytest.mark.parametrize("V", VOCABS)
def test_sampler_draws_match_fp64_reference(V):
    rng = np.random.default_rng(V)
    stats = dict(draws=0, skipped=0, edge=0, max_delta=0.0, max_value_err=0.0)
    for ci, (T, top_p, top_k) in enumerate(GRID):
        _check_draws(V, ci, T, top_p, top_k, rng, stats)
    frac = stats["skipped"] / stats["draws"]
    print(f"\nsampler V={V} kernels={_impls(V)}: {stats['draws']} draws, {stats['skipped']} skipped ({100 * frac:.2f} %), "
          f"max delta {stats['max_delta']:.3g}, rows with a top-p edge token {stats['edge']}, "
          f"max kept-value error {stats['max_value_err']:.3g}")
    assert frac < MAX_SKIPPED, stats


@pytest.mark.parametrize("V", VOCABS)
def test_greedy_returns_lowest_tied_index(V):
    """Ties inside one thread's strided range (i, i + 1024), across lanes (i, i + 1) and across warps; the bad and
    begin-suppress masks removing the lower tied token; an all-equal row; greedy by do_sample = 0 and by T < 1e-5."""
    rng = np.random.default_rng(V + 1)
    B = 8
    rows = (rng.standard_normal((B, V)) * 3).astype(np.float32)
    i = int(rng.integers(0, max(1, V - 1025)))
    pairs = [(i, i + 1024), (i, i + 1), (3, V - 1), (V // 2, V // 2 + 32)]
    for r, (a, b) in enumerate(pairs):
        a, b = min(a, V - 1), min(b, V - 1)
        rows[r, [a, b]] = rows[r].max() + 2.0
    rows[4] = 0.25                                           # all equal: token 0
    a, b = V // 3, V // 3 + 1024 if V // 3 + 1024 < V else V - 1
    rows[5, [a, b]] = rows[5].max() + 2.0                    # the bad token removes the lower tied index
    bad = a
    rows[6, [a + 1, b]] = rows[6].max() + 3.0                # three-way tie, lowest masked by the begin-suppress token
    rows[6, 0] = rows[6, b]
    bs = 0
    rows[7, [1, 2]] = rows[7].max() + 1.0
    suppress = [0, 0, 0, 0, 0, 0, 1, 1]
    want = so.greedy(rows, bad, bs, np.array(suppress, bool))
    dev = torch.from_numpy(rows).cuda()
    for do_sample, T in ((False, 0.8), (True, 5e-6)):
        params = _params(T, 0.95, 0, do_sample=do_sample, bad_token=bad, bs_token=bs, seed=3 << 40)
        for impl in _impls(V):
            out, _ = dbg_sample(dev, params, suppress, [0] * B, list(range(B)), impl)
            assert out.cpu().tolist() == want.tolist(), (V, impl, do_sample)


def test_generic_kernel_distribution_at_128k():
    """12 800 draws (64 rows x 200 steps) of the generic kernel at V = 128256 over a nucleus of about 20 tokens, G-test
    against the fp64 vector over the tokens with p > 1e-4 (the rest pooled in one bin)."""
    from scipy.stats import power_divergence
    V, rows, n_steps = 128256, 64, 200
    rng = np.random.default_rng(128256)
    x = rng.standard_normal(V)
    top = rng.choice(V, 24, replace=False)
    x[top] = 14.0 + rng.standard_normal(24) * 0.7
    logits = torch.from_numpy(np.tile(x.astype(np.float32), (rows, 1))).cuda()
    T, top_p = 1.0, 0.95
    params = _params(T, top_p, 0, seed=(0xA5A5 << 32) | 99)
    ref = so.processed_probs(x.astype(np.float32)[None], T, top_p, 0)["probs"][0]
    seq_ids = [0x01000193 * (r + 1) % 2**32 for r in range(rows)]
    probs = torch.empty(rows, V, device="cuda")
    toks = []
    for s in range(n_steps):
        out, _ = dbg_sample(logits, params, [0] * rows, [s] * rows, seq_ids, 1, probs)
        toks.append(out)
    toks = torch.cat(toks).cpu().numpy()
    counts = np.bincount(toks, minlength=V)
    assert counts[probs[0].cpu().numpy() == 0].sum() == 0
    big = ref > 1e-4
    n = toks.size
    f_obs = np.append(counts[big], counts[~big].sum()).astype(np.float64)
    f_exp = np.append(ref[big], ref[~big].sum()) * n
    if f_exp[-1] == 0:
        f_obs, f_exp = f_obs[:-1], f_exp[:-1]
    g, pval = power_divergence(f_obs, f_exp, lambda_="log-likelihood")
    print(f"\nG-test at V={V}: {n} draws over {int(big.sum())} tokens with p > 1e-4 "
          f"(nucleus {int((ref > 0).sum())}), G = {g:.2f}, p = {pval:.3f}")
    assert 15 <= (ref > 0).sum() <= 25
    assert pval > 1e-3, (g, pval)


# ---------------------------------------------------------------- fused generation loop with sampling
_ENGINES = {}


def _engine(name):
    """A tiny engine with room for 8 sequences in one step. Built here rather than through conftest.engine_for, whose
    model_bundle also builds the HF oracle that these tests do not need."""
    if name not in _ENGINES:
        from detikzify_b200.engine import Engine, pack_arena
        from detikzify_b200.model.configuration import preset
        from detikzify_b200.model.weights import random_init
        cfg = preset(name)
        _ENGINES[name] = (cfg, Engine(cfg, pack_arena(cfg, random_init(cfg, seed=0)), device=0, max_seqs=8, max_batch=8))
    return _ENGINES[name]


def _pixels(cfg, seed=1000):
    g = torch.Generator().manual_seed(seed)
    S = cfg.vision_config.image_size
    return torch.rand(1, 3, S, S, generator=g) * 2 - 1


def _prompt(cfg, n_text=7, seed=2000):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(0, min(cfg.vocab_size, cfg.patch_token_id), (n_text,), generator=g)
    return torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), text]).long()


@pytest.mark.parametrize("name,B,impl", [("tiny", 1, 1), ("tiny", 1, 0), ("tiny2", 1, 1), ("tiny2", 1, 0), ("tiny", 2, 1),
                                         ("tiny", 5, 1)],
                         ids=["tiny-B1-persistent", "tiny-B1-graph", "tiny2-B1-persistent", "tiny2-B1-graph", "tiny-B2",
                              "tiny-B5-gemm"])
def test_generation_loop_equals_stepwise_sampling(name, B, impl):
    """gen_begin / gen_step / gen_wait with do_sample draw the same tokens as decode + sample one step at a time: the first
    token with RNG counter 0, the n-th after it with counter n, each sequence on its own stream (seq_id) of a 64-bit seed.
    Both sides run the same engine and decode kernels, so the logits are bit-identical and the tokens must be equal.
    B = 5 takes the batched-GEMM decode step."""
    cfg, eng = _engine(name)
    eng.set_option("decode_impl", impl)
    img = eng.image_embeds(_pixels(cfg).cuda())[0]
    prompts = [_prompt(cfg, n_text=5 + 3 * i, seed=4000 + i) for i in range(B)]
    T0 = [p.numel() for p in prompts]
    steps = min(20, cfg.model_max_length - max(T0) - 1)
    params = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id,
                          begin_suppress_token=cfg.eos_token_id, seed=(0xC0FFEE << 32) | 0x1234)
    seq_ids = [(0x9E3779B9 + 7919 * i) % 2**32 for i in range(B)]
    slots = [eng.seq_alloc() for _ in range(B)]
    try:
        last = torch.stack([eng.prefill(s, p.cuda(), 0, img, 0)[0] for s, p in zip(slots, prompts)])
        first, _ = eng.sample(last, params, suppress=[1] * B, steps=[0] * B, seq_ids=seq_ids)
        # stepwise reference on the engine itself
        toks = [first.cpu().tolist()]
        for n in range(1, steps + 1):
            lg = eng.decode(slots, [t + n - 1 for t in T0], torch.tensor(toks[-1], device="cuda"))
            nxt, _ = eng.sample(lg, params, suppress=[0] * B, steps=[n] * B, seq_ids=seq_ids)
            toks.append(nxt.cpu().tolist())
        # fused loop
        for s, p in zip(slots, prompts):
            eng.prefill(s, p.cuda(), 0, img, 0)
        eng.gen_begin(slots, T0, toks[0], params, seq_ids=seq_ids)
        got = [toks[0]]
        eng.gen_step()
        for i in range(steps):
            if i + 1 < steps:
                eng.gen_step()  # one step of lookahead
            got.append(eng.gen_wait(i))
        eng.gen_end()
    finally:
        for s in slots:
            eng.seq_free(s)
        eng.set_option("decode_impl", 1)
    assert got == toks
    assert len({tuple(t) for t in toks}) > steps // 2      # the draws do vary from step to step
