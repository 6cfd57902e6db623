"""
Prefill and scoring held layer by layer to an fp64 restatement (tests/prefill_restatement.py), each layer restated from the
engine's OWN input residual to it (dev option ``prefill_layers`` + ``dtk_dbg_residual_read``) and attending over the
engine's own bf16 KV cache (``dtk_dbg_kv_read``). A whole-stack restatement of bf16-operand GEMMs is only as tight as the
random-init decoders' layer-to-layer amplification of rounding flips allows; restated one layer at a time, the bound is set
by that layer's roundings alone.

Models (``load(..., device_init=True)``), max_len 2048:
  ds-1.3b (MHA, hd 128), tl-1.1b (GQA 32/4, hd 64), v2-8b-2l (GQA 32/8, llama3 RoPE, V 128256), ds-7b-2l (H 4096).

Cases, where the kernels change shape: full prefills of T in {1, 17, 32, 33, 63, 64, 65, 129, 1000, 2047} (GEMM tiles
below and above M = 64; ragged and exact 64-row query tiles and 64-key tiles); suffixes of T in {1, 40, 300} at start_pos
253 (a query tile straddles the cached prefix); a borrower (``seq_share`` of 253 positions: 240 lent, 13 copied) prefilling
a 40-token suffix (``split_row`` 240 inside the 192-255 key tile); ds-1.3b's 243-row image span at position 700 of 1100.
T = 2047 checks every layer, the others layers {0, 1, L/2, L - 1}.

Checks:
  * x_0 (``prefill_layers`` = 0) is the fp32 embedding row, or the given image row at a spliced position, bit for bit;
  * per layer l: |x_{l+1} - restated| <= LAMBDA * sigma_row + flip_eps at every element (sigma_row = the larger over four
    error-model draws of the RMS change of that row; flip_eps = what ambiguous roundings of the bf16 norm operands can do).
    Every new K / V row of layer l holds the restated bf16 bits except elements within eps of a rounding boundary (the
    rule of test_gpu_decode_restatement.check_rows);
  * head, from the engine's own x_L: the last row's GEMV logits, every row's GEMM logits (``dtk_prefill`` and
    ``dtk_score``), ``dtk_score``'s lse and logprob (targets include -1, 0, V - 1 and V; an out-of-range target gives
    logprob exactly 0), each against ``restate_head`` under its own error-model bound.
LAMBDA = 10: the largest of H Gaussian draws is about 4 sigma, which leaves a factor two for the model's approximations.

Negative controls run on the restatement only; collected over the module, each must exceed the bound at least once.
"""
import ctypes as C
import gc
import time

import pytest
import torch

from decode_restatement import Weights, bf16, bf16_ulp
from prefill_restatement import flip_eps, head_noise, layer_noise, restate_head, restate_layer

pytestmark = pytest.mark.gpu
LAMBDA = 10.0
FULL_T = (1, 17, 32, 33, 63, 64, 65, 129, 1000, 2047)
SUFFIX_T = (1, 40, 300)
CONTROL_T = (65, 129, 1000)
MODELS = ["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b", "v2-8b-2l", "ds-7b-2l"]
SLOTS = 4
REPORT = []
controls_hit = {}


def release_memory():
    """Return every block torch's allocator caches to the device (see test_gpu_decode_restatement.release_memory)."""
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=MODELS)
def model(request):
    from detikzify_b200.model import load
    release_memory()   # the previous parameter's arena
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=SLOTS)
    m.name = request.param
    m.engine._w64 = Weights(m.engine.cfg, m.engine.arena, m.engine.ccfg)
    yield m
    m.engine.close()
    del m
    release_memory()


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.perf_counter()
    yield
    release_memory()
    free, total = torch.cuda.mem_get_info()
    REPORT.append(f"PREFILL RESTATE module end: {time.perf_counter() - t0:.0f} s, {free / 2**30:.1f} of "
                  f"{total / 2**30:.1f} GiB free, {torch.cuda.memory_reserved() / 2**30:.2f} GiB reserved by torch")
    for line in REPORT:
        print(line)


def prompt(cfg, T, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, min(cfg.vocab_size, 30000), (T,), generator=g)
    ids[ids == cfg.image_token_id] = 2
    return ids


def kv_read(eng, slot, layer, pos0, n):
    c = eng.cfg
    k = torch.empty(c.num_key_value_heads, n, c.head_dim, dtype=torch.bfloat16, device=eng.device)
    v = torch.empty_like(k)
    rc = eng.lib.dtk_dbg_kv_read(eng._h, slot, layer, pos0, n, C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                 eng._stream())
    assert rc == 0, eng.lib.dtk_last_error(eng._h).decode()
    return k, v


def residual(eng, T):
    out = torch.empty(T, eng.cfg.hidden_size, dtype=torch.float32, device=eng.device)
    rc = eng.lib.dtk_dbg_residual_read(eng._h, 0, T, C.c_void_p(out.data_ptr()), eng._stream())
    assert rc == 0, eng.lib.dtk_last_error(eng._h).decode()
    torch.cuda.synchronize()
    return out


def run(eng, slot, ids, start, n_layers, img=None, img_start=0):
    """The residual stream after the first n_layers layers of a prefill (n_layers = -1: every layer)."""
    eng.set_option("prefill_layers", n_layers)
    try:
        eng.prefill(slot, ids.cuda(), start, img, img_start)
    finally:
        eng.set_option("prefill_layers", -1)
    return residual(eng, ids.numel())


def pair_norm(t):
    return torch.sqrt(t * t + t.roll(t.shape[-1] // 2, -1) ** 2)


def check_rows(tag, got, pre, sig, kv_eps):
    """got [T, kv_heads, hd] bf16 read back, pre the restated rows before rounding (rule of the decode test)."""
    want = bf16(pre)
    got = got.double()
    eps = LAMBDA * sig[:, :, None] + kv_eps + 2.0 ** -20 * pair_norm(pre)
    bad = (got != want) & ((got - pre).abs() > bf16_ulp(want) / 2 + eps)
    i = bad.nonzero()[:3].tolist()
    assert not bad.any(), (tag, int(bad.sum()), [(j, float(pre[tuple(j)]), float(want[tuple(j)]), float(got[tuple(j)]),
                                                   float(eps[tuple(j)])) for j in i])
    return int((got != want).sum())


def _controls(cfg, T, start):
    c = {"causal mask + 1": dict(causal_shift=1), "causal mask - 1": dict(causal_shift=-1),
         "RoPE at pos + 1": dict(rope_shift=1), "fp32 q": dict(fp32_q=True), "fp32 attention output": dict(fp32_att=True),
         "fp32 SwiGLU output": dict(fp32_swiglu=True)}
    if start + T > 64:
        c["key 64 dropped"] = dict(drop_key=64)
    if 1 < cfg.num_key_value_heads < cfg.num_attention_heads:
        c["GQA h % kv_heads"] = dict(gqa_mod=True)
    return c


def control_names(cfg):
    return list(_controls(cfg, 2047, 0))


def check_layer(model, tag, slot, ids, start, l, img=None, img_start=0, controls=None, x_in=None, subst=None):
    """Layer l of a prefill of ids at start: x_l and x_{l+1} from two runs, layer l's cache rows [0, start + T) after the
    second. ``x_in``: replaces x_l in extra (control) restatements; ``subst(K, V)``: replaces the cache read there.
    Returns {control name: exceeded}."""
    eng, cfg, w = model.engine, model.config, model.engine._w64
    T = ids.numel()
    x_l = run(eng, slot, ids, start, l, img, img_start).double()
    x_n = run(eng, slot, ids, start, l + 1, img, img_start).double()
    K, V = kv_read(eng, slot, l, 0, start + T)
    K, V = K.double(), V.double()

    def kv(ll, n):
        assert ll == l and n == start + T
        return K, V
    ref = restate_layer(w, l, x_l, start, kv, "prefill")
    sig = layer_noise(w, l, x_l, start, kv, "prefill", ref)
    x_eps = flip_eps(w, l, x_l, start, kv, ref)
    bound = LAMBDA * sig["x"][:, None] + x_eps
    err = (x_n - ref["x"]).abs()
    ratio = (err / bound).amax(-1)
    rms = x_n.pow(2).mean(-1).sqrt()
    worst = ratio.max().item()
    REPORT.append(f"PREFILL RESTATE {tag} L{l}: x worst err/bound {worst:.3f}, bound/RMS "
                  f"{(LAMBDA * sig['x'] / rms).max().item():.2e}, flip_eps/RMS {(x_eps.amax(-1) / rms).max().item():.2e}")
    assert torch.isfinite(x_n).all(), tag
    assert worst <= 1.0, (tag, l, worst, int(ratio.argmax()))
    Kn, Vn = K[:, start:].transpose(0, 1), V[:, start:].transpose(0, 1)
    check_rows((tag, l, "k"), Kn, ref["k"], sig["k"], ref["kv_eps"][0])
    check_rows((tag, l, "v"), Vn, ref["v"], sig["v"], ref["kv_eps"][1])
    hit = {}
    for name, kw in (controls or {}).items():
        xi = x_in if x_in is not None else x_l
        kvc = kv if subst is None else (lambda ll, n: subst(K, V))
        r = restate_layer(w, l, xi, start, kvc, "prefill", **kw)
        hit[name] = bool((~((x_n - r["x"]).abs() <= bound)).any())
        key = (model.name, name)
        controls_hit[key] = controls_hit.get(key, False) or hit[name]
        del r
    return hit


def check_head(model, tag, slot, ids, start, img=None, img_start=0):
    """Last-row GEMV and all-row GEMM logits of dtk_prefill, then dtk_score's logits, lse and logprob, each from the x_L
    the call left."""
    eng, cfg, w = model.engine, model.config, model.engine._w64
    T, V = ids.numel(), cfg.vocab_size
    last, alll = eng.prefill(slot, ids.cuda(), start, img, img_start, want_all_logits=True)
    x = residual(eng, T).double()
    ref = restate_head(w, x, "prefill")
    sig = head_noise(w, x, "prefill", ref)
    rms = ref["logits"].pow(2).mean(-1).sqrt()
    b_last = LAMBDA * sig["last_logits"]
    r_last = ((last.double() - ref["last_logits"]).abs().max() / b_last).item()
    b_all = LAMBDA * sig["logits"][:, None] + ref["logits_eps"]
    r_all = ((alll.double() - ref["logits"]).abs() / b_all).amax(-1).max().item()
    REPORT.append(f"PREFILL RESTATE {tag} head: last worst err/bound {r_last:.3f} (bound/RMS "
                  f"{(b_last / rms[-1]).item():.2e}), all worst err/bound {r_all:.3f} (bound/RMS "
                  f"{(LAMBDA * sig['logits'] / rms).max().item():.2e})")
    assert torch.isfinite(last).all() and torch.isfinite(alll).all(), tag
    assert r_last <= 1.0, (tag, "last", r_last)
    assert r_all <= 1.0, (tag, "all", r_all)
    del alll

    g = torch.Generator().manual_seed(T + start)
    targets = torch.randint(0, V, (T,), generator=g)
    for i, t in enumerate([-1, 0, V - 1, V][:T]):   # no target, both ends of the vocabulary, past its end
        targets[i] = t
    logprob, lse, slog = eng.score(slot, ids.cuda(), start, img, img_start, targets.cuda(), want_all_logits=True)
    x = residual(eng, T).double()
    ref = restate_head(w, x, "prefill")
    valid = (targets >= 0) & (targets < V)
    tv = targets.clamp(0, V - 1).cuda()
    sig = head_noise(w, x, "prefill", ref, tv)
    rows = torch.arange(T, device="cuda")
    eps_max = ref["logits_eps"].amax(-1)
    b_all = LAMBDA * sig["logits"][:, None] + ref["logits_eps"]
    r_all = ((slog.double() - ref["logits"]).abs() / b_all).amax(-1).max().item()
    b_lse = LAMBDA * sig["lse"] + eps_max
    r_lse = ((lse.double() - ref["lse"]).abs() / b_lse).max().item()
    lp_ref = ref["logits"][rows, tv] - ref["lse"]
    b_lp = LAMBDA * sig["logprob"] + ref["logits_eps"][rows, tv] + eps_max
    vc = valid.cuda()
    r_lp = ((logprob.double() - lp_ref).abs() / b_lp)[vc].max().item() if bool(vc.any()) else 0.0
    REPORT.append(f"PREFILL RESTATE {tag} score: logits worst err/bound {r_all:.3f}, lse {r_lse:.3f} (bound "
                  f"{b_lse.max().item():.2e}), logprob {r_lp:.3f} (bound {b_lp.max().item():.2e})")
    assert r_all <= 1.0, (tag, "score logits", r_all)
    assert r_lse <= 1.0, (tag, "lse", r_lse)
    assert r_lp <= 1.0, (tag, "logprob", r_lp)
    assert (logprob[~vc] == 0).all(), (tag, logprob[~vc])


def _layers(L, T):
    return list(range(L)) if T == 2047 else sorted({0, 1, L // 2, L - 1})


def test_option_and_residual_read_reject_bad_arguments(model):
    eng = model.engine
    L, ml = eng.cfg.num_hidden_layers, eng.max_len
    assert eng.get_option("prefill_layers") == -1
    buf = torch.empty(2, eng.cfg.hidden_size, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    try:
        for v in (-2, L + 1, 1 << 40):
            assert eng.lib.dtk_set_option(eng._h, b"prefill_layers", v) == -1, v
            assert eng.get_option("prefill_layers") == -1
        for v in (0, L, -1):
            eng.set_option("prefill_layers", v)
            assert eng.get_option("prefill_layers") == v
        for args in [(-1, 1), (0, -1), (ml, 1), (ml - 1, 2), (0, ml + 1)]:
            assert eng.lib.dtk_dbg_residual_read(eng._h, *args, p, None) == -1, args
        assert eng.lib.dtk_dbg_residual_read(eng._h, 0, 1, None, None) == -1
        assert eng.lib.dtk_dbg_residual_read(eng._h, ml - 2, 2, p, None) == 0
        torch.cuda.synchronize()
    finally:
        eng.set_option("prefill_layers", -1)


def test_x0_is_the_embedding(model):
    """prefill_layers = 0: every row is the fp32 embedding row, or the image row at a spliced position (ds-1.3b: a
    243-row span at 700 of 1100)."""
    eng, cfg, w = model.engine, model.config, model.engine._w64
    T, img, start = 1100, None, 700
    ids = prompt(cfg, T, 3)
    if model.name.endswith("ds-1.3b"):
        ids[start:start + cfg.num_patches] = cfg.image_token_id
        img = torch.randn(cfg.num_patches, cfg.hidden_size, generator=torch.Generator().manual_seed(4)).cuda() * 0.05
    slot = eng.seq_alloc()
    try:
        x = run(eng, slot, ids, 0, 0, img, start)
        want = w("dec.embed")[ids.cuda()].float()
        if img is not None:
            want[start:start + img.shape[0]] = img
        assert torch.equal(x, want)
    finally:
        eng.seq_free(slot)


@pytest.mark.parametrize("T", FULL_T)
def test_full_prefill(model, T):
    eng, cfg = model.engine, model.config
    ids = prompt(cfg, T, 100 + T)
    slot = eng.seq_alloc()
    try:
        tag = f"{model.name} full T={T}"
        for l in _layers(cfg.num_hidden_layers, T):
            check_layer(model, tag, slot, ids, 0, l, controls=_controls(cfg, T, 0) if T in CONTROL_T else None)
        check_head(model, tag, slot, ids, 0)
    finally:
        eng.seq_free(slot)


@pytest.mark.parametrize("T", SUFFIX_T)
def test_suffix_prefill(model, T):
    """253 cached positions, then T more: q_pos0 = 253 is not a multiple of 64, so a query tile straddles the prefix."""
    eng, cfg = model.engine, model.config
    pre, suf = prompt(cfg, 253, 7), prompt(cfg, T, 200 + T)
    slot = eng.seq_alloc()
    try:
        eng.prefill(slot, pre.cuda(), 0, None, 0)
        tag = f"{model.name} suffix 253+{T}"
        for l in _layers(cfg.num_hidden_layers, T):
            check_layer(model, tag, slot, suf, 253, l, controls=_controls(cfg, T, 253) if T == 40 else None)
        check_head(model, tag, slot, suf, 253)
    finally:
        eng.seq_free(slot)


def test_borrower_prefill(model):
    """seq_share(base, sub, 253): 240 positions lent (split_row 240 inside the 192-255 key tile), 13 copied; then a
    40-token suffix. The control reads the lent positions from the borrower's own slot, which holds another prompt."""
    eng, cfg = model.engine, model.config
    pre, own, suf = prompt(cfg, 253, 31), prompt(cfg, 253, 32), prompt(cfg, 40, 33)
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    try:
        eng.prefill(base, pre.cuda(), 0, None, 0)
        eng.prefill(sub, own.cuda(), 0, None, 0)
        own_rows = [[t.double() for t in kv_read(eng, sub, l, 0, 240)] for l in range(cfg.num_hidden_layers)]
        eng.seq_share(base, sub, 253)
        tag = f"{model.name} borrower 253+40"
        hit = False
        for l in _layers(cfg.num_hidden_layers, 40):
            def own_slot(K, V, l=l):
                K, V = K.clone(), V.clone()
                K[:, :240], V[:, :240] = own_rows[l]
                return K, V
            hit |= check_layer(model, tag, sub, suf, 253, l, controls={"lent rows from the own slot": {}},
                               subst=own_slot)["lent rows from the own slot"]
        check_head(model, tag, sub, suf, 253)
        assert hit
    finally:
        eng.seq_free(sub)
        eng.seq_free(base)


def test_image_span_prefill(model):
    """ds-1.3b: a 243-row image span at position 700 of a 1100-token prompt. The control restates layer 0 from the
    embedding rows of the image token instead of the image rows."""
    if not model.name.endswith("ds-1.3b"):
        pytest.skip("the image span case runs on ds-1.3b")
    eng, cfg, w = model.engine, model.config, model.engine._w64
    T, start, n = 1100, 700, cfg.num_patches
    ids = prompt(cfg, T, 41)
    ids[start:start + n] = cfg.image_token_id
    img = torch.randn(n, cfg.hidden_size, generator=torch.Generator().manual_seed(42)).cuda() * 0.05
    slot = eng.seq_alloc()
    try:
        tag = f"{model.name} image span 700+243 T=1100"
        unspliced = w("dec.embed")[ids.cuda()].clone()
        for l in _layers(cfg.num_hidden_layers, T):
            hit = check_layer(model, tag, slot, ids, 0, l, img, start,
                              controls={"image rows not spliced": {}} if l == 0 else None, x_in=unspliced)
            if l == 0:
                assert hit["image rows not spliced"]
        check_head(model, tag, slot, ids, 0, img, start)
    finally:
        eng.seq_free(slot)


ROUNDING_CONTROLS = ("fp32 q", "fp32 attention output", "fp32 SwiGLU output")


def test_controls_exceed_the_bound(model):
    """Every negative control exceeded the bound at least once: the structural ones on each model, the removed rounding
    points over the module's models (checked at the last one)."""
    hit_anywhere = {n for (m, n), h in controls_hit.items() if h}
    missed = [n for n in control_names(model.config) if n not in ROUNDING_CONTROLS and not controls_hit.get((model.name, n))]
    if model.name == MODELS[-1]:
        missed += [n for n in ROUNDING_CONTROLS if n not in hit_anywhere]
    REPORT.append(f"PREFILL RESTATE {model.name} controls exceeded: "
                  f"{sorted(n for (m, n), hit in controls_hit.items() if m == model.name and hit)}")
    assert not missed, (missed, controls_hit)
