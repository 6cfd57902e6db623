"""
Every decode path against an fp64 restatement of the same step (tests/decode_restatement.py), read against the engine's own
bf16 KV cache through ``dtk_dbg_kv_read``: the cache noise of a comparison with an fp32 oracle is gone, so the bound can be
orders of magnitude tighter than a fraction of the logits' RMS.

Models (``load(..., device_init=True)``), with ``max_seqs`` slots of ``max_len`` 2048:
  ds-1.3b (MHA, hd 128)    36 slots x 0.40 GB = 14.5 GB of KV
  tl-1.1b (GQA 32/4, hd 64) 36 slots x 0.05 GB =  1.7 GB
  v2-8b-2l (GQA 32/8, llama3 RoPE, V 128256) 36 slots x 0.017 GB = 0.6 GB
  ds-7b-2l (H 4096)        36 slots x 0.07 GB =  2.4 GB

Bound on the logits. The restatement is run a second time with the kernel path's roundings replaced by random errors of
their modelled size (a length-K fp32 dot product: sqrt(K u_acc^2 + u_in^2) times the root sum of squares of its products;
fp32 elementwise results: 4 u relative; bf16 operands: the error is added before rounding, so boundary flips happen as in
the kernel; the cascade's bf16 P: half a bf16 ulp relative). sigma = the larger, over two such runs, of the RMS over the
vocabulary of the logit change. A row passes when max |kernel - restated| <= LAMBDA * sigma: the largest of B * V
Gaussian draws is about 5 sigma, LAMBDA = 10 leaves a factor two for the model's approximations.

The batched and cascade bounds come out near 5-14 % of the logits' RMS, against 4e-4 at batch 1. That is the path, not
the model. The random-init decoders amplify a perturbation from layer to layer, and at the bf16 operands an amplified
difference becomes more rounding flips, each one bf16 ulp. So an ulp-level difference in one fp32 sum grows to about 1 %
of RMS at the logits. The kernels land at about 4.5 sigma, where the largest of B * V draws of the model is expected.

Cache rows. A K / V row read back must hold the restated bf16 bits, except elements whose stored value is a bf16 neighbour
of a value within eps of the restated one (for |value| above eps that is one ulp, where the restated value lies within eps
of a rounding boundary): eps = LAMBDA * (the error model's RMS change of that head's row) + the shift that ambiguous
roundings of the bf16 norm operand can cause (batched paths) + 2^-20 |(k_i, k_i+hd/2)| for the fp32 RoPE rotation.

Negative controls run on the restatement only: each perturbed restatement must exceed the bound on at least one case.
"""
import ctypes as C
import gc
import math

import pytest
import torch

from decode_restatement import Weights, bf16, bf16_ulp, noise_scale, restate_step

pytestmark = pytest.mark.gpu
LAMBDA = 10.0
CONTEXTS = (243, 255, 256, 257, 271, 272, 512, 1023, 1024, 1145, 1536, 2000, 2047)
MODELS = ["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b", "v2-8b-2l", "ds-7b-2l"]
SLOTS = 36
REPORT = []


def release_memory():
    """Return every block torch's allocator caches to the device. The fp64 restatement's temporaries and the arenas of
    models already dropped would otherwise stay reserved, and engines created later (their own cudaMalloc) run out of
    memory."""
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", params=MODELS)
def model(request):
    from detikzify_b200.model import load
    release_memory()   # the previous parameter's arena
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=SLOTS,
                max_batch=33)
    m.name = request.param
    yield m
    m.engine.close()   # KV slots and decode tiles now, whoever still holds the model object
    del m
    release_memory()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    release_memory()   # torn down after the model fixture: nothing of this module stays on the device
    free, total = torch.cuda.mem_get_info()
    REPORT.append(f"RESTATE module end: {free / 2**30:.1f} of {total / 2**30:.1f} GiB free, "
                  f"{torch.cuda.memory_reserved() / 2**30:.2f} GiB reserved by torch")
    for line in REPORT:
        print(line)


def kv_read(eng, slot, layer, pos0, n):
    c = eng.cfg
    k = torch.empty(c.num_key_value_heads, n, c.head_dim, dtype=torch.bfloat16, device=eng.device)
    v = torch.empty_like(k)
    rc = eng.lib.dtk_dbg_kv_read(eng._h, slot, layer, pos0, n, C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                 eng._stream())
    assert rc == 0, eng.lib.dtk_last_error(eng._h).decode()
    return k, v


def reader(eng, slots, subst=None):
    def kv(b, l, n):
        k, v = kv_read(eng, slots[b], l, 0, n)
        k, v = k.double(), v.double()
        if subst is not None:
            k, v = subst(b, l, k, v)
        return k, v
    return kv


def weights(eng):
    if not hasattr(eng, "_w64"):
        eng._w64 = Weights(eng.cfg, eng.arena, eng.ccfg)
    return eng._w64


def check_logits(tag, got, ref, sig):
    err = (got.double() - ref["logits"]).abs().amax(-1)
    bound = LAMBDA * sig["logits"]
    rms = ref["logits"].pow(2).mean(-1).sqrt()
    ratio = (err / bound).max().item()
    REPORT.append(f"RESTATE {tag}: worst err/bound {ratio:.3f}, bound/RMS {(bound / rms).max().item():.2e}")
    assert torch.isfinite(got).all(), tag
    assert ratio <= 1.0, (tag, ratio)
    return bound


def exceeds(got, ctrl, bound):
    err = (got.double() - ctrl["logits"]).abs().amax(-1)
    return bool((~(err <= bound)).any())


def check_rows(tag, eng, slots, positions, ref, sig):
    for l in range(eng.cfg.num_hidden_layers):
        for b, (s, p) in enumerate(zip(slots, positions)):
            k, v = kv_read(eng, s, l, p, 1)
            for name, got, pre, sg in (("k", k[:, 0], ref["k"][l][b], sig["k"][l][b]),
                                       ("v", v[:, 0], ref["v"][l][b], sig["v"][l][b])):
                want = bf16(pre)
                got = got.double()
                eps = LAMBDA * sg[:, None] + ref["kv_eps"][l][b] + 2.0 ** -20 * pair_norm(pre)
                bad = (got != want) & ((got - pre).abs() > bf16_ulp(want) / 2 + eps)
                i = bad.nonzero()[:3].tolist()
                assert not bad.any(), (tag, name, l, b, int(bad.sum()), [(float(pre[tuple(j)]), float(want[tuple(j)]),
                                                                         float(got[tuple(j)]), float(eps[tuple(j)])) for j in i])


def pair_norm(t):
    """|(t_i, t_{i + hd/2})|: the fp32 RoPE rotation of a pair errs by a few ulps of this, not of its (possibly cancelled)
    result."""
    return torch.sqrt(t * t + t.roll(t.shape[-1] // 2, -1) ** 2)


def prompt(cfg, T, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(3, min(cfg.vocab_size, 30000), (T,), generator=g)


def test_kv_read_rejects_bad_arguments(model):
    eng = model.engine
    buf = torch.empty(1 << 20, dtype=torch.bfloat16, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    slot = eng.seq_alloc()
    try:
        other = (slot + 1) % SLOTS   # not allocated
        L, ml = eng.cfg.num_hidden_layers, eng.max_len
        for args in [(other, 0, 0, 1), (-1, 0, 0, 1), (SLOTS, 0, 0, 1), (slot, L, 0, 1), (slot, -1, 0, 1),
                     (slot, 0, -1, 1), (slot, 0, ml, 1), (slot, 0, ml - 1, 2), (slot, 0, 0, -1)]:
            assert eng.lib.dtk_dbg_kv_read(eng._h, *args, p, p, None) == -1, args
        assert eng.lib.dtk_dbg_kv_read(eng._h, slot, 0, 0, 1, None, p, None) == -1
        assert eng.lib.dtk_dbg_kv_read(eng._h, slot, L - 1, ml - 1, 1, p, p, None) == 0
    finally:
        eng.seq_free(slot)


def test_prefill_rows_layer0(model):
    """Layer 0's cache rows at every position of a 2047-token prefill: embedding (or image row) -> RMSNorm -> bf16 -> qkv ->
    RoPE -> bf16. ds-1.3b splices an image span mid-prompt."""
    eng, cfg = model.engine, model.config
    w = weights(eng)
    T = 2047
    ids = prompt(cfg, T, 11)
    img, start = None, 0
    if model.name.endswith("ds-1.3b"):
        start, n = 700, cfg.num_patches
        ids[start:start + n] = cfg.image_token_id
        img = torch.randn(n, cfg.hidden_size, generator=torch.Generator().manual_seed(12)).cuda() * 0.05
    slot = eng.seq_alloc()
    try:
        eng.prefill(slot, ids.cuda(), 0, img, start)
        k, v = kv_read(eng, slot, 0, 0, T)
        x = w("dec.embed")[ids.cuda()].clone()
        if img is not None:
            x[start:start + img.shape[0]] = img.double()
        H, nh, nkv, HD = cfg.hidden_size, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        r = torch.rsqrt((x * x).mean(-1, keepdim=True) + cfg.rms_norm_eps)
        h = x * r * w("dec.L0.norm1")
        hb = bf16(h)
        near = ((h - hb).abs() - bf16_ulp(hb) / 2).abs() <= 2.0 ** -18 * h.abs()
        wk = w("dec.L0.wqkv")[nh * HD:]
        kv = hb @ wk.T
        amb = (near * bf16_ulp(hb)) @ wk.abs().T + math.sqrt(H) * 2.0 ** -23 * torch.sqrt((hb * hb) @ (wk * wk).T) * LAMBDA
        kk, vv = kv[:, :nkv * HD].view(T, nkv, HD), kv[:, nkv * HD:].view(T, nkv, HD)
        cs = w.rope[:T][:, None]
        kk = torch.cat([kk[..., :HD // 2] * cs[..., 0] - kk[..., HD // 2:] * cs[..., 1],
                        kk[..., HD // 2:] * cs[..., 0] + kk[..., :HD // 2] * cs[..., 1]], -1)
        eps_k = amb[:, :nkv * HD].view(T, nkv, HD).abs()
        eps_k = eps_k + eps_k.roll(HD // 2, -1) + 2.0 ** -20 * pair_norm(kk)
        eps_v = amb[:, nkv * HD:].view(T, nkv, HD)
        for name, got, pre, eps in (("k", k.permute(1, 0, 2), kk, eps_k), ("v", v.permute(1, 0, 2), vv, eps_v)):
            want = bf16(pre)
            got = got.double()
            bad = (got != want) & ((got - pre).abs() > bf16_ulp(want) / 2 + eps)
            REPORT.append(f"RESTATE {model.name} prefill L0 {name}: {int((got != want).sum())} boundary elements of {got.numel()}")
            i = bad.nonzero()[:3]
            assert not bad.any(), (name, i.tolist(), [(float(pre[tuple(j)]), float(want[tuple(j)]), float(got[tuple(j)]),
                                                      float(eps[tuple(j)])) for j in i.tolist()])
    finally:
        eng.seq_free(slot)


def _single(eng, cfg, w, path, slot, T, ids, tag, controls=None):
    pos, tok = [T], [int(ids[T])]
    got = eng.decode([slot], pos, ids[T:T + 1].cuda())
    torch.cuda.synchronize()
    kv = reader(eng, [slot])
    ref = restate_step(w, pos, tok, kv, path)
    sig = noise_scale(w, pos, tok, kv, path, ref)
    bound = check_logits(tag, got, ref, sig)
    check_rows(tag, eng, [slot], pos, ref, sig)
    if controls is not None:
        for name, kw in controls.items():
            key = (cfg.name_or_path, name)
            controls_hit.setdefault(key, False)
            if exceeds(got, restate_step(w, pos, tok, kv, path, **kw), bound):
                controls_hit[key] = True
    return got


controls_hit = {}


def _controls(cfg, path):
    c = {"drop last cached key": dict(drop_key=lambda n: n - 1),
         "drop first key of an item": dict(drop_key=lambda n: 16 * (n // 32)),
         "RoPE at pos + 1": dict(rope_shift=1)}
    if cfg.num_key_value_heads > 1 and cfg.num_attention_heads != cfg.num_key_value_heads:
        c["GQA h % kv_heads"] = dict(gqa_mod=True)
    if path == "persistent":
        c["unrounded current K/V"] = dict(fp32_current=True)
    return c


@pytest.mark.parametrize("path", ["persistent", "per_op"])
def test_batch1_step(model, path):
    eng, cfg = model.engine, model.config
    w = weights(eng)
    ids = prompt(cfg, 2048, 21)
    slot = eng.seq_alloc()
    eng.set_option("decode_impl", 1 if path == "persistent" else 0)
    try:
        for T in CONTEXTS:
            eng.prefill(slot, ids[:T].cuda(), 0, None, 0)
            _single(eng, cfg, w, path, slot, T, ids, f"{model.name} {path} T={T}",
                    _controls(cfg, path) if T in (243, 2047) else None)
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)


@pytest.mark.parametrize("path", ["persistent", "per_op"])
def test_borrower_step(model, path):
    """253 shared positions: 240 lent, 13 copied. The control reads the lent positions from the borrower's own slot (which
    holds another prompt's rows)."""
    eng, cfg = model.engine, model.config
    w = weights(eng)
    pre, own, suf = prompt(cfg, 253, 31), prompt(cfg, 253, 32), prompt(cfg, 40, 33)
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    eng.set_option("decode_impl", 1 if path == "persistent" else 0)
    try:
        eng.prefill(base, pre.cuda(), 0, None, 0)
        eng.prefill(sub, own.cuda(), 0, None, 0)
        own_rows = [kv_read(eng, sub, l, 0, 240) for l in range(cfg.num_hidden_layers)]
        eng.seq_share(base, sub, 253)
        eng.prefill(sub, suf.cuda(), 253, None, 0)
        T = 293
        got = eng.decode([sub], [T], torch.tensor([17], device="cuda"))
        torch.cuda.synchronize()
        kv = reader(eng, [sub])
        ref = restate_step(w, [T], [17], kv, path)
        sig = noise_scale(w, [T], [17], kv, path, ref)
        bound = check_logits(f"{model.name} {path} borrower", got, ref, sig)
        check_rows(f"{model.name} {path} borrower", eng, [sub], [T], ref, sig)

        def own_slot(b, l, k, v):
            k, v = k.clone(), v.clone()
            k[:, :240], v[:, :240] = own_rows[l][0].double(), own_rows[l][1].double()
            return k, v
        assert exceeds(got, restate_step(w, [T], [17], reader(eng, [sub], own_slot), path), bound)
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(sub)
        eng.seq_free(base)


def test_batched_steps(model):
    eng, cfg = model.engine, model.config
    w = weights(eng)
    slots = [eng.seq_alloc() for _ in range(33)]
    g = torch.Generator().manual_seed(41)
    try:
        lens = torch.randint(200, 1200, (33,), generator=g).tolist()
        ids = [prompt(cfg, n + 1, 100 + i) for i, n in enumerate(lens)]
        for s, n, t in zip(slots, lens, ids):
            eng.prefill(s, t[:n].cuda(), 0, None, 0)
        for B in (4, 5, 17, 32, 33):
            # each B decodes at the same positions: the step rewrites row n and reads rows [0, n) of the prompt
            pos, tok = lens[:B], [int(t[n]) for t, n in zip(ids[:B], lens)]
            got = eng.decode(slots[:B], pos, torch.tensor(tok, device="cuda"))
            torch.cuda.synchronize()
            kv = reader(eng, slots[:B])
            ref = restate_step(w, pos, tok, kv, "batched")
            sig = noise_scale(w, pos, tok, kv, "batched", ref)
            bound = check_logits(f"{model.name} batched B={B}", got, ref, sig)
            check_rows(f"{model.name} batched B={B}", eng, slots[:B], pos, ref, sig)
            if B == 5:
                for name, kw in _controls(cfg, "batched").items():
                    assert exceeds(got, restate_step(w, pos, tok, kv, "batched", **kw), bound), name
    finally:
        for s in slots:
            eng.seq_free(s)


def test_cascade_step(model):
    """32 rows that borrow one 253-position prefix (240 lent), each with a private suffix of its own length."""
    eng, cfg = model.engine, model.config
    w = weights(eng)
    base = eng.seq_alloc()
    subs = [eng.seq_alloc() for _ in range(32)]
    try:
        eng.prefill(base, prompt(cfg, 253, 51).cuda(), 0, None, 0)
        pos, tok = [], []
        for i, s in enumerate(subs):
            eng.seq_share(base, s, 253)
            n = 3 + 5 * i
            suf = prompt(cfg, n + 1, 200 + i)
            eng.prefill(s, suf[:n].cuda(), 253, None, 0)
            pos.append(253 + n)
            tok.append(int(suf[n]))
        got = eng.decode(subs, pos, torch.tensor(tok, device="cuda"))
        torch.cuda.synchronize()
        kv = reader(eng, subs)
        ref = restate_step(w, pos, tok, kv, "cascade", cas_len=240)
        sig = noise_scale(w, pos, tok, kv, "cascade", ref, cas_len=240)
        bound = check_logits(f"{model.name} cascade B=32", got, ref, sig)
        check_rows(f"{model.name} cascade B=32", eng, subs, pos, ref, sig)
        assert exceeds(got, restate_step(w, pos, tok, kv, "cascade", cas_len=240, drop_key=lambda n: 16 * (n // 32)), bound)
    finally:
        for s in subs:
            eng.seq_free(s)
        eng.seq_free(base)


def test_controls_exceed_the_bound(model):
    """Every negative control of the batch-1 steps (collected over the module's cases) exceeded the bound at least once."""
    cfg = model.config
    for path in ("persistent", "per_op"):
        for name in _controls(cfg, path):
            assert controls_hit.get((cfg.name_or_path, name)), (name, controls_hit)


def test_fused_greedy_loop(model):
    """gen_begin / gen_step on the persistent kernel: each step restated on the cache read back after it."""
    eng, cfg = model.engine, model.config
    w = weights(eng)
    ids = prompt(cfg, 300, 61)
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False)
    try:
        last, _ = eng.prefill(slot, ids.cuda(), 0, None, 0)
        first = int(last.argmax())
        eng.gen_begin([slot], [300], [first], params)
        toks = [first]
        decided = 0
        for i in range(6):
            eng.gen_step()
            toks.append(eng.gen_wait(i)[0])
            torch.cuda.synchronize()
            T = 300 + i
            kv = reader(eng, [slot])
            ref = restate_step(w, [T], [toks[i]], kv, "persistent")
            sig = noise_scale(w, [T], [toks[i]], kv, "persistent", ref)
            top = ref["logits"][0].topk(2)
            if (top.values[0] - top.values[1]).item() > 2 * LAMBDA * sig["logits"][0].item():
                assert toks[i + 1] == int(top.indices[0]), (i, toks)
                decided += 1
        eng.gen_end()
        assert decided >= 3
    finally:
        eng.seq_free(slot)


def test_fp8_persistent_and_batched():
    from detikzify_b200.model import load
    m, _ = load("nllg/detikzify-ds-1.3b", device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=6,
                max_batch=5, quantize="fp8")
    eng, cfg = m.engine, m.config
    w = Weights(cfg, eng.arena, eng.ccfg)
    slots = [eng.seq_alloc() for _ in range(5)]
    try:
        lens = [243, 300, 511, 1024, 2047]
        ids = [prompt(cfg, n + 1, 300 + i) for i, n in enumerate(lens)]
        for s, n, t in zip(slots, lens, ids):
            eng.prefill(s, t[:n].cuda(), 0, None, 0)
        _single(eng, cfg, w, "persistent", slots[4], 2047, ids[4], "ds-1.3b fp8 persistent T=2047")
        pos, tok = lens, [int(t[n]) for t, n in zip(ids, lens)]
        got = eng.decode(slots, pos, torch.tensor(tok, device="cuda"))
        torch.cuda.synchronize()
        kv = reader(eng, slots)
        ref = restate_step(w, pos, tok, kv, "batched")
        sig = noise_scale(w, pos, tok, kv, "batched", ref)
        check_logits("ds-1.3b fp8 batched B=5", got, ref, sig)
        check_rows("ds-1.3b fp8 batched B=5", eng, slots, pos, ref, sig)
    finally:
        for s in slots:
            eng.seq_free(s)
        eng.close()
        del m, eng, w
        release_memory()
