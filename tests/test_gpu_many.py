"""Continuous batching on the GPU: row retirement and admission inside the running batched decode loop.

- ``generate_many``'s first ``batch_size`` requests equal ``generate_batch`` of those prompts token for token (one shared
  figure; greedy and sampled, with and without processors; tiny shapes and ``ds-7b-2l`` at B = 32 on the swap-GEMM path
  with the shared-prefix cascade).
- A loop with retirements and admissions draws exactly the tokens of the same schedule run one step at a time through
  ``dtk_decode`` + ``dtk_sample`` with each row's counters (``steps = 1 + t - s0``, ``seq_id``); an inactive row sits on a
  scratch slot there (rows are independent columns of every kernel).
- A retired row's slot reads back byte-identical after further steps; a slot reused inside the loop holds the KV a fresh
  prefill writes; ``dtk_gen_wait`` and ``dtk_gen_first`` return with rows inactive; every refused admission returns its status
  and message."""
import ctypes as C
import gc

import pytest
import torch

from conftest import model_bundle

pytestmark = pytest.mark.gpu

_ENGINES = {}
_MODELS = {}


def engine_for(name, max_seqs, max_batch):
    """this module's engines (not the session cache): the ds-7b-2l one holds 36 KV slots, released when the module ends"""
    key = (name, max_seqs, max_batch)
    if key not in _ENGINES:
        from detikzify_b200.engine import Engine, pack_arena
        cfg, sd, _ = model_bundle(name)
        _ENGINES[key] = Engine(cfg, pack_arena(cfg, sd), device=0, max_seqs=max_seqs, max_batch=max_batch)
    return _ENGINES[key]


@pytest.fixture(scope="module", autouse=True)
def _release():
    """Close every engine of this module and return torch's cached blocks to the device, so that the engines of the test
    modules that run after this one find the memory free."""
    yield
    _MODELS.clear()
    for eng in _ENGINES.values():
        eng.close()
    _ENGINES.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _pixels(cfg, seed=1000):
    g = torch.Generator().manual_seed(seed)
    S = cfg.vision_config.image_size
    return torch.rand(1, 3, S, S, generator=g) * 2 - 1


def _prompt(cfg, n_text, seed):
    g = torch.Generator().manual_seed(seed)
    text = torch.randint(3, 200, (n_text,), generator=g)
    return torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), text]).long()


def _model(name, max_seqs, max_batch):
    """one model object per cached engine (each model keeps a prefix-cache slot of its own)"""
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    key = (name, max_seqs, max_batch)
    if key not in _MODELS:
        cfg, _, _ = model_bundle(name)
        _MODELS[key] = DetikzifyForCausalLM(cfg, engine=engine_for(name, max_seqs=max_seqs, max_batch=max_batch),
                                            max_seqs=max_seqs, max_batch=max_batch)
    return _MODELS[key]


def _stop_after(prompts, new):
    return [[(lambda ids, scores, n=p.numel() + k: ids.shape[1] >= n)] for p, k in zip(prompts, new)]


@pytest.mark.parametrize("do_sample,proc", [(False, False), (True, False), (False, True), (True, True)],
                         ids=["greedy", "sampled", "greedy-proc", "sampled-proc"])
@pytest.mark.parametrize("B", [2, 5])
def test_first_wave_equals_generate_batch(B, do_sample, proc):
    model = _model("tiny", 24, 8)
    cfg = model.config
    pix = _pixels(cfg)
    base = _prompt(cfg, 30, 7)
    N = 3 * B + 1
    prompts = [base] * N                                     # samples of one prompt: every request shares its whole prefix
    new = [(5 * i + 3) % 23 + 4 for i in range(N)]
    kw = dict(do_sample=do_sample, temperature=0.8, top_p=0.95, seed=1234, max_new_tokens=40,
              bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id])
    if proc:
        kw.update(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5)
    crit = _stop_after(prompts, new)
    outs = dict(model.generate_many(prompts, pix, batch_size=B, stopping_criteria=crit, **kw))
    ref = model.generate_batch(prompts[:B], pix, stopping_criteria=crit[:B], **kw)
    assert [outs[i].tolist() for i in range(B)] == [r.cpu().tolist() for r in ref]
    assert sorted(outs) == list(range(N)) and all(len(outs[i]) == base.numel() + new[i] for i in range(N))


def _run_schedule(eng, cfg, B, prompts, n_steps, do_sample, img):
    """The loop with retirements and admissions: request i stays for n_steps[i] loop tokens after its first one; rows are
    refilled in request order as soon as the host sees a request end. Returns per request (first token + loop tokens, s0,
    row, slot) and every ring row read."""
    params = eng.sampling(temperature=1.3, top_p=0.97, do_sample=do_sample, seed=(0xABCD << 32) | 5)
    N = len(prompts)
    slots = {}
    got = {i: [] for i in range(N)}
    s0, row_of = {}, {}
    for i in range(B):
        slots[i] = eng.seq_alloc()
    last = torch.stack([eng.prefill(slots[i], prompts[i].cuda(), 0, img, 0)[0] for i in range(B)])
    first, _ = eng.sample(last, params, suppress=[1] * B, steps=[0] * B, seq_ids=list(range(B)))
    for i, t in enumerate(first.tolist()):
        got[i].append(t)
        s0[i], row_of[i] = 0, i
    eng.gen_begin([slots[i] for i in range(B)], [prompts[i].numel() for i in range(B)], first.tolist(), params,
                  list(range(B)))
    rows = list(range(B))
    queue = list(range(B, N))
    launched = waited = 0
    pending = []
    ring = []
    try:
        while any(o is not None for o in rows):
            while launched < waited + 2:
                eng.gen_step()
                launched += 1
            for r in pending:
                got[rows[r]].append(eng.gen_first(r))
            pending = []
            entry = eng.gen_wait(waited)
            ring.append((waited, list(entry), list(rows)))
            for r, i in enumerate(rows):
                if i is not None and waited >= s0[i] and len(got[i]) <= n_steps[i]:
                    got[i].append(entry[r])
            waited += 1
            for r, i in enumerate(rows):
                if i is not None and len(got[i]) > n_steps[i]:
                    eng.gen_retire(r)
                    eng.seq_free(slots[i])
                    rows[r] = None
                    if queue:
                        j = queue.pop(0)
                        slots[j] = eng.seq_alloc()
                        lg, _ = eng.prefill(slots[j], prompts[j].cuda(), 0, img, 0)
                        eng.gen_admit(r, slots[j], prompts[j].numel(), lg, j)
                        rows[r], s0[j], row_of[j] = j, launched, r
                        pending.append(r)
    finally:
        eng.gen_end()
    return params, got, s0, row_of, slots, ring


def _stepwise(eng, cfg, B, prompts, n_steps, params, s0, row_of, img):
    """The same schedule one step at a time: dtk_decode + dtk_sample with counter 1 + t - s0 on stream seq_id; a row without
    an occupant decodes a scratch slot."""
    N = len(prompts)
    slots = [eng.seq_alloc() for _ in range(N)]
    scratch = eng.seq_alloc()
    try:
        want = {}
        for i in range(N):
            lg, _ = eng.prefill(slots[i], prompts[i].cuda(), 0, img, 0)
            t, _ = eng.sample(lg[None], params, suppress=[1], steps=[0], seq_ids=[i])
            want[i] = [int(t.item())]
        T = max(s0[i] + n_steps[i] for i in range(N))
        for t in range(T):
            occ = [None] * B
            for i in range(N):
                if s0[i] <= t < s0[i] + n_steps[i]:
                    occ[row_of[i]] = i
            sl = [slots[i] if i is not None else scratch for i in occ]
            pos = [prompts[i].numel() + t - s0[i] if i is not None else 0 for i in occ]
            tok = [want[i][-1] if i is not None else 0 for i in occ]
            lg = eng.decode(sl, pos, torch.tensor(tok, device="cuda"))
            nxt, _ = eng.sample(lg, params, suppress=[0] * B,
                                steps=[(1 + t - s0[i]) & 0xFFFFFFFF if i is not None else 0 for i in occ],
                                seq_ids=[i if i is not None else 0 for i in occ])
            for r, i in enumerate(occ):
                if i is not None:
                    want[i].append(int(nxt[r]))
        return want
    finally:
        for s in slots + [scratch]:
            eng.seq_free(s)


@pytest.mark.parametrize("B,do_sample", [(2, True), (5, True), (5, False)], ids=["B2-gemv", "B5-gemm", "B5-gemm-greedy"])
def test_admitted_rows_equal_stepwise_run(B, do_sample):
    cfg, _, _ = model_bundle("tiny")
    eng = engine_for("tiny", max_seqs=24, max_batch=8)
    img = eng.image_embeds(_pixels(cfg).cuda())[0]
    N = 2 * B + 3
    prompts = [_prompt(cfg, 4 + (7 * i) % 13, 300 + i) for i in range(N)]
    n_steps = [(11 * i + 5) % 17 + 1 for i in range(N)]
    params, got, s0, row_of, slots, ring = _run_schedule(eng, cfg, B, prompts, n_steps, do_sample, img)
    assert any(s > 0 for s in s0.values())                   # some requests really entered a running loop
    want = _stepwise(eng, cfg, B, prompts, n_steps, params, s0, row_of, img)
    for i in range(N):
        assert got[i] == want[i], (i, s0[i], row_of[i])
    # a row without an occupant publishes the sentinel from the first step launched after its retirement
    assert any(-1 in entry for _, entry, _ in ring)
    for t, entry, rows in ring:
        for r, i in enumerate(rows):
            if i is not None and t >= s0[i]:
                assert entry[r] >= 0


def _kv(eng, slot, n):
    L, kvh, hd = eng.cfg.num_hidden_layers, eng.cfg.num_key_value_heads, eng.cfg.head_dim
    out = []
    for layer in range(L):
        k = torch.empty(kvh, n, hd, dtype=torch.bfloat16, device="cuda")
        v = torch.empty_like(k)
        assert eng.lib.dtk_dbg_kv_read(eng._h, slot, layer, 0, n, C.c_void_p(k.data_ptr()), C.c_void_p(v.data_ptr()),
                                       C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
        out += [k, v]
    torch.cuda.synchronize()
    return [t.view(torch.int16).cpu() for t in out]


@pytest.mark.parametrize("B", [3, 5])
def test_retired_rows_write_nothing_and_reused_slots_hold_a_fresh_prefill(B):
    cfg, _, _ = model_bundle("tiny")
    eng = engine_for("tiny", max_seqs=24, max_batch=8)
    img = eng.image_embeds(_pixels(cfg).cuda())[0]
    params = eng.sampling(temperature=1.0, do_sample=True, seed=99)
    prompts = [_prompt(cfg, 6 + i, 500 + i) for i in range(B + 1)]
    slots = [eng.seq_alloc() for _ in range(B)]
    spare = eng.seq_alloc()
    try:
        last = torch.stack([eng.prefill(s, p.cuda(), 0, img, 0)[0] for s, p in zip(slots, prompts)])
        first, _ = eng.sample(last, params, suppress=[1] * B, steps=[0] * B)
        eng.gen_begin(slots, [p.numel() for p in prompts[:B]], first.tolist(), params)
        try:
            for t in range(3):
                eng.gen_step()
                eng.gen_wait(t)
            eng.gen_retire(1)
            ml = eng.max_len
            before = _kv(eng, slots[1], ml)
            for t in range(3, 9):
                eng.gen_step()
                row = eng.gen_wait(t)
                assert row[1] == -1 and all(x >= 0 for r, x in enumerate(row) if r != 1)
            after = _kv(eng, slots[1], ml)
            assert all(torch.equal(a, b) for a, b in zip(before, after))
            # the retired slot goes to a new request inside the same loop
            eng.seq_free(slots[1])
            reused = eng.seq_alloc()
            assert reused == slots[1]
            T0 = prompts[B].numel()
            lg, _ = eng.prefill(reused, prompts[B].cuda(), 0, img, 0)
            eng.gen_admit(1, reused, T0, lg, 7)
            eng.gen_step()
            tok = eng.gen_first(1)
            assert 0 <= tok < cfg.vocab_size
            assert eng.gen_wait(9)[1] >= 0
        finally:
            eng.gen_end()
        eng.prefill(spare, prompts[B].cuda(), 0, img, 0)
        fresh = _kv(eng, spare, T0)
        held = _kv(eng, reused, T0)
        assert all(torch.equal(a, b) for a, b in zip(fresh, held))
    finally:
        for s in slots + [spare]:
            try:
                eng.seq_free(s)
            except Exception:
                pass


def test_refused_admissions():
    cfg, _, _ = model_bundle("tiny")
    eng = engine_for("tiny", max_seqs=24, max_batch=8)
    lib, h = eng.lib, eng._h
    img = eng.image_embeds(_pixels(cfg).cuda())[0]
    params = eng.sampling(do_sample=False)
    logits = torch.zeros(cfg.vocab_size, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def admit(row, slot, pos):
        return lib.dtk_gen_admit(h, row, slot, pos, C.c_void_p(logits.data_ptr()), 0, None, 0, 0, stream)

    def msg():
        return lib.dtk_last_error(h).decode()

    p = _prompt(cfg, 70, 9)
    if eng.get_option("decode_persistent"):     # B = 1 on the persistent kernel: no admissions
        s = eng.seq_alloc()
        try:
            eng.prefill(s, p.cuda(), 0, img, 0)
            eng.gen_begin([s], [p.numel()], [3], params)
            try:
                assert admit(0, s, p.numel()) == -5 and "persistent" in msg()
                assert lib.dtk_gen_retire(h, 0, stream) == -5
            finally:
                eng.gen_end()
        finally:
            eng.seq_free(s)
    # B = 4 rows sharing one 64-position prefix: the loop runs the cascade
    base = eng.seq_alloc()
    slots = [eng.seq_alloc() for _ in range(4)]
    other = eng.seq_alloc()
    free_slot = eng.seq_alloc()
    eng.seq_free(free_slot)
    try:
        eng.prefill(base, p.cuda(), 0, img, 0)
        for s in slots:
            eng.seq_share(base, s, 64)
            eng.prefill(s, p[64:].cuda(), 64, None, 0)
        eng.gen_begin(slots, [p.numel()] * 4, [3] * 4, params)
        try:
            assert admit(0, slots[0], p.numel()) == -1 and "active" in msg()
            assert eng.lib.dtk_gen_retire(h, 0, stream) == 0
            assert admit(0, free_slot, p.numel()) == -1 and "allocated" in msg()
            assert admit(0, slots[0], 40) == -1 and "shared prefix" in msg()
            eng.prefill(other, p.cuda(), 0, img, 0)                       # unshared: another prefix than the cascade's
            assert admit(0, other, p.numel()) == -1 and "cascade" in msg()
            assert admit(9, slots[0], p.numel()) == -1
            assert admit(0, slots[0], p.numel()) == 0                     # the borrower of the loop's prefix is taken
            eng.gen_step()
            assert 0 <= eng.gen_first(0) < cfg.vocab_size
            assert eng.gen_wait(0)[0] >= 0
        finally:
            eng.gen_end()
    finally:
        for s in slots + [other, base]:
            eng.seq_free(s)


def test_ds7b_2l_b32_cascade_first_wave():
    """The real shape: ds-7b-2l, 40 samples of one figure at batch_size 32 (swap-GEMM step with the shared-prefix cascade)."""
    model = _model("ds-7b-2l", 36, 32)
    cfg = model.config
    pix = _pixels(cfg)
    p = _prompt(cfg, 100, 11)                                 # 104 shared positions: 96 lent, the cascade's prefix
    N = 40
    new = [(13 * i + 5) % 29 + 3 for i in range(N)]
    prompts = [p] * N
    crit = _stop_after(prompts, new)
    kw = dict(do_sample=True, temperature=0.8, top_p=0.95, seed=77, max_new_tokens=40,
              bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id])
    outs = dict(model.generate_many(prompts, pix, batch_size=32, stopping_criteria=crit, **kw))
    ref = model.generate_batch(prompts[:32], pix, stopping_criteria=crit[:32], **kw)
    assert [outs[i].tolist() for i in range(32)] == [r.cpu().tolist() for r in ref]
    assert sorted(outs) == list(range(N)) and all(len(outs[i]) == p.numel() + new[i] for i in range(N))
