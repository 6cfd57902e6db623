"""
The persistent decode kernel marks its weight-tile bulk copies with an L2 ``evict_first`` cache policy. A cache policy only
decides which lines the L2 drops first, so with it (``mega_variant`` 0, the default) and without it (bit 0) every logit is
bit-identical.

Checked at the ds-1.3b shape (head_dim 128, MHA) and the tl-1.1b shape (head_dim 64, GQA 32/4), weights generated on the
device: single decode steps at contexts around the 16-position KV items up to 2047, a borrower whose cached prefix lives
partly in another slot (253 shared positions: 240 lent, 13 copied), a run of consecutive launches, and the greedy ids of the
device-resident generation loop.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
ON, OFF = 0, 1
CONTEXTS = (243, 255, 256, 257, 271, 272, 1023, 1145, 1536, 2000, 2047)


@pytest.fixture(scope="module", params=["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b"])
def model(request):
    from detikzify_b200.model import load
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=4, max_batch=1)
    yield m
    m.engine.set_option("mega_variant", 0)
    del m
    torch.cuda.empty_cache()


def _decode(eng, slot, pos, tok, variant):
    eng.set_option("mega_variant", variant)
    try:
        return eng.decode([slot], [pos], torch.tensor([tok], device="cuda"))[0].clone()
    finally:
        eng.set_option("mega_variant", 0)


def test_l2_policy_is_bit_identical_across_contexts(model):
    eng = model.engine
    assert eng.get_option("decode_persistent") == 1
    g = torch.Generator().manual_seed(4100)
    ids = torch.randint(3, 30000, (2048,), generator=g).cuda()
    slot = eng.seq_alloc()
    try:
        for T in CONTEXTS:
            eng.prefill(slot, ids[:T], 0, None, 0)
            on = _decode(eng, slot, T, int(ids[T]), ON)
            off = _decode(eng, slot, T, int(ids[T]), OFF)
            assert torch.isfinite(on).all(), T
            assert torch.equal(on, off), T
    finally:
        eng.seq_free(slot)


def test_l2_policy_is_bit_identical_on_a_borrower(model):
    eng = model.engine
    g = torch.Generator().manual_seed(4200)
    prefix = torch.randint(3, 30000, (253,), generator=g).cuda()
    suffix = torch.randint(3, 30000, (40,), generator=g).cuda()
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    try:
        eng.prefill(base, prefix, 0, None, 0)
        eng.seq_share(base, sub, prefix.numel())
        eng.prefill(sub, suffix, prefix.numel(), None, 0)
        T = prefix.numel() + suffix.numel()
        on = _decode(eng, sub, T, 17, ON)
        off = _decode(eng, sub, T, 17, OFF)
        assert torch.equal(on, off)
    finally:
        eng.seq_free(sub)
        eng.seq_free(base)


def test_l2_policy_is_bit_identical_over_consecutive_launches_and_greedy_loop(model):
    eng, cfg = model.engine, model.config
    g = torch.Generator().manual_seed(4300)
    ids = torch.randint(3, 30000, (300,), generator=g).cuda()
    toks = torch.randint(3, 30000, (12,), generator=g).tolist()
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    steps = 40
    logits, greedy = {}, {}
    try:
        for variant in (ON, OFF):
            eng.set_option("mega_variant", variant)
            eng.prefill(slot, ids, 0, None, 0)
            # back-to-back launches without a host round trip in between
            logits[variant] = torch.stack([eng.decode([slot], [ids.numel() + i], torch.tensor([t], device="cuda"))[0].clone()
                                           for i, t in enumerate(toks)]).cpu()
            last, _ = eng.prefill(slot, ids, 0, None, 0)
            first, _ = eng.sample(last, params)
            eng.gen_begin([slot], [ids.numel()], [int(first)], params)
            got = [int(first)]
            for i in range(steps):
                eng.gen_step()
                got.append(eng.gen_wait(i)[0])
            eng.gen_end()
            greedy[variant] = got
    finally:
        eng.set_option("mega_variant", 0)
        eng.seq_free(slot)
    assert torch.equal(logits[ON], logits[OFF])
    assert greedy[ON] == greedy[OFF]
