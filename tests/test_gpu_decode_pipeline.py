"""
Consumer order of the batch-1 persistent decode kernel on the GPU.

A consumer warp reads a weight tile out of the ring, hands the slot back and rebuilds the tile's A fragments before it stages
the tile's input slice (the wait for the previous phase's output); ``mega_variant`` bit 1 stages first, as earlier builds
did. Neither order changes an operation or its operands, so the logits must be bit-identical with the bit on and off:
  * bf16 tiles, packed tiles (also with injected escape tiles) and FP8 tiles, on one quantized arena;
  * head_dim 128 (ds-1.3b shape) and head_dim 64 (tl-1.1b shape);
  * ring depths of 8 slots (one per consumer warp), 16 and the configured default;
  * contexts 1, 15, 16, 17, 243 and 2047, and a borrower of a shared prefix;
  * the greedy ids of 64 consecutive launches of the device-resident loop.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
CONTEXTS = (1, 15, 16, 17, 243, 2047)
FORMATS = {"bf16": (0, 0), "packed": (0, 1), "fp8": (1, 0)}   # (decode_fp8, decode_pack)
NSLOTS = (8, 16, 0)                                             # 0 = the configured ring depth
STAGE_FIRST = 2                                                  # mega_variant bit 1


@pytest.fixture(scope="module", params=["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b"])
def model(request):
    from detikzify_b200.model import load
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=4, max_batch=1,
                quantize="fp8")
    yield m
    del m
    torch.cuda.empty_cache()


def _format(eng, name):
    fp8, pk = FORMATS[name]
    eng.set_option("decode_fp8", 0)
    eng.set_option("decode_pack", pk)
    eng.set_option("decode_fp8", fp8)
    assert (eng.get_option("decode_fp8"), eng.get_option("decode_pack")) == (fp8, pk)


def _reset(eng):
    eng.set_option("mega_variant", 0)
    eng.set_option("mega_nslots", 0)
    _format(eng, "fp8")


def _both_orders(eng, slot, pos, tok):
    out = []
    for variant in (0, STAGE_FIRST):
        eng.set_option("mega_variant", variant)
        out.append(eng.decode([slot], [pos], torch.tensor([tok], device="cuda"))[0].clone())
    eng.set_option("mega_variant", 0)
    return out


def test_orders_are_bit_identical_across_formats_ring_depths_and_contexts(model):
    eng = model.engine
    g = torch.Generator().manual_seed(7100)
    ids = torch.randint(3, 30000, (2048,), generator=g).cuda()
    slot = eng.seq_alloc()
    try:
        for T in CONTEXTS:
            eng.prefill(slot, ids[:T], 0, None, 0)
            ref = None
            for name in FORMATS:
                _format(eng, name)
                for ns in NSLOTS:
                    eng.set_option("mega_nslots", ns)
                    new, old = _both_orders(eng, slot, T, int(ids[T]))
                    assert torch.isfinite(new).all(), (T, name, ns)
                    assert torch.equal(new, old), (T, name, ns)
                    if name != "fp8":   # bf16 and packed tiles hold the same bits
                        ref = new if ref is None else ref
                        assert torch.equal(new, ref), (T, name, ns)
    finally:
        _reset(eng)
        eng.seq_free(slot)


def test_orders_are_bit_identical_on_a_borrower(model):
    eng = model.engine
    g = torch.Generator().manual_seed(7200)
    prefix = torch.randint(3, 30000, (253,), generator=g).cuda()
    suffix = torch.randint(3, 30000, (40,), generator=g).cuda()
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    try:
        eng.prefill(base, prefix, 0, None, 0)
        eng.seq_share(base, sub, prefix.numel())
        eng.prefill(sub, suffix, prefix.numel(), None, 0)
        T = prefix.numel() + suffix.numel()
        for name in FORMATS:
            _format(eng, name)
            new, old = _both_orders(eng, sub, T, 17)
            assert torch.equal(new, old), name
    finally:
        _reset(eng)
        eng.seq_free(sub)
        eng.seq_free(base)


def test_orders_are_bit_identical_on_escape_tiles(model):
    """Packed tiles with escape tiles (exponent bytes from the side buffer, base 0) and a base-0 row of subnormals."""
    from test_gpu_pack import _matrices
    eng = model.engine
    mats = _matrices(eng)
    edits = [("dec.L0.wqkv", 3, 5, 0x0000), ("dec.L0.wo", 17, 300, 0x0001), ("dec.L0.wgu", 40, 7, 0x2000),
             ("dec.L0.wd", 2, 1000, 0x4300), ("dec.lm_head", 33, 100, 0x0000)]
    g = torch.Generator().manual_seed(7300)
    ids = torch.randint(3, 30000, (400,), generator=g).cuda()
    slot = eng.seq_alloc()
    flat = eng.arena.view(torch.int16)
    saved = []
    try:
        _format(eng, "packed")
        n0 = eng.get_option("decode_pack_escapes")
        for name, r, c, v in edits:
            i = mats[name].offset // 2 + r * mats[name].cols + c
            saved.append((i, flat[i].clone()))
            flat[i] = int(np.array(v, np.uint16).view(np.int16))
        info = mats["dec.L0.wo"]
        i0 = info.offset // 2 + 50 * info.cols
        saved.append((slice(i0, i0 + info.cols), flat[i0:i0 + info.cols].clone()))
        flat[i0:i0 + info.cols] = torch.randint(1, 0x80, (info.cols,), device=flat.device).to(torch.int16)
        eng.set_option("decode_pack", 0)   # rebuild the tiles from the edited arena
        eng.set_option("decode_pack", 1)
        assert eng.get_option("decode_pack_escapes") >= n0 + 3
        eng.prefill(slot, ids, 0, None, 0)
        for ns in NSLOTS:
            eng.set_option("mega_nslots", ns)
            new, old = _both_orders(eng, slot, ids.numel(), 11)
            assert torch.equal(new, old), ns
    finally:
        for i, v in saved:
            flat[i] = v
        eng.set_option("decode_pack", 0)
        _reset(eng)
        eng.seq_free(slot)


def test_orders_give_the_same_greedy_ids_over_64_launches(model):
    eng, cfg = model.engine, model.config
    g = torch.Generator().manual_seed(7400)
    ids = torch.randint(3, 30000, (300,), generator=g).cuda()
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    steps = 64
    greedy = {}
    try:
        for name in FORMATS:
            _format(eng, name)
            for ns in (8, 0):
                eng.set_option("mega_nslots", ns)
                for variant in (0, STAGE_FIRST):
                    eng.set_option("mega_variant", variant)
                    last, _ = eng.prefill(slot, ids, 0, None, 0)
                    first, _ = eng.sample(last, params)
                    eng.gen_begin([slot], [ids.numel()], [int(first)], params)
                    got = [int(first)]
                    for i in range(steps):
                        eng.gen_step()
                        got.append(eng.gen_wait(i)[0])
                    eng.gen_end()
                    greedy[name, ns, variant] = got
    finally:
        _reset(eng)
        eng.seq_free(slot)
    for name in FORMATS:
        for ns in (8, 0):
            assert greedy[name, ns, 0] == greedy[name, ns, STAGE_FIRST], (name, ns)
    assert greedy["bf16", 0, 0] == greedy["packed", 0, 0]
