"""
Packed decoder weights (engine option ``decode_pack``, on by default in ``load()``) on the GPU.

The batch-1 persistent kernel streams every matrix, lm_head included, as 13-bit packed tiles (sign | mantissa7 plus a 5-bit
exponent code against a per-row base, escape tiles for the rest) and rebuilds the exact bf16 bits in registers, so on one
engine its logits must be bit-identical with the option on and off:
  * the device packer writes the bytes of the numpy restatement (test_cpu_pack.py) for every matrix of one layer;
  * at the ds-1.3b (head_dim 128, MHA), tl-1.1b (head_dim 64, GQA 32/4) and v2-8b-2l (GQA 32/8, V 128256) shapes: single steps
    at contexts around the 16-position KV items up to 2047, a borrower of a shared prefix, back-to-back launches, and the
    greedy ids of the device-resident loop with mega_variant 0 and 1;
  * an arena with injected escape values, zeros and subnormals (escape tiles, base-0 rows);
  * ``decode_weight_bytes`` counts the packed tiles and escape planes;
  * switching ``decode_pack`` and ``decode_fp8`` in any order leaves each mode's logits unchanged, and a generation loop whose
    per-token graph was captured before a switch is captured again after it.
"""
import ctypes as C
import re

import numpy as np
import pytest
import torch

from test_cpu_pack import TILE, TILE_GLU, TILE_ROPE, TILE_SEQ, geometry, pack

pytestmark = pytest.mark.gpu
CONTEXTS = (243, 255, 256, 257, 271, 272, 1023, 1145, 1536, 2000, 2047)
MODES = {"wqkv": TILE_ROPE, "wo": TILE_SEQ, "wgu": TILE_GLU, "wd": TILE_SEQ}


@pytest.fixture(scope="module", params=["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b", "v2-8b-2l"])
def model(request):
    from detikzify_b200.model import load
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=4, max_batch=1)
    yield m
    del m
    torch.cuda.empty_cache()


def _decode(eng, slot, pos, tok, pk):
    eng.set_option("decode_pack", pk)
    return eng.decode([slot], [pos], torch.tensor([tok], device="cuda"))[0].clone()


def _matrices(eng):
    from detikzify_b200.engine import weight_table
    out = {}
    for info in weight_table(eng.ccfg):
        name = info.name.decode()
        if re.fullmatch(r"dec\.L\d+\.(wqkv|wo|wgu|wd)", name) or name == "dec.lm_head":
            out[name] = info
    return out


def _bits(eng, info):
    view = eng.arena[info.offset // 2: info.offset // 2 + info.rows * info.cols]
    return view.view(torch.int16).cpu().numpy().view(np.uint16).reshape(info.rows, info.cols)


def _packed_bytes(cfg, mats):
    layer = sum(np.prod(geometry(mats[f"dec.L0.{n}"].rows, mats[f"dec.L0.{n}"].cols, MODES[n])) for n in MODES)
    lm = np.prod(geometry(mats["dec.lm_head"].rows, mats["dec.lm_head"].cols, TILE_SEQ))
    return int(layer * cfg.num_hidden_layers + lm) * TILE


def test_device_packer_matches_numpy(model):
    eng, cfg = model.engine, model.config
    assert eng.get_option("decode_pack") == 1 and eng.get_option("decode_persistent") == 1
    mats = _matrices(eng)
    off = esc0 = 0
    for n in MODES:   # layer 0: wqkv | wo | wgu | wd (the restatement of the larger v2-8b MLP matrices would take minutes)
        info = mats[f"dec.L0.{n}"]
        if info.rows * info.cols > 30_000_000:
            off += int(np.prod(geometry(info.rows, info.cols, MODES[n]))) * TILE
            continue
        want, planes = pack(_bits(eng, info), MODES[n], cfg.head_dim, esc0)   # escape entries are numbered in tile order
        esc0 += planes.shape[0]
        got = np.empty(want.size, np.uint8)
        assert eng.lib.dtk_dbg_pack_bytes(eng._h, off, got.size, got.ctypes.data_as(C.c_void_p)) == 0
        assert np.array_equal(got.reshape(want.shape), want), n
        off += want.size


def test_pack_is_bit_identical_across_contexts(model):
    eng = model.engine
    g = torch.Generator().manual_seed(6100)
    ids = torch.randint(3, 30000, (2048,), generator=g).cuda()
    slot = eng.seq_alloc()
    try:
        for T in CONTEXTS:
            eng.prefill(slot, ids[:T], 0, None, 0)
            on = _decode(eng, slot, T, int(ids[T]), 1)
            off = _decode(eng, slot, T, int(ids[T]), 0)
            assert torch.isfinite(on).all(), T
            assert torch.equal(on, off), T
    finally:
        eng.set_option("decode_pack", 1)
        eng.seq_free(slot)


def test_pack_is_bit_identical_on_a_borrower(model):
    eng = model.engine
    g = torch.Generator().manual_seed(6200)
    prefix = torch.randint(3, 30000, (253,), generator=g).cuda()
    suffix = torch.randint(3, 30000, (40,), generator=g).cuda()
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    try:
        eng.prefill(base, prefix, 0, None, 0)
        eng.seq_share(base, sub, prefix.numel())
        eng.prefill(sub, suffix, prefix.numel(), None, 0)
        T = prefix.numel() + suffix.numel()
        assert torch.equal(_decode(eng, sub, T, 17, 1), _decode(eng, sub, T, 17, 0))
    finally:
        eng.set_option("decode_pack", 1)
        eng.seq_free(sub)
        eng.seq_free(base)


def test_pack_is_bit_identical_over_consecutive_launches_and_greedy_loop(model):
    eng, cfg = model.engine, model.config
    g = torch.Generator().manual_seed(6300)
    ids = torch.randint(3, 30000, (300,), generator=g).cuda()
    toks = torch.randint(3, 30000, (12,), generator=g).tolist()
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    steps = 40
    logits, greedy = {}, {}
    try:
        for pk in (1, 0):
            eng.set_option("decode_pack", pk)
            eng.prefill(slot, ids, 0, None, 0)
            logits[pk] = torch.stack([eng.decode([slot], [ids.numel() + i], torch.tensor([t], device="cuda"))[0].clone()
                                      for i, t in enumerate(toks)]).cpu()
            for variant in (0, 1):
                eng.set_option("mega_variant", variant)
                last, _ = eng.prefill(slot, ids, 0, None, 0)
                first, _ = eng.sample(last, params)
                eng.gen_begin([slot], [ids.numel()], [int(first)], params)
                got = [int(first)]
                for i in range(steps):
                    eng.gen_step()
                    got.append(eng.gen_wait(i)[0])
                eng.gen_end()
                greedy[pk, variant] = got
                eng.set_option("mega_variant", 0)
    finally:
        eng.set_option("mega_variant", 0)
        eng.set_option("decode_pack", 1)
        eng.seq_free(slot)
    assert torch.equal(logits[1], logits[0])
    assert greedy[1, 0] == greedy[0, 0] == greedy[1, 1] == greedy[0, 1]


def test_pack_decode_weight_bytes(model):
    eng, cfg = model.engine, model.config
    mats = _matrices(eng)
    want = _packed_bytes(cfg, mats) + eng.get_option("decode_pack_escapes") * 4096
    assert eng.get_option("decode_pack_escapes") < 1e-3 * want / TILE   # rare: exact zeros of the random init, mostly
    assert eng.get_option("decode_weight_bytes") == want
    kv = eng.lib.dtk_decode_bytes(C.byref(eng.ccfg), 512) - eng.lib.dtk_decode_bytes(C.byref(eng.ccfg), 0)
    assert eng.decode_bytes(512) == want + kv
    try:
        eng.set_option("decode_pack", 0)
        H, I, V, L = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_hidden_layers
        qd, kd = cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
        assert eng.get_option("decode_weight_bytes") == 2 * L * ((qd + 2 * kd) * H + H * qd + 3 * H * I) + 2 * V * H
    finally:
        eng.set_option("decode_pack", 1)


def test_pack_escape_tiles_are_bit_identical(model):
    """Values the 5-bit code cannot reach: a zero and a subnormal in rows with base > 0, a value 58 binades below its row's
    largest one (escape tiles), +-128 (a row base far above the others), and a row of subnormals (base 0: no escape by
    itself), in layer 0 and the lm_head."""
    eng, cfg = model.engine, model.config
    mats = _matrices(eng)
    edits = [("dec.L0.wqkv", 3, 5, 0x0000), ("dec.L0.wo", 17, 300, 0x0001), ("dec.L0.wgu", 40, 7, 0x2000),
             ("dec.L0.wd", 2, 1000, 0x4300), ("dec.L0.wd", 3, 1001, 0xC300), ("dec.lm_head", 33, 100, 0x0000)]
    saved = []
    g = torch.Generator().manual_seed(6400)
    ids = torch.randint(3, 30000, (400,), generator=g).cuda()
    slot = eng.seq_alloc()
    flat = eng.arena.view(torch.int16)
    n0 = eng.get_option("decode_pack_escapes")
    try:
        for name, r, c, v in edits:
            info = mats[name]
            i = info.offset // 2 + r * info.cols + c
            saved.append((i, flat[i].clone()))
            flat[i] = int(np.array(v, np.uint16).view(np.int16))
        info = mats["dec.L0.wo"]
        i0 = info.offset // 2 + 50 * info.cols
        saved.append((slice(i0, i0 + info.cols), flat[i0:i0 + info.cols].clone()))
        flat[i0:i0 + info.cols] = torch.randint(1, 0x80, (info.cols,), device=flat.device).to(torch.int16)   # subnormals
        eng.set_option("decode_pack", 0)   # rebuild both tile sets from the edited arena
        eng.set_option("decode_pack", 1)
        assert eng.get_option("decode_pack_escapes") >= n0 + 3
        assert eng.get_option("decode_weight_bytes") == _packed_bytes(cfg, mats) + eng.get_option("decode_pack_escapes") * 4096
        eng.prefill(slot, ids, 0, None, 0)
        on = _decode(eng, slot, ids.numel(), 11, 1)
        off = _decode(eng, slot, ids.numel(), 11, 0)
        assert torch.equal(on, off)
    finally:
        for i, v in saved:
            flat[i] = v
        eng.set_option("decode_pack", 0)
        eng.set_option("decode_pack", 1)
        eng.seq_free(slot)
    assert eng.get_option("decode_pack_escapes") == n0


def test_switching_formats_keeps_each_modes_logits():
    """A quantized arena runs in all three formats (bf16, e4m3, packed) with the same logits; every switch frees the previous
    tiles, and a per-token graph captured before a switch (per-op batch-1 loop) is rebuilt after it."""
    from detikzify_b200.model import load
    m, _ = load("nllg/detikzify-ds-1.3b", device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=2,
                max_batch=1, quantize="fp8")
    eng, cfg = m.engine, m.config
    g = torch.Generator().manual_seed(6500)
    ids = torch.randint(3, 30000, (300,), generator=g).cuda()
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)

    def step():
        return eng.decode([slot], [ids.numel()], torch.tensor([19], device="cuda"))[0].clone()

    def loop(impl):
        eng.set_option("decode_impl", impl)
        last, _ = eng.prefill(slot, ids, 0, None, 0)
        first, _ = eng.sample(last, params)
        eng.gen_begin([slot], [ids.numel()], [int(first)], params)
        got = [int(first)]
        for i in range(8):
            eng.gen_step()
            got.append(eng.gen_wait(i)[0])
        eng.gen_end()
        eng.set_option("decode_impl", 1)
        return got

    try:
        eng.prefill(slot, ids, 0, None, 0)
        assert eng.get_option("decode_fp8") == 1 and eng.get_option("decode_pack") == 0
        ref = step()
        ref_ids = loop(1)
        per_op = loop(0)   # captures the per-op graph of the loop
        for key, value in [("decode_pack", 1), ("decode_fp8", 0), ("decode_pack", 1), ("decode_fp8", 1), ("decode_pack", 1),
                           ("decode_pack", 0), ("decode_fp8", 1), ("decode_fp8", 0), ("decode_pack", 1)]:
            eng.set_option(key, value)
            assert eng.get_option("decode_fp8") + eng.get_option("decode_pack") <= 1
            eng.prefill(slot, ids, 0, None, 0)
            assert torch.equal(step(), ref), (key, value)
            assert loop(1) == ref_ids and loop(0) == per_op, (key, value)
    finally:
        eng.seq_free(slot)
        del m
        torch.cuda.empty_cache()
