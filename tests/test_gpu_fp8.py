"""
FP8 decoder weights (``load(..., quantize="fp8")``, engine option ``decode_fp8``) on the GPU.

The quantized arena holds W~ = e4m3 code x 2^k_r per row, exactly representable in bf16. With ``decode_fp8`` the batch-1
persistent kernel streams the codes and row exponents instead of the bf16 values and rebuilds the same bf16 bits in
registers, so on one engine its logits must be bit-identical with the option on and off:
  * at the ds-1.3b (head_dim 128, MHA), tl-1.1b (head_dim 64, GQA 32/4) and v2-8b-2l (GQA 32/8, V 128256) shapes, weights
    generated on the device and quantized as load() does: single steps at contexts around the 16-position KV items up to
    2047, a borrower of a 253-position shared prefix, back-to-back launches, and the greedy ids of the device-resident
    loop with mega_variant 0 and 1;
  * the public path against the fp32 oracle built from the quantized state dict: generate() at tiny / tiny-tl / tiny-v2,
    teacher-forced persistent decode at ds-7b-2l and v2-8b-2l (8 % of the reference logits' RMS, as test_gpu_ds7b.py);
  * an arena that is not quantized is refused, and the engine keeps decoding as before;
  * ``decode_weight_bytes`` counts the bytes the kernel streams in each mode.
"""
import ctypes as C
import re

import pytest
import torch

from conftest import model_bundle

pytestmark = pytest.mark.gpu
CONTEXTS = (243, 255, 256, 257, 271, 272, 1023, 1145, 1536, 2000, 2047)
LAYER_MATRIX = re.compile(r"model\.layers\.\d+\.(self_attn\.[qkvo]_proj|mlp\.(gate|up|down)_proj)\.weight$")


def _quantized_sd(sd):
    from detikzify_b200.quant import quantize_fp8_rows
    return {k: quantize_fp8_rows(v.to(torch.bfloat16)) if LAYER_MATRIX.match(k) else v for k, v in sd.items()}


def _weight_bytes(cfg, fp8):
    H, I, V, L = cfg.hidden_size, cfg.intermediate_size, cfg.vocab_size, cfg.num_hidden_layers
    qd, kd = cfg.num_attention_heads * cfg.head_dim, cfg.num_key_value_heads * cfg.head_dim
    w = L * ((qd + 2 * kd) * H + H * qd + 3 * H * I)
    rows = L * ((qd + 2 * kd) + H + 2 * I + H)
    return (w + rows if fp8 else 2 * w) + 2 * V * H


@pytest.fixture(scope="module", params=["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b", "v2-8b-2l"])
def model(request):
    from detikzify_b200.model import load
    m, _ = load(request.param, device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=4, max_batch=1,
                quantize="fp8")
    yield m
    del m
    torch.cuda.empty_cache()


def _decode(eng, slot, pos, tok, fp8):
    eng.set_option("decode_fp8", fp8)
    return eng.decode([slot], [pos], torch.tensor([tok], device="cuda"))[0].clone()


def test_fp8_is_bit_identical_across_contexts(model):
    eng = model.engine
    assert eng.get_option("decode_persistent") == 1 and eng.get_option("decode_fp8") == 1
    g = torch.Generator().manual_seed(5100)
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
        eng.set_option("decode_fp8", 1)
        eng.seq_free(slot)


def test_fp8_is_bit_identical_on_a_borrower(model):
    eng = model.engine
    g = torch.Generator().manual_seed(5200)
    prefix = torch.randint(3, 30000, (253,), generator=g).cuda()
    suffix = torch.randint(3, 30000, (40,), generator=g).cuda()
    base, sub = eng.seq_alloc(), eng.seq_alloc()
    try:
        eng.prefill(base, prefix, 0, None, 0)
        eng.seq_share(base, sub, prefix.numel())
        eng.prefill(sub, suffix, prefix.numel(), None, 0)
        T = prefix.numel() + suffix.numel()
        on = _decode(eng, sub, T, 17, 1)
        off = _decode(eng, sub, T, 17, 0)
        assert torch.equal(on, off)
    finally:
        eng.set_option("decode_fp8", 1)
        eng.seq_free(sub)
        eng.seq_free(base)


def test_fp8_is_bit_identical_over_consecutive_launches_and_greedy_loop(model):
    eng, cfg = model.engine, model.config
    g = torch.Generator().manual_seed(5300)
    ids = torch.randint(3, 30000, (300,), generator=g).cuda()
    toks = torch.randint(3, 30000, (12,), generator=g).tolist()
    slot = eng.seq_alloc()
    params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    steps = 40
    logits, greedy = {}, {}
    try:
        for fp8 in (1, 0):
            eng.set_option("decode_fp8", fp8)
            eng.prefill(slot, ids, 0, None, 0)
            # back-to-back launches without a host round trip in between
            logits[fp8] = torch.stack([eng.decode([slot], [ids.numel() + i], torch.tensor([t], device="cuda"))[0].clone()
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
                greedy[fp8, variant] = got
                eng.set_option("mega_variant", 0)
    finally:
        eng.set_option("mega_variant", 0)
        eng.set_option("decode_fp8", 1)
        eng.seq_free(slot)
    assert torch.equal(logits[1], logits[0])
    assert greedy[1, 0] == greedy[0, 0] == greedy[1, 1] == greedy[0, 1]


def test_fp8_decode_weight_bytes(model):
    eng, cfg = model.engine, model.config
    try:
        for fp8 in (1, 0):
            eng.set_option("decode_fp8", fp8)
            assert eng.get_option("decode_weight_bytes") == _weight_bytes(cfg, fp8)
            kv = eng.lib.dtk_decode_bytes(C.byref(eng.ccfg), 512) - eng.lib.dtk_decode_bytes(C.byref(eng.ccfg), 0)
            assert eng.decode_bytes(512) == _weight_bytes(cfg, fp8) + kv
    finally:
        eng.set_option("decode_fp8", 1)


@pytest.mark.parametrize("name", ["tiny", "tiny-tl", "tiny-v2"])
def test_fp8_generate_matches_oracle_on_quantized_weights(name):
    from detikzify_b200.model import load
    from oracle.hf_oracle import Oracle, synthetic_pixels
    cfg, sd, _ = model_bundle(name)
    sdq = _quantized_sd(sd)
    oracle = Oracle(cfg.to_dict(), sdq)
    model, _ = load(name, device_map=0, state_dict=sd, quantize="fp8", max_seqs=2)
    assert model.engine.get_option("decode_fp8") == 1 and model.engine.get_option("decode_persistent") == 1
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=1000)
    ids = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.tensor([5, 6, 7])]).long()
    T0, steps, TOL = ids.numel(), 16, 3e-2
    ref = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
    got = model.generate(input_ids=ids[None], pixel_values=pix, bad_words_ids=[[cfg.image_token_id]],
                         begin_suppress_tokens=[cfg.eos_token_id], max_length=T0 + steps, do_sample=False)[0].cpu()
    n = min(got.numel(), ref.numel())
    assert n > T0
    ref_logits, _ = oracle.forward_logits(ref[None], pix)
    diff = (got[:n] != ref[:n]).nonzero()
    if diff.numel():   # a divergence is only tolerated at a near-tie of the fp32 logits
        t = int(diff[0])
        top2 = ref_logits[0, t - 1].topk(2).values
        assert (top2[0] - top2[1]).item() < 2 * TOL, (t, top2)
    # the engine's own teacher-forced logits along the oracle's ids, on the persistent fp8 kernel
    eng = model.engine
    img = eng.image_embeds(pix.cuda())[0]
    slot = eng.seq_alloc()
    try:
        last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
        worst = (last.cpu() - ref_logits[0, T0 - 1]).abs().max().item()
        for t in range(T0, T0 + 8):
            lg = eng.decode([slot], [t], ref[t:t + 1].cuda())[0].cpu()
            worst = max(worst, (lg - ref_logits[0, t]).abs().max().item())
        assert worst < TOL, worst
    finally:
        eng.seq_free(slot)


@pytest.mark.parametrize("name", ["ds-7b-2l", "v2-8b-2l"])
def test_fp8_persistent_decode_matches_oracle_at_large_shapes(name):
    from detikzify_b200.engine import Engine, pack_arena
    from oracle.hf_oracle import Oracle, synthetic_pixels
    cfg, sd, _ = model_bundle(name)
    sdq = _quantized_sd(sd)
    oracle = Oracle(cfg.to_dict(), sdq)
    eng = Engine(cfg, pack_arena(cfg, sdq), device=0, max_seqs=2, max_batch=1)
    try:
        eng.set_option("decode_fp8", 1)
        assert eng.get_option("decode_persistent") == 1
        pix = synthetic_pixels(1, cfg.vision_config.image_size)
        img = eng.image_embeds(pix.cuda())[0]
        g = torch.Generator().manual_seed(7100)
        P = cfg.num_patches
        ids = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(3, 32000, (30,), generator=g)]).long()
        T0, steps = ids.numel(), 6
        ref_ids = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
        ref_all, _ = oracle.forward_logits(ref_ids[None], pix)
        TOL = max(3e-2, 0.08 * ref_all.float().pow(2).mean().sqrt().item())
        slot = eng.seq_alloc()
        last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
        worst = (last.cpu() - ref_all[0, T0 - 1]).abs().max().item()
        for t in range(T0, T0 + steps - 1):
            lg = eng.decode([slot], [t], ref_ids[t:t + 1].cuda())[0].cpu()
            worst = max(worst, (lg - ref_all[0, t]).abs().max().item())
        assert worst < TOL, worst
        eng.seq_free(slot)
    finally:
        eng.close()


def test_fp8_refused_on_unquantized_weights():
    from detikzify_b200.engine import Engine, EngineError, pack_arena
    cfg, sd, _ = model_bundle("tiny")
    eng = Engine(cfg, pack_arena(cfg, sd), device=0, max_seqs=2, max_batch=1)
    try:
        slot = eng.seq_alloc()
        ids = torch.arange(3, 40).cuda()
        eng.prefill(slot, ids, 0, None, 0)
        before = [eng.decode([slot], [ids.numel() + i], torch.tensor([9 + i], device="cuda"))[0].clone() for i in range(3)]
        with pytest.raises(EngineError, match=r"decode_fp8: layer 0 wqkv"):
            eng.set_option("decode_fp8", 1)
        assert eng.get_option("decode_fp8") == 0
        assert eng.get_option("decode_weight_bytes") == _weight_bytes(cfg, 0)
        eng.prefill(slot, ids, 0, None, 0)
        after = [eng.decode([slot], [ids.numel() + i], torch.tensor([9 + i], device="cuda"))[0].clone() for i in range(3)]
        for a, b in zip(before, after):
            assert torch.equal(a, b)
    finally:
        eng.close()
