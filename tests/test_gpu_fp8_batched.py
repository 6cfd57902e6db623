"""
FP8 decoder weights on the batched decode step (4 <= B < 64: MCTS rollouts, ``generate_batch``, ``sample_batch``).

With ``decode_fp8`` the four layer GEMMs of the batched step read the e4m3 decode tiles on the swapped-operand wgmma tile
and rebuild W~ = code x 2^k_r in registers. The arena of a quantized model holds the same W~ in bf16, and the FP8 tile cuts
K at the same 64-k blocks and sums the split-K ranks in the same order, so on one engine the batched logits must be
bit-identical with the option on and off:
  * at the ds-1.3b (head_dim 128; wd K = 5504 is not a multiple of 256), tl-1.1b (head_dim 64, GQA 32/4) and v2-8b-2l
    (GQA 32/8, V 128256) shapes, weights generated on the device and quantized as load() does: B in {4, 5, 17, 32, 33, 63}
    (both column widths of the tile, ragged column counts) at ragged positions, every forced split-K factor at B = 32,
    32 rows borrowing one 253-position prefix (shared-prefix attention), and the device-resident loop at B = 8 run with
    the option 1 -> 0 -> 1 (the cached step graph must follow the re-tiled weights);
  * the step really reads the tiles: zeroing a matrix in the arena leaves the FP8 logits unchanged;
  * the public path against the fp32 oracle on the quantized state dict: generate_batch of 4 prompts at tiny / tiny-tl /
    tiny-v2, and teacher-forced batched logits at ds-7b-2l (8 % of the reference logits' RMS, as test_gpu_ds7b.py).
"""
import re

import pytest
import torch

from conftest import model_bundle

pytestmark = pytest.mark.gpu
BATCHES = (4, 5, 17, 32, 33, 63)
LAYER_MATRIX = re.compile(r"model\.layers\.\d+\.(self_attn\.[qkvo]_proj|mlp\.(gate|up|down)_proj)\.weight$")


def _quantized_sd(sd):
    from detikzify_b200.quant import quantize_fp8_rows
    return {k: quantize_fp8_rows(v.to(torch.bfloat16)) if LAYER_MATRIX.match(k) else v for k, v in sd.items()}


@pytest.fixture(scope="module", params=["nllg/detikzify-ds-1.3b", "nllg/detikzify-tl-1.1b", "v2-8b-2l"])
def model(request):
    """the model load(..., device_init=True, quantize="fp8") builds, with 64 KV slots of 512 positions (every row of a
    63-row step needs a slot of its own; 2048-position slots would hold 26 GB at ds-1.3b)"""
    from detikzify_b200.engine import random_arena_device, to_c_config, weight_table
    from detikzify_b200.model import DetikzifyForCausalLM, preset
    from detikzify_b200.quant import quantize_arena_fp8
    cfg = preset(request.param)
    arena = random_arena_device(cfg, 0, seed=0)
    quantize_arena_fp8(arena, weight_table(to_c_config(cfg)))
    m = DetikzifyForCausalLM(cfg, arena, device=0, max_seqs=64, max_batch=64, max_len=512)
    del arena
    m.engine.set_option("decode_fp8", 1)
    yield m
    m.engine.close()
    del m
    torch.cuda.empty_cache()


def _prefill_rows(eng, n, seed):
    """n slots with ragged prompts (30 + 7 i tokens) and one next token each"""
    g = torch.Generator().manual_seed(seed)
    slots, lens = [], []
    for i in range(n):
        ids = torch.randint(3, 30000, (30 + 7 * i,), generator=g)
        s = eng.seq_alloc()
        eng.prefill(s, ids.cuda(), 0, None, 0)
        slots.append(s)
        lens.append(ids.numel())
    return slots, lens, torch.randint(3, 30000, (n,), generator=g)


def _step(eng, slots, lens, toks, fp8):
    eng.set_option("decode_fp8", fp8)
    return eng.decode(slots, lens, toks.cuda()).clone()


def test_fp8_batched_step_is_bit_identical(model):
    eng = model.engine
    assert eng.get_option("decode_fp8") == 1 and eng.get_option("decode_gemm_min_batch") == 4
    slots, lens, toks = _prefill_rows(eng, max(BATCHES), 6100)
    try:
        for B in BATCHES:
            on = _step(eng, slots[:B], lens[:B], toks[:B], 1)
            off = _step(eng, slots[:B], lens[:B], toks[:B], 0)
            assert torch.isfinite(on).all(), B
            assert torch.equal(on, off), B
    finally:
        eng.set_option("decode_fp8", 1)
        for s in slots:
            eng.seq_free(s)


def test_fp8_batched_step_is_bit_identical_at_every_split(model):
    eng = model.engine
    B = 32
    slots, lens, toks = _prefill_rows(eng, B, 6200)
    try:
        for split in (1, 2, 3, 8, 0):   # forced split-K factors, then the heuristic
            eng.set_option("gemm_swap_split", split)
            on = _step(eng, slots, lens, toks, 1)
            off = _step(eng, slots, lens, toks, 0)
            assert torch.equal(on, off), split
    finally:
        eng.set_option("gemm_swap_split", 0)
        eng.set_option("decode_fp8", 1)
        for s in slots:
            eng.seq_free(s)


def test_fp8_batched_step_reads_the_tiles(model):
    from detikzify_b200.engine import weight_table
    eng = model.engine
    B = 17
    slots, lens, toks = _prefill_rows(eng, B, 6300)
    info = next(w for w in weight_table(eng.ccfg) if w.name.decode() == "dec.L0.wd")
    view = eng.arena[info.offset // 2: info.offset // 2 + info.rows * info.cols]
    saved = view.clone()
    try:
        on = _step(eng, slots, lens, toks, 1)
        view.zero_()
        torch.cuda.synchronize()
        assert torch.equal(_step(eng, slots, lens, toks, 1), on)    # the FP8 step does not read the arena's matrix
        assert not torch.equal(_step(eng, slots, lens, toks, 0), on)   # the bf16 step does
    finally:
        view.copy_(saved)
        torch.cuda.synchronize()
        eng.set_option("decode_fp8", 0)   # re-tile from the restored arena
        eng.set_option("decode_fp8", 1)
        for s in slots:
            eng.seq_free(s)


def test_fp8_batched_step_on_a_shared_prefix(model):
    eng = model.engine
    B = 32
    g = torch.Generator().manual_seed(6400)
    prefix = torch.randint(3, 30000, (253,), generator=g).cuda()
    base = eng.seq_alloc()
    subs = []
    try:
        eng.prefill(base, prefix, 0, None, 0)
        lens = []
        for i in range(B):
            s = eng.seq_alloc()
            subs.append(s)
            eng.seq_share(base, s, prefix.numel())
            suf = torch.randint(3, 30000, (1 + i % 5,), generator=g).cuda()
            eng.prefill(s, suf, prefix.numel(), None, 0)
            lens.append(prefix.numel() + suf.numel())
        toks = torch.randint(3, 30000, (B,), generator=g)
        on = _step(eng, subs, lens, toks, 1)
        off = _step(eng, subs, lens, toks, 0)
        assert torch.isfinite(on).all()
        assert torch.equal(on, off)
    finally:
        eng.set_option("decode_fp8", 1)
        for s in subs:
            eng.seq_free(s)
        eng.seq_free(base)


def test_fp8_generation_loop_follows_the_retiled_weights(model):
    eng, cfg = model.engine, model.config
    B, steps = 8, 24
    slots, lens, toks = _prefill_rows(eng, B, 6500)
    runs = {}
    try:
        for name, params in (("greedy", eng.sampling(do_sample=False, bad_token=cfg.image_token_id)),
                             ("nucleus", eng.sampling(temperature=0.8, top_p=0.95, do_sample=True,
                                                      bad_token=cfg.image_token_id, seed=11))):
            for i, fp8 in enumerate((1, 0, 1)):   # the same graph key after each re-tile
                eng.set_option("decode_fp8", fp8)
                eng.gen_begin(slots, lens, toks.tolist(), params, seq_ids=list(range(B)))
                got = []
                for t in range(steps):
                    eng.gen_step()
                    got.append(eng.gen_wait(t))
                eng.gen_end()
                runs[name, i] = got
    finally:
        eng.set_option("decode_fp8", 1)
        for s in slots:
            eng.seq_free(s)
    for name in ("greedy", "nucleus"):
        assert runs[name, 0] == runs[name, 1] == runs[name, 2], name


@pytest.mark.parametrize("name", ["tiny", "tiny-tl", "tiny-v2"])
def test_fp8_generate_batch_matches_oracle_on_quantized_weights(name):
    from detikzify_b200.model import load
    from oracle.hf_oracle import Oracle, synthetic_pixels
    cfg, sd, _ = model_bundle(name)
    oracle = Oracle(cfg.to_dict(), _quantized_sd(sd))
    model, _ = load(name, device_map=0, state_dict=sd, quantize="fp8", max_seqs=6, max_batch=4)
    assert model.engine.get_option("decode_fp8") == 1
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=1000)
    span = torch.full((cfg.num_patches,), cfg.patch_token_id)
    prompts = [torch.cat([span, torch.tensor(t)]).long() for t in ([5, 6, 7], [5, 6, 9, 11], [5, 8], [5, 6, 7, 12, 13])]
    steps, TOL = 16, 3e-2
    got = model.generate_batch(prompts, pix, bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
                               max_new_tokens=steps, do_sample=False)
    for ids, out in zip(prompts, got):
        T0 = ids.numel()
        ref = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
        out = out.cpu()
        n = min(out.numel(), ref.numel())
        assert n > T0
        diff = (out[:n] != ref[:n]).nonzero()
        if diff.numel():   # a divergence is only tolerated at a near-tie of the fp32 logits
            t = int(diff[0])
            ref_logits, _ = oracle.forward_logits(ref[None], pix)
            top2 = ref_logits[0, t - 1].topk(2).values
            assert (top2[0] - top2[1]).item() < 2 * TOL, (t, top2)


def test_fp8_batched_decode_matches_oracle_at_ds7b_shape():
    from detikzify_b200.engine import Engine, pack_arena
    from oracle.hf_oracle import Oracle, synthetic_pixels
    cfg, sd, _ = model_bundle("ds-7b-2l")
    sdq = _quantized_sd(sd)
    oracle = Oracle(cfg.to_dict(), sdq)
    B = 8
    eng = Engine(cfg, pack_arena(cfg, sdq), device=0, max_seqs=B, max_batch=B)
    try:
        eng.set_option("decode_fp8", 1)
        pix = synthetic_pixels(1, cfg.vision_config.image_size)
        img = eng.image_embeds(pix.cuda())[0]
        g = torch.Generator().manual_seed(7200)
        P = cfg.num_patches
        prompts = [torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(0, 32000, (10 + 5 * i,), generator=g)]).long()
                   for i in range(B)]
        tok = torch.randint(0, 32000, (B,), generator=g)
        slots = [eng.seq_alloc() for _ in range(B)]
        for s, ids in zip(slots, prompts):
            eng.prefill(s, ids.cuda(), 0, img, 0)
        step = eng.decode(slots, [p.numel() for p in prompts], tok.cuda()).cpu()
        for i in (0, 3, 7):
            ref, _ = oracle.forward_logits(torch.cat([prompts[i], tok[i:i + 1]])[None], pix)
            TOL = max(3e-2, 0.08 * ref.float().pow(2).mean().sqrt().item())
            assert (step[i] - ref[0, -1]).abs().max().item() < TOL, i
    finally:
        eng.close()
