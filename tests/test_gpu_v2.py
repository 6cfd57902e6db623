"""
v2 / v2.5 model shapes on the CUDA path (SURVEY.md section 8 f4; reference detikzify/model/configuration_detikzify.py:31-58,
83-120, modeling_detikzify.py:62-86,165-179,181-271): 420-px-style tower (N % 3 == 0), bias-free connector, GQA decoder with
llama3 RoPE scaling, V = 128256 (the generic sampler: the register-resident one holds 32768 logits).
  * tiny-v2: against the golden vectors the REFERENCE's own v2 module produced (tests/golden/reference_v2_tiny.pt);
  * v2-8b-2l: every detikzify-v2-8b matrix shape with two decoder layers against the fp32 oracle, batch 1 on the persistent
    kernel and on the per-op kernels, batched-GEMM decode, and the sampler at V = 128256.
Tolerance: logits max-abs 3e-2 at the tiny shape; at the 8b shapes 8 % of the reference logits' RMS (see test_gpu_ds7b.py).
"""
from pathlib import Path

import pytest
import torch

from conftest import engine_for, model_bundle

pytestmark = pytest.mark.gpu
TOL = 3e-2
GOLD = Path(__file__).parent / "golden" / "reference_v2_tiny.pt"


def _pixels(cfg, batch, seed=1000):
    from oracle.hf_oracle import synthetic_pixels
    return synthetic_pixels(batch, cfg.vision_config.image_size, seed)


@pytest.mark.parametrize("impl", [1, 0], ids=["persistent", "per-op"])
def test_tiny_v2_matches_reference_v2_module(impl):
    gold = torch.load(GOLD, weights_only=False)["tiny-v2"]
    cfg, sd, oracle = model_bundle("tiny-v2", seed=gold["seed"])
    eng = engine_for("tiny-v2", seed=gold["seed"])
    pix = _pixels(cfg, 1, seed=gold["pixel_seed"])
    ids = gold["input_ids"].long()
    start = int((ids == cfg.image_token_id).nonzero()[0])
    img = eng.image_embeds(pix.cuda())[0]
    assert (img.cpu() - gold["image_embeds"]).abs().max().item() < 2e-2
    slot = eng.seq_alloc()
    eng.set_option("decode_impl", impl)
    try:
        last, alll = eng.prefill(slot, ids.cuda(), 0, img, start, want_all_logits=True)
        assert (alll.cpu() - gold["logits"]).abs().max().item() < TOL
        lg = eng.decode([slot], [ids.numel()], torch.tensor([gold["next_id"]], device="cuda"))[0].cpu()
        assert (lg - gold["decode_logits"]).abs().max().item() < TOL
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)


def test_tiny_v2_public_generate_matches_reference_ids():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    gold = torch.load(GOLD, weights_only=False)["tiny-v2"]
    cfg, sd, oracle = model_bundle("tiny-v2", seed=gold["seed"])
    model = DetikzifyForCausalLM(cfg, engine=engine_for("tiny-v2", seed=gold["seed"]))
    pix = _pixels(cfg, 1, seed=gold["pixel_seed"])
    ref = gold["generate_ids"]
    out = model.generate(input_ids=gold["generate_prompt"][None], pixel_values=pix, bad_words_ids=[[cfg.image_token_id]],
                         begin_suppress_tokens=[cfg.eos_token_id], max_length=ref.numel(), do_sample=False)
    got = out[0].cpu()
    n = min(got.numel(), ref.numel())
    diff = (got[:n] != ref[:n]).nonzero()
    if diff.numel():
        t = int(diff[0])   # a divergence is only tolerated at a near-tie of the fp32 logits
        logits, _ = oracle.forward_logits(ref[None, :t], pix)
        top2 = logits[0, -1].topk(2).values
        assert (top2[0] - top2[1]).item() < 2 * TOL, (t, top2)
    else:
        assert got.numel() == ref.numel()


def test_v2_8b_shapes_decode_and_sampler():
    name = "v2-8b-2l"
    cfg, sd, oracle = model_bundle(name)
    assert (cfg.num_attention_heads, cfg.num_key_value_heads, cfg.vocab_size, cfg.intermediate_size) == (32, 8, 128256, 14336)
    B = 8
    eng = engine_for(name, max_seqs=B + 1, max_batch=B)
    pix = _pixels(cfg, 1)
    img = eng.image_embeds(pix.cuda())[0]
    P = cfg.num_patches
    g = torch.Generator().manual_seed(8000)
    prompts = [torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(0, 128000, (30 + 5 * i,), generator=g)]).long() for i in range(B)]
    tok1 = torch.randint(0, 128000, (B,), generator=g)
    slots = [eng.seq_alloc() for _ in range(B)]
    try:
        lens = []
        for s, ids in zip(slots, prompts):
            last, _ = eng.prefill(s, ids.cuda(), 0, img, 0)
            lens.append(ids.numel())
        ref0, _ = oracle.forward_logits(torch.cat([prompts[B - 1], tok1[B - 1:]])[None], pix)
        TOL = max(3e-2, 0.08 * ref0.pow(2).mean().sqrt().item())
        assert (last.cpu() - ref0[0, -2]).abs().max().item() < TOL          # prefill last row of the longest prompt
        # batch-1 decode on both implementations (GQA attention: several key ranges per head)
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            lg = eng.decode([slots[B - 1]], [lens[B - 1]], tok1[B - 1:].cuda())[0].cpu()
            assert (lg - ref0[0, -1]).abs().max().item() < TOL, impl
        eng.set_option("decode_impl", 1)
        # kernel variants (bit 1: arrival counter, bit 2: two tiles per consumer-warp iteration) sum in the same order
        base = eng.decode([slots[B - 1]], [lens[B - 1]], tok1[B - 1:].cuda())[0].clone()
        for variant in (2, 4, 6):
            eng.set_option("mega_variant", variant)
            assert torch.equal(eng.decode([slots[B - 1]], [lens[B - 1]], tok1[B - 1:].cuda())[0], base), variant
        eng.set_option("mega_variant", 0)
        # batched-GEMM decode of all 8 sequences (rewrites the same KV rows)
        step = eng.decode(slots, lens, tok1.cuda()).clone()
        for i in (0, 3, B - 1):
            ref, _ = oracle.forward_logits(torch.cat([prompts[i], tok1[i:i + 1]])[None], pix)
            assert (step[i].cpu() - ref[0, -1]).abs().max().item() < TOL, i
        # sampler at V = 128256 (generic kernel): nucleus probability vector vs the HF processor chain, greedy = argmax
        params = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id,
                              begin_suppress_token=cfg.eos_token_id, seed=5)
        out, probs = eng.sample(step, params, suppress=[1] * B, steps=list(range(B)), seq_ids=list(range(B)), want_probs=True)
        for i in (0, B - 1):
            ref_p = oracle.processed_probs(torch.zeros(1, lens[i], dtype=torch.long), step[i:i + 1].cpu(), lens[i],
                                           temperature=0.8, top_p=0.95, top_k=0)[0]
            got = probs[i].cpu()
            mism = ((ref_p > 0) != (got > 0)).sum()
            assert mism <= 1, (i, mism)
            if mism == 0:
                assert (got - ref_p).abs().max() < 1e-5
            assert got[cfg.image_token_id] == 0 and got[cfg.eos_token_id] == 0 and got[int(out[i])] > 0
        gp = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
        gout, _ = eng.sample(step, gp, suppress=[0] * B)
        masked = step.clone()
        masked[:, cfg.image_token_id] = -float("inf")
        assert gout.cpu().tolist() == masked.argmax(-1).cpu().tolist()
    finally:
        eng.set_option("decode_impl", 1)
        for s in slots:
            eng.seq_free(s)
