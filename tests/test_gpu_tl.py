"""
detikzify-tl-1.1b (TinyLlama-1.1B decoder: head_dim 64, GQA 32/4, V 32008) on the CUDA engine, and the cl-7b matrix shapes:

  * ``tiny-tl`` against the reference's own model code (tests/golden/reference_v1_tl.pt), through the C ABI and ``generate()``;
  * ``tl-1.1b`` at the real shape against the reference golden and the fp32 oracle: prefill, 24 teacher-forced decode steps on
    the persistent kernel and the per-op kernels, context checkpoints 512 / 1024 / 1536 / 2047;
  * B = 2 (per-op GEMV) and B = 32 (batched GEMM) decode on ragged contexts, two steps, and the nucleus probability vector;
  * shared KV prefixes: cascade on / off, persistent decode on a borrower, prefix-cache reuse in ``generate()``,
    ``generate_batch`` against per-sequence ``generate()``;
  * ``cl-7b-2l`` (every CodeLlama-7b matrix shape, two layers): prefill and batch-1 decode on both implementations.

Tolerance and greedy-margin rule as in test_gpu_ds13b.py: logits max-abs 3e-2 (|logits| ~ 1), greedy ids equal wherever the
oracle's top-1 margin exceeds twice that.
"""
from pathlib import Path

import pytest
import torch

from conftest import engine_for, model_bundle

pytestmark = pytest.mark.gpu
NAME = "nllg/detikzify-tl-1.1b"
TOL = 3e-2
GOLD = torch.load(Path(__file__).parent / "golden" / "reference_v1_tl.pt", weights_only=False)
B = 32


def _ids_agree_up_to_near_tie(got, ref, oracle, pix):
    """Greedy ids equal, or the first divergence is at a step whose fp32 top-1 margin is below the parity tolerance."""
    n = min(got.numel(), ref.numel())
    diff = (got[:n] != ref[:n]).nonzero()
    if diff.numel() == 0:
        assert got.numel() == ref.numel()
        return
    t = int(diff[0])
    logits, _ = oracle.forward_logits(ref[None, :t], pix)
    top2 = logits[0, -1].topk(2).values
    assert (top2[0] - top2[1]).item() < 2 * TOL, (t, top2)


# ---------------------------------------------------------------- tiny-tl against the reference's model code
def test_tiny_tl_matches_reference_golden():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny-tl")
    g = GOLD["tiny-tl"]
    eng = engine_for("tiny-tl")
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=g["pixel_seed"])
    img = eng.image_embeds(pix.cuda())[0]
    ids = g["input_ids"]
    img_start = ids.tolist().index(cfg.patch_token_id)
    slot = eng.seq_alloc()
    try:
        _, all_logits = eng.prefill(slot, ids.cuda(), 0, img, img_start, want_all_logits=True)
        assert (all_logits.cpu() - g["logits"]).abs().max().item() < TOL
        T = ids.numel()
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            lg = eng.decode([slot], [T], torch.tensor([g["next_id"]]).cuda())[0].cpu()
            assert (lg - g["decode_logits"]).abs().max().item() < TOL, impl
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)
    model = DetikzifyForCausalLM(cfg, engine=eng)
    ref = g["generate_ids"]
    out = model.generate(input_ids=g["generate_prompt"][None], pixel_values=pix, bad_words_ids=[[cfg.image_token_id]],
                         begin_suppress_tokens=[cfg.eos_token_id], max_length=ref.numel(), do_sample=False)
    _ids_agree_up_to_near_tie(out[0].cpu(), ref, oracle, pix)


# ---------------------------------------------------------------- tl-1.1b at the real shape
@pytest.fixture(scope="module")
def tl():
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle(NAME)
    eng = engine_for(NAME, max_seqs=B + 4, max_batch=B)
    assert eng.get_option("decode_persistent") == 1
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=GOLD["tl-1.1b"]["pixel_seed"])
    img = eng.image_embeds(pix.cuda())[0]
    return cfg, oracle, eng, pix, img


def test_tl11b_prefill_decode_and_2k_context(tl):
    cfg, oracle, eng, pix, img = tl
    gold = GOLD["tl-1.1b"]
    P = cfg.num_patches
    assert P == 243
    slot = eng.seq_alloc()
    try:
        # the reference's own model code at this shape: last prompt row and one cached decode step
        ids = gold["input_ids"]
        last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
        assert (last.cpu() - gold["last_logits"]).abs().max().item() < TOL
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            lg = eng.decode([slot], [ids.numel()], torch.tensor([gold["next_id"]]).cuda())[0].cpu()
            assert (lg - gold["decode_logits"]).abs().max().item() < TOL, impl
        # 24 teacher-forced greedy steps on both implementations against the fp32 oracle
        T0, steps = ids.numel(), 24
        ref_ids = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
        ref_all, _ = oracle.forward_logits(ref_ids[None], pix)
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
            worst = (last.cpu() - ref_all[0, T0 - 1]).abs().max().item()
            agree = checked = 0
            for t in range(T0, T0 + steps - 1):
                lg = eng.decode([slot], [t], ref_ids[t:t + 1].cuda())[0].cpu()
                worst = max(worst, (lg - ref_all[0, t]).abs().max().item())
                top2 = ref_all[0, t].topk(2).values
                if (top2[0] - top2[1]) > 2 * TOL:
                    checked += 1
                    agree += int(lg.argmax() == ref_all[0, t].argmax())
            assert worst < TOL, (impl, worst)
            assert agree == checked, impl
        # context checkpoints (split-KV ranges of the persistent kernel change shape) and the 2k end of the cache
        g = torch.Generator().manual_seed(2100)
        long_ids = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(3, 32000, (2048 - P,), generator=g)]).long()
        ref_long, _ = oracle.forward_logits(long_ids[None], pix)
        for T in (512, 1024, 1536, 2047):
            lastp, _ = eng.prefill(slot, long_ids[:T].cuda(), 0, img, 0)
            assert (lastp.cpu() - ref_long[0, T - 1]).abs().max().item() < TOL, T
            for impl in (1, 0):
                eng.set_option("decode_impl", impl)
                lgT = eng.decode([slot], [T], long_ids[T:T + 1].cuda())[0].cpu()
                assert (lgT - ref_long[0, T]).abs().max().item() < TOL, (T, impl)
                top2 = ref_long[0, T].topk(2).values
                if (top2[0] - top2[1]) > 2 * TOL:
                    assert int(lgT.argmax()) == int(ref_long[0, T].argmax()), (T, impl)
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)


@pytest.mark.parametrize("nb", [2, B])
def test_tl11b_batched_decode_and_nucleus(tl, nb):
    """nb = 2 runs the per-op GEMV kernels, nb = 32 the batched-GEMM step (swapped tile at N 2560 / 4096 / 11264 / 32008,
    K 2048 / 5632); ragged contexts, two consecutive steps, then the nucleus probability vector at V 32008."""
    cfg, oracle, eng, pix, img = tl
    P = cfg.num_patches
    g = torch.Generator().manual_seed(2200 + nb)
    prompts = [torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(3, 32000, (5 + 3 * i,), generator=g)]).long()
               for i in range(nb)]
    tok1 = torch.randint(3, 32000, (nb,), generator=g)
    tok2 = torch.randint(3, 32000, (nb,), generator=g)
    slots = [eng.seq_alloc() for _ in range(nb)]
    try:
        lens = []
        for s, ids in zip(slots, prompts):
            eng.prefill(s, ids.cuda(), 0, img, 0)
            lens.append(ids.numel())
        step1 = eng.decode(slots, lens, tok1.cuda()).clone()
        step2 = eng.decode(slots, [n + 1 for n in lens], tok2.cuda()).clone()
        torch.cuda.synchronize()
        for i in sorted({0, 1, nb // 2, nb - 1}):
            ref, _ = oracle.forward_logits(torch.cat([prompts[i], tok1[i:i + 1], tok2[i:i + 1]])[None], pix)
            assert (step1[i].cpu() - ref[0, -2]).abs().max().item() < TOL, i
            assert (step2[i].cpu() - ref[0, -1]).abs().max().item() < TOL, i
        params = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id,
                              begin_suppress_token=cfg.eos_token_id, seed=5)
        out, probs = eng.sample(step2, params, suppress=[0] * nb, steps=list(range(nb)), seq_ids=list(range(nb)), want_probs=True)
        torch.cuda.synchronize()
        assert probs.shape[-1] == 32008
        for i in (0, nb - 1):
            ref_p = oracle.processed_probs(torch.zeros(1, lens[i] + 2, dtype=torch.long), step2[i:i + 1].cpu(), lens[i],
                                           temperature=0.8, top_p=0.95, top_k=0)[0]
            got = probs[i].cpu()
            mism = ((ref_p > 0) != (got > 0)).sum()
            assert mism <= 1, (i, mism)
            if mism == 0:
                assert (got - ref_p).abs().max() < 1e-5
            assert got[int(out[i])] > 0 and got[cfg.image_token_id] == 0
    finally:
        for s in slots:
            eng.seq_free(s)


def test_tl11b_shared_prefix_cascade_and_persistent_borrower(tl):
    """Eight rollouts borrow a 253-position prefix (not a multiple of 16 or 32: 240 positions lent, 13 copied). The
    tensor-core prefix pass (cascade_attn 1) and the per-row kernel (0) agree and match the oracle; the persistent kernel
    decodes a borrower, whose 16-position KV items come partly from the base slot and partly from its own."""
    cfg, oracle, eng, pix, img = tl
    P = cfg.num_patches
    R = 8
    g = torch.Generator().manual_seed(2300)
    prefix = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(3, 32000, (10,), generator=g)]).long()
    cut = prefix.numel()
    assert cut % 16 and cut % 32
    sufs = [torch.randint(3, 32000, (1 + 2 * i,), generator=g) for i in range(R)]
    toks = torch.randint(3, 32000, (R,), generator=g)
    base = eng.seq_alloc()
    subs = [eng.seq_alloc() for _ in range(R)]
    try:
        eng.prefill(base, prefix.cuda(), 0, img, 0)
        lens = []
        for s, suf in zip(subs, sufs):
            eng.seq_share(base, s, cut)
            eng.prefill(s, suf.cuda(), cut, None, 0)
            lens.append(cut + suf.numel())
        out = {}
        for cas in (1, 0):
            eng.set_option("cascade_attn", cas)
            out[cas] = eng.decode(subs, lens, toks.cuda()).clone()
        torch.cuda.synchronize()
        assert (out[1] - out[0]).abs().max().item() < TOL   # the prefix pass rounds q to bf16 (tensor-core operand)
        for i in (0, R - 1):
            ref, _ = oracle.forward_logits(torch.cat([prefix, sufs[i], toks[i:i + 1]])[None], pix)
            assert (out[1][i].cpu() - ref[0, -1]).abs().max().item() < TOL, i
            for impl in (1, 0):
                eng.set_option("decode_impl", impl)
                lg = eng.decode([subs[i]], [lens[i]], toks[i:i + 1].cuda())[0].cpu()
                assert (lg - ref[0, -1]).abs().max().item() < TOL, (i, impl)
            eng.set_option("decode_impl", 1)
    finally:
        eng.set_option("cascade_attn", 1)
        eng.set_option("decode_impl", 1)
        for s in subs:
            eng.seq_free(s)
        eng.seq_free(base)


# ---------------------------------------------------------------- public generate paths (tiny-tl)
def _tiny_prompts(cfg, n, seed):
    g = torch.Generator().manual_seed(seed)
    stem = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.randint(0, 500, (6,), generator=g)])
    return [torch.cat([stem, torch.randint(0, 500, (2 + i,), generator=g)]).long() for i in range(n)]


def test_tiny_tl_generate_prefix_cache_equals_cold_call():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny-tl")
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=5)
    a, b = _tiny_prompts(cfg, 2, 2400)
    kw = dict(pixel_values=pix, bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
              max_new_tokens=20, do_sample=False)
    warm = DetikzifyForCausalLM(cfg, engine=engine_for("tiny-tl", max_seqs=6, max_batch=2))
    warm.generate(input_ids=a[None], **kw)
    got = warm.generate(input_ids=b[None], **kw)[0].cpu()          # reuses the KV of the shared stem
    cold = DetikzifyForCausalLM(cfg, engine=engine_for("tiny-tl", max_seqs=3, max_batch=1))
    ref = cold.generate(input_ids=b[None], **kw)[0].cpu()
    assert got.tolist() == ref.tolist()


def test_tiny_tl_generate_batch_shared_prefix_equals_generate():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny-tl")
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=6)
    prompts = _tiny_prompts(cfg, 6, 2500)
    kw = dict(pixel_values=pix, bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
              max_new_tokens=16, do_sample=False)
    model = DetikzifyForCausalLM(cfg, engine=engine_for("tiny-tl", max_seqs=10, max_batch=6))
    outs = model.generate_batch(prompts, share_prefix=True, **kw)
    for p, o in zip(prompts, outs):
        single = model.generate(input_ids=p[None], **kw)[0].cpu()
        _ids_agree_up_to_near_tie(o.cpu(), single, oracle, pix)


# ---------------------------------------------------------------- cl-7b matrix shapes
def test_cl7b_2l_prefill_and_batch1_decode():
    from oracle.hf_oracle import synthetic_pixels
    name = "cl-7b-2l"
    cfg, sd, oracle = model_bundle(name)
    assert (cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.vocab_size) == (4096, 11008, 32, 32024)
    eng = engine_for(name, max_seqs=2, max_batch=1)
    pix = synthetic_pixels(1, cfg.vision_config.image_size)
    img = eng.image_embeds(pix.cuda())[0]
    g = torch.Generator().manual_seed(2600)
    ids = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.randint(3, 32000, (30,), generator=g)]).long()
    T0, steps = ids.numel(), 6
    ref_ids = oracle.generate(ids[None], pix, max_length=T0 + steps, stop_on_eos=False)[0]
    ref_all, _ = oracle.forward_logits(ref_ids[None], pix)
    tol = max(TOL, 0.08 * ref_all.float().pow(2).mean().sqrt().item())   # two-layer fixture: as test_gpu_ds7b.py
    slot = eng.seq_alloc()
    try:
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            last, _ = eng.prefill(slot, ids.cuda(), 0, img, 0)
            worst = (last.cpu() - ref_all[0, T0 - 1]).abs().max().item()
            for t in range(T0, T0 + steps - 1):
                lg = eng.decode([slot], [t], ref_ids[t:t + 1].cuda())[0].cpu()
                worst = max(worst, (lg - ref_all[0, t]).abs().max().item())
                top2 = ref_all[0, t].topk(2).values
                if (top2[0] - top2[1]) > 2 * tol:
                    assert int(lg.argmax()) == int(ref_all[0, t].argmax())
            assert worst < tol, (impl, worst)
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)
