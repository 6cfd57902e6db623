"""
Oracle-backed parity of paths that would otherwise only be checked against the engine itself:
  * image span in the MIDDLE of the prompt through dtk_prefill, against the logits the REFERENCE's own
    DetikzifyForCausalLM produced (tests/golden/reference_v1_tiny.pt, detikzify/model/v1/modeling_detikzify.py:157-200);
  * dtk_seq_fork and suffix prefill against oracle.forward_logits;
  * ImageSim.get_similarity on the CUDA vision tower against oracle.selfsim_cos (detikzify/evaluate/imagesim.py:91-125).
Tolerances as in test_gpu_model.py: logits max-abs 3e-2 (bf16 operand storage, fp32 accumulation).
"""
from pathlib import Path

import pytest
import torch

from conftest import engine_for, model_bundle

pytestmark = pytest.mark.gpu
TOL = 3e-2
GOLD = Path(__file__).parent / "golden" / "reference_v1_tiny.pt"


def _pixels(cfg, batch, seed=1000):
    from oracle.hf_oracle import synthetic_pixels
    return synthetic_pixels(batch, cfg.vision_config.image_size, seed)


@pytest.mark.parametrize("impl", [1, 0], ids=["persistent", "per-op"])
@pytest.mark.parametrize("name", ["tiny", "tiny2"])
def test_mid_prompt_image_span_matches_reference_logits(name, impl):
    """The reference's forward on a prompt [text, 243-style image span, text] (golden: all-position logits + one cached
    decode step). The engine splices the projector rows at img_start > 0 inside dtk_prefill."""
    gold = torch.load(GOLD, weights_only=False)[name]
    cfg, sd, oracle = model_bundle(name, seed=gold["seed"])
    eng = engine_for(name, seed=gold["seed"])
    ids = gold["input_ids"].long()
    pix = _pixels(cfg, 1, seed=gold["pixel_seed"])
    start = int((ids == cfg.image_token_id).nonzero()[0])
    assert start > 0 and int((ids == cfg.image_token_id).sum()) == cfg.num_patches
    img = eng.image_embeds(pix.cuda())[0]
    slot = eng.seq_alloc()
    eng.set_option("decode_impl", impl)
    try:
        last, alll = eng.prefill(slot, ids.cuda(), 0, img, start, want_all_logits=True)
        assert (alll.cpu() - gold["logits"]).abs().max().item() < TOL
        assert (last.cpu() - gold["logits"][-1]).abs().max().item() < TOL
        lg = eng.decode([slot], [ids.numel()], torch.tensor([gold["next_id"]], device="cuda"))[0].cpu()
        assert (lg - gold["decode_logits"]).abs().max().item() < TOL
    finally:
        eng.set_option("decode_impl", 1)
        eng.seq_free(slot)


@pytest.mark.parametrize("name", ["tiny", "tiny2"])
def test_fork_and_suffix_prefill_against_oracle(name):
    """MCTS prefix reuse: prefill(prefix) -> fork -> prefill(suffix, start_pos) -> decode. Every logits row is compared
    with the oracle's full forward of the same token sequence (not with the engine's own full prefill)."""
    cfg, sd, oracle = model_bundle(name)
    eng = engine_for(name)
    pix = _pixels(cfg, 1)
    g = torch.Generator().manual_seed(4000)
    P = cfg.num_patches
    text = torch.randint(0, min(cfg.vocab_size, cfg.patch_token_id), (30,), generator=g)
    ids = torch.cat([torch.full((P,), cfg.patch_token_id), text]).long()
    alt = ids.clone()
    alt[P + 12:] = torch.randint(0, min(cfg.vocab_size, cfg.patch_token_id), (18,), generator=g)  # a sibling branch
    ref_a, _ = oracle.forward_logits(ids[None], pix)
    ref_b, _ = oracle.forward_logits(alt[None], pix)
    img = eng.image_embeds(pix.cuda())[0]
    a, b = eng.seq_alloc(), eng.seq_alloc()
    try:
        cut = P + 12
        eng.prefill(a, ids[:cut].cuda(), 0, img, 0)
        eng.seq_fork(a, b, cut)
        # branch a: suffix prefill with all-position logits
        last_a, all_a = eng.prefill(a, ids[cut:].cuda(), cut, None, 0, want_all_logits=True)
        assert (all_a.cpu() - ref_a[0, cut:]).abs().max().item() < TOL
        # branch b (forked copy of the prefix): its own suffix, then one decode step
        last_b, _ = eng.prefill(b, alt[cut:-1].cuda(), cut, None, 0)
        assert (last_b.cpu() - ref_b[0, -2]).abs().max().item() < TOL
        lg = eng.decode([b], [alt.numel() - 1], alt[-1:].cuda())[0].cpu()
        assert (lg - ref_b[0, -1]).abs().max().item() < TOL
        # the fork did not disturb branch a
        assert (last_a.cpu() - ref_a[0, -1]).abs().max().item() < TOL
    finally:
        eng.seq_free(a)
        eng.seq_free(b)


@pytest.mark.parametrize("mode", ["cos", "cos_avg"])
def test_imagesim_on_cuda_tower_matches_oracle(mode):
    """SelfSim reward through the public ImageSim object (PIL in, float out) on the CUDA vision tower vs the oracle's
    fp64 cosine of HF-SigLIP features of the same preprocessed pixels (evaluate/imagesim.py:91-125)."""
    import torch.nn.functional as F
    from PIL import Image, ImageDraw
    from detikzify_b200.evaluate.imagesim import ImageSim
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from detikzify_b200.model import build_processor
    from detikzify_b200.util.image import expand, load
    name = "tiny2"
    cfg, sd, oracle = model_bundle(name)
    model = DetikzifyForCausalLM(cfg, engine=engine_for(name))
    proc = build_processor(cfg)
    ims = []
    for k in range(2):
        im = Image.new("RGB", (200, 160), "white")
        d = ImageDraw.Draw(im)
        for j in range(6):
            d.line([(10 + 25 * j, 20 + 9 * k * j), (180 - 20 * j, 140 - 15 * k)], fill="black", width=2 + k)
        d.ellipse([60, 40 + 30 * k, 140, 120], outline="black", width=3)
        ims.append(im)
    sim = ImageSim.from_detikzify(model, proc, mode=mode)
    got = sim.get_similarity(ims[0], ims[1])
    feats = []
    for im in ims:
        im = expand(load(im), max(im.size), do_trim=True)
        pix = proc.image_processor(images=im, return_tensors="pt")["pixel_values"]
        tok, pool = oracle.vision(pix)
        feats.append(pool.squeeze() if mode == "cos" else tok.squeeze().mean(dim=0))
    ref = F.cosine_similarity(feats[0].double(), feats[1].double(), dim=0).item()
    assert abs(got - ref) < 5e-3, (got, ref)
    assert abs(sim.get_similarity(ims[0], ims[0]) - 1.0) < 1e-6
    # batched form (candidate renders of parallel rollouts through one ViT pass): same values as pair by pair
    both = sim.get_similarities([ims[1], ims[0]], ims[0])
    assert abs(both[0] - got) < 2e-3 and abs(both[1] - 1.0) < 1e-6
    if mode == "cos":
        p0 = proc.image_processor(images=expand(load(ims[0]), max(ims[0].size), do_trim=True), return_tensors="pt")["pixel_values"]
        p1 = proc.image_processor(images=expand(load(ims[1]), max(ims[1].size), do_trim=True), return_tensors="pt")["pixel_values"]
        assert abs(oracle.selfsim_cos(p0, p1) - ref) < 1e-9


@pytest.mark.parametrize("name", ["tiny2", "tiny-v2"])
def test_imagesim_emd_on_cuda_tower_matches_oracle(name):
    """The v2 models' SelfSim ("emd": 2 tanh(-EMD) + 1 over the patch tokens, evaluate/imagesim.py:105-107,121-123) on the CUDA
    vision tower (assignment solver on the host) vs the oracle (HF SigLIP tokens, the transport LP itself)."""
    from PIL import Image, ImageDraw
    from detikzify_b200.evaluate.imagesim import ImageSim
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from detikzify_b200.model import build_processor
    from detikzify_b200.util.image import expand, load
    cfg, sd, oracle = model_bundle(name)
    model = DetikzifyForCausalLM(cfg, engine=engine_for(name))
    proc = build_processor(cfg)
    ims = []
    for k in range(2):
        im = Image.new("RGB", (200, 160), "white")
        d = ImageDraw.Draw(im)
        for j in range(6):
            d.line([(10 + 25 * j, 20 + 9 * k * j), (180 - 20 * j, 140 - 15 * k)], fill="black", width=2 + k)
        d.ellipse([60, 40 + 30 * k, 140, 120], outline="black", width=3)
        ims.append(im)
    sim = ImageSim.from_detikzify(model, proc, mode="emd")
    if name == "tiny-v2":
        assert ImageSim.from_detikzify(model, proc).mode == "emd"   # the v2 default
    got = sim.get_similarity(ims[0], ims[1])
    pix = [proc.image_processor(images=expand(load(im), max(im.size), do_trim=True), return_tensors="pt")["pixel_values"] for im in ims]
    ref = oracle.selfsim_emd(pix[0], pix[1])
    assert abs(got - ref) < 5e-3, (got, ref)
    assert abs(sim.get_similarity(ims[0], ims[0]) - 1.0) < 1e-6
    both = sim.get_similarities([ims[1], ims[0]], ims[0])
    assert abs(both[0] - got) < 2e-3 and abs(both[1] - 1.0) < 1e-6


def test_shared_prefix_rollouts_against_oracle():
    """dtk_seq_share: four rollouts READ the first 41 positions (image span + path prefix) from one base slot — whole
    16-position blocks shared, the 9-position remainder copied — then prefill their own suffixes and decode. Every logits
    row (suffix prefill, batch-1 decode on both implementations, batched-GEMM decode of all four) is checked against the
    oracle's full forward of the same token sequence; reference counting protects the base slot."""
    from detikzify_b200.engine import EngineError
    name = "tiny2"
    cfg, sd, oracle = model_bundle(name)
    eng = engine_for(name, max_seqs=8, max_batch=8)
    pix = _pixels(cfg, 1)
    img = eng.image_embeds(pix.cuda())[0]
    P = cfg.num_patches
    g = torch.Generator().manual_seed(4100)
    hi = min(cfg.vocab_size, cfg.patch_token_id)
    prefix = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(0, hi, (14,), generator=g)]).long()
    cut = prefix.numel()
    assert cut % 16 != 0
    R = 4
    suffixes = [torch.randint(0, hi, (5 + 3 * i,), generator=g) for i in range(R)]
    toks = torch.randint(0, hi, (R,), generator=g)
    base = eng.seq_alloc()
    subs = [eng.seq_alloc() for _ in range(R)]
    try:
        eng.prefill(base, prefix.cuda(), 0, img, 0)
        refs, lens = [], []
        for s, suf in zip(subs, suffixes):
            eng.seq_share(base, s, cut)
            last, _ = eng.prefill(s, suf.cuda(), cut, None, 0)
            full = torch.cat([prefix, suf])
            ref, _ = oracle.forward_logits(torch.cat([full, toks[len(refs):len(refs) + 1]])[None], pix)
            assert (last.cpu() - ref[0, -2]).abs().max().item() < TOL
            refs.append(ref[0, -1]); lens.append(full.numel())
        # the base is protected while borrowers exist
        with pytest.raises(EngineError):
            eng.seq_free(base)
        with pytest.raises(EngineError):
            eng.prefill(base, prefix[:8].cuda(), 4, None, 0)
        for impl in (1, 0):
            eng.set_option("decode_impl", impl)
            for i in (0, R - 1):
                lg = eng.decode([subs[i]], [lens[i]], toks[i:i + 1].cuda())[0].cpu()
                assert (lg - refs[i]).abs().max().item() < TOL, (impl, i)
        eng.set_option("decode_impl", 1)
        batched = eng.decode(subs, lens, toks.cuda())
        for i in range(R):
            assert (batched[i].cpu() - refs[i]).abs().max().item() < TOL, i
        # a fork of a borrower is self-contained
        extra = eng.seq_alloc()
        try:
            eng.seq_fork(subs[1], extra, lens[1])
            lg = eng.decode([extra], [lens[1]], toks[1:2].cuda())[0].cpu()
            assert (lg - refs[1]).abs().max().item() < TOL
        finally:
            eng.seq_free(extra)
    finally:
        eng.set_option("decode_impl", 1)
        for s in subs:
            eng.seq_free(s)
        eng.seq_free(base)


def test_shared_prefix_cascade_attention_matches_plain_and_oracle():
    """Batched decode of rollouts that share one long prefix: the shared keys are reduced once per head by the tensor-core
    prefix kernel (the rollouts are its query rows) and merged with each row's private suffix. Same logits as the per-row
    path (option cascade_attn = 0) up to the bf16 rounding of q, and both match the oracle."""
    name = "tiny2"
    cfg, sd, oracle = model_bundle(name)
    R = 6
    eng = engine_for(name, max_seqs=R + 2, max_batch=R)
    pix = _pixels(cfg, 1)
    img = eng.image_embeds(pix.cuda())[0]
    P = cfg.num_patches
    g = torch.Generator().manual_seed(4200)
    hi = min(cfg.vocab_size, cfg.patch_token_id)
    prefix = torch.cat([torch.full((P,), cfg.patch_token_id), torch.randint(0, hi, (107 - P,), generator=g)]).long()
    cut = prefix.numel()                      # 107: 96 positions shared (cascade needs >= 64), 11 copied
    suffixes = [torch.randint(0, hi, (2 + 4 * i,), generator=g) for i in range(R)]
    toks = torch.randint(0, hi, (R,), generator=g)
    base = eng.seq_alloc()
    subs = [eng.seq_alloc() for _ in range(R)]
    try:
        eng.prefill(base, prefix.cuda(), 0, img, 0)
        refs, lens = [], []
        for i, (s, suf) in enumerate(zip(subs, suffixes)):
            eng.seq_share(base, s, cut)
            eng.prefill(s, suf.cuda(), cut, None, 0)
            full = torch.cat([prefix, suf])
            ref, _ = oracle.forward_logits(torch.cat([full, toks[i:i + 1]])[None], pix)
            refs.append(ref[0, -1]); lens.append(full.numel())
        out = {}
        for cas in (1, 0):
            eng.set_option("cascade_attn", cas)
            out[cas] = eng.decode(subs, lens, toks.cuda()).clone()
        torch.cuda.synchronize()
        assert (out[1] - out[0]).abs().max().item() < 2e-2
        for i in range(R):
            assert (out[1][i].cpu() - refs[i]).abs().max().item() < TOL, i
        # the generation loop (CUDA graph keyed by the shared slot and length) agrees with stepwise decode + argmax
        eng.set_option("cascade_attn", 1)
        first = [int(out[1][i].argmax()) for i in range(R)]
        params = eng.sampling(do_sample=False, bad_token=cfg.image_token_id)
        eng.gen_begin(subs, [n + 1 for n in lens], first, params)
        got = []
        for step in range(3):
            eng.gen_step()
            got.append(eng.gen_wait(step))
        eng.gen_end()
        # stepwise: feed the same tokens through dtk_decode
        cur, pos = first, [n + 1 for n in lens]
        # rewind is implicit: decode rewrites the same KV rows
        for step in range(3):
            lg = eng.decode(subs, pos, torch.tensor(cur).cuda())
            lg[:, cfg.image_token_id] = -float("inf")
            cur = [int(x) for x in lg.argmax(-1)]
            assert cur == [int(x) for x in got[step]], step
            pos = [n + 1 for n in pos]
    finally:
        eng.set_option("cascade_attn", 1)
        for s in subs:
            eng.seq_free(s)
        eng.seq_free(base)


def test_device_image_preprocessing_is_pillow_exact():
    """dtk_image_preprocess: the resized uint8 image equals Pillow's bicubic resize bit for bit and the normalised fp32 pixels
    equal the host image processor's (reference v1/processing_detikzify.py:242-251), for ragged input sizes."""
    import numpy as np
    from PIL import Image
    from detikzify_b200.model import build_processor
    name = "tiny2"
    cfg, sd, oracle = model_bundle(name)
    eng = engine_for(name)
    ip = build_processor(cfg).image_processor
    S = cfg.vision_config.image_size
    rng = np.random.default_rng(5)
    ims = []
    for h, w in [(500, 500), (S, S), (97, 233), (640, 200), (60, 60)]:
        arr = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        arr[: h // 3] = 255                                    # renders are mostly white
        ims.append(Image.fromarray(arr))
        out = torch.empty(3, S, S, device="cuda")
        u8 = eng.image_preprocess(torch.from_numpy(arr).cuda(), S, ip.rescale_factor, ip.image_mean, ip.image_std, out, want_uint8=True)
        ref_u8 = np.asarray(ims[-1].resize((S, S), resample=Image.Resampling.BICUBIC))
        assert np.array_equal(u8.cpu().numpy(), ref_u8), (h, w)
    host = ip.preprocess(ims)["pixel_values"]
    dev = ip.preprocess_device(ims, eng)
    torch.cuda.synchronize()
    assert (dev.cpu() - host).abs().max().item() < 1e-6
