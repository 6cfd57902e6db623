"""Fused lm_head log-softmax (``dtk_dbg_lm_logprob``, ``dtk_score`` / ``Engine.score``) and the public ``forward()`` /
``score()`` of the model on the GPU:
  * the kernel against fp64 ``log_softmax(A W^T)`` of the same bf16 operands at the lm_head's scale and shapes;
  * ``Engine.score`` against ``log_softmax`` of the same engine's prefill logits (ds-1.3b, tl-1.1b, v2-8b-2l);
  * ``forward()`` logits and loss against the reference goldens, ``score()`` prefix sharing, no interference with
    ``generate()``, and the memory a 2047-token score of a 128 256-word vocabulary needs."""
import ctypes as C
from pathlib import Path

import pytest
import torch

from conftest import engine_for, model_bundle

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden"


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def _lm_logprob(A, W, targets):
    from detikzify_b200 import _lib
    M, N, K = A.shape[0], W.shape[0], A.shape[1]
    lp = torch.empty(M, device="cuda", dtype=torch.float32)
    lse = torch.empty(M, device="cuda", dtype=torch.float32)
    rc = _lib.load_library().dtk_dbg_lm_logprob(_p(A), _p(W), M, N, K, _p(targets), _p(lp), _p(lse),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    return lp, lse


_W = {}


def _weights(V, K):
    if (V, K) not in _W:
        _W.clear()
        g = torch.Generator(device="cuda").manual_seed(V + K)
        _W[(V, K)] = (torch.randn(V, K, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    return _W[(V, K)]


def _check_against_fp64(A, W, targets):
    V = W.shape[0]
    lp, lse = _lm_logprob(A, W, targets)
    lp2, lse2 = _lm_logprob(A, W, targets)
    torch.cuda.synchronize()
    assert torch.equal(lp, lp2) and torch.equal(lse, lse2)   # deterministic
    ref = A.double() @ W.double().T
    rlse = torch.logsumexp(ref, -1)
    ok = (targets >= 0) & (targets < V)
    rlp = torch.where(ok, ref.gather(1, targets.clamp(0, V - 1)[:, None])[:, 0] - rlse, torch.zeros_like(rlse))
    tol = 1e-4 * rlse.abs().clamp(min=1)
    assert ((lse.double() - rlse).abs() <= tol).all(), (lse.double() - rlse).abs().max()
    assert ((lp.double() - rlp).abs() <= tol).all(), (lp.double() - rlp).abs().max()
    assert (lp[~ok] == 0).all()


@pytest.mark.parametrize("V,K", [(520, 2048), (32008, 2048), (32256, 2048), (32008, 4096), (128256, 4096)])
@pytest.mark.parametrize("M", [1, 3, 17, 64, 200, 2047])
def test_lm_logprob_kernel_matches_fp64(M, V, K):
    g = torch.Generator(device="cuda").manual_seed(M)
    A = torch.randn(M, K, device="cuda", generator=g).to(torch.bfloat16)
    W = _weights(V, K)
    pool = torch.tensor([0, 255, 256, V - 1, -100, V], device="cuda")
    targets = torch.randint(0, V, (M,), device="cuda", generator=g)
    targets[: min(M, 6)] = pool[: min(M, 6)]
    if M > 6:
        targets[6::7] = pool[torch.arange(len(targets[6::7]), device="cuda") % 6]
    _check_against_fp64(A, W, targets)


def test_lm_logprob_kernel_zero_fill_stays_out_near_minus_50():
    """Every logit near -50 (a constant column of A against W[:, 0] = -50): a zero-filled column past V = 32008 entering the
    sum would move the lse from about -39.6 to about 0."""
    M, V, K = 64, 32008, 2048
    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn(M, K, device="cuda", generator=g)
    A[:, 0] = 1.0
    W = (torch.randn(V, K, device="cuda", generator=g) * 0.02)
    W[:, 0] = -50.0
    targets = torch.tensor([0, 255, 256, V - 1, -100, V] * 11, device="cuda")[:M]
    _check_against_fp64(A.to(torch.bfloat16), W.to(torch.bfloat16), targets)


# ---------------------------------------------------------------- Engine.score against the engine's own prefill logits
@pytest.mark.parametrize("name", ["nllg/detikzify-ds-1.3b", "tl-1.1b", "v2-8b-2l"])
def test_engine_score_matches_prefill_logits(name):
    cfg, _, _ = model_bundle(name)
    eng = engine_for(name)
    V = cfg.vocab_size
    g = torch.Generator().manual_seed(7)
    slots = [eng.seq_alloc(), eng.seq_alloc()]
    try:
        for T in (5, 64, 300):
            ids = torch.randint(0, min(V, 32000), (T,), generator=g).cuda()
            targets = torch.randint(0, V, (T,), generator=g).cuda()
            targets[::5] = -1
            _, ref = eng.prefill(slots[0], ids, 0, want_all_logits=True)
            lp, lse, alll = eng.score(slots[1], ids, 0, targets=targets, want_all_logits=True)
            lp2, _, _ = eng.score(slots[1], ids, 0, targets=targets)
            with pytest.raises(ValueError, match="targets"):
                eng.score(slots[1], ids, 0)
            torch.cuda.synchronize()
            assert torch.equal(lp, lp2)
            rlse = torch.logsumexp(ref.double(), -1)
            ok = targets >= 0
            rlp = torch.where(ok, ref.double().gather(1, targets.clamp(min=0)[:, None])[:, 0] - rlse, torch.zeros_like(rlse))
            assert (lse.double() - rlse).abs().max() <= 1e-3, T
            assert (lp.double() - rlp).abs().max() <= 1e-3, T
            if T >= 64:   # both run the persistent 128 x 256 wgmma kernel on the same operands
                assert torch.equal(alll, ref), T
            else:
                assert (alll - ref).abs().max() <= 1e-3, T
        # a borrower of a shared prefix: scoring positions [96, 300) equals the rows of the full prefill
        ids = torch.randint(0, min(V, 32000), (300,), generator=g).cuda()
        _, ref = eng.prefill(slots[0], ids, 0, want_all_logits=True)
        eng.seq_share(slots[0], slots[1], 96)
        targets = torch.randint(0, V, (204,), generator=g).cuda()
        lp, _, _ = eng.score(slots[1], ids[96:], 96, targets=targets)
        r = torch.log_softmax(ref[96:].double(), -1).gather(1, targets[:, None])[:, 0]
        assert (lp.double() - r).abs().max() <= 1e-3
    finally:
        for s in reversed(slots):
            eng.seq_free(s)


# ---------------------------------------------------------------- public forward() against the reference goldens
_MODELS = {}


def _model(name):
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    if name not in _MODELS:
        cfg, _, _ = model_bundle(name)
        _MODELS[name] = DetikzifyForCausalLM(cfg, engine=engine_for(name, max_seqs=6, max_batch=4))
    return _MODELS[name]


@pytest.mark.parametrize("file,name", [("reference_v1_tiny", "tiny"), ("reference_v1_tiny", "tiny2"),
                                       ("reference_v2_tiny", "tiny-v2"), ("reference_v1_tl", "tiny-tl")])
def test_forward_logits_match_reference_golden(file, name):
    from oracle.hf_oracle import synthetic_pixels
    g = torch.load(GOLDEN / f"{file}.pt", weights_only=False)[name]
    model = _model(name)
    pix = synthetic_pixels(1, model.config.vision_config.image_size, seed=g["pixel_seed"])
    out = model(input_ids=g["input_ids"][None], pixel_values=pix)
    assert out.loss is None and out.logits.shape == (1, g["input_ids"].numel(), model.config.vocab_size)
    assert (out.logits[0].cpu() - g["logits"]).abs().max().item() < 3e-2


@pytest.mark.parametrize("case,name", [("v1", "tiny"), ("v2", "tiny-v2"), ("v2_right", "tiny-v2"), ("v2_left", "tiny-v2")])
def test_forward_loss_matches_reference_golden(case, name):
    from oracle.hf_oracle import synthetic_pixels
    g = torch.load(GOLDEN / "reference_loss_tiny.pt", weights_only=False)[case]
    model = _model(name)
    B = g["input_ids"].shape[0]
    pix = synthetic_pixels(B, model.config.vision_config.image_size, seed=g["pixel_seed"])
    out = model(input_ids=g["input_ids"], pixel_values=pix, attention_mask=g.get("attention_mask"), labels=g["labels"])
    assert abs(out.loss.item() - g["loss"].item()) < 3e-2
    if "logits" in g:
        assert (out.logits.cpu() - g["logits"]).abs().max().item() < 3e-2
    else:
        assert not out.logits[~g["attention_mask"].bool().cuda()].any()
    # the loss comes from the fused log-probs; cross-entropy over the returned logits agrees
    lab = g["labels"][:, 1:].clone()
    if "attention_mask" in g:
        lab[g["attention_mask"][:, 1:] == 0] = -100
    ce = torch.nn.functional.cross_entropy(out.logits[:, :-1].reshape(-1, out.logits.shape[-1]).cpu(), lab.reshape(-1))
    assert abs(out.loss.item() - ce.item()) < 1e-3


def test_forward_with_caption_matches_adapter_golden():
    from test_gpu_adapter import _bundle
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels
    cfg, acfg, _, _, eng, _ = _bundle("tiny-v2")
    model = DetikzifyForCausalLM(cfg, engine=eng)
    model.adapter = A.CrossAttentionAdapter(cfg, acfg, eng.adapter_arena)
    model.embedding_model = A.CaptionEmbedder(acfg)
    gold = torch.load(GOLDEN / "reference_adapter_tiny.pt", weights_only=False)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=gold["pixel_seed"])
    cap, prompt = gold["caption"], gold["prompt"]
    for key, p in (("image", pix), ("text", None)):
        out = model(input_ids=prompt[None], pixel_values=p, adapter_input_ids=cap[None],
                    adapter_attention_mask=torch.ones(1, cap.numel(), dtype=torch.long))
        assert (out.logits[0].cpu() - gold[f"{key}_logits"]).abs().max().item() < 3e-2, key
    eng.close()


# ---------------------------------------------------------------- score(): prefix sharing, determinism, no interference
def test_score_with_shared_prefix_equals_forward_alone():
    from oracle.hf_oracle import synthetic_pixels
    name = "nllg/detikzify-ds-1.3b"
    model = _model(name)
    cfg = model.config
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=11)
    g = torch.Generator().manual_seed(12)
    head = [cfg.patch_token_id] * cfg.num_patches + torch.randint(0, 32000, (20,), generator=g).tolist()
    # every candidate's own prefill keeps >= 64 rows, as forward() does: both then run each decoder GEMM on the same dense
    # tile (fewer rows take the swapped-operand tile, whose bf16 activations round differently: ~1e-2 after 24 layers)
    cands = [head + torch.randint(0, 32000, (70 + 5 * i,), generator=g).tolist() for i in range(8)]
    seqs = [torch.tensor(c) for c in cands]
    ref = [torch.log_softmax(model(input_ids=torch.tensor([c]), pixel_values=pix).logits[0].double(), -1) for c in cands]
    # the last 4 shared code tokens scored as well; and scoring from the first token after the image span (v1 layout)
    for start in (len(head) - 4, cfg.num_patches):
        got = model.score(seqs, pix, start=start)
        again = model.score(seqs, pix, start=start)
        for i, c in enumerate(cands):
            assert torch.equal(got[i], again[i])
            r = ref[i][start - 1:-1].gather(1, torch.tensor(c[start:]).cuda()[:, None])[:, 0]
            assert got[i].shape == (len(c) - start,)
            assert (got[i].double() - r).abs().max().item() <= 1e-3, (start, i)


def test_generate_unchanged_by_forward_and_score():
    from oracle.hf_oracle import synthetic_pixels
    model = _model("tiny")
    cfg = model.config
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=77)
    prompt = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.tensor([5, 6, 7])]).long()[None]
    kw = dict(pixel_values=pix, bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
              max_new_tokens=24, do_sample=False)
    before = model.generate(input_ids=prompt, **kw)
    ids = torch.cat([prompt[0], torch.randint(0, 400, (30,))])
    model(input_ids=ids[None], pixel_values=pix, labels=ids[None])
    model.score([ids, ids[:20]], pix, start=10)
    mid = model.generate(input_ids=prompt, **kw)
    model(input_ids=ids[None, :12], pixel_values=pix)
    after = model.generate(input_ids=prompt, **kw)
    assert torch.equal(before, mid) and torch.equal(before, after)


def test_score_memory_at_128k_vocab():
    name = "v2-8b-2l"
    cfg, _, _ = model_bundle(name)
    eng = engine_for(name, max_seqs=2, max_batch=1)   # an engine of its own: its first call allocates the partials
    T, V = 2047, cfg.vocab_size
    budget = 4 * T * V // 8
    ids = torch.randint(0, 128000, (T,), device="cuda")
    targets = torch.randint(0, V, (T,), device="cuda")
    slot = eng.seq_alloc()
    try:
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.max_memory_allocated()
        lp, _, _ = eng.score(slot, ids, 0, targets=targets)
        torch.cuda.synchronize()
        assert torch.cuda.max_memory_allocated() - base < budget
        assert free0 - torch.cuda.mem_get_info()[0] < budget
        assert torch.isfinite(lp).all()
    finally:
        eng.seq_free(slot)
