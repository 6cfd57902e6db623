"""
TikZero text conditioning on the CUDA path (reference detikzify/model/adapter): the cross-attention kernel, the per-head
LayerNorm and the gated GEMM epilogue at the real so400m shapes against fp32 torch, the caption encoder at the real
Llama-3.2-1B widths against HF ``LlamaModel``, and the conditioned model end to end against ``oracle.adapter_oracle``.
Engines are built here (not shared through conftest): attaching an adapter changes an engine's state.
Tolerances: kernels as in test_gpu_kernels.py; end to end at the real widths 8 % of the reference RMS (test_gpu_ds7b.py).
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

D, HEADS, DH = 1152, 16, 72


def _bundle(cfg_name, vision=None, adapter_name="tiny", seed=0, max_seqs=4, max_batch=4):
    from detikzify_b200.engine import Engine, pack_arena
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.weights import random_init
    from oracle.adapter_oracle import AdapterOracle
    cfg = preset(cfg_name)
    if vision is not None:
        cfg.vision_config = vision
    sd = random_init(cfg, seed=seed)
    acfg = A.adapter_preset(adapter_name)
    asd = A.random_init(cfg, acfg, seed=seed + 1)
    eng = Engine(cfg, pack_arena(cfg, sd), device=0, max_seqs=max_seqs, max_batch=max_batch)
    eng.adapter_attach(A.to_c_adapter_config(acfg), A.pack_arena(cfg, acfg, asd))
    return cfg, acfg, sd, asd, eng, AdapterOracle(cfg.to_dict(), sd, acfg, asd)


def _rel(got, ref):
    return ((got.float() - ref.float()).abs().max() / ref.float().pow(2).mean().sqrt()).item()


def _xattn_ref(q, kv, lens, N, Tk):
    """fp32 softmax(q k^T / sqrt(72)) v over the first lens[b] keys of image b."""
    B = len(lens)
    qf = q.float().view(B, N, HEADS, DH).transpose(1, 2)
    kf = kv[:, :D].float().view(B, Tk, HEADS, DH).transpose(1, 2)
    vf = kv[:, D:].float().view(B, Tk, HEADS, DH).transpose(1, 2)
    out = torch.empty(B, HEADS, N, DH, device=q.device)
    for b, L in enumerate(lens):
        s = qf[b] @ kf[b, :, :L].transpose(1, 2) / DH ** 0.5
        out[b] = torch.softmax(s, -1) @ vf[b, :, :L]
    return out.transpose(1, 2).reshape(B * N, D)


@pytest.mark.parametrize("N", [729, 900])
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("Tk", [1, 7, 77, 300, 512])
def test_xattn_kernel_masks_padded_keys(N, B, Tk):
    from detikzify_b200 import _lib
    import ctypes as C
    lib = _lib.load_library()
    g = torch.Generator(device="cuda").manual_seed(N * 7 + B * 3 + Tk)
    q = torch.randn(B * N, D, device="cuda", generator=g).bfloat16()
    kv = torch.randn(B * Tk, 2 * D, device="cuda", generator=g).bfloat16()
    lens = [Tk if b == 0 else max(1, (Tk * 2) // 3) for b in range(B)]
    kv3 = kv.view(B, Tk, 2 * D)
    for b, L in enumerate(lens):   # large finite garbage in the masked key / value rows
        kv3[b, L:] = 3.0e4
    np_ = (Tk + 127) // 128 * 128
    vt = torch.empty(B * HEADS * 80, np_, device="cuda", dtype=torch.bfloat16)
    o = torch.empty(B * N, D, device="cuda", dtype=torch.bfloat16)
    rc = lib.dtk_dbg_xattn_tc(q.data_ptr(), kv.data_ptr(), (C.c_int * B)(*lens), Tk, vt.data_ptr(), o.data_ptr(), B, HEADS, N,
                              DH ** -0.5, None)
    assert rc == 0
    torch.cuda.synchronize()
    ref = _xattn_ref(q, kv, lens, N, Tk)
    assert torch.isfinite(o.float()).all()
    assert (o.float() - ref).abs().max().item() < 2e-2


def test_head_layernorm_and_gated_epilogue():
    from detikzify_b200 import _lib
    lib = _lib.load_library()
    g = torch.Generator(device="cuda").manual_seed(3)
    M = 1000
    x = (torch.randn(M, D, device="cuda", generator=g) * 3 + 1).bfloat16()
    w = (1 + 0.1 * torch.randn(DH, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(DH, device="cuda", generator=g)).bfloat16()
    out = torch.empty_like(x)
    assert lib.dtk_dbg_head_layernorm(x.data_ptr(), w.data_ptr(), b.data_ptr(), 1e-6, M, HEADS, DH, out.data_ptr(), None) == 0
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x.float().view(M, HEADS, DH), (DH,), w.float(), b.float(), 1e-6).view(M, D)
    assert (out.float() - ref).abs().max().item() < 3e-2
    # gated residual GEMM: out = resid + sigmoid(gate) * gelu_tanh(A W^T + bias), on both GEMM families
    K, N = 1152, 4304
    A = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    W = (torch.randn(N, K, device="cuda", generator=g) * 0.03).bfloat16()
    bias = (torch.randn(N, device="cuda", generator=g) * 0.1).bfloat16()
    resid = torch.randn(M, N, device="cuda", generator=g)
    gate = torch.tensor([-0.7], device="cuda").bfloat16()
    ref = resid + torch.sigmoid(gate.float()) * torch.nn.functional.gelu(A.float() @ W.float().T + bias.float(), approximate="tanh")
    prev = lib.dtk_dbg_gemm_impl(-1)
    try:
        for impl in (0, 1, 2):
            lib.dtk_dbg_gemm_impl(impl)
            o = torch.empty(M, N, device="cuda")
            assert lib.dtk_dbg_gemm_gated(A.data_ptr(), W.data_ptr(), bias.data_ptr(), gate.data_ptr(), resid.data_ptr(), M, N, K,
                                          1, o.data_ptr(), None) == 0
            torch.cuda.synchronize()
            assert (o - ref).abs().max().item() < 3e-2, impl
        # M < 64 without an activation: the swapped-operand tile of the batched decode path (impl 1 / 2)
        Ms = 40
        ref = resid[:Ms] + torch.sigmoid(gate.float()) * (A[:Ms].float() @ W.float().T + bias.float())
        for impl in (0, 1, 2):
            lib.dtk_dbg_gemm_impl(impl)
            o = torch.empty(Ms, N, device="cuda")
            assert lib.dtk_dbg_gemm_gated(A.data_ptr(), W.data_ptr(), bias.data_ptr(), gate.data_ptr(), resid.data_ptr(), Ms, N, K,
                                          0, o.data_ptr(), None) == 0
            torch.cuda.synchronize()
            assert (o - ref).abs().max().item() < 3e-2, ("M<64", impl)
    finally:
        lib.dtk_dbg_gemm_impl(prev)


@pytest.fixture(scope="module")
def real_width():
    """Every real cross-layer and embedder matrix shape: so400m tower (2 layers, 420 px) and Llama-3.2-1B (2 layers)."""
    from detikzify_b200.model.configuration import VisionConfig
    return _bundle("tiny-v2", vision=VisionConfig(num_hidden_layers=2, image_size=420), adapter_name="llama-3.2-1b-2l")


@pytest.mark.parametrize("T", [1, 13, 77, 512])
def test_caption_encoder_real_widths(real_width, T):
    cfg, acfg, sd, asd, eng, oracle = real_width
    g = torch.Generator().manual_seed(T)
    ids = torch.randint(0, 128000, (T,), generator=g)
    hidden, cond = eng.text_encode(ids.cuda(), want_hidden=True)
    h_ref, c_ref = oracle.caption_states(ids)
    assert _rel(hidden.cpu(), h_ref[0]) < 0.08
    assert _rel(cond.cpu(), c_ref[0]) < 0.08


def test_conditioned_tower_real_widths(real_width):
    from oracle.hf_oracle import synthetic_pixels
    cfg, acfg, sd, asd, eng, oracle = real_width
    pix = synthetic_pixels(2, 420)
    g = torch.Generator().manual_seed(5)
    caps = [torch.randint(0, 128000, (77,), generator=g), torch.randint(0, 128000, (20,), generator=g)]
    tok, pooled = eng.vit_encode_cond(pix.cuda(), [c.cuda() for c in caps])
    for b in range(2):
        ref_t, ref_p = oracle.vision_cond(pix[b:b + 1], caps[b])
        assert _rel(tok[b].cpu(), ref_t[0]) < 0.08, b
        assert _rel(pooled[b].cpu(), ref_p[0]) < 0.08, b
    # right-padded batch: the padded caption positions are masked keys
    ids = torch.full((2, 77), acfg.pad_token_id)
    mask = torch.zeros(2, 77, dtype=torch.long)
    for b, c in enumerate(caps):
        ids[b, : c.numel()], mask[b, : c.numel()] = c, 1
    ref_t, _ = oracle.vision_cond(pix, ids, mask)
    assert _rel(tok[1].cpu(), ref_t[1]) < 0.08
    # the plain tower is unchanged by an attached adapter, and the captions change the result
    plain, _ = eng.vit_encode(pix.cuda())
    assert _rel(plain[0].cpu(), oracle.vision(pix[:1])[0][0]) < 0.08
    assert _rel(plain[0].cpu(), tok[0].cpu()) > 0.1


@pytest.fixture(scope="module")
def tiny_model():
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from detikzify_b200.model import adapter as A
    cfg, acfg, sd, asd, eng, oracle = _bundle("tiny-v2")
    model = DetikzifyForCausalLM(cfg, engine=eng)
    model.adapter = A.CrossAttentionAdapter(cfg, acfg, eng.adapter_arena)
    model.embedding_model = A.CaptionEmbedder(acfg)
    return cfg, model, oracle


def _prompt(cfg, extra):
    return torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.tensor(extra)]).long()


def _gold():
    from pathlib import Path
    return torch.load(Path(__file__).parent / "golden" / "reference_adapter_tiny.pt", weights_only=False)


def test_tiny_matches_reference_adapter_golden(tiny_model):
    """Against what the reference's own modeling_adapter.py computed (tests/golden/make_reference_golden_adapter.py, same
    seeds as ``_bundle``): adapted tower, prefill logits and greedy ids of public generate(), text only and image + text."""
    from oracle.hf_oracle import synthetic_pixels
    cfg, model, oracle = tiny_model
    gold = _gold()
    eng = model.engine
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=gold["pixel_seed"])
    cap, prompt = gold["caption"], gold["prompt"]
    hidden, cond = eng.text_encode(cap.cuda(), want_hidden=True)
    assert (hidden.cpu() - gold["embed_hidden"]).abs().max().item() < 3e-2
    assert (cond.cpu() - gold["connector"]).abs().max().item() < 3e-2
    for key, p in (("image", pix), ("text", None)):
        p_dev = p if p is not None else model.adapter.dummy_pixels()
        tok, _ = eng.vit_encode_cond(p_dev.cuda(), [cap.cuda()], want_pooled=False)
        assert (tok[0].cpu() - gold[f"{key}_vision"]).abs().max().item() < 5e-2, key
        ref = gold[f"{key}_generate_ids"]
        out = model.generate(input_ids=prompt[None], pixel_values=p, adapter_input_ids=cap[None],
                             adapter_attention_mask=torch.ones(1, cap.numel(), dtype=torch.long),
                             bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
                             max_length=ref.numel(), do_sample=False)[0].cpu()
        # prefill logits of the prompt with the conditioned image span the call used
        _, alll = eng.prefill(model._slot, prompt.cuda(), 0, model._img_cache[1], 0, want_all_logits=True)
        model._slot_tokens = []
        assert (alll.cpu() - gold[f"{key}_logits"]).abs().max().item() < 3e-2, key
        n = min(out.numel(), ref.numel())
        diff = (out[:n] != ref[:n]).nonzero()
        if diff.numel():   # a divergence is only tolerated at a near-tie of the fp32 logits
            t = int(diff[0])
            top2 = oracle.forward_logits_cond(ref[None, :t], p, cap)[0, -1].topk(2).values
            assert (top2[0] - top2[1]).item() < 6e-2, (key, t, top2)
        else:
            assert out.numel() == ref.numel(), key
    # right-padded batch of two captions, no image: the padded positions are masked keys
    caps = [gold["batch_ids"][i][gold["batch_mask"][i].bool()].cuda() for i in range(2)]
    tok, _ = eng.vit_encode_cond(model.adapter.dummy_pixels().expand(2, -1, -1, -1).cuda(), caps, want_pooled=False)
    assert (tok.cpu() - gold["batch_vision"]).abs().max().item() < 5e-2


def test_tiny_caption_keys_the_caches(tiny_model):
    """One image under two captions: the KV the call leaves in its slot is the oracle's for THAT caption (a decode step on it
    matches the fp32 logits); a repeat of the same (image, caption) re-runs neither the caption encoder nor the tower."""
    from oracle.hf_oracle import synthetic_pixels
    cfg, model, oracle = tiny_model
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=77)
    ids = _prompt(cfg, [17, 40])
    kw = dict(bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id], max_length=ids.numel() + 1,
              do_sample=False)
    nxt = torch.tensor([123])
    for cap in (torch.tensor([3, 4, 5]), torch.tensor([200, 201, 202, 203, 9]), torch.tensor([3, 4, 5])):
        model.generate(input_ids=ids[None], pixel_values=pix, adapter_input_ids=cap[None], **kw)
        assert model._slot_tokens == ids.tolist()      # the slot holds the prompt's KV (image span included)
        lg = model.engine.decode([model._slot], [ids.numel()], nxt.cuda())[0].cpu()
        ref = oracle.forward_logits_cond(torch.cat([ids, nxt])[None], pix, cap)[0, -1]
        assert (lg - ref).abs().max().item() < 3e-2, cap
    before = model.engine.launch_count
    model.generate(input_ids=ids[None], pixel_values=pix, adapter_input_ids=torch.tensor([[7, 8]]), **kw)
    miss = model.engine.launch_count - before
    before = model.engine.launch_count
    model.generate(input_ids=ids[None], pixel_values=pix, adapter_input_ids=torch.tensor([[7, 8]]), **kw)
    hit = model.engine.launch_count - before
    # the repeat re-runs neither the caption encoder nor the tower (>= 19 launches per vision layer with its cross layer)
    assert miss - hit >= 19 * cfg.vision_config.num_hidden_layers, (miss, hit)
    with pytest.raises(ValueError):
        model.generate_batch([ids, ids], pixel_values=pix, adapter_input_ids=torch.tensor([[1, 2], [3, 4], [5, 6]]), **kw)


def test_selfsim_with_caption_on_the_target_side(tiny_model):
    """ImageSim (reference evaluate/imagesim.py:61-142): the target side (image or none, plus text2) on the adapted tower,
    candidates on the plain tower, against the oracle; the batched path gives the same values and encodes the target once."""
    import torch.nn.functional as F
    from PIL import Image
    from detikzify_b200.evaluate.imagesim import ImageSim
    from detikzify_b200.model import build_processor
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.processing import AdapterProcessor
    cfg, model, oracle = tiny_model
    proc = AdapterProcessor(processor=build_processor(cfg), tokenizer=A._load_tokenizer("tiny", model.adapter.config))
    sim = ImageSim.from_detikzify(model, proc, mode="cos", preprocess=False)
    figs = [Image.new("RGB", (60, 50), c) for c in ("white", "red")]
    for i, f in enumerate(figs):
        f.paste((0, 0, 255), (5 + 10 * i, 5, 30, 40))
    caption = "a blue square"
    ids = torch.tensor(list(caption.encode()))
    ip = proc.processor.image_processor
    for target in (figs[1], None):
        sim.reset()
        sim.update(img1=figs[0], img2=target, text2=caption)
        got = sim.compute()
        p0 = ip(images=figs[0], return_tensors="pt")["pixel_values"]
        pt = ip(images=target, return_tensors="pt")["pixel_values"] if target is not None else None
        ref = F.cosine_similarity(oracle.vision(p0)[1][0].double(), oracle.vision_cond(pt, ids)[1][0].double(), dim=0).item()
        assert abs(got - ref) < 2e-2, (target is None, got, ref)
        before = model.engine.launch_count
        both = sim.get_similarities(figs, target, text=caption)
        assert both[0] == pytest.approx(got, abs=1e-3)
        # the conditioned target is cached: one plain batched tower pass for the candidates (no caption encoder launches)
        assert model.engine.launch_count - before < 19 * cfg.vision_config.num_hidden_layers
    with pytest.raises(ValueError):
        ImageSim.from_detikzify(model, proc.processor, mode="cos").update(img1=figs[0], text2=caption)


def test_tiny_generate_batch_per_sequence_captions(tiny_model):
    cfg, model, oracle = tiny_model
    caps = torch.tensor([[3, 4, 5, 0], [200, 201, 202, 203]])
    mask = torch.tensor([[1, 1, 1, 0], [1, 1, 1, 1]])
    ids = _prompt(cfg, [17, 40])
    outs = model.generate_batch([ids, ids], adapter_input_ids=caps, adapter_attention_mask=mask,
                                bad_words_ids=[[cfg.image_token_id]], begin_suppress_tokens=[cfg.eos_token_id],
                                max_length=ids.numel() + 1, do_sample=False)
    for i, cap in enumerate((caps[0, :3], caps[1])):
        ref = oracle.forward_logits_cond(ids[None], None, cap)[0, -1]
        ref[cfg.image_token_id] = ref[cfg.eos_token_id] = -float("inf")
        top2 = ref.topk(2).values
        assert int(outs[i][-1]) == int(ref.argmax()) or (top2[0] - top2[1]).item() < 6e-2, i


def test_pipeline_text_only_sample():
    from detikzify_b200.infer.pipeline import DetikzifyPipeline
    from detikzify_b200.infer.tikz import TikzDocument
    from detikzify_b200.model import adapter, load
    model, processor = load("tiny", device_map=0)
    model, processor = adapter.load(model, processor, embedding_model="tiny")
    assert hasattr(model, "adapter")
    doc = DetikzifyPipeline(model, processor, metric="fast").sample(text="a blue square")
    assert isinstance(doc, TikzDocument)
    model.unload_cross_attn_adapter()
    assert not hasattr(model, "adapter")
