"""
TikZero adapter host logic without a GPU: the adapter arena layout through the C ABI, checkpoint-directory mapping, the
AdapterProcessor (reference model/adapter/processing_adapter.py), ``has_adapter`` / ``unload_cross_attn_adapter`` / the
reference's ValueError, and the caption path of ``generate`` / the pipeline on a scripted engine.
"""
import ctypes as C

import pytest
import torch

from scripted_engine import ScriptedEngine


def test_adapter_weight_table_through_abi():
    from detikzify_b200 import _lib
    from detikzify_b200.engine import to_c_config
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    cfg, acfg = preset("v2-8b"), A.adapter_preset("llama-3.2-1b")
    table = A.adapter_weight_table(cfg, acfg)
    names = [t.name.decode() for t in table]
    assert names[0] == "emb.embed" and names[-1] == "ad.dummy"
    assert names.index("emb.norm") == 1 + 6 * 16 and names[1 + 6 * 16 + 1: 1 + 6 * 16 + 3] == ["ad.connector_w", "ad.connector_b"]
    shape = {t.name.decode(): (t.rows, t.cols) for t in table}
    assert shape["emb.embed"] == (128256, 2048)
    assert shape["emb.L0.wqkv"] == ((32 + 16) * 64, 2048) and shape["emb.L15.wgu"] == (2 * 8192, 2048)
    assert shape["ad.connector_w"] == (1152, 2048)
    assert shape["ad.L26.wkv"] == (2304, 1152) and shape["ad.L26.bkv"] == (1, 2304) and shape["ad.L26.q_norm_w"] == (1, 72)
    assert shape["ad.L0.attn_gate"] == (1, 1) and shape["ad.dummy"] == (3, 420 * 420)
    assert sum(n.startswith("ad.L") and n.endswith(".wq") for n in names) == 27
    offs = [t.offset for t in table]
    assert all(o % 256 == 0 for o in offs) and offs == sorted(offs)
    lib = _lib.load_library()
    total = lib.dtk_adapter_arena_bytes(C.byref(to_c_config(cfg)), C.byref(A.to_c_adapter_config(acfg)))
    assert total >= table[-1].offset + table[-1].nbytes
    # cross layer every 3rd vision layer; embedder head_dim other than 64 is rejected
    acfg3 = A.adapter_preset("llama-3.2-1b")
    acfg3.cross_attn_every_n_layers = 3
    assert A.cross_layers(cfg, acfg3) == [2, 5, 8, 11, 14, 17, 20, 23, 26]
    assert sum(t.name.decode().endswith(".wq") for t in A.adapter_weight_table(cfg, acfg3)) == 9
    bad = A.to_c_adapter_config(acfg)
    bad.head_dim = 128
    assert lib.dtk_adapter_weight_count(C.byref(to_c_config(cfg)), C.byref(bad)) < 0


def test_pack_arena_places_every_tensor():
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    cfg, acfg = preset("tiny-v2"), A.adapter_preset("tiny")
    sd = A.random_init(cfg, acfg, seed=3)
    assert set(sd) == set(A.canonical_shapes(cfg, acfg))
    assert all(tuple(v.shape) == A.canonical_shapes(cfg, acfg)[k] for k, v in sd.items())
    g0, g1 = sd["adapter.layers.0.cross_attn_attn_gate"], sd["adapter.layers.0.cross_attn_mlp_gate"]
    assert g0.item() != 0 and g1.item() != 0 and g0.item() != g1.item()
    arena = A.pack_arena(cfg, acfg, sd)
    table = {t.name.decode(): t for t in A.adapter_weight_table(cfg, acfg)}

    def get(name):
        t = table[name]
        return arena[t.offset // 2: t.offset // 2 + t.rows * t.cols].view(t.rows, t.cols).float()
    p = "adapter.layers.1.cross_attn."
    wkv = torch.cat([sd[p + "k_proj.weight"], sd[p + "v_proj.weight"]]).bfloat16().float()
    assert torch.equal(get("ad.L1.wkv"), wkv)
    assert torch.equal(get("ad.L1.mlp_gate").view(1), sd["adapter.layers.1.cross_attn_mlp_gate"].bfloat16().float())
    g, u = sd["embedding_model.layers.0.mlp.gate_proj.weight"], sd["embedding_model.layers.0.mlp.up_proj.weight"]
    assert torch.equal(get("emb.L0.wgu")[0::2], g.bfloat16().float()) and torch.equal(get("emb.L0.wgu")[1::2], u.bfloat16().float())


def test_checkpoint_directories_map_to_canonical_names(tmp_path):
    from safetensors.torch import save_file
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    cfg, acfg = preset("tiny-v2"), A.adapter_preset("tiny")
    sd = A.random_init(cfg, acfg, seed=1)
    (tmp_path / "adapter").mkdir()
    (tmp_path / "emb").mkdir()
    save_file({k[len("adapter."):]: v.contiguous() for k, v in sd.items() if k.startswith("adapter.")},
              str(tmp_path / "adapter" / "model.safetensors"))
    emb = {"model." + k[len("embedding_model."):]: v.contiguous() for k, v in sd.items() if k.startswith("embedding_model.")}
    emb["lm_head.weight"] = torch.zeros(4, 4)
    save_file(emb, str(tmp_path / "emb" / "model.safetensors"))
    got = {**A.load_adapter_dir(str(tmp_path / "adapter")), **A.load_embedder_dir(str(tmp_path / "emb"))}
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    assert A.load_adapter_dir(str(tmp_path / "missing")) is None


def _processor(cfg_name="tiny"):
    from detikzify_b200.model import build_processor
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.processing import AdapterProcessor
    cfg, acfg = preset(cfg_name), A.adapter_preset("tiny")
    return cfg, acfg, AdapterProcessor(processor=build_processor(cfg), tokenizer=A._load_tokenizer("tiny", acfg))


def test_adapter_processor_keys_dummy_image_truncation_padding():
    from PIL import Image
    cfg, acfg, proc = _processor()
    enc = proc(text="a blue square", return_tensors="pt")
    assert set(enc) == {"input_ids", "attention_mask", "adapter_input_ids", "adapter_attention_mask"}   # no pixel_values
    assert (enc["input_ids"][0] == cfg.image_token_id).sum() == cfg.num_patches
    assert enc["adapter_input_ids"].tolist() == [list(b"a blue square")]
    enc = proc(images=Image.new("RGB", (40, 30), "red"), text="x", return_tensors="pt")
    assert {"pixel_values", "input_ids", "adapter_input_ids"} <= set(enc)
    assert "adapter_input_ids" not in proc(images=Image.new("RGB", (8, 8)), return_tensors="pt")
    long = "y" * (acfg.max_text + 40)
    enc = proc(text=long, text_kwargs={"truncation": True}, return_tensors="pt")
    assert enc["adapter_input_ids"].shape == (1, acfg.max_text)
    enc = proc(text=["ab", "abcd"], text_kwargs={"padding": True}, return_tensors="pt")
    assert enc["adapter_input_ids"].tolist() == [[97, 98, acfg.pad_token_id, acfg.pad_token_id], [97, 98, 99, 100]]
    assert enc["adapter_attention_mask"].tolist() == [[1, 1, 0, 0], [1, 1, 1, 1]]
    with pytest.raises(ValueError):
        proc()


class CaptionEngine(ScriptedEngine):
    """Scripted engine with the conditioned tower: records the caption each tower pass is conditioned on."""

    def image_embeds_cond(self, pix, captions):
        self.calls.append(("image_embeds_cond", tuple(pix.shape), tuple(tuple(c.tolist()) for c in captions)))
        return torch.zeros(pix.shape[0], self.P, self.H)

    def adapter_detach(self):
        self.calls.append(("adapter_detach",))


def _scripted_model():
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    cfg, acfg = preset("tiny"), A.adapter_preset("tiny")   # "tiny": the synthetic tokenizer knows its image token
    eng = CaptionEngine(cfg)
    model = DetikzifyForCausalLM(cfg, engine=eng, max_seqs=4)
    return cfg, acfg, eng, model


def _attach(model, cfg, acfg):
    from detikzify_b200.model import adapter as A
    S = cfg.vision_config.image_size
    model.adapter = A.CrossAttentionAdapter.__new__(A.CrossAttentionAdapter)
    model.adapter.config, model.adapter.layers = acfg, A.cross_layers(cfg, acfg)
    model.adapter.dummy_input = torch.linspace(-2, 2, 3 * S * S).view(3, S, S)
    model.embedding_model = A.CaptionEmbedder(acfg)


def test_has_adapter_value_error_and_caption_keyed_caches():
    from detikzify_b200.infer.pipeline import has_adapter
    cfg, acfg, eng, model = _scripted_model()
    ids = torch.cat([torch.full((cfg.num_patches,), cfg.patch_token_id), torch.tensor([40, 41])])[None]
    kw = dict(max_length=ids.shape[1] + 2, bad_words_ids=[[cfg.image_token_id]])
    assert not has_adapter(model) and not model.has_adapter()
    with pytest.raises(ValueError, match="no adapter is loaded"):
        model.generate(input_ids=ids, adapter_input_ids=torch.tensor([[1, 2]]), **kw)
    _attach(model, cfg, acfg)
    assert has_adapter(model) and model.has_adapter()
    pix = torch.zeros(1, 3, cfg.vision_config.image_size, cfg.vision_config.image_size)
    model.generate(input_ids=ids, pixel_values=pix, adapter_input_ids=torch.tensor([[5, 6, 0]]),
                   adapter_attention_mask=torch.tensor([[1, 1, 0]]), **kw)
    model.generate(input_ids=ids, pixel_values=pix, adapter_input_ids=torch.tensor([[5, 6]]), **kw)   # same (image, caption)
    model.generate(input_ids=ids, pixel_values=pix, adapter_input_ids=torch.tensor([[7]]), **kw)      # same image, new caption
    model.generate(input_ids=ids, pixel_values=pix, **kw)                                             # same image, no caption
    towers = [c for c in eng.calls if c[0] in ("image_embeds", "image_embeds_cond")]
    assert [c[0] for c in towers] == ["image_embeds_cond", "image_embeds_cond", "image_embeds"]
    assert towers[0][2] == ((5, 6),) and towers[1][2] == ((7,),)
    prefills = [c for c in eng.calls if c[0] == "prefill"]
    # a new caption invalidates the image-span KV: every tower pass is followed by a prefill from position 0
    assert [p[2] for p in prefills] == [0, ids.shape[1] - 1, 0, 0]
    # text only: the tower input is the clamped dummy image
    eng.calls.clear()
    model.generate(input_ids=ids, adapter_input_ids=torch.tensor([[9, 9]]), **kw)
    assert [c for c in eng.calls if c[0] == "image_embeds_cond"][0][1] == (1, 3, cfg.vision_config.image_size, cfg.vision_config.image_size)
    assert model._img_cache[0].min() == -1 and model._img_cache[0].max() == 1
    model.unload_cross_attn_adapter()
    assert not has_adapter(model) and ("adapter_detach",) in eng.calls and model._img_cache is None


def test_pipeline_text_only_sample_forwards_the_caption():
    from detikzify_b200.infer.pipeline import DetikzifyPipeline
    from detikzify_b200.infer.tikz import TikzDocument
    cfg, acfg, eng, model = _scripted_model()
    _, _, proc = _processor()
    pipe = DetikzifyPipeline(model, proc, metric="fast")
    with pytest.raises(AssertionError):
        pipe.sample(text="a circle")          # no adapter loaded
    _attach(model, cfg, acfg)
    doc = pipe.sample(text="a blue square")
    assert isinstance(doc, TikzDocument)
    conds = [c for c in eng.calls if c[0] == "image_embeds_cond"]
    assert conds and conds[0][2] == (tuple(b"a blue square"),)


def test_adapter_oracle_matches_reference_golden():
    """oracle/adapter_oracle.py against what the reference's own modeling_adapter.py computed
    (tests/golden/make_reference_golden_adapter.py): fp32, greedy ids equal."""
    from pathlib import Path
    from detikzify_b200.model import adapter as A
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.weights import random_init
    from oracle.adapter_oracle import AdapterOracle
    from oracle.hf_oracle import synthetic_pixels
    gold = torch.load(Path(__file__).parent / "golden" / "reference_adapter_tiny.pt", weights_only=False)
    cfg, acfg = preset("tiny-v2"), A.adapter_preset("tiny")
    oracle = AdapterOracle(cfg.to_dict(), random_init(cfg, seed=gold["seed"]), acfg,
                           A.random_init(cfg, acfg, seed=gold["adapter_seed"]))
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=gold["pixel_seed"])
    cap, prompt = gold["caption"], gold["prompt"]
    tol = 2e-5
    h, c = oracle.caption_states(cap)
    assert (h[0] - gold["embed_hidden"]).abs().max() < tol and (c[0] - gold["connector"]).abs().max() < tol
    for key, p in (("image", pix), ("text", None)):
        vis, _ = oracle.vision_cond(p, cap)
        assert (vis[0] - gold[f"{key}_vision"]).abs().max() < tol, key
        assert (oracle.forward_logits_cond(prompt[None], p, cap)[0] - gold[f"{key}_logits"]).abs().max() < tol, key
        ids = oracle.generate_cond(prompt[None], p, cap, max_length=gold[f"{key}_generate_ids"].numel())
        assert torch.equal(ids[0], gold[f"{key}_generate_ids"]), key
    vis, _ = oracle.vision_cond(None, gold["batch_ids"], gold["batch_mask"])
    assert (vis - gold["batch_vision"]).abs().max() < tol
