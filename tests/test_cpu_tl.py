"""
detikzify-tl-1.1b (TinyLlama-1.1B decoder: head_dim 64, GQA 32/4) and detikzify-cl-7b on the CPU side: the fp32 oracle
against the reference's own v1 model code at the ``tiny-tl`` test shape (tests/golden/reference_v1_tl.pt, written by
make_reference_golden_tl.py), the presets, ``config_from_dict`` on a TinyLlama-style flat v1 config.json, and the C ABI's
weight table / byte counts at head_dim 64.
"""
import ctypes as C
from dataclasses import replace
from pathlib import Path

import torch

from conftest import model_bundle

GOLD = torch.load(Path(__file__).parent / "golden" / "reference_v1_tl.pt", weights_only=False)


def test_oracle_matches_reference_model_code_tiny_tl():
    from oracle.hf_oracle import synthetic_pixels
    cfg, sd, oracle = model_bundle("tiny-tl")
    g = GOLD["tiny-tl"]
    ids = g["input_ids"][None]
    assert cfg.patch_token_id in ids[0, 1:-1].tolist()    # the image span sits in mid-prompt
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=g["pixel_seed"])
    logits, cache = oracle.forward_logits(ids, pix, use_cache=True)
    assert (logits[0] - g["logits"]).abs().max().item() < 2e-5
    assert int(logits[0, -1].argmax()) == g["next_id"]
    dec, _ = oracle.decode_logits(torch.tensor([[g["next_id"]]]), cache)
    assert (dec[0, -1] - g["decode_logits"]).abs().max().item() < 2e-5
    tokens, _ = oracle.vision(pix)
    n, c = cfg.num_patches, cfg.concat_patches
    feats = tokens[:, tokens.shape[1] - n * c:].reshape(-1, n, tokens.shape[-1] * c)[0]
    assert (feats - g["vision_features"]).abs().max().item() < 2e-5
    out = oracle.generate(g["generate_prompt"][None], pix, max_length=g["generate_ids"].numel())
    assert out[0].tolist() == g["generate_ids"].tolist()


def test_oracle_matches_reference_model_code_at_tl11b_shape():
    from oracle.hf_oracle import synthetic_pixels
    g = GOLD["tl-1.1b"]
    cfg, sd, oracle = model_bundle("nllg/detikzify-tl-1.1b")
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=g["pixel_seed"])
    logits, cache = oracle.forward_logits(g["input_ids"][None], pix, use_cache=True)
    assert (logits[0, -1] - g["last_logits"]).abs().max().item() < 2e-4
    assert int(logits[0, -1].argmax()) == g["next_id"]
    dec, _ = oracle.decode_logits(torch.tensor([[g["next_id"]]]), cache)
    assert (dec[0, -1] - g["decode_logits"]).abs().max().item() < 2e-4


def test_presets_cover_every_v1_checkpoint():
    from detikzify_b200.model import v1_models
    from detikzify_b200.model.configuration import preset
    assert v1_models == ["nllg/detikzify-ds-1.3b", "nllg/detikzify-ds-7b", "nllg/detikzify-tl-1.1b", "nllg/detikzify-cl-7b"]
    for name in v1_models:
        assert preset(name).name_or_path == name
    tl = preset("nllg/detikzify-tl-1.1b")
    assert (tl.hidden_size, tl.intermediate_size, tl.num_hidden_layers) == (2048, 5632, 22)
    assert (tl.num_attention_heads, tl.num_key_value_heads, tl.head_dim) == (32, 4, 64)
    assert (tl.vocab_size, tl.bos_token_id, tl.eos_token_id, tl.pad_token_id, tl.patch_token_id) == (32008, 1, 2, 32000, 1)
    assert (tl.rope_theta, tl.rope_factor, tl.rms_norm_eps, tl.model_max_length) == (10000.0, 1.0, 1e-5, 2048)
    assert replace(preset("tl-1.1b"), name_or_path="") == replace(tl, name_or_path="")
    cl = preset("nllg/detikzify-cl-7b")
    assert (cl.hidden_size, cl.intermediate_size, cl.num_hidden_layers, cl.num_attention_heads, cl.head_dim) == (4096, 11008, 32, 32, 128)
    assert (cl.rope_theta, cl.rope_factor, cl.vocab_size) == (1e6, 1.0, 32024)
    cl2 = preset("cl-7b-2l")
    assert cl2.num_hidden_layers == 2 and (cl2.hidden_size, cl2.vocab_size) == (4096, 32024)
    tiny = preset("tiny-tl")
    assert tiny.head_dim == 64 and tiny.hidden_size // tiny.num_attention_heads == 64
    assert tiny.num_attention_heads // tiny.num_key_value_heads == 8
    assert tiny.vocab_size % 16 == 8 and tiny.rope_factor == 1.0


def test_config_from_tinyllama_style_v1_config_json():
    from detikzify_b200.model.configuration import config_from_dict, preset
    d = {   # flat LLaMA config + the fields initialize_vision_modules writes; no head_dim key (derived from hidden / heads)
        "architectures": ["DetikzifyForCausalLM"], "model_type": "detikzify", "hidden_size": 2048, "intermediate_size": 5632,
        "num_hidden_layers": 22, "num_attention_heads": 32, "num_key_value_heads": 4, "vocab_size": 32008,
        "max_position_embeddings": 2048, "rms_norm_eps": 1e-05, "rope_theta": 10000.0, "rope_scaling": None,
        "bos_token_id": 1, "eos_token_id": 2, "pad_token_id": 32000, "hidden_act": "silu", "tie_word_embeddings": False,
        "patch_token_id": 1, "concat_patches": 3, "num_patches": 243, "use_mm_proj": True, "mm_hidden_size": 3456,
        "vision_tower": "vit_so400m_patch14_siglip_384.webli", "feature_layer": -1}
    cfg = config_from_dict(d, name="local-tl")
    ref = preset("nllg/detikzify-tl-1.1b")
    for f in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "num_key_value_heads", "head_dim",
              "vocab_size", "rms_norm_eps", "rope_theta", "rope_factor", "rope_type", "bos_token_id", "eos_token_id",
              "pad_token_id", "patch_token_id", "concat_patches", "projector_bias"):
        assert getattr(cfg, f) == getattr(ref, f), f
    assert cfg.num_patches == 243


def test_abi_accepts_head_dim_64_and_rejects_others():
    from detikzify_b200 import _lib
    from detikzify_b200.engine import to_c_config, weight_table
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.weights import param_count
    lib = _lib.load_library()
    for name in ("tiny-tl", "nllg/detikzify-tl-1.1b"):
        cfg = preset(name)
        cc = to_c_config(cfg)
        assert lib.dtk_weight_count(C.byref(cc)) > 0
        table = weight_table(cc)
        pad = cfg.vision_config.hidden_size * (-(3 * 14 * 14) % 64)   # patch-embed K padded to a multiple of 64
        assert sum(t.rows * t.cols for t in table) == param_count(cfg) + pad
        wqkv = next(t for t in table if t.name.decode() == "dec.L0.wqkv")
        assert (wqkv.rows, wqkv.cols) == ((cfg.num_attention_heads + 2 * cfg.num_key_value_heads) * 64, cfg.hidden_size)
        assert lib.dtk_arena_bytes(C.byref(cc)) > 0
    for hd in (96, 32, 256):
        cc = to_c_config(preset("tiny-tl"))
        cc.head_dim = hd
        assert lib.dtk_weight_count(C.byref(cc)) < 0
        assert lib.dtk_arena_bytes(C.byref(cc)) == 0
    cc = to_c_config(preset("tiny"))   # head_dim 64 with heads * head_dim != hidden
    cc.head_dim = 64
    assert lib.dtk_weight_count(C.byref(cc)) < 0


def test_decode_bytes_tl11b():
    from detikzify_b200 import _lib
    from detikzify_b200.engine import to_c_config
    from detikzify_b200.model.configuration import preset
    lib = _lib.load_library()
    cc = to_c_config(preset("nllg/detikzify-tl-1.1b"))
    for T in (0, 243, 2048):
        assert lib.dtk_decode_bytes(C.byref(cc), T) == 2_068_873_216 + T * 22_528

