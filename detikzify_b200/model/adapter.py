"""
``detikzify_b200.model.adapter.load`` — drop-in for ``detikzify.model.adapter.load`` (reference
detikzify/model/adapter/__init__.py:9-22): TikZero text conditioning.

    model, processor = load("nllg/detikzify-v2.5-8b", device_map=0)
    model, processor = adapter.load(model, processor)
    DetikzifyPipeline(model, processor).sample(text="a blue square")

A caption is embedded by a Llama-3.2-1B ``LlamaModel`` (final-norm hidden states), mapped to the vision width by the
adapter's ``connector`` and read by one gated cross-attention layer before every ``cross_attn_every_n_layers``-th ViT layer
(reference model/adapter/modeling_adapter.py:293-394). Everything runs in the engine: ``dtk_text_encode`` and
``dtk_vit_encode_cond`` over a second bf16 weight arena attached to the model's engine.

Weights: the adapter from ``adapter_name_or_path`` (or ``<model>/adapter``) ``*.safetensors`` with the reference's names,
the embedder from a local Llama-3.2-1B directory (with or without the ``model.`` prefix). Whatever is not found is, offline,
a seeded random init (``random_init_weights=False`` raises instead).
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import asdict, dataclass, replace
from glob import glob
from typing import Dict, List, Optional

import torch

from .. import _lib
from .._lib import DtkAdapterConfig, DtkWeightInfo
from ..engine import EngineError, to_c_config
from .processing import AdapterProcessor, SyntheticTokenizer

EMB = "embedding_model."
AD = "adapter."


@dataclass
class AdapterConfig:
    """Caption embedder dims (a LlamaModel with head_dim 64) and the adapter's layout. Defaults: Llama-3.2-1B, the public
    base config (like the decoder dims of the model presets, configuration input rather than reference source)."""
    hidden_size: int = 2048
    intermediate_size: int = 8192
    num_hidden_layers: int = 16
    num_attention_heads: int = 32
    num_key_value_heads: int = 8
    head_dim: int = 64
    vocab_size: int = 128256
    rms_norm_eps: float = 1e-5
    rope_theta: float = 500000.0
    rope_type: str = "llama3"
    rope_factor: float = 32.0
    rope_low_freq_factor: float = 1.0
    rope_high_freq_factor: float = 4.0
    rope_original_max_position: int = 8192
    max_text: int = 512                  # tokenizer model_max_length (reference adapter/__init__.py:17)
    pad_token_id: int = 128004           # <|finetune_right_pad_id|>
    cross_attn_every_n_layers: int = 1
    name_or_path: str = "meta-llama/Llama-3.2-1B"

    def to_dict(self):
        return asdict(self)


def adapter_preset(name: str) -> AdapterConfig:
    """``llama-3.2-1b`` (the reference's embedder), ``llama-3.2-1b-2l`` (every embedder matrix shape, two layers: parity tests)
    and ``tiny`` (head_dim 64 at a CPU-test size)."""
    key = name.split("/")[-1].lower()
    if key == "llama-3.2-1b":
        return AdapterConfig(name_or_path=name)
    if key == "llama-3.2-1b-2l":
        return AdapterConfig(num_hidden_layers=2, name_or_path=name)
    if key == "tiny":
        # short original context so that all three llama3 frequency bands occur
        return AdapterConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                             num_key_value_heads=2, vocab_size=640, rope_factor=8.0, rope_original_max_position=64,
                             max_text=96, pad_token_id=604, name_or_path=name)
    raise KeyError(f"unknown adapter embedder preset {name!r}")


def _config_from_json(path: str, name: str) -> AdapterConfig:
    import json
    with open(os.path.join(path, "config.json")) as f:
        d = json.load(f)
    rs = d.get("rope_scaling") or d.get("rope_parameters") or {}
    heads = int(d["num_attention_heads"])
    return AdapterConfig(
        hidden_size=int(d["hidden_size"]), intermediate_size=int(d["intermediate_size"]),
        num_hidden_layers=int(d["num_hidden_layers"]), num_attention_heads=heads,
        num_key_value_heads=int(d.get("num_key_value_heads", heads)), head_dim=int(d.get("head_dim") or d["hidden_size"] // heads),
        vocab_size=int(d["vocab_size"]), rms_norm_eps=float(d.get("rms_norm_eps", 1e-5)),
        rope_theta=float(d.get("rope_theta", rs.get("rope_theta", 500000.0))),
        rope_type="llama3" if rs.get("rope_type", rs.get("type")) == "llama3" else "linear",
        rope_factor=float(rs.get("factor", 1.0)), rope_low_freq_factor=float(rs.get("low_freq_factor", 1.0)),
        rope_high_freq_factor=float(rs.get("high_freq_factor", 4.0)),
        rope_original_max_position=int(rs.get("original_max_position_embeddings", 8192)), name_or_path=name)


def to_c_adapter_config(acfg: AdapterConfig) -> DtkAdapterConfig:
    return DtkAdapterConfig(
        hidden=acfg.hidden_size, inter=acfg.intermediate_size, layers=acfg.num_hidden_layers, heads=acfg.num_attention_heads,
        kv_heads=acfg.num_key_value_heads, head_dim=acfg.head_dim, vocab=acfg.vocab_size, rms_eps=acfg.rms_norm_eps,
        rope_theta=acfg.rope_theta, rope_factor=acfg.rope_factor, rope_type={"linear": 0, "llama3": 1}[acfg.rope_type],
        rope_low_freq=acfg.rope_low_freq_factor, rope_high_freq=acfg.rope_high_freq_factor,
        rope_orig_max_pos=acfg.rope_original_max_position, max_text=acfg.max_text,
        cross_every_n=acfg.cross_attn_every_n_layers)


def adapter_weight_table(cfg, acfg: AdapterConfig) -> List[DtkWeightInfo]:
    lib = _lib.load_library()
    ccfg, cacfg = to_c_config(cfg), to_c_adapter_config(acfg)
    n = lib.dtk_adapter_weight_count(C.byref(ccfg), C.byref(cacfg))
    if n <= 0:
        raise EngineError("invalid adapter configuration (dtk_adapter_weight_count): the embedder head_dim must be 64")
    out = []
    for i in range(n):
        info = DtkWeightInfo()
        if lib.dtk_adapter_weight_get(C.byref(ccfg), C.byref(cacfg), i, C.byref(info)) != 0:
            raise EngineError("dtk_adapter_weight_get failed")
        out.append(info)
    return out


def cross_layers(cfg, acfg: AdapterConfig) -> List[int]:
    n = acfg.cross_attn_every_n_layers
    return [l for l in range(cfg.vision_config.num_hidden_layers) if (l + 1) % n == 0]


def canonical_shapes(cfg, acfg: AdapterConfig) -> Dict[str, tuple]:
    """Canonical state dict: ``embedding_model.`` + LlamaModel names, ``adapter.`` + CrossAttentionAdapter names."""
    E, I, hd = acfg.hidden_size, acfg.intermediate_size, acfg.head_dim
    qd, kd = acfg.num_attention_heads * hd, acfg.num_key_value_heads * hd
    vc = cfg.vision_config
    D, VI, dh = vc.hidden_size, vc.intermediate_size, vc.head_dim
    s = {EMB + "embed_tokens.weight": (acfg.vocab_size, E), EMB + "norm.weight": (E,)}
    for l in range(acfg.num_hidden_layers):
        p = f"{EMB}layers.{l}."
        s.update({p + "input_layernorm.weight": (E,), p + "post_attention_layernorm.weight": (E,),
                  p + "self_attn.q_proj.weight": (qd, E), p + "self_attn.k_proj.weight": (kd, E),
                  p + "self_attn.v_proj.weight": (kd, E), p + "self_attn.o_proj.weight": (E, qd),
                  p + "mlp.gate_proj.weight": (I, E), p + "mlp.up_proj.weight": (I, E), p + "mlp.down_proj.weight": (E, I)})
    s.update({AD + "connector.weight": (D, E), AD + "connector.bias": (D,), AD + "dummy_input": (3, vc.image_size, vc.image_size)})
    for l in cross_layers(cfg, acfg):
        p = f"{AD}layers.{l}."
        for n in ("q", "k", "v", "out"):
            s[p + f"cross_attn.{n}_proj.weight"], s[p + f"cross_attn.{n}_proj.bias"] = (D, D), (D,)
        for n in ("q_norm", "k_norm"):
            s[p + f"cross_attn.{n}.weight"], s[p + f"cross_attn.{n}.bias"] = (dh,), (dh,)
        for n in ("layer_norm1", "layer_norm2"):
            s[p + f"{n}.weight"], s[p + f"{n}.bias"] = (D,), (D,)
        s.update({p + "mlp.fc1.weight": (VI, D), p + "mlp.fc1.bias": (VI,), p + "mlp.fc2.weight": (D, VI),
                  p + "mlp.fc2.bias": (D,), p + "cross_attn_attn_gate": (1,), p + "cross_attn_mlp_gate": (1,)})
    return s


def random_init(cfg, acfg: AdapterConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """Seeded synthetic weights (fp32, CPU): matrices and biases N(0, 0.02^2), norm gains 1 + N(0, 0.02^2), gates N(0, 1)
    (non-zero and different per layer, so that a swapped attention / MLP gate changes the result), and a dummy image that
    exceeds [-1, 1] (the clamp is exercised)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in canonical_shapes(cfg, acfg).items():
        if k.endswith("_gate"):
            sd[k] = torch.randn(shp, generator=g)
        elif k.endswith("dummy_input"):
            sd[k] = 3 * torch.rand(shp, generator=g) - 1.5
        elif k.endswith("norm.weight") or k.endswith("layernorm.weight") or "layer_norm" in k and k.endswith(".weight") \
                or k.endswith("_norm.weight"):
            sd[k] = 1 + 0.02 * torch.randn(shp, generator=g)
        else:
            sd[k] = 0.02 * torch.randn(shp, generator=g)
    return sd


def _arena_source(name: str, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    parts = name.split(".")
    if name == "emb.embed":
        return sd[EMB + "embed_tokens.weight"]
    if name == "emb.norm":
        return sd[EMB + "norm.weight"]
    if parts[0] == "emb":
        p, k = f"{EMB}layers.{int(parts[1][1:])}.", parts[2]
        if k == "norm1":
            return sd[p + "input_layernorm.weight"]
        if k == "norm2":
            return sd[p + "post_attention_layernorm.weight"]
        if k == "wqkv":
            return torch.cat([sd[p + f"self_attn.{n}_proj.weight"] for n in "qkv"], dim=0)
        if k == "wo":
            return sd[p + "self_attn.o_proj.weight"]
        if k == "wgu":   # interleaved rows: 2i = gate_i, 2i+1 = up_i
            g, u = sd[p + "mlp.gate_proj.weight"], sd[p + "mlp.up_proj.weight"]
            return torch.stack([g, u], dim=1).reshape(-1, g.shape[1])
        if k == "wd":
            return sd[p + "mlp.down_proj.weight"]
    if name == "ad.connector_w":
        return sd[AD + "connector.weight"]
    if name == "ad.connector_b":
        return sd[AD + "connector.bias"]
    if name == "ad.dummy":
        return sd[AD + "dummy_input"]
    if parts[0] == "ad":
        p, k = f"{AD}layers.{int(parts[1][1:])}.", parts[2]
        simple = {"ln1_w": "layer_norm1.weight", "ln1_b": "layer_norm1.bias", "ln2_w": "layer_norm2.weight",
                  "ln2_b": "layer_norm2.bias", "wq": "cross_attn.q_proj.weight", "bq": "cross_attn.q_proj.bias",
                  "wo": "cross_attn.out_proj.weight", "bo": "cross_attn.out_proj.bias",
                  "q_norm_w": "cross_attn.q_norm.weight", "q_norm_b": "cross_attn.q_norm.bias",
                  "k_norm_w": "cross_attn.k_norm.weight", "k_norm_b": "cross_attn.k_norm.bias",
                  "w1": "mlp.fc1.weight", "b1": "mlp.fc1.bias", "w2": "mlp.fc2.weight", "b2": "mlp.fc2.bias",
                  "attn_gate": "cross_attn_attn_gate", "mlp_gate": "cross_attn_mlp_gate"}
        if k in simple:
            return sd[p + simple[k]]
        if k == "wkv":   # k_proj and v_proj packed: one GEMM over the caption rows
            return torch.cat([sd[p + "cross_attn.k_proj.weight"], sd[p + "cross_attn.v_proj.weight"]], dim=0)
        if k == "bkv":
            return torch.cat([sd[p + "cross_attn.k_proj.bias"], sd[p + "cross_attn.v_proj.bias"]], dim=0)
    raise KeyError(name)


def pack_arena(cfg, acfg: AdapterConfig, sd: Dict[str, torch.Tensor]) -> torch.Tensor:
    """Pack the canonical state dict into the adapter arena (CPU bf16)."""
    lib = _lib.load_library()
    nbytes = lib.dtk_adapter_arena_bytes(C.byref(to_c_config(cfg)), C.byref(to_c_adapter_config(acfg)))
    if nbytes == 0:
        raise EngineError("invalid adapter configuration (dtk_adapter_arena_bytes)")
    arena = torch.zeros(nbytes // 2, dtype=torch.bfloat16)
    for info in adapter_weight_table(cfg, acfg):
        name = info.name.decode()
        src = _arena_source(name, sd).to(torch.bfloat16).reshape(-1)
        if src.numel() != info.rows * info.cols:
            raise EngineError(f"{name}: expected {info.rows}x{info.cols}, got {src.numel()} elements")
        arena[info.offset // 2: info.offset // 2 + src.numel()] = src
    return arena


def random_arena_device(cfg, acfg: AdapterConfig, device, seed: int = 0) -> torch.Tensor:
    """Synthetic adapter weights generated in the device arena (seconds instead of a 1.2 B-parameter host init); same
    distribution as ``random_init``, different random stream."""
    lib = _lib.load_library()
    nbytes = lib.dtk_adapter_arena_bytes(C.byref(to_c_config(cfg)), C.byref(to_c_adapter_config(acfg)))
    if nbytes == 0:
        raise EngineError("invalid adapter configuration (dtk_adapter_arena_bytes)")
    g = torch.Generator(device=device).manual_seed(seed)
    arena = (torch.randn(nbytes // 2, device=device, generator=g) * 0.02).to(torch.bfloat16)
    gains = ("norm1", "norm2", "norm", "ln1_w", "ln2_w", "q_norm_w", "k_norm_w")
    for info in adapter_weight_table(cfg, acfg):
        name, n = info.name.decode(), info.rows * info.cols
        sl = arena[info.offset // 2: info.offset // 2 + n]
        last = name.split(".")[-1]
        if last in gains:
            sl.copy_((sl.float() + 1.0).to(torch.bfloat16))
        elif last.endswith("_gate"):
            sl.copy_((sl.float() * 50.0).to(torch.bfloat16))
        elif last == "dummy":
            sl.copy_((torch.rand(n, device=device, generator=g) * 3 - 1.5).to(torch.bfloat16))
    return arena


def _safetensors(path: Optional[str]) -> Optional[Dict[str, torch.Tensor]]:
    if not path or not os.path.isdir(path):
        return None
    files = sorted(glob(os.path.join(path, "*.safetensors")))
    if not files:
        return None
    from safetensors.torch import load_file
    sd: Dict[str, torch.Tensor] = {}
    for f in files:
        sd.update(load_file(f))
    return sd


def load_adapter_dir(path: str) -> Optional[Dict[str, torch.Tensor]]:
    """Adapter weights of a ``CrossAttentionAdapter.save_pretrained`` directory, canonical names."""
    sd = _safetensors(path)
    return None if sd is None else {AD + k: v for k, v in sd.items()}


def load_embedder_dir(path: str) -> Optional[Dict[str, torch.Tensor]]:
    """LlamaModel weights (with or without the ``model.`` prefix of a causal-LM checkpoint; ``lm_head`` is unused)."""
    sd = _safetensors(path)
    if sd is None:
        return None
    return {EMB + (k[len("model."):] if k.startswith("model.") else k): v for k, v in sd.items() if not k.startswith("lm_head.")}


def _load_tokenizer(path: str, acfg: AdapterConfig):
    if os.path.isdir(path) and any(os.path.exists(os.path.join(path, f)) for f in ("tokenizer.json", "tokenizer_config.json")):
        from transformers import AutoTokenizer   # host-side text -> ids only
        return AutoTokenizer.from_pretrained(path, pad_token="<|finetune_right_pad_id|>", model_max_length=acfg.max_text,
                                             padding_side="right")
    return SyntheticTokenizer(acfg.vocab_size, 128000 if acfg.vocab_size > 128001 else 0, 128001 if acfg.vocab_size > 128001 else 1,
                              acfg.pad_token_id, model_max_length=acfg.max_text)


class CaptionEmbedder:
    """``model.embedding_model``: the caption encoder's configuration (its weights live in the engine's adapter arena)."""

    def __init__(self, acfg: AdapterConfig):
        self.config = acfg


class CrossAttentionAdapter:
    """``model.adapter``: configuration, cross-layer indices and the learned dummy image (fp32 on the device)."""

    def __init__(self, cfg, acfg: AdapterConfig, arena: torch.Tensor):
        self.config = acfg
        self.layers = cross_layers(cfg, acfg)
        info = next(i for i in adapter_weight_table(cfg, acfg) if i.name.decode() == "ad.dummy")
        S = cfg.vision_config.image_size
        self.dummy_input = arena[info.offset // 2: info.offset // 2 + 3 * S * S].view(3, S, S).float()

    def dummy_pixels(self) -> torch.Tensor:
        """The tower input without an image (reference modeling_adapter.py:489-491): ``dummy_input.clamp(-1, 1)``."""
        return self.dummy_input.clamp(-1, 1)[None]


def load(model, processor, adapter_name_or_path: Optional[str] = None, embedding_model: str = "meta-llama/Llama-3.2-1B", *,
         random_init_weights: Optional[bool] = None, seed: int = 0, state_dict: Optional[Dict[str, torch.Tensor]] = None,
         config: Optional[AdapterConfig] = None, device_init: bool = False):
    """Returns ``(model, AdapterProcessor)``; afterwards ``has_adapter(model)`` is True and ``generate`` / the pipeline accept
    captions (``adapter_input_ids`` / ``adapter_attention_mask``). ``state_dict`` (canonical names, see ``canonical_shapes``)
    replaces every file source. ``device_init=True``: synthetic weights generated on the device (benches)."""
    cfg = model.config
    acfg = replace(config) if config is not None else None   # the tokenizer's pad id is written into a copy
    if acfg is None:
        emb_dir = isinstance(embedding_model, str) and os.path.isdir(embedding_model)
        acfg = (_config_from_json(embedding_model, embedding_model)
                if emb_dir and os.path.exists(os.path.join(embedding_model, "config.json")) else adapter_preset(embedding_model))
    if acfg.head_dim != 64:
        raise EngineError(f"the caption embedder must have head_dim 64 (got {acfg.head_dim})")
    device = model.engine.device
    if state_dict is None and device_init:
        arena = random_arena_device(cfg, acfg, device, seed=seed)
    else:
        sd = state_dict
        if sd is None:
            ad = load_adapter_dir(adapter_name_or_path or os.path.join(model.name_or_path or "", "adapter"))
            emb = load_embedder_dir(embedding_model)
            if ad is None or emb is None:
                if random_init_weights is False:
                    raise FileNotFoundError("adapter or embedder weights not found (offline) and random init disabled")
                if (ad is None) != (emb is None) and random_init_weights is not True:
                    # trained adapter weights on a random caption embedder (or the reverse) give meaningless output
                    raise FileNotFoundError(
                        f"found {'adapter' if ad is not None else 'embedder'} weights but no "
                        f"{'embedder (embedding_model=' + repr(embedding_model) + ' is not a local directory)' if ad is not None else 'adapter'}"
                        " weights; pass both, or random_init_weights=True to fill the missing part with random weights")
                sd = random_init(cfg, acfg, seed=seed)
            else:
                sd = {}
            sd.update(ad or {})
            sd.update(emb or {})
        arena = pack_arena(cfg, acfg, sd)
        del sd
    model.engine.adapter_attach(to_c_adapter_config(acfg), arena)
    model.adapter = CrossAttentionAdapter(cfg, acfg, model.engine.adapter_arena)
    model.embedding_model = CaptionEmbedder(acfg)
    model._img_cache = None
    model._slot_tokens = []
    tokenizer = _load_tokenizer(embedding_model, acfg)
    acfg.pad_token_id = tokenizer.pad_token_id
    return model, AdapterProcessor(processor=processor, tokenizer=tokenizer)


__all__ = ["load", "AdapterConfig", "adapter_preset", "adapter_weight_table", "canonical_shapes", "random_init", "pack_arena",
           "to_c_adapter_config", "load_adapter_dir", "load_embedder_dir", "CrossAttentionAdapter", "CaptionEmbedder"]
