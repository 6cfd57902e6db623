"""
Plain configuration objects for the CUDA engine (no HF dependency).

Mirrors the attribute names the reference's callers read:
  * ``config.image_token_id`` / ``config.patch_token_id`` and ``config.pooling_mode``
    (reference: detikzify/model/v1/configuration_detikzify.py:3-13),
  * ``config.text_config.eos_token_id`` (read at detikzify/infer/generate.py:221 for every
    model although the v1 config is flat -> ``text_config`` is an alias to ``self``),
  * ``config.vision_config.image_size`` (examples/refine.py:174),
  * ``config.num_patches`` / ``concat_patches`` / ``feature_layer`` / ``mm_hidden_size``
    (detikzify/model/v1/modeling_detikzify.py:98-107).

Decoder dims of the named checkpoints are the public DeepSeek-Coder, TinyLlama-1.1B and CodeLlama-7b base configs
(SURVEY.md Appendix A); they are config input, not reference source. The tl-1.1b / cl-7b vocab sizes follow the v1
loader's rule (add ``<pad>``, resize to a multiple of 8: reference v1/__init__.py:43-44) and are unverified against
the hub; a checkpoint directory's ``config.json`` always wins.
"""
from __future__ import annotations

from dataclasses import dataclass, field, asdict
from typing import Any, Dict


@dataclass
class VisionConfig:
    hidden_size: int = 1152
    intermediate_size: int = 4304
    num_hidden_layers: int = 27
    num_attention_heads: int = 16
    image_size: int = 384
    patch_size: int = 14
    num_channels: int = 3
    layer_norm_eps: float = 1e-6
    hidden_act: str = "gelu_pytorch_tanh"  # or "gelu" (exact erf); SURVEY §8c open parameter

    @property
    def head_dim(self) -> int:
        return self.hidden_size // self.num_attention_heads

    @property
    def num_positions(self) -> int:
        return (self.image_size // self.patch_size) ** 2

    def to_dict(self) -> Dict[str, Any]:
        return asdict(self)


@dataclass
class DetikzifyConfig:
    # decoder (LLaMA)
    hidden_size: int = 2048
    intermediate_size: int = 5504
    num_hidden_layers: int = 24
    num_attention_heads: int = 16
    num_key_value_heads: int = 16
    head_dim: int = 128
    vocab_size: int = 32256
    max_position_embeddings: int = 16384
    rms_norm_eps: float = 1e-6
    rope_theta: float = 100000.0
    rope_factor: float = 4.0  # linear scaling (DeepSeek-Coder)
    rope_type: str = "linear"  # "llama3" for the LLaMA-3.x decoders of the v2 checkpoints
    rope_low_freq_factor: float = 1.0
    rope_high_freq_factor: float = 4.0
    rope_original_max_position: int = 8192
    model_max_length: int = 2048  # v1 tokenizer limit, detikzify/model/v1/__init__.py:28
    # special tokens (v1: patch token := tokenizer BOS, v1/__init__.py:49)
    bos_token_id: int = 32013
    eos_token_id: int = 32014
    pad_token_id: int = 32018
    patch_token_id: int = 32013
    # glue
    concat_patches: int = 3
    feature_layer: int = -1
    projector_bias: bool = True  # v1: nn.Linear with bias (v1/modeling_detikzify.py:82)
    model_type: str = "detikzify"
    name_or_path: str = ""
    vision_config: VisionConfig = field(default_factory=VisionConfig)

    # --- attribute aliases the reference's callers use -------------------------------------
    @property
    def image_token_id(self) -> int:
        return self.patch_token_id

    @property
    def pooling_mode(self) -> str:
        # v1 configs pool with "cos" (v1/configuration_detikzify.py:11-13); the v2 config has no such attribute and
        # ImageSim.from_detikzify then defaults to "emd" (evaluate/imagesim.py:64)
        return "cos" if self.projector_bias else "emd"

    @property
    def text_config(self) -> "DetikzifyConfig":
        return self

    @property
    def num_patches(self) -> int:
        """image tokens fed to the decoder (243 @384px)."""
        return self.vision_config.num_positions // self.concat_patches

    @property
    def mm_hidden_size(self) -> int:
        return self.vision_config.hidden_size * self.concat_patches

    @property
    def use_mm_proj(self) -> bool:
        return True

    def to_dict(self) -> Dict[str, Any]:
        d = asdict(self)
        d["image_token_id"] = self.image_token_id
        d["num_patches"] = self.num_patches
        return d


def preset(name: str) -> DetikzifyConfig:
    """Named checkpoint shapes. ``tiny``/``tiny2`` are test shapes (ragged on purpose:
    16 patches -> 5 image tokens drops the first patch, K=176 is not a multiple of 32)."""
    key = name.split("/")[-1].lower()
    if key in ("detikzify-ds-1.3b", "ds-1.3b"):
        return DetikzifyConfig(name_or_path=name)
    if key in ("detikzify-ds-7b", "ds-7b"):
        return DetikzifyConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=32,
                               num_attention_heads=32, num_key_value_heads=32, name_or_path=name)
    if key in ("detikzify-ds-7b-2l", "ds-7b-2l"):
        # parity-test shape: every ds-7b matrix shape (H 4096, I 11008, 32 heads, V 32256) with two decoder layers and a
        # small vision tower, so that the fp32 CPU oracle fits in memory and finishes in seconds
        return DetikzifyConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=2,
                               num_attention_heads=32, num_key_value_heads=32, name_or_path=name,
                               vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                                          num_attention_heads=2, image_size=56, patch_size=14))
    if key in ("detikzify-tl-1.1b", "tl-1.1b"):
        # TinyLlama-1.1B: head_dim 64, GQA 32/4; V = 32000 + <pad> -> 32008; patch token = BOS (v1/__init__.py:49)
        return DetikzifyConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=22, num_attention_heads=32,
                               num_key_value_heads=4, head_dim=64, vocab_size=32008, max_position_embeddings=2048,
                               rms_norm_eps=1e-5, rope_theta=10000.0, rope_factor=1.0,
                               bos_token_id=1, eos_token_id=2, pad_token_id=32000, patch_token_id=1, name_or_path=name)
    if key in ("detikzify-cl-7b", "cl-7b", "detikzify-cl-7b-2l", "cl-7b-2l"):
        # CodeLlama-7b: MHA 32 x 128, theta 1e6; V = 32016 + <pad> -> 32024. "-2l": parity-test shape (two decoder layers,
        # small tower) with every cl-7b matrix shape
        two = key.endswith("-2l")
        return DetikzifyConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=2 if two else 32,
                               num_attention_heads=32, num_key_value_heads=32, vocab_size=32024, max_position_embeddings=16384,
                               rms_norm_eps=1e-5, rope_theta=1000000.0, rope_factor=1.0,
                               bos_token_id=1, eos_token_id=2, pad_token_id=32016, patch_token_id=1, name_or_path=name,
                               vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                                          num_attention_heads=2, image_size=56, patch_size=14)
                               if two else VisionConfig())
    if key == "tiny-tl":   # TinyLlama wiring at a CPU-test size: head_dim 64, GQA 8/1, V = 520 (8 mod 16), no RoPE scaling
        return DetikzifyConfig(
            hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=8,
            num_key_value_heads=1, head_dim=64, vocab_size=520, model_max_length=128, max_position_embeddings=2048,
            rms_norm_eps=1e-5, rope_theta=10000.0, rope_factor=1.0,
            bos_token_id=500, eos_token_id=501, pad_token_id=502, patch_token_id=500,
            name_or_path=name,
            vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                       num_attention_heads=2, image_size=56, patch_size=14))
    if key in ("detikzify-v2-8b", "detikzify-v2.5-8b", "v2-8b", "v2.5-8b"):
        # v2 / v2.5 (reference detikzify/model/configuration_detikzify.py:31-58,83-120, modeling_detikzify.py:62-86): SigLIP
        # so400m at 420 px -> 900 patches -> 300 image tokens, bias-free connector, LLaMA-3.1-8B decoder (GQA 32/8,
        # V 128256, llama3 RoPE scaling; public base config, not in the reference tree), image token 128005
        return DetikzifyConfig(hidden_size=4096, intermediate_size=14336, num_hidden_layers=32, num_attention_heads=32,
                               num_key_value_heads=8, vocab_size=128256, max_position_embeddings=131072, rms_norm_eps=1e-5,
                               rope_theta=500000.0, rope_factor=8.0, rope_type="llama3", rope_low_freq_factor=1.0,
                               rope_high_freq_factor=4.0, rope_original_max_position=8192,
                               bos_token_id=128000, eos_token_id=128001, pad_token_id=128004, patch_token_id=128005,
                               projector_bias=False, name_or_path=name, vision_config=VisionConfig(image_size=420))
    if key in ("detikzify-v2-8b-2l", "v2-8b-2l"):   # parity-test shape: every v2-8b matrix shape, two decoder layers, small tower
        return DetikzifyConfig(hidden_size=4096, intermediate_size=14336, num_hidden_layers=2, num_attention_heads=32,
                               num_key_value_heads=8, vocab_size=128256, max_position_embeddings=131072, rms_norm_eps=1e-5,
                               rope_theta=500000.0, rope_factor=8.0, rope_type="llama3", rope_low_freq_factor=1.0,
                               rope_high_freq_factor=4.0, rope_original_max_position=8192,
                               bos_token_id=128000, eos_token_id=128001, pad_token_id=128004, patch_token_id=128005,
                               projector_bias=False, name_or_path=name,
                               vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                                          num_attention_heads=2, image_size=84, patch_size=14))
    if key == "tiny-v2":   # v2 wiring at a CPU-test size: GQA 4/2, llama3 RoPE (short original context so all three
        # frequency bands occur), bias-free connector, 6x6 patches -> 12 image tokens
        return DetikzifyConfig(
            hidden_size=512, intermediate_size=1376, num_hidden_layers=2, num_attention_heads=4,
            num_key_value_heads=2, vocab_size=640, model_max_length=128, rms_norm_eps=1e-5,
            rope_theta=500000.0, rope_factor=8.0, rope_type="llama3", rope_low_freq_factor=1.0, rope_high_freq_factor=4.0,
            rope_original_max_position=64,
            bos_token_id=600, eos_token_id=601, pad_token_id=604, patch_token_id=605, projector_bias=False,
            name_or_path=name,
            vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                       num_attention_heads=2, image_size=84, patch_size=14))
    if key == "tiny":
        return DetikzifyConfig(
            hidden_size=256, intermediate_size=688, num_hidden_layers=2, num_attention_heads=2,
            num_key_value_heads=2, vocab_size=512, model_max_length=96,
            bos_token_id=500, eos_token_id=501, pad_token_id=502, patch_token_id=500,
            name_or_path=name,
            vision_config=VisionConfig(hidden_size=144, intermediate_size=176, num_hidden_layers=2,
                                       num_attention_heads=2, image_size=56, patch_size=14))
    if key == "tiny2":  # more layers/heads, 3x3 patches
        return DetikzifyConfig(
            hidden_size=384, intermediate_size=1040, num_hidden_layers=3, num_attention_heads=3,
            num_key_value_heads=3, vocab_size=1000, model_max_length=160,
            bos_token_id=990, eos_token_id=991, pad_token_id=992, patch_token_id=990,
            name_or_path=name,
            vision_config=VisionConfig(hidden_size=216, intermediate_size=400, num_hidden_layers=3,
                                       num_attention_heads=3, image_size=126, patch_size=14))
    raise KeyError(f"unknown model preset {name!r}")


def config_from_dict(d: Dict[str, Any], name: str = "") -> DetikzifyConfig:
    """``config.json`` of a checkpoint directory -> DetikzifyConfig. Two layouts exist: v1 checkpoints carry a flat LLaMA
    config plus the fields ``initialize_vision_modules`` wrote (reference v1/configuration_detikzify.py:3-13,
    v1/modeling_detikzify.py:98-107: patch_token_id, concat_patches, num_patches, vision_tower ...; the tower itself is a timm
    so400m/14@384 SigLIP and is NOT described in the file), v2 / v2.5 nest ``text_config`` / ``vision_config`` and name the
    image token ``image_token_id`` (reference configuration_detikzify.py:83-120)."""
    def rope(t: Dict[str, Any]) -> Dict[str, Any]:
        rs = t.get("rope_scaling") or t.get("rope_parameters") or {}
        kind = rs.get("rope_type", rs.get("type", "default"))
        out = dict(rope_theta=float(t.get("rope_theta", rs.get("rope_theta", 10000.0))), rope_factor=float(rs.get("factor", 1.0)))
        if kind == "llama3":
            out.update(rope_type="llama3", rope_low_freq_factor=float(rs.get("low_freq_factor", 1.0)),
                       rope_high_freq_factor=float(rs.get("high_freq_factor", 4.0)),
                       rope_original_max_position=int(rs.get("original_max_position_embeddings", 8192)))
        elif kind not in ("default", "linear"):
            raise ValueError(f"unsupported rope scaling {kind!r}")
        return out

    v2 = "text_config" in d
    t = d["text_config"] if v2 else d
    heads = int(t["num_attention_heads"])
    head_dim = int(t.get("head_dim") or t["hidden_size"] // heads)
    common = dict(
        hidden_size=int(t["hidden_size"]), intermediate_size=int(t["intermediate_size"]), num_hidden_layers=int(t["num_hidden_layers"]),
        num_attention_heads=heads, num_key_value_heads=int(t.get("num_key_value_heads", heads)), head_dim=head_dim,
        vocab_size=int(t["vocab_size"]), max_position_embeddings=int(t.get("max_position_embeddings", 2048)),
        rms_norm_eps=float(t.get("rms_norm_eps", 1e-6)), bos_token_id=int(t.get("bos_token_id") or 0),
        eos_token_id=int(t["eos_token_id"] if not isinstance(t.get("eos_token_id"), list) else t["eos_token_id"][0]),
        pad_token_id=int(t.get("pad_token_id") if t.get("pad_token_id") is not None else d.get("pad_token_id", 0)),
        name_or_path=name, **rope(t))
    if v2:
        vc = d.get("vision_config") or {}
        vision = VisionConfig(**{k: vc[k] for k in ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads",
                                                   "image_size", "patch_size", "num_channels", "layer_norm_eps", "hidden_act") if k in vc})
        if "image_size" not in vc:
            vision.image_size = 420
        return DetikzifyConfig(patch_token_id=int(d.get("image_token_id", 128005)), concat_patches=int(d.get("concat_factor", 3)),
                               projector_bias=False, vision_config=vision, **common)
    return DetikzifyConfig(patch_token_id=int(d["patch_token_id"]), concat_patches=int(d.get("concat_patches", 3)),
                           projector_bias=True, vision_config=VisionConfig(), **common)
