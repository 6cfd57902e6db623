"""
``detikzify_b200.model.load`` — drop-in for ``detikzify.model.load``
(reference detikzify/model/__init__.py:28-61 and v1 loader detikzify/model/v1/__init__.py:24-56).

    model, processor = load("nllg/detikzify-ds-1.3b", device_map=0, torch_dtype=torch.bfloat16)

Accepted kwargs are the ones the reference's callers pass (examples/infer.py:32-37,
examples/eval.py:110-115, webui/webui.py:76-81): ``device_map`` ("auto" | int | "cuda:N"),
``torch_dtype`` (torch dtype or string, bf16/fp16 both map to the engine's bf16 storage),
``attn_implementation`` (ignored: the engine has its own attention kernels).
Weights come from ``<path>/*.safetensors`` when ``model_name_or_path`` is a local directory;
otherwise — there is no network in the build environment — a deterministic random init of the named
checkpoint shape is used (``random_init=True`` / ``seed=``), which is what the benches measure.
"""
from __future__ import annotations

import os
from glob import glob
from typing import Dict, Optional

import torch

from .configuration import DetikzifyConfig, VisionConfig, config_from_dict, preset
from .modeling import DetikzifyForCausalLM
from .processing import DetikzifyImageProcessor, DetikzifyProcessor, SyntheticTokenizer
from .weights import canonical_shapes, convert_timm_vision, convert_v2_state_dict, random_init

# the v1 checkpoints the reference lists (reference detikzify/model/v1/__init__.py:10-15), each with a shape preset
v1_models = [
    "nllg/detikzify-ds-1.3b",
    "nllg/detikzify-ds-7b",
    "nllg/detikzify-tl-1.1b",
    "nllg/detikzify-cl-7b",
]


def _device_index(device_map) -> int:
    if device_map is None or device_map == "auto":
        return int(os.environ.get("LOCAL_RANK", torch.cuda.current_device() if torch.cuda.is_available() else 0))
    if isinstance(device_map, int):
        return device_map
    if isinstance(device_map, torch.device):
        return device_map.index or 0
    if isinstance(device_map, str):
        return torch.device(device_map).index or 0
    if isinstance(device_map, dict):
        return _device_index(next(iter(device_map.values())))
    raise ValueError(f"unsupported device_map {device_map!r}")


def _load_safetensors_dir(path: str, vision_tower: Optional[str] = None) -> Dict[str, torch.Tensor]:
    """Canonical state dict of a checkpoint directory. v2 / v2.5 names are mapped onto the canonical ones; v1 checkpoints do
    NOT contain the vision tower (the reference wraps the timm model in a list so that it stays out of the state dict and
    pulls the pretrained timm weights instead, v1/modeling_detikzify.py:49-57,84-96) — pass ``vision_tower`` (a timm
    ``vit_so400m_patch14_siglip_384`` safetensors file or directory) to supply it."""
    from safetensors.torch import load_file
    sd: Dict[str, torch.Tensor] = {}
    for f in sorted(glob(os.path.join(path, "*.safetensors"))):
        sd.update(load_file(f))
    if any(k.startswith("model.text_model.") or k.startswith("model.connector.") for k in sd):
        sd = convert_v2_state_dict(sd)
    if vision_tower is not None:
        files = sorted(glob(os.path.join(vision_tower, "*.safetensors"))) if os.path.isdir(vision_tower) else [vision_tower]
        tower: Dict[str, torch.Tensor] = {}
        for f in files:
            tower.update(load_file(f))
        sd.update(convert_timm_vision(tower))
    elif any(k.startswith("blocks.") or k.startswith("patch_embed.") for k in sd):
        sd.update(convert_timm_vision(sd))
    if not any(k.startswith("model.vision_model.") for k in sd):
        raise FileNotFoundError(
            f"{path}: the checkpoint holds no vision tower (v1 checkpoints never do); pass vision_tower=<timm "
            "vit_so400m_patch14_siglip_384 safetensors> to load()")
    return sd


def _load_tokenizer(path: str, cfg: DetikzifyConfig):
    """The checkpoint's own tokenizer when its files are present (v1 settings: reference v1/__init__.py:24-33); None otherwise."""
    if not any(os.path.exists(os.path.join(path, f)) for f in ("tokenizer.json", "tokenizer.model", "tokenizer_config.json")):
        return None
    from transformers import AutoTokenizer   # host-side text <-> ids only, not on the GPU path
    tok = AutoTokenizer.from_pretrained(path, model_max_length=cfg.model_max_length, add_bos_token=False, add_eos_token=True,
                                        pad_token="<pad>", padding_side="right", legacy=False)
    return tok


def build_processor(cfg: DetikzifyConfig, tokenizer=None) -> DetikzifyProcessor:
    tokenizer = tokenizer or SyntheticTokenizer(cfg.vocab_size, cfg.bos_token_id, cfg.eos_token_id,
                                                cfg.pad_token_id, model_max_length=cfg.model_max_length)
    return DetikzifyProcessor(
        image_processor=DetikzifyImageProcessor(size=cfg.vision_config.image_size),
        tokenizer=tokenizer,
        image_seq_len=cfg.num_patches,
        image_token=tokenizer.convert_ids_to_tokens(cfg.patch_token_id))


def load(model_name_or_path, modality_projector: Optional[str] = None, is_v1: bool = False, *,
         random_init_weights: Optional[bool] = None, seed: int = 0, state_dict: Optional[Dict[str, torch.Tensor]] = None,
         config: Optional[DetikzifyConfig] = None, max_seqs: int = 2, max_batch: int = 1, broadcast: bool = False,
         prefix_slots: Optional[int] = None, device_init: bool = False, vision_tower: Optional[str] = None,
         quantize: Optional[str] = None, **kwargs):
    """Returns ``(model, processor)``.

    ``max_seqs`` KV slots are preallocated (0.40 GB each for ds-1.3b at 2k context); ``generate()`` keeps a prefix cache
    over ``prefix_slots`` of them (default ``max_seqs - max_batch``, at least 1) — for MCTS use e.g. ``max_seqs=8``;
    ``generate_batch`` / ``sample_batch`` need ``max_batch`` (and as many free slots) >= the number of sequences.

    ``device_init=True`` (benches): synthetic weights are generated directly on the device (``random_arena_device``)
    instead of on the host — seconds instead of minutes for ds-7b; the values differ from the CPU-seeded init.

    ``broadcast=True`` (multi-GPU, one process per GPU): only rank 0 materialises the weights; the
    packed arena is sent with ONE ``torch.distributed.broadcast`` over NCCL (SURVEY.md §8e).

    ``quantize="fp8"``: weight-only e4m3 quantization of the decoder-layer matrices (q/k/v/o, gate/up, down) with one
    power-of-two scale per output row (``detikzify_b200.quant``). The arena holds the dequantized values, so every path
    computes the same quantized model, and batch-1 decode and batched decode steps of 4 <= B < 64 rows (rollouts,
    ``generate_batch``) stream the layer matrices as e4m3 (about half the bytes) with bit-identical logits.
    Embeddings, norms, lm_head, projector, vision tower and KV cache stay bf16. ``None`` (default) keeps the weights as
    they are, and batch-1 decode streams them as lossless 13-bit packed tiles (engine option ``decode_pack``: the same
    logits as bf16 tiles, about 17 % fewer bytes per token).
    """
    from ..engine import pack_arena, to_c_config, weight_table
    from ..quant import quantize_arena_fp8
    from .. import _lib
    import ctypes as C

    if quantize not in (None, "fp8"):
        raise ValueError(f"quantize must be None or 'fp8', got {quantize!r}")

    is_dir = isinstance(model_name_or_path, str) and os.path.isdir(model_name_or_path)
    cfg = config
    if cfg is None and is_dir and os.path.exists(os.path.join(model_name_or_path, "config.json")):
        import json
        with open(os.path.join(model_name_or_path, "config.json")) as f:
            cfg = config_from_dict(json.load(f), name=model_name_or_path)
    if cfg is None:
        cfg = preset(model_name_or_path)
    device = _device_index(kwargs.pop("device_map", None))
    dtype = kwargs.pop("torch_dtype", kwargs.pop("dtype", torch.bfloat16))
    if isinstance(dtype, str):
        dtype = getattr(torch, dtype)
    kwargs.pop("attn_implementation", None)

    rank0 = True
    if broadcast:
        import torch.distributed as dist
        rank0 = dist.get_rank() == 0
    arena = None
    if rank0 and device_init and state_dict is None:
        from ..engine import random_arena_device
        arena = random_arena_device(cfg, device, seed=seed)
    elif rank0:
        sd = state_dict
        if sd is None and isinstance(model_name_or_path, str) and os.path.isdir(model_name_or_path) \
                and glob(os.path.join(model_name_or_path, "*.safetensors")):
            sd = _load_safetensors_dir(model_name_or_path, vision_tower)
        if sd is None:
            if random_init_weights is False:
                raise FileNotFoundError(f"no weights found for {model_name_or_path!r} (offline) and random init disabled")
            sd = random_init(cfg, seed=seed)
        if modality_projector is not None:
            from safetensors.torch import load_file
            try:
                proj = torch.load(modality_projector, map_location="cpu")
            except Exception:
                proj = load_file(modality_projector)
            for k, v in proj.items():
                sd["model.mm_projector." + k.split(".")[-1]] = v
        arena = pack_arena(cfg, sd)
        del sd
    if rank0 and quantize == "fp8":   # before the broadcast: every rank holds the same bytes
        quantize_arena_fp8(arena, weight_table(to_c_config(cfg)))
    if broadcast:
        import torch.distributed as dist
        lib = _lib.load_library()
        nbytes = lib.dtk_arena_bytes(C.byref(to_c_config(cfg)))
        dev = torch.device(f"cuda:{device}")
        arena = arena.to(dev) if rank0 else torch.empty(nbytes // 2, dtype=torch.bfloat16, device=dev)
        dist.broadcast(arena, src=0)  # the single collective of the whole path

    model = DetikzifyForCausalLM(cfg, arena, device=device, dtype=dtype, max_seqs=max_seqs, max_batch=max_batch,
                                 prefix_slots=prefix_slots, decode_pack=quantize != "fp8")
    if quantize == "fp8":
        model.engine.set_option("decode_fp8", 1)
    tokenizer = _load_tokenizer(model_name_or_path, cfg) if is_dir else None
    return model, build_processor(cfg, tokenizer)


__all__ = ["load", "v1_models", "DetikzifyConfig", "VisionConfig", "DetikzifyForCausalLM", "DetikzifyProcessor",
           "DetikzifyImageProcessor", "SyntheticTokenizer", "preset", "build_processor"]
