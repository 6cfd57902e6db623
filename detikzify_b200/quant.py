"""
FP8 (e4m3) weight-only quantization of the decoder-layer matrices.

Each output row ``r`` of a matrix ``W`` is stored as ``W~[r] = q[r] * 2^k_r``: ``k_r`` is the smallest integer with
``max |W[r]| <= 448 * 2^k_r`` (at least -117, so that every nonzero value stays a bf16 normal; 0 for a row of zeros) and
``q[r] = e4m3fn(W[r] / 2^k_r)`` rounded to nearest even. Because the scale is a power of two, ``W~`` is exactly
representable in bf16: the quantized model is the bf16 model with ``W~`` in place of ``W``, on every path. The batch-1
persistent decode kernel and the layer GEMMs of batched decode steps with 4 <= B < 64 rows stream ``q`` and ``k_r`` instead
of the bf16 values (engine option ``decode_fp8``).
"""
from __future__ import annotations

import re

import torch

E4M3_MAX = 448.0
K_MIN = -117
# the decoder-layer matrices of the weight arena that are quantized (embeddings, norms, lm_head, projector and ViT stay bf16)
LAYER_MATRIX = re.compile(r"dec\.L\d+\.(wqkv|wo|wgu|wd)$")


def fp8_row_exponents(w: torch.Tensor) -> torch.Tensor:
    """k_r (int32 [rows]) of a 2-D matrix: the smallest k with max |w[r]| <= 448 * 2^k, at least -117; 0 for a zero row."""
    amax = w.float().abs().amax(dim=1)
    f, e = torch.frexp(amax)          # amax = f * 2^e exactly, f in [0.5, 1); 448 = 0.875 * 2^9
    k = e - 9 + (f > 0.875).to(e.dtype)
    return torch.where(amax > 0, k.clamp(min=K_MIN), torch.zeros_like(k))


def quantize_fp8_rows(w: torch.Tensor) -> torch.Tensor:
    """W~ (bf16, same shape and device) of a 2-D matrix under the per-row power-of-two e4m3 rule. Raises ValueError on
    non-finite weights. Quantizing W~ again returns it bit for bit."""
    if w.dim() != 2:
        raise ValueError(f"expected a 2-D matrix, got shape {tuple(w.shape)}")
    x = w.float()
    if not torch.isfinite(x).all():
        raise ValueError("fp8 quantization: the matrix holds inf or NaN")
    scale = ((fp8_row_exponents(x).to(torch.int32) + 127) << 23).view(torch.float32)[:, None]   # 2^k_r from its bits
    q = (x / scale).to(torch.float8_e4m3fn)          # |x / 2^k_r| <= 448: round to nearest even, no saturation needed
    out = (q.float() * scale).to(torch.bfloat16)     # exact: q has 4 significant bits and q * 2^k_r is a bf16 normal
    if not torch.isfinite(out).all():                # only a row whose max rounds up to 2^128
        raise ValueError("fp8 quantization: a row's maximum rounds past the bf16 range")
    return out


def quantize_arena_fp8(arena: torch.Tensor, table) -> None:
    """Replace, in place, every decoder-layer matrix of a packed bf16 weight arena (host or device) by its W~.
    ``table``: the arena's weight table (``engine.weight_table``)."""
    for info in table:
        name = info.name.decode()
        if LAYER_MATRIX.match(name):
            n = info.rows * info.cols
            view = arena[info.offset // 2: info.offset // 2 + n].view(info.rows, info.cols)
            try:
                view.copy_(quantize_fp8_rows(view))
            except ValueError as e:
                raise ValueError(f"{name}: {e}") from None
