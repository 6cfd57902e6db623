"""
One decoder step restated in float64, on the engine's own weights and KV cache, rounded where a given decode path rounds.

``restate_step`` takes B rows (position, token id), a reader of each row's cached bf16 keys / values and a ``path``:

  * ``None``: no rounding point at all (the CPU self-test runs it on its own fp64 cache against the HF model);
  * ``"persistent"`` (the batch-1 persistent kernel): fp32-grade matrix inputs (the kernel splits them into bf16 hi + lo);
    the current token's key / value enter attention as the bf16 cache row the qkv phase writes (it publishes the rounded
    values, so the step reads what the cache holds);
  * ``"per_op"`` (``decode_impl`` 0, fp32 GEMVs): the current key / value read back from the bf16 cache;
  * ``"batched"`` (B >= 4, tensor-core GEMMs): the RMSNorm outputs, the attention output and the SwiGLU output are bf16 GEMM
    operands, the current key / value come from the bf16 cache, q and the residual stream stay fp32;
  * ``"cascade"``: as ``"batched"``, and the keys below ``cas_len`` are reduced with a bf16 q (the prefix kernel's operand).
    Its bf16 P is not restated: the error model carries it.

Weights come from the arena through the C ABI's weight table (fused wqkv, gate/up interleaved row by row in wgu). RoPE uses
the engine's table: fp32 inv_freq from libm ``powf``, llama3 band scaling in fp32, fp32 angle = pos * inv_freq, cos / sin of
that angle rounded to fp32.

Error model (``Noise``). The same step is run again with every rounding of the kernel replaced by an explicit random error:
  * a length-K fp32 dot product: N(0, s^2) with s = sqrt(K u_acc^2 + u_in^2) * sqrt(sum_j (w_j x_j)^2), u_acc = 2^-23 (twice
    the unit roundoff: tensor-core accumulation does not round to nearest), u_in = 2^-18 / sqrt(3) for the persistent
    kernel's hi + lo operands (the lo part is itself rounded to bf16), 0 elsewhere;
  * an elementwise fp32 result (RoPE, residual adds, SiLU * up with ``__expf``, RMSNorm with ``rsqrtf``, softmax weights with
    ``exp2f``): relative N(0, (4 u)^2), u = 2^-24;
  * a bf16 rounding point: the error is added *before* rounding, so rounding-boundary flips occur as in the kernel;
  * cascade: each prefix softmax weight carries a relative uniform error of half a bf16 ulp (its bf16 P).
The spread of the logits between that run and the exact restatement is the logit noise scale of the path at this step.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Callable, Dict, Optional, Sequence

import torch

U = 2.0 ** -24
U_ACC = 2.0 ** -23
U_IN_PERSISTENT = 2.0 ** -18 / math.sqrt(3.0)
PATHS = (None, "persistent", "per_op", "batched", "cascade")


def bf16(x: torch.Tensor) -> torch.Tensor:
    """Round to the nearest bf16 (fp64 -> fp32 first: exact for every value a kernel's fp32 result can round from)."""
    return x.to(torch.float32).to(torch.bfloat16).to(x.dtype)


def bf16_ulp(x: torch.Tensor) -> torch.Tensor:
    """Spacing of bf16 values at |x| (normal range)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e - 7)


def rope_table(cfg, T: int) -> torch.Tensor:
    """[T, head_dim / 2, 2] (cos, sin) float32, computed as the engine computes it (fp32 host arithmetic, libm powf)."""
    import numpy as np
    powf = C.CDLL("libm.so.6").powf
    powf.restype, powf.argtypes = C.c_float, [C.c_float, C.c_float]
    f32 = np.float32
    hd = cfg.head_dim
    theta, factor = f32(cfg.rope_theta), f32(cfg.rope_factor)
    inv = np.empty(hd // 2, np.float32)
    for i in range(hd // 2):
        v = f32(1.0) / f32(powf(theta, f32(f32(2 * i) / f32(hd))))
        if cfg.rope_type == "llama3":
            lo, hi, old = f32(cfg.rope_low_freq_factor), f32(cfg.rope_high_freq_factor), f32(cfg.rope_original_max_position)
            low_wl, high_wl = old / lo, old / hi
            wl = f32(f32(2.0) * f32(3.14159265358979323846)) / v
            if wl > low_wl:
                v = v / factor
            elif not wl < high_wl:
                smooth = (old / wl - lo) / (hi - lo)
                v = (f32(1.0) - smooth) * v / factor + smooth * v
        else:
            v = v / factor
        inv[i] = v
    ang = np.arange(T, dtype=np.float32)[:, None] * inv[None, :]          # fp32 products
    cs = np.stack([np.vectorize(math.cos)(ang.astype(np.float64)), np.vectorize(math.sin)(ang.astype(np.float64))], -1)
    return torch.from_numpy(cs.astype(np.float32))


class Weights:
    """The decoder matrices of an arena (bf16, CPU or device) as float64 on ``device``, read through the weight table."""

    def __init__(self, cfg, arena: torch.Tensor, ccfg, device=None):
        from detikzify_b200.engine import weight_table
        self.cfg, self.arena = cfg, arena
        self.device = device if device is not None else arena.device
        self.info = {t.name.decode(): t for t in weight_table(ccfg)}
        self._cache: Dict[str, torch.Tensor] = {}
        self.rope = rope_table(cfg, ccfg.max_len + 1).to(self.device, torch.float64)   # + 1: the RoPE-shift control

    def __call__(self, name: str) -> torch.Tensor:
        if name in self._cache:
            return self._cache[name]
        t = self.info[name]
        w = self.arena[t.offset // 2: t.offset // 2 + t.rows * t.cols].view(t.rows, t.cols)
        w = w.to(self.device).to(torch.float64)
        if t.rows == 1 or name in ("dec.embed",):   # small or gathered: keep
            self._cache[name] = w
        return w


class Noise:
    """Random stand-in for the kernel's roundings (see the module docstring); ``None`` in place of a Noise = exact."""

    def __init__(self, seed: int, device, u_in: float = 0.0):
        self.g = torch.Generator(device=device).manual_seed(seed)
        self.u_in = u_in

    def _n(self, like):
        return torch.randn(like.shape, generator=self.g, device=like.device, dtype=like.dtype)

    def dot(self, y, x, w):
        """y = x @ w.T of length-K rows (x [B, K], w [N, K])."""
        K = x.shape[-1]
        s = math.sqrt(K * U_ACC ** 2 + self.u_in ** 2) * torch.sqrt((x * x) @ (w * w).T)
        return y + s * self._n(y)

    def elem(self, y, rel=4 * U):
        return y + rel * y.abs() * self._n(y)

    def uniform_rel(self, y, rel):
        return y * (1 + rel * (2 * torch.rand(y.shape, generator=self.g, device=y.device, dtype=y.dtype) - 1))


def _mm(x, w, nz, path_dot=True):
    y = x @ w.T
    return nz.dot(y, x, w) if (nz is not None and path_dot) else y


def _rms(x, g, eps, nz):
    r = torch.rsqrt((x * x).mean(-1, keepdim=True) + eps)
    y = x * r * g
    return nz.elem(y) if nz is not None else y


def _rope(t, cs):
    """rotate-half RoPE of t [..., hd] with cs [..., hd/2, 2]."""
    h = t.shape[-1] // 2
    a, b = t[..., :h], t[..., h:]
    c, s = cs[..., 0], cs[..., 1]
    return torch.cat([a * c - b * s, b * c + a * s], -1)


def restate_step(w: Weights, positions: Sequence[int], tokens: Sequence[int], kv: Callable, path: Optional[str] = None,
                 nz: Optional[Noise] = None, cas_len: int = 0, drop_key: Optional[Callable[[int], int]] = None,
                 rope_shift: int = 0, gqa_mod: bool = False, fp32_current: bool = False) -> dict:
    """One decode step of B rows. ``kv(b, layer, n)`` -> (K, V) float64 [kv_heads, n, hd]: row b's cached positions [0, n).

    Negative controls (perturbed restatements the comparison must reject): ``drop_key(pos)`` -> a cached position left out
    of the softmax; ``rope_shift`` rotates q and the new key as at pos + shift; ``gqa_mod`` routes query head h to kv head
    h % kv_heads; ``fp32_current`` uses the unrounded current key / value in attention.

    Returns ``logits`` [B, V] and, per layer, ``k`` / ``v`` [B, kv_heads, hd]: the new cache row before its bf16 rounding,
    with ``kv_eps`` [B, kv_heads, hd]: how far the kernel's own bf16 norm operand can move it (ambiguous roundings, batched
    paths only; 0 elsewhere)."""
    assert path in PATHS, path
    cfg = w.cfg
    dev = w.device
    B = len(positions)
    H, HD, nh, nkv = cfg.hidden_size, cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
    qd, kd, I, eps = nh * HD, nkv * HD, cfg.intermediate_size, cfg.rms_norm_eps
    rb = path in ("batched", "cascade")             # bf16 GEMM operands
    cur_fp32 = fp32_current
    rnd = (lambda t: bf16(t)) if path is not None else (lambda t: t)
    pos = torch.tensor(list(positions), device=dev)
    cs = w.rope[pos + rope_shift]                    # [B, hd/2, 2]
    x = w("dec.embed")[torch.tensor(list(tokens), device=dev)].clone()
    out = {"k": [], "v": [], "kv_eps": []}
    for l in range(cfg.num_hidden_layers):
        p = f"dec.L{l}."
        h = _rms(x, w(p + "norm1"), eps, nz)
        wqkv = w(p + "wqkv")
        amb = torch.zeros(B, kd, device=dev, dtype=torch.float64)
        if rb:
            # elements of the bf16 operand within 2^-18 (relative) of a rounding boundary may round either way in the kernel
            hb = bf16(h)
            near = ((h - hb).abs() - bf16_ulp(hb) / 2).abs() <= 2.0 ** -18 * h.abs()
            amb = (near * bf16_ulp(hb)) @ wqkv[qd:qd + kd].abs().T
            h = hb
        qkv = _mm(h, wqkv, nz)
        q = qkv[:, :qd].view(B, nh, HD)
        k = qkv[:, qd:qd + kd].view(B, nkv, HD)
        v = qkv[:, qd + kd:].view(B, nkv, HD)
        q, k = _rope(q, cs[:, None]), _rope(k, cs[:, None])
        if nz is not None:
            q, k = nz.elem(q), nz.elem(k)
        out["k"].append(k)
        out["v"].append(v)
        out["kv_eps"].append(amb.view(B, nkv, HD))
        kc, vc = (k, v) if cur_fp32 else (rnd(k), rnd(v))
        att = torch.empty(B, nh, HD, device=dev, dtype=torch.float64)
        for b in range(B):
            n = int(positions[b])
            K, V = kv(b, l, n)
            K = torch.cat([K, kc[b][:, None]], 1)
            V = torch.cat([V, vc[b][:, None]], 1)
            keep = torch.ones(n + 1, dtype=torch.bool, device=dev)
            if drop_key is not None:
                keep[drop_key(n)] = False
            heads = torch.arange(nh, device=dev)
            kvh = heads % nkv if gqa_mod else heads // (nh // nkv)
            Kh, Vh = K[kvh][:, keep], V[kvh][:, keep]             # [nh, T, hd]
            qb = q[b]
            s = torch.einsum("hd,htd->ht", qb, Kh) / math.sqrt(HD)
            if path == "cascade" and cas_len > 0:
                npre = int(keep[:cas_len].sum())
                s[:, :npre] = torch.einsum("hd,htd->ht", bf16(qb), Kh[:, :npre]) / math.sqrt(HD)
            if nz is not None:
                s = s + math.sqrt(HD) * U_ACC * torch.sqrt(torch.einsum("hd,htd->ht", qb * qb, Kh * Kh)) / math.sqrt(HD) \
                    * nz._n(s)
            pr = torch.softmax(s, -1)
            if nz is not None:
                pr = nz.elem(pr)
                if path == "cascade" and cas_len > 0:
                    pr[:, :npre] = nz.uniform_rel(pr[:, :npre], 2.0 ** -9)
            o = torch.einsum("ht,htd->hd", pr, Vh)
            if nz is not None:
                o = o + math.sqrt(Vh.shape[1]) * U_ACC * torch.sqrt(torch.einsum("ht,htd->hd", pr * pr, Vh * Vh)) * nz._n(o)
            att[b] = o / pr.sum(-1, keepdim=True)
        a = att.view(B, qd)
        if rb:
            a = bf16(nz.elem(a) if nz is not None else a)
        x = x + _mm(a, w(p + "wo"), nz)
        if nz is not None:
            x = nz.elem(x)
        h = _rms(x, w(p + "norm2"), eps, nz)
        if rb:
            h = bf16(h)
        wgu = w(p + "wgu")
        gu = _mm(h, wgu, nz)
        g, u = gu[:, 0::2], gu[:, 1::2]
        hh = g / (1 + torch.exp(-g)) * u
        if nz is not None:
            hh = nz.elem(hh)
        if rb:
            hh = bf16(hh)
        x = x + _mm(hh, w(p + "wd"), nz)
        if nz is not None:
            x = nz.elem(x)
    h = _rms(x, w("dec.norm"), eps, nz)
    if rb:
        h = bf16(h)
    out["logits"] = _mm(h, w("dec.lm_head"), nz)
    return out


def noise_for(path: Optional[str], seed: int, device) -> Noise:
    return Noise(seed, device, u_in=U_IN_PERSISTENT if path == "persistent" else 0.0)


def noise_scale(w: Weights, positions, tokens, kv, path, ref: dict, draws: int = 2, seed: int = 0, **kw) -> dict:
    """Per-row RMS (over the vocabulary) of the logit change the error model produces, and per (row, layer, kv head) the RMS
    change of the new cache row before rounding; the larger of ``draws`` runs."""
    sig = torch.zeros(len(positions), device=w.device, dtype=torch.float64)
    ksig = [torch.zeros(len(positions), w.cfg.num_key_value_heads, device=w.device, dtype=torch.float64)
            for _ in range(w.cfg.num_hidden_layers)]
    vsig = [t.clone() for t in ksig]
    for d in range(draws):
        r = restate_step(w, positions, tokens, kv, path, nz=noise_for(path, seed + d, w.device), **kw)
        sig = torch.maximum(sig, (r["logits"] - ref["logits"]).pow(2).mean(-1).sqrt())
        for l in range(w.cfg.num_hidden_layers):
            ksig[l] = torch.maximum(ksig[l], (r["k"][l] - ref["k"][l]).pow(2).mean(-1).sqrt())
            vsig[l] = torch.maximum(vsig[l], (r["v"][l] - ref["v"][l]).pow(2).mean(-1).sqrt())
    return {"logits": sig, "k": ksig, "v": vsig}
