"""
One prefill decoder layer restated in float64, from the engine's own input residual to that layer, on the engine's own
weights and KV cache, rounded where ``decoder_stack`` (engine.cu) rounds; and the head that follows the last layer.

``restate_layer`` takes the residual stream x [T, H] entering layer l at positions [start_pos, start_pos + T), a reader
``kv(l, n)`` of the layer's cached keys / values [0, n) and a ``path``:

  * ``None``: no rounding point at all. The reader holds the positions below ``start_pos`` only; the new rows enter
    attention as restated (the CPU self-test chains the layers on its own fp64 cache against the HF model);
  * ``"prefill"``: the rounding points of the prefill kernels, checked against the code:
      - RMSNorm in fp32, rounded to the bf16 GEMM operand ``p_xn`` (``rmsnorm_kernel``);
      - the qkv GEMM writes fp32 (``p_qkv``);
      - RoPE in fp32, q rounded to bf16 ``p_q``, k and v rounded to bf16 into the cache (``rope_kv_prefill_kernel``);
      - causal flash attention (``flash_attn_kernel``, attn_mma.cu): fp32 scores of the bf16 q and cached keys; over
        64-key tiles from key 0, P = exp(s - m) with m the running maximum up to and including the tile, rounded to bf16
        in the PV product while the row sum ``l_run`` adds the unrounded fp32 P; partials rescaled in fp32 as the maximum
        grows; output rounded to bf16 ``p_att``;
      - the wo and wd GEMMs add into the fp32 residual in their epilogue;
      - norm2 rounded to bf16; the wgu GEMM's GLU epilogue writes silu(gate) * up rounded to bf16 ``p_h``.
    The reader holds every position [0, start_pos + T), the rows this prefill wrote included, so attention sees the bf16
    keys and values the kernel saw.

``restate_head`` restates what follows the last layer: the final RMSNorm rounded to bf16 and the lm_head GEMM (every row's
logits of ``dtk_prefill`` and ``dtk_score``), the fp32-operand GEMV of the last row (``dtk_prefill``'s last logits) and the
log-softmax normaliser of ``dtk_score``.

Error model (``Noise`` of decode_restatement.py): fp32 dot products N(0, K u_acc^2 sum (w_j x_j)^2), elementwise fp32
results 4 u relative (the attention weights' ``exp2f`` included, before their bf16 rounding), the error added before each
bf16 rounding so boundary flips occur as in the kernel; the log-softmax normaliser carries an absolute N(0, s^2), s =
2^-21 (``__expf``) + u (|lse| + 4 sqrt(256 + V / 256)) (fp32 sums within each 256-column tile and the merge of the tiles'
partials). A uniform half-ulp error on every P instead of its rounding (the decode cascade's model) comes out near 4 % of
the residual's RMS: at T = 1 the kernel's only P is exactly 1, and a layer's bound could no longer tell its own rounding
points apart.

Ambiguous roundings. An element of a bf16 norm operand within 2^-18 (relative) of a rounding boundary may round either way
in the kernel (its fp32 RMSNorm differs from the exact one by a few u). ``kv_eps`` bounds what that does to the new K / V
rows (norm1; linear), ``logits_eps`` what it does to the logits (final norm; linear) and ``flip_eps`` what it does to the
layer's output residual. That one is not linear: one flipped norm element moves every q or SwiGLU input of its row and so
flips further bf16 roundings downstream, far more than the error model flips in that row. Rows are independent within a
layer (attention reads the cache), so ``flip_eps`` restates the layer once per rank k, with the k-th ambiguous element
of every row rounded the other way, and sums the changes.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch

from decode_restatement import U, U_ACC, Noise, Weights, _mm, _rms, _rope, bf16, bf16_ulp

PATHS = (None, "prefill")
NEAR = 2.0 ** -18          # relative distance to a bf16 rounding boundary below which the kernel may round either way
LSE_TILE = 256             # columns per log-softmax partial of the lm_head GEMM (launch.h)
BKV = 64                   # keys per tile of flash_attn_kernel


def _near(h: torch.Tensor, hb: torch.Tensor, rel: float = NEAR) -> torch.Tensor:
    """h lies within rel (relative) of a rounding boundary of its bf16 value hb."""
    return ((h - hb).abs() - bf16_ulp(hb) / 2).abs() <= rel * h.abs()


def _near_ulp(h: torch.Tensor, hb: torch.Tensor) -> torch.Tensor:
    """ulp(hb) where h lies within NEAR of a rounding boundary of its bf16 value hb, else 0."""
    return _near(h, hb) * bf16_ulp(hb)


def _round(h: torch.Tensor, flip: Optional[torch.Tensor]) -> torch.Tensor:
    """bf16(h), the elements of ``flip`` rounded to the other neighbour (h lies near the midpoint of the two, so 2h - hb
    rounds to it)."""
    hb = bf16(h)
    return hb if flip is None else torch.where(flip, bf16(2 * h - hb), hb)


def _attend(q, K, V, start_pos, nz, rb, gqa_mod, drop_key, causal_shift):
    """Causal attention of q [T, nh, hd] (query t at position start_pos + t) over K, V [nkv, n, hd]; -> [T, nh, hd].
    ``rb``: the kernel's bf16 P, taken over 64-key tiles relative to the running maximum."""
    T, nh, HD = q.shape
    nkv, n = K.shape[0], K.shape[1]
    dev = q.device
    heads = torch.arange(nh, device=dev)
    kvh = heads % nkv if gqa_mod else heads // (nh // nkv)
    Kh, Vh = K[kvh], V[kvh]                                   # [nh, n, hd]
    keys = torch.arange(n, device=dev)
    nt = (n + BKV - 1) // BKV
    out = torch.empty(T, nh, HD, device=dev, dtype=q.dtype)
    step = max(1, (1 << 24) // (nh * max(nt * BKV, 1)))      # query rows per chunk: ~128 MB per [nh, rows, n] temporary
    for t0 in range(0, T, step):
        t1 = min(T, t0 + step)
        qc = q[t0:t1]
        rows = t1 - t0
        s = torch.einsum("thd,hnd->htn", qc, Kh) / math.sqrt(HD)
        if nz is not None:
            s = s + U_ACC * torch.sqrt(torch.einsum("thd,hnd->htn", qc * qc, Kh * Kh)) * nz._n(s)
        qpos = start_pos + torch.arange(t0, t1, device=dev)
        vis = keys[None, :] <= qpos[:, None] + causal_shift     # [rows, n]
        if drop_key is not None:
            vis = vis & (keys != drop_key)[None, :]
        s = torch.nn.functional.pad(s.masked_fill(~vis[None], -math.inf), (0, nt * BKV - n), value=-math.inf)
        s = s.view(nh, rows, nt, BKV)
        m_fin = s.amax((-2, -1))[..., None, None]                # [nh, rows, 1, 1]
        m_run = s.amax(-1).cummax(-1).values[..., None] if rb else m_fin   # [nh, rows, nt, 1]
        p = torch.exp(s - m_run).nan_to_num(0.0)               # a row with no visible key: the kernel writes 0
        resc = torch.exp(m_run - m_fin).nan_to_num(0.0)        # fp32 rescaling of the earlier tiles' partials
        if nz is not None:
            p, resc = nz.elem(p), nz.elem(resc)
        pn = (bf16(p) if rb else p) * resc
        pr = p * resc
        pn, pr = pn.view(nh, rows, -1)[..., :n], pr.view(nh, rows, -1)[..., :n]
        o = torch.einsum("htn,hnd->htd", pn, Vh)
        if nz is not None:
            o = o + math.sqrt(n) * U_ACC * torch.sqrt(torch.einsum("htn,hnd->htd", pn * pn, Vh * Vh)) * nz._n(o)
        den = pr.sum(-1, keepdim=True)
        out[t0:t1] = torch.where(den > 0, o / den.clamp_min(1e-300), torch.zeros_like(o)).transpose(0, 1)
    return out


def restate_layer(w: Weights, l: int, x: torch.Tensor, start_pos: int, kv: Callable, path: Optional[str] = None,
                  nz: Optional[Noise] = None, causal_shift: int = 0, drop_key: Optional[int] = None, rope_shift: int = 0,
                  gqa_mod: bool = False, fp32_q: bool = False, fp32_att: bool = False, fp32_swiglu: bool = False,
                  flip1: Optional[torch.Tensor] = None, flip2: Optional[torch.Tensor] = None) -> dict:
    """Layer l over x [T, H] (float64) at positions [start_pos, start_pos + T). ``kv(l, n)`` -> (K, V) float64
    [kv_heads, n, hd]: the layer's cached positions [0, n) (see the module docstring for what it must hold per path).

    Negative controls (perturbed restatements the comparison must reject): ``causal_shift`` lets query t see the keys up to
    position start_pos + t + shift; ``drop_key`` leaves one cached position out of every softmax; ``rope_shift`` rotates q
    and k as at pos + shift; ``gqa_mod`` routes query head h to kv head h % kv_heads; ``fp32_q`` / ``fp32_att`` /
    ``fp32_swiglu`` remove the bf16 rounding of q, of the attention output and of the SwiGLU output. ``flip1`` / ``flip2``
    [T, H] (bool): elements of the bf16 norm1 / norm2 operand rounded the other way (``flip_eps``).

    Returns ``x`` [T, H]: the layer's output residual; ``k`` / ``v`` [T, kv_heads, hd]: the new cache rows before their bf16
    rounding, with ``kv_eps`` (k, v): how far ambiguous roundings of the bf16 norm1 operand can move them; ``near1`` /
    ``near2`` [T, H]: the norm operands' elements within NEAR of a rounding boundary (path "prefill")."""
    assert path in PATHS, path
    cfg = w.cfg
    dev = w.device
    T = x.shape[0]
    H, HD, nh, nkv = cfg.hidden_size, cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads
    qd, kd, eps = nh * HD, nkv * HD, cfg.rms_norm_eps
    rb = path == "prefill"
    p = f"dec.L{l}."
    zero = torch.zeros(T, nkv, HD, device=dev, dtype=torch.float64)
    kv_eps, near1, near2 = (zero, zero), None, None

    h = _rms(x, w(p + "norm1"), eps, nz)
    wqkv = w(p + "wqkv")
    if rb:
        hb = _round(h, flip1)
        if nz is None:
            amb = _near_ulp(h, hb) @ wqkv[qd:].abs().T        # [T, 2 kd]
            ak, av = amb[:, :kd].view(T, nkv, HD), amb[:, kd:].view(T, nkv, HD)
            kv_eps = (ak + ak.roll(HD // 2, -1), av)         # RoPE mixes the pair (i, i + hd/2) with |cos|, |sin| <= 1
            near1 = _near(h, hb)
        h = hb
    qkv = _mm(h, wqkv, nz)
    q = qkv[:, :qd].view(T, nh, HD)
    k = qkv[:, qd:qd + kd].view(T, nkv, HD)
    v = qkv[:, qd + kd:].view(T, nkv, HD)
    cs = w.rope[start_pos + rope_shift + torch.arange(T, device=dev)][:, None]   # [T, 1, hd/2, 2]
    q, k = _rope(q, cs), _rope(k, cs)
    if nz is not None:
        q, k = nz.elem(q), nz.elem(k)
    if rb and not fp32_q:
        q = bf16(q)
    if rb:
        K, V = kv(l, start_pos + T)
    else:
        K, V = kv(l, start_pos)
        K, V = torch.cat([K, k.transpose(0, 1)], 1), torch.cat([V, v.transpose(0, 1)], 1)
    a = _attend(q, K, V, start_pos, nz, rb, gqa_mod, drop_key, causal_shift).reshape(T, qd)
    if nz is not None:
        a = nz.elem(a)
    if rb and not fp32_att:
        a = bf16(a)
    x = x + _mm(a, w(p + "wo"), nz)
    if nz is not None:
        x = nz.elem(x)

    h = _rms(x, w(p + "norm2"), eps, nz)
    wgu = w(p + "wgu")
    if rb:
        hb = _round(h, flip2)
        if nz is None:
            near2 = _near(h, hb)
        h = hb
    gu = _mm(h, wgu, nz)
    g, u = gu[:, 0::2], gu[:, 1::2]
    sg = torch.sigmoid(g)
    hh = g * sg * u
    if nz is not None:
        hh = nz.elem(hh)
    if rb and not fp32_swiglu:
        hh = bf16(hh)
    wd = w(p + "wd")
    x = x + _mm(hh, wd, nz)
    if nz is not None:
        x = nz.elem(x)
    return {"x": x, "k": k, "v": v, "kv_eps": kv_eps, "near1": near1, "near2": near2}


def flip_eps(w: Weights, l: int, x, start_pos: int, kv, ref: dict) -> torch.Tensor:
    """[T, H]: per row, the sum over its ambiguous norm1 and norm2 elements (``ref["near1"]`` / ``["near2"]`` of the
    "prefill" restatement) of |output residual with that element rounded the other way - ``ref["x"]``."""
    eps = torch.zeros_like(ref["x"])
    for key in ("near1", "near2"):
        near = ref[key]
        rank = near.cumsum(-1) * near                          # 1, 2, ... along each row's ambiguous elements
        for k in range(1, int(rank.max()) + 1):
            r = restate_layer(w, l, x, start_pos, kv, "prefill", **{"flip" + key[-1]: rank == k})
            eps += (r["x"] - ref["x"]).abs()
            del r
    return eps


def restate_head(w: Weights, x: torch.Tensor, path: Optional[str] = None, nz: Optional[Noise] = None) -> dict:
    """The final RMSNorm and lm_head over the last layer's residual x [T, H] (float64).

    Returns ``logits`` [T, V] (bf16 norm operand with path "prefill": the GEMM of every row's logits) with ``logits_eps``
    [T, V] (path "prefill" without noise; else None), ``last_logits`` [V] (fp32 norm operand: the last row's GEMV) and
    ``lse`` [T]: log sum exp of ``logits``."""
    assert path in PATHS, path
    cfg = w.cfg
    lm = w("dec.lm_head")
    h = _rms(x, w("dec.norm"), cfg.rms_norm_eps, nz)
    last = _mm(h[-1:], lm, nz)[0]
    eps = None
    if path is not None:
        hb = bf16(h)
        if nz is None:
            eps = _near_ulp(h, hb) @ lm.abs().T
        h = hb
    logits = _mm(h, lm, nz)
    lse = torch.logsumexp(logits, -1)
    if nz is not None:
        V = lm.shape[0]
        s = 2.0 ** -21 + U * (lse.abs() + 4 * math.sqrt(LSE_TILE + V / LSE_TILE))
        lse = lse + s * nz._n(lse)
    return {"logits": logits, "logits_eps": eps, "last_logits": last, "lse": lse}


def layer_noise(w: Weights, l: int, x, start_pos: int, kv, path, ref: dict, draws: int = 4, seed: int = 0) -> dict:
    """Per row, the RMS (over the hidden size) change of the output residual under the error model; per (row, kv head) the
    RMS change of the new K / V rows before rounding; the larger of ``draws`` runs. A row's change comes from a handful of
    discrete rounding flips whose count varies from run to run, so it takes four."""
    T = x.shape[0]
    sig = torch.zeros(T, device=w.device, dtype=torch.float64)
    ksig = torch.zeros(T, w.cfg.num_key_value_heads, device=w.device, dtype=torch.float64)
    vsig = ksig.clone()
    for d in range(draws):
        r = restate_layer(w, l, x, start_pos, kv, path, nz=Noise(seed + d, w.device))
        sig = torch.maximum(sig, (r["x"] - ref["x"]).pow(2).mean(-1).sqrt())
        ksig = torch.maximum(ksig, (r["k"] - ref["k"]).pow(2).mean(-1).sqrt())
        vsig = torch.maximum(vsig, (r["v"] - ref["v"]).pow(2).mean(-1).sqrt())
        del r
    return {"x": sig, "k": ksig, "v": vsig}


def head_noise(w: Weights, x, path, ref: dict, targets: Optional[torch.Tensor] = None, draws: int = 2,
               seed: int = 0) -> dict:
    """Under the error model, the larger over ``draws`` runs of: per row, the RMS (over the vocabulary) change of the
    logits; the RMS change of the last row's GEMV logits; the RMS over the rows of the change of ``lse`` and, with
    ``targets`` (in range), of each row's log-probability (one value per row: a scale from one row would be one draw)."""
    T = x.shape[0]
    z = torch.zeros((), device=w.device, dtype=torch.float64)
    out = {"logits": torch.zeros(T, device=w.device, dtype=torch.float64), "last_logits": z, "lse": z, "logprob": z}
    rows = torch.arange(T, device=w.device)
    for d in range(draws):
        r = restate_head(w, x, path, nz=Noise(seed + d, w.device))
        out["logits"] = torch.maximum(out["logits"], (r["logits"] - ref["logits"]).pow(2).mean(-1).sqrt())
        out["last_logits"] = torch.maximum(out["last_logits"], (r["last_logits"] - ref["last_logits"]).pow(2).mean().sqrt())
        out["lse"] = torch.maximum(out["lse"], (r["lse"] - ref["lse"]).pow(2).mean().sqrt())
        if targets is not None:
            lp = r["logits"][rows, targets] - r["lse"]
            lp0 = ref["logits"][rows, targets] - ref["lse"]
            out["logprob"] = torch.maximum(out["logprob"], (lp - lp0).pow(2).mean().sqrt())
        del r
    return out
