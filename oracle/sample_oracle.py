"""
fp64 restatement of the fused sampler (detikzify_b200/csrc/sample.cu) in numpy: the Philox4x32-10 uniform, the processor
chain and the inverse-CDF draw, plus the fp32 prefix sums the kernel's draw compares the uniform against.

The processor chain follows the kernel's documented rule, which differs from HF's TopPLogitsWarper only inside a tie group:
  mask bad token -> mask the begin-suppress token (first new token only) -> /T -> top-k (keep every score >= the k-th
  largest; off when k <= 0 or k >= V) -> softmax -> top-p (drop every token whose probability p satisfies
  sum_{q <= p} q <= (float)(1 - top_p), always keep the maximum) -> renormalise.
A tie group is kept or dropped as a whole; HF sorts the vocabulary and may split one.

The draw of sequence ``seq_id`` at RNG counter ``step`` (+ the generation loop's ``gen_step``) is
  x = Philox4x32-10(counter = (step + gen_step mod 2^32, seq_id, 0x243F6A88, 0x85A308D3), key = (seed_lo, seed_hi)),
  u = (x0 >> 8) / 2^24,
  token = the first index, in index order, where the running sum of the probability vector exceeds u.
"""
from __future__ import annotations

import numpy as np

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
CTR2, CTR3 = 0x243F6A88, 0x85A308D3
MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC'11; the constants of Random123 and of CUDA's curand_philox4x32_x.h).
    ctr: [..., 4] words, key: [..., 2] words (broadcast against each other) -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    key = np.asarray(key, dtype=np.uint64)
    x0, x1, x2, x3 = (ctr[..., i] for i in range(4))
    k0, k1 = key[..., 0], key[..., 1]
    for _ in range(10):
        p0 = np.uint64(M0) * x0
        p1 = np.uint64(M1) * x2
        x0, x1, x2, x3 = ((p1 >> np.uint64(32)) ^ x1 ^ k0, p1 & MASK32, (p0 >> np.uint64(32)) ^ x3 ^ k1, p0 & MASK32)
        k0 = (k0 + np.uint64(W0)) & MASK32
        k1 = (k1 + np.uint64(W1)) & MASK32
    return np.stack([x0, x1, x2, x3], axis=-1).astype(np.uint32)


def uniform(seed: int, step, seq_id, gen_step: int = 0) -> np.ndarray:
    """The sampler's uniform in [0, 1) for a 64-bit seed; step / seq_id broadcast (uint32 each)."""
    step = np.asarray(step, dtype=np.uint64)
    seq_id = np.asarray(seq_id, dtype=np.uint64)
    step, seq_id = np.broadcast_arrays(step, seq_id)
    c0 = (step + np.uint64(gen_step & 0xFFFFFFFF)) & MASK32
    ctr = np.stack([c0, seq_id, np.full_like(c0, CTR2), np.full_like(c0, CTR3)], axis=-1)
    seed = int(seed) & (2**64 - 1)
    x = philox4x32_10(ctr, [seed & 0xFFFFFFFF, seed >> 32])
    return (x[..., 0] >> np.uint32(8)).astype(np.float64) / 2.0**24


def is_sampling(do_sample: bool, temperature: float) -> bool:
    """dtk_sampling: greedy when do_sample is off or the temperature is below 1e-5."""
    return bool(do_sample) and temperature >= 1e-5


def masked_scores(logits, bad_token: int = -1, begin_suppress_token: int = -1, suppress=False) -> np.ndarray:
    """fp64 [B, V] logits with the bad token and, on rows with ``suppress``, the begin-suppress token set to -inf."""
    s = np.array(logits, dtype=np.float64, ndmin=2)
    B, V = s.shape
    if 0 <= bad_token < V:
        s[:, bad_token] = -np.inf
    sup = np.broadcast_to(np.asarray(suppress, dtype=bool), (B,))
    if 0 <= begin_suppress_token < V:
        s[sup, begin_suppress_token] = -np.inf
    return s


def greedy(logits, bad_token: int = -1, begin_suppress_token: int = -1, suppress=False) -> np.ndarray:
    """Greedy tokens: the lowest index among the maxima of the masked logits (np.argmax returns the first)."""
    return masked_scores(logits, bad_token, begin_suppress_token, suppress).argmax(axis=1)


def mass_at_or_below(p: np.ndarray) -> np.ndarray:
    """S[b, i] = sum of p[b, j] over every j with p[b, j] <= p[b, i] (ties included), in fp64."""
    B, V = p.shape
    S = np.empty_like(p)
    idx = np.arange(V)
    for b, row in enumerate(p):
        order = np.argsort(row)
        ps = row[order]
        last = np.append(ps[:-1] != ps[1:], True)       # last member of its tie group in ascending order
        end = np.minimum.accumulate(np.where(last, idx, V - 1)[::-1])[::-1]
        S[b, order] = np.cumsum(ps)[end]
    return S


def top_p_limit(top_p: float) -> float:
    """The kernel removes ascending cumulative mass <= (float)(1 - top_p) (dtk_sampling keeps top_p in double)."""
    return float(np.float32(1.0 - top_p))


def processed_probs(logits, temperature: float = 1.0, top_p: float = 1.0, top_k: int = 0, bad_token: int = -1,
                    begin_suppress_token: int = -1, suppress=False, do_sample: bool = True) -> dict:
    """The probability vector the sampler draws from, in fp64. Returns a dict of [B, V] arrays:
    ``probs`` (renormalised over the kept tokens), ``kept`` (bool), ``softmax`` (after top-k, before top-p), ``mass_below``
    (``mass_at_or_below`` of ``softmax``, what the top-p rule compares with the limit; None when top-p is off) and ``rel`` = exp(score - max) (the
    unnormalised softmax term). Greedy (``is_sampling`` false): ``probs`` = softmax of the masked logits, like the kernel's
    returned vector."""
    s = masked_scores(logits, bad_token, begin_suppress_token, suppress)
    B, V = s.shape
    sampling = is_sampling(do_sample, temperature)
    if sampling:
        s = s / temperature
        if 0 < top_k < V:
            kth = np.partition(s, V - top_k, axis=1)[:, V - top_k][:, None]
            s = np.where(s >= kth, s, -np.inf)
    m = s.max(axis=1, keepdims=True)
    rel = np.exp(s - m)
    sm = rel / rel.sum(axis=1, keepdims=True)
    S = None
    kept = sm > 0
    if sampling and top_p < 1.0:
        S = mass_at_or_below(sm)
        drop = S <= top_p_limit(top_p)
        drop &= sm < sm.max(axis=1, keepdims=True)          # min_tokens_to_keep = 1
        kept &= ~drop
    p = np.where(kept, sm, 0.0)
    p = p / p.sum(axis=1, keepdims=True)
    return {"probs": p, "kept": kept, "softmax": sm, "mass_below": S, "rel": rel}


def draw(probs, u) -> np.ndarray:
    """Inverse-CDF draw in index order over each row of ``probs`` (summed in fp64): the first index whose running sum
    exceeds u. Returns V where u is not below the row's total (the kernel falls back to the argmax there)."""
    cdf = np.cumsum(np.array(probs, dtype=np.float64, ndmin=2), axis=1)
    u = np.broadcast_to(np.asarray(u, dtype=np.float64), (cdf.shape[0],))
    return np.array([np.searchsorted(c, x, side="right") for c, x in zip(cdf, u)])


def kernel_prefix_sums(probs32, threads: int = 1024):
    """The CDF boundaries of one fp32 probability row as the kernel's draw computes them, next to the same boundaries in fp64.

    The kernel gives thread t the chunk [t * per, (t + 1) * per) with per = ceil(V / threads), sums it sequentially (loc),
    scans the chunk sums with two 32-wide Hillis-Steele scans (within each warp, then over the warp totals), forms the exclusive
    offset excl = (warp offset + inclusive) - loc, and the thread whose [excl, excl + loc) holds u walks its chunk adding
    the positive entries to excl. Returns (b64, b32): every boundary the search compares u against (each chunk's excl and
    excl + loc, and excl plus each positive entry's running sum) in fp64 over the same fp32 values, and as the kernel's fp32
    arithmetic rounds it. |b32 - b64| is the summation error at that boundary."""
    p = np.asarray(probs32, dtype=np.float32).reshape(-1)
    V = p.size
    per = -(-V // threads)
    w = np.zeros(threads * per, dtype=np.float32)
    w[:V] = p
    w = w.reshape(threads, per)
    loc = np.zeros(threads, dtype=np.float32)
    for j in range(per):
        loc = loc + w[:, j]
    lane = np.arange(threads) % 32

    def warp_scan(x):
        x = x.reshape(-1, 32).copy()
        for o in (1, 2, 4, 8, 16):
            sh = np.zeros_like(x)
            sh[:, o:] = x[:, :-o]
            x = np.where((np.arange(32) >= o)[None, :], x + sh, x)
        return x.reshape(-1)

    inc = warp_scan(loc)
    tot = inc[lane == 31]
    woff = warp_scan(tot) - tot
    excl = (woff[np.arange(threads) // 32] + inc) - loc
    c = excl.copy()
    run32 = np.empty_like(w)
    for j in range(per):
        c = np.where(w[:, j] > 0, c + w[:, j], c)
        run32[:, j] = c
    w64 = w.astype(np.float64)
    start64 = np.concatenate([[0.0], np.cumsum(w64.sum(axis=1))[:-1]])
    run64 = start64[:, None] + np.cumsum(w64, axis=1)
    pos, act = w > 0, loc > 0      # a chunk without mass never claims the draw
    b64 = np.concatenate([start64[act], (start64 + w64.sum(axis=1))[act], run64[pos]])
    b32 = np.concatenate([excl[act], (excl + loc)[act], run32[pos]]).astype(np.float64)
    return b64, b32
