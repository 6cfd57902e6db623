"""
fp64 restatement of the sampler's HF logits processors (dtk_processors; detikzify_b200/csrc/sample.cu, PROC instantiations),
on top of the processor chain of oracle/sample_oracle.py:
  repetition penalty (fp32, on every distinct id of the row's history: x < 0 ? x * p : x / p) -> bans (-inf): no-repeat
  n-gram, single ids, bad-word sequences whose prefix ends the history (skipped when longer than the history), EOS while the
  history is shorter than eos_min_len, begin-suppress ids on rows with the suppress flag -> /T -> top-k -> softmax -> top-p
  -> min-p (drop p < min_p * p_max; sampling only) -> renormalise.
"""
from __future__ import annotations

import numpy as np

from oracle import sample_oracle as so


def banned_ngram_tokens(hist, n: int):
    """HF _calc_banned_ngram_tokens for one row: ids that followed an earlier occurrence of the last n - 1 ids."""
    L = len(hist)
    if n <= 0 or L + 1 < n:
        return []
    tail = list(hist[L - n + 1:]) if n > 1 else []
    return [hist[j + n - 1] for j in range(L - n + 1) if list(hist[j:j + n - 1]) == tail]


def processed_logits(logits, histories, penalty: float = 1.0, ngram: int = 0, ban_ids=(), begin_ids=(), words=(),
                     eos: int = -1, eos_min_len=None, suppress=False) -> np.ndarray:
    """fp64 [B, V] scores after the processors, before the temperature (the penalty rounds in fp32 as HF's does)."""
    s = np.array(logits, dtype=np.float32, ndmin=2).copy()
    B, V = s.shape
    sup = np.broadcast_to(np.asarray(suppress, dtype=bool), (B,))
    eml = np.zeros(B, dtype=np.int64) if eos_min_len is None else np.asarray(eos_min_len)
    p32 = np.float32(penalty)
    for b, h in enumerate(histories):
        if penalty != 1.0 and len(h):
            ids = np.unique(np.asarray(h, dtype=np.int64))
            x = s[b, ids]
            s[b, ids] = np.where(x < 0, x * p32, x / p32)
    out = s.astype(np.float64)
    for b, h in enumerate(histories):
        h = [int(i) for i in h]
        ban = list(ban_ids) + banned_ngram_tokens(h, ngram)
        for w in words:
            if len(w) <= len(h) and h[len(h) - len(w) + 1:] == list(w[:-1]):
                ban.append(w[-1])
        if sup[b]:
            ban += list(begin_ids)
        if 0 <= eos < V and len(h) < eml[b]:
            ban.append(eos)
        if ban:
            out[b, np.asarray(ban, dtype=np.int64)] = -np.inf
    return out


def processed_probs(logits, histories, temperature: float = 1.0, top_p: float = 1.0, top_k: int = 0, min_p: float = 0.0,
                    do_sample: bool = True, **proc) -> dict:
    """so.processed_probs on the processed scores, plus min-p after top-p when sampling. Adds ``min_p_rel`` = p / p_max
    (what the min-p rule compares with min_p)."""
    s = processed_logits(logits, histories, **proc)
    r = so.processed_probs(s, temperature=temperature, top_p=top_p, top_k=top_k, do_sample=do_sample)
    sm = r["softmax"]
    r["min_p_rel"] = sm / sm.max(axis=1, keepdims=True)
    if so.is_sampling(do_sample, temperature) and min_p > 0:
        kept = r["kept"] & (r["min_p_rel"] >= min_p)
        p = np.where(kept, sm, 0.0)
        r["kept"], r["probs"] = kept, p / p.sum(axis=1, keepdims=True)
    return r
