"""
Sequence scoring on one GPU, at the ds-1.3b and v2-8b shapes. Prints ONE JSON line:

  * lm_head: the lm_head phase alone at T = --T rows (A bf16 [T,H] ~ N(0,1), W bf16 [V,H] ~ N(0, 0.02^2)):
      - fused: the GEMM with the log-softmax epilogue + the partials merge (dtk_dbg_lm_logprob);
      - unfused: the same GEMM writing fp32 [T,V] logits (dtk_dbg_gemm), then torch.log_softmax and a gather;
    median ms of --reps calls from CUDA events, TFLOP/s (2 T V H flop over that time, beside the 989 TFLOP/s BF16 dense data-sheet peak), and the
    extra device memory of each path (fused: T ceil(V/256) 8 B of partials; unfused: the torch allocator's peak growth);
  * ranking: --cands candidates of --code code tokens right after one image prefix (243 tokens at ds-1.3b, 300 at v2-8b),
    scored from the first code token with one model.score() call (one tower pass, the image prefix prefilled once), with one
    score() per candidate (no sharing, no logits) and with one forward(labels=...) per candidate (no sharing, [T,V]
    logits): scored tokens/s of the median repetition, the time of every repetition and the allocator's peak growth;
  * the GPU's name and power limit, read in the same run.

Weights: device_init=True (seeded random init on the GPU; the kernels' cost does not depend on the values).
    python tools/bench_score.py [--T 2047] [--cands 32] [--code 512] [--reps 20] [--models ds-1.3b,v2-8b]
"""
import argparse
import ctypes as C
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_tl import gpu_info   # noqa: E402

PEAK_TFLOPS = 989.0   # H100 SXM data sheet, dense BF16
NAMES = {"ds-1.3b": "nllg/detikzify-ds-1.3b", "v2-8b": "nllg/detikzify-v2-8b"}


def _p(t):
    return C.c_void_p(0 if t is None else t.data_ptr())


def timed(fn, reps):
    """ms of each of ``reps`` calls after one warm-up call (CUDA events around each call)."""
    fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        fn()
        ev[i + 1].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(reps)]


def med(xs):
    return sorted(xs)[len(xs) // 2]


def lm_head_phase(cfg, T, reps):
    from detikzify_b200 import _lib
    lib = _lib.load_library()
    H, V = cfg.hidden_size, cfg.vocab_size
    g = torch.Generator(device="cuda").manual_seed(0)
    A = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    W = (torch.randn(V, H, device="cuda", generator=g) * 0.02).to(torch.bfloat16)
    tg = torch.randint(0, V, (T,), device="cuda", generator=g)
    lp, lse = torch.empty(T, device="cuda"), torch.empty(T, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def fused():
        assert lib.dtk_dbg_lm_logprob(_p(A), _p(W), T, V, H, _p(tg), _p(lp), _p(lse), st) == 0

    def unfused():
        logits = torch.empty(T, V, device="cuda")
        assert lib.dtk_dbg_gemm(_p(A), _p(W), None, None, T, V, H, 0, 0, _p(logits), None, st) == 0
        return torch.log_softmax(logits, -1).gather(1, tg[:, None])[:, 0]

    flop = 2.0 * T * V * H
    ms_f = med(timed(fused, reps))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ms_u = med(timed(unfused, reps))
    extra_u = torch.cuda.max_memory_allocated() - base
    err = (unfused() - lp).abs().max().item()
    return {"T": T, "V": V, "H": H,
            "fused_ms": round(ms_f, 4), "fused_tflops": round(flop / ms_f / 1e9, 1),
            "unfused_ms": round(ms_u, 4), "unfused_tflops": round(flop / ms_u / 1e9, 1),
            "peak_tflops_datasheet": PEAK_TFLOPS, "fused_frac_of_peak": round(flop / ms_f / 1e9 / PEAK_TFLOPS, 3),
            "fused_extra_bytes": T * ((V + 255) // 256) * 8 + 4 * T, "unfused_extra_bytes_measured": int(extra_u),
            "max_abs_diff_logprob": err}


def ranking(model, cands, code, reps):
    from oracle.hf_oracle import synthetic_pixels
    cfg = model.config
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=3).cuda()
    g = torch.Generator().manual_seed(1)
    P = cfg.num_patches
    head = torch.full((P,), cfg.patch_token_id)
    seqs = [torch.cat([head, torch.randint(0, 32000, (code,), generator=g)]) for _ in range(cands)]
    n_tok = cands * code

    def by_score():          # one call: one tower pass, the image prefix prefilled once and lent to every candidate
        return model.score(seqs, pix, start=P)

    def by_score_each():     # one score() per candidate: tower and whole-sequence prefill per candidate, no logits
        for q in seqs:
            model.score([q], pix, start=P)

    def by_forward():        # one forward(labels=...) per candidate: as above, plus the [T, V] fp32 logits
        for q in seqs:
            lab = q.clone()
            lab[:P] = -100
            model(input_ids=q[None], pixel_values=pix, labels=lab[None])

    out = {"candidates": cands, "code_tokens": code, "image_tokens": P, "reps": reps}
    for name, fn in (("score", by_score), ("score_each", by_score_each), ("forward", by_forward)):
        fn()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        ms = timed(fn, reps)
        out[f"{name}_tok_s"] = round(n_tok / med(ms) * 1e3, 1)
        out[f"{name}_ms"] = [round(x, 2) for x in ms]
        out[f"{name}_peak_extra_bytes"] = int(torch.cuda.max_memory_allocated() - base)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--T", type=int, default=2047)
    ap.add_argument("--cands", type=int, default=32)
    ap.add_argument("--code", type=int, default=512)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rank-reps", type=int, default=5)
    ap.add_argument("--models", default="ds-1.3b,v2-8b")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_score.py measures the GPU; no CUDA device found")
    from detikzify_b200.model import load
    res = {"bench": "score", **gpu_info()}
    for key in args.models.split(","):
        model, _ = load(NAMES[key], device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=4, max_batch=1)
        res[key] = {"lm_head": lm_head_phase(model.config, args.T, args.reps),
                    "ranking": ranking(model, args.cands, args.code, args.rank_reps)}
        model.close()
        del model
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
