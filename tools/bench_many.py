"""
Continuous batching (``generate_many``) against lock-step ``generate_batch`` chunks on a stream of requests whose program
lengths vary. Prints ONE JSON line per (shape, workload, arm).

Workloads: 256 requests as 8 figures x 32 samples, and as 1 figure x 256 samples; nucleus sampling (T 0.8, top-p 0.95).
Random weights never stop on their own, so request i stops after L_i new tokens (its stopping criterion), L_i drawn
log-uniformly from [64, max_len - prompt length] (seed 0) and EOS is disabled; both arms get the same L_i. Arms, alternated
in one process, --runs runs each:
  * lock-step: ``generate_batch`` in chunks of --batch requests, one figure per chunk (a chunk runs as long as its longest
    program);
  * many: ``generate_many(batch_size=--batch)`` over all requests (a finished row takes the next request at once).
Each line: generated tokens/s over the whole call (ViT, prefill and admissions included; median and all runs), decode steps
launched, mean rows per step that produced a kept token, and the card's name and power limit read in the same run.

Without a GPU the tool prints the step and occupancy counts of both arms, which follow from the lengths and the host's
schedule alone, and exits with status 1: it never falls back to a CPU run.
    python tools/bench_many.py [--shapes ds-1.3b,ds-7b] [--workloads 8x32,1x256] [--runs 3] [--batch 32]
"""
import argparse
import json
import math
import sys
import time
from collections import deque
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

SHAPES = {"ds-1.3b": "nllg/detikzify-ds-1.3b", "ds-7b": "nllg/detikzify-ds-7b"}
MAX_LEN = 2048
TEXT = [185, 186, 187, 188]   # a few text tokens after the image span: the samples of a figure share the whole prompt


def lengths(n, prefix, seed=0):
    g = torch.Generator().manual_seed(seed)
    lo, hi = math.log(64), math.log(MAX_LEN - prefix)
    return [int(round(math.exp(lo + (hi - lo) * float(u)))) for u in torch.rand(n, generator=g, dtype=torch.float64)]


def lockstep_counts(L, B, F):
    """decode steps and kept-token row-steps of generate_batch chunks of B requests, one figure per chunk"""
    per = len(L) // F
    steps = 0
    for f in range(F):
        fl = L[f * per:(f + 1) * per]
        steps += sum(max(fl[c:c + B]) - 1 for c in range(0, per, B))
    return steps, sum(x - 1 for x in L)


def many_counts(L, B):
    """decode steps of generate_many's schedule (two steps in flight, a finished row refilled after the host reads its last
    token): the same policy as DetikzifyForCausalLM._many, on lengths alone"""
    N = len(L)
    queue = deque(range(N))
    got = [0] * N
    rows, s0 = [], []
    for _ in range(min(B, N)):
        i = queue.popleft()
        rows.append(i); s0.append(0); got[i] = 1
    cap = max(L[i] for i in rows) - 1
    launched = waited = 0
    pending = []
    while True:
        for r, i in enumerate(rows):
            if i is not None and got[i] >= L[i]:
                rows[r] = None
        for r in range(len(rows)):
            if rows[r] is None and queue:
                i = queue.popleft()
                rows[r], s0[r] = i, launched
                cap = max(cap, launched + L[i] - 1)
                pending.append(r)
        if all(i is None for i in rows):
            break
        while launched < waited + 2 and launched < cap:
            launched += 1
        for r in pending:
            got[rows[r]] += 1
        pending = []
        if not any(i is not None and got[i] < L[i] for i in rows):
            continue
        for r, i in enumerate(rows):
            if i is not None and waited >= s0[r] and got[i] < L[i]:
                got[i] += 1
        waited += 1
    return launched, sum(x - 1 for x in L)


def counts(L, B, F):
    ls, useful = lockstep_counts(L, B, F)
    ms, _ = many_counts(L, B)
    return {"lockstep": {"steps": ls, "mean_active_rows": round(useful / ls, 2)},
            "many": {"steps": ms, "mean_active_rows": round(useful / ms, 2)}}


def workload(spec):
    F, per = (int(x) for x in spec.split("x"))
    return F, per


def bench_shape(key, args):
    from bench_tl import gpu_info
    from detikzify_b200.engine import random_arena_device
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.model.modeling import DetikzifyForCausalLM
    from oracle.hf_oracle import synthetic_pixels

    cfg = preset(SHAPES[key])
    B = args.batch
    dev = torch.device("cuda:0")
    F_max = max(workload(w)[0] for w in args.workloads.split(","))
    model = DetikzifyForCausalLM(cfg, random_arena_device(cfg, dev, seed=0), device=0, max_seqs=B + args.spare_slots,
                                 max_batch=B, max_len=MAX_LEN)
    eng = model.engine
    steps = [0]
    gen_step = eng.gen_step

    def counted():
        steps[0] += 1
        gen_step()
    eng.gen_step = counted
    info = gpu_info()
    pixels = synthetic_pixels(F_max, cfg.vision_config.image_size, seed=3)
    prompt = torch.tensor([cfg.image_token_id] * cfg.num_patches + TEXT, dtype=torch.int64)
    kw = dict(do_sample=True, temperature=0.8, top_p=0.95, eos_token_id=-1, bad_words_ids=[[cfg.image_token_id]],
              max_length=MAX_LEN)
    for spec in args.workloads.split(","):
        F, per = workload(spec)
        N = F * per
        L = lengths(N, prompt.numel())
        prompts = [prompt] * N
        crit = [[(lambda ids, scores, n=prompt.numel() + k: ids.shape[1] >= n)] for k in L]
        figure = [i // per for i in range(N)]

        def lockstep():
            out = {}
            for f in range(F):
                for c in range(0, per, B):
                    idx = [f * per + c + j for j in range(min(B, per - c))]
                    res = model.generate_batch([prompts[i] for i in idx], pixels[f:f + 1], seed=f * per + c,
                                               stopping_criteria=[crit[i] for i in idx], **kw)
                    out.update(zip(idx, res))
            return out

        def many():
            return dict(model.generate_many(prompts, pixels[:F], figure=figure, batch_size=B, seed=0,
                                            stopping_criteria=crit, **kw))

        arms = (("lockstep", lockstep), ("many", many))
        res = {name: {"rates": [], "steps": None} for name, _ in arms}
        for _ in range(args.runs):
            for name, fn in arms:
                torch.cuda.synchronize()
                steps[0] = 0
                t0 = time.perf_counter()
                out = fn()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                new = sum(len(out[i]) - prompt.numel() for i in range(N))
                assert new == sum(L), (name, new, sum(L))
                res[name]["rates"].append(new / dt)
                res[name]["steps"] = steps[0]
        for name, _ in arms:
            r = res[name]
            rates = sorted(r["rates"])
            print(json.dumps({
                "shape": key, "model": SHAPES[key], "workload": f"{F} figures x {per} samples", "arm": name,
                "batch": B, "requests": N, "length_distribution": f"log-uniform integer new tokens on [64, {MAX_LEN - prompt.numel()}], seed 0",
                "mean_new_tokens": round(sum(L) / N, 1), "tok_per_s": round(rates[len(rates) // 2], 1),
                "tok_per_s_runs": [round(x, 1) for x in r["rates"]], "steps": r["steps"],
                "mean_active_rows": round(sum(x - 1 for x in L) / r["steps"], 2), **info}), flush=True)
    model.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="ds-1.3b,ds-7b")
    ap.add_argument("--workloads", default="8x32,1x256")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--spare-slots", type=int, default=6, help="KV slots beyond --batch: figure prefixes and generate()'s own")
    args = ap.parse_args()
    P = 243 + len(TEXT)   # the checkpoints' image span (num_patches) + the text
    for spec in args.workloads.split(","):
        F, per = workload(spec)
        L = lengths(F * per, P)
        print(json.dumps({"workload": f"{F} figures x {per} samples", "batch": args.batch,
                          "mean_new_tokens": round(sum(L) / len(L), 1), "counts": counts(L, args.batch, F)}), flush=True)
    if not torch.cuda.is_available():
        print("bench_many: no CUDA device; the counts above follow from the lengths, the tokens/s need an H100",
              file=sys.stderr)
        sys.exit(1)
    for key in args.shapes.split(","):
        bench_shape(key, args)


if __name__ == "__main__":
    main()
