"""
FP8 decoder weights (engine option ``decode_fp8``) against bf16 on the batched decode step. Prints ONE JSON line per shape.

For each of ds-1.3b, tl-1.1b, ds-7b and v2-8b, with ``device_init`` weights quantized in place as
``load(..., quantize="fp8")`` does, on one engine with ``decode_fp8`` alternating 0 / 1, --reps runs each (medians):
  * batched step: ``Engine.decode`` of B in --batches rows at ragged contexts around 512, CUDA-event time over --steps
    steps; ms per step and the weight bytes each step streams (``decode_weight_bytes``: the four layer matrices as bf16
    or as e4m3 codes plus one exponent per row, the lm_head in bf16);
  * kernel split: in a separate ``torch.profiler`` run, the summed time per step of the swapped-operand GEMM kernels
    (every dense matrix of the step, lm_head included), its share of all kernel time, and the GB/s it achieves over the
    bytes each mode streams;
  * rollouts (BASELINE configs[3] shape): per figure ViT + projector + prefill of the image prompt, then --rollouts
    nucleus rollouts (T 0.8, top-p 0.95) that borrow the image prefix (``seq_share``), --rollout-tokens new tokens each,
    in the device-resident loop; tok/s per mode, and whether both modes sampled the same ids (every step of one run each);
  * the card's name and power limit, read in the same run.
    python tools/bench_fp8_rollouts.py [--shapes ds-1.3b,tl-1.1b,ds-7b,v2-8b] [--batches 4,32,63] [--steps 50] [--reps 3]
"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_tl import gpu_info, hbm_peak  # noqa: E402

SHAPES = {"ds-1.3b": "nllg/detikzify-ds-1.3b", "tl-1.1b": "nllg/detikzify-tl-1.1b", "ds-7b": "nllg/detikzify-ds-7b",
          "v2-8b": "nllg/detikzify-v2-8b"}
MODES = ((0, "bf16"), (1, "fp8"))


def median(xs):
    return sorted(xs)[len(xs) // 2]


def bench_shape(key, args, peak, peak_src):
    from detikzify_b200.engine import Engine, random_arena_device, weight_table
    from detikzify_b200.model.configuration import preset
    from detikzify_b200.quant import quantize_arena_fp8
    from oracle.hf_oracle import synthetic_pixels

    cfg = preset(SHAPES[key])
    batches = [int(b) for b in args.batches.split(",")]
    nrows = max(max(batches), args.rollouts)
    P = cfg.num_patches
    dev = torch.device("cuda:0")
    arena = random_arena_device(cfg, dev, seed=0)
    eng = Engine(cfg, arena, device=0, max_seqs=nrows + 1, max_batch=nrows,
                 max_len=max(1024, P + args.rollout_tokens + 64))   # every row a KV slot: 2k slots of ds-7b do not fit 64 times
    quantize_arena_fp8(eng.arena, weight_table(eng.ccfg))
    eng.set_option("decode_fp8", 1)                                  # tiles of the quantized arena
    stream = torch.cuda.Stream(device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    g = torch.Generator().manual_seed(9100)
    slots = [eng.seq_alloc() for _ in range(nrows + 1)]
    out = {"shape": key, "model": SHAPES[key], **gpu_info(), "hbm_peak_gbs": peak, "hbm_peak_source": peak_src}

    with torch.cuda.stream(stream):
        # ---- batched step at ragged contexts 480 + i
        lens = [480 + i for i in range(nrows)]
        for s, n in zip(slots, lens):
            eng.prefill(s, torch.randint(3, 30000, (n,), generator=g).to(dev), 0, None, 0)
        toks = torch.randint(3, 30000, (nrows,), generator=g).to(dev)

        def step_run(B):
            for _ in range(3):
                eng.decode(slots[:B], lens[:B], toks[:B])
            ev[0].record(stream)
            for _ in range(args.steps):
                eng.decode(slots[:B], lens[:B], toks[:B])
            ev[1].record(stream)
            stream.synchronize()
            return ev[0].elapsed_time(ev[1]) / args.steps

        step_ms = {(m, B): [] for m, _ in MODES for B in batches}
        for _ in range(args.reps):
            for m, _ in MODES:
                eng.set_option("decode_fp8", m)
                for B in batches:
                    step_ms[m, B].append(step_run(B))
        wbytes = {}
        for m, _ in MODES:
            eng.set_option("decode_fp8", m)
            wbytes[m] = eng.get_option("decode_weight_bytes")

        # ---- kernel split (profiler run of its own)
        split = {}
        for m, name in MODES:
            eng.set_option("decode_fp8", m)
            for B in batches:
                step_run(B)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(args.steps):
                        eng.decode(slots[:B], lens[:B], toks[:B])
                    stream.synchronize()
                gemm_us = all_us = 0.0
                for e in prof.key_averages():
                    t = e.device_time_total
                    all_us += t
                    if "gemm_tc_swap_kernel" in e.key:
                        gemm_us += t
                gemm_ms = gemm_us / 1e3 / args.steps
                split[name, B] = {"swap_gemm_ms_per_step": gemm_ms, "kernel_ms_per_step": all_us / 1e3 / args.steps,
                                  "swap_gemm_share": gemm_us / all_us, "swap_gemm_gbs": wbytes[m] / (gemm_ms * 1e-3) / 1e9}

        # ---- rollouts: ViT + projector + prefill, R rollouts borrowing the image prefix
        R, NT = args.rollouts, args.rollout_tokens
        pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=5000).to(dev)
        ids = torch.full((P,), cfg.patch_token_id, dtype=torch.int64, device=dev)
        nuc = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id, begin_suppress_token=-1,
                           seed=3)
        base, rows = slots[nrows], slots[:R]

        def figure(every_step=False):
            for sl in rows:
                eng.seq_share(base, sl, 0)            # release the previous prefix loan
            ev[0].record(stream)
            img = eng.image_embeds(pix)[0]
            last, _ = eng.prefill(base, ids, 0, img, 0)
            for sl in rows:
                eng.seq_share(base, sl, P)            # rollouts read the image prefix in place
            first, _ = eng.sample(last[None].expand(R, -1).contiguous(), nuc, suppress=[0] * R, steps=[0] * R, seq_ids=list(range(R)))
            eng.gen_begin(rows, [P] * R, [int(t) for t in first.tolist()], nuc, list(range(R)))
            got = [[int(t) for t in first.tolist()]]
            for t in range(NT - 1):
                eng.gen_step()
                if every_step:
                    got.append(eng.gen_wait(t))
            if not every_step:
                got.append(eng.gen_wait(NT - 2))
            eng.gen_end()
            ev[1].record(stream)
            stream.synchronize()
            return ev[0].elapsed_time(ev[1]), got

        roll_ms, roll_ids = {0: [], 1: []}, {}
        for m, _ in MODES:
            eng.set_option("decode_fp8", m)
            roll_ids[m] = figure(every_step=True)[1]   # warm-up (graph capture) and the ids of every step
        for _ in range(args.reps):
            for m, _ in MODES:
                eng.set_option("decode_fp8", m)
                roll_ms[m].append(figure()[0])

    for m, name in MODES:
        out[name] = {"weight_bytes_per_step": wbytes[m],
                     "step": {str(B): {"ms": median(step_ms[m, B]), "all_ms": step_ms[m, B], **split[name, B]} for B in batches},
                     "rollouts": {"n": R, "new_tokens": NT, "ms": median(roll_ms[m]),
                                  "tok_s": R * NT / (median(roll_ms[m]) * 1e-3), "all_ms": roll_ms[m]}}
    out["step_speedup"] = {str(B): out["bf16"]["step"][str(B)]["ms"] / out["fp8"]["step"][str(B)]["ms"] for B in batches}
    out["swap_gemm_speedup"] = {str(B): out["bf16"]["step"][str(B)]["swap_gemm_ms_per_step"] /
                                out["fp8"]["step"][str(B)]["swap_gemm_ms_per_step"] for B in batches}
    out["rollout_speedup"] = out["fp8"]["rollouts"]["tok_s"] / out["bf16"]["rollouts"]["tok_s"]
    out["rollout_ids_equal"] = roll_ids[0] == roll_ids[1]
    for s in slots[:nrows]:                            # borrowers before the lender
        eng.seq_free(s)
    eng.seq_free(slots[nrows])
    eng.close()
    del eng, arena
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="ds-1.3b,tl-1.1b,ds-7b,v2-8b")
    ap.add_argument("--batches", default="4,32,63")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rollouts", type=int, default=32)
    ap.add_argument("--rollout-tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_rollouts.py measures the GPU; no CUDA device found")
    peak, peak_src = hbm_peak()
    for key in args.shapes.split(","):
        print(json.dumps(bench_shape(key, args, peak, peak_src)), flush=True)


if __name__ == "__main__":
    main()
