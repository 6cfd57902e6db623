"""
detikzify-tl-1.1b (TinyLlama-1.1B decoder, head_dim 64, GQA 32/4) on one GPU. Prints ONE JSON line:

  * decode: batch-1 greedy loop from the 243-token image prefix to --total-len, device-resident (persistent kernel + fused
    argmax, token ring to the host), tokens/s over CUDA-event time, and the decode HBM fraction: the algorithmic bytes
    sum over T of dtk_decode_bytes(T) (weights once + the KV rows read) over that time, against MEASURED_PEAKS.json
    (hbm_gbs) or the H100 SXM data sheet's 3.35 TB/s;
  * prefill_ms: the 243-row image-prefix prefill (projector output given);
  * rollouts: --rollouts nucleus rollouts (T 0.8, top-p 0.95) that read one image prefix in place (dtk_seq_share), each
    --rollout-tokens new tokens, tokens/s over the whole figure (ViT + prefill + rollouts);
  * the GPU's name and power limit, read in the same run.

Weights: device_init=True (seeded random init on the GPU; the kernels' cost does not depend on the values).
    python tools/bench_tl.py [--total-len 2048] [--rollouts 32] [--rollout-tokens 128] [--reps 3]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power, "sm_max_clock": clock}
    except (OSError, IndexError, ValueError, subprocess.TimeoutExpired):
        return {"gpu": torch.cuda.get_device_name(0), "power_limit": None, "sm_max_clock": None}


def hbm_peak():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        return float(json.loads(p.read_text())["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "H100 SXM data sheet (3.35 TB/s HBM3)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--total-len", type=int, default=2048)
    ap.add_argument("--rollouts", type=int, default=32)
    ap.add_argument("--rollout-tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tl.py measures the GPU; no CUDA device found")
    from detikzify_b200.model import load
    from oracle.hf_oracle import synthetic_pixels

    R = args.rollouts
    model, _ = load("nllg/detikzify-tl-1.1b", device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True,
                    max_seqs=R + 1, max_batch=R)
    cfg, eng = model.config, model.engine
    dev = torch.device("cuda:0")
    P = cfg.num_patches
    total = min(args.total_len, eng.max_len)
    n_new = total - P
    ids = torch.full((P,), cfg.patch_token_id, dtype=torch.int64, device=dev)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=1000).to(dev)
    greedy = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    nuc = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id, begin_suppress_token=-1, seed=3)
    slots = [eng.seq_alloc() for _ in range(R)]
    stream = torch.cuda.Stream(device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]

    def decode_run():
        img = eng.image_embeds(pix)[0]
        ev[0].record(stream)
        last, _ = eng.prefill(slots[0], ids, 0, img, 0)
        ev[1].record(stream)
        first, _ = eng.sample(last, greedy, suppress=[0])
        eng.gen_begin([slots[0]], [P], [int(first.item())], greedy)
        ev[2].record(stream)
        for _ in range(n_new - 1):
            eng.gen_step()
        ev[3].record(stream)
        eng.gen_wait(n_new - 2)
        eng.gen_end()
        stream.synchronize()
        return ev[0].elapsed_time(ev[1]), ev[2].elapsed_time(ev[3])

    def rollout_run():
        for sl in slots[1:]:
            eng.seq_share(slots[0], sl, 0)        # drop the previous prefix loan
        ev[0].record(stream)
        img = eng.image_embeds(pix)[0]
        last, _ = eng.prefill(slots[0], ids, 0, img, 0)
        for sl in slots[1:]:
            eng.seq_share(slots[0], sl, P)        # rollouts read the image prefix from slot 0
        first, _ = eng.sample(last[None].expand(R, -1).contiguous(), nuc, suppress=[0] * R, steps=[0] * R, seq_ids=list(range(R)))
        eng.gen_begin(slots, [P] * R, [int(t) for t in first.tolist()], nuc, list(range(R)))
        for _ in range(args.rollout_tokens - 1):
            eng.gen_step()
        eng.gen_wait(args.rollout_tokens - 2)
        eng.gen_end()
        ev[1].record(stream)
        stream.synchronize()
        return ev[0].elapsed_time(ev[1])

    with torch.cuda.stream(stream):
        decode_run()                              # warm-up: module load, graph capture
        runs = [decode_run() for _ in range(args.reps)]
        rollout_run()
        rolls = [rollout_run() for _ in range(args.reps)]
    for s in reversed(slots):                   # borrowers before the lender
        eng.seq_free(s)

    peak, peak_src = hbm_peak()
    # decode step s (s = 1 .. n_new - 1) appends the token at position P + s and reads P + s + 1 cached positions
    bytes_dec = sum(eng.decode_bytes(P + 1 + i) for i in range(n_new - 1))
    dec_ms = sorted(r[1] for r in runs)[len(runs) // 2]
    pre_ms = sorted(r[0] for r in runs)[len(runs) // 2]
    roll_ms = sorted(rolls)[len(rolls) // 2]
    gbs = bytes_dec / (dec_ms * 1e-3) / 1e9
    print(json.dumps({
        "model": "nllg/detikzify-tl-1.1b", **gpu_info(),
        "decode": {"tokens": n_new - 1, "ctx": [P + 1, total - 1], "ms": dec_ms, "tok_s": (n_new - 1) / (dec_ms * 1e-3),
                   "ms_per_token": dec_ms / (n_new - 1), "achieved_gbs": gbs, "hbm_fraction": gbs / peak, "hbm_peak_gbs": peak,
                   "hbm_peak_source": peak_src, "persistent_kernel": eng.get_option("decode_persistent"),
                   "all_ms": [r[1] for r in runs]},
        "prefill_ms": pre_ms,
        "rollouts": {"n": R, "new_tokens": args.rollout_tokens, "ms": roll_ms,
                     "tok_s": R * args.rollout_tokens / (roll_ms * 1e-3), "all_ms": rolls},
    }))


if __name__ == "__main__":
    main()
