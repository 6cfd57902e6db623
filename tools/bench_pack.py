"""
Packed decoder weights (engine option ``decode_pack``, on by default in ``load()``) against bf16 tiles on one GPU. Prints ONE
JSON line per shape.

For each of ds-1.3b, tl-1.1b, ds-7b and v2-8b, with ``device_init`` weights, on one engine ``decode_pack`` alternates 0 / 1,
--reps runs each: batch-1 greedy decode from the image prefix to --total-len in the device-resident loop (persistent kernel +
fused argmax), tok/s and ms/token over CUDA-event time (median), the streamed bytes per token (``Engine.decode_bytes``: the
weights as the current mode streams them, plus the cached keys/values) and their fraction of the HBM peak (MEASURED_PEAKS.json,
else the H100 SXM data sheet's 3.35 TB/s), whether both modes ended on the same greedy token, the time of one pack and one bf16
re-tile, the escape-tile count; ds-7b also at context 512 (64 steps from a 512-token prefill); the card's name and power limit,
read in the same run.
    python tools/bench_pack.py [--shapes ds-1.3b,tl-1.1b,ds-7b,v2-8b] [--total-len 2048] [--reps 3]
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_tl import gpu_info, hbm_peak  # noqa: E402

SHAPES = {"ds-1.3b": "nllg/detikzify-ds-1.3b", "tl-1.1b": "nllg/detikzify-tl-1.1b", "ds-7b": "nllg/detikzify-ds-7b",
          "v2-8b": "nllg/detikzify-v2-8b"}


def bench_shape(key, args, peak, peak_src):
    from detikzify_b200.model import load
    from oracle.hf_oracle import synthetic_pixels

    model, _ = load(SHAPES[key], device_map=0, torch_dtype=torch.bfloat16, seed=0, device_init=True, max_seqs=2, max_batch=1)
    cfg, eng = model.config, model.engine
    dev = torch.device("cuda:0")
    P = cfg.num_patches
    total = min(args.total_len, eng.max_len)
    n_new = total - P
    img_ids = torch.full((P,), cfg.patch_token_id, dtype=torch.int64, device=dev)
    pix = synthetic_pixels(1, cfg.vision_config.image_size, seed=1000).to(dev)
    greedy = eng.sampling(do_sample=False, bad_token=cfg.image_token_id, begin_suppress_token=-1)
    slot = eng.seq_alloc()
    stream = torch.cuda.Stream(device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    g = torch.Generator().manual_seed(9000)
    text = torch.randint(3, 30000, (512,), generator=g).to(dev)

    with torch.cuda.stream(stream):
        pack_ms = {}
        for mode in (0, 1):   # load() packed the tiles already: time one rebuild of each format
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.set_option("decode_pack", mode)
            pack_ms[mode] = (time.perf_counter() - t0) * 1e3
        escapes = eng.get_option("decode_pack_escapes")

        def decode_run():
            img = eng.image_embeds(pix)[0]
            last, _ = eng.prefill(slot, img_ids, 0, img, 0)
            first, _ = eng.sample(last, greedy, suppress=[0])
            eng.gen_begin([slot], [P], [int(first.item())], greedy)
            ev[0].record(stream)
            for _ in range(n_new - 1):
                eng.gen_step()
            ev[1].record(stream)
            last_tok = eng.gen_wait(n_new - 2)[0]
            eng.gen_end()
            stream.synchronize()
            return ev[0].elapsed_time(ev[1]), last_tok

        def ctx512_run(steps=64):
            last, _ = eng.prefill(slot, text, 0, None, 0)
            first, _ = eng.sample(last, greedy, suppress=[0])
            eng.gen_begin([slot], [text.numel()], [int(first.item())], greedy)
            ev[0].record(stream)
            for _ in range(steps):
                eng.gen_step()
            ev[1].record(stream)
            eng.gen_wait(steps - 1)
            eng.gen_end()
            stream.synchronize()
            return ev[0].elapsed_time(ev[1]) / steps

        runs, runs512, ids = {0: [], 1: []}, {0: [], 1: []}, {}
        for mode in (0, 1):                   # warm-up of both modes
            eng.set_option("decode_pack", mode)
            decode_run()
        for _ in range(args.reps):
            for mode in (0, 1):
                eng.set_option("decode_pack", mode)
                ms, ids[mode] = decode_run()
                runs[mode].append(ms)
                if key == "ds-7b":
                    runs512[mode].append(ctx512_run())
        out = {"shape": key, "model": SHAPES[key], **gpu_info(), "persistent_kernel": eng.get_option("decode_persistent"),
               "pack_ms": pack_ms[1], "bf16_retile_ms": pack_ms[0], "escape_tiles": escapes,
               "same_last_token": ids[0] == ids[1], "hbm_peak_gbs": peak, "hbm_peak_source": peak_src}
        for mode, name in ((0, "bf16"), (1, "packed")):
            eng.set_option("decode_pack", mode)
            # decode step s (s = 1 .. n_new - 1) appends the token at position P + s and reads P + s + 1 cached positions
            bytes_dec = sum(eng.decode_bytes(P + 1 + i) for i in range(n_new - 1))
            ms = sorted(runs[mode])[len(runs[mode]) // 2]
            gbs = bytes_dec / (ms * 1e-3) / 1e9
            out[name] = {"tokens": n_new - 1, "ctx": [P + 1, total - 1], "ms": ms, "tok_s": (n_new - 1) / (ms * 1e-3),
                         "ms_per_token": ms / (n_new - 1), "bytes_per_token": bytes_dec / (n_new - 1),
                         "weight_bytes": eng.get_option("decode_weight_bytes"), "achieved_gbs": gbs, "hbm_fraction": gbs / peak,
                         "all_ms": runs[mode]}
            if runs512[mode]:
                ms512 = sorted(runs512[mode])[len(runs512[mode]) // 2]
                b512 = eng.decode_bytes(text.numel() + 32)
                out[name]["ctx512"] = {"ms_per_token": ms512, "tok_s": 1e3 / ms512, "bytes_per_token": b512,
                                       "hbm_fraction": b512 / (ms512 * 1e-3) / 1e9 / peak, "all_ms": runs512[mode]}
        out["speedup_tok_s"] = out["packed"]["tok_s"] / out["bf16"]["tok_s"]
        if key == "ds-7b":
            out["speedup_ctx512"] = out["packed"]["ctx512"]["tok_s"] / out["bf16"]["ctx512"]["tok_s"]
    eng.seq_free(slot)
    eng.close()
    del model, eng
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="ds-1.3b,tl-1.1b,ds-7b,v2-8b")
    ap.add_argument("--total-len", type=int, default=2048)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pack.py measures the GPU; no CUDA device found")
    peak, peak_src = hbm_peak()
    for key in args.shapes.split(","):
        print(json.dumps(bench_shape(key, args, peak, peak_src)), flush=True)


if __name__ == "__main__":
    main()
