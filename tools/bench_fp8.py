"""
FP8 decoder weights (engine option ``decode_fp8``) against bf16 on one GPU. Prints ONE JSON line per shape.

For each of ds-1.3b, tl-1.1b, ds-7b and v2-8b, with ``device_init`` weights:
  * the teacher-forced logits of a 512-token prefill are taken with the original bf16 weights;
  * the arena's four decoder-layer matrices are then quantized in place exactly as ``load(..., quantize="fp8")`` does, and
    the same prefill is repeated: KL(original || fp8) per position (mean and max) and the top-1 agreement are reported.
    The weights are random, so these two numbers say nothing about a real checkpoint;
  * on that one engine ``decode_fp8`` alternates 0 / 1, --reps runs each: batch-1 greedy decode from the image prefix to
    --total-len in the device-resident loop (persistent kernel + fused argmax), tok/s and ms/token over CUDA-event time,
    the streamed bytes per token (``Engine.decode_bytes``: the weights as the current mode streams them, plus the cached
    keys/values) and their fraction of the HBM peak (MEASURED_PEAKS.json, else the H100 SXM data sheet's 3.35 TB/s);
  * ds-7b also at context 512 (64 steps from a 512-token prefill);
  * the one-time re-tile time of each direction, and the card's name and power limit, read in the same run.
    python tools/bench_fp8.py [--shapes ds-1.3b,tl-1.1b,ds-7b,v2-8b] [--total-len 2048] [--reps 3]
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


def kl_top1(ref: torch.Tensor, got: torch.Tensor):
    lp, lq = torch.log_softmax(ref.double(), -1), torch.log_softmax(got.double(), -1)
    kl = (lp.exp() * (lp - lq)).sum(-1)
    return kl.mean().item(), kl.max().item(), (ref.argmax(-1) == got.argmax(-1)).double().mean().item()


def bench_shape(key, args, peak, peak_src):
    from detikzify_b200.engine import weight_table
    from detikzify_b200.model import load
    from detikzify_b200.quant import quantize_arena_fp8
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
        ref = eng.prefill(slot, text, 0, None, 0, want_all_logits=True)[1].float().cpu()
        quantize_arena_fp8(eng.arena, weight_table(eng.ccfg))
        torch.cuda.synchronize()
        retile = {}
        for mode in (1, 0, 1):   # the first switch builds the fp8 tiles, then bf16 tiles of the quantized arena, then fp8
            t0 = time.perf_counter()
            eng.set_option("decode_fp8", mode)
            retile[mode] = (time.perf_counter() - t0) * 1e3
        got = eng.prefill(slot, text, 0, None, 0, want_all_logits=True)[1].float().cpu()
        kl_mean, kl_max, top1 = kl_top1(ref, got)
        del ref, got

        def decode_run():
            img = eng.image_embeds(pix)[0]
            last, _ = eng.prefill(slot, img_ids, 0, img, 0)
            first, _ = eng.sample(last, greedy, suppress=[0])
            eng.gen_begin([slot], [P], [int(first.item())], greedy)
            ev[0].record(stream)
            for _ in range(n_new - 1):
                eng.gen_step()
            ev[1].record(stream)
            eng.gen_wait(n_new - 2)
            eng.gen_end()
            stream.synchronize()
            return ev[0].elapsed_time(ev[1])

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

        runs = {0: [], 1: []}
        runs512 = {0: [], 1: []}
        for mode in (0, 1):                   # warm-up of both modes
            eng.set_option("decode_fp8", mode)
            decode_run()
        for _ in range(args.reps):
            for mode in (0, 1):
                eng.set_option("decode_fp8", mode)
                runs[mode].append(decode_run())
                if key == "ds-7b":
                    runs512[mode].append(ctx512_run())
        out = {"shape": key, "model": SHAPES[key], **gpu_info(), "persistent_kernel": eng.get_option("decode_persistent"),
               "kl_orig_fp8_mean": kl_mean, "kl_orig_fp8_max": kl_max, "top1_agreement": top1, "teacher_forced_tokens": 512,
               "retile_ms": {"fp8": retile[1], "bf16": retile[0]}, "hbm_peak_gbs": peak, "hbm_peak_source": peak_src}
        for mode, name in ((0, "bf16"), (1, "fp8")):
            eng.set_option("decode_fp8", mode)
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
        out["speedup_tok_s"] = out["fp8"]["tok_s"] / out["bf16"]["tok_s"]
        if key == "ds-7b":
            out["speedup_ctx512"] = out["fp8"]["ctx512"]["tok_s"] / out["bf16"]["ctx512"]["tok_s"]
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
        raise SystemExit("bench_fp8.py measures the GPU; no CUDA device found")
    peak, peak_src = hbm_peak()
    for key in args.shapes.split(","):
        print(json.dumps(bench_shape(key, args, peak, peak_src)), flush=True)


if __name__ == "__main__":
    main()
