"""
Cost of the sampler's HF logits processors (dtk_processors) on one GPU. Prints ONE JSON line.

  * sampler kernel time per call (torch.profiler device time, median over --reps calls) with the processors off
    (dtk_dbg_sample) and on (dtk_dbg_sample_proc: repetition penalty 1.3, no-repeat 3-gram, eight bad-word sequences, min-p
    0.05), sampling at T = 0.8 / top-p 0.95, at V = 32256 and 128256, B = 1 and 32, histories of 243 and 2048 ids;
  * batch-1 greedy ds-1.3b decode tok/s (random device weights, packed tiles as load() uses them, 243-token prompt, 512 new
    tokens in the device-resident loop) with the processors off (fused argmax in the persistent kernel) and on (the
    sampler kernel after every step), alternating, --reps runs each;
  * the card's name and power limit, read in the same run.
    python tools/bench_sampler.py [--reps 3]
"""
import argparse
import ctypes as C
import json
import statistics
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from bench_tl import gpu_info  # noqa: E402

PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_p=0.05, eos_token_id=2,
            words=[[11, 12], [13, 14, 15], [16, 17], [18, 19, 20, 21], [22, 23], [24, 25], [26, 27, 28], [29, 30]])


def sampler_times(V, B, L, reps):
    from detikzify_b200 import _lib
    from detikzify_b200.engine import Engine, c_histories, c_processors
    lib = _lib.load_library()
    rng = np.random.default_rng(0)
    logits = torch.tensor(rng.normal(0, 3, size=(B, V)).astype(np.float32), device="cuda")
    out = torch.empty(B, dtype=torch.int64, device="cuda")
    probs = torch.empty(B, V, dtype=torch.float32, device="cuda")
    params = Engine.sampling(temperature=0.8, top_p=0.95, do_sample=True, seed=1)
    hist = [rng.integers(0, 64, size=L).tolist() for _ in range(B)]
    ids, lens = c_histories(hist)
    proc = c_processors(**PROC)
    eml = (C.c_int32 * B)(*([0] * B))
    P = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731

    def off():
        assert lib.dtk_dbg_sample(P(logits), B, V, C.byref(params), None, None, None, 0, P(out), P(probs), None) == 0

    def on():
        assert lib.dtk_dbg_sample_proc(P(logits), B, V, C.byref(params), None, None, None, 0, C.byref(proc), ids, lens, eml,
                                       L, P(out), P(probs), None) == 0

    res = {}
    for name, fn in (("off", off), ("on", on)):
        fn()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
        ts = [e.device_time for e in prof.events() if "sample" in e.name and e.device_time > 0]
        res[name] = round(statistics.median(ts), 2)
    return res


def decode_tps(eng, cfg, prompt, new, proc):
    slot = eng.seq_alloc()
    try:
        last, _ = eng.prefill(slot, prompt, 0)
        params = eng.sampling(do_sample=False)
        hist = prompt.tolist()
        if proc:
            eng.set_processors(PROC, [hist], [0])
        first, _ = eng.sample(last, params, suppress=[1])
        tok = int(first)
        if proc:
            eng.set_processors(PROC, [hist + [tok]], [0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.gen_begin([slot], [len(hist)], [tok], params)
        launched = 0
        for i in range(new):
            while launched < i + 2 and launched < new:
                eng.gen_step()
                launched += 1
            last_tok = eng.gen_wait(i)[0]
        eng.gen_end()
        dt = time.perf_counter() - t0
    finally:
        eng.set_processors(None)
        eng.seq_free(slot)
    return new / dt, last_tok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    out = {"metric": "sampler_processors", **gpu_info(), "sampler_us": {}}
    for V in (32256, 128256):
        for B in (1, 32):
            for L in (243, 2048):
                out["sampler_us"][f"V{V}_B{B}_L{L}"] = sampler_times(V, B, L, 20)
    from detikzify_b200.engine import Engine, random_arena_device
    from detikzify_b200.model.configuration import preset
    cfg = preset("nllg/detikzify-ds-1.3b")
    eng = Engine(cfg, random_arena_device(cfg, 0), device=0, max_seqs=2, max_batch=1, max_len=2048)
    eng.set_option("decode_pack", 1)
    g = torch.Generator().manual_seed(0)
    prompt = torch.randint(3, 1000, (243,), generator=g).cuda()
    tps = {"off": [], "on": []}
    toks = {}
    for _ in range(args.reps):
        for mode in ("off", "on"):
            t, last = decode_tps(eng, cfg, prompt, 512, mode == "on")
            tps[mode].append(round(t, 1))
            toks[mode] = last
    out["ds13b_greedy_tok_s"] = tps
    out["ds13b_ratio_on_off"] = round(statistics.median(tps["on"]) / statistics.median(tps["off"]), 4)
    eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
