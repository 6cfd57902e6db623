"""BASELINE.json configs[3] shape check (dev tool): detikzify-ds-7b random-init, (1) batch-1 decode: persistent kernel
vs per-op kernels (logits agreement, ms/token), (2) 32 parallel rollouts with nucleus sampling through the fused generation
loop (CUDA graph of per-op kernels): tokens/s, and batched-vs-single logits agreement."""
import sys, time
import torch
sys.path.insert(0, ".")
from detikzify_b200.model import load

name = "nllg/detikzify-ds-7b"
t0 = time.time()
model, _ = load(name, device_map=0, max_seqs=40, max_batch=32)
eng, cfg = model.engine, model.config
print(f"load {time.time() - t0:.1f}s; persistent={eng.get_option('decode_persistent')}", flush=True)
ctx = 512
ids = torch.randint(0, 30000, (ctx,), generator=torch.Generator().manual_seed(1)).cuda()
slots = [eng.seq_alloc() for _ in range(32)]
eng.prefill(slots[0], ids, 0, None, 0)
for s in slots[1:]:
    eng.seq_fork(slots[0], s, ctx)
tok = torch.tensor([5], device="cuda")
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
res = {}
for impl in (1, 0):
    eng.set_option("decode_impl", impl)
    for _ in range(3):
        lg = eng.decode([slots[0]], [ctx], tok)
    torch.cuda.synchronize(); ev0.record()
    for _ in range(10):
        lg = eng.decode([slots[0]], [ctx], tok)
    ev1.record(); torch.cuda.synchronize()
    res[impl] = lg[0].clone()
    ms = ev0.elapsed_time(ev1) / 10
    print(f"B=1 decode_impl={impl}: {ms:.3f} ms/token, {eng.decode_bytes(ctx) / ms / 1e6:.0f} GB/s", flush=True)
eng.set_option("decode_impl", 1)
print(f"persistent vs per-op logits max abs diff {(res[1] - res[0]).abs().max().item():.3e} (|logits| max {res[0].abs().max().item():.2f})")
toks = torch.full((32,), 5, device="cuda")
lgb = eng.decode(slots, [ctx] * 32, toks)
print(f"batched (B=32) row 0 vs single logits max abs diff {(lgb[0] - res[0]).abs().max().item():.3e}; rows identical: {bool((lgb[0] == lgb[31]).all())}")
params = eng.sampling(temperature=0.8, top_p=0.95, do_sample=True, bad_token=cfg.image_token_id, begin_suppress_token=-1, seed=3)
steps = 64
for rep in range(2):
    for i, s in enumerate(slots):
        pass
    eng.gen_begin(slots, [ctx + 1] * 32, [7] * 32, params)
    torch.cuda.synchronize(); t0 = time.time()
    for _ in range(steps):
        eng.gen_step()
    out = eng.gen_wait(steps - 1)
    dt = time.time() - t0
    eng.gen_end()
    print(f"32 rollouts x {steps} sampled tokens at ctx {ctx}..: {32 * steps / dt:.0f} tokens/s ({dt / steps * 1e3:.2f} ms/step), distinct last tokens {len(set(out))}", flush=True)

# ---- the same rollouts READING one shared prefix (dtk_seq_share): shared-prefix attention on / off
for s in slots:
    eng.seq_free(s)
base = eng.seq_alloc()
eng.prefill(base, ids, 0, None, 0)
slots = [eng.seq_alloc() for _ in range(32)]
for s in slots:
    eng.seq_share(base, s, ctx - 16)   # 496 positions shared, 16 copied
for cas in (1, 0, 1):
    eng.set_option("cascade_attn", cas)
    eng.gen_begin(slots, [ctx] * 32, [7] * 32, params)
    torch.cuda.synchronize(); t0 = time.time()
    for _ in range(steps):
        eng.gen_step()
    out = eng.gen_wait(steps - 1)
    dt = time.time() - t0
    eng.gen_end()
    print(f"shared prefix, cascade_attn={cas}: {32 * steps / dt:.0f} tokens/s ({dt / steps * 1e3:.2f} ms/step), distinct last tokens {len(set(out))}", flush=True)
