"""Phase-level timeline of the persistent decode kernel across all CTAs (dev tool).
Usage: python tools/mega_profile.py [--fp8 | --bf16] [model] [ctx] [trace.pt]  (the trace goes to the temporary directory by
default; the decode streams packed tiles as load() sets them up; --fp8: weights quantized as load(..., quantize="fp8") does,
decode on the FP8 layer tiles; --bf16: decode on bf16 tiles)."""
import ctypes as C, os, sys, tempfile
import torch
sys.path.insert(0, ".")
from detikzify_b200.model import load
fp8, bf16 = "--fp8" in sys.argv, "--bf16" in sys.argv
sys.argv = [a for a in sys.argv if a not in ("--fp8", "--bf16")]
name = sys.argv[1] if len(sys.argv) > 1 else "nllg/detikzify-ds-1.3b"
ctx = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
model, _ = load(name, device_map=0, quantize="fp8" if fp8 else None)
eng, cfg = model.engine, model.config
if bf16:
    eng.set_option("decode_pack", 0)
print(f"tile format: {'fp8' if eng.get_option('decode_fp8') else 'packed' if eng.get_option('decode_pack') else 'bf16'}")
slot = eng.seq_alloc()
g = torch.Generator().manual_seed(1)
ids = torch.randint(0, 30000, (ctx,), generator=g).cuda()
eng.prefill(slot, ids, 0, None, 0)
tok = torch.tensor([5], device="cuda")
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
def timeit(label):
    for _ in range(3):
        eng.decode([slot], [ctx], tok)
    torch.cuda.synchronize()
    ev0.record()
    for _ in range(10):
        eng.decode([slot], [ctx], tok)
    ev1.record(); torch.cuda.synchronize()
    print(f"{label}: ms/token {ev0.elapsed_time(ev1) / 10:.4f}")
import subprocess
print(subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.mem,power.draw,temperature.gpu,clocks_event_reasons.active", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
timeit("default")
for variant in (1, 0, 1, 0):
    eng.set_option("mega_variant", variant)
    timeit(f"variant={variant} (bit 0: weight copies without the evict_first L2 policy)")
    lgv = eng.decode([slot], [ctx], tok)[0].clone()
    if variant == 1:
        lg_ref = lgv
    print(f"   logits vs variant 1: max diff {(lgv - lg_ref).abs().max().item():.2e}")
for flags in (1, 2, 0):
    eng.set_option("mega_flags", flags)
    timeit(f"flags={flags} (1=no mma, 2=no waiting at all)")
print(subprocess.run(["nvidia-smi", "--query-gpu=name,clocks.sm,clocks.mem,power.draw,temperature.gpu,clocks_event_reasons.active", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
eng.set_option("mega_debug", 1)
eng.decode([slot], [ctx], tok)
L = cfg.num_hidden_layers
NP = L * 5 + 1
G = torch.cuda.get_device_properties(0).multi_processor_count   # the kernel runs one CTA per SM
n = G * NP * 4
buf = (C.c_longlong * n)()
got = eng.lib.dtk_dbg_mega_times(eng._h, buf, n)
G = got // (NP * 4)
t = torch.tensor(list(buf[:got]), dtype=torch.float64).view(G, NP, 4)
t0 = t[:, 0, 0].min()
names = ["qkv", "attn", "o", "gu", "down"]
print(f"kernel span: {(t[:, -1, 2].max() - t0).item() / 1e3:.1f} us  (G={G})")
for layer in (1, L // 2):
    print(f"layer {layer}: per phase over CTAs (us rel. to kernel start): start[min,max] staged[min,max] done[min,max] | mean(stage) mean(items) | n_active")
    for ph in range(5):
        d = t[:, layer * 5 + ph]
        act = (d[:, 2] - d[:, 1]) > 300  # CTAs that did work (ns)
        a = d[act] if act.any() else d
        f = lambda x: f"[{(x.min() - t0).item() / 1e3:8.2f},{(x.max() - t0).item() / 1e3:8.2f}]"
        print(f"  {names[ph]:5s} {f(a[:, 0])} {f(a[:, 1])} {f(a[:, 2])} | {(a[:, 1] - a[:, 0]).mean().item() / 1e3:6.2f} {(a[:, 2] - a[:, 1]).mean().item() / 1e3:6.2f} | {int(act.sum())}")
# slowest CTAs per phase kind (who finishes last), aggregated over layers
import collections
cnt = collections.Counter()
for layer in range(L):
    for ph in range(5):
        d = t[:, layer * 5 + ph, 2]
        cnt[int(d.argmax())] += 1
print("CTAs most often last to finish a phase:", cnt.most_common(12))


# ---- per-tile SM-clock trace of one layer: where does the weight stream stall?
TL = L // 2
eng.set_option("mega_trace_layer", TL)
eng.decode([slot], [ctx], tok)
ROWS = 168
buf2 = (C.c_longlong * (G * ROWS * 4))()
got = eng.lib.dtk_dbg_mega_trace(eng._h, buf2, G * ROWS * 4)
tr = torch.tensor(list(buf2[:got]), dtype=torch.float64).view(-1, ROWS, 4)
import os
out = sys.argv[3] if len(sys.argv) > 3 else os.path.join(tempfile.gettempdir(), "mega_trace.pt")
torch.save({"trace": tr, "phases": t, "layer": TL}, out)
MHZ = 1965.0
ntile = [24, 8, 40, 22] if "1.3b" in name else None
print(f"\nper-tile trace of layer {TL} (us, SM clock at {MHZ:.0f} MHz, relative to the CTA's own layer start stamp)")
print("columns per tile: issue(producer) landed asked done | landed-issue")
for cta in (0, 1, G // 3, 2 * G // 3, G - 1):
    d = tr[cta]
    t0c = d[160, 0]
    ph = (d[160:165] - t0c) / MHZ
    print(f"CTA {cta}: phase stamps start/staged/done/bar: " + " | ".join(" ".join(f"{v:6.2f}" for v in ph[i]) for i in range(5)))
    rows = [(i, d[i]) for i in range(160) if d[i, 1] > 0]
    for i, r in rows:
        v = (r - t0c) / MHZ
        print(f"   tile {i:3d}: issue {v[0]:7.2f} landed {v[1]:7.2f} asked {v[3]:7.2f} done {v[2]:7.2f} | fetch {v[1]-v[0]:6.2f} proc {v[2]-v[1]:5.2f}")
# aggregate: fetch latency distribution, and how many of a phase's tiles had landed before the phase was staged
lat = []
ready = collections.defaultdict(list)
for cta in range(tr.shape[0]):
    d = tr[cta]
    rows = [i for i in range(160) if d[i, 1] > 0]
    if not rows:
        continue
    for i in rows:
        if d[i, 0] > 0:
            lat.append(((d[i, 1] - d[i, 0]) / MHZ).item())
    # phase boundaries by consumer order: tiles are consumed in index order; assign phase by 'asked' time vs stamps
    for phi, stamp_row in ((0, 160), (2, 162), (3, 163), (4, 164)):
        staged = d[stamp_row, 1]
        nxt = d[stamp_row, 3]
        mine = [i for i in rows if d[i, 3] >= d[stamp_row, 0] and d[i, 3] <= nxt]
        if mine:
            # a tile was "already in the ring" if its issue time precedes the staged stamp by > 1 us
            ready[phi].append((sum(1 for i in mine if d[i, 0] > 0 and d[i, 0] < staged - 1.0 * MHZ), len(mine)))
lat = torch.tensor(lat)
print(f"fetch latency (issue -> consumer saw it), all CTAs: median {lat.median():.2f} us, p10 {lat.quantile(0.1):.2f}, p90 {lat.quantile(0.9):.2f}, max {lat.max():.2f}")
for phi, nm in ((0, "qkv"), (2, "o"), (3, "gu"), (4, "down")):
    if ready[phi]:
        a = torch.tensor(ready[phi], dtype=torch.float64)
        print(f"  {nm:5s}: tiles per CTA {a[:,1].mean():5.1f}; issued >1us before the phase was staged: {a[:,0].mean():5.1f}")
