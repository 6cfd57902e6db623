"""Per-tile trace of one layer of the persistent decode kernel with every tagged-word wait skipped (dev flag 2): what one CTA
costs by itself when it never waits for another CTA (dev tool; the logits of such a run are garbage)."""
import ctypes as C, sys
import torch
sys.path.insert(0, ".")
from detikzify_b200.model import load
name = sys.argv[1] if len(sys.argv) > 1 else "nllg/detikzify-ds-1.3b"
ctx = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
flags = int(sys.argv[3]) if len(sys.argv) > 3 else 2
model, _ = load(name, device_map=0)
eng, cfg = model.engine, model.config
slot = eng.seq_alloc()
ids = torch.randint(0, 30000, (ctx,), generator=torch.Generator().manual_seed(1)).cuda()
eng.prefill(slot, ids, 0, None, 0)
tok = torch.tensor([5], device="cuda")
L = cfg.num_hidden_layers
eng.set_option("mega_flags", flags)
eng.set_option("mega_debug", 1)
TL = L // 2
eng.set_option("mega_trace_layer", TL)
for _ in range(3):
    eng.decode([slot], [ctx], tok)
torch.cuda.synchronize()
props = torch.cuda.get_device_properties(0)
ROWS, G, MHZ = 168, props.multi_processor_count, props.clock_rate / 1e3   # one CTA per SM; SM clock at its maximum
buf2 = (C.c_longlong * (G * ROWS * 4))()
got = eng.lib.dtk_dbg_mega_trace(eng._h, buf2, G * ROWS * 4)
tr = torch.tensor(list(buf2[:got]), dtype=torch.float64).view(-1, ROWS, 4)
print(f"flags={flags}: per-tile trace of layer {TL} (us at {MHZ:.0f} MHz, relative to the CTA's layer start)")
for cta in (1, 50, 100):
    d = tr[cta]
    t0c = d[160, 0]
    ph = (d[160:165] - t0c) / MHZ
    print(f"CTA {cta}: phase stamps start/staged/done/bar: " + " | ".join(" ".join(f"{v:6.2f}" for v in ph[i]) for i in range(5)))
    for i in range(160):
        if d[i, 1] > 0:
            v = (d[i] - t0c) / MHZ
            print(f"   tile {i:3d}: issue {v[0]:7.2f} asked {v[3]:7.2f} got {v[1]:7.2f} done {v[2]:7.2f}")
dur = (tr[:, 164, 3] - tr[:, 160, 0]) / MHZ
print(f"layer duration per CTA: median {dur.median():.2f} us, min {dur.min():.2f}, max {dur.max():.2f}")
eng.set_option("mega_flags", 0)
