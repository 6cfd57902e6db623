"""Dense-GEMM timing at the model shapes (mma.sync kernel vs the wgmma kernels) + ViT / prefill wall time per implementation.
Dev tool:  python tools/gemm_bench.py [model]"""
import ctypes as C, math, sys
import torch
sys.path.insert(0, ".")
from detikzify_b200 import _lib as L
from detikzify_b200.model import load

lib = L.load_library()
P = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
S = lambda: C.c_void_p(torch.cuda.current_stream().cuda_stream)
SHAPES = [  # (M, N, K, out_bf16, label)
    (729, 3456, 1152, True, "vit qkv B=1"), (729, 4304, 1152, True, "vit fc1 B=1"), (729, 1152, 4304, False, "vit fc2 B=1"),
    (5832, 3456, 1152, True, "vit qkv B=8"), (5832, 4304, 1152, True, "vit fc1 B=8"), (5832, 1152, 4304, False, "vit fc2 B=8"),
    (243, 6144, 2048, False, "llama qkv T=243"), (243, 11008, 2048, True, "llama gate/up T=243"), (243, 2048, 5504, False, "llama down T=243"),
    (2048, 6144, 2048, False, "llama qkv T=2048"), (2048, 11008, 2048, True, "llama gate/up T=2048"), (2048, 2048, 5504, False, "llama down T=2048"),
]
IMPLS = [int(v) for v in sys.argv[2].split(",")] if len(sys.argv) > 2 else [0, 1, 2]
ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
for M, N, K, obf, label in SHAPES:
    A = (torch.randn(M, K, device="cuda") * 0.5).bfloat16()
    W = (torch.randn(N, K, device="cuda") / math.sqrt(K)).bfloat16()
    out = torch.empty(M, N, device="cuda", dtype=torch.bfloat16 if obf else torch.float32)
    res = []
    for impl in IMPLS:
        lib.dtk_dbg_gemm_impl(impl)
        call = lambda: lib.dtk_dbg_gemm(P(A), P(W), P(None), P(None), M, N, K, 0, 0, P(None if obf else out), P(out if obf else None), S())
        for _ in range(3):
            call()
        torch.cuda.synchronize(); ev0.record()
        for _ in range(20):
            call()
        ev1.record(); torch.cuda.synchronize()
        us = ev0.elapsed_time(ev1) / 20 * 1e3
        res.append((us, 2.0 * M * N * K / us / 1e6))
    print(f"{label:24s} M={M:5d} N={N:5d} K={K:5d}  mma.sync {res[0][0]:8.1f} us {res[0][1]:7.1f} TF/s | wgmma 128x128 {res[1][0]:8.1f} us {res[1][1]:7.1f} TF/s | persistent {res[2][0]:8.1f} us {res[2][1]:7.1f} TF/s")

name = sys.argv[1] if len(sys.argv) > 1 else "nllg/detikzify-ds-1.3b"
model, _ = load(name, device_map=0)
eng, cfg = model.engine, model.config
from oracle.hf_oracle import synthetic_pixels
for impl in IMPLS:
    eng.set_option("gemm_impl", impl)
    for B in (1, 8, 32):
        pix = synthetic_pixels(B, cfg.vision_config.image_size).cuda()
        for _ in range(2):
            eng.vit_encode(pix)
        torch.cuda.synchronize(); ev0.record()
        for _ in range(5):
            eng.vit_encode(pix)
        ev1.record(); torch.cuda.synchronize()
        print(f"gemm_impl={impl} ViT B={B}: {ev0.elapsed_time(ev1) / 5 / B:.3f} ms/img")
    slot = eng.seq_alloc()
    for T in (243, 2047):
        ids = torch.randint(0, 30000, (T,), generator=torch.Generator().manual_seed(1)).cuda()
        for _ in range(2):
            eng.prefill(slot, ids, 0, None, 0)
        torch.cuda.synchronize(); ev0.record()
        for _ in range(5):
            eng.prefill(slot, ids, 0, None, 0)
        ev1.record(); torch.cuda.synchronize()
        print(f"gemm_impl={impl} prefill T={T}: {ev0.elapsed_time(ev1) / 5:.3f} ms")
    eng.seq_free(slot)
eng.set_option("gemm_impl", 0)
