"""Streaming-primitive microbenchmark (dev tool).

Builds tools/csrc/stream_bench.cu into tools/libdtk_dev.so (NOT part of the product library) and measures
how fast persistent CTAs pull a large buffer from HBM: chip-wide, and per SM when only `grid` CTAs run
(the per-SM ingest cap decides how much of a stall a CTA of the decode kernel can make up later).
`python tools/stream_bench.py build` only compiles (works without a GPU)."""
import ctypes as C, subprocess, sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
LIB = ROOT / "libdtk_dev.so"


def build():
    src = ROOT / "csrc" / "stream_bench.cu"
    if LIB.exists() and LIB.stat().st_mtime > src.stat().st_mtime:
        return LIB
    cmd = ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
           "-shared", "-Xcompiler", "-fPIC", "-o", str(LIB), str(src)]
    subprocess.run(cmd, check=True)
    return LIB


if __name__ == "__main__":
    build()
    if len(sys.argv) > 1 and sys.argv[1] == "build":
        sys.exit(0)
    import torch
    lib = C.CDLL(str(LIB))
    lib.dtk_dbg_stream_bench.restype = C.c_int
    lib.dtk_dbg_stream_bench.argtypes = [C.c_void_p, C.c_uint64] + [C.c_int] * 8 + [C.c_void_p, C.c_void_p]
    nbytes = 3 * 2**30
    buf = torch.empty(nbytes, dtype=torch.uint8, device="cuda").random_(0, 255)
    sink = torch.zeros(4, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(mode, chunk, nslots, ncw, npw, read, hint, grid=132, iters=5, nb=nbytes):
        args = (C.c_void_p(buf.data_ptr()), nb, mode, chunk, nslots, ncw, npw, read, hint, grid, C.c_void_p(sink.data_ptr()), s)
        rc = lib.dtk_dbg_stream_bench(*args)
        assert rc == 0, rc
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            lib.dtk_dbg_stream_bench(*args)
        e1.record(); torch.cuda.synchronize()
        return nb * iters / (e0.elapsed_time(e1) * 1e-3) / 1e9

    quick = len(sys.argv) > 1 and sys.argv[1] == "quick"
    print("per-SM ingest when only `grid` CTAs stream (GB/s total | GB/s per SM):")
    for grid in (1, 2, 8, 32, 66, 99, 132):
        nb = min(nbytes, grid * 96 * 2**20)
        row = [f"grid {grid:3d}:"]
        for label, a in (("tma 8K x24 p4", (0, 8192, 24, 8, 4, 1, 0)), ("tma 8K x24 p8", (0, 8192, 24, 8, 8, 1, 0)),
                         ("tma 16K x12 p4", (0, 16384, 12, 4, 4, 1, 0)), ("tma 32K x6 p2", (0, 32768, 6, 2, 2, 1, 0)),
                         ("ldg 16 warps", (1, 8192, 1, 16, 0, 0, 0)), ("ldg 8 warps", (1, 8192, 1, 8, 0, 0, 0))):
            v = run(*a, grid=grid, nb=nb)
            row.append(f"{label} {v:7.0f} | {v / grid:6.1f}")
        print("  " + "   ".join(row), flush=True)
    if quick:
        sys.exit(0)
    print("LDG all warps:")
    for chunk in (4096, 8192, 16384):
        for warps in (8, 12, 16):
            print(f"  chunk {chunk:6d} warps {warps:2d}: {run(1, chunk, 1, warps, 0, 0, 0):7.0f} GB/s")
    print("TMA bulk ring:")
    for chunk, nslots in ((4096, 32), (4096, 48), (8192, 16), (8192, 24), (16384, 8), (16384, 12), (32768, 4), (32768, 6), (65536, 3)):
        for ncw, npw in ((8, 4), (4, 4), (8, 1), (8, 8)):
            if nslots % ncw or nslots % npw:
                continue
            for read in (0, 1):
                for hint in (0, 1):
                    print(f"  chunk {chunk:6d} slots {nslots:2d} ({chunk*nslots//1024:3d} KB) ncw {ncw} npw {npw} read {read} hint {hint}: {run(0, chunk, nslots, ncw, npw, read, hint):7.0f} GB/s")
