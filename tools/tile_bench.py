"""Tile-loop microbenchmark (dev tool): cycles per 8 KB tile per warp and bytes/clk per SM for the consumer side of
the decode kernel, by variant (bit 0: 128-bit LDS of fragment-ordered tiles instead of ldmatrix; bit 1: four accumulator
chains instead of two; bit 2: no per-tile bookkeeping; bit 3: no mma). `python tools/tile_bench.py build` only compiles."""
import ctypes as C, subprocess, sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
LIB = ROOT / "libdtk_tile.so"


def build():
    src = ROOT / "csrc" / "tile_bench.cu"
    if LIB.exists() and LIB.stat().st_mtime > src.stat().st_mtime:
        return LIB
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
                    "-shared", "-Xcompiler", "-fPIC", "-o", str(LIB), str(src)], check=True)
    return LIB


if __name__ == "__main__":
    build()
    if len(sys.argv) > 1 and sys.argv[1] == "build":
        sys.exit(0)
    import torch
    lib = C.CDLL(str(LIB))
    lib.dtk_dbg_tile_bench.restype = C.c_int
    lib.dtk_dbg_tile_bench.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    out = torch.zeros(4, device="cuda")
    cyc = torch.zeros(132, dtype=torch.int64, device="cuda")
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    iters, nslots = 4000, 24
    names = {0: "ldmatrix, 2 chains, bookkeeping (decode kernel today)", 1: "LDS.128 fragments, 2 chains, bookkeeping",
             2: "ldmatrix, 4 chains, bookkeeping", 3: "LDS.128, 4 chains, bookkeeping", 4: "ldmatrix, 2 chains, no bookkeeping",
             5: "LDS.128, 2 chains, no bookkeeping", 6: "ldmatrix, 4 chains, no bookkeeping", 7: "LDS.128, 4 chains, no bookkeeping",
             8: "ldmatrix, NO mma, bookkeeping", 9: "LDS.128, NO mma, bookkeeping", 12: "ldmatrix, NO mma, no bookkeeping",
             13: "LDS.128, NO mma, no bookkeeping", 16: "TWO tiles interleaved per warp iteration, bookkeeping",
             20: "TWO tiles interleaved per warp iteration, no bookkeeping"}
    for grid in (132,):
        print(f"grid {grid}:")
        for v, nm in names.items():
            for _ in range(2):
                rc = lib.dtk_dbg_tile_bench(v, iters, nslots, grid, C.c_void_p(out.data_ptr()), C.c_void_p(cyc.data_ptr()), s)
                assert rc == 0, rc
                torch.cuda.synchronize()
            c = cyc[:grid].double().mean().item()
            per_round = c / iters                      # one round = 8 tiles (one per warp)
            print(f"  var {v:2d} {nm:58s}: {per_round:7.1f} cycles per round of 8 tiles = {8 * 8192 / per_round:6.1f} B/clk/SM")
