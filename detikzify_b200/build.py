"""
In-tree build of the C-ABI CUDA library (``detikzify_b200/csrc/libdtk_b200.so``) for sm_90a.

nvcc cross-compiles without a GPU. Each ``.cu`` is compiled to an object in ``csrc/build/`` (parallel,
re-compiled only when the source or a header is newer) and linked into one shared library that exports
exactly the ``extern "C"`` symbols of ``include/detikzify_b200.h``.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent / "csrc"
ROOT = Path(__file__).resolve().parent.parent
LIB = CSRC / "libdtk_b200.so"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden",
          "-Xptxas", "-v", "-I", str(ROOT / "include")]


def sources():
    return sorted(CSRC.glob("*.cu"))


def headers():
    return sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted((ROOT / "include").glob("*.h"))


def _stale(target: Path, deps) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def _compile(src: Path, obj: Path, verbose: bool):
    cmd = [NVCC, *ARCH, *CFLAGS, "-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}\n")
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src.name}")
    (obj.with_suffix(".ptxas.txt")).write_text(r.stderr)
    return obj


def build(force: bool = False, verbose: bool = False) -> Path:
    bdir = CSRC / "build"
    bdir.mkdir(exist_ok=True)
    hdrs = headers()
    jobs, objs = [], []
    for src in sources():
        obj = bdir / (src.stem + ".o")
        objs.append(obj)
        if force or _stale(obj, [src, *hdrs]):
            jobs.append((src, obj))
    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(lambda j: _compile(j[0], j[1], verbose), jobs))
    if force or jobs or _stale(LIB, objs):
        tmp = LIB.with_suffix(".so.tmp")   # link beside the target and rename: a concurrent reader never sees a half-written library
        cmd = [NVCC, *ARCH, "-shared", "-o", str(tmp), *map(str, objs)]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
