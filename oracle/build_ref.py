"""
Recipe for ``oracle/_ref/``: the reference implementation's own driver modules, byte-compiled so that the drop-in tests can
execute them unmodified on top of this package's objects. Nothing of the reference is kept in the repository: ``build()``
runs this recipe where a reference checkout is available: the directory named by ``DETIKZIFY_REFERENCE``, else the nearest
checkout called ``reference`` next to this repository or next to one of the directories that enclose it (a work tree or a
test clone usually sits somewhere below the directory that holds both). Byte code is specific to the Python version that wrote it; the tests skip
where ``oracle/_ref/`` was not built or was built by another version.
"""
from __future__ import annotations

import os
import py_compile
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
OUT = ROOT / "oracle" / "_ref" / "detikzify"
MODULES = [
    "mcts/node.py", "mcts/montecarlo.py", "util/functools.py", "util/generation.py", "util/torch.py",
    "evaluate/imagesim.py", "infer/generate.py", "model/v1/processing_detikzify.py",
]


def build_ref(reference: str | os.PathLike | None = None) -> Path | None:
    """Byte-compile the reference modules into ``oracle/_ref/detikzify``; returns None when there is no reference checkout."""
    given = reference or os.environ.get("DETIKZIFY_REFERENCE")
    roots = [Path(given)] if given else [d / "reference" for d in ROOT.parents]
    src = next((r / "detikzify" for r in roots if (r / "detikzify").is_dir()), None)
    if src is None:
        return None
    for rel in MODULES:
        dst = (OUT / rel).with_suffix(".pyc")
        dst.parent.mkdir(parents=True, exist_ok=True)
        py_compile.compile(str(src / rel), cfile=str(dst), dfile=f"detikzify/{rel}", doraise=True)
    return OUT


if __name__ == "__main__":
    import sys
    print(build_ref(sys.argv[1] if len(sys.argv) > 1 else None))
