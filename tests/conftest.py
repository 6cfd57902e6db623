import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope="session", autouse=True)
def _built_library():
    """Make sure the in-tree C-ABI library exists (nvcc cross-compiles on CPU boxes)."""
    from detikzify_b200 import build
    if not build.LIB.exists():
        build.build()
    return build.LIB


_CACHE = {}


def model_bundle(name: str, seed: int = 0, lm_head_std: float = 0.02):
    """(cfg, canonical state dict, fp32 oracle) — cached per session."""
    key = (name, seed, lm_head_std)
    if key not in _CACHE:
        from detikzify_b200.model.configuration import preset
        from detikzify_b200.model.weights import random_init
        from oracle.hf_oracle import Oracle
        cfg = preset(name)
        sd = random_init(cfg, seed=seed, lm_head_std=lm_head_std)
        _CACHE[key] = (cfg, sd, Oracle(cfg.to_dict(), sd))
    return _CACHE[key]


_ENGINES = {}


def engine_for(name: str, seed: int = 0, lm_head_std: float = 0.02, max_seqs: int = 4, max_batch: int = 4):
    key = (name, seed, lm_head_std, max_seqs, max_batch)
    if key not in _ENGINES:
        from detikzify_b200.engine import Engine, pack_arena
        cfg, sd, _ = model_bundle(name, seed, lm_head_std)
        _ENGINES[key] = Engine(cfg, pack_arena(cfg, sd), device=0, max_seqs=max_seqs, max_batch=max_batch)
    return _ENGINES[key]
