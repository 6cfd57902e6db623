"""
Stores what the drop-in tests compare with when no reference checkout is at hand: the reference's own image processor and
its ImageSim ("emd" mode), executed from oracle/_ref (oracle/build_ref.py), on the test images of
tests/test_cpu_reference_dropin.py. Run:  python tests/golden/make_reference_dropin_golden.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import test_cpu_reference_dropin as t   # noqa: E402

assert t._ref_usable(), "build oracle/_ref first (oracle/build_ref.py)"
f1, f2, sim, self_sim = t.reference_emd_case()
attrs, pixels = t.reference_preprocess_case()
idx = t._pixel_sample(60000)
np.savez_compressed(t.GOLDEN, emd_f1=f1.float().numpy(), emd_f2=f2.float().numpy(), emd_sim=np.float64(sim),
                    emd_self=np.float64(self_sim), proc_attrs=np.array(attrs, dtype=np.float64),
                    proc_pixels=np.stack([p.reshape(-1).numpy()[idx] for p in pixels]).astype(np.float32))
print(t.GOLDEN)
