"""Generates tests/golden/png16_golden.npz: the 16-bit depth PNG streams of tests/test_oracle_rgbd.py::cases and what python-cv2 (here
4.13.0, libpng) makes of them: cv2.imdecode(IMREAD_UNCHANGED).  Run from the repo root."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_oracle_rgbd as T   # noqa: E402

out = {}
for name, png in T.cases():
    out[name + "_png"] = np.frombuffer(png, np.uint8)
    out[name + "_depth"] = T.cv2_reference(png)
np.savez_compressed(T.GOLD, **out)
print(T.GOLD, T.GOLD.stat().st_size, "bytes,", len(out), "arrays")
