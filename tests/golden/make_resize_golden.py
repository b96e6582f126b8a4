"""Generates tests/golden/resize_golden.npz: the small cases of tests/test_oracle_resize.py and what python-cv2 (here 4.13.0) makes of them:
cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR), the call System::TrackRGBD / System::TrackStereo make when Settings::needToResize().
Run from the repo root."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_oracle_resize as T   # noqa: E402

out = {}
for name, src, dw, dh in T.cases():
    if src.size <= T.GOLD_MAX_PIXELS:
        out[name + "_src"], out[name + "_cv2"] = src, T.cv2_resize(src, dw, dh)
np.savez_compressed(T.GOLD, **out)
print(T.GOLD, T.GOLD.stat().st_size, "bytes,", len(out), "arrays")
