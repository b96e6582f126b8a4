"""Generates tests/golden/remap_golden.npz: the images and maps of tests/test_oracle_rectify.py and what python-cv2 (here 4.13.0) makes of
them: cv2.remap(src, mapx, mapy, cv2.INTER_LINEAR), the call System::TrackStereo makes to rectify a pair.  Run from the repo root."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_oracle_rectify as T   # noqa: E402

out = {}
for name, src, mx, my in T.cases():
    out[name + "_src"], out[name + "_mapx"], out[name + "_mapy"] = src, mx, my
    out[name + "_cv2"] = T.cv2_remap(src, mx, my)
np.savez_compressed(T.GOLD, **out)
print(T.GOLD, T.GOLD.stat().st_size, "bytes,", len(out), "arrays")
