"""Generates tests/golden/undistort_golden.npz: the points and distortion sets of tests/test_oracle_undistort.py and what python-cv2 (here
4.13.0) makes of them: cv2.undistortPoints(points, K, dist, None, K), the call of Frame::UndistortKeyPoints.  Run from the repo root."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_oracle_undistort as T   # noqa: E402

out = {}
for name, dist in T.sets():
    xy = T.points(name, 4000)
    out[name + "_xy"] = xy
    out[name + "_dist"] = dist
    out[name + "_cv2"] = T.cv2_undistort(xy, dist)
np.savez_compressed(T.GOLD, **out)
print(T.GOLD, T.GOLD.stat().st_size, "bytes,", len(out), "arrays")
