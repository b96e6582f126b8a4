"""Generates tests/golden/colour_golden.npz: the colour images of tests/test_oracle_colour.py and what python-cv2 (here 4.13.0) makes of
them: cv2.resize / cv2.remap (INTER_LINEAR, BORDER_CONSTANT 0) of the colour image, then cv2.cvtColor to gray - what System::TrackRGBD /
TrackStereo and Tracking::GrabImage* do to a colour camera image.  Run from the repo root."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_oracle_colour as T   # noqa: E402

out = {}
for name, kind, img, arg, w0 in T.CASES:
    if img.shape[0] * img.shape[1] > T.GOLD_MAX_PIXELS:
        continue
    out[name + "_src"] = img
    out[name + "_cv2"] = T.cv2_result(kind, img, arg, w0)
np.savez_compressed(T.GOLD, **out)
print(T.GOLD, T.GOLD.stat().st_size, "bytes,", len(out), "arrays")
