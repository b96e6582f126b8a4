"""The stereo additions that need no GPU: the right camera's view of the synthetic plane sequence, and the stereo entry points of the C ABI."""
import ctypes as C
import hashlib

import numpy as np
import pytest

from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import synthetic as S

STEREO_SYMBOLS = ("rgbl_resident_upload_stereo", "rgbl_resident_upload_stereo_png", "rgbl_resident_process_stereo", "rgbl_resident_stage_stereo",
                  "rgbl_track_sequence_stereo")


def test_library_exports_the_stereo_entry_points():
    lib = C.CDLL(str(L.LIB_PATH))
    hdr = (L._PKG.parent / "include" / "rgbl_b200.h").read_text()
    for name in STEREO_SYMBOLS:
        assert hasattr(lib, name) and name in L.SYMBOLS and f"int {name}(" in hdr, name


@pytest.mark.parametrize("kw", [dict(), dict(loop=8), dict(shift_px=3, Z=10.0), dict(W=300, H=160, Z=12.5)])
def test_right_image_is_the_left_view_shifted_by_the_disparity(kw):
    seq = S.PlaneSequence(17, 9, **kw)
    d = seq.disparity_px()
    assert d == round(S.KITTI_BF / seq.Z)
    for t in range(9):
        left, right = seq.image(t), seq.right_image(t)
        assert right.shape == left.shape and right.dtype == np.uint8
        assert (right[:, :-d] == left[:, d:]).all()                 # right(x) = left(x + d)
        assert not (right == left).all()
        nxt = seq.texture[:, seq.step_index(t) * seq.shift + d:][:, :seq.W]
        assert (right == nxt).all()


def test_right_image_refuses_what_it_cannot_render():
    with pytest.raises(ValueError, match="slack"):
        S.PlaneSequence(3, 2, shift_px=1, Z=5.0).right_image(0)              # 20 px > shift_px + 8
    with pytest.raises(ValueError, match="whole-pixel"):
        S.PlaneSequence(3, 2, Z=30.0).right_image(0)                         # 3.33 px
    with pytest.raises(ValueError, match="pinhole"):
        S.PlaneSequence(3, 2, W=200, H=120, cam=(300.0, 300.0, 100.0, 60.0, 100.0), dist=S.TUM1_DIST).right_image(0)


# SHA-256 (first 32 hex digits) of image(0) .. image(n - 1) concatenated, as the previous release of synthetic.py rendered them
PARENT_IMAGE_DIGESTS = [
    (dict(seed=36, n=16), "1aa322637d3f961268db8146a2eb7d4c"),
    (dict(seed=21, n=3), "4dbd7fce16cef67fb5350380d84f09cf"),
    (dict(seed=41, n=9), "09819df007d3c93800e227bcd9bee985"),
    (dict(seed=9, n=2, W=300, H=160), "39c814bc7694fc032096fc9400500c03"),
    (dict(seed=2000, n=5, loop=8), "e37f6c580ead74c33309b342b89d20d3"),
    (dict(seed=61, n=4, shift_px=3, Z=10.0), "fc48205360df2cf2e74c27238425f891"),
]


@pytest.mark.parametrize("case,digest", PARENT_IMAGE_DIGESTS)
def test_left_images_are_unchanged(case, digest):
    kw = {k: v for k, v in case.items() if k not in ("seed", "n")}
    seq = S.PlaneSequence(case["seed"], case["n"], **kw)
    assert hashlib.sha256(b"".join(seq.image(t).tobytes() for t in range(case["n"]))).hexdigest()[:32] == digest
