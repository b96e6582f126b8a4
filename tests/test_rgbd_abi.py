"""The RGB-D entry points are part of the library's C ABI (they are declared in include/rgbl_b200.h and exported)."""
import ctypes as C

from orb_slam3_rgbl_b200 import _lib as L

RGBD_SYMBOLS = ("rgbl_resident_upload_rgbd", "rgbl_resident_upload_rgbd_png", "rgbl_decode_png_depth16", "rgbl_resident_process_rgbd",
                "rgbl_resident_stage_rgbd", "rgbl_track_sequence_rgbd")


def test_library_exports_the_rgbd_entry_points():
    lib = C.CDLL(str(L.LIB_PATH))
    hdr = (L._PKG.parent / "include" / "rgbl_b200.h").read_text()
    for name in RGBD_SYMBOLS:
        assert hasattr(lib, name) and name in L.SYMBOLS and f"int {name}(" in hdr, name
