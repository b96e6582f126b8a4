"""The camera-distortion entry points are part of the library's C ABI (they are declared in include/rgbl_b200.h and exported)."""
import ctypes as C

from orb_slam3_rgbl_b200 import _lib as L

UNDISTORT_SYMBOLS = ("rgbl_set_camera_distortion", "rgbl_resident_download_keys_un")


def test_library_exports_the_undistortion_entry_points():
    lib = C.CDLL(str(L.LIB_PATH))
    hdr = (L._PKG.parent / "include" / "rgbl_b200.h").read_text()
    for name in UNDISTORT_SYMBOLS:
        assert hasattr(lib, name) and name in L.SYMBOLS and f"int {name}(" in hdr, name
