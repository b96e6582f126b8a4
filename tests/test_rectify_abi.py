"""The stereo rectification entry point is part of the library's C ABI (declared in include/rgbl_b200.h and exported)."""
import ctypes as C

from orb_slam3_rgbl_b200 import _lib as L


def test_library_exports_the_rectification_entry_point():
    lib = C.CDLL(str(L.LIB_PATH))
    hdr = (L._PKG.parent / "include" / "rgbl_b200.h").read_text()
    name = "rgbl_set_stereo_rectification"
    assert hasattr(lib, name) and name in L.SYMBOLS and f"int {name}(" in hdr
