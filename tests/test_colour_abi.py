"""The colour-input entry point is part of the library's C ABI (declared in include/rgbl_b200.h, exported, bound in _lib.SYMBOLS), and
the ABI version counts it."""
import ctypes as C

from orb_slam3_rgbl_b200 import _lib as L


def test_library_exports_the_colour_input_entry_point():
    lib = C.CDLL(str(L.LIB_PATH))
    hdr = (L._PKG.parent / "include" / "rgbl_b200.h").read_text()
    name = "rgbl_set_input_channels"
    assert hasattr(lib, name) and name in L.SYMBOLS and f"int {name}(rgbl_ctx* ctx, int channels" in hdr
    assert L.SYMBOLS[name][1] == [C.c_void_p, C.c_int, C.c_int]


def test_abi_version_counts_the_colour_input():
    assert L.lib().rgbl_abi_version() >= 3
