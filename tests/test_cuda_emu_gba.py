"""rgbl_global_bundle_adjustment and the tiled factorisation of ba_factor.cu run through the library compiled over the CUDA-on-CPU shim
(tests/cuda_emu; ba_factor.cuh's emulated build forms the FP64 mma.sync from warp shuffles in the PTX fragment layout, and
cuda_emu/emu_ba_factor.cpp compiles it into the library): a subset of gba_cases.py against the oracle, the solve export against numpy at the
tile edges, the argument and capacity refusals, and, with the oracle alone at full size, that every case reaches the path it exists for."""
import ctypes as C

import numpy as np
import pytest

import gba_cases as GC
import gba_dense_reference as GD
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L

EXPORT_NS = (1, 5, 63, 64, 65, 128, 129)


class EmuGBA:
    def __init__(self, path):
        self.so = C.CDLL(str(path))
        for name, (res, args) in L.SYMBOLS.items():
            fn = getattr(self.so, name)
            fn.restype, fn.argtypes = res, args
        self.so.rgbl_testing_reduced_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        cfg = L.Config(0, 160, 120, 1, 0, 0, L.OrbParams(200, 1.2, 4, 20, 7))
        self.h = C.c_void_p()
        assert self.so.rgbl_create(C.byref(cfg), C.byref(self.h)) == 0

    def raw(self, p, po, pt, it, stop=None):
        a = GC.args(p)
        return self.so.rgbl_global_bundle_adjustment(self.h, len(a[0]), L.ptr(a[0]), L.ptr(a[1]), len(a[2]), L.ptr(a[2]), len(a[3]), L.ptr(a[3]),
                                                     L.ptr(a[4]), L.ptr(a[5]), L.ptr(a[6]), L.ptr(a[7]), *a[8:], p["iterations"], int(p["robust"]),
                                                     stop, L.ptr(po), L.ptr(pt), C.byref(it))

    def __call__(self, p):
        po = np.empty_like(p["poses"]); pt = np.empty_like(p["points"]); it = C.c_int(-1)
        stop = np.array([1 if p["stop"] else 0], np.uint8)
        rc = self.raw(p, po, pt, it, L.ptr(stop))
        assert rc == 0, self.so.rgbl_last_error(self.h)
        return po, pt, it.value

    def solve(self, A, b, path):
        n = len(b); x = np.full(n, np.nan); st = np.full(1, -1, np.int32)
        A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
        assert self.so.rgbl_testing_reduced_solve(n, A.ctypes.data, b.ctypes.data, path, x.ctypes.data, st.ctypes.data) == 0
        return x, int(st[0])

    def close(self):
        self.so.rgbl_destroy(self.h)


@pytest.fixture(scope="module")
def emu():
    e = EmuGBA(build.build_full())
    yield e
    e.close()


CASES = GC.emulated_cases()


def spd(n, seed):
    rng = np.random.default_rng(seed)
    M = rng.normal(size=(n, n))
    A = M @ M.T + n * np.eye(n)
    return np.tril(A) + np.triu(rng.normal(size=(n, n)) * 1e3, 1), A, rng.normal(size=n)     # the upper triangle is never read


def test_subset_has_every_launch_shape():
    """One tile full / partial, several tiles with a full / partial last one, from the export; the graph reaches the tiled path."""
    shapes = {GC.tiled_shape(n) for n in EXPORT_NS}
    assert {("one_tile", "full"), ("one_tile", "partial"), ("tiles", "full"), ("tiles", "partial")} <= shapes
    assert any(GC.solver_path(int((c["problem"]["pose_fixed"] == 0).sum())) == "tiled" for c in CASES)


@pytest.mark.parametrize("n", EXPORT_NS)
def test_solve_export_emulated(emu, n):
    A_low, A, b = spd(n, n)
    ref = np.linalg.solve(A, b)
    for path in (1, 2):
        x, st = emu.solve(A_low, b, path)
        assert st == 0 and np.abs(x - ref).max() <= 1e-12 * np.abs(ref).max(), (n, path)


def test_solve_export_failing_pivot_emulated(emu):
    for n, bad in ((129, 128), (129, 3), (64, 63)):
        A = np.eye(n)
        A[bad, bad] = -1.0
        for path in (1, 2):
            x, st = emu.solve(A, np.ones(n), path)
            assert st == 1 and not x.any(), (n, bad, path)
        A[bad, bad] = 1.0
        A[bad, 0 if bad else 1] = np.nan
        x, st = emu.solve(A, np.ones(n), 2)
        assert st == 1 and not x.any(), (n, bad)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_gba_emulated(emu, c):
    ref = GC.reference(c["problem"])
    GC.check_coverage(c, ref[3])
    bar, d_pose, d_pt = GC.compare(c, emu(c["problem"]), ref)
    print(f"{c['name']}: {bar} bar, pose {d_pose:.1e}, point {d_pt:.1e}")


def test_refusals_leave_the_context_usable(emu):
    """Bad arguments: RGBL_E_INVALID; 4097 free poses: RGBL_E_CAPACITY with nothing written; a call after each works."""
    good = GC.stopped()[0]["problem"]
    p = GC.refused()
    po = np.full_like(p["poses"], 7.0); pt = np.full_like(p["points"], 7.0); it = C.c_int(-5)
    assert emu.raw(p, po, pt, it) == L.RGBL_E_CAPACITY
    assert (po == 7.0).all() and (pt == 7.0).all() and it.value == -5
    emu(good)
    bad = dict(good, e_point=good["e_point"].copy())
    bad["e_point"][0] = len(good["points"])
    po = np.empty_like(good["poses"]); pt = np.empty_like(good["points"])
    assert emu.raw(bad, po, pt, C.c_int(0)) == L.RGBL_E_INVALID
    assert emu.raw(dict(good, iterations=-1), po, pt, C.c_int(0)) == L.RGBL_E_INVALID
    assert emu.so.rgbl_global_bundle_adjustment(emu.h, 2, None, None, 0, None, 0, None, None, None, None, None, *GC.CAM, 1, 0, None, None, None,
                                                None) == L.RGBL_E_INVALID
    ref = GC.reference(good)
    GC.compare(GC.stopped()[0], emu(good), ref)


def test_families_reach_their_paths():
    """Through the oracle at full size: every case reaches what it exists for and is well-conditioned (gba_cases.sensitivity), both
    sides of the selection and of a tile multiple are present, and the dense one-step case is the oracle's own first step to 1e-6."""
    n_opt = set()
    for c in GC.all_cases():
        tr = GC.reference(c["problem"])[3]
        GC.check_coverage(c, tr)
        if c["problem"]["iterations"] and not c["expect"].get("unchanged"):
            assert GC.sensitivity(c["problem"]) < GC.SENSITIVITY, c["name"]
        n_opt.add(int((c["problem"]["pose_fixed"] == 0).sum()))
    assert {64, 65, 95, 96, 97, 200} <= n_opt
    c = GC.dense_case()
    po, pt, it, tr = GC.reference(c["problem"])
    GC.check_first_accepted(c, tr)
    GD.compare(c["problem"], po, pt)


def test_stop_flag_semantics_in_the_oracle():
    """Raised before the call: no iteration; not raised: the run goes on to the iteration limit or a stop test."""
    c = GC.stopped()[0]
    assert GC.reference(c["problem"])[2] == 0
    assert GC.reference(dict(c["problem"], stop=False))[2] > 0
