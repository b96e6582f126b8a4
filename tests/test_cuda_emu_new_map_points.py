"""rgbl_create_new_map_points through the whole library compiled over the CUDA-on-CPU shim (tests/cuda_emu): the search, triangulation
and ordered kernels run on a machine without a GPU, on a subset of tests/new_map_points_cases.py that still reaches every branch, and
equal the oracle bit for bit."""
import ctypes as C

import pytest

import new_map_points_cases as M
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F

CASES = M.emulated_cases()


@pytest.fixture(scope="module")
def ctx():
    so = C.CDLL(str(build.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "_lib", so)                 # frontend calls go to the emulated library for this module
    c = F.Context(160, 120, 200, nlevels=4)
    yield c
    c.close()
    mp.undo()


def test_subset_reaches_every_branch():
    tags = set()
    for c in CASES:
        tags |= M.tags(c, M.oracle_create(c))
    assert M.REQUIRED_TAGS - {"n1_strided"} <= tags, sorted(M.REQUIRED_TAGS - tags)


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_case_emulated(ctx, c):
    M.assert_same(M.run_device(ctx, c), M.oracle_create(c))


def test_one_neighbour_at_a_time_emulated(ctx):
    c = next(c for c in CASES if c["name"] == "claimed")
    whole = M.run_device(ctx, c)
    kf1 = dict(c["kf1"]); kf1["has_mp"] = c["kf1"]["has_mp"].copy()
    for j in range(len(c["neighbours"])):
        part = dict(c, kf1=kf1, neighbours=c["neighbours"][j:j + 1], F12=c["F12"][j:j + 1], ep=c["ep"][j:j + 1])
        r = M.run_device(ctx, part)
        a, b = whole["created_start"][j], whole["created_start"][j + 1]
        assert (r["idx1"] == whole["idx1"][a:b]).all() and (r["idx2"] == whole["idx2"][a:b]).all()
        assert r["x3d"].tobytes() == whole["x3d"][a:b].tobytes() and r["n_matches"][0] == whole["n_matches"][j]
        kf1["has_mp"][r["idx1"]] = 1


def test_capacity_emulated(ctx):
    c = next(c for c in CASES if c["name"] == "claimed")
    total = int(M.oracle_create(c)["created_start"][-1])
    M.assert_same(M.run_device(ctx, c, cap=total), M.oracle_create(c))
    with pytest.raises(L.RgblError) as e:
        M.run_device(ctx, c, cap=total - 1)
    assert e.value.code == L.RGBL_E_CAPACITY
