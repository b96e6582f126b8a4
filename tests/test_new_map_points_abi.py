"""rgbl_create_new_map_points' argument checks: bad arguments return RGBL_E_INVALID before anything is written, whether or not a
device is present (the checks run before any CUDA call), and the ABI version counts the entry point."""
import ctypes as C

import numpy as np
import pytest

import new_map_points_cases as M
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F


def test_abi_version_counts_create_new_map_points():
    assert L.lib().rgbl_abi_version() >= 4


def _call(ctx_handle, case, **over):
    v1 = F.KeyFrameView(case["kf1"]); v2 = [F.KeyFrameView(k) for k in case["neighbours"]]
    for k, v in over.pop("kf1_fields", {}).items():
        setattr(v1.c, k, v)
    n = over.pop("n", len(v2))
    arr = (L.KeyFrameViewC * max(len(v2), 1))(*[v.c for v in v2])
    F12 = np.ascontiguousarray(case["F12"], np.float32); ep = np.ascontiguousarray(case["ep"], np.float32)
    start = np.full(len(v2) + 1, -7, np.int32); nm = np.full(max(len(v2), 1), -7, np.int32)
    cap = len(v1.desc)
    i1 = np.full(cap, -7, np.int32); i2 = np.full(cap, -7, np.int32); x = np.full((cap, 3), -7, np.float32)
    a = dict(n_levels=M.N_LEVELS, fx=M.FX, cap=cap, start=L.ptr(start))
    a.update(over)
    rc = L.lib().rgbl_create_new_map_points(ctx_handle, C.byref(v1.c), n, arr, L.ptr(F12), L.ptr(ep), a["fx"], M.FY, M.CX, M.CY, M.BF, a["n_levels"],
                                            L.ptr(M.SF), L.ptr(M.SG), 0.0, 0, 0, a["start"], L.ptr(i1), L.ptr(i2), L.ptr(x), a["cap"], L.ptr(nm))
    untouched = (start == -7).all() and (nm == -7).all() and (i1 == -7).all() and (i2 == -7).all() and (x == -7).all()
    return rc, untouched


@pytest.fixture(scope="module")
def handle(have_gpu):
    if not have_gpu:
        yield None
        return
    c = F.Context(M.W, M.H, 2000)
    yield c.handle
    c.close()


def _bad_octave(case):
    case["kf1"]["keys_un"]["octave"][0] = M.N_LEVELS
    return case


def _bad_feat(case):
    ids, start, feat = case["neighbours"][0]["fv"]
    feat = feat.copy(); feat[0] = len(case["neighbours"][0]["desc"])
    case["neighbours"][0]["fv"] = (ids, start, feat)
    return case


def _bad_pose(case):
    case["neighbours"][1]["Tcw"] = case["neighbours"][1]["Tcw"].copy()
    case["neighbours"][1]["Tcw"][5] = np.nan
    return case


@pytest.mark.parametrize("what", ["levels_low", "levels_high", "negative_n", "null_start", "null_desc", "octave", "feature_index", "pose", "fx",
                                  "negative_cap"])
def test_invalid_arguments(handle, what):
    c = M.case_claimed()
    over = {}
    if what == "levels_low":
        over["n_levels"] = 1
    elif what == "levels_high":
        over["n_levels"] = 17
    elif what == "negative_n":
        over["n"] = -1
    elif what == "null_start":
        over["start"] = None
    elif what == "null_desc":
        over["kf1_fields"] = {"desc": None}
    elif what == "octave":
        c = _bad_octave(c)
    elif what == "feature_index":
        c = _bad_feat(c)
    elif what == "pose":
        c = _bad_pose(c)
    elif what == "fx":
        over["fx"] = float("inf")
    elif what == "negative_cap":
        over["cap"] = -1
    if handle is None:
        # without a device the library refuses every context; the null-context check is the first one and also returns RGBL_E_INVALID
        rc, untouched = _call(None, c, **over)
    else:
        rc, untouched = _call(handle, c, **over)
    assert rc == L.RGBL_E_INVALID and untouched
