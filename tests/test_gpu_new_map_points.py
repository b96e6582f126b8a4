"""rgbl_create_new_map_points on the device against the CreateNewMapPoints oracle, bit for bit: every case of
tests/new_map_points_cases.py and 20 seeded scenes of about 2000 features and 10 neighbours; one call per neighbour with has_mp1
carried equals one call; the per-pair counts equal rgbl_search_for_triangulation with the carried has_mp1."""
import numpy as np
import pytest

import new_map_points_cases as M
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F

pytestmark = pytest.mark.gpu

CASES = M.all_cases()


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(M.W, M.H, 2000)
    yield c
    c.close()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_case(ctx, c):
    M.assert_same(M.run_device(ctx, c), M.oracle_create(c))


@pytest.mark.parametrize("seed", range(20))
def test_full_scene(ctx, seed):
    c = M.full_scene(seed)
    assert len(c["neighbours"]) == 10 and 1500 < len(c["kf1"]["desc"]) < 2600
    got, ref = M.run_device(ctx, c), M.oracle_create(c)
    M.assert_same(got, ref)
    assert ref["created_start"][-1] > 300


@pytest.mark.parametrize("seed", [0, 1])
def test_one_neighbour_at_a_time(ctx, seed):
    c = M.full_scene(seed)
    whole = M.run_device(ctx, c)
    kf1 = dict(c["kf1"]); kf1["has_mp"] = c["kf1"]["has_mp"].copy()
    for j in range(len(c["neighbours"])):
        part = dict(c, kf1=kf1, neighbours=c["neighbours"][j:j + 1], F12=c["F12"][j:j + 1], ep=c["ep"][j:j + 1])
        r = M.run_device(ctx, part)
        a, b = whole["created_start"][j], whole["created_start"][j + 1]
        assert np.array_equal(r["idx1"], whole["idx1"][a:b]) and np.array_equal(r["idx2"], whole["idx2"][a:b])
        assert r["x3d"].tobytes() == whole["x3d"][a:b].tobytes() and r["n_matches"][0] == whole["n_matches"][j]
        kf1["has_mp"][r["idx1"]] = 1


@pytest.mark.parametrize("seed", [2, 3])
def test_counts_equal_device_search(ctx, seed):
    c = M.full_scene(seed)
    got = M.run_device(ctx, c)
    kf1 = c["kf1"]; has = kf1["has_mp"].astype(np.uint8).copy()
    for j, nb in enumerate(c["neighbours"]):
        k1 = dict(desc=kf1["desc"], keys=kf1["keys_un"], has_mp=has, uright=kf1["uright"], fv=kf1["fv"])
        k2 = dict(desc=nb["desc"], keys=nb["keys_un"], has_mp=nb["has_mp"], uright=nb["uright"], fv=nb["fv"])
        nm, m = F.search_for_triangulation(ctx, k1, k2, c["F12"][j], c["ep"][j], M.SF, M.SG, False, c["coarse"], c["check_orientation"])
        assert nm == got["n_matches"][j]
        a, b = got["created_start"][j], got["created_start"][j + 1]
        assert (m[got["idx1"][a:b]] == got["idx2"][a:b]).all()
        has[got["idx1"][a:b]] = 1


def test_capacity(ctx):
    c = next(c for c in CASES if c["name"] == "large")
    total = int(M.oracle_create(c)["created_start"][-1])
    M.assert_same(M.run_device(ctx, c, cap=total), M.oracle_create(c))
    with pytest.raises(L.RgblError) as e:
        M.run_device(ctx, c, cap=total - 1)
    assert e.value.code == L.RGBL_E_CAPACITY
    M.assert_same(M.run_device(ctx, c), M.oracle_create(c))          # the context stays usable
