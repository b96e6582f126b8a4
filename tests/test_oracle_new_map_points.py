"""CPU checks of the CreateNewMapPoints oracle (tests/new_map_points_oracle.cpp): every branch is reached by the cases, its decisions
equal an independent float64 restatement away from thresholds, its triangulated points equal numpy's SVD null vector on
well-conditioned matches, and its per-pair counts are SearchForTriangulation's with has_mp1 carried."""
import numpy as np
import pytest

import new_map_points_cases as M

CASES = M.all_cases()


@pytest.fixture(scope="module")
def refs():
    return {c["name"]: M.oracle_create(c) for c in CASES}


def test_every_branch_is_reached(refs):
    tags = set()
    for c in CASES:
        t = M.tags(c, refs[c["name"]])
        assert c["expect"] <= t, (c["name"], sorted(c["expect"] - t))
        tags |= t
    assert M.REQUIRED_TAGS <= tags, sorted(M.REQUIRED_TAGS - tags)


def _decide64(case, j, i1, i2):
    """(route, result, x3D) of one match in float64; `near` collects the relative margins of every threshold it compares against"""
    kf1, nb = case["kf1"], case["neighbours"][j]
    T1, T2 = kf1["Tcw"].astype(float), nb["Tcw"].astype(float)
    R1, R2 = M.quat_to_rot(T1[:4]), M.quat_to_rot(T2[:4]); t1, t2 = T1[4:], T2[4:]
    O1, O2 = -R1.T @ t1, -R2.T @ t2
    k1, k2 = kf1["keys_un"][i1], nb["keys_un"][i2]
    u1, u2 = float(kf1["uright"][i1]), float(nb["uright"][i2])
    s1, s2 = u1 >= 0, u2 >= 0
    xn1 = np.array([(k1["x"] - M.CX) / M.FX, (k1["y"] - M.CY) / M.FY, 1.0]); xn2 = np.array([(k2["x"] - M.CX) / M.FX, (k2["y"] - M.CY) / M.FY, 1.0])
    r1, r2 = R1.T @ xn1, R2.T @ xn2
    cr = r1 @ r2 / (np.linalg.norm(r1) * np.linalg.norm(r2))
    mb = M.BF / M.FX
    c1 = c2 = cr + 1
    if s1:
        c1 = np.cos(2 * np.arctan2(mb / 2, kf1["depth"][i1]))
    elif s2:
        c2 = np.cos(2 * np.arctan2(mb / 2, nb["depth"][i2]))
    cs = min(c1, c2)
    near = [(cr, cs), (cr, 0.9998), (c1, c2)]
    x = None
    if cr < cs and cr > 0 and (s1 or s2 or cr < 0.9998):
        route = 1
        P1, P2 = np.c_[R1, t1], np.c_[R2, t2]
        A = np.array([xn1[0] * P1[2] - P1[0], xn1[1] * P1[2] - P1[1], xn2[0] * P2[2] - P2[0], xn2[1] * P2[2] - P2[1]])
        v = np.linalg.svd(A)[2][3]
        x = v[:3] / v[3]
    elif s1 and c1 < c2:
        route = 2
        if not kf1["depth"][i1] > 0:
            return route, 3, None, near
        z = float(kf1["depth"][i1]); k = kf1["keys"][i1]
        x = R1.T @ np.array([(k["x"] - M.CX) * z / M.FX, (k["y"] - M.CY) * z / M.FY, z]) + O1
    elif s2 and c2 < c1:
        route = 3
        if not nb["depth"][i2] > 0:
            return route, 3, None, near
        z = float(nb["depth"][i2]); k = nb["keys"][i2]
        x = R2.T @ np.array([(k["x"] - M.CX) * z / M.FX, (k["y"] - M.CY) * z / M.FY, z]) + O2
    else:
        return 0, 1, None, near
    pc1, pc2 = R1 @ x + t1, R2 @ x + t2
    near += [(pc1[2], 0.0), (pc2[2], 0.0)]
    if pc1[2] <= 0:
        return route, 4, x, near
    if pc2[2] <= 0:
        return route, 5, x, near
    for res, pc, k, s, ur in ((6, pc1, k1, s1, u1), (7, pc2, k2, s2, u2)):
        u = M.FX * pc[0] / pc[2] + M.CX; v = M.FY * pc[1] / pc[2] + M.CY
        e = (u - k["x"]) ** 2 + (v - k["y"]) ** 2
        if s:
            e += (u - M.BF / pc[2] - ur) ** 2
        th = (7.8 if s else 5.991) * M.SG[k["octave"]]
        near.append((e, th))
        if e > th:
            return route, res, x, near
    d1, d2 = np.linalg.norm(x - O1), np.linalg.norm(x - O2)
    if case["th_far"] > 0:
        near += [(d1, case["th_far"]), (d2, case["th_far"])]
        if d1 >= case["th_far"] or d2 >= case["th_far"]:
            return route, 9, x, near
    rd, ro, rf = d2 / d1, M.SF[k1["octave"]] / M.SF[k2["octave"]], 1.5 * M.SF[1]
    near += [(rd * rf, ro), (rd, ro * rf)]
    if rd * rf < ro or rd > ro * rf:
        return route, 10, x, near
    return route, 0, x, near


def _far_from(near, rel=1e-4):
    return all(abs(a - b) > rel * max(abs(a), abs(b), 1e-12) for a, b in near)


def test_decisions_equal_float64_restatement(refs):
    checked = 0
    for c in CASES:
        for j, i1, i2, route, result, st in refs[c["name"]]["trace"]:
            r64, res64, x64, near = _decide64(c, j, i1, i2)
            if not _far_from(near):
                continue
            assert (route, result) == (r64, res64), (c["name"], j, i1, i2)
            checked += 1
    assert checked > 1000


def test_triangulated_points_equal_svd_null_vector(refs):
    checked = 0
    for c in CASES:
        r = refs[c["name"]]
        created = {(j, i1): i for i, (j, i1) in enumerate((j, i1) for j, i1, i2, route, result, st in r["trace"] if result == 0)}
        for (j, i1, i2, route, result, st) in r["trace"]:
            if result != 0 or route != 1:
                continue
            r64, res64, x64, near = _decide64(c, j, i1, i2)
            if not _far_from(near) or np.linalg.norm(x64) > 30:
                continue
            x = r["x3d"][created[(j, i1)]]
            assert np.allclose(x, x64, rtol=1e-4, atol=1e-4 * np.linalg.norm(x64)), (c["name"], j, i1, x, x64)
            checked += 1
    assert checked > 500


def test_counts_equal_search_with_carried_has_mp(refs):
    for c in CASES:
        r = refs[c["name"]]
        for j, (nm, m, has) in enumerate(M.search_with_carried(c, r)):
            assert r["n_matches"][j] == nm, (c["name"], j)
            a, b = r["created_start"][j], r["created_start"][j + 1]
            assert (m[r["idx1"][a:b]] == r["idx2"][a:b]).all()
            assert (np.diff(r["idx1"][a:b]) > 0).all()


def test_capacity(refs):
    c = next(c for c in CASES if c["name"] == "claimed")
    total = int(refs["claimed"]["created_start"][-1])
    assert M.oracle_create(c, cap=total)["rc"] == 0
    assert M.oracle_create(c, cap=total - 1)["rc"] == -3
