"""CPU-side checks of the product library: it loads, exports every symbol include/rgbl_b200.h declares,
fails loudly without a GPU, and its host-side pieces (tables, geometry, quad-tree, masks) match the oracle."""
import ctypes as C
import re
from pathlib import Path

import numpy as np
import pytest

import oracle
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol():
    hdr = (ROOT / "include" / "rgbl_b200.h").read_text()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(rgbl_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 15
    lib = C.CDLL(str(L.LIB_PATH))
    for name in sorted(declared):
        assert hasattr(lib, name), f"librgbl_b200.so does not export {name}"
    assert declared == set(L.SYMBOLS), f"python binding out of sync: {declared ^ set(L.SYMBOLS)}"
    assert L.lib().rgbl_abi_version() >= 1


def test_no_cpu_fallback(have_gpu):
    if have_gpu:
        pytest.skip("GPU present")
    with pytest.raises(L.RgblError) as e:
        F.Context(S.KITTI_W, S.KITTI_H)
    assert e.value.code == L.RGBL_E_CUDA and "no CPU fallback" in str(e.value)


def test_product_never_imports_oracle():
    for p in (ROOT / "orb_slam3_rgbl_b200").rglob("*"):
        if p.suffix in (".py", ".cu", ".cpp", ".h", ".cuh") and p.is_file():
            txt = p.read_text(errors="ignore")
            assert "import oracle" not in txt and "liborb_oracle" not in txt and "oracle/" not in txt, p
    for p in (ROOT / "tools").rglob("*"):              # development tools that need the oracle live under tests/tools
        if p.is_file() and p.suffix in (".py", ".sh", ".cpp"):
            txt = p.read_text(errors="ignore")
            assert "import oracle" not in txt and "liborb_oracle" not in txt and "_oracle.cpp" not in txt, p


@pytest.mark.parametrize("nf,sf,nl", [(2000, 1.2, 8), (1000, 1.2, 8), (4000, 1.2, 8), (1200, 1.5, 5), (500, 1.1, 12)])
def test_orb_tables_match_oracle(nf, sf, nl):
    t = F.orb_tables(nf, sf, nl)
    ex = oracle.Extractor(nf, sf, nl)
    assert (t["scale"] == ex.scale_factors).all() and (t["inv_scale"] == ex.inv_scale_factors).all()
    assert (t["features_per_level"] == ex.features_per_level).all() and (t["umax"] == ex.umax).all()
    assert list(t["umax"]) == [15, 15, 15, 15, 14, 14, 14, 13, 13, 12, 11, 10, 9, 8, 6, 3]     # SURVEY a1


def test_structuring_elements_match_reference_tables():
    for kind in ("Rectangle", "Cross", "Ellipse"):
        for ku, kv in ((3, 3), (5, 3), (7, 5), (9, 9), (1, 1), (4, 6)):
            assert (F.structuring_element(kind, ku, kv) == S.structuring_element(kind, ku, kv)).all()
    d5 = F.structuring_element("Diamond", 5)
    assert d5.tolist() == [[0, 0, 1, 0, 0], [0, 1, 1, 1, 0], [1, 1, 1, 1, 1], [0, 1, 1, 1, 0], [0, 0, 1, 0, 0]]   # DepthModule.h:141-145
    with pytest.raises(L.RgblError):
        F.structuring_element("Diamond", 4)
    with pytest.raises(L.RgblError):
        F.structuring_element("Hexagon", 5)


def test_descriptor_distance_is_popcount():
    rng = np.random.default_rng(0)
    for _ in range(200):
        a = rng.integers(0, 256, 32, dtype=np.uint8); b = rng.integers(0, 256, 32, dtype=np.uint8)
        assert L.lib().rgbl_descriptor_distance(L.ptr(a), L.ptr(b)) == int(np.unpackbits(a ^ b).sum())
    z = np.zeros(32, np.uint8); o = np.full(32, 255, np.uint8)
    assert L.lib().rgbl_descriptor_distance(L.ptr(z), L.ptr(o)) == 256


def _quadtree(cand, w, h, n):
    out = np.empty(max(n + 3, 4 * max(1, round((w - 32) / (h - 32)))), np.int32)
    m = L.testing_lib().rgbl_quadtree_select(L.ptr(np.ascontiguousarray(cand, np.int32)), len(cand), 16, w - 16, 16, h - 16, n, L.ptr(out), len(out))
    assert m >= 0
    return out[:m]


def _oracle_quadtree(cand, w, h, n):
    k = np.zeros(len(cand), oracle.KP_DTYPE)
    k["x"], k["y"], k["response"] = cand[:, 0], cand[:, 1], cand[:, 2]
    return oracle.distribute_quadtree(k, 16, w - 16, 16, h - 16, n)


@pytest.mark.parametrize("seed", range(6))
def test_quadtree_matches_oracle_on_real_candidates(seed):
    img = S.make_image(100 + seed, 900, 300)
    ex = oracle.Extractor(1500); ex(img)
    for l in range(8):
        cand = ex.level_candidates(l)
        h, w = ex.level_image(l).shape
        sel = cand[_quadtree(cand, w, h, int(ex.features_per_level[l]))]
        ref = ex.level_keypoints(l)
        assert len(sel) == len(ref)
        assert (sel[:, 0] + 16 == ref["x"]).all() and (sel[:, 1] + 16 == ref["y"]).all() and (sel[:, 2] == ref["response"]).all()


@pytest.mark.parametrize("seed", range(12))
def test_quadtree_matches_oracle_random(seed):
    """Random candidate clouds incl. heavy score ties and tiny/huge budgets: the tie-sensitive paths
    (std::sort order, first-max) must agree with the oracle's std::list restatement."""
    rng = np.random.default_rng(seed)
    w, h = int(rng.integers(120, 1300)), int(rng.integers(100, 420))
    n = int(rng.integers(1, 6000))
    xy = np.unique(np.stack([rng.integers(0, w - 32, n) // 2 * 2, rng.integers(0, h - 32, n) // 2 * 2], 1), axis=0)
    order = np.lexsort((xy[:, 0], xy[:, 1]))             # row-major like cv::FAST
    xy = xy[order]
    sc = rng.integers(7, 12 if seed % 2 else 200, len(xy))
    cand = np.concatenate([xy, sc[:, None]], 1).astype(np.int32)
    for budget in (1, 5, 60, 434, 5000):
        if round((w - 32) / (h - 32)) < 1:
            continue
        sel = cand[_quadtree(cand, w, h, budget)]
        ref = _oracle_quadtree(cand, w, h, budget)
        assert len(sel) == len(ref)
        assert (sel[:, 0] == ref["x"]).all() and (sel[:, 1] == ref["y"]).all() and (sel[:, 2] == ref["response"]).all()


def test_quadtree_empty_and_single():
    assert len(_quadtree(np.zeros((0, 3), np.int32), 400, 200, 50)) == 0
    one = np.array([[10, 10, 30]], np.int32)
    assert _quadtree(one, 400, 200, 50).tolist() == [0]


# ---- device quad-tree logic, executed on the host (same source as the kernel: quadtree_block.cuh) ----

def _block(cand, w, h, n):
    out = np.empty((max(n + 3, 4 * max(1, round((w - 32) / (h - 32)))), 3), np.int32)
    m = L.testing_lib().rgbl_quadtree_select_block_emulation(L.ptr(np.ascontiguousarray(cand, np.int32)), len(cand), 16, w - 16, 16, h - 16, n, L.ptr(out), len(out))
    assert m >= 0
    return out[:m]


def test_std_sort_restatement_matches_python_reference_order_on_distinct_keys():
    """With distinct keys every correct sort agrees; tie behaviour is checked against the oracle's std::sort through the
    quad-tree tests below (and was checked against libstdc++ directly on 20 200 arrays during development)."""
    rng = np.random.default_rng(0)
    for n in (0, 1, 2, 15, 16, 17, 33, 200, 1500):
        keys = rng.permutation(n * 2)[:n]
        su = np.stack([keys, np.zeros(n, np.int64)], 1).astype(np.int32)
        perm = np.empty(max(n, 1), np.int32)
        L.testing_lib().rgbl_std_sort_emulation(L.ptr(np.ascontiguousarray(su)), n, L.ptr(perm))
        assert (keys[perm[:n]] == np.sort(keys)).all()


@pytest.mark.parametrize("seed", range(4))
def test_block_quadtree_matches_oracle_on_real_candidates(seed):
    img = S.make_image(300 + seed, 1000, 320)
    ex = oracle.Extractor(2000); ex(img)
    for l in range(8):
        cand = ex.level_candidates(l)
        h, w = ex.level_image(l).shape
        got = _block(cand, w, h, int(ex.features_per_level[l]))
        ref = ex.level_keypoints(l)
        assert len(got) == len(ref)
        assert (got[:, 0] + 16 == ref["x"]).all() and (got[:, 1] + 16 == ref["y"]).all() and (got[:, 2] == ref["response"]).all()


@pytest.mark.parametrize("seed", range(10))
def test_block_quadtree_matches_oracle_random_ties(seed):
    rng = np.random.default_rng(100 + seed)
    w, h = int(rng.integers(120, 1300)), int(rng.integers(100, 420))
    if round((w - 32) / (h - 32)) < 1:
        return
    n = int(rng.integers(1, 6000))
    xy = np.unique(np.stack([rng.integers(0, w - 32, n) // 2 * 2, rng.integers(0, h - 32, n) // 2 * 2], 1), axis=0)
    xy = xy[np.lexsort((xy[:, 0], xy[:, 1]))]
    sc = rng.integers(7, 12 if seed % 2 else 200, len(xy))
    cand = np.concatenate([xy, sc[:, None]], 1).astype(np.int32)
    for budget in (1, 5, 60, 434, 900):
        ref = _oracle_quadtree(cand, w, h, budget)
        got = _block(cand, w, h, budget)
        assert len(got) == len(ref)
        assert (got[:, 0] == ref["x"]).all() and (got[:, 1] == ref["y"]).all() and (got[:, 2] == ref["response"]).all()


def test_header_is_plain_c():
    """The drop-in boundary is a C ABI: include/rgbl_b200.h must compile as C99 and as C++11 on its own (no torch / CUDA types)."""
    import subprocess
    from pathlib import Path
    hdr = Path(__file__).resolve().parent.parent / "include" / "rgbl_b200.h"
    for cmd in (["gcc", "-std=c99", "-fsyntax-only", "-x", "c"], ["g++", "-std=c++11", "-fsyntax-only", "-x", "c++"]):
        r = subprocess.run(cmd + [str(hdr)], capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    txt = hdr.read_text()
    assert "torch" not in txt and "#include <cuda" not in txt and "cudaStream_t" not in txt      # no torch / CUDA types in the signatures


def test_plain_c_client_links_against_the_library(tmp_path):
    """examples/abi_demo.c is a C99 program using nothing but include/rgbl_b200.h; it must compile, link against librgbl_b200.so and run:
    on a box without a CUDA device rgbl_create reports RGBL_E_CUDA (exit code 3) - there is no CPU fallback."""
    import subprocess
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    libdir = root / "orb_slam3_rgbl_b200"
    exe = tmp_path / "abi_demo"
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", f"-I{root / 'include'}", str(root / "examples" / "abi_demo.c"), f"-L{libdir}", "-lrgbl_b200",
                        f"-Wl,-rpath,{libdir}", "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    run = subprocess.run([str(exe)], capture_output=True, text=True, timeout=300)
    import torch
    if torch.cuda.is_available():
        assert run.returncode == 0 and "keypoints" in run.stdout, run.stdout + run.stderr
    else:
        assert run.returncode == 3 and "no CPU fallback" in run.stdout, run.stdout + run.stderr


# ---- strip formulation of the per-cell FAST (fast_strip.cuh), executed on the host ----------------------------------------
def _strip_fast(img_level, width, height, level, nfeatures=1500, scale=1.2, nlevels=8, ini_th=12, min_th=7, max_cells=8, max_width=264):
    prm = L.OrbParams(nfeatures, scale, nlevels, ini_th, min_th)
    lv = np.ascontiguousarray(img_level, np.uint8)
    out = np.empty((1 << 18, 3), np.int32)
    n = L.testing_lib().rgbl_fast_strips_emulation(C.byref(prm), width, height, level, L.ptr(lv), lv.strides[0], max_cells, max_width, L.ptr(out), len(out))
    assert n >= 0, n
    return out[:n]


@pytest.mark.parametrize("seed,size,ths,strip", [
    (0, (900, 300), (20, 7), (8, 264)), (1, (900, 300), (20, 7), (3, 120)), (2, (1241, 376), (20, 7), (8, 264)),
    (3, (640, 480), (12, 7), (5, 200)), (4, (501, 260), (40, 5), (1, 78)), (5, (752, 480), (20, 7), (8, 250)),
    (6, (900, 300), (255, 60), (8, 264)), (7, (333, 250), (20, 7), (2, 264))])
def test_fast_strips_match_the_oracle_cell_by_cell(seed, size, ths, strip):
    """Every level of a real pyramid: same candidates, same scores, same (cell-major, row-major) order as the per-cell cv::FAST
    restatement with the iniTh -> minTh fallback (src/ORBextractor.cc:805-868)."""
    w, h = size
    img = S.make_image(300 + seed, w, h)
    ex = oracle.Extractor(1500, ini_th=ths[0], min_th=ths[1]); ex(img)
    total = 0
    for l in range(8):
        got = _strip_fast(ex.level_image(l), w, h, l, ini_th=ths[0], min_th=ths[1], max_cells=strip[0], max_width=strip[1])
        ref = ex.level_candidates(l)
        assert got.shape == ref.shape, (l, got.shape, ref.shape)
        assert (got == ref).all(), l
        total += len(ref)
    assert total > 200


def test_fast_strips_on_flat_and_saturated_images():
    for val in (0, 255, 128):
        img = np.full((250, 333), val, np.uint8)
        ex = oracle.Extractor(500); ex(img)
        for l in range(8):
            assert len(_strip_fast(ex.level_image(l), 333, 250, l, nfeatures=500)) == len(ex.level_candidates(l)) == 0
    # checkerboard: many equal scores next to each other (NMS ties) and every cell needs the fallback decision
    yy, xx = np.mgrid[0:240, 0:400]
    img = (((xx // 5 + yy // 5) & 1) * 200 + 20).astype(np.uint8)
    ex = oracle.Extractor(1000); ex(img)
    for l in range(8):
        got, ref = _strip_fast(ex.level_image(l), 400, 240, l, nfeatures=1000), ex.level_candidates(l)
        assert got.shape == ref.shape and (got == ref).all(), l


def test_fast_strips_when_every_pixel_passes_the_high_speed_test():
    """Vertical stripes of period 6 (plus noise): p[-3] and p[+3] differ from every pixel by ~200, so the high-speed test passes
    everywhere and the list of listed pixels fills its buffer - the strip kernel then cannot put its second list (score-carrying
    words) into the same buffer and walks all words in the NMS phase instead."""
    rng = np.random.default_rng(77)
    yy, xx = np.mgrid[0:260, 0:420]
    img = (((xx % 6) < 3) * 200 + 20 + rng.integers(0, 30, xx.shape)).astype(np.uint8)
    ex = oracle.Extractor(1000); ex(img)
    total = 0
    for l in range(8):
        got, ref = _strip_fast(ex.level_image(l), 420, 260, l, nfeatures=1000), ex.level_candidates(l)
        assert got.shape == ref.shape and (got == ref).all(), l
        total += len(ref)
    assert total > 100


# ---- block-parallel std::sort (quadtree_block.cuh: block_std_sort), executed on the host -----------------------------------
def _sort_perm(su, mode):
    perm = np.empty(len(su), np.int32)
    assert L.testing_lib().rgbl_std_sort_block_emulation(L.ptr(np.ascontiguousarray(su, np.int32)), len(su), mode, L.ptr(perm)) == 0
    return perm


@pytest.mark.parametrize("seed", range(40))
def test_block_std_sort_equals_libstdcxx_sort_including_ties(seed):
    """Same permutation as the C++ library's std::sort with compareNodes (src/ORBextractor.cc:538-553): the order of equal
    (size, UL.x) pairs is decided by the introsort's swaps, which the block formulation has to reproduce exactly."""
    rng = np.random.default_rng(900 + seed)
    for n in [0, 1, 2, 15, 16, 17, 18, 33, 64, 100, 257, 430, 777, 1024][seed % 7::7] + [int(rng.integers(17, 1025))]:
        k_size, k_x = [(3, 4), (8, 30), (40, 40), (2, 2), (1000, 1000)][seed % 5]
        su = np.stack([rng.integers(2, 2 + k_size, n), rng.integers(0, k_x, n) * 37], 1).astype(np.int32)
        if seed % 4 == 1:
            su = su[np.lexsort((su[:, 1], su[:, 0]))]                  # already sorted
        if seed % 4 == 2:
            su = su[np.lexsort((su[:, 1], su[:, 0]))][::-1]            # reversed
        ref = _sort_perm(su, -1)
        assert (_sort_perm(su, 0) == ref).all(), n
        serial = np.empty(n, np.int32)
        L.testing_lib().rgbl_std_sort_emulation(L.ptr(np.ascontiguousarray(su)), n, L.ptr(serial))
        assert (serial == ref).all(), n
        for forced in (1, 2, 4):                                       # depth limit 0, 1, 3: heapsort fallback path
            assert (_sort_perm(su, forced) == ref).all(), (n, forced)


@pytest.mark.parametrize("seed", range(6))
def test_block_quadtree_with_block_sort_matches_oracle(seed):
    img = S.make_image(140 + seed, 900, 300)
    ex = oracle.Extractor(1500); ex(img)
    for l in range(8):
        cand = ex.level_candidates(l)
        h, w = ex.level_image(l).shape
        n = int(ex.features_per_level[l])
        out = np.empty((n + 64, 3), np.int32)
        m = L.testing_lib().rgbl_quadtree_select_block_emulation(L.ptr(np.ascontiguousarray(cand, np.int32)), len(cand), 16, w - 16, 16, h - 16, n, L.ptr(out), len(out))
        ref = ex.level_keypoints(l)
        assert m == len(ref)
        assert (out[:m, 0] + 16 == ref["x"]).all() and (out[:m, 1] + 16 == ref["y"]).all() and (out[:m, 2] == ref["response"]).all()


# ---- staged describe kernel (describe_warp.cuh), host twin ----------------------------------------------------------------
@pytest.mark.parametrize("seed,size", [(0, (900, 300)), (1, (1241, 376)), (2, (640, 480)), (3, (333, 250))])
def test_staged_describe_matches_the_oracle(seed, size):
    """Angles (bit-exact floats) and descriptors of every keypoint of a real extraction, level by level."""
    w, h = size
    img = S.make_image(500 + seed, w, h)
    ex = oracle.Extractor(1200)
    kps, desc, _ = ex(img)
    prm = L.OrbParams(1200, 1.2, 8, 12, 7)
    base = 0
    for l in range(8):
        lv = ex.level_image(l)
        bl = oracle.gaussian_blur7(lv)
        kl = ex.level_keypoints(l)
        n = len(kl)
        if n == 0:
            continue
        xy = np.ascontiguousarray(np.stack([kl["x"], kl["y"]], 1).astype(np.int32))
        ang = np.empty(n, np.float32); d = np.empty((n, 32), np.uint8)
        rc = L.testing_lib().rgbl_describe_staged_emulation(C.byref(prm), L.ptr(lv), L.ptr(bl), lv.shape[1], lv.shape[0], lv.strides[0], n,
                                                    L.ptr(xy), L.ptr(ang), L.ptr(d))
        assert rc == 0
        ref = kps[base:base + n]
        assert (ref["octave"] == l).all()
        assert (ang.view(np.uint32) == np.ascontiguousarray(ref["angle"]).view(np.uint32)).all(), l
        assert (d == desc[base:base + n]).all(), l
        base += n
    assert base == len(kps) > 500
