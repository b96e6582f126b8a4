"""The batched Frame::ComputeStereoMatches kernels (stereo_kernels.cu: row index count / scan / fill, match, median rejection) on the
CUDA-on-CPU shim (tests/cuda_emu), several pairs in one launch, against the oracle's restatement of the reference (stereo_oracle.cpp)."""
import ctypes as C
import importlib.util
import subprocess
from pathlib import Path

import numpy as np
import pytest

import oracle
from oracle import _p
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import synthetic as S

HERE = Path(__file__).resolve().parent
W, H = 320, 160


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("cuda_emu_build", HERE / "cuda_emu" / "build.py")
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    d = mod.BUILD / "stereo"
    d.mkdir(parents=True, exist_ok=True)
    for f in mod.CSRC.iterdir():
        if f.suffix in (".h", ".cuh", ".inc"):
            (d / f.name).write_text(mod._transform(f.read_text()))
    (d / "stereo_kernels.emu.cpp").write_text(mod._transform((mod.CSRC / "stereo_kernels.cu").read_text()))
    lib = d / "libcuda_emu_stereo.so"
    subprocess.run(["g++", "-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes",
                    f"-I{HERE / 'cuda_emu'}", f"-I{d}", "-o", str(lib), str(HERE / "cuda_emu" / "emu_stereo.cpp"),
                    str(HERE / "cuda_emu" / "emu_runtime.cpp")], check=True)
    L_ = C.CDLL(str(lib))
    L_.emu_stereo_idx_cap.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_int]
    L_.emu_stereo_matches.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L_


def _oracle_matches(kl, dl, kr, dr, lv_l, lv_r, scale, inv_scale, mb, mbf):
    """oracle.stereo_matches on explicit level images (the pyramids of hand-made pairs are not an extractor's)."""
    lib = oracle.lib()
    oracle._late(lib)
    kl = np.ascontiguousarray(kl, L.KP_DTYPE); kr = np.ascontiguousarray(kr, L.KP_DTYPE)
    dl = np.ascontiguousarray(dl, np.uint8); dr = np.ascontiguousarray(dr, np.uint8)
    nl = len(lv_l)
    pl = (C.c_void_p * nl)(*[a.ctypes.data for a in lv_l]); pr = (C.c_void_p * nl)(*[a.ctypes.data for a in lv_r])
    lw = np.array([a.shape[1] for a in lv_l], np.int32); lh = np.array([a.shape[0] for a in lv_l], np.int32)
    d = np.empty(len(kl), np.float32); u = np.empty(len(kl), np.float32)
    lib.orc_stereo_matches(len(kl), _p(kl), _p(dl), len(kr), _p(kr), _p(dr), nl, _p(scale), _p(inv_scale), pl, pr, _p(lw), _p(lh), mb, mbf, _p(d), _p(u))
    return d, u


def _extracted(ex, img):
    k, d, _ = ex(img)
    return k, d, [np.ascontiguousarray(ex.level_image(l)) for l in range(ex.nlevels)]


def _periodic_pair(ex):
    """A hand-made pair whose SADs tie: columns alternate between two values (period 2) and every row is the same, so the 11 shifts of
    the SAD window give two values only, and every matched keypoint has the same SAD (the right image's values differ by 2, so it is
    not 0 and the median rejection keeps them).  Right keypoints are listed twice with the same descriptor (Hamming ties: the first one
    must win)."""
    def levels(a, b):
        img = np.tile(np.array([a, b], np.uint8), W // 2)[None, :].repeat(H, 0)
        return [np.ascontiguousarray(np.resize(img, (int(round(H / s)), int(round(W / s))))) for s in ex.scale_factors]
    rng = np.random.default_rng(3)
    n = 40
    kl = np.zeros(n, L.KP_DTYPE)
    kl["x"] = rng.integers(60, W - 40, n).astype(np.float32) + rng.choice([0.0, 0.5], n).astype(np.float32)
    kl["y"] = rng.integers(20, H - 20, n).astype(np.float32)
    kl["octave"] = rng.integers(0, 3, n)
    kl["size"] = 31.0
    kr = kl.copy(); kr["x"] -= rng.integers(2, 9, n).astype(np.float32)
    kr = np.concatenate([kr, kr])
    dl = rng.integers(0, 256, (n, 32)).astype(np.uint8)
    dr = np.concatenate([dl, dl])
    dr[:n, 0] ^= 1                           # one bit off in the first copy: the exact copy (later index) wins on distance
    dr[n // 2:n, :] = dl[n // 2:]            # ... except for the second half, where both copies tie and the first must win
    return (kl, dl, levels(40, 200)), (kr, dr, levels(42, 198))


def _check_row_index(row_start, row_idx, kr, scale):
    """The CSR row index equals vRowIndices (src/Frame.cc:918-940) and lists each row's right keypoints in ascending order."""
    rows = [[] for _ in range(H)]
    for i, k in enumerate(kr):
        r = np.float32(2.0) * scale[k["octave"]]
        for y in range(int(np.floor(np.float32(k["y"] - r))), int(np.ceil(np.float32(k["y"] + r))) + 1):
            if 0 <= y < H:
                rows[y].append(i)
    assert row_start[0] == 0
    for y in range(H):
        assert row_idx[row_start[y]:row_start[y + 1]].tolist() == rows[y], y


def test_batched_stereo_kernels_match_oracle(emu):
    ex_l, ex_r = oracle.Extractor(500), oracle.Extractor(500)
    scale, inv_scale = ex_l.scale_factors.copy(), ex_l.inv_scale_factors.copy()
    nlev = ex_l.nlevels
    mb, mbf = np.float32(S.KITTI_BF) / np.float32(S.KITTI_FX), np.float32(S.KITTI_BF)
    pairs = []
    for seed in (5, 6):                                  # the non-uniform disparity field of stereo_pair
        l, r = S.stereo_pair(seed, W, H)
        pairs.append((_extracted(ex_l, l), _extracted(ex_r, r)))
    tex = S.make_image(7, W + 16, H)                     # a whole-pixel shift: most SADs are 0, the median ties
    pairs.append((_extracted(ex_l, np.ascontiguousarray(tex[:, 8:8 + W])), _extracted(ex_r, np.ascontiguousarray(tex[:, 13:13 + W]))))
    (kl, dl, lv), (kr, dr, rv) = pairs[0]
    pairs.append(((kl[: len(kl) // 2], dl[: len(kl) // 2], lv), (kr[:0], dr[:0], rv)))      # no right keypoints: no match at all
    pairs.append(_periodic_pair(ex_l))
    n_pairs = len(pairs)
    cap = max(max(len(a[0]), len(b[0])) for a, b in pairs)
    lw = np.array([a.shape[1] for a in pairs[0][0][2]], np.int32); lh = np.array([a.shape[0] for a in pairs[0][0][2]], np.int32)
    slots = [p[0] for p in pairs] + [p[1] for p in pairs]
    levels = np.concatenate([np.concatenate([a.reshape(-1) for a in s[2]]) for s in slots])
    n_kp = np.array([len(s[0]) for s in slots], np.int32)
    kps = np.zeros((2 * n_pairs, cap), L.KP_DTYPE); desc = np.zeros((2 * n_pairs, cap, 32), np.uint8)
    for i, s in enumerate(slots):
        kps[i, :len(s[0])] = s[0]; desc[i, :len(s[0])] = s[1]
    idx_cap = emu.emu_stereo_idx_cap(cap, _p(scale), nlev, H)
    depth = np.full((2 * n_pairs, cap), 7.0, np.float32); ur = np.full((2 * n_pairs, cap), 7.0, np.float32)
    row_start = np.zeros((n_pairs, H + 1), np.int32); row_idx = np.full((n_pairs, idx_cap), -1, np.int32)
    assert emu.emu_stereo_matches(n_pairs, nlev, _p(lw), _p(lh), _p(scale), _p(inv_scale), _p(levels), _p(n_kp), _p(kps), _p(desc), cap, mb, mbf,
                                  _p(depth), _p(ur), _p(row_start), _p(row_idx)) == 0
    n_matched = []
    for p, ((kl, dl, lv), (kr, dr, rv)) in enumerate(pairs):
        rd, ru = _oracle_matches(kl, dl, kr, dr, lv, rv, scale, inv_scale, mb, mbf)
        n = len(kl)
        assert (depth[p, :n].view(np.uint32) == rd.view(np.uint32)).all(), (p, int((depth[p, :n] != rd).sum()))
        assert (ur[p, :n].view(np.uint32) == ru.view(np.uint32)).all(), p
        assert (depth[p, n:] == 7.0).all() and (depth[n_pairs + p] == 7.0).all()           # nothing written beyond the left keypoints
        _check_row_index(row_start[p], row_idx[p], kr, scale)
        n_matched.append(int((rd > 0).sum()))
    assert n_matched[0] > 50 and n_matched[1] > 50 and n_matched[2] > 50 and n_matched[3] == 0 and n_matched[4] > 0, n_matched
    assert (depth[3, :len(pairs[3][0][0])] == -1.0).all()


def test_row_index_capacity_bounds_every_keypoint(emu):
    """stereo_row_index_cap's per-keypoint bound (2 r + 4 rows, r = 2 scale) holds for every octave and sub-pixel row, near the image's
    top and bottom too, and is clipped to the image height."""
    for nlev, sf in ((8, 1.2), (5, 1.44), (3, 2.0)):
        t = oracle.Extractor(100, sf, nlev)
        scale = t.scale_factors.copy()
        per_kp = emu.emu_stereo_idx_cap(1, _p(scale), nlev, 10 ** 6)
        for o in range(nlev):
            r = np.float32(2.0) * scale[o]
            for y in np.linspace(0.0, 50.0, 2001, dtype=np.float32):
                assert int(np.ceil(np.float32(y + r))) - int(np.floor(np.float32(y - r))) + 1 <= per_kp
        assert emu.emu_stereo_idx_cap(1, _p(scale), nlev, 7) == 7
