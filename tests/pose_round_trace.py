"""TEST INFRASTRUCTURE: what each round of PoseOptimization did, from the oracle's own code.  oracle/pose_oracle.cpp stays as it is; this
module compiles a copy of it with counters inserted (text only, every anchor must match exactly as often as expected, so a change of the
oracle fails here instead of silently counting something else) into tests/cuda_emu/build/pose_round_trace/.  The counters read values the
oracle computes anyway and change none of its arithmetic: the outputs equal oracle.pose_optimize_trace's (test_cuda_emu_pose_replica.py
checks it).

Per round r: changed[r], the edges whose level r's classification changed; linear[r], r's robust Huber evaluations in the linear region
(e2 > dsqr, or NaN); linear_first[r] / linear_rejected[r], those at r's initial pose (before its first system is built) and in its
rejected trials.  replica_rounds: the rounds that repeat the round before them bit for bit (no level changed after it, and the same
robust flag or no linear-region evaluation in it), which pose_optimize_kernel does not run.  The oracle itself runs every round, as g2o."""
from __future__ import annotations

import ctypes as C
import subprocess
from pathlib import Path

import numpy as np

import oracle

HERE = Path(__file__).resolve().parent
SRC = HERE.parent / "oracle" / "pose_oracle.cpp"
OUT = HERE / "cuda_emu" / "build" / "pose_round_trace"

# (anchor, replacement, occurrences)
_EDITS = [
    ("    double min_rho_margin, min_stop_margin, min_chi2_margin;\n};",
     "    double min_rho_margin, min_stop_margin, min_chi2_margin;\n"
     "    int changed[4], linear[4], linear_first[4], linear_rejected[4], replica_rounds;\n};", 1),
    ("    PoseTrace* tr = nullptr;\n",
     "    PoseTrace* tr = nullptr;\n"
     "    mutable int linear = 0;\n"
     "    void count_linear(double e2, float dsqr) const { if (!(e2 <= dsqr)) ++linear; }\n", 1),
    ("huber(edge_chi2(e), e.stereo ? delta_stereo : delta_mono, e.stereo ? dsqr_stereo : dsqr_mono, rho);",
     "count_linear(edge_chi2(e), e.stereo ? dsqr_stereo : dsqr_mono); "
     "huber(edge_chi2(e), e.stereo ? delta_stereo : delta_mono, e.stereo ? dsqr_stereo : dsqr_mono, rho);", 2),
    ("        const double ini = current;\n",
     "        const double ini = current;\n"
     "        if (tr && iteration == 0) tr->linear_first[tr->rounds] = linear;\n", 1),
    ("            compute_active_errors();\n            temp = active_robust_chi2();\n",
     "            compute_active_errors();\n            const int linear0 = linear;\n            temp = active_robust_chi2();\n", 1),
    ("lambda *= ni; ni *= 2; est = backup;",
     "lambda *= ni; ni *= 2; est = backup; if (tr) tr->linear_rejected[tr->rounds] += linear - linear0;", 1),
    ("        lm.est = init;\n        const int iters = lm.optimize(10);\n",
     "        lm.est = init; lm.linear = 0;\n        const int iters = lm.optimize(10);\n"
     "        if (tr) { tr->linear[it] = lm.linear; tr->changed[it] = 0; }\n", 1),
    ("            if (outlier[i]) edge_error(e, lm.est, cam);\n",
     "            const int level0 = e.level;\n            if (outlier[i]) edge_error(e, lm.est, cam);\n", 1),
    ("            if (it == 2) e.robust = false;\n",
     "            if (tr) tr->changed[it] += e.level != level0;\n            if (it == 2) e.robust = false;\n", 1),
    ("    // Sophus::SE3<float> pose(rotation()",
     "    if (tr)\n"
     "        for (int r = 1; r < tr->rounds; ++r)\n"
     "            tr->replica_rounds += tr->changed[r - 1] == 0 && ((r < 3) == (r - 1 < 3) || tr->linear[r - 1] == 0);\n"
     "    // Sophus::SE3<float> pose(rotation()", 1),
]


def _source() -> str:
    text = SRC.read_text()
    for anchor, repl, count in _EDITS:
        found = text.count(anchor)
        if found != count:
            raise RuntimeError(f"oracle/pose_oracle.cpp changed: {anchor!r} found {found} times, expected {count}")
        text = text.replace(anchor, repl)
    return text


def build() -> Path:
    lib = OUT / "libpose_round_trace.so"
    if lib.exists() and lib.stat().st_mtime > max(SRC.stat().st_mtime, Path(__file__).stat().st_mtime):
        return lib
    OUT.mkdir(parents=True, exist_ok=True)
    src = OUT / "pose_round_trace.cpp"
    src.write_text(_source())
    # the oracle's own flags (oracle/Makefile)
    subprocess.run(["g++", "-O3", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wno-unused-function",
                    f"-I{SRC.parent}", "-shared", "-o", str(lib), str(src), "-lm"], check=True)
    return lib


class _Trace(C.Structure):
    _fields_ = oracle.PoseTraceC._fields_ + [("changed", C.c_int * 4), ("linear", C.c_int * 4), ("linear_first", C.c_int * 4),
                                             ("linear_rejected", C.c_int * 4), ("replica_rounds", C.c_int)]


_lib = None


def pose_optimize_trace(pose, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf):
    """oracle.pose_optimize_trace with the per-round fields above -> (n_inliers, pose_out[7], outlier[n], trace)"""
    global _lib
    if _lib is None:
        _lib = C.CDLL(str(build()))
        _lib.orc_pose_optimize_trace.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] * 5 + [C.c_void_p, C.c_void_p, C.POINTER(_Trace)]
        _lib.orc_pose_optimize_trace.restype = C.c_int
    pose = np.ascontiguousarray(pose, np.float32); xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    stereo = np.ascontiguousarray(stereo, np.uint8)
    n = len(xw)
    out = np.empty(7, np.float32); outlier = np.zeros(n, np.uint8); tr = _Trace()
    r = _lib.orc_pose_optimize_trace(pose.ctypes.data, n, xw.ctypes.data, obs.ctypes.data, inv_sigma2.ctypes.data, stereo.ctypes.data,
                                     fx, fy, cx, cy, bf, out.ctypes.data, outlier.ctypes.data, C.byref(tr))
    per_round = ("iters", "changed", "linear", "linear_first", "linear_rejected")
    trace = {name: (list(getattr(tr, name))[:tr.rounds] if name in per_round else getattr(tr, name)) for name, _ in _Trace._fields_}
    return r, out, outlier, trace
