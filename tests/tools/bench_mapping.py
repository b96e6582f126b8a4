"""Time LocalMapping::CreateNewMapPoints for one key frame of about 2000 features and 10 neighbours (a scene of
tests/new_map_points_cases.py) two ways, and print one JSON line:
  - new:  one rgbl_create_new_map_points call (three launches, one download, one synchronise);
  - loop: what a shim does without it: per neighbour, rgbl_search_for_triangulation on the device, then the oracle's host
          triangulation and checks (tests/new_map_points_oracle.cpp) on one core, has_mp1 carried between neighbours.
Host clock around synchronised calls, after warm-up; the process is pinned to one core for both.  The card's name and power
limit are read in the same run.  Needs a GPU.
    python tests/tools/bench_mapping.py [--iters 50] [--seed 0]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

import numpy as np  # noqa: E402

import new_map_points_cases as M  # noqa: E402
from orb_slam3_rgbl_b200 import _lib as L  # noqa: E402
from orb_slam3_rgbl_b200 import frontend as F  # noqa: E402

SEARCH_FN = C.CFUNCTYPE(C.c_int, *([C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 4 + [C.c_int] +
                                   [C.c_void_p] * 7 + [C.c_int] * 3 + [C.c_void_p]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    os.sched_setaffinity(0, {sorted(os.sched_getaffinity(0))[0]})
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          check=True).stdout.strip().splitlines()[0]
    ctx = F.Context(M.W, M.H, 2000)
    case = M.full_scene(a.seed)
    nm = C.c_int(0)
    lib = L.lib()

    def device_search(n1, d1, k1, m1, u1, nn1, i1, s1, f1, n2, d2, k2, m2, u2, nn2, i2, s2, f2, F12, ep, sf, sg, only, coarse, ori, match):
        L.check(lib.rgbl_search_for_triangulation(ctx.handle, n1, d1, k1, m1, u1, nn1, i1, s1, f1, n2, d2, k2, m2, u2, nn2, i2, s2, f2, F12, ep,
                                                  M.N_LEVELS, sf, sg, only, coarse, ori, match, C.byref(nm)), ctx.handle)
        return nm.value
    cb = SEARCH_FN(device_search)
    M._search_fn = lambda: C.cast(cb, C.c_void_p)          # the oracle's loop, with its search on the device

    def timed(fn):
        for _ in range(5):
            fn()
        t = []
        for _ in range(a.iters):
            t0 = time.perf_counter(); fn(); t.append(time.perf_counter() - t0)
        return float(np.median(t)) * 1e3, float(np.min(t)) * 1e3

    new = M.run_device(ctx, case)
    loop = M.oracle_create(case)
    M.assert_same(new, loop)
    new_ms = timed(lambda: M.run_device(ctx, case))
    loop_ms = timed(lambda: M.oracle_create(case))
    print(json.dumps(dict(card=card, n1=len(case["kf1"]["desc"]), neighbours=len(case["neighbours"]), created=int(new["created_start"][-1]),
                          new_ms_median=round(new_ms[0], 3), new_ms_min=round(new_ms[1], 3), loop_ms_median=round(loop_ms[0], 3),
                          loop_ms_min=round(loop_ms[1], 3), iters=a.iters)))
    ctx.close()


if __name__ == "__main__":
    main()
