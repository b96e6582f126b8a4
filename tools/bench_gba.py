"""Global bundle adjustment on the device (rgbl_global_bundle_adjustment): per call on seeded loop-closed maps of about 100, 500, 1500 and
3000 free key frames (points seen by 3-10 key frames, tests/gba_cases.loop_graph), the time, LM iterations and trials, the time share of
linearisation, Schur build, factorisation, substitutions and updates (kernel times from torch.profiler, by kernel name), and the achieved
FP64 rate of the factorisation (n^3 / 3 per factorisation over its kernel time) against the data sheet's 67 TFLOP/s (H100 SXM, FP64
tensor core).  Then the two factorisation paths of ba_factor.cu side by side at 32 / 64 / 96 / 128 free key frames (rgbl_testing_reduced_solve
on an SPD matrix, factorisation and substitution kernel time per solve).  GPU only; prints the card name and power limit read in the same
run, and one JSON line.  Usage: python tools/bench_gba.py [--sizes 100 500 1500 3000] [--out FILE]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tests")]

PHASES = {"linearisation": ("ba_linearize", "ba_point_sum", "ba_pose_sum", "ba_maxdiag"),
          "schur": ("ba_schur_init", "ba_schur_kernel"),
          "factorisation": ("ba_cholesky", "chol_potrf", "chol_trsm", "chol_update"),
          "substitutions": ("chol_rhs", "chol_forward", "chol_back", "chol_out"),
          "updates": ("ba_point_update", "ba_pose_update", "ba_errors", "ba_final_sum", "ba_init_state", "ba_export")}
PEAK_FP64 = 67e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def kernel_times(prof):
    """{kernel name: (total device us, launches)}"""
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t > 0 and e.count:
            out[e.key] = (t, e.count)
    return out


def phase_of(name):
    for ph, keys in PHASES.items():
        if any(k in name for k in keys):
            return ph
    return None


def profiled(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return kernel_times(prof)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[100, 500, 1500, 3000])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_gba needs a GPU")
    torch.zeros(1, device="cuda")
    import gba_cases as GC
    from orb_slam3_rgbl_b200 import _lib as L
    from orb_slam3_rgbl_b200 import frontend as F
    from orb_slam3_rgbl_b200 import synthetic as S
    info = card()
    print("card:", info, flush=True)
    ctx = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=1)

    def call(p):
        return F.global_bundle_adjustment(ctx, *GC.args(p), iterations=p["iterations"], robust=p["robust"])

    call(GC.loop_graph(1, 80, iterations=2))                       # warm-up: module load, both solve paths' first launches
    call(GC.loop_graph(2, 30, iterations=2))
    rows = []
    for n_free in a.sizes:
        p = GC.loop_graph(5000 + n_free, n_free + 1, iterations=10)
        n = 6 * n_free
        t0 = time.perf_counter(); po, pt, it = call(p); t_call = time.perf_counter() - t0      # returns after a stream synchronise
        kt = profiled(lambda: call(p))
        trials = sum(c for k, (t, c) in kt.items() if "ba_point_update" in k)
        share = {ph: 0.0 for ph in PHASES}
        for k, (t, c) in kt.items():
            ph = phase_of(k)
            if ph:
                share[ph] += t
        total = sum(share.values())
        fact_s = share["factorisation"] * 1e-6
        rate = trials * n ** 3 / 3 / fact_s if fact_s > 0 else 0.0
        row = dict(free_kf=n_free, n=n, points=len(p["points"]), edges=len(p["e_point"]), call_s=round(t_call, 4), iterations=it, trials=trials,
                   kernel_s=round(total * 1e-6, 4), share={k: round(v / total, 4) for k, v in share.items()},
                   factorisation_ms_per_trial=round(fact_s * 1e3 / max(trials, 1), 3), factorisation_tflops=round(rate / 1e12, 2),
                   share_of_fp64_peak=round(rate / PEAK_FP64, 4))
        rows.append(row)
        print(json.dumps(row), flush=True)

    so = L.testing_lib()
    paths = []
    rng = np.random.default_rng(0)
    for n_free in (32, 64, 96, 128):
        n = 6 * n_free
        M = rng.normal(size=(n, n)); A = np.ascontiguousarray(np.tril(M @ M.T + n * np.eye(n))); b = rng.normal(size=n)
        x = np.empty(n); st = np.zeros(1, np.int32)
        r = dict(free_kf=n_free, n=n)
        for path, name in ((1, "single_cta"), (2, "tiled")):
            solve = lambda: so.rgbl_testing_reduced_solve(n, A.ctypes.data, b.ctypes.data, path, x.ctypes.data, st.ctypes.data)
            for _ in range(3):
                solve()
            kt = profiled(lambda: [solve() for _ in range(10)])
            t = sum(v for k, (v, c) in kt.items() if phase_of(k) in ("factorisation", "substitutions"))
            r[name + "_ms"] = round(t / 10 * 1e-3, 4)
        paths.append(r)
        print(json.dumps(r), flush=True)
    ctx.close()
    res = dict(card=info, gba=rows, paths=paths)
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
