"""RGB-D throughput (needs a GPU; writes nothing): System::TrackRGBD as in Examples/RGB-D/rgbd_kitti.cc on the workload of bench.py's
config B, with uint16 depth images (KITTI depth PNG scale x256, 5 % holes) instead of point clouds, tracked through
rgbl_track_sequence_rgbd from staged device slots; and 32 KITTI-size 16-bit depth PNGs through rgbl_decode_png_depth16, with a
one-core python-cv2 imdecode arm.  Prints one JSON line.
    python tools/bench_rgbd.py [--steps K] [--no-cpu]"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench as B                                                    # noqa: E402  (CONFIGS, make_sequence, chain thresholds)
from orb_slam3_rgbl_b200 import frontend as F, synthetic as S       # noqa: E402


def sequence(steps, factor):
    cfg = B.CONFIGS["B"]
    T, M, W, H, cam = cfg["T"], cfg["M"], cfg["W"], cfg["H"], cfg["cam"]
    seq = B.make_sequence(cfg, 2000)
    ctx = F.Context(W, H, cfg["nfeat"], max_batch=T)
    try:
        runner = F.SequenceRunner.rgbd(ctx, F.depth_map_factor(factor), cam[4], T, W, H, M, pinned=True)
        for m in range(M):
            ts = range(m * T, (m + 1) * T)
            runner.set_batch(m, [seq.image(t) for t in ts], [seq.depth16(t, factor) for t in ts])
            runner.stage(m, m)
        chain = lambda cont: F.make_chain_params(seq.pose(0), *cam, th_last=B.TH_LAST, continue_sequence=cont, local_map_frames=cfg["K"],
                                                 th_local=B.TH_LOCAL)
        runner.reserve(steps, False)
        runner.run(chain(False), 3, first=0, resident_slots=M)          # warm-up of the same shape
        ctx.timer_mark(0)
        out = runner.run(chain(True), steps, first=3 % M, resident_slots=M)
        ctx.timer_mark(1)
        ms = ctx.timer_elapsed_ms() / steps
        last_t = (3 + steps) * T - 1
        return {"workload": f"config-B plane sequence as RGB-D: {W}x{H} gray + uint16 depth (x{factor:g}, 5% holes), nFeatures={cfg['nfeat']}, "
                            f"{T} frames per batch, {M} staged batches cycled, local map K={cfg['K']}",
                "value": T / (ms * 1e-3), "unit": B.UNIT, "ms_per_step": ms, "steps": steps,
                "matches_per_frame": float(out["n_matches"].mean()), "local_matches_per_frame": float(out["n_local_matches"].mean()),
                "inliers_per_frame": float(out["n_inliers"].mean()),
                "pose_x_error_m_last_frame": float(abs(out["poses"][-1, 4] - seq.pose(last_t)[4])),
                "timing": "CUDA events on the library stream around ONE rgbl_track_sequence_rgbd call of K steps (resident-staged inputs)"}
    finally:
        ctx.close()


def depth_png(factor, with_cpu, n=32, reps=5):
    cfg = B.CONFIGS["B"]
    W, H = cfg["W"], cfg["H"]
    seq = B.make_sequence(cfg, 2000)
    pngs = [S.encode_png16(seq.depth16(f, factor)) for f in range(n)]
    ctx = F.Context(W, H, cfg["nfeat"], max_batch=n)
    try:
        F.decode_png_depth16(ctx, pngs)
        t0 = time.perf_counter()
        for _ in range(reps):
            F.decode_png_depth16(ctx, pngs)
        ms = (time.perf_counter() - t0) * 1e3 / reps
    finally:
        ctx.close()
    res = {"workload": f"{n} 16-bit depth PNG files of {W}x{H} (all five scanline filters), {sum(map(len, pngs)) / n / 1e6:.2f} MB each",
           "ms_per_batch": ms, "frames_per_s": n / (ms * 1e-3),
           "timing": "host wall clock per rgbl_decode_png_depth16 call (it returns after its D2H): parallel zlib inflate on the host, H2D of the "
                     "filtered scanlines, reconstruction on the device, D2H of the uint16 images"}
    if with_cpu:
        import cv2
        cv2.setNumThreads(1)
        t0 = time.perf_counter()
        for b in pngs[:8]:
            cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED)
        res["cpu_reference"] = {"frames_per_s": 8 / (time.perf_counter() - t0), "cores": 1,
                                "kind": "reference (python-cv2 = OpenCV imgcodecs + libpng, the reference's own reader)"}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--factor", type=float, default=256.0)
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    line = {"rgbd_sequence": sequence(args.steps, args.factor), "depth_png_input": depth_png(args.factor, not args.no_cpu),
            "device": gpu.splitlines()[0] if gpu else None}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
