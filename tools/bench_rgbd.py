"""RGB-D throughput (needs a GPU; writes nothing): System::TrackRGBD as in Examples/RGB-D/rgbd_kitti.cc on the workload of bench.py's
config B, with uint16 depth images (KITTI depth PNG scale x256, 5 % holes) instead of point clouds, tracked through
rgbl_track_sequence_rgbd from staged device slots; and 32 KITTI-size 16-bit depth PNGs through rgbl_decode_png_depth16, with a
one-core python-cv2 imdecode arm.  Prints one JSON line.
--camera tum1: the RGB-D sequence on a 640x480 camera with TUM1's calibration and distortion (k1..k3 != 0; a plane 3 m away, depth x5000),
so that every frame construction also undistorts its keypoints: frames/s, the depth-gather stage per batch with and without the
distortion (profiling mode 2, no overlap between kernels), and the final pose error, also for the same images tracked as if k1 = 0.
--resize WxH: RGB-D frames of a 1280x720 camera (gray + uint16 depth) tracked at W x H (integer factors), resized on the device
(rgbl_set_input_resize) against the same context fed frames resized on the host beforehand, from staged slots and from pinned host
buffers; the `pyramid` and `depth_gather` stages of one batch with and without the resize (profiling mode 2); and cv2.resize of one image
and its depth image on one host core.
    python tools/bench_rgbd.py [--steps K] [--no-cpu] [--camera kitti|tum1] [--resize WxH]"""
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


TUM1_K = (S.TUM1_FX, S.TUM1_FY, S.TUM1_CX, S.TUM1_CY)


def sequence_tum1(steps, reps=20):
    T, M, K, nfeat, W, H = 32, 4, 3, 1000, S.TUM_W, S.TUM_H
    cam = TUM1_K + (S.TUM1_BF,)
    seq = S.PlaneSequence(2000, M * T, Z=3.0, W=W, H=H, loop=M * T, cam=cam, dist=S.TUM1_DIST)
    batches = [[seq.image(t) for t in range(m * T, (m + 1) * T)] for m in range(M)]
    depths = [[seq.depth16(t, S.TUM_DEPTH_FACTOR) for t in range(m * T, (m + 1) * T)] for m in range(M)]
    scale = F.depth_map_factor(S.TUM_DEPTH_FACTOR)

    def run(dist):
        ctx = F.Context(W, H, nfeat, max_batch=T)
        try:
            bounds = ctx.set_camera_distortion(*TUM1_K, dist)
            runner = F.SequenceRunner.rgbd(ctx, scale, S.TUM1_BF, T, W, H, M, pinned=True)
            for m in range(M):
                runner.set_batch(m, batches[m], depths[m])
                runner.stage(m, m)
            chain = lambda cont: F.make_chain_params(seq.pose(0), *cam, th_last=B.TH_LAST, continue_sequence=cont, local_map_frames=K,
                                                     th_local=B.TH_LOCAL)
            runner.reserve(steps, False)
            runner.run(chain(False), 3, first=0, resident_slots=M)          # warm-up of the same shape
            ctx.timer_mark(0)
            out = runner.run(chain(True), steps, first=3 % M, resident_slots=M)
            ctx.timer_mark(1)
            ms = ctx.timer_elapsed_ms() / steps
            truth = np.array([seq.pose(t)[4] for t in range(3 * T, (3 + steps) * T)])
            # frame construction alone, stage by stage (profiling mode 2: no two kernels of the context overlap), in a run of its own
            b = F.RgbdBatch(ctx, batches[0], depths[0], pinned=False)
            b.upload(); b.process_resident(scale, S.TUM1_BF)
            ctx.profile_enable(2); ctx.profile_reset()
            for _ in range(reps):
                b.process_resident(scale, S.TUM1_BF)
            prof = ctx.profile_read()
            ctx.profile_enable(0)
            g = prof["depth_gather"]
            return {"frames_per_s": T / (ms * 1e-3), "ms_per_step": ms, "bounds": [float(v) for v in bounds],
                    "inliers_per_frame": float(out["n_inliers"].mean()),
                    "pose_x_error_m_last_frame": float(abs(out["poses"][-1, 4] - truth[-1])),
                    "pose_x_error_m_max": float(np.abs(out["poses"][:, 4] - truth).max()),
                    "depth_gather_ms_per_batch": g["ms"] / max(g["calls"], 1), "depth_gather_launches_per_batch": g["launches"] / max(g["calls"], 1),
                    "frame_construction_ms_per_batch": sum(v["ms"] for k, v in prof.items() if not k.startswith("_") and k not in ("match", "pose")) / reps}
        finally:
            ctx.close()

    dist_on, k1_zero = run(S.TUM1_DIST), run(np.zeros(5, np.float32))
    return {"workload": f"plane sequence {W}x{H} through TUM1's lens (k1..k3 != 0) as RGB-D: gray + uint16 depth (x5000, 5% holes), "
                        f"nFeatures={nfeat}, {T} frames per batch, {M} staged batches cycled, local map K={K}",
            "value": dist_on["frames_per_s"], "unit": B.UNIT, "steps": steps, "distortion": dist_on, "same_images_as_if_k1_0": k1_zero,
            "undistort_ms_per_batch": dist_on["depth_gather_ms_per_batch"] - k1_zero["depth_gather_ms_per_batch"],
            "timing": "frames/s: CUDA events around ONE rgbl_track_sequence_rgbd call of K steps (resident-staged inputs); stage times: "
                      f"rgbl_profile_enable(ctx, 2) over {reps} rgbl_resident_process_rgbd calls of one batch; undistort_ms_per_batch = the "
                      "difference of the depth-gather stage with and without the distortion"}


RESIZE_SRC, RESIZE_CAM = (1280, 720), (700.0, 700.0, 640.0, 360.0, 140.0)      # the camera's size and fx, fy, cx, cy, bf


def resize_line(steps, gpu, w, h, factor=1000.0, reps=20):
    import cv2
    T, M, K, nfeat = 32, 4, 3, 2000
    seq = S.PlaneSequence(2000, M * T, W=RESIZE_SRC[0], H=RESIZE_SRC[1], cam=RESIZE_CAM, loop=M * T)
    sx, sy = np.float32(w / seq.W), np.float32(h / seq.H)
    fx, fy, cx, cy, bf = (np.float32(v) for v in RESIZE_CAM)
    cam = (float(fx * sx), float(fy * sy), float(cx * sx), float(cy * sy), float(bf * sx))      # Settings' intrinsics at the new size
    scale = F.depth_map_factor(factor)
    big = [([seq.image(t) for t in range(m * T, (m + 1) * T)], [seq.depth16(t, factor) for t in range(m * T, (m + 1) * T)]) for m in range(M)]
    rs = lambda a: cv2.resize(a, (w, h), interpolation=cv2.INTER_LINEAR)
    small = [([rs(i) for i in imgs], [rs(d) for d in deps]) for imgs, deps in big]

    def run(batches, on, resident):
        ctx = F.Context(w, h, nfeat, max_batch=T)
        try:
            if on:
                ctx.set_input_resize(*RESIZE_SRC)
            iw, ih = batches[0][0][0].shape[::-1]
            runner = F.SequenceRunner.rgbd(ctx, scale, cam[4], T, iw, ih, M, pinned=True)
            for m in range(M):
                runner.set_batch(m, *batches[m])
                if resident:
                    runner.stage(m, m)
            chain = lambda cont: F.make_chain_params(seq.pose(0), *cam, th_last=B.TH_LAST, continue_sequence=cont, local_map_frames=K, th_local=B.TH_LOCAL)
            slots = M if resident else 0
            runner.reserve(steps, False)
            runner.run(chain(False), 3, first=0, resident_slots=slots)          # warm-up of the same shape
            ctx.timer_mark(0)
            out = runner.run(chain(True), steps, first=3 % M, resident_slots=slots)
            ctx.timer_mark(1)
            ms = ctx.timer_elapsed_ms() / steps
            res = {"frames_per_s": T / (ms * 1e-3), "ms_per_step": ms, "inliers_per_frame": float(out["n_inliers"].mean())}
            if resident:       # frame construction alone, stage by stage (profiling mode 2), in a run of its own
                b = F.RgbdBatch(ctx, *batches[0], pinned=False)
                b.upload(); b.process_resident(scale, cam[4])
                ctx.profile_enable(2); ctx.profile_reset()
                for _ in range(reps):
                    b.process_resident(scale, cam[4])
                prof = ctx.profile_read()
                ctx.profile_enable(0)
                res["stages_ms_per_batch"] = {k: v["ms"] / reps for k, v in prof.items() if not k.startswith("_") and v["calls"]}
            return res
        finally:
            ctx.close()

    cv2.setNumThreads(1)
    img, dep = big[0][0][0], big[0][1][0]
    for _ in range(3):
        rs(img); rs(dep)
    t0 = time.perf_counter()
    for _ in range(50):
        rs(img); rs(dep)
    host_ms = (time.perf_counter() - t0) * 1e3 / 50
    on_res, off_res = run(big, True, True), run(small, False, True)
    return {"workload": f"plane sequence {seq.W}x{seq.H} as RGB-D (gray + uint16 depth x{factor:g}, 5% holes) tracked at {w}x{h}, nFeatures={nfeat}, "
                        f"{T} frames per batch, {M} batches cycled, local map K={K}",
            "device_resize": {"resident": on_res, "host": run(big, True, False)},
            "host_resized_inputs": {"resident": off_res, "host": run(small, False, False)},
            "pyramid_stage_ms_per_batch": {"device_resize": on_res["stages_ms_per_batch"].get("pyramid", 0.0),
                                           "host_resized_inputs": off_res["stages_ms_per_batch"].get("pyramid", 0.0)},
            "depth_gather_stage_ms_per_batch": {"device_resize": on_res["stages_ms_per_batch"].get("depth_gather", 0.0),
                                                "host_resized_inputs": off_res["stages_ms_per_batch"].get("depth_gather", 0.0)},
            "cv2_resize_image_and_depth_one_host_core_ms": host_ms,
            "timing": "frames/s: CUDA events around ONE rgbl_track_sequence_rgbd call of K steps (resident: staged device slots; host: pinned host "
                      "buffers, H2D inside the call); host_resized_inputs: the same context without the resize, fed frames resized on the host "
                      f"before the measurement; stages: rgbl_profile_enable(ctx, 2) over {reps} rgbl_resident_process_rgbd calls of one batch; "
                      "cv2: host wall clock, cv2.setNumThreads(1), one image and its depth image",
            "device": gpu.splitlines()[0] if gpu else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--factor", type=float, default=256.0)
    ap.add_argument("--no-cpu", action="store_true")
    ap.add_argument("--camera", choices=("kitti", "tum1"), default="kitti")
    ap.add_argument("--resize", metavar="WxH", help="measure the input resize from 1280x720 to W x H instead (see the module docstring)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if args.resize:
        w, h = (int(v) for v in args.resize.lower().split("x"))
        line = {"rgbd_resize": resize_line(args.steps, gpu, w, h)}
    elif args.camera == "tum1":
        line = {"rgbd_sequence_tum1": sequence_tum1(args.steps), "device": gpu.splitlines()[0] if gpu else None}
    else:
        line = {"rgbd_sequence": sequence(args.steps, args.factor), "depth_png_input": depth_png(args.factor, not args.no_cpu),
                "device": gpu.splitlines()[0] if gpu else None}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
