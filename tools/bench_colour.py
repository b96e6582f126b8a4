"""Colour camera input (needs a GPU; writes nothing): the cvtColor of Tracking::GrabImageRGBL / GrabImageRGBD / GrabImageStereo on the
device (rgbl_set_input_channels) against the same context fed images converted to gray on the host beforehand.  Per input kind, with
3-channel RGB images (Camera.RGB = 1): frames (pairs) per second through the sequence runner from staged device slots and from pinned
host images; the `pyramid` stage of one batch (profiling mode 2: no two kernels of the context overlap), which holds the gray conversion
(fused with the resize or the remap when they are on); and cv2 on one host core (cvtColor, after resize / remap when they are on) of one
image (pair), for comparison.  Prints one JSON line.
    --kind rgbl    KITTI-like RGB-L sequence of bench.py's config B (1241x376, 32 frames per batch, LiDAR clouds);
    --kind rgbd    the same images with uint16 depth images (x256), as tools/bench_rgbd.py;
    --kind stereo  the rectified plane sequence of tools/bench_stereo.py (1241x376, 32 pairs per batch); --resize WxH: 1280x720 pairs
                   tracked at W x H; --rectify: the raw pairs of the EuRoC-like rig (752x480), or with --resize the scale maps at W x H.
    python tools/bench_colour.py --kind rgbl|rgbd|stereo [--steps K] [--resize WxH] [--rectify]"""
import argparse
import json
import subprocess
import sys
import time
import zlib
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import bench as B                                                    # noqa: E402  (CONFIGS, make_sequence, chain thresholds)
import bench_stereo as BS                                            # noqa: E402  (stereo workloads)
from orb_slam3_rgbl_b200 import frontend as F, synthetic as S       # noqa: E402

M = 4


class Workload:
    """the sequence of one kind: colour(t) the camera's RGB image(s) of frame t, gray(t) the host's conversion (after cv2's resize or
    remap of the colour image); the context's size, camera and settings"""

    def __init__(self, kind, size, rectify):
        import cv2
        self.kind, self.size, self.rectify = kind, size, rectify
        self.maps = None
        if kind == "stereo":
            self.T, nfeat = BS.T, 2000
            if size:
                seq = S.PlaneSequence(2000, M * self.T, W=BS.RESIZE_SRC[0], H=BS.RESIZE_SRC[1], cam=BS.RESIZE_CAM, loop=M * self.T)
                self.maps = BS.scale_maps(seq, *size) * 2 if rectify else None
                self.cam = BS.resized_cam(seq, *size)
            elif rectify:
                seq = S.PlaneSequence(2000, M * self.T, W=S.EUROC_W, H=S.EUROC_H, cam=S.EUROC_CAM, dist=S.EUROC_DIST, loop=M * self.T)
                self.maps = seq.rectification_maps() * 2
                self.cam = seq.cam
            else:
                seq = BS.make_sequence()
                self.cam = seq.cam
            self.W, self.H = size or (seq.W, seq.H)
            self.colour = lambda t: [np.ascontiguousarray(S.colorize(side[0], t + 7 * s)) for s, side in enumerate(BS.pair_images(seq, [t]))]
        else:
            cfg = B.CONFIGS["B"]
            self.T, nfeat, self.cam = cfg["T"], cfg["nfeat"], cfg["cam"]
            seq = B.make_sequence(cfg, 1000)
            self.W, self.H = seq.W, seq.H
            self.colour = lambda t: [np.ascontiguousarray(S.colorize(seq.image(t), t))]
        self.seq, self.nfeat = seq, nfeat
        self.in_size = (seq.W, seq.H)

        def to_gray(img, cam_idx=0):
            if self.maps is not None:
                img = cv2.remap(img, self.maps[2 * cam_idx], self.maps[2 * cam_idx + 1], cv2.INTER_LINEAR)
            elif size:
                img = cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)
            return cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
        self.to_gray = to_gray
        self.cache = {}

    def frames(self, t, colour):
        if (t, colour) not in self.cache:
            c = self.colour(t)
            self.cache[(t, colour)] = c if colour else [self.to_gray(i, k) for k, i in enumerate(c)]
        return self.cache[(t, colour)]

    def context(self, colour):
        """a context at the tracking size; colour: RGB input (converted on the device, with the resize / remap when on)"""
        ctx = F.Context(self.W, self.H, self.nfeat, max_batch=2 * self.T if self.kind == "stereo" else self.T,
                        max_points=self.seq.cloud(0).shape[1] if self.kind == "rgbl" else 0)
        if colour:
            ctx.set_input_channels(3, True)
            if self.size:
                ctx.set_input_resize(*self.in_size)
            if self.maps is not None:
                ctx.set_stereo_rectification(*self.maps)
        return ctx


def runner_for(wl, ctx, colour):
    T = wl.T
    W, H = wl.in_size if colour else (wl.W, wl.H)
    ch = 3 if colour else 1
    if wl.kind == "stereo":
        r = F.SequenceRunner.stereo(ctx, float(np.float32(wl.cam[4]) / np.float32(wl.cam[0])), float(wl.cam[4]), T, W, H, M, channels=ch)
    elif wl.kind == "rgbd":
        r = F.SequenceRunner.rgbd(ctx, F.depth_map_factor(256.0), wl.cam[4], T, W, H, M, channels=ch)
    else:
        r = F.SequenceRunner(ctx, wl.seq.P, F.make_depth_params(bf=wl.cam[4]), T, W, H, wl.seq.cloud(0).shape[1], M, channels=ch)
    for m in range(M):
        ts = range(m * T, (m + 1) * T)
        imgs = [wl.frames(t, colour) for t in ts]
        second = ([i[1] for i in imgs] if wl.kind == "stereo" else [wl.seq.depth16(t, 256.0) for t in ts] if wl.kind == "rgbd"
                  else [wl.seq.cloud(t) for t in ts])
        r.set_batch(m, [i[0] for i in imgs], second)
    return r


def throughput(wl, colour, resident, steps):
    ctx = wl.context(colour)
    try:
        runner = runner_for(wl, ctx, colour)
        if resident:
            for m in range(M):
                runner.stage(m, m)
        th_last, th_local = (BS.TH_LAST, BS.TH_LOCAL) if wl.kind == "stereo" else (B.TH_LAST, B.TH_LOCAL)
        chain = lambda cont: F.make_chain_params(wl.seq.pose(0), *wl.cam, th_last=th_last, continue_sequence=cont, local_map_frames=3, th_local=th_local)
        slots = M if resident else 0
        runner.reserve(steps, False)
        runner.run(chain(False), 3, first=0, resident_slots=slots)          # warm-up of the same shape
        ctx.timer_mark(0)
        out = runner.run(chain(True), steps, first=3 % M, resident_slots=slots)
        ctx.timer_mark(1)
        ms = ctx.timer_elapsed_ms() / steps
        return {"value": wl.T / (ms * 1e-3), "unit": "stereo pairs/s" if wl.kind == "stereo" else "frames/s", "ms_per_step": ms,
                "h2d_MB_per_step": runner.h2d_bytes_per_batch() / 1e6, "inliers_per_frame": float(out["n_inliers"].mean()),
                "poses_crc32": zlib.crc32(out["poses"].tobytes())}
    finally:
        ctx.close()


def pyramid_stage(wl, colour, reps=20):
    ctx = wl.context(colour)
    try:
        imgs = [wl.frames(t, colour) for t in range(wl.T)]
        if wl.kind == "stereo":
            b = F.StereoBatch(ctx, [i[0] for i in imgs], [i[1] for i in imgs], pinned=False)
            run = lambda: b.process_resident(float(np.float32(wl.cam[4]) / np.float32(wl.cam[0])), float(wl.cam[4]))
        elif wl.kind == "rgbd":
            b = F.RgbdBatch(ctx, [i[0] for i in imgs], [wl.seq.depth16(t, 256.0) for t in range(wl.T)], pinned=False)
            run = lambda: b.process_resident(F.depth_map_factor(256.0), wl.cam[4])
        else:
            b = F.RgblBatch(ctx, [i[0] for i in imgs], [wl.seq.cloud(t) for t in range(wl.T)], wl.seq.P, F.make_depth_params(bf=wl.cam[4]), pinned=False)
            run = b.process_resident
        b.upload()
        run()
        ctx.profile_enable(2); ctx.profile_reset()
        for _ in range(reps):
            run()
        prof = ctx.profile_read()
        ctx.profile_enable(0)
        return prof["pyramid"]["ms"] / reps
    finally:
        ctx.close()


def host_ms(wl, reps=30):
    """cv2 on one host core: what the host does per image (pair) in the host-converted arm"""
    import cv2
    cv2.setNumThreads(1)
    imgs = wl.frames(0, True)
    for _ in range(3):
        [wl.to_gray(i, k) for k, i in enumerate(imgs)]
    t0 = time.perf_counter()
    for _ in range(reps):
        [wl.to_gray(i, k) for k, i in enumerate(imgs)]
    return (time.perf_counter() - t0) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", choices=["rgbl", "rgbd", "stereo"], required=True)
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--resize", metavar="WxH", help="stereo: 1280x720 pairs tracked at W x H (rgbl_set_input_resize)")
    ap.add_argument("--rectify", action="store_true", help="stereo: remapped pairs (rgbl_set_stereo_rectification)")
    args = ap.parse_args()
    if args.kind != "stereo" and (args.resize or args.rectify):
        ap.error("--resize and --rectify apply to --kind stereo")
    size = tuple(int(v) for v in args.resize.lower().split("x")) if args.resize else None
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    wl = Workload(args.kind, size, args.rectify)
    step = "resize + cvtColor" if size and not args.rectify else "remap + cvtColor" if wl.maps is not None else "cvtColor"
    line = {"workload": f"{args.kind}: RGB camera images {wl.in_size[0]}x{wl.in_size[1]}x3 tracked at {wl.W}x{wl.H} ({step}), nFeatures {wl.nfeat}, "
                        f"{wl.T} {'pairs' if args.kind == 'stereo' else 'frames'} per batch, {M} batches cycled, local map K=3",
            "device_colour": {"resident": throughput(wl, True, True, args.steps), "host": throughput(wl, True, False, args.steps)},
            "host_converted_gray": {"resident": throughput(wl, False, True, args.steps), "host": throughput(wl, False, False, args.steps)},
            "pyramid_stage_ms_per_batch": {"device_colour": pyramid_stage(wl, True), "host_converted_gray": pyramid_stage(wl, False)},
            f"cv2_{step.replace(' + ', '_').lower()}_one_{'pair' if args.kind == 'stereo' else 'image'}_one_host_core_ms": host_ms(wl),
            "timing": "rates: CUDA events around ONE sequence-runner call of K steps (resident: staged device slots; host: pinned host images, H2D "
                      "inside the call); poses_crc32 equal in both arms = bitwise the same poses; pyramid: rgbl_profile_enable(ctx, 2) over 20 "
                      "process calls of one batch; cv2: host wall clock, cv2.setNumThreads(1)",
            "device": gpu.splitlines()[0] if gpu else None}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
