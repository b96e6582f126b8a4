"""Stereo throughput (needs a GPU; writes nothing): System::TrackStereo as in Examples/Stereo/stereo_kitti.cc at the geometry of bench.py's
config C (1241x376, nFeatures 2000) on a rectified plane sequence (PlaneSequence.right_image: 5 px disparity), 32 pairs per batch (one
batched extraction of 64 images + ComputeStereoMatches), tracked through rgbl_track_sequence_stereo from staged device slots and from pinned
host buffers.  Also the stage times of one batch's frame construction (profiling mode 2: no two kernels of the context overlap): the
extraction of the 64 images and the stereo `match` stage, at nFeatures 2000 and 4000.  Prints one JSON line.
--rectify: instead, the raw pairs of a distorted EuRoC-like rig (752x480, PlaneSequence.raw_left_image / raw_right_image) tracked with and
without rectification on the device (rgbl_set_stereo_rectification), from staged slots and from pinned host images; the `pyramid` stage of
one batch with and without rectification (profiling mode 2); and, for comparison, cv2.remap of one pair on one host core.
--resize WxH: camera pairs of 1280x720 (a pinhole plane sequence) tracked at W x H, resized on the device (rgbl_set_input_resize) against the
same context fed pairs resized on the host beforehand, from staged slots and from pinned host images; the `pyramid` stage of one batch with
and without the resize (profiling mode 2); and cv2.resize of one pair on one host core.  With --rectify too, the pairs are remapped instead
(maps at W x H whose coordinates index the 1280x720 images, as Settings builds them with a new image size).
    python tools/bench_stereo.py [--steps K] [--rectify] [--resize WxH]"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench as B                                                    # noqa: E402  (CONFIGS, UNIT)
from orb_slam3_rgbl_b200 import frontend as F, synthetic as S       # noqa: E402

T, M, K = 32, 4, 3
TH_LAST, TH_LOCAL = 7.0, 1.0          # System::STEREO: src/Tracking.cc:2913-2917, :3432-3436


def make_sequence():
    cfg = B.CONFIGS["C"]
    return S.PlaneSequence(2000, M * T, W=cfg["W"], H=cfg["H"], loop=M * T)


def sequence(seq, steps, resident, maps=None, size=None, images=None):
    """size: (w, h) of the context with the input resize on (the pairs keep the sequence's size); images(ts): the pairs of frames ts
    (default pair_images), cam: the camera of the context (default the sequence's)"""
    W, H, nfeat = seq.W, seq.H, B.CONFIGS["C"]["nfeat"]
    cam = seq.cam if size is None else resized_cam(seq, *size)
    mb, mbf = float(np.float32(cam[4]) / np.float32(cam[0])), float(cam[4])
    ctx = F.Context(*(size or (W, H)), nfeat, max_batch=2 * T)
    images = images or (lambda ts: pair_images(seq, ts))
    try:
        if size is not None:
            ctx.set_input_resize(W, H)
        if maps is not None:
            ctx.set_stereo_rectification(*maps)
        W, H = images([0])[0][0].shape[::-1]
        runner = F.SequenceRunner.stereo(ctx, mb, mbf, T, W, H, M, pinned=True)
        for m in range(M):
            ts = range(m * T, (m + 1) * T)
            runner.set_batch(m, *images(ts))
            if resident:
                runner.stage(m, m)
        chain = lambda cont: F.make_chain_params(seq.pose(0), *cam, th_last=TH_LAST, continue_sequence=cont, local_map_frames=K, th_local=TH_LOCAL)
        slots = M if resident else 0
        runner.reserve(steps, False)
        runner.run(chain(False), 3, first=0, resident_slots=slots)          # warm-up of the same shape
        ctx.timer_mark(0)
        out = runner.run(chain(True), steps, first=3 % M, resident_slots=slots)
        ctx.timer_mark(1)
        ms = ctx.timer_elapsed_ms() / steps
        truth = np.array([seq.pose(t)[4] for t in range(3 * T, (3 + steps) * T)])
        return {"value": T / (ms * 1e-3), "unit": "stereo pairs/s", "ms_per_step": ms, "steps": steps,
                "matches_per_frame": float(out["n_matches"].mean()), "local_matches_per_frame": float(out["n_local_matches"].mean()),
                "inliers_per_frame": float(out["n_inliers"].mean()), "pose_x_error_m_max": float(np.abs(out["poses"][:, 4] - truth).max())}
    finally:
        ctx.close()


def pair_images(seq, ts):
    """(lefts, rights) of frames ts: the rectified views of a pinhole sequence, the raw views of a distorted one"""
    if seq.dist is None:
        return [seq.image(t) for t in ts], [seq.right_image(t) for t in ts]
    return [seq.raw_left_image(t) for t in ts], [seq.raw_right_image(t) for t in ts]


def stages(seq, nfeat, reps=20, maps=None, size=None, images=None):
    """one batch of T pairs: rgbl_resident_process_stereo under profiling mode 2 -> per-batch stage times (size, images: as for sequence)"""
    W, H = seq.W, seq.H
    cam = seq.cam if size is None else resized_cam(seq, *size)
    mb, mbf = float(np.float32(cam[4]) / np.float32(cam[0])), float(cam[4])
    ctx = F.Context(*(size or (W, H)), nfeat, max_batch=2 * T)
    images = images or (lambda ts: pair_images(seq, ts))
    try:
        if size is not None:
            ctx.set_input_resize(W, H)
        if maps is not None:
            ctx.set_stereo_rectification(*maps)
        b = F.StereoBatch(ctx, *images(range(T)), pinned=False)
        b.upload()
        n = b.process_resident(mb, mbf).copy()
        depth = [np.array(fr[2]) for fr in b.download()]
        ctx.profile_enable(2); ctx.profile_reset()
        for _ in range(reps):
            b.process_resident(mb, mbf)
        prof = ctx.profile_read()
        ctx.profile_enable(0)
        per = {k: v["ms"] / reps for k, v in prof.items() if not k.startswith("_") and v["calls"]}
        return {"nfeatures": nfeat, "left_keypoints_per_frame": float(n.mean()), "stereo_matches_per_frame": float(np.mean([(d > 0).sum() for d in depth])),
                "extract_64_images_ms": sum(v for k, v in per.items() if k not in ("match", "pose")),
                "stereo_match_ms": per.get("match", 0.0), "match_launches_per_batch": prof["match"]["launches"] / reps,
                "stages_ms": per}
    finally:
        ctx.close()


def host_remap_ms(seq, maps, reps=50):
    """cv2.remap of one raw pair (both images) on one host core, wall clock per pair"""
    import time
    import cv2
    cv2.setNumThreads(1)
    l, r = pair_images(seq, [0])
    m1l, m2l, m1r, m2r = maps
    for _ in range(3):
        cv2.remap(l[0], m1l, m2l, cv2.INTER_LINEAR); cv2.remap(r[0], m1r, m2r, cv2.INTER_LINEAR)
    t0 = time.perf_counter()
    for _ in range(reps):
        cv2.remap(l[0], m1l, m2l, cv2.INTER_LINEAR); cv2.remap(r[0], m1r, m2r, cv2.INTER_LINEAR)
    return (time.perf_counter() - t0) * 1e3 / reps


RESIZE_SRC = (1280, 720)
RESIZE_CAM = (700.0, 700.0, 640.0, 360.0, 140.0)      # fx, fy, cx, cy, bf of the 1280x720 camera (baseline 0.2 m, 7 px disparity)


def resized_cam(seq, w, h):
    """Settings' intrinsics at the new size: fx, cx by w / width, fy, cy by h / height, bf = b * fx"""
    sx, sy = np.float32(w / seq.W), np.float32(h / seq.H)
    fx, fy, cx, cy, bf = (np.float32(v) for v in seq.cam)
    return float(fx * sx), float(fy * sy), float(cx * sx), float(cy * sy), float(bf * sx)


def scale_maps(seq, w, h):
    """M1, M2 at w x h indexing the sequence's images: a pure scale, as a rig without distortion would have"""
    xs, ys = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    return [np.ascontiguousarray((xs + 0.5) * seq.W / w - 0.5, np.float32), np.ascontiguousarray((ys + 0.5) * seq.H / h - 0.5, np.float32)]


def host_resize_ms(seq, w, h, reps=50):
    """cv2.resize of one pair (both images) on one host core, wall clock per pair"""
    import time
    import cv2
    cv2.setNumThreads(1)
    l, r = pair_images(seq, [0])
    for _ in range(3):
        cv2.resize(l[0], (w, h), interpolation=cv2.INTER_LINEAR); cv2.resize(r[0], (w, h), interpolation=cv2.INTER_LINEAR)
    t0 = time.perf_counter()
    for _ in range(reps):
        cv2.resize(l[0], (w, h), interpolation=cv2.INTER_LINEAR); cv2.resize(r[0], (w, h), interpolation=cv2.INTER_LINEAR)
    return (time.perf_counter() - t0) * 1e3 / reps


def resize_line(steps, gpu, w, h, rectify):
    import cv2
    seq = S.PlaneSequence(2000, M * T, W=RESIZE_SRC[0], H=RESIZE_SRC[1], cam=RESIZE_CAM, loop=M * T)
    maps = scale_maps(seq, w, h) * 2 if rectify else None
    if rectify:
        small = lambda ts: tuple([cv2.remap(i, maps[0], maps[1], cv2.INTER_LINEAR) for i in side] for side in pair_images(seq, ts))
    else:
        small = lambda ts: tuple([cv2.resize(i, (w, h), interpolation=cv2.INTER_LINEAR) for i in side] for side in pair_images(seq, ts))
    on = dict(size=(w, h), maps=maps)
    off = dict(size=(w, h), images=small)
    st_on, st_off = stages(seq, 2000, **on), stages_plain(seq, 2000, w, h, small)
    return {"workload": f"pinhole plane sequence {seq.W}x{seq.H} tracked at {w}x{h}" + (" (rectification maps at the new size)" if rectify else "")
                        + f", nFeatures 2000, {T} pairs per batch, {M} batches cycled, local map K={K}, th_last {TH_LAST:g}, th_local {TH_LOCAL:g}",
            "device_resize": {"resident": sequence(seq, steps, True, **on), "host": sequence(seq, steps, False, **on)},
            "host_resized_inputs": {"resident": sequence_plain(seq, steps, True, w, h, small), "host": sequence_plain(seq, steps, False, w, h, small)},
            "pyramid_stage_ms_per_batch": {"device_resize": st_on["stages_ms"].get("pyramid", 0.0), "host_resized_inputs": st_off["stages_ms"].get("pyramid", 0.0)},
            "stages_per_batch": {"device_resize": st_on, "host_resized_inputs": st_off},
            ("cv2_remap_one_pair_one_host_core_ms" if rectify else "cv2_resize_one_pair_one_host_core_ms"):
                host_remap_ms(seq, maps) if rectify else host_resize_ms(seq, w, h),
            "timing": "pairs/s: CUDA events around ONE rgbl_track_sequence_stereo call of K steps (resident: staged device slots; host: pinned host "
                      "images, H2D inside the call); host_resized_inputs: the same context without the resize, fed pairs resized (remapped) on "
                      "the host before the measurement; stages: rgbl_profile_enable(ctx, 2) over 20 rgbl_resident_process_stereo calls of one "
                      "batch; cv2: host wall clock, cv2.setNumThreads(1), both images of one pair",
            "device": gpu.splitlines()[0] if gpu else None}


def sequence_plain(seq, steps, resident, w, h, images):
    """the context at w x h without the resize, fed the pairs images(ts) already at w x h"""
    ctx_seq = _Resized(seq, w, h)
    return sequence(ctx_seq, steps, resident, images=images)


def stages_plain(seq, nfeat, w, h, images):
    return stages(_Resized(seq, w, h), nfeat, images=images)


class _Resized:
    """the sequence seen by a context of w x h without the input resize: its size and Settings' scaled camera"""

    def __init__(self, seq, w, h):
        self.W, self.H, self.cam, self.pose, self.dist = w, h, resized_cam(seq, w, h), seq.pose, None


def rectify_line(steps, gpu):
    seq = S.PlaneSequence(2000, M * T, W=S.EUROC_W, H=S.EUROC_H, cam=S.EUROC_CAM, dist=S.EUROC_DIST, loop=M * T)
    maps = seq.rectification_maps() * 2
    st_on, st_off = stages(seq, 2000, maps=maps), stages(seq, 2000)
    host_ms = host_remap_ms(seq, maps)
    return {"workload": f"raw pairs of a distorted EuRoC-like rig {seq.W}x{seq.H} (k1 {S.EUROC_DIST[0]:g}, k2 {S.EUROC_DIST[1]:g}), nFeatures 2000, "
                        f"{T} pairs per batch, {M} batches cycled, local map K={K}, th_last {TH_LAST:g}, th_local {TH_LOCAL:g}",
            "rectified": {"resident": sequence(seq, steps, True, maps), "host": sequence(seq, steps, False, maps)},
            "not_rectified": {"resident": sequence(seq, steps, True), "host": sequence(seq, steps, False)},
            "pyramid_stage_ms_per_batch": {"rectified": st_on["stages_ms"].get("pyramid", 0.0), "not_rectified": st_off["stages_ms"].get("pyramid", 0.0)},
            "stages_per_batch": {"rectified": st_on, "not_rectified": st_off},
            "cv2_remap_one_pair_one_host_core_ms": host_ms,
            "timing": "pairs/s: CUDA events around ONE rgbl_track_sequence_stereo call of K steps (resident: staged device slots; host: pinned host "
                      "images, H2D inside the call); stages: rgbl_profile_enable(ctx, 2) over 20 rgbl_resident_process_stereo calls of one batch; "
                      "cv2.remap: host wall clock, cv2.setNumThreads(1), both images of one pair",
            "device": gpu.splitlines()[0] if gpu else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--rectify", action="store_true", help="measure stereo rectification on the device instead (see the module docstring)")
    ap.add_argument("--resize", metavar="WxH", help="measure the input resize from 1280x720 to W x H instead (see the module docstring)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    if args.resize:
        w, h = (int(v) for v in args.resize.lower().split("x"))
        print(json.dumps(resize_line(args.steps, gpu, w, h, args.rectify)))
        return
    if args.rectify:
        print(json.dumps(rectify_line(args.steps, gpu)))
        return
    seq = make_sequence()
    line = {"workload": f"rectified plane sequence {seq.W}x{seq.H} (config-C geometry), disparity {seq.disparity_px()} px, nFeatures "
                        f"{B.CONFIGS['C']['nfeat']}, {T} pairs per batch (one extraction of {2 * T} images), {M} batches cycled, local map K={K}, "
                        f"th_last {TH_LAST:g}, th_local {TH_LOCAL:g}",
            "resident": sequence(seq, args.steps, True), "host": sequence(seq, args.steps, False),
            "stages_per_batch": [stages(seq, 2000), stages(seq, 4000)],
            "timing": "pairs/s: CUDA events around ONE rgbl_track_sequence_stereo call of K steps (resident: staged device slots; host: pinned host "
                      "images, H2D inside the call); stages: rgbl_profile_enable(ctx, 2) over 20 rgbl_resident_process_stereo calls of one batch",
            "device": gpu.splitlines()[0] if gpu else None}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
