"""Stereo throughput (needs a GPU; writes nothing): System::TrackStereo as in Examples/Stereo/stereo_kitti.cc at the geometry of bench.py's
config C (1241x376, nFeatures 2000) on a rectified plane sequence (PlaneSequence.right_image: 5 px disparity), 32 pairs per batch (one
batched extraction of 64 images + ComputeStereoMatches), tracked through rgbl_track_sequence_stereo from staged device slots and from pinned
host buffers.  Also the stage times of one batch's frame construction (profiling mode 2: no two kernels of the context overlap): the
extraction of the 64 images and the stereo `match` stage, at nFeatures 2000 and 4000.  Prints one JSON line.
--rectify: instead, the raw pairs of a distorted EuRoC-like rig (752x480, PlaneSequence.raw_left_image / raw_right_image) tracked with and
without rectification on the device (rgbl_set_stereo_rectification), from staged slots and from pinned host images; the `pyramid` stage of
one batch with and without rectification (profiling mode 2); and, for comparison, cv2.remap of one pair on one host core.
    python tools/bench_stereo.py [--steps K] [--rectify]"""
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


def sequence(seq, steps, resident, maps=None):
    W, H, nfeat = seq.W, seq.H, B.CONFIGS["C"]["nfeat"]
    cam = seq.cam
    mb, mbf = float(np.float32(cam[4]) / np.float32(cam[0])), float(cam[4])
    ctx = F.Context(W, H, nfeat, max_batch=2 * T)
    try:
        if maps is not None:
            ctx.set_stereo_rectification(*maps)
        runner = F.SequenceRunner.stereo(ctx, mb, mbf, T, W, H, M, pinned=True)
        for m in range(M):
            ts = range(m * T, (m + 1) * T)
            runner.set_batch(m, *pair_images(seq, ts))
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


def stages(seq, nfeat, reps=20, maps=None):
    """one batch of T pairs: rgbl_resident_process_stereo under profiling mode 2 -> per-batch stage times"""
    W, H, cam = seq.W, seq.H, seq.cam
    mb, mbf = float(np.float32(cam[4]) / np.float32(cam[0])), float(cam[4])
    ctx = F.Context(W, H, nfeat, max_batch=2 * T)
    try:
        if maps is not None:
            ctx.set_stereo_rectification(*maps)
        b = F.StereoBatch(ctx, *pair_images(seq, range(T)), pinned=False)
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
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
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
