"""Several sequences on one GPU (needs a GPU; writes nothing unless --out): S independent config-B sequences (bench.py's workload, each lane its
own seed) tracked two ways, alternating in one call:
  lanes      one context with rgbl_set_sequences(S): every batch holds S lanes of m frames, one rgbl_track_sequence call;
  contexts   S one-lane contexts, each driven by its own host thread calling rgbl_track_sequence (ctypes drops the GIL during the call).
For S in --lanes, from staged device slots and from pinned host buffers: frames/s in total and per lane and ms per step (one step = one
batch of every lane), best of --reps alternating rounds; each lane's poses and counters compared bit for bit between the two arms; the
chain's ms per step in profiling mode (lanes arm, staged slots); the pose clusters the device runs at once (rgbl_sequence_lanes_resident);
the card's name, power limit and SM clocks from a read-only nvidia-smi query.  Prints one JSON line per measurement and a summary line.
    python tools/bench_sequences.py [--lanes 1,2,4,6,8] [--m 16] [--steps 8] [--reps 3] [--out FILE]"""
import argparse
import json
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import bench as B                                                    # noqa: E402  (CONFIGS, make_sequence, chain thresholds)
from orb_slam3_rgbl_b200 import frontend as F                        # noqa: E402

NB = 2                    # distinct host batches per lane (the looped sequence is back at its start after NB * m frames)


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, check=True)
    return dict(zip(q.split(","), [v.strip() for v in r.stdout.strip().splitlines()[0].split(",")]))


class Lane:
    def __init__(self, cfg, seed):
        self.seq = B.make_sequence(cfg, seed)
        n = NB * cfg["T"]
        self.img = [self.seq.image(t) for t in range(n)]
        self.cloud = [self.seq.cloud(t) for t in range(n)]


def chain(cfg, lane):
    return F.make_chain_params(lane.seq.pose(0), *cfg["cam"], th_last=B.TH_LAST, local_map_frames=cfg["K"], th_local=B.TH_LOCAL)


def make_runner(cfg, lanes, staged):
    """a context and runner for `lanes` (one lane: the separate-contexts arm), host batches filled and, if staged, staged"""
    m, W, H = cfg["T"], cfg["W"], cfg["H"]
    maxp = max(c.shape[1] for l in lanes for c in l.cloud)
    ctx = F.Context(W, H, cfg["nfeat"], max_batch=len(lanes) * m, max_points=maxp)
    ctx.set_sequences(len(lanes), [l.seq.pose(0) for l in lanes])
    r = F.SequenceRunner(ctx, lanes[0].seq.P, F.make_depth_params(bf=cfg["cam"][4]), len(lanes) * m, W, H, maxp, NB)
    for b in range(NB):
        r.set_batch(b, [l.img[b * m + k] for l in lanes for k in range(m)], [l.cloud[b * m + k] for l in lanes for k in range(m)])
        if staged:
            r.stage(b, b)
    return ctx, r


def run(cfg, r, lanes, steps, staged):
    o = r.run(chain(cfg, lanes[0]), steps, resident_slots=NB if staged else 0)
    return {k: np.array(o[k]) for k in ("poses", "n_matches", "n_inliers", "n_local_matches")}


def lane_of(out, S, s, m, steps):
    idx = [b * S * m + s * m + k for b in range(steps) for k in range(m)]
    return {k: v[idx] for k, v in out.items()}


def measure(cfg, lanes, steps, reps, staged):
    S, m = len(lanes), cfg["T"]
    ctx, r = make_runner(cfg, lanes, staged)
    singles = [make_runner(cfg, [l], staged) for l in lanes]
    try:
        run(cfg, r, lanes, 2, staged)                                  # warm-up: graphs, modules, allocations
        for (_, rs), l in zip(singles, lanes):
            run(cfg, rs, [l], 2, staged)
        best_l = best_c = float("inf")
        for _ in range(reps):
            t0 = time.perf_counter(); out_l = run(cfg, r, lanes, steps, staged); best_l = min(best_l, time.perf_counter() - t0)
            outs = [None] * S

            def one(i):
                outs[i] = run(cfg, singles[i][1], [lanes[i]], steps, staged)
            th = [threading.Thread(target=one, args=(i,)) for i in range(S)]
            t0 = time.perf_counter()
            for t in th:
                t.start()
            for t in th:
                t.join()
            best_c = min(best_c, time.perf_counter() - t0)
        same = all(lane_of(out_l, S, s, m, steps)[k].tobytes() == outs[s][k].tobytes() for s in range(S) for k in out_l)
        chain_ms = None
        if staged:
            ctx.profile_enable(True); ctx.profile_reset()
            run(cfg, r, lanes, steps, staged)
            chain_ms = ctx.profile_read()["match"]["ms"] / steps
            ctx.profile_enable(False)
        frames = S * m * steps
        return dict(lanes=S, frames_per_lane_per_step=m, steps=steps, source="staged_slots" if staged else "pinned_host",
                    lanes_fps=frames / best_l, lanes_fps_per_lane=frames / best_l / S, lanes_ms_per_step=1e3 * best_l / steps,
                    contexts_fps=frames / best_c, contexts_fps_per_lane=frames / best_c / S, contexts_ms_per_step=1e3 * best_c / steps,
                    lanes_over_contexts=best_c / best_l, poses_identical=bool(same), chain_ms_per_step_profiled=chain_ms)
    finally:
        ctx.close()
        for c, _ in singles:
            c.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", default="1,2,4,6,8")
    ap.add_argument("--m", type=int, default=16, help="frames per lane per step")
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    cfg = dict(B.CONFIGS["B"], T=a.m, M=NB)
    Ss = [int(x) for x in a.lanes.split(",")]
    pool = [Lane(cfg, 2000 + 17 * i) for i in range(max(Ss))]
    info = gpu_info()
    probe = F.Context(cfg["W"], cfg["H"], cfg["nfeat"])
    resident = probe.sequence_lanes_resident()
    probe.close()
    rows = []
    for staged in (True, False):
        for S in Ss:
            row = measure(cfg, pool[:S], a.steps, a.reps, staged)
            print(json.dumps(row), flush=True)
            rows.append(row)
    summary = dict(gpu=info, lanes_resident=resident, workload=f"config B lanes: {cfg['W']}x{cfg['H']}, {cfg['nfeat']} features, K={cfg['K']}",
                   all_poses_identical=all(r["poses_identical"] for r in rows))
    print(json.dumps(summary), flush=True)
    if a.out:
        Path(a.out).write_text(json.dumps(dict(summary=summary, rows=rows), indent=1))


if __name__ == "__main__":
    main()
