"""Development aid (CPU only): how much of PoseOptimization's work repeats itself on the bench sequence.  Runs the oracle chain
(bench.CpuSequence: frame construction, TrackWithMotionModel and TrackLocalMap per frame) over a config's sequence and, for every pose
optimisation, reads the per-round trace of the oracle's code (tests/pose_round_trace.py): a round r >= 1 repeats round r - 1 bit for
bit when no edge level changed after round r - 1 and either the robust flag stays the same or round r - 1 had no Huber linear-region
evaluation.  pose_optimize_kernel skips such rounds; this
prints the share of LM iterations that sit in them.

    python tests/tools/count_pose_rounds.py [--config B] [--frames 128] [--seed 1000]

--frames defaults to the config's whole loop (M x T frames: 128 for config B)."""
import argparse
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import bench  # noqa: E402
import oracle  # noqa: E402
import pose_round_trace  # noqa: E402


def replica_rounds(t):
    """Indices of the rounds of one trace that repeat the round before them."""
    return [r for r in range(1, t["rounds"]) if t["changed"][r - 1] == 0 and ((r < 3) == (r - 1 < 3) or t["linear"][r - 1] == 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="B")
    ap.add_argument("--frames", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1000)
    args = ap.parse_args()
    cfg = dict(bench.CONFIGS[args.config])
    frames = args.frames or cfg["M"] * cfg["T"]
    calls = []
    traced = pose_round_trace.pose_optimize_trace

    def pose_optimize(*a):
        ni, pose, outlier, t = traced(*a)
        calls.append(t)
        return ni, pose, outlier
    oracle.pose_optimize = pose_optimize            # oracle/chain.py calls it through the module
    bench.CpuSequence(cfg, bench.make_sequence(cfg, args.seed)).advance(frames)

    iters = sum(sum(t["iters"]) for t in calls)
    rounds = sum(t["rounds"] for t in calls)
    rep = [replica_rounds(t) for t in calls]
    rep_iters = sum(t["iters"][r] for t, rs in zip(calls, rep) for r in rs)
    per_round = [sum(r in rs for rs in rep) for r in range(4)]
    print(f"config {args.config}, seed {args.seed}, {frames} frames: {len(calls)} pose optimisations, {rounds} rounds, {iters} LM iterations")
    print(f"repeat rounds: {sum(map(len, rep))} (round 1: {per_round[1]}, round 2: {per_round[2]}, round 3: {per_round[3]}), "
          f"holding {rep_iters} LM iterations = {100.0 * rep_iters / max(iters, 1):.1f} %")
    # these start round 3 from the robust system the classification built for round 2: reused when its build had no linear-region edge
    print(f"calls that skip round 2 and run round 3: {sum(1 for rs in rep if 2 in rs and 3 not in rs)}")


if __name__ == "__main__":
    main()
