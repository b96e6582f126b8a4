"""Sequence lanes (rgbl_set_sequences) on the GPU at config-B geometry (1241 x 376, 2000 features, local map of K = 3 frames): every lane
of a context that tracks S sequences in lockstep equals, bit for bit, a one-lane context given that lane's frames alone.  The one-lane
chain is tied to the oracle by tests/test_gpu_tracking.py.  Covered: the RGB-L runner from staged slots and from pinned host buffers
(S = 2, 4, 8), the manual rgbl_resident_track_begin2 / _end2 API with two chains queued (S = 3), the PDL / graph switches, and a
frame-construction overflow with lanes on."""
import numpy as np
import pytest

from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

W, H, FEAT, K = S.KITTI_W, S.KITTI_H, 2000, 3
M, NB = 2, 3                      # frames per lane per batch; batches (each after the first continues the sequences)
CAM = (S.KITTI_FX, S.KITTI_FY, S.KITTI_CX, S.KITTI_CY, S.KITTI_BF)
PRM = F.make_depth_params(bf=S.KITTI_BF)
KEYS = ("poses", "n_matches", "n_inliers", "n_local_matches")


class Seq:
    """One lane's sequence: NB * M frames of a plane sequence of its own seed, speed and start."""

    def __init__(self, i):
        self.ps = S.PlaneSequence(300 + 11 * i, NB * M + 1, shift_px=5 + (i % 4))
        self.img = [self.ps.image(t) for t in range(NB * M)]
        self.cloud = [self.ps.cloud(t) for t in range(NB * M)]
        self.pose0 = self.ps.pose(0)


SEQS = {}


def seq(i):
    if i not in SEQS:
        SEQS[i] = Seq(i)
    return SEQS[i]


def _frames(lanes, b, attr):
    return [getattr(l, attr)[b * M + k] for l in lanes for k in range(M)]


def _context(lanes, **kw):
    maxp = max(c.shape[1] for l in lanes for c in l.cloud)
    ctx = F.Context(W, H, FEAT, max_batch=len(lanes) * M, max_points=maxp, **kw)
    ctx.set_sequences(len(lanes), [l.pose0 for l in lanes])
    return ctx, maxp


def run_runner(lanes, resident):
    """rgbl_track_sequence over NB batches of len(lanes) * M frames -> dict of per-frame outputs in batch order"""
    ctx, maxp = _context(lanes)
    try:
        T = len(lanes) * M
        r = F.SequenceRunner(ctx, lanes[0].ps.P, PRM, T, W, H, maxp, NB)
        for b in range(NB):
            r.set_batch(b, _frames(lanes, b, "img"), _frames(lanes, b, "cloud"))
        chain = F.make_chain_params(lanes[0].pose0, *CAM, local_map_frames=K)
        if resident:
            for b in range(NB):
                r.stage(b, b)
            o = r.run(chain, NB, resident_slots=NB)
        else:
            o = r.run(chain, NB)
        return {k: np.array(o[k]) for k in KEYS}
    finally:
        ctx.close()


def run_manual(lanes):
    """rgbl_resident_track_begin2 / _end2, batch by batch, with the chains of batches 0 and 1 queued together -> outputs in batch order"""
    ctx, _ = _context(lanes)
    try:
        batches = [F.RgblBatch(ctx, _frames(lanes, b, "img"), _frames(lanes, b, "cloud"), lanes[0].ps.P, PRM, pinned=False) for b in range(NB)]
        outs = []
        for b, batch in enumerate(batches):
            batch.upload(); batch.process_resident()
            batch.track_begin2(F.make_chain_params(lanes[0].pose0, *CAM, continue_sequence=b > 0, local_map_frames=K))
            if b >= 1:
                outs.append(batches[b - 1].track_end2())             # two chains were in flight
        outs.append(batches[-1].track_end2())
        return {k: np.concatenate([o[k] for o in outs]) for k in KEYS + ("n_inliers_first",)}
    finally:
        ctx.close()


def lane_of(out, n_lanes, s):
    idx = [b * n_lanes * M + s * M + k for b in range(NB) for k in range(M)]
    return {k: v[idx] for k, v in out.items()}


SINGLE = {}


def single(i, how):
    key = (i, how)
    if key not in SINGLE:
        SINGLE[key] = run_manual([seq(i)]) if how == "manual" else run_runner([seq(i)], how == "resident")
    return SINGLE[key]


def assert_lanes_equal(out, ids, how):
    for s, i in enumerate(ids):
        got, want = lane_of(out, len(ids), s), single(i, how)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), f"lane {s}: {k} differs from the one-lane run"


@pytest.mark.parametrize("resident", [True, False], ids=["staged_slots", "pinned_host"])
@pytest.mark.parametrize("n_lanes", [2, 4, 8])
def test_runner_lanes_equal_single_sequence(n_lanes, resident):
    ids = list(range(n_lanes))
    out = run_runner([seq(i) for i in ids], resident)
    assert_lanes_equal(out, ids, "resident" if resident else "host")
    assert out["n_local_matches"].max() > 50              # the local map took part


def test_manual_chain_two_queued_three_lanes():
    ids = [1, 3, 5]
    out = run_manual([seq(i) for i in ids])
    assert_lanes_equal(out, ids, "manual")
    assert out["n_inliers_first"].max() > 50


def test_switches_give_the_same_bits(monkeypatch):
    ids = [2, 4, 6]
    results = []
    for env in ({}, {"RGBL_CHAIN_PDL": "0"}, {"RGBL_CHAIN_GRAPH": "0"}):
        for k in ("RGBL_CHAIN_PDL", "RGBL_CHAIN_GRAPH"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)                       # read by rgbl_create
        results.append(run_manual([seq(i) for i in ids]))
    for other in results[1:]:
        for k in results[0]:
            assert results[0][k].tobytes() == other[k].tobytes(), k


def test_frame_construction_overflow_with_lanes():
    lanes = [seq(0), seq(1)]
    ctx, maxp = _context(lanes, max_candidates=256)        # far fewer FAST candidates than a KITTI frame has
    try:
        r = F.SequenceRunner(ctx, lanes[0].ps.P, PRM, 2 * M, W, H, maxp, 1)
        r.set_batch(0, _frames(lanes, 0, "img"), _frames(lanes, 0, "cloud"))
        with pytest.raises(L.RgblError) as e:
            r.run(F.make_chain_params(lanes[0].pose0, *CAM, local_map_frames=K), 1)
        assert e.value.code == L.RGBL_E_CAPACITY
    finally:
        ctx.close()


def test_lanes_resident_query():
    ctx = F.Context(W, H, FEAT)
    try:
        assert ctx.sequence_lanes_resident() >= 1
    finally:
        ctx.close()
