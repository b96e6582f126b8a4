"""Seeded small problems at the edges of the matcher and mapping entry points, shared by the device (test_gpu_match_edges.py) and the
emulated (test_cuda_emu_match.py) tests, with the comparison against the pinned oracle (oracle/matcher_oracle.cpp, mapping_oracle.cpp,
bow_oracle.cpp):

  rgbl_search_by_bow              bow_collect_kernel + resolve_kernel mode 2      (match_kernels.cu)
  rgbl_search_by_projection_reloc search_reloc_collect_kernel + resolve_kernel mode 0
  rgbl_fuse_search                fuse_search_kernel
  rgbl_search_for_triangulation   triangulation_search_kernel + triangulation_finish_kernel   (api_mapping.cu)
  rgbl_distinctive_descriptors    distinctive_kernel
  rgbl_compute_bow                bow_descend_kernel + bow_assemble_kernel     (bow_kernels.cu)

Frames are built directly (keypoints, octaves, angles, uright and descriptors in a 160 x 120 image), not extracted, so a case is a few
hundred features and runs under emulation in seconds.  Every case is dict(name, kind, problem, expect): `expect` names the paths the case
exists for, and `paths(case)` recomputes them from the case data alone (admissible list lengths, the resolution's shared-memory need,
the waiting queries of the round model, histogram counts), so a generator change cannot silently stop reaching a path."""
import math

import numpy as np

import oracle
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F

W, H = 160, 120
FX, FY, CX, CY, BF = 100.0, 100.0, 80.0, 60.0, 40.0
SF = (np.float32(1.2) ** np.arange(8)).astype(np.float32)
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)

# the constants of resolve_kernel and its launchers (match_kernels.cu, api_track.cu, rgbl_ctx.h)
TH_LOW = 50
LIST_CAP = 512                   # kMatchListCap: admissible candidates kept per query; more is RGBL_E_CAPACITY
SORTED_MAX = 32                  # warp_finish_list: longer lists stay in scan order (kListUnsorted)
DYN_BYTES = 160 * 1024           # resolve_dyn_bytes(): on-chip rounds when need <= this, global-memory rounds above
PRELOAD = 4096                   # dense-run entries the on-chip set-up keeps in registers; the rest go through the loop after it
WARP_TAIL = 32                   # block rounds run while more than this many queries wait; warp 0 finishes the rest
FINISH_THREADS = 1024            # triangulation_finish_kernel: one CTA, strided over n1
ASSEMBLE_MAX = 8192              # bow_assemble_kernel: the one-CTA sort holds this many features


def keep_max(th_dist, ratio):
    """api_track.cu keep_max: candidates beyond it cannot change a ratio-tested decision (float division, as in C++)."""
    return min(256, int(math.floor(float(np.float32(th_dist) / np.float32(ratio)))) + 1)


def need_bytes(n_f, n_q, E):
    """resolve_kernel's shared-memory need (match_kernels.cu) for n_f frame features, n_q queries and E list entries."""
    return 12 * (n_f + 1) + 4 * (n_q + 1) + 12 * (E + 4) + 12 * n_q + n_f + 2 * n_q + 4 * n_q + 64


# ---- descriptors --------------------------------------------------------------------------------------------------------------
def hamming(a, b):
    return np.unpackbits(np.bitwise_xor(a, b), axis=-1).sum(-1)


def at_dist(rng, d, k):
    """d with exactly k of its 256 bits flipped"""
    out = d.copy()
    for b in rng.choice(256, k, replace=False):
        out[b >> 3] ^= np.uint8(1 << (b & 7))
    return out


def rand_desc(rng, n=None):
    return rng.integers(0, 256, (32,) if n is None else (n, 32), dtype=np.uint8)


def rot_bin(q_angle, f_angle):
    """rotation_bin of match_kernels.cu / the reference's rot histogram bin, in float32"""
    rot = np.float32(q_angle) - np.float32(f_angle)
    if rot < 0:
        rot = np.float32(rot + np.float32(360.0))
    x = float(np.float32(rot * np.float32(1.0 / 30)))
    b = int(math.floor(x + 0.5)) if x >= 0 else -int(math.floor(-x + 0.5))
    return 0 if b == 30 else b


def three_maxima(hist):
    """ComputeThreeMaxima: the kept bins"""
    order = sorted([i for i in range(30) if hist[i] > 0], key=lambda i: (-hist[i], i))[:3]
    c = [hist[i] for i in order] + [0, 0, 0]
    keep = order + [-1, -1, -1]
    if c[1] < float(np.float32(0.1) * np.float32(c[0])):
        keep[1] = keep[2] = -1
    elif c[2] < float(np.float32(0.1) * np.float32(c[0])):
        keep[2] = -1
    return [k for k in keep[:3] if k >= 0]


# ---- SearchByBoW problems -------------------------------------------------------------------------------------------------------
class BowBuilder:
    """Key-frame features (queries) and frame features (candidates) placed in vocabulary nodes; build() gives the CSR feature vectors
    with node ids ascending and, inside a node, features in ascending index order (as DBoW2's FeatureVector holds them)."""

    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.kf, self.f = [], []

    def query(self, node, desc, angle=0.0, valid=1):
        self.kf.append((node, desc, angle, valid))

    def cand(self, node, desc, angle=0.0):
        self.f.append((node, desc, angle))

    @staticmethod
    def _csr(items, perm):
        nodes = np.array([it[0] for it in items], np.int64)
        ids = np.unique(nodes)
        start, feat = [0], []
        for n in ids:
            feat.extend(sorted(perm[np.nonzero(nodes == n)[0]].tolist()))
            start.append(len(feat))
        return ids.astype(np.uint32) * 7 + 3, np.array(start, np.int32), np.array(feat, np.int32)

    def build(self, ratio, check=True, shuffle=True):
        pk = self.rng.permutation(len(self.kf)) if shuffle else np.arange(len(self.kf))
        pf = self.rng.permutation(len(self.f)) if shuffle else np.arange(len(self.f))
        kd = np.zeros((len(self.kf), 32), np.uint8); ka = np.zeros(len(self.kf), np.float32); kv = np.zeros(len(self.kf), np.uint8)
        for i, (_, d, a, v) in enumerate(self.kf):
            kd[pk[i]] = d; ka[pk[i]] = a; kv[pk[i]] = v
        fd = np.zeros((len(self.f), 32), np.uint8); fa = np.zeros(len(self.f), np.float32)
        for i, (_, d, a) in enumerate(self.f):
            fd[pf[i]] = d; fa[pf[i]] = a
        return dict(kf_desc=kd, kf_angle=ka, kf_valid=kv, kf_csr=self._csr(self.kf, pk), f_desc=fd, f_angle=fa,
                    f_csr=self._csr(self.f, pf), ratio=ratio, check=check)


def bow_lists(p):
    """The queries of SearchByBoW in the reference's order (merge-join of the feature vectors) with their admissible candidates
    (distance <= keep_max(TH_LOW, ratio)) as (distance, position in the frame's node list, frame feature), in scan order."""
    km = keep_max(TH_LOW, p["ratio"])
    ki, ks, kfeat = p["kf_csr"]; fi, fs, ffeat = p["f_csr"]
    out, a, b = [], 0, 0
    while a < len(ki) and b < len(fi):
        if ki[a] == fi[b]:
            for ik in kfeat[ks[a]:ks[a + 1]]:
                if not p["kf_valid"][ik]:
                    continue
                pos = np.arange(fs[b], fs[b + 1])
                d = hamming(p["kf_desc"][ik][None], p["f_desc"][ffeat[pos]])
                out.append([(int(dd), int(pp), int(ffeat[pp])) for dd, pp in zip(d, pos) if dd <= km])
            a += 1; b += 1
        elif ki[a] < fi[b]:
            a += 1
        else:
            b += 1
    return out


def rounds_model(lists, mode, ratio=0.0, th_accept=TH_LOW, taken0=()):
    """The resolution's rounds under the state each round starts with (resolve_kernel: a waiting query is final when it is the
    lowest waiting lister of its best - and in mode 2 its second-best - available candidate).  -> waiting queries before each round."""
    taken = set(taken0)
    lists = [sorted(l)[:LIST_CAP] for l in lists]
    waiting = [q for q, l in enumerate(lists) if l]
    hist = [len(waiting)]
    while waiting:
        minq = {}
        for q in waiting:
            for _, _, ft in lists[q]:
                if ft not in taken:
                    minq.setdefault(ft, q)
        nxt, commits = [], []
        for q in waiting:
            av = [e for e in lists[q] if e[2] not in taken]
            dep = av[:1] if mode == 0 else av[:2]
            if all(minq.get(e[2]) == q for e in dep):
                commits.append(av)
            else:
                nxt.append(q)
        for av in commits:
            if not av or av[0][0] > th_accept:
                continue
            if mode == 2 and not float(av[0][0]) < float(np.float32(ratio) * np.float32(av[1][0] if len(av) > 1 else 256)):
                continue
            taken.add(av[0][2])
        waiting = nxt
        hist.append(len(waiting))
    return hist


def resolve_paths(lists, n_f, mode, ratio=0.0, th_accept=TH_LOW, taken0=()):
    """What resolve_kernel does with these lists, from the data alone."""
    counts = [len(l) for l in lists]
    E = sum(min(c, LIST_CAP) for c in counts)
    need = need_bytes(n_f, len(lists), E)
    hist = rounds_model(lists, mode, ratio, th_accept, taken0)
    tail = next((h for h in hist if h <= WARP_TAIL), 0)
    return dict(counts=counts, E=E, need=need, on_chip=need <= DYN_BYTES, waiting=hist[0], after_first=hist[1] if len(hist) > 1 else 0,
                block_rounds=next(i for i, h in enumerate(hist) if h <= WARP_TAIL), tail=tail, rounds=len(hist) - 1)


def _bow_single(b, node, best, rest, rng, base=None, angle=(0.0, 0.0)):
    """one query in its own node: a candidate at distance `best` and one per distance in `rest`"""
    q = rand_desc(rng) if base is None else base
    b.query(node, q, angle[0])
    b.cand(node, at_dist(rng, q, best), angle[1])
    for d in rest:
        b.cand(node, at_dist(rng, q, d), float(rng.uniform(0, 360)))


def bow_case_lists():
    """admissible lists of 0, 1, 2, 32, 33 and ~200 candidates (the 33 and 200 ones stay in scan order, the best placed anywhere), and a
    node whose three queries share 33 candidates, so the later ones walk past taken entries"""
    rng = np.random.default_rng(10)
    b = BowBuilder(11)
    km = keep_max(TH_LOW, 0.7)
    q = rand_desc(rng); b.query(0, q)
    for _ in range(5):
        b.cand(0, at_dist(rng, q, int(rng.integers(km + 1, 120))))              # candidates, none admissible
    for node, n in ((1, 1), (2, 2), (3, 32), (4, 33), (5, 201)):
        _bow_single(b, node, 12, list(rng.integers(20, km + 1, n - 1)) + [km + 3, 110], rng)
    base = rand_desc(rng)
    for _ in range(3):
        b.query(6, at_dist(rng, base, 4))
    for _ in range(33):
        b.cand(6, at_dist(rng, base, int(rng.integers(4, 30))))
    p = b.build(0.7)
    return dict(name="bow_lists", kind="bow", problem=p, expect=dict(list_lengths=[0, 1, 2, 32, 33, 201], sorted=True, unsorted=True))


def bow_case_list33():
    """lists of exactly 33 candidates (the shortest left in scan order) where the 33rd scan entry decides: in node 0 it is the best, in
    node 1 it is the second that makes the ratio test reject the best at scan position 0.  A resolution that loses or misplaces an entry
    of a 33-entry list changes both decisions."""
    rng = np.random.default_rng(15)
    b = BowBuilder(16)
    q = rand_desc(rng); b.query(0, q)
    for _ in range(32):
        b.cand(0, at_dist(rng, q, int(rng.integers(30, 51))))
    b.cand(0, at_dist(rng, q, 5))                      # scan position 32: the best
    q = rand_desc(rng); b.query(1, q)
    b.cand(1, at_dist(rng, q, 5))                      # scan position 0: the best ...
    for _ in range(31):
        b.cand(1, at_dist(rng, q, int(rng.integers(40, 61))))
    b.cand(1, at_dist(rng, q, 7))                      # ... rejected by the second at scan position 32: 5 >= 0.7 x 7
    p = b.build(0.7, shuffle=False)
    return dict(name="bow_list33", kind="bow", problem=p, expect=dict(list_lengths=[33], list33_decides=True))


def bow_case_capacity(n):
    """one query with n admissible candidates, one of them exactly at keep_max: 512 pass, 513 are RGBL_E_CAPACITY"""
    rng = np.random.default_rng(20 + n)
    b = BowBuilder(21 + n)
    km = keep_max(TH_LOW, 0.7)
    _bow_single(b, 0, 15, [km] + list(rng.integers(30, km + 1, n - 2)) + [km + 1] * 3, rng)
    _bow_single(b, 1, 10, [60], rng)
    p = b.build(0.7)
    return dict(name=f"bow_cap{n}", kind="bow", problem=p, expect=dict(list_lengths=[n], refused=n > LIST_CAP, at_keep_max=True))


def bow_case_ratio(ratio):
    """ratio-test edges: equal best and second-best, best at TH_LOW with the second at keep_max - 1, keep_max and keep_max + 1 (the
    last one is not kept: the query then sees no second candidate), best one above TH_LOW"""
    rng = np.random.default_rng(int(ratio * 100))
    b = BowBuilder(int(ratio * 100) + 1)
    km = keep_max(TH_LOW, ratio)
    _bow_single(b, 0, 20, [20], rng)
    _bow_single(b, 1, 20, [20, 40], rng)
    for node, d2 in ((2, km - 1), (3, km), (4, km + 1)):
        _bow_single(b, node, TH_LOW, [d2], rng)
    _bow_single(b, 5, TH_LOW + 1, [200], rng)
    _bow_single(b, 6, 30, [], rng)
    _bow_single(b, 7, 0, [0], rng)
    p = b.build(ratio)
    return dict(name=f"bow_ratio{ratio}", kind="bow", problem=p, expect=dict(second_at=[km - 1, km, km + 1], equal_best=True))


def bow_case_sides():
    """kf_valid masks, nodes present on one side only (interleaved ids), several queries per node"""
    rng = np.random.default_rng(30)
    b = BowBuilder(31)
    for node in range(40):
        side = node % 4                       # 0, 1: both sides; 2: key frame only; 3: frame only
        base = rand_desc(rng)
        if side != 3:
            for _ in range(int(rng.integers(1, 6))):
                b.query(node, at_dist(rng, base, int(rng.integers(0, 25))), float(rng.uniform(0, 20)), int(rng.random() < 0.7))
        if side != 2:
            for _ in range(int(rng.integers(1, 8))):
                b.cand(node, at_dist(rng, base, int(rng.integers(0, 40))), float(rng.uniform(0, 20)))
    p = b.build(0.75)
    return dict(name="bow_sides", kind="bow", problem=p, expect=dict(one_sided=True, invalid_kf=True))


def bow_case_need(over):
    """the shared-memory need of the resolution tuned to exactly DYN_BYTES (on chip) or DYN_BYTES + 1 (global-memory rounds), with
    more than PRELOAD entries: nodes of 4 contending queries and ~50 candidates, and a last node whose candidates settle the byte count"""
    rng = np.random.default_rng(40)
    b = BowBuilder(41)
    km = keep_max(TH_LOW, 0.7)
    for node in range(51):
        base = rand_desc(rng)
        for _ in range(4):
            b.query(node, at_dist(rng, base, 3), float(rng.uniform(0, 40)))
        for _ in range(50):
            b.cand(node, at_dist(rng, base, int(rng.integers(2, 40))), float(rng.uniform(0, 40)))
    q = rand_desc(rng)
    b.query(99, q, 5.0)
    b.cand(99, at_dist(rng, q, 9))

    def cur():
        p = b.build(0.7, shuffle=False)
        return need_bytes(len(p["f_desc"]), *(lambda l: (len(l), sum(len(x) for x in l)))(bow_lists(p)))
    target = DYN_BYTES + (1 if over else 0)
    rest = target - cur()
    assert rest > 0, rest
    # an admissible candidate adds 13 (frame feature) + 12 (entry) bytes, a non-admissible one 13
    for n_out in range(25):
        if (rest - 13 * n_out) % 25 == 0 and rest - 13 * n_out >= 0:
            break
    for _ in range((rest - 13 * n_out) // 25):
        b.cand(99, at_dist(rng, q, int(rng.integers(5, km + 1))))
    for _ in range(n_out):
        b.cand(99, at_dist(rng, q, int(rng.integers(km + 1, 130))))
    assert cur() == target
    p = b.build(0.7, shuffle=False)
    return dict(name="bow_need_over" if over else "bow_need_at", kind="bow", problem=p, expect=dict(on_chip=not over, need=target, preload_loop=True))


def bow_case_contention():
    """200 queries whose best candidates are the same few features (noisy copies of three base descriptors per node): block rounds
    with more than 32 waiting queries, then the warp-0 tail"""
    rng = np.random.default_rng(50)
    b = BowBuilder(51)
    for node in range(4):
        bases = rand_desc(rng, 3)
        for _ in range(50):
            b.query(node, at_dist(rng, bases[rng.integers(3)], int(rng.integers(2, 12))), float(rng.uniform(0, 25)))
        for _ in range(12):
            b.cand(node, at_dist(rng, bases[rng.integers(3)], int(rng.integers(2, 12))), float(rng.uniform(0, 25)))
    p = b.build(0.9)
    return dict(name="bow_contention", kind="bow", problem=p, expect=dict(block_rounds=True, tail=True))


def bow_case_chain(n=80):
    """a serial chain: query k's descriptor is query k-1's with 40 bits flipped and its best candidate is its own descriptor, which
    query k-1 (and k-2) list as well, so exactly one query becomes final per round: more than 32 rounds, block rounds then the tail"""
    rng = np.random.default_rng(60)
    b = BowBuilder(61)
    d = rand_desc(rng)
    for k in range(n):
        b.query(0, d, 0.0)
        b.cand(0, d.copy(), 0.0)
        d = at_dist(rng, d, 40)
    p = b.build(0.9, shuffle=False)
    return dict(name="bow_chain", kind="bow", problem=p, expect=dict(min_rounds=WARP_TAIL + 1, exact_rounds=n, block_rounds=True, tail=True))


def bow_case_far_lister(n_nodes=40):
    """per node two queries: q0 lists {a, b}, q1 lists {c, d, a} with a its third candidate.  The on-chip rounds only wait for the
    listers of a query's best two, so every query is final in the first round; the global-memory rounds wait for the listers of every
    available candidate, so q1 waits a round for q0.  The round count tells the two paths apart (exact: no query's decision depends
    on a commit of the same round)."""
    rng = np.random.default_rng(65)
    b = BowBuilder(66)

    def flip(d, bits):
        out = d.copy()
        for x in bits:
            out[x >> 3] ^= np.uint8(1 << (x & 7))
        return out
    for node in range(n_nodes):
        bits = rng.permutation(256)
        A = rand_desc(rng)
        q1 = flip(A, bits[:54])                        # keep_max(50, 0.9) = 56: q1 lists a at 54
        b.query(node, A); b.query(node, q1)
        b.cand(node, A)                                 # a: 0 from q0, 54 from q1
        b.cand(node, flip(A, bits[62:72]))             # b: 10 from q0, 64 from q1 (not listed)
        b.cand(node, flip(q1, bits[54:57]))            # c: 3 from q1, 57 from q0 (not listed)
        b.cand(node, flip(q1, bits[57:62]))            # d: 5 from q1, 59 from q0 (not listed)
    p = b.build(0.9, shuffle=False)
    return dict(name="bow_far_lister", kind="bow", problem=p, expect=dict(exact_rounds=1))


def _hist_builder(seed, counts, rot_of_bin=None, ratio=0.7):
    """one accepted match per (node, query, candidate) with its rotation in the bin given by `counts` {bin: n}"""
    rng = np.random.default_rng(seed)
    b = BowBuilder(seed + 1)
    node = 0
    for binv, n in counts.items():
        for _ in range(n):
            fa = float(np.float32(rng.uniform(0, 200)))
            rot = rot_of_bin(binv, rng) if rot_of_bin else 30.0 * binv
            _bow_single(b, node, 8, [], rng, angle=(float(np.float32(fa + rot)) if fa + rot < 360 else float(np.float32(fa + rot - 360)), fa))
            node += 1
    return b.build(ratio)


HIST_PATTERNS = {
    "tie": {3: 5, 1: 5, 7: 5, 2: 5},                 # four equal bins: the three lowest indices are kept
    "at_tenth": {4: 20, 9: 2, 1: 2},                 # second and third exactly at 0.1 x the largest: kept
    "second_below": {4: 21, 9: 2, 1: 2},             # second and third just below: both cleared
    "third_below": {4: 20, 9: 2, 1: 1},              # third just below: cleared
    "two_bins": {5: 7, 0: 3},                        # fewer than three non-empty bins
    "one_bin": {11: 4},
}


def bow_case_hist(kind):
    p = _hist_builder(70 + len(kind), HIST_PATTERNS[kind])
    return dict(name=f"bow_hist_{kind}", kind="bow", problem=p, expect=dict(hist=HIST_PATTERNS[kind]))


def bow_case_angles():
    """rotations of exactly 0, 345 and 359.9 degrees, halves of a bin width and negative differences (q - f < 0 wraps by 360)"""
    rng = np.random.default_rng(80)
    b = BowBuilder(81)
    node = 0
    for qa, fa in ((10.0, 10.0), (345.0, 0.0), (359.9, 0.0), (0.0, 0.1), (15.0, 0.0), (45.0, 0.0), (100.0, 130.0), (5.0, 20.0), (0.0, 345.0),
                   (200.0, 200.5), (359.5, 0.0)) * 3:
        _bow_single(b, node, 6, [], rng, angle=(qa, fa))
        node += 1
    p = b.build(0.7)
    return dict(name="bow_angles", kind="bow", problem=p, expect=dict(negative_rot=True, wrap_bins=[0, 12]))


def bow_cases():
    return ([bow_case_lists(), bow_case_list33(), bow_case_capacity(512), bow_case_capacity(513)] + [bow_case_ratio(r) for r in (0.5, 0.6, 0.7)]
            + [bow_case_sides(), bow_case_need(False), bow_case_need(True), bow_case_contention(), bow_case_chain(), bow_case_far_lister()]
            + [bow_case_hist(k) for k in HIST_PATTERNS] + [bow_case_angles()])


# ---- frames for SearchByProjection(reloc) and Fuse --------------------------------------------------------------------------------
def frame_view_args(keys, uright, desc):
    """the argument tuple of oracle.FrameView / frontend.FrameView for a 160 x 120 frame"""
    return (keys, uright, desc, W, H, SF, FX, FY, CX, CY, BF)


def keypoints(xy, octave, angle):
    k = np.zeros(len(xy), oracle.KP_DTYPE)
    k["x"], k["y"] = np.asarray(xy, np.float32).T
    k["octave"] = octave; k["angle"] = angle; k["size"] = 31 * SF[np.asarray(octave)]
    return k


def point_at(u, v, z):
    """a world point (identity pose) that projects to (u, v) at depth z (z < 0: behind the camera)"""
    return np.array([(u - CX) * z / FX, (v - CY) * z / FY, z], np.float32)


def level_dists(xw, pl):
    """mfMinDistance / mfMaxDistance that predict level pl for a camera at the origin (pl >= 8 clamps to the top level)"""
    d = float(np.linalg.norm(xw.astype(np.float64)))
    mx = d * 1.2 ** pl * 0.9
    return np.float32(min(mx / 1.2 ** 7, 0.9 * d)), np.float32(mx)


def kernel_level(xw, mx):
    """the predicted level before clamping as search_reloc_collect_kernel computes it (identity pose: PO = xw), and its distance test"""
    f = np.float32
    x = xw.astype(f)
    dist = f(np.sqrt(f(f(x[0] * x[0]) + f(f(x[1] * x[1]) + f(x[2] * x[2])))))
    lg = f(math.log(float(f(f(mx) / dist))))
    return math.ceil(float(f(lg / f(np.log(f(SF[1])))))), not dist > f(f(1.2) * f(mx))


def lower_clamp_dists(xw):
    """(mfMinDistance, mfMaxDistance) at the distance boundary dist == 1.2 mfMaxDistance where the predicted level is -1"""
    d = float(np.linalg.norm(xw.astype(np.float64)))
    m = np.float32(d / 1.2)
    for _ in range(8):
        m = np.nextafter(m, np.float32(0))
    for _ in range(16):                                 # the smallest mfMaxDistance that still passes the distance test
        pl, inside = kernel_level(xw, m)
        if inside:
            assert pl < 0, (xw, m, pl)
            return np.float32(m / SF[7]), m
        m = np.nextafter(m, np.float32(1e9))
    raise AssertionError(xw)


def predicted_level(xw, mn, mx):
    d = float(np.linalg.norm(xw.astype(np.float64)))
    return int(math.ceil(math.log(float(mx) / d) / math.log(1.2)))


class RelocBuilder:
    """a frame with keypoints on a 12 px lattice (so windows of different sites do not overlap) plus extra keypoints near some sites,
    and map points projecting onto them"""

    def __init__(self, seed, n_sites=100, extra=60):
        self.rng = rng = np.random.default_rng(seed)
        sites = [(6.0 + 12 * i, 6.0 + 12 * j) for i in range(13) for j in range(10)]
        self.sites = [sites[k] for k in rng.permutation(len(sites))[:n_sites]]
        xy = list(self.sites); oc = list(rng.integers(1, 7, n_sites))
        for _ in range(extra):
            s = int(rng.integers(n_sites))
            xy.append((self.sites[s][0] + float(rng.uniform(-1.5, 1.5)), self.sites[s][1] + float(rng.uniform(-1.5, 1.5)))); oc.append(oc[s])
        self.xy, self.oc = xy, np.array(oc, np.int32)
        self.desc = rand_desc(rng, len(xy))
        for k in range(n_sites, len(xy)):              # the extra keypoints look like the site's own
            s = next(i for i in range(n_sites) if abs(self.sites[i][0] - xy[k][0]) < 2 and abs(self.sites[i][1] - xy[k][1]) < 2)
            self.desc[k] = at_dist(rng, self.desc[s], int(rng.integers(3, 20)))
        self.angle = rng.uniform(0, 360, len(xy)).astype(np.float32)
        self.pts = []                                  # (xw, desc, kf_angle, mf_min, mf_max, valid)

    def point(self, site, dist_bits, z=None, pl=None, rot=0.0, valid=1, jitter=0.5):
        rng = self.rng
        u = self.sites[site][0] + float(rng.uniform(-jitter, jitter)); v = self.sites[site][1] + float(rng.uniform(-jitter, jitter))
        xw = point_at(u, v, float(rng.uniform(4, 30)) if z is None else z)
        mn, mx = level_dists(xw, int(self.oc[site]) if pl is None else pl)
        self.pts.append((xw, at_dist(rng, self.desc[site], dist_bits), float(np.float32(self.angle[site] + rot) % np.float32(360)), mn, mx, valid))

    def build(self, th=3.0, orb_dist=64, check=True, occupied=None):
        k = keypoints(self.xy, self.oc, self.angle)
        ur = np.full(len(k), -1.0, np.float32)
        P = list(zip(*self.pts))
        return dict(keys=k, uright=ur, desc=self.desc.copy(), pose=IDENTITY.copy(), valid=np.array(P[5], np.uint8), xw=np.stack(P[0]),
                    mp_desc=np.stack(P[1]), kf_angle=np.array(P[2], np.float32), mf_min=np.array(P[3], np.float32),
                    mf_max=np.array(P[4], np.float32), th=th, orb_dist=orb_dist, check=check,
                    occupied=None if occupied is None else np.asarray(occupied, np.uint8))


def reloc_lists(p):
    """admissible candidates of every map point: the oracle's features_in_area around the projection, levels pl - 1 .. pl + 1,
    distance <= orb_dist (the occupancy is a state of the resolution, not of the lists)"""
    fv = oracle.FrameView(*frame_view_args(p["keys"], p["uright"], p["desc"]))
    out = []
    for i in range(len(p["valid"])):
        x = p["xw"][i].astype(np.float32)
        if not p["valid"][i]:
            out.append([]); continue
        u = np.float32(np.float32(np.float32(FX) * x[0]) / x[2]) + np.float32(CX)
        v = np.float32(np.float32(np.float32(FY) * x[1]) / x[2]) + np.float32(CY)
        pl = min(max(predicted_level(x, p["mf_min"][i], p["mf_max"][i]), 0), 7)
        cand = oracle.features_in_area(fv, float(u), float(v), float(p["th"] * SF[pl]), pl - 1, pl + 1)
        d = hamming(p["mp_desc"][i][None], p["desc"][cand]) if len(cand) else []
        out.append([(int(dd), k, int(c)) for k, (dd, c) in enumerate(zip(d, cand)) if dd <= p["orb_dist"]])
    return out


def reloc_case_mixed():
    """orb_dist at the kept boundary (isolated sites at exactly orb_dist and orb_dist + 1), occupied features, points behind the camera
    (the reference has no depth test: they match), predicted levels clamped at the top, invalid points, contention on shared sites"""
    b = RelocBuilder(90)
    rng = b.rng
    for s in range(0, 60):
        b.point(s, int(rng.integers(0, 40)))
    for s in range(0, 20):                             # a second and third point on the same sites
        b.point(s, int(rng.integers(0, 40))); b.point(s, int(rng.integers(0, 40)))
    b.point(60, 64, jitter=0.0); b.point(61, 65, jitter=0.0); b.point(62, 64, jitter=0.0)
    for s in (63, 64, 65):
        b.point(s, 10, z=-float(rng.uniform(5, 20)))
    for s in (66, 67):
        b.point(s, 12, pl=9)
    b.point(68, 5, valid=0)
    # the clamp at level 0: a point on the optical axis at a depth where dist == 1.2 mfMaxDistance still passes the distance test and
    # the predicted level is -1 (lower_clamp_dists), with a keypoint of level 0 under it
    kp = len(b.xy)
    b.xy.append((CX, CY)); b.oc = np.append(b.oc, np.int32(0)); b.desc = np.vstack([b.desc, rand_desc(rng)[None]])
    b.angle = np.append(b.angle, np.float32(40.0))
    xw = np.array([0, 0, 5.26], np.float32)
    mn, mx = lower_clamp_dists(xw)
    b.pts.append((xw, at_dist(rng, b.desc[kp], 7), 40.0, mn, mx, 1))
    occ = np.zeros(len(b.xy), np.uint8); occ[rng.choice(len(b.xy) - 1, 25, replace=False)] = 1; occ[62] = 1
    p = b.build(occupied=occ)
    p["low_clamp"] = (len(b.pts) - 1, kp)
    return dict(name="reloc_mixed", kind="reloc", problem=p, expect=dict(orb_dist_boundary=True, behind=True, top_clamp=True, low_clamp=True,
                                                                          occupied=True, block_rounds=True))


def reloc_case_hist(kind):
    """the rotation histogram of mode 0: one isolated match per point, rotations chosen per bin"""
    pat = HIST_PATTERNS[kind]
    n = sum(pat.values())
    b = RelocBuilder(100 + len(kind), n_sites=max(n, 30), extra=0)
    s = 0
    for binv, c in pat.items():
        for _ in range(c):
            b.point(s, 5, rot=30.0 * binv, jitter=0.0); s += 1
    return dict(name=f"reloc_hist_{kind}", kind="reloc", problem=b.build(), expect=dict(hist=pat))


def reloc_cases():
    return [reloc_case_mixed()] + [reloc_case_hist(k) for k in ("tie", "at_tenth", "second_below", "two_bins")]


def fuse_case():
    """points projecting exactly onto max_x / max_y (excluded by IsInImage) and min_x / min_y (included), points behind the camera
    (rejected by the depth test alone: their normals face away from the camera), ties in the best distance (the first in scan order
    wins), stereo and mono keypoints.  Every edge and behind point has a mono keypoint with its own descriptor inside its search window,
    so it would match if its boundary or depth test were dropped."""
    rng = np.random.default_rng(110)
    xy = [(float(x), float(y)) for x, y in rng.uniform((1, 1), (W - 1, H - 1), (150, 2))]
    xy += [(W - 1.5, 30.0), (80.0, H - 1.5), (0.5, 30.0), (80.0, 0.5), (W - 0.5, H - 0.5)]     # the first four in the 64 x 48 grid
    n0 = len(xy)
    for k in range(20):                                 # ties: two keypoints near one projection with equal descriptors
        x, y = float(rng.uniform(20, 140)), float(rng.uniform(20, 100))
        xy += [(x + 0.3, y), (x - 0.4, y + 0.2)]
    oc = np.zeros(len(xy), np.int32)
    desc = rand_desc(rng, len(xy))
    for k in range(n0, len(xy), 2):
        desc[k + 1] = desc[k]
    kps = keypoints(xy, oc, rng.uniform(0, 360, len(xy)).astype(np.float32))
    z = rng.uniform(5, 30, len(xy)).astype(np.float32)
    ur = np.where(rng.random(len(xy)) < 0.5, kps["x"] - np.float32(BF) / z, -1).astype(np.float32)
    ur[[0, 1, 2, n0 - 5, n0 - 4, n0 - 3, n0 - 2]] = -1                  # the targets of the behind and edge points are mono
    pts, pdesc = [], []
    for k in range(len(xy)):
        pts.append(point_at(float(kps["x"][k]), float(kps["y"][k]), float(z[k]))); pdesc.append(at_dist(rng, desc[k], int(rng.integers(0, 60))))
    edge = [point_at(W, 30.0, 10.0), point_at(80.0, H, 10.0), point_at(0.0, 30.0, 10.0), point_at(80.0, 0.0, 10.0)]
    targets = []
    for e, k in zip(edge, range(n0 - 5, n0 - 1)):
        targets.append((len(pts), k)); pts.append(e); pdesc.append(desc[k])
    for k in range(3):                                  # behind the camera, projecting into the image
        targets.append((len(pts), k)); pts.append(point_at(float(xy[k][0]), float(xy[k][1]), -8.0)); pdesc.append(desc[k])
    xw = np.stack(pts).astype(np.float32)
    dist = np.linalg.norm(xw, axis=1).astype(np.float32)
    normal = (xw / dist[:, None]).astype(np.float32)
    mx = (dist * 1.08).astype(np.float32); mn = (mx / SF[7]).astype(np.float32)
    valid = (rng.random(len(xw)) < 0.95).astype(np.uint8); valid[-7:] = 1
    p = dict(keys=kps, uright=ur, desc=desc, pose=IDENTITY.copy(), Ow=np.zeros(3, np.float32), valid=valid, xw=xw, normal=normal, mf_min=mn,
             mf_max=mx, mp_desc=np.stack(pdesc), th=3.0, edge=(len(xw) - 7, len(xw) - 3), targets=targets)
    return dict(name="fuse_edges", kind="fuse", problem=p, expect=dict(on_max_edge=2, on_min_edge=2, behind=3, ties=True))


def fuse_projection(p, i):
    """(u, v, z) of point i as fuse_search_kernel computes them (identity pose)"""
    x = p["xw"][i]
    u = np.float32(np.float32(np.float32(FX) * x[0]) / x[2]) + np.float32(CX)
    v = np.float32(np.float32(np.float32(FY) * x[1]) / x[2]) + np.float32(CY)
    return u, v, x[2]


# ---- SearchForTriangulation --------------------------------------------------------------------------------------------------------
# A forward-moving camera pair with fx = fy = 128 and cx = cy = 64 (exact in float): F12 = K^-T [t]x K^-1 for t = (0, 0, 1) has entries
# 0, +-2^-14, +-2^-8 and its epipolar lines meet at (64, 64); a key-frame-1 feature exactly there has la = lb = 0 (den == 0).
TRI_K = 128.0
TRI_C = 64.0
_a = 1.0 / TRI_K
TRI_F12 = np.array([[0, -_a * _a, 0.5 * _a], [_a * _a, 0, -0.5 * _a], [-0.5 * _a, 0.5 * _a, 0]], np.float32)


def tri_case(name, seed, n1=300, n_nodes=30, wide=40, hist=None, only_stereo=False, coarse=False, check=True):
    """Key frame 2's features lie on the epipolar lines of key frame 1's (pushed outward from the epipole), so most pairs pass the
    epipolar test.  Node 0 holds `wide` (> 32) key-frame-2 features of which several tie at the minimum distance; one key-frame-1
    feature sits at the epipole (den == 0); key-frame-2 features at exactly 10 px (kept) and just under 10 px (rejected) from the
    epipole argument; key frame 1 has n1 features (> 1024: the finish kernel's strided loop).  `hist` {bin: n}: one isolated
    match per entry, rotation in that bin."""
    rng = np.random.default_rng(seed)
    ep = np.array([TRI_C + 1.0, TRI_C - 20.0], np.float32)
    k1, k2, d1, d2, n1s, n2s, ur1, ur2, mp1, mp2 = [], [], [], [], [], [], [], [], [], []

    def add1(x, y, d, node, ang=0.0, stereo=False, mp=False):
        k1.append((x, y, ang, 0)); d1.append(d); n1s.append(node); ur1.append(x - 5.0 if stereo else -1.0); mp1.append(mp)

    def add2(x, y, d, node, ang=0.0, stereo=False, mp=False, oc=0):
        k2.append((x, y, ang, oc)); d2.append(d); n2s.append(node); ur2.append(x - 5.0 if stereo else -1.0); mp2.append(mp)

    def outward(x, y, s):
        return TRI_C + s * (x - TRI_C), TRI_C + s * (y - TRI_C)
    if hist is None:
        base = rand_desc(rng)
        for j in range(4):                              # node 0: wide, with ties at the minimum
            x, y = float(rng.uniform(0, 128)), float(rng.uniform(0, 128))
            q = at_dist(rng, base, 2)
            add1(x, y, q, 0, float(rng.uniform(0, 30)), stereo=bool(rng.random() < 0.5))
            for c in range(wide // 4):
                xx, yy = outward(x, y, float(rng.uniform(1.02, 1.3)))
                dd = 7 if c in (2, 5, 8) else int(rng.integers(8, 45))
                add2(xx, yy, at_dist(rng, q, dd), 0, float(rng.uniform(0, 30)), stereo=bool(rng.random() < 0.5))
        q = rand_desc(rng)
        add1(TRI_C, TRI_C, q, 1)                       # at the epipole: den == 0
        add2(TRI_C + 3.0, TRI_C + 4.0, at_dist(rng, q, 5), 1)
        add2(TRI_C - 3.0, TRI_C, at_dist(rng, q, 9), 1, stereo=True)
        # the epipole radius: candidates exactly 10 px (kept) and just under 10 px (rejected, though nearer in descriptor distance) from
        # the epipole argument, both on the epipolar line of a mono key-frame-1 feature (the line through (64, 64) and it)
        q = rand_desc(rng)
        near = (float(ep[0]) + 6.0, float(ep[1]) + 8.0)
        radius_pair = (len(k1), len(k2))
        add1(TRI_C + 0.8 * (near[0] - TRI_C), TRI_C + 0.8 * (near[1] - TRI_C), q, 2)
        for xy2, dd in ((near, 5), ((near[0], float(ep[1]) + 7.99), 4), ((float(ep[0]) + 10.0, float(ep[1])), 6)):
            add2(xy2[0], xy2[1], at_dist(rng, q, dd), 2)
        for node in range(3, n_nodes):
            base = rand_desc(rng)
            qs = []
            for _ in range(int(rng.integers(1, 6))):
                x, y = float(rng.uniform(0, 128)), float(rng.uniform(0, 128))
                q = at_dist(rng, base, int(rng.integers(0, 10)))
                add1(x, y, q, node, float(rng.uniform(0, 40)), stereo=bool(rng.random() < 0.5), mp=bool(rng.random() < 0.15)); qs.append((x, y))
            for _ in range(int(rng.integers(1, 8))):
                x, y = qs[int(rng.integers(len(qs)))]
                xx, yy = outward(x, y, float(rng.uniform(1.02, 1.4)))
                if rng.random() < 0.2:
                    yy += float(rng.uniform(2, 6))      # off the line
                add2(xx, yy, at_dist(rng, base, int(rng.integers(0, 40))), node, float(rng.uniform(0, 40)), stereo=bool(rng.random() < 0.5),
                     mp=bool(rng.random() < 0.15), oc=int(rng.integers(0, 4)))
    else:
        node = 0
        for binv, c in hist.items():
            for _ in range(c):
                x, y = float(rng.uniform(0, 128)), float(rng.uniform(0, 128))
                q = rand_desc(rng); fa = float(rng.uniform(0, 100))
                add1(x, y, q, node, fa + 30.0 * binv)
                xx, yy = outward(x, y, 1.2)
                add2(xx, yy, at_dist(rng, q, 6), node, fa)
                node += 1
    while len(k1) < n1:                                 # features of key frame 1 in nodes key frame 2 does not have
        add1(float(rng.uniform(0, 128)), float(rng.uniform(0, 128)), rand_desc(rng), 10_000 + len(k1))

    def frame(ks, ds, ns, urs, mps, seed_):
        r = np.random.default_rng(seed_)
        perm = r.permutation(len(ks))                  # feature indices independent of the node order
        kp = np.zeros(len(ks), oracle.KP_DTYPE)
        for i, (x, y, a, oc) in enumerate(ks):
            kp[perm[i]] = (x, y, 31.0, a % 360.0, 0.0, oc, -1)
        d = np.zeros((len(ks), 32), np.uint8); d[perm] = np.stack(ds)
        ur = np.zeros(len(ks), np.float32); ur[perm] = urs
        mp = np.zeros(len(ks), np.uint8); mp[perm] = mps
        nodes = np.array(ns); ids = np.unique(nodes); start, feat = [0], []
        for n in ids:
            feat.extend(sorted(perm[np.nonzero(nodes == n)[0]].tolist())); start.append(len(feat))
        return dict(desc=d, keys=kp, has_mp=mp, uright=ur, fv=(ids.astype(np.uint32), np.array(start, np.int32), np.array(feat, np.int32)), perm=perm)
    kf1 = frame(k1, d1, n1s, ur1, mp1, seed + 1)
    kf2 = frame(k2, d2, n2s, ur2, mp2, seed + 2)
    sg = (SF * SF).astype(np.float32)
    p = dict(kf1=kf1, kf2=kf2, F12=TRI_F12.copy(), ep=ep, sf=SF.copy(), sg=sg, only_stereo=only_stereo, coarse=coarse, check=check)
    ex = dict(n1_strided=n1 > FINISH_THREADS)
    if hist is None:
        ex.update(wide_node=wide, ties=True, den_zero=True, epipole_radius=not only_stereo)
        p["radius_pair"] = (int(kf1["perm"][radius_pair[0]]), int(kf2["perm"][radius_pair[1]]))
    else:
        ex["hist"] = hist
    return dict(name=name, kind="tri", problem=p, expect=ex)


def tri_cases():
    return [tri_case("tri_edges", 120, n1=1300), tri_case("tri_only_stereo", 121, only_stereo=True), tri_case("tri_coarse", 122, coarse=True),
            tri_case("tri_no_orientation", 123, check=False)] + [tri_case(f"tri_hist_{k}", 130 + i, n1=1100 if k == "tie" else 200,
                                                                          hist=HIST_PATTERNS[k]) for i, k in enumerate(("tie", "at_tenth", "second_below", "third_below", "two_bins"))]


def tri_den(p, idx1):
    """den of key-frame-1 feature idx1 as triangulation_search_kernel computes it"""
    k = p["kf1"]["keys"][idx1]; Fm = p["F12"].reshape(9).astype(np.float32)
    x, y = np.float32(k["x"]), np.float32(k["y"])
    la = np.float32(np.float32(x * Fm[0]) + np.float32(y * Fm[3])) + Fm[6]
    lb = np.float32(np.float32(x * Fm[1]) + np.float32(y * Fm[4])) + Fm[7]
    return np.float32(np.float32(la * la) + np.float32(lb * lb))


# ---- ComputeDistinctiveDescriptors ---------------------------------------------------------------------------------------------------
def distinctive_case(name, seed, sizes, mode="noisy"):
    rng = np.random.default_rng(seed)
    start = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    rows = []
    for n in sizes:
        base = rand_desc(rng)
        if mode == "identical":
            rows.append(np.repeat(base[None], n, 0))
        elif mode == "complement":                     # the first row is the complement of all the others: its median is 256
            r = np.repeat(base[None], n, 0); r[0] = ~base; rows.append(r)
        else:
            r = np.repeat(base[None], n, 0)
            r ^= rng.integers(0, 256, r.shape, dtype=np.uint8) & rng.integers(0, 256, r.shape, dtype=np.uint8) & rng.integers(0, 256, r.shape, dtype=np.uint8)
            rows.append(r)
    desc = np.concatenate(rows) if rows else np.zeros((0, 32), np.uint8)
    return dict(name=name, kind="distinctive", problem=dict(obs_start=start, desc=desc), expect=dict(sizes=sorted(set(sizes)), mode=mode))


def distinctive_cases():
    rng = np.random.default_rng(140)
    return [distinctive_case("dist_sizes", 141, [1, 2, 3, 4, 32, 33, 300, 0, 5, 6] + list(rng.integers(1, 12, 200))),
            distinctive_case("dist_identical", 142, [1, 2, 3, 32, 33, 40], "identical"),
            distinctive_case("dist_complement", 143, [3, 5, 33], "complement")]


def distinctive_medians(p, point):
    b, e = p["obs_start"][point], p["obs_start"][point + 1]
    D = np.array([[0 if i == j else hamming(p["desc"][i], p["desc"][j]) for j in range(b, e)] for i in range(b, e)])
    return np.sort(D, 1)[:, (e - b - 1) // 2]


# ---- ComputeBoW --------------------------------------------------------------------------------------------------------------------
def vocabulary(seed, k, levels, ragged=False, stop=0.05, ties=False):
    import bow_data as B
    v = B.make_vocabulary(seed, k, levels, ragged, stop)
    if ties:                                            # every node's second child a copy of its first: the first in list order wins
        for i in range(len(v["child_begin"]) - 1):
            c = v["child_index"][v["child_begin"][i]:v["child_begin"][i + 1]]
            if len(c) >= 2:
                v["node_desc"][c[1]] = v["node_desc"][c[0]]
    return v


def compute_bow_case(name, seed, n, k=10, levels=3, levelsup=2, ragged=False, stop=0.05, ties=False):
    import bow_data as B
    v = vocabulary(seed, k, levels, ragged, stop, ties)
    d = B.descriptors_near_words(v, n, seed + 1) if n else np.zeros((0, 32), np.uint8)
    return dict(name=name, kind="compute_bow", problem=dict(vocab=v, desc=d, levelsup=levelsup),
                expect=dict(n=n, refused=n > ASSEMBLE_MAX, root_children=k, ties=ties, levelsup_ge_L=levelsup >= levels, ragged=ragged))


def compute_bow_cases():
    return [compute_bow_case("cbow_n31", 150, 31), compute_bow_case("cbow_n32", 151, 32), compute_bow_case("cbow_n33", 152, 33),
            compute_bow_case("cbow_n8192", 153, 8192, levels=3), compute_bow_case("cbow_n8193", 154, 8193),
            compute_bow_case("cbow_k32", 155, 300, k=32, levels=2, levelsup=1), compute_bow_case("cbow_k33", 156, 300, k=33, levels=2, levelsup=1),
            compute_bow_case("cbow_ties", 157, 400, k=6, levels=3, ties=True),
            compute_bow_case("cbow_levelsup_L", 158, 200, levels=3, levelsup=3), compute_bow_case("cbow_levelsup_gt_L", 159, 200, levels=2, levelsup=4),
            compute_bow_case("cbow_ragged_stopped", 160, 600, k=6, levels=4, ragged=True, stop=0.4)]


def all_cases():
    return bow_cases() + reloc_cases() + [fuse_case()] + tri_cases() + distinctive_cases() + compute_bow_cases()


# ---- what each case reaches, from its data alone --------------------------------------------------------------------------------
def paths(c):
    """-> the set of path tags the case reaches, computed without running any matcher"""
    p, k, out = c["problem"], c["kind"], set()
    if k == "bow":
        r = resolve_paths(bow_lists(p), len(p["f_desc"]), 2, p["ratio"])
        out |= _resolve_tags(r, "bow")
    elif k == "reloc":
        taken = set(np.nonzero(p["occupied"])[0].tolist()) if p["occupied"] is not None else set()
        r = resolve_paths(reloc_lists(p), len(p["keys"]), 0, th_accept=p["orb_dist"], taken0=taken)
        out |= _resolve_tags(r, "reloc")
    elif k == "tri":
        out.add("tri")
        if len(p["kf1"]["desc"]) > FINISH_THREADS:
            out.add("tri:n1_strided")
        n2 = np.diff(p["kf2"]["fv"][1])
        if (n2 > 32).any():
            out.add("tri:wide_node")
    elif k == "distinctive":
        out.add("distinctive")
    elif k == "compute_bow":
        n = len(p["desc"])
        out.add("cbow:refused" if n > ASSEMBLE_MAX else "cbow")
        if n > 4096:
            out.add("cbow:big")
    elif k == "fuse":
        out.add("fuse")
    if "hist" in c["expect"]:
        out.add(f"{k}:hist")
    return out


def _resolve_tags(r, k):
    t = {k}
    cnt = r["counts"]
    if any(0 < x <= SORTED_MAX for x in cnt):
        t.add(f"{k}:sorted")
    if any(SORTED_MAX < x <= LIST_CAP for x in cnt):
        t.add(f"{k}:unsorted")
    if any(x > LIST_CAP for x in cnt):
        t.add(f"{k}:capacity")
    t.add(f"{k}:on_chip" if r["on_chip"] else f"{k}:global")
    if r["on_chip"] and r["E"] > PRELOAD:
        t.add(f"{k}:preload_loop")
    if r["waiting"] > WARP_TAIL:
        t.add(f"{k}:block_rounds")
        if r["tail"] > 0:
            t.add(f"{k}:block_to_tail")
    if r["rounds"] > WARP_TAIL:
        t.add(f"{k}:many_rounds")
    return t


def check_expect(c):
    """the case reaches what its expect names (asserts); returns the tags"""
    p, e, name = c["problem"], c["expect"], c["name"]
    tags = paths(c)
    if c["kind"] == "bow":
        lists = bow_lists(p)
        r = resolve_paths(lists, len(p["f_desc"]), 2, p["ratio"])
        km = keep_max(TH_LOW, p["ratio"])
        for m in e.get("list_lengths", []):
            assert m in r["counts"], (name, m, sorted(set(r["counts"])))
        if e.get("list33_decides"):
            ki, ks, kfeat = p["kf_csr"]; fi, fs, ffeat = p["f_csr"]
            last0, last1 = ffeat[fs[1] - 1], ffeat[fs[2] - 1]
            assert [len(l) for l in lists] == [33, 33] and min(lists[0])[2] == last0 and sorted(lists[1])[1][2] == last1, name
            n, m = run_oracle(c)
            assert n == 1 and m[last0] == kfeat[ks[0]] and (m[ffeat[fs[1]:fs[2]]] == -1).all(), name
        if e.get("at_keep_max"):
            assert any(len(l) > LIST_CAP - 1 and any(x[0] == km for x in l) for l in lists), name
        if "on_chip" in e:
            assert r["on_chip"] == e["on_chip"] and r["need"] == e["need"] and r["E"] > PRELOAD, (name, r["need"], r["E"])
        if e.get("block_rounds"):
            assert r["waiting"] > WARP_TAIL and r["after_first"] > 0 and r["block_rounds"] >= 1, (name, r)
        if e.get("tail"):
            assert 0 < r["tail"] <= WARP_TAIL, (name, r)
        if "min_rounds" in e:
            assert r["rounds"] >= e["min_rounds"] and r["after_first"] > WARP_TAIL, (name, r)
        if "exact_rounds" in e:
            assert r["rounds"] == e["exact_rounds"] and r["on_chip"], (name, r)
        if "second_at" in e:
            seconds = {sorted(l)[1][0] for l in lists if len(l) >= 2 and sorted(l)[0][0] == TH_LOW}
            singles = [l for l in lists if len(l) == 1 and l[0][0] == TH_LOW]
            assert {km - 1, km} <= seconds and singles, (name, seconds)   # km + 1 is not kept: that query's list has one entry
            ds = [sorted(x[0] for x in l) for l in lists]
            assert any(len(d) >= 2 and d[0] == d[1] for d in ds), name
        if e.get("one_sided"):
            ki, fi = set(p["kf_csr"][0].tolist()), set(p["f_csr"][0].tolist())
            assert ki - fi and fi - ki and ki & fi, name
        if e.get("invalid_kf"):
            assert (p["kf_valid"] == 0).any() and (p["kf_valid"] == 1).any(), name
    if "hist" in e and c["kind"] in ("bow", "reloc"):
        if c["kind"] == "bow":
            h = _bow_hist(p)
        else:
            h = _reloc_hist(p)
        assert h == {b_: n for b_, n in e["hist"].items()}, (name, h)
    if c["kind"] == "bow" and "wrap_bins" in e:
        bins = [rot_bin(p["kf_angle"][i], p["f_angle"][j]) for i, j in _bow_pairs(p)]
        assert set(e["wrap_bins"]) <= set(bins), (name, sorted(set(bins)))
        assert any(p["kf_angle"][i] < p["f_angle"][j] for i, j in _bow_pairs(p)), name
    if c["kind"] == "reloc" and c["expect"].get("orb_dist_boundary"):
        lists = reloc_lists(p)
        best = [min(x[0] for x in l) for l in lists if l]
        assert p["orb_dist"] in best, name
        assert (p["xw"][:, 2] < 0).any() and any(lists[i] for i in np.nonzero(p["xw"][:, 2] < 0)[0]), name
        pls = [predicted_level(p["xw"][i], p["mf_min"][i], p["mf_max"][i]) for i in range(len(p["xw"]))]
        assert max(pls) >= 8, name
        if c["expect"].get("low_clamp"):
            i, kp = p["low_clamp"]
            pl, inside = kernel_level(p["xw"][i], p["mf_max"][i])
            assert pl < 0 and inside, (name, pl, inside)
            assert run_oracle(c)[1][kp] == i, name                       # the clamped point matches its level-0 keypoint
        assert "reloc:block_rounds" in tags, (name, tags)
    if c["kind"] == "fuse":
        i0, i1 = p["edge"]
        uv = [fuse_projection(p, i) for i in range(i0, i1)]
        assert uv[0][0] == np.float32(W) and uv[1][1] == np.float32(H) and uv[2][0] == 0 and uv[3][1] == 0, (name, uv)
        assert (p["xw"][i1:, 2] < 0).all(), name
        for i, k in p["targets"]:                      # dropping the boundary or depth test would give the point this keypoint
            d = float(np.linalg.norm(p["xw"][i].astype(np.float64)))
            level = min(max(math.ceil(math.log(float(p["mf_max"][i]) / d) / math.log(1.2)), 0), 7)
            u, v, _ = fuse_projection(p, i)
            kp = p["keys"][k]
            assert p["uright"][k] < 0 and abs(float(kp["x"]) - float(u)) < p["th"] * SF[level] and abs(float(kp["y"]) - float(v)) < p["th"] * SF[level], (name, i)
            assert level - 1 <= kp["octave"] <= level and hamming(p["mp_desc"][i], p["desc"][k]) == 0, (name, i)
            gx = round(float(np.float32(kp["x"] * np.float32(64 / W)))); gy = round(float(np.float32(kp["y"] * np.float32(48 / H))))
            assert 0 <= gx < 64 and 0 <= gy < 48, (name, k)                # Frame::PosInGrid keeps it
            assert float(np.dot(p["xw"][i], p["normal"][i])) >= 0.5 * d and p["mf_max"][i] * 1.2 >= d, (name, i)
        best = run_oracle(c)[0]                        # max_x / max_y and behind: nothing; min_x / min_y: their keypoint
        assert [int(best[i]) for i, _ in p["targets"]] == [-1, -1, p["targets"][2][1], p["targets"][3][1], -1, -1, -1], (name, best[i0:])
    if c["kind"] == "tri":
        kf1 = p["kf1"]
        if e.get("den_zero"):
            assert any(tri_den(p, i) == 0 for i in range(len(kf1["desc"]))), name
            assert "tri:wide_node" in tags, name
            ep = p["ep"]; k2 = p["kf2"]["keys"]
            r2 = (np.float32(ep[0]) - k2["x"]) ** 2 + (np.float32(ep[1]) - k2["y"]) ** 2
            assert (r2 == np.float32(100)).any() and ((r2 < 100) & (r2 > 99)).any(), name
        if e.get("epipole_radius"):                     # the pair at exactly 10 px is the match: the nearer one was rejected by the radius
            i1, i2 = p["radius_pair"]
            assert run_oracle(c)[1][i1] == i2, (name, run_oracle(c)[1][i1], i2)
        if e.get("n1_strided"):
            assert "tri:n1_strided" in tags, name
        if "hist" in e:
            h = {}
            ids1, s1, f1 = kf1["fv"]; ids2, s2, f2 = p["kf2"]["fv"]
            for a, node in enumerate(ids1):
                bidx = np.nonzero(ids2 == node)[0]
                if len(bidx):
                    i, j = f1[s1[a]], f2[s2[bidx[0]]]
                    b_ = rot_bin(kf1["keys"]["angle"][i], p["kf2"]["keys"]["angle"][j]); h[b_] = h.get(b_, 0) + 1
            assert h == e["hist"], (name, h)
    if c["kind"] == "distinctive":
        sizes = set(np.diff(p["obs_start"]).tolist())
        assert set(e["sizes"]) <= sizes, name
        if e["mode"] == "complement":
            pt = int(np.nonzero(np.diff(p["obs_start"]) >= 3)[0][0])
            assert distinctive_medians(p, pt)[0] == 256, name
        if e["mode"] == "noisy":
            meds = [distinctive_medians(p, q) for q in range(len(p["obs_start"]) - 1) if p["obs_start"][q + 1] > p["obs_start"][q]]
            assert any((m == m.min()).sum() > 1 for m in meds), name                 # tied medians
    if c["kind"] == "compute_bow":
        v = p["vocab"]
        cb = v["child_begin"]
        assert e["ragged"] or cb[1] - cb[0] == e["root_children"], name
        if e["ragged"]:
            leaves = v["word_id"] >= 0
            assert (v["node_weight"][leaves] == 0).any(), name             # stopped words
            depth = np.zeros(len(cb) - 1, int)
            for i in range(len(cb) - 1):
                depth[v["child_index"][cb[i]:cb[i + 1]]] = depth[i] + 1
            assert len(set(depth[leaves].tolist())) > 1, name             # leaves above the last level
    return tags


def _bow_pairs(p):
    """(key-frame feature, frame feature) of every node that holds exactly one of each"""
    ki, ks, kfeat = p["kf_csr"]; fi, fs, ffeat = p["f_csr"]
    out = []
    for a, node in enumerate(ki):
        b = np.nonzero(fi == node)[0]
        if len(b) and ks[a + 1] - ks[a] == 1 and fs[b[0] + 1] - fs[b[0]] == 1:
            out.append((int(kfeat[ks[a]]), int(ffeat[fs[b[0]]])))
    return out


def _bow_hist(p):
    h = {}
    for i, j in _bow_pairs(p):
        b_ = rot_bin(p["kf_angle"][i], p["f_angle"][j]); h[b_] = h.get(b_, 0) + 1
    return h


def _reloc_hist(p):
    h = {}
    for i, l in enumerate(reloc_lists(p)):
        if l:
            j = min(l)[2]
            b_ = rot_bin(p["kf_angle"][i], p["keys"]["angle"][j]); h[b_] = h.get(b_, 0) + 1
    return h


# ---- running a case: through the frontend and through the oracle ----------------------------------------------------------------
def run_device(ctx, c):
    """the case through orb_slam3_rgbl_b200.frontend (whatever library it has loaded) -> comparable result"""
    p, k = c["problem"], c["kind"]
    if k == "bow":
        m = F.ORBmatcher(ctx, p["ratio"], p["check"])
        return m.SearchByBoW(p["kf_desc"], p["kf_angle"], p["kf_valid"], p["kf_csr"], p["f_desc"], p["f_angle"], p["f_csr"])
    if k == "reloc":
        fv = F.FrameView(*frame_view_args(p["keys"], p["uright"], p["desc"]))
        return F.ORBmatcher(ctx, 0.9, p["check"]).SearchByProjectionReloc(fv, p["pose"], p["valid"], p["xw"], p["mp_desc"], p["kf_angle"], p["mf_min"],
                                                                          p["mf_max"], p["th"], p["orb_dist"], p["occupied"])
    if k == "fuse":
        fv = F.FrameView(*frame_view_args(p["keys"], p["uright"], p["desc"]))
        return F.fuse_search(ctx, fv, p["pose"], p["Ow"], p["valid"], p["xw"], p["normal"], p["mf_min"], p["mf_max"], p["mp_desc"], p["th"])
    if k == "tri":
        return F.search_for_triangulation(ctx, p["kf1"], p["kf2"], p["F12"], p["ep"], p["sf"], p["sg"], p["only_stereo"], p["coarse"], p["check"])
    if k == "distinctive":
        return F.distinctive_descriptors(ctx, p["obs_start"], p["desc"])
    if k == "compute_bow":
        v = p["vocab"]
        voc = F.ORBVocabulary(ctx, v["child_begin"], v["child_index"], v["node_desc"], v["node_weight"], v["word_id"], v["levels"])
        try:
            return voc.transform(p["desc"], p["levelsup"])
        finally:
            voc.close()
    raise ValueError(k)


def run_oracle(c):
    p, k = c["problem"], c["kind"]
    if k == "bow":
        return oracle.search_by_bow(p["kf_desc"], p["kf_angle"], p["kf_valid"], p["kf_csr"], p["f_desc"], p["f_angle"], p["f_csr"], p["ratio"], p["check"])
    if k == "reloc":
        fv = oracle.FrameView(*frame_view_args(p["keys"], p["uright"], p["desc"]))
        return oracle.search_by_projection_reloc(fv, p["pose"], p["valid"], p["xw"], p["mp_desc"], p["kf_angle"], p["mf_min"], p["mf_max"], p["th"],
                                                 p["orb_dist"], p["check"], p["occupied"])
    if k == "fuse":
        fv = oracle.FrameView(*frame_view_args(p["keys"], p["uright"], p["desc"]))
        return oracle.fuse_search(fv, p["pose"], p["Ow"], p["valid"], p["xw"], p["normal"], p["mf_min"], p["mf_max"], p["mp_desc"], p["th"])
    if k == "tri":
        return oracle.search_for_triangulation(p["kf1"], p["kf2"], p["F12"], p["ep"], p["sf"], p["sg"], p["only_stereo"], p["coarse"], p["check"])
    if k == "distinctive":
        return oracle.distinctive_descriptors(p["obs_start"], p["desc"])
    if k == "compute_bow":
        return oracle.compute_bow(p["vocab"], p["desc"], p["levelsup"])
    raise ValueError(k)


def refused(c):
    return bool(c["expect"].get("refused"))


REFUSAL_TEXT = {"bow": "matcher candidate list overflow", "compute_bow": "too many features for one BoW transform"}


def compare(c, got, ref):
    """bit for bit: matches and counts, best indices and distances, BoW words, values (as bits), nodes and features"""
    k, name = c["kind"], c["name"]
    if k in ("bow", "reloc", "tri"):
        assert got[0] == ref[0], (name, got[0], ref[0])
        assert np.array_equal(got[1], ref[1]), (name, int((got[1] != ref[1]).sum()), np.nonzero(got[1] != ref[1])[0][:10])
    elif k == "fuse":
        assert np.array_equal(got[0], ref[0]) and np.array_equal(got[1], ref[1]), (name, int((got[0] != ref[0]).sum()), int((got[1] != ref[1]).sum()))
    elif k == "distinctive":
        assert np.array_equal(got, ref), (name, np.nonzero(got != ref)[0][:10])
    elif k == "compute_bow":
        (gw, gv), (gn, gs, gf) = got
        (rw, rv), (rn, rs, rf) = ref
        assert np.array_equal(gw, rw) and np.array_equal(gv.view(np.uint64), rv.view(np.uint64)), name
        assert np.array_equal(gn, rn) and np.array_equal(gs, rs) and np.array_equal(gf, rf), name


def check_case(ctx, c):
    """run the case on the loaded library and compare it with the oracle (or check the refusal) -> one line for the log"""
    if refused(c):
        try:
            run_device(ctx, c)
        except L.RgblError as e:
            assert e.code == L.RGBL_E_CAPACITY and REFUSAL_TEXT[c["kind"]] in str(e), (c["name"], str(e))
            return f"{c['name']}: refused ({e})"
        raise AssertionError(f"{c['name']}: not refused")
    got, ref = run_device(ctx, c), run_oracle(c)
    compare(c, got, ref)
    if c["kind"] in ("bow", "reloc", "tri"):
        return f"{c['name']}: {ref[0]} matches"
    return f"{c['name']}: equal"


def emulated_cases():
    """The subset run at one OS thread per CUDA thread: every resolution path (sorted and unsorted lists, the capacity refusal, on-chip
    rounds with the loop after the register preload, the global-memory rounds, block rounds handing over to the warp tail, a chain of
    more than 32 rounds), the ratio edges at a ratio whose 50 / ratio is not an integer, both rotation histograms at 0.1 x the largest,
    reloc with its boundaries, fuse, triangulation with n1 > 1024 and a wide node, distinctive descriptors, and ComputeBoW around 32
    features, 33 children, ties and the refusal above 8192."""
    names = {"bow_lists", "bow_list33", "bow_cap513", "bow_ratio0.6", "bow_need_at", "bow_need_over", "bow_contention", "bow_chain", "bow_far_lister", "bow_hist_at_tenth",
             "bow_hist_tie", "bow_angles", "reloc_mixed", "reloc_hist_second_below", "fuse_edges", "tri_edges", "tri_coarse", "tri_hist_at_tenth",
             "dist_sizes", "dist_identical", "dist_complement", "cbow_n33", "cbow_k33", "cbow_ties", "cbow_levelsup_gt_L", "cbow_n8193"}
    return [c for c in all_cases() if c["name"] in names]


# the tags the emulated subset must keep (test_subset_has_every_launch_shape)
REQUIRED_TAGS = {"bow:sorted", "bow:unsorted", "bow:capacity", "bow:on_chip", "bow:global", "bow:preload_loop", "bow:block_rounds",
                 "bow:block_to_tail", "bow:many_rounds", "bow:hist", "reloc:on_chip", "reloc:block_rounds", "reloc:hist", "fuse", "tri:n1_strided",
                 "tri:wide_node", "tri:hist", "distinctive", "cbow", "cbow:refused"}
