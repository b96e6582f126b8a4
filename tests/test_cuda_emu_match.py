"""The matcher and mapping entry points of tests/match_cases.py run through the whole library compiled over the CUDA-on-CPU shim
(tests/cuda_emu), so a machine without a GPU executes their kernels: a subset of the cases that still reaches every resolution path,
compared bit for bit with the oracle through orb_slam3_rgbl_b200.frontend (pointed at the emulated library), and, from the case data
alone, that every case reaches the path it exists for."""
import ctypes as C

import pytest

import match_cases as MC
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F

CASES = MC.emulated_cases()


@pytest.fixture(scope="module")
def ctx():
    so = C.CDLL(str(build.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    so.rgbl_last_match_rounds.restype, so.rgbl_last_match_rounds.argtypes = C.c_int, [C.c_void_p]
    mp = pytest.MonkeyPatch()
    mp.setattr(L, "_lib", so)                 # frontend calls go to the emulated library for this module
    c = F.Context(MC.W, MC.H, 200, nlevels=4)
    c.so = so
    yield c
    c.close()
    mp.undo()


def test_subset_has_every_launch_shape():
    tags = set().union(*(MC.paths(c) for c in CASES))
    assert MC.REQUIRED_TAGS <= tags, sorted(MC.REQUIRED_TAGS - tags)


def test_cases_reach_their_paths():
    """every case, at full size: what its expect names holds for its data (list lengths around 32 / 33 / 512 / 513, the need against
    160 KB, waiting queries of the round model, histogram counts, boundary projections), and over all cases every tag is reached"""
    tags = set()
    for c in MC.all_cases():
        tags |= MC.check_expect(c)
    assert MC.REQUIRED_TAGS <= tags


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_case_emulated(ctx, c):
    MC.check_expect(c)
    print(MC.check_case(ctx, c))


def test_refusal_leaves_the_context_usable(ctx):
    by = {c["name"]: c for c in CASES}
    MC.check_case(ctx, by["bow_cap513"])
    MC.check_case(ctx, by["bow_lists"])


@pytest.mark.parametrize("name", ["bow_chain", "bow_far_lister"])
def test_round_count(ctx, name):
    """resolve_kernel's round counter where the round model is exact: a serial chain of 80 queries (48 block rounds, then 32 rounds of
    the warp tail) and 80 queries that are all final in the first on-chip round (the global-memory rounds would take two)"""
    c = next(c for c in CASES if c["name"] == name)
    MC.check_case(ctx, c)
    assert ctx.so.rgbl_last_match_rounds(ctx.handle) == c["expect"]["exact_rounds"]
