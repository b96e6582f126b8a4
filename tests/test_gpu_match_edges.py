"""The matcher and mapping entry points at their list, capacity, contention, tie and histogram edges (tests/match_cases.py) on the
device, through orb_slam3_rgbl_b200.frontend, against the pinned oracle: matches, counts, best indices and distances and BoW values bit
for bit, and the error code and text of the refusals.  A refusal leaves the context usable: the next call equals the oracle."""
import pytest

import match_cases as MC
from orb_slam3_rgbl_b200 import frontend as F

pytestmark = pytest.mark.gpu

CASES = MC.all_cases()


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(MC.W, MC.H, 200, nlevels=4)
    yield c
    c.close()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_case_matches_oracle(ctx, c):
    MC.check_expect(c)
    print(MC.check_case(ctx, c))


def test_context_usable_after_refusals(ctx):
    by = {c["name"]: c for c in CASES}
    for refusal, after in (("bow_cap513", "bow_lists"), ("cbow_n8193", "cbow_n33"), ("bow_cap513", "bow_need_over"), ("bow_cap513", "bow_need_at")):
        MC.check_case(ctx, by[refusal])
        MC.check_case(ctx, by[after])
