"""The fixtures of tests/test_gpu_tas_paths.py reach the branches they claim, and the oracle's output on them passes the
same invariants as the device's: checked on the CPU, so a machine without a GPU proves what the device tests exercise."""
import pytest

import oracle
from tests.test_gpu_tas_paths import FIXTURES, build, check_invariants, facts


@pytest.mark.parametrize("name", list(FIXTURES))
def test_fixtures_reach_their_branches(name):
    topo, reqs, cap, claims, pairs = build(name)
    want = oracle.tas_find(topo, reqs, cap)
    check_invariants(topo, reqs, want)
    got = facts(topo, reqs, want, pairs)
    assert claims <= got, sorted(claims - got)
