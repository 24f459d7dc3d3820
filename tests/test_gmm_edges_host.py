"""CPU checks of the GMM edge table (tests/test_gpu_gmm_edges.py): against the restated launch plan
(test_gmm_host.plan_restated) it reaches every instantiation, both thread plans at their boundary, the largest and
smallest shapes, every source of phi, the batch sizes around a CTA, and one, two and many row chunks on every
path.  Also the plan's boundary itself through zk_gmm_plan."""

import ctypes

import gmm_reference as R
import pytest
from test_gmm_host import plan_restated
from test_gpu_gmm_edges import CASES, threads

from zuko_b200 import _engine as E


def T_of(case) -> int:
    return plan_restated(case.D, case.K, R.COV[case.cov], int(case.tied))[0]


def test_thread_rule_matches_the_plan():
    for case in CASES:
        assert threads(case.D, case.K) == T_of(case), case.id


@pytest.mark.parametrize("D,K,T", [(32, 32, 128), (40, 16, 128), (33, 31, 64), (40, 17, 64), (64, 32, 64), (1, 1, 128)])
@pytest.mark.parametrize("cov", ["full", "diagonal", "spherical"])
@pytest.mark.parametrize("tied", [False, True])
def test_plan_boundary(D, K, T, cov, tied):
    """128 threads while 2D + K <= 96, 64 above."""
    threads_ = ctypes.c_int()
    E.check(E.lib().zk_gmm_plan(D, K, R.COV[cov], int(tied), ctypes.byref(threads_), None, None, None, None))
    assert threads_.value == T == plan_restated(D, K, R.COV[cov], int(tied))[0]


def test_every_instantiation_and_source():
    cells = {(c.cov, c.tied) for c in CASES}
    assert cells == {(cov, tied) for cov in R.COV for tied in (False, True)}  # x 3 families: every case runs all
    assert {c.src for c in CASES} == {"table", "rows", "bcast"}
    assert {c.hyper for c in CASES if c.src != "table"} == {"fp32", "tc"}
    assert {c.src for c in CASES if c.hyper == "tc"} >= {"rows", "bcast"}


def test_both_plans_and_shape_edges():
    pairs = {(c.D, c.K) for c in CASES}
    assert {T_of(c) for c in CASES} == {128, 64}
    assert {(32, 32), (40, 16), (33, 31), (40, 17), (64, 32), (1, 1)} <= pairs
    assert any(c.D == 64 and c.K == 32 and c.cov == "full" and c.tied for c in CASES)
    assert {(c.cov, c.tied) for c in CASES if (c.D, c.K) == (1, 1)} >= {("full", False), ("full", True)}
    for T in (128, 64):
        assert {c.src for c in CASES if T_of(c) == T} == {"table", "rows", "bcast"}, T


def test_batches_around_a_cta():
    for T in (128, 64):
        batches = {c.B for c in CASES if c.B is not None and T_of(c) == T}
        assert {1, T - 1, T, T + 1, 2 * T + 1} <= batches, T
        assert any(b >= 1000 and b % T for b in batches), T


def test_row_chunks_on_every_path():
    """One, two and many chunks (the last holding one row) on the three backward paths (per-row, broadcast,
    unconditional) and the per-row forward of log_prob and sample; the chunk plan is restated exactly for fp32
    conditioners, so the counted chunks use those and the table."""
    for src in ("rows", "bcast", "table"):
        counts = {c.chunks for c in CASES if c.src == src and (src == "table" or c.hyper == "fp32")}
        assert {1, 2, "many"} <= counts, src
    assert {c.chunks for c in CASES if c.hyper == "tc"} >= {1, "min"}
