"""The L2 screen's lower bound (tests/sparse_l2_bound_model.py) against the reference's L2 distance D_ref, the fp32
restatement of vector.cpp (test_gpu_sparse.ref_distances): LB <= D_ref for every pair the bound covers, and every pair
whose D_ref is NaN (or whose inputs are not finite) is left uncovered, so it is always re-scored.  Runs without a GPU."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
from sparse_l2_bound_model import MAX_TERMS, adversarial, csr_norm2, lower_bound  # noqa: E402
from test_gpu_sparse import IP, L2, densify, ref_distances, sparse_rows  # noqa: E402


def bounds_and_ref(rows, qs, vocab):
    R, Qd = densify(rows, vocab), densify(qs, vocab)
    with np.errstate(all="ignore"):
        d_ref = ref_distances(R, Qd, L2)
        dot = -ref_distances(R, Qd, IP)   # the matched products in index order (absent elements add an exact +-0)
    lb = lower_bound(dot, csr_norm2(rows)[None, :], csr_norm2(qs)[:, None], np.diff(rows[0])[None, :],
                     np.diff(qs[0])[:, None])
    return lb, d_ref


def check(lb, d_ref, what):
    covered = np.isfinite(lb)
    assert not np.isnan(d_ref[covered]).any(), what + ": a pair with a NaN distance is screened"
    bad = covered & ~(lb.astype(np.float64) <= d_ref.astype(np.float64))
    assert not bad.any(), "%s: LB > D_ref at %s (LB %r, D_ref %r)" % (
        what, np.argwhere(bad)[:3].tolist(), lb[bad][:3], d_ref[bad][:3])
    return covered


def test_bound_holds_on_the_golden_l2_table():
    from make_sparse_golden import table
    n, vocab, rows, qs, _, _, _ = table(L2)
    lb, d_ref = bounds_and_ref(rows, qs, vocab)
    covered = check(lb, d_ref, "golden L2 table")
    assert covered.all()   # finite values only
    # tight enough to screen: the slack is about 3 m u (|row|^2 + |q|^2), m <= 100 elements here
    rn, qn = csr_norm2(rows)[None, :], csr_norm2(qs)[:, None]
    assert (d_ref - lb <= 300 * 2.0 ** -24 * (rn + qn) + 1e-30).all()


def test_bound_holds_on_random_pairs():
    """More than 10^5 pairs: rows and queries of sparse_rows with values scaled by 10^[-6, 6]."""
    rng = np.random.default_rng(7)
    pairs = 0
    for seed in range(3):
        vocab = 1500
        rows = sparse_rows(420, vocab, 300 + seed, max_nnz=80)
        qs = sparse_rows(90, vocab, 400 + seed, max_nnz=40, empty_every=0, dup_every=0)
        rs = (10.0 ** rng.uniform(-6, 6, rows[0].size - 1)).astype(np.float32)
        rows = (rows[0], rows[1], (rows[2] * np.repeat(rs, np.diff(rows[0]))).astype(np.float32))
        lb, d_ref = bounds_and_ref(rows, qs, vocab)
        assert check(lb, d_ref, "random pairs, seed %d" % seed).all()
        pairs += lb.size
    assert pairs >= 100_000


def test_bound_holds_on_adversarial_rows_and_queries():
    for seed in (1, 2, 3):
        rows, qs, vocab = adversarial(seed)
        lb, d_ref = bounds_and_ref(rows, qs, vocab)
        covered = check(lb, d_ref, "adversarial, seed %d" % seed)
        rn, qn = csr_norm2(rows), csr_norm2(qs)
        # exactly the pairs with a non-finite |row|^2 or |q|^2 are left to the merge (no dot overflows here)
        assert np.array_equal(~covered, ~np.isfinite(rn)[None, :] | ~np.isfinite(qn)[:, None])
        assert (~np.isfinite(rn)).any() and (~np.isfinite(qn)).any() and np.isnan(d_ref).any()
        # cancellation: a row equal to a covered query is at distance 0 and its bound may not exceed 0
        assert ((d_ref == 0) & covered).any() and (lb[(d_ref == 0) & covered] <= 0).all()
        # products that underflow: the tiny query against the tiny rows, and distances that overflow to +inf
        assert (covered & (d_ref > 0) & (d_ref < 1e-37)).any()
        assert (covered & np.isinf(d_ref)).any()


def test_pairs_beyond_the_formula_are_uncovered():
    lb = lower_bound(np.zeros(3, np.float32), np.ones(3, np.float32), np.ones(3, np.float32),
                     np.array([10, MAX_TERMS - 12, MAX_TERMS - 11]), np.array([10, 10, 10]))
    assert np.isfinite(lb[:2]).all() and lb[2] == np.inf
    lb = lower_bound(np.float32(np.inf), np.float32(1), np.float32(1), 1, 1)
    assert lb == np.inf


@pytest.mark.parametrize("seed", [11, 12])
def test_bound_is_zero_or_below_for_identical_rows(seed):
    rows = sparse_rows(50, 300, seed, max_nnz=60, empty_every=0, dup_every=0)
    lb, d_ref = bounds_and_ref(rows, rows, 300)
    check(lb, d_ref, "rows against themselves")
    assert (np.diag(d_ref) == 0).all() and (np.diag(lb) <= 0).all()
