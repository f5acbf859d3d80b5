"""CPU tests of the posting-list extension: its two entry points are declared in the header, exported, bound by lib.py,
reachable from SparseIndex and refused without an index; the numpy model of the lists is pinned on a hand-worked
table, and the restatement of the device merge gives the model's lists on seeded tables."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from sparse_postings_model import extend_model, postings_model, same_postings  # noqa: E402
from test_sparse_abi import ROOT, _lib  # noqa: E402

CALLS = ("eps_index_extend_sparse_postings", "eps_index_get_sparse_postings")


def test_postings_calls_declared_exported_and_bound():
    L = _lib()
    hdr = open(os.path.join(ROOT, "include", "epsilla_b200.h")).read()
    assert "EPS_API int eps_index_extend_sparse_postings(eps_index* ix, int64_t n);" in hdr
    assert re.search(r"EPS_API int eps_index_get_sparse_postings\(eps_index\* ix, int64_t\* n_rows, int64_t\* n_terms, "
                     r"int64_t\* n_postings,\s+uint32_t\* terms, int64_t\* ptr, int32_t\* rows, float\* values\);", hdr)
    from vectordb_b200.lib import EXPORTS
    for name in CALLS:
        assert name in EXPORTS
        assert getattr(L, name).argtypes, "%s has no ctypes signature" % name
    from vectordb_b200.index import SparseIndex
    assert callable(SparseIndex.extend_postings) and callable(SparseIndex.postings)


def test_postings_calls_null_index_refused():
    L = _lib()
    for n in (-1, 0, 5):
        assert L.eps_index_extend_sparse_postings(None, n) == 40005   # EPS_ERR_INVALID_ARGUMENT: no index
    assert L.eps_index_get_sparse_postings(None, None, None, None, None, None, None, None) == 40005


def csr(rows):
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    idx = np.array([i for r in rows for i, _ in r], np.int64)
    val = np.array([v for r in rows for _, v in r], np.float32)
    return off, idx, val


# row 0: {2: 1, 5: 2}; row 1: empty; row 2: {0: 3, 2: 4}; row 3: {5: 5, 7: 6}
HAND = csr([[(2, 1.0), (5, 2.0)], [], [(0, 3.0), (2, 4.0)], [(5, 5.0), (7, 6.0)]])


def test_model_on_a_hand_worked_table():
    same_postings(postings_model(HAND, 4), dict(rows=4, terms=[0, 2, 5, 7], ptr=[0, 1, 3, 5, 6],
                                                post_rows=[2, 0, 2, 0, 3, 3],
                                                post_values=np.float32([3, 1, 4, 2, 5, 6])), "rows [0, 4)")
    same_postings(postings_model(HAND, 2), dict(rows=2, terms=[2, 5], ptr=[0, 1, 2], post_rows=[0, 0],
                                                post_values=np.float32([1, 2])), "rows [0, 2)")
    same_postings(dict(postings_model(HAND, 1), rows=2), postings_model(HAND, 2), "an empty row adds no posting")
    # extending [0, 2) over rows 2 and 3: term 0 is new below every old term, 7 above, 2 and 5 are shared
    same_postings(extend_model(postings_model(HAND, 2), HAND, 4), postings_model(HAND, 4), "hand-worked extension")


def random_table(rng, n, dim, empty=0.1):
    rows = []
    for _ in range(n):
        k = 0 if rng.random() < empty else int(rng.integers(1, 12))
        idx = np.sort(rng.choice(dim, size=min(k, dim), replace=False))
        rows.append([(int(i), float(rng.standard_normal())) for i in idx])
    return csr(rows)


@pytest.mark.parametrize("seed", range(6))
def test_merge_restatement_matches_the_model(seed):
    rng = np.random.default_rng(seed)
    dim = int(rng.integers(2, 60))
    t = random_table(rng, 300, dim)
    n0 = int(rng.integers(1, 150))
    lists = postings_model(t, n0)
    steps = sorted(set(int(x) for x in rng.integers(n0, 301, 4))) + [300]
    for n in steps:
        lists = extend_model(lists, t, n)
        same_postings(lists, postings_model(t, n), "seed %d, [0, %d) extended to %d" % (seed, n0, n))
