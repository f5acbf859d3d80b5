"""CPU check of the sparse golden file: the numpy fp32 restatement of the reference's sparse distances that the GPU
tests use (tests/test_gpu_sparse.py) reproduces tests/golden/sparse.npz, the reference's own Search answers."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_sparse_golden import CASES, THR, crc, table  # noqa: E402
from sparse_golden_check import check_against_golden  # noqa: E402
from test_gpu_sparse import densify, ref_distances, ref_search  # noqa: E402


def case_filter(name, n, attr, codes, alive, use_del, metric):
    keep = alive.copy() if use_del else np.ones(n, bool)
    dyn = None
    if name == "numeric":
        keep &= attr < 30
    if name == "prefilter":
        keep &= attr < 10
    if name == "string":
        keep &= codes != 3
    if name == "distance":
        dyn = lambda d, t=THR[metric]: d < t  # noqa: E731
    return keep, dyn


def test_restatement_reproduces_reference_golden():
    g = np.load(os.path.join(HERE, "golden", "sparse.npz"))
    for metric in (1, 2, 3):
        n, vocab, rows, qs, attr, codes, dead = table(metric)
        assert crc(*rows, *qs) == int(g["m%d_table_crc32" % metric]), "numpy no longer draws the golden table"
        D = ref_distances(densify(rows, vocab), densify(qs, vocab), metric)
        alive = np.ones(n, bool)
        alive[dead] = False
        for name, _, ll, limit, _, use_del in CASES:
            keep, dyn = case_filter(name, n, attr, codes, alive, use_del, metric)
            ids, ds, cnt = ref_search(D, limit, min(limit, ll), keep=keep, dyn=dyn)
            check_against_golden(g, "m%d_%s" % (metric, name), ids, ds, cnt, metric)
