"""CPU test: the bit-exact model of sparse graph search (sparse_graph_model.port_model with the numpy fp32 distances of
test_gpu_sparse.ref_distances) reproduces the reference's own build and Search answers in tests/golden/sparse_graph.npz
(make_sparse_graph_golden.py): identical ids and counts, bitwise-equal distances, and per query as many distance
evaluations as the reference's SparseVecDistFunc calls.  The GPU tests compare the device against the same model."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))

from make_sparse_golden import THR, crc, table  # noqa: E402
from make_sparse_graph_golden import CASES, N_GRAPH, drop_empty_query  # noqa: E402
from sparse_graph_model import port_model  # noqa: E402
from test_gpu_sparse import (NT_INT4_ATTR, NT_INT_CONST, NT_NE, assert_bitwise, attr_lt, densify,  # noqa: E402
                             distance_lt, ref_distances)

GOLDEN = os.path.join(HERE, "golden", "sparse_graph.npz")


@pytest.mark.parametrize("metric", [1, 2, 3])
def test_port_model_reproduces_reference_sparse_graph_search(port, metric):
    g = np.load(GOLDEN)
    n, vocab, rows, qs, attr, codes, dead = table(metric)
    assert crc(*rows, *qs) == int(g["m%d_table_crc32" % metric])
    if metric == 2:
        qs = drop_empty_query(qs)
    D = ref_distances(densify(rows, vocab), densify(qs, vocab), metric)
    off = g["m%d_graph_offsets" % metric]
    graph = (N_GRAPH, off, g["m%d_graph_nbrs" % metric].astype(np.int64), int(g["m%d_graph_nav" % metric]))
    assert off.size == N_GRAPH + 1 and off[-1] == graph[2].size
    attrs = np.ascontiguousarray(np.stack([attr, codes], 1).astype(np.int32)).view(np.uint8).ravel()
    deleted = np.zeros((n + 7) // 8, np.uint8)
    np.bitwise_or.at(deleted, dead >> 3, (1 << (dead & 7)).astype(np.uint8))
    code_ne3 = np.array([[NT_INT4_ATTR, 1, -1, -1, 0, 0, 0, 4], [NT_INT_CONST, 1, -1, -1, 3, 0, 0, -1],
                         [NT_NE, 3, 0, 1, 0, 0, 0, -1]], np.int64)   # the string codes as an INT4 column
    nodes = {"numeric": attr_lt(30), "distance": distance_lt(THR[metric]), "string": code_ne3}
    for name, L, limit, visible, _, use_del in CASES:
        total = n if visible is None else visible
        key = "m%d_%s" % (metric, name)
        got = port_model(port, D[:, :total], graph, L, limit, deleted=deleted if use_del else None, attrs=attrs,
                         stride=8, nodes=nodes.get(name))
        want = (g[key + "_ids"].astype(np.int64), g[key + "_dists"].astype(np.float64), g[key + "_counts"].astype(np.int64))
        assert_bitwise(got[:3], want, key)
        assert np.array_equal(got[3], g[key + "_calls"]), key + ": distance evaluations differ from the reference's calls"
