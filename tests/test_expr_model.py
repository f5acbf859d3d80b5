"""tests/expr_model.py against the reference's own answers (tests/golden/exprs.npz), on the CPU: LogicalEvaluate bits
exactly equal, NumEvaluate doubles bit-equal (NaN matches NaN, the sign of zero counts), facet groups and counts
exact and aggregate values within 1e-9.  The variant readings of the model must each disagree with the golden file,
so a device that read the rules that way would fail the GPU tests held to it."""
import numpy as np
import pytest

import expr_model as em


@pytest.fixture(scope="module")
def g():
    return em.Golden()


def logical(g, nodes, rules=em.REFERENCE):
    return em.filter_rows(nodes, g.table, g.filter_dists[:, None], rules)


def same_doubles(a, b):
    """Bit-equal, except that any NaN matches any NaN."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return (np.isnan(a) & np.isnan(b)) | (a.view(np.int64) == b.view(np.int64))


def test_golden_covers_the_table_edges(g):
    t = g.table
    x, y = t.column(em.FLOAT_ATTR, g.col_offset["x"]), t.column(em.DOUBLE_ATTR, g.col_offset["y"])
    a8 = t.column(em.INT8, g.col_offset["a8"])
    for v in (x, y):
        assert np.isnan(v).any() and np.isposinf(v).any() and np.isneginf(v).any()
        assert np.any((v == 0) & np.signbit(v)) and np.any((v == 0) & ~np.signbit(v))
        assert np.any((v != 0) & (np.abs(v) < np.finfo(v.dtype).tiny))
    assert {2 ** 53 - 1, 2 ** 53 + 1, -2 ** 53 - 1, -2 ** 63, 2 ** 63 - 1} <= set(a8.tolist())
    assert {0, 1, 2, 0x80, 0xFF} <= set(t.raw[:, g.col_offset["t"]].tolist())
    assert (t.column(em.INT4, g.col_offset["b4"]) == 0).sum() > 8
    assert len(g.filters) >= 2000 and len(g.values) >= 300
    assert sum(len(n) == 64 for n in g.filters) >= 1


def test_logical_matches_golden(g):
    bad = [i for i, nodes in enumerate(g.filters) if not np.array_equal(logical(g, nodes), g.filter_bits[i])]
    assert not bad, "%d programs differ, first %r" % (len(bad), g.filter_text[bad[0]])


def test_numeric_matches_golden_bitwise(g):
    for i, nodes in enumerate(g.values):
        got = np.broadcast_to(em.num_eval(nodes, g.table, g.value_dists[:, None]), g.value_num[i].shape)
        ok = same_doubles(got, g.value_num[i])
        assert ok.all(), "%r: %d values differ, first %r vs %r" % (g.value_text[i], (~ok).sum(), got[~ok][0],
                                                                    g.value_num[i][~ok][0])


def test_facets_match_golden(g):
    for case in g.facets:
        aggs = list(zip(case["agg_types"], case["agg_nodes"]))
        got = em.facet(case["key_nodes"], case["key_type"], aggs, g.table, case["ids"], case["dists"])
        msg = em.facet_mismatch(case, got, g.words)
        assert msg is None, msg


def test_int_key_example(g):
    """The grouping of include/epsilla_b200.h's eps_facet example: a4 / b4 and a4 % b4 over rows 0..7."""
    want = {"a4 / b4": {2: 1, 1: 1, 0: 1, 3: 2, em.INT64_MIN: 3}, "a4 % b4": {0: 4, 1: 1, em.INT64_MIN: 3}}
    saturating = {"a4 / b4": {0: 2, 2: 1, 1: 1, 3: 2, 2 ** 63 - 1: 1, em.INT64_MIN: 1}, "a4 % b4": {0: 7, 1: 1}}
    for case in g.facets[:2]:
        aggs = list(zip(case["agg_types"], case["agg_nodes"]))
        assert case["aggs"] == ["COUNT(*)"] and list(case["ids"]) == list(range(8))
        for rules, w in ((em.REFERENCE, want), (em.Rules(int_key_saturating=True), saturating)):
            got = em.facet(case["key_nodes"], case["key_type"], aggs, g.table, case["ids"], case["dists"], rules)
            assert {k: v[0] for k, v in got} == w[case["group"]]


def test_variant_readings_disagree(g):
    """Each plausible misreading is caught by the golden file."""
    for rules in (em.Rules(dist_in_logical=True), em.Rules(bool_byte_one=True)):
        wrong = sum(not np.array_equal(logical(g, nodes, rules), g.filter_bits[i]) for i, nodes in enumerate(g.filters))
        assert wrong > 0, rules
    sat = em.Rules(int_key_saturating=True)
    wrong = 0
    for case in g.facets:
        aggs = list(zip(case["agg_types"], case["agg_nodes"]))
        got = em.facet(case["key_nodes"], case["key_type"], aggs, g.table, case["ids"], case["dists"], sat)
        wrong += em.facet_mismatch(case, got, g.words) is not None
    assert wrong > 0
