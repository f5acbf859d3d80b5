"""Restatement in numpy float64 of the reference's expression evaluator and facet grouping, independent of the device
(filter.cuh, facet.cu), for the tests.

    num_eval(nodes, table, dist)       ExprEvaluator::NumEvaluate (engine/query/expr/expr_evaluator.cpp:127-164)
    logical_eval(nodes, table, dist)   ExprEvaluator::LogicalEvaluate (:170-258)
    facet(key, key_type, aggs, table, ids, dists)   FacetExecutor::Aggregate (engine/db/execution/aggregation.hpp:232-300)

`nodes` are the parser's [n, 8] int64 PODs (node_type, value_type, left, right, int_value, double_value bits,
bool_value, field_offset; field_offset -2 is "@distance"), with a StringConst's int_value holding the literal's
dictionary code and a StringAttr's field_offset its string column.  Evaluation is vectorised over the table's rows;
`dist` broadcasts against them (a scalar, one value per row, or a column [D, 1] for D distances at once).

The rules restated:
  * integer attributes widen to int64 and then to double (round to nearest), floats to double; IntConst is its int64
    value as a double;
  * NumEvaluate of any node that is not a constant, an attribute or + - * / % (fmod) is 0.0;
  * a BoolAttr is true for any non-zero byte (:56-59);
  * NOT, AND, OR and an EQ / NE of bools evaluate their children with distance 0 (:166-168), so "@distance" reads the
    real distance only under a numeric comparison at the root;
  * an INT group-by key is (int64_t) of the double, which on x86-64 (cvttsd2si) turns NaN and everything outside
    [-2^63, 2^63) into INT64_MIN.

Variant readings, used to show that the golden file tells them apart: Rules(dist_in_logical=True) lets the distance
through AND / OR / NOT / bool EQ, Rules(bool_byte_one=True) reads only byte 1 as true, and
Rules(int_key_saturating=True) casts INT keys with NaN to 0 and saturation at the int64 limits.
"""
from collections import namedtuple

import numpy as np

import like_model as lm

Rules = namedtuple("Rules", "dist_in_logical bool_byte_one int_key_saturating", defaults=(False, False, False))
REFERENCE = Rules()

INT_CONST, STRING_CONST, DOUBLE_CONST, BOOL_CONST = 1, 2, 3, 4
INT1, INT2, INT4, INT8, STRING_ATTR, DOUBLE_ATTR, FLOAT_ATTR, BOOL_ATTR = 5, 6, 7, 8, 9, 10, 11, 12
ADD, SUB, MUL, DIV, MOD = 14, 15, 16, 17, 18
LT, LTE, EQ, GT, GTE, NE, AND, OR, NOT, LIKE, IN = 19, 20, 21, 22, 23, 24, 25, 26, 27, 29, 34
SUM, MIN, MAX, COUNT = 30, 31, 32, 33
VT_STRING, VT_INT, VT_DOUBLE, VT_BOOL = 0, 1, 2, 3
INT64_MIN = -(1 << 63)
_WIDTH = {INT1: np.int8, INT2: np.int16, INT4: np.int32, INT8: np.int64, FLOAT_ATTR: np.float32, DOUBLE_ATTR: np.float64}


class Table:
    """Row-major attribute bytes [n_rows x stride], the string columns' dictionary codes [columns x n_rows] and the
    dictionary (bytes per code)."""

    def __init__(self, attrs, stride, n_rows, str_codes=None, words=None):
        self.raw = np.asarray(attrs, np.uint8)[:n_rows * stride].reshape(n_rows, stride)
        self.n = n_rows
        self.str_codes = None if str_codes is None else np.asarray(str_codes, np.int64)
        self.words = None if words is None else [w.encode() if isinstance(w, str) else bytes(w) for w in words]

    def column(self, node_type, offset):
        dt = np.dtype(_WIDTH[node_type])
        return self.raw[:, offset:offset + dt.itemsize].copy().view(dt)[:, 0]

    def rows(self, ids):
        """The table restricted to rows `ids` (in that order)."""
        t = Table.__new__(Table)
        t.raw, t.n, t.words = self.raw[ids], len(ids), self.words
        t.str_codes = None if self.str_codes is None else self.str_codes[:, ids]
        return t


def _double(bits):
    return float(np.int64(bits).view(np.float64))


def num_eval(nodes, table, dist, i=None):
    """NumEvaluate(i, row, dist) for every row (i defaults to the root)."""
    nodes = np.asarray(nodes, np.int64)
    i = len(nodes) - 1 if i is None else i
    t, left, right, iv, fo = (int(v) for v in nodes[i, [0, 2, 3, 4, 7]])
    if t == INT_CONST:
        return np.float64(iv)
    if t == DOUBLE_CONST:
        return np.float64(_double(nodes[i, 5]))
    if t in (INT1, INT2, INT4, INT8):
        return table.column(t, fo).astype(np.int64).astype(np.float64)
    if t in (DOUBLE_ATTR, FLOAT_ATTR):
        if fo == -2:
            return np.asarray(dist, np.float64)
        return table.column(t, fo).astype(np.float64)
    if left != -1 and right != -1:
        a, b = num_eval(nodes, table, dist, left), num_eval(nodes, table, dist, right)
        with np.errstate(all="ignore"):
            if t == ADD:
                return a + b
            if t == SUB:
                return a - b
            if t == MUL:
                return a * b
            if t == DIV:
                return np.true_divide(a, b)
            if t == MOD:
                return np.fmod(a, b)
    return np.float64(0.0)


def _codes(nodes, table, i):
    t, fo, iv = int(nodes[i, 0]), int(nodes[i, 7]), int(nodes[i, 4])
    if t == STRING_CONST:
        return np.int64(iv)
    if t == STRING_ATTR:
        return table.str_codes[fo]
    raise NotImplementedError("string node type %d (concatenation is out of scope)" % t)


def _like(nodes, table, left, right):
    a, b = np.broadcast_arrays(_codes(nodes, table, left), _codes(nodes, table, right), np.zeros(table.n, np.int64))[:2]
    return lm.like_many([table.words[c] for c in a], [table.words[c] for c in b])


def logical_eval(nodes, table, dist, i=None, rules=REFERENCE):
    """LogicalEvaluate(i, row, dist) for every row (i defaults to the root)."""
    nodes = np.asarray(nodes, np.int64)
    i = len(nodes) - 1 if i is None else i
    t, vt, left, right, fo = (int(v) for v in nodes[i, [0, 1, 2, 3, 7]])
    inner = dist if rules.dist_in_logical else 0.0   # the two-argument overload passes distance 0 (:166-168)
    sub = lambda j: logical_eval(nodes, table, inner, j, rules)
    if t == BOOL_CONST:
        return np.bool_(nodes[i, 6] != 0)
    if t == BOOL_ATTR:
        byte = table.raw[:, fo]
        return byte == 1 if rules.bool_byte_one else byte != 0
    if t == NOT:
        return ~np.asarray(sub(left))
    if t == IN:
        raise NotImplementedError("IN is lowered to an OR of EQs before it reaches an evaluator")
    if left == -1 or right == -1:
        return np.bool_(False)
    if t in (EQ, NE):
        cvt = int(nodes[left, 1])
        if cvt == VT_STRING:
            r = np.asarray(_codes(nodes, table, left) == _codes(nodes, table, right))
        elif cvt == VT_BOOL:
            r = np.asarray(sub(left) == sub(right))
        else:
            r = np.asarray(num_eval(nodes, table, dist, left) == num_eval(nodes, table, dist, right))
        return r if t == EQ else ~r
    if t in (AND, OR):
        a, b = np.asarray(sub(left)), np.asarray(sub(right))
        return (a & b) if t == AND else (a | b)
    if t == LIKE:
        return _like(nodes, table, left, right)
    if t in (LT, LTE, GT, GTE):
        a, b = num_eval(nodes, table, dist, left), num_eval(nodes, table, dist, right)
        return {LT: np.less, LTE: np.less_equal, GT: np.greater, GTE: np.greater_equal}[t](a, b)
    return np.bool_(False)


def filter_rows(nodes, table, dist, rules=REFERENCE):
    """The filter's verdict for every row, broadcast to the shape of rows x dist."""
    shape = np.broadcast_shapes(np.shape(dist), (table.n,))
    if nodes is None or len(nodes) == 0:
        return np.ones(shape, bool)
    return np.broadcast_to(logical_eval(nodes, table, dist, rules=rules), shape).copy()


def int_key(v, saturating=False):
    """(int64_t)v of an INT group-by key, as an int: x86-64 (the reference), or NaN to 0 and saturation when
    saturating."""
    v = float(v)
    if saturating:
        if v != v:
            return 0
        if v >= 2.0 ** 63:
            return (1 << 63) - 1
        if v < -2.0 ** 63:
            return INT64_MIN
        return int(v)
    if not (-2.0 ** 63 <= v < 2.0 ** 63):
        return INT64_MIN
    return int(v)


def facet(key_nodes, key_type, aggs, table, ids, dists=None, rules=REFERENCE):
    """FacetExecutor::Aggregate over one result list: groups in order of first appearance, [(key, [values])].  Keys are
    ints (INT), floats (DOUBLE), bools (BOOL) or dictionary codes (STRING); aggs is [(agg type, nodes)], values are the
    aggregated doubles (before Project's (int64_t) cast of INT-typed aggregates)."""
    ids = np.asarray(ids, np.int64)
    sub = table.rows(ids)
    d = np.zeros(ids.size) if dists is None else np.asarray(dists, np.float64)
    if key_type == VT_BOOL:
        keys = [bool(k) for k in filter_rows(key_nodes, sub, d, rules)]
    elif key_type == VT_STRING:
        root = len(key_nodes) - 1
        keys = [int(k) for k in np.broadcast_to(_codes(np.asarray(key_nodes), sub, root), ids.shape)]
    else:
        v = np.broadcast_to(num_eval(key_nodes, sub, d), ids.shape)
        keys = [int_key(k, rules.int_key_saturating) for k in v] if key_type == VT_INT else [float(k) for k in v]
    vals = [np.broadcast_to(num_eval(n, sub, d), ids.shape) for _, n in aggs]
    groups = {}
    for r, k in enumerate(keys):
        acc = groups.setdefault(k, [k, [None] * len(aggs)])[1]
        for g, (t, _) in enumerate(aggs):
            v = float(vals[g][r])
            if t in (COUNT, SUM):   # a new key starts at +0.0 (unordered_map's value-initialised double)
                acc[g] = (0.0 if acc[g] is None else acc[g]) + (1.0 if t == COUNT else v)
            elif acc[g] is None or (t == MIN and v < acc[g]) or (t == MAX and v > acc[g]):
                acc[g] = v
    return [(k, acc) for k, acc in groups.values()]


class Golden:
    """tests/golden/exprs.npz (written by tests/golden/make_expr_golden.py): the table, the filter programs with their
    LogicalEvaluate bits [program, distance, row], the value expressions with their NumEvaluate doubles [expression,
    distance, row], and the facet cases with the reference's JSON."""

    def __init__(self, path=None):
        import json
        import os
        path = path or os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "exprs.npz")
        g = np.load(path, allow_pickle=False)
        self.n, self.stride = int(g["n_rows"]), int(g["stride"])
        self.attrs = g["attrs"]
        self.words = [str(w) for w in g["words"]]
        self.str_codes = g["str_codes"]
        self.table = Table(self.attrs, self.stride, self.n, self.str_codes, self.words)
        self.col_offset = dict(zip([str(c) for c in g["col_names"]], g["col_offsets"].tolist()))
        off, nodes, codes = g["filter_off"], g["filter_nodes"].copy(), g["filter_lit_codes"]
        sc = nodes[:, 0] == STRING_CONST
        nodes[sc, 4] = codes[sc]
        self.filter_text = [str(t) for t in g["filter_text"]]
        self.filters = [nodes[off[i]:off[i + 1]] for i in range(off.size - 1)]
        self.filter_dists = g["filter_dists"]
        self.filter_bits = np.unpackbits(g["filter_bits"], axis=2, count=self.n).astype(bool)
        off, nodes = g["value_off"], g["value_nodes"]
        self.value_text = [str(t) for t in g["value_text"]]
        self.values = [nodes[off[i]:off[i + 1]] for i in range(off.size - 1)]
        self.value_type = g["value_type"]
        self.value_dists = g["value_dists"]
        self.value_num = g["value_num"]
        self.facets = []
        for i, group in enumerate(g["facet_group"]):
            aggs = json.loads(str(g["facet_aggs"][i]))
            agg_nodes = [g["facet_agg_nodes_%d_%d" % (i, j)] for j in range(len(aggs))]
            self.facets.append(dict(group=str(group), aggs=aggs, key_type=int(g["facet_key_type"][i]),
                                    key_nodes=g["facet_key_nodes_%d" % i], agg_nodes=agg_nodes,
                                    agg_types=[AGG_TYPE[a[:a.index("(")].upper()] for a in aggs],
                                    ids=g["facet_ids_%d" % i], dists=g["facet_dists_%d" % i],
                                    want=json.loads(str(g["facet_json"][i]))))


AGG_TYPE = {"SUM": SUM, "MIN": MIN, "MAX": MAX, "COUNT": COUNT}


def facet_mismatch(case, got, words):
    """Compare one list's groups [(key, [values])] with the reference's Project() JSON; returns None or a message.
    Keys and group counts are exact; INT-typed aggregates go through Project's (int64_t) cast and must be equal,
    DOUBLE-typed ones within 1e-9 relative (non-finite ones are JSON null)."""
    group, aggs, kt = case["group"], case["aggs"], case["key_type"]
    want = {}
    for obj in case["want"]:
        k = obj[group]
        want[words.index(k) if kt == VT_STRING else k] = [obj[a] for a in aggs]
    if len(got) != len(want):
        return "%s: %d groups, reference %d" % (group, len(got), len(want))
    int_typed = [int(n[-1, 1]) == VT_INT for n in case["agg_nodes"]]
    for key, vals in got:
        k = int(key) if kt in (VT_INT, VT_STRING) else (bool(key) if kt == VT_BOOL else float(key))
        if k not in want:
            return "%s: key %r is not among the reference's %s" % (group, k, sorted(want, key=str)[:8])
        for a, v, w, it in zip(aggs, vals, want[k], int_typed):
            if it:
                ok = int_key(v) == w
            elif w is None:
                ok = not np.isfinite(v)
            else:
                ok = abs(v - w) <= 1e-9 * max(1.0, abs(w))
            if not ok:
                return "%s: key %r %s = %r, reference %r" % (group, k, a, v, w)
    return None
