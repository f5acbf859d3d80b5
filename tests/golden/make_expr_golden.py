"""Writes tests/golden/exprs.npz: the reference's own answers for filter and value expressions on a typed table.

    python tests/golden/make_expr_golden.py

Needs oracle/_ref/libepsilla_ref.so (built by __graft_entry__.build() from a reference checkout) and that checkout's
headers ($EPSILLA_REFERENCE or oracle.reference_dir()).  Everything is drawn from fixed seeds, so a re-run writes the same
file bit for bit.

The table has N_ROWS rows and the columns of COLS: every integer width, float, double, two bool columns and two string
columns.  Its values hold the integer limits, int64 values around +-2^53 and at the int64 limits, zeros in the divisor
column b4, NaN, +-inf, +-0.0 and subnormals in x and y, the literals the programs use, and bool bytes 2, 0x80 and 0xFF
(ExprEvaluator reads any non-zero byte as true).  The numeric columns are written into the reference's own attribute
table through oracle.Ref, whose parser also supplies each program's node PODs (ref_filter_nodes / ref_value_nodes).

The small driver below is test infrastructure: it parses an expression with the reference's parser once and asks
ExprEvaluator for every row at every distance: LogicalEvaluate(root, row, d) for filter programs, the raw float64
NumEvaluate(root, row, d) for value expressions (stored as doubles, never through JSON).  Facet cases go through the
reference's FacetExecutor (oracle.Ref.facet), whose Project() output is JSON.

Stored: the table (attrs, stride, string values), the filter programs (text, PODs, the dictionary code of each string
literal, LogicalEvaluate bits [program, distance, row] packed along rows), the value expressions (text, PODs, root
value type, NumEvaluate [expression, distance, row]) and the facet cases (key, aggregates, id lists, distances, JSON).
String codes index the sorted set of every string in the table and every literal; a literal of a filter that appears
in no row keeps its code, so EQ against it matches no row.
"""
import ctypes as C
import io
import json
import os
import re
import subprocess
import sys
import tempfile
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

DRIVER = r'''
#include <cstdint>
#include <string>
#include <unordered_map>
#include <vector>
#include "db/catalog/meta_types.hpp"
#include "db/vector.hpp"
#include "query/expr/expr.hpp"
#include "query/expr/expr_evaluator.hpp"
using namespace vectordb;
using namespace vectordb::query::expr;

struct Table {
  std::unordered_map<std::string, engine::meta::FieldType> types;
  std::unordered_map<std::string, size_t> offsets;
  int64_t stride = 0, n_str = 0;
  char* attrs = nullptr;
  std::vector<engine::VariableLenAttrColumnContainer> strs;
};

extern "C" void* table_new(char* attrs, int64_t stride, int64_t n_rows, int n_fields, const char* const* names,
                           const int* types, const int64_t* offsets) {
  auto* t = new Table();
  t->attrs = attrs;
  t->stride = stride;
  for (int i = 0; i < n_fields; ++i) {
    t->types[names[i]] = static_cast<engine::meta::FieldType>(types[i]);
    t->offsets[names[i]] = static_cast<size_t>(offsets[i]);
    if (types[i] == static_cast<int>(engine::meta::FieldType::STRING)) ++t->n_str;
  }
  t->types["@distance"] = engine::meta::FieldType::DOUBLE;
  t->strs.resize(t->n_str, engine::VariableLenAttrColumnContainer(n_rows));
  return t;
}

extern "C" void table_set_string(void* h, int64_t col, int64_t row, const char* s) {
  static_cast<Table*>(h)->strs[col][row] = std::string(s);
}

// LogicalEvaluate (logical != 0) or NumEvaluate of the root for every row at every distance: out[d * n_rows + row].
// Returns the node count, or -1 when the text does not parse.
extern "C" int64_t eval_expr(void* h, const char* text, int logical, int64_t n_rows, const double* dists, int64_t nd,
                             uint8_t* bits, double* nums) {
  auto* t = static_cast<Table*>(h);
  std::vector<ExprNodePtr> nodes;
  if (!Expr::ParseNodeFromStr(text, nodes, t->types, logical != 0).ok() || nodes.empty()) return -1;
  ExprEvaluator ev(nodes, t->offsets, t->stride, t->n_str, t->attrs, t->strs);
  const int root = static_cast<int>(nodes.size()) - 1;
  for (int64_t d = 0; d < nd; ++d)
    for (int64_t r = 0; r < n_rows; ++r) {
      if (logical) bits[d * n_rows + r] = ev.LogicalEvaluate(root, r, dists[d]) ? 1 : 0;
      else nums[d * n_rows + r] = ev.NumEvaluate(root, r, dists[d]);
    }
  return static_cast<int64_t>(nodes.size());
}
'''

N_ROWS = 256
COLS = [("a1", "int1"), ("a2", "int2"), ("a4", "int4"), ("a8", "int8"), ("b4", "int4"), ("x", "float"), ("y", "double"),
        ("t", "bool"), ("u", "bool"), ("s", "string"), ("w", "string")]
INT_COLS = ["a1", "a2", "a4", "a8", "b4"]
REAL_COLS = ["x", "y"]
BOOL_COLS = ["t", "u"]
STR_COLS = ["s", "w"]

# Column values.  The first 8 rows of a4 / b4 are the grouping example of include/epsilla_b200.h (eps_facet).
A4_HEAD, B4_HEAD = [0, 5, -5, 7, 0, 1, 2, 3], [0, 0, 0, 2, 1, 1, 1, 1]
POOLS = {
    "a1": [-128, 127, 0, 1, -1, 2, -2, 3, 5, 7, -7],
    "a2": [-32768, 32767, 0, 1, -1, 2, 3, 5, 7, -300, 1000],
    "a4": [-2147483648, 2147483647, 0, 1, -1, 2, 3, 5, 7, -5, 65536],
    "a8": [2 ** 53 - 1, 2 ** 53, 2 ** 53 + 1, -2 ** 53 - 1, -2 ** 53, -2 ** 53 + 1, -2 ** 63, 2 ** 63 - 1, 0, 1, -1, 2,
           7, 3],
    "b4": [0, 0, 0, 1, -1, 2, -2, 3, -3, 7],
    "x": [np.nan, np.inf, -np.inf, 0.0, -0.0, 1e-40, -1e-45, 1.5, -0.5, 2.25, 3.0, 0.25, 2.0, 7.0, -3.0, 1e30, 0.1, -1.5],
    "y": [np.nan, np.inf, -np.inf, 0.0, -0.0, 5e-324, -2.2250738585072014e-308, 1.5, -0.5, 2.25, 3.0, 0.25, 2.0, 7.0,
          -3.0, 2.0 ** 63, -2.0 ** 63, 1e300, 0.1, 9007199254740993.0, -1.5],
    "t": [0, 1, 2, 0x80, 0xFF],
    "u": [0, 1, 0, 1, 0xFF],
    "s": ["", "a", "b", "ab", "a%", "x y"],
    "w": ["", "a", "ab", "zz", "b"],
}
INT_LITS = ["0", "1", "-1", "2", "3", "5", "7", "-5", "127", "-128", "32767", "-32768", "2147483647", "-2147483647",
            "65536", "1000"]
REAL_LITS = ["0.0", "-0.0", "1.5", "-0.5", "2.25", "0.25", "3.0", "2.0", "7.0", "0.1", "1000000.5", "-1.5"]
STR_LITS = ["a", "ab", "", "zzz", "x y", "b"]      # 'zzz' is in no row
LIKE_PATS = ["a%", "%b", "_", "%", "", "%a%"]
# "@distance" of the filter programs: zeros of both signs, IP-style negatives, and values the columns and literals hold
FILTER_DISTS = [0.0, -0.0, -1.5, 2.0, 7.0, 0.25, -3.0, 1.5]
VALUE_DISTS = [0.0, -0.0, -1.5, 7.0]
N_RANDOM_FILTERS, N_RANDOM_VALUES = 2000, 300
MAX_NODES = 64

NT = dict(IntConst=1, StringConst=2, DoubleConst=3, BoolConst=4, Int1=5, Int2=6, Int4=7, Int8=8, StringAttr=9,
          DoubleAttr=10, FloatAttr=11, BoolAttr=12, Add=14, Sub=15, Mul=16, Div=17, Mod=18, LT=19, LTE=20, EQ=21, GT=22,
          GTE=23, NE=24, AND=25, OR=26, NOT=27, LIKE=29)
ARITH = (14, 15, 16, 17, 18)
CMP = (19, 20, 22, 23)
VT_INT, VT_DOUBLE, VT_BOOL = 1, 2, 3

# Hand-written programs: every family at least once whatever the random draw.
CURATED_FILTERS = [
    "a1 < 2", "a2 >= -32768", "a4 <= 2147483647", "a8 > 2147483647", "a8 = a8 + 1", "a8 - 1 < a8", "b4 <> 0",
    "x < 1.5", "x = 2.0", "x <> x", "y >= y", "y = 0.0", "y = -0.0", "x > -0.0", "y <= 7.0",
    "a4 / b4 > 1", "a4 % b4 = 0", "a4 % b4 <> a4 % b4", "-5 % b4 = -1", "a1 % -3 < 0", "a4 / 0 > 0", "x / 0 < 0",
    "x % 0.0 = x % 0.0", "y % 2 = -1.5", "a1 + x > 2.25", "a2 * y < 0.25", "a8 / 3 = y", "(a4 - b4) * 2.25 >= 3.0",
    "x * y <> y * x", "a8 + 0.1 = a8",
    "t", "u", "NOT (t)", "NOT (NOT (u))", "t AND u", "(t OR u) AND (NOT (t))", "((t AND (a1 < 2)) OR (u AND (x > 0.0))) AND (NOT ((y < 0.0) OR u))",
    "t = true", "t = u", "t <> u", "(a1 < 2) = (t)", "(x > 0.0) <> (y > 0.0)", "(t) = (NOT (u))", "false OR t", "true",
    "@distance < 1.5", "@distance >= 0.0", "@distance = -0.0", "@distance > -1.5", "@distance = a1", "y <= @distance",
    "@distance * 2 + a1 > 3", "1 / @distance > 0", "(@distance - x) * y < 0.25", "@distance % 2 = 0",
    "(@distance < 1.5) AND t", "(@distance < 1.5) OR u", "NOT (@distance < 1.5)", "NOT (@distance >= 0.0)",
    "(@distance >= 0.0) = (t)", "(t) <> (@distance < 2.0)", "((@distance > 1.5) AND (a1 > 0)) OR (NOT (@distance < 0.0))",
    "s = 'a'", "s <> 'ab'", "s = 'zzz'", "s <> 'zzz'", "s = w", "s <> w", "'x y' = s", "s = ''",
    "s LIKE 'a%' AND a1 > 0", "(w LIKE '%b') OR (x < 1.5)", "NOT (s LIKE '_') AND (@distance < 2.0)",
]


def load_driver():
    from oracle.oracle import reference_dir
    ref = reference_dir()
    so = os.path.join(ROOT, "oracle", "_ref", "libepsilla_ref.so")
    if not ref or not os.path.exists(so):
        sys.exit("make_expr_golden: needs a reference checkout and oracle/_ref/libepsilla_ref.so (run build())")
    tmp = tempfile.mkdtemp(prefix="expr_ref_")
    src, out = os.path.join(tmp, "expr_driver.cpp"), os.path.join(tmp, "libexpr_driver.so")
    open(src, "w").write(DRIVER)
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-DNDEBUG", "-fopenmp", "-fPIC", "-w", "-shared",
                           "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ref, "engine"), src, "-o", out,
                           so, "-Wl,-rpath," + os.path.dirname(so)])
    L = C.CDLL(out)
    vp, i64 = C.c_void_p, C.c_int64
    L.table_new.restype = vp
    L.table_new.argtypes = [vp, i64, i64, C.c_int, vp, vp, vp]
    L.table_set_string.argtypes = [vp, i64, i64, C.c_char_p]
    L.eval_expr.restype = i64
    L.eval_expr.argtypes = [vp, C.c_char_p, C.c_int, i64, vp, i64, vp, vp]
    return L


def column_values(rng):
    """Every column's N_ROWS values: each pool value at least once, the rest drawn from the pool."""
    vals = {}
    for name, _ in COLS:
        pool = POOLS[name]
        idx = np.concatenate([np.arange(len(pool)), rng.integers(0, len(pool), N_ROWS - len(pool))])
        rng.shuffle(idx)
        vals[name] = [pool[i] for i in idx]
    vals["a4"][:8], vals["b4"][:8] = A4_HEAD, B4_HEAD
    return vals


def build_table(vals):
    from oracle.oracle import Ref
    ref = Ref("l2", 2, N_ROWS, attr_cols=COLS)
    ref.set_rows(np.zeros((N_ROWS, 2), np.float32))
    for name, typ in COLS:
        if typ == "string":
            ref.set_string_column(name, vals[name])
        elif typ == "bool":   # the raw bytes, 2, 0x80 and 0xFF among them, through the Ref.attrs view
            raw = ref.attrs.reshape(ref.capacity, ref.stride)
            raw[:N_ROWS, ref.attr_offset(name)] = np.array(vals[name], np.uint8)
        else:
            ref.set_attr_column(name, np.array(vals[name]))
    return ref


class Gen:
    """Seeded random filter programs and value expressions over COLS, within the reference parser's grammar: '<>' for
    not-equal, no unary minus (negative literals only), no exponent or leading-dot literals, int32 integer literals."""

    def __init__(self, rng):
        self.rng = rng

    def pick(self, seq):
        return seq[int(self.rng.integers(0, len(seq)))]

    def num(self, depth):
        r = self.rng.random()
        if depth <= 0 or r < 0.45:
            k = self.rng.random()
            if k < 0.35:
                return self.pick(INT_COLS)
            if k < 0.55:
                return self.pick(REAL_COLS)
            if k < 0.7:
                return self.pick(INT_LITS)
            if k < 0.85:
                return self.pick(REAL_LITS)
            return "@distance"
        op = self.pick(["+", "-", "*", "/", "%"])
        return "(%s %s %s)" % (self.num(depth - 1), op, self.num(depth - 1))

    def boolean(self, depth):
        r = self.rng.random()
        if depth <= 0:
            r = r * 0.5
        if r < 0.3:
            return "(%s %s %s)" % (self.num(depth - 1), self.pick(["<", "<=", ">", ">=", "=", "<>"]), self.num(depth - 1))
        if r < 0.36:
            return self.pick(BOOL_COLS)
        if r < 0.38:
            return self.pick(["true", "false"])
        if r < 0.44:
            return "(%s %s '%s')" % (self.pick(STR_COLS), self.pick(["=", "<>"]), self.pick(STR_LITS))
        if r < 0.47:
            return "(s %s w)" % self.pick(["=", "<>"])
        if r < 0.5:
            return "(%s LIKE '%s')" % (self.pick(STR_COLS), self.pick(LIKE_PATS))
        if r < 0.62:
            return "(NOT %s)" % self.paren(self.boolean(depth - 1))
        if r < 0.9:
            return "(%s %s %s)" % (self.boolean(depth - 1), self.pick(["AND", "OR"]), self.boolean(depth - 1))
        return "(%s %s %s)" % (self.paren(self.boolean(depth - 1)), self.pick(["=", "<>"]), self.paren(self.boolean(depth - 1)))

    @staticmethod
    def paren(e):
        return e if e.startswith("(") else "(%s)" % e

    def value(self):
        return self.num(int(self.rng.integers(0, 5)))


def families(nodes):
    """The families of FILTER_FAMILIES a program's nodes belong to."""
    t, vt, left, right, iv, fo = nodes[:, 0], nodes[:, 1], nodes[:, 2], nodes[:, 3], nodes[:, 4], nodes[:, 7]
    root = t[-1]
    found = set()
    n = len(nodes)
    uses_dist = bool(np.any(((t == 10) | (t == 11)) & (fo == -2)))
    for i in range(n):
        ti = t[i]
        if ti in CMP + (21, 24):
            for c in (left[i], right[i]):
                if t[c] in (5, 6, 7, 8, 10, 11) and fo[c] != -2:
                    found.add("cmp_%d" % t[c])
        if ti in ARITH:
            found.add("op_%d" % ti)
            if {vt[left[i]], vt[right[i]]} == {VT_INT, VT_DOUBLE}:
                found.add("mixed_int_float")
            rc = right[i]
            if ti in (17, 18) and ((t[rc] == 1 and iv[rc] == 0) or t[rc] == 7 and fo[rc] == 15):
                found.add("by_zero_%d" % ti)
            if ti == 18 and any(t[c] == 1 and iv[c] < 0 for c in (left[i], right[i])):
                found.add("mod_negative")
        if ti == 12:
            found.add("bool_attr")
        if ti == 27:
            found.add("not")
        if ti in (25, 26) and (t[left[i]] in (25, 26) or t[right[i]] in (25, 26)):
            found.add("nested_and_or")
        if ti in (21, 24) and vt[left[i]] == VT_BOOL:
            found.add("bool_eq")
        if ti in (21, 24) and vt[left[i]] == 0:
            found.add("string_eq")
        if ti == 29 and np.any(np.isin(t, CMP)):
            found.add("like_with_numeric")
    if uses_dist:
        if root in CMP + (21, 24) and vt[left[-1]] not in (0, VT_BOOL):
            if any(t[c] in (10, 11) and fo[c] == -2 for c in (left[-1], right[-1])):
                found.add("dist_root_cmp")
            if any(t[i] in ARITH and (fo[left[i]] == -2 or fo[right[i]] == -2) for i in range(n)):
                found.add("dist_in_arith")
        if root in (25, 26):
            found.add("dist_under_and_or")
        if root == 27:
            found.add("dist_under_not")
        if root in (21, 24) and vt[left[-1]] == VT_BOOL:
            found.add("dist_under_bool_eq")
    if n == MAX_NODES:
        found.add("64_nodes")
    return found


FILTER_FAMILIES = ["cmp_5", "cmp_6", "cmp_7", "cmp_8", "cmp_10", "cmp_11", "op_14", "op_15", "op_16", "op_17", "op_18",
                   "mixed_int_float", "by_zero_17", "by_zero_18", "mod_negative", "bool_attr", "not", "nested_and_or",
                   "bool_eq", "string_eq", "like_with_numeric", "dist_root_cmp", "dist_in_arith", "dist_under_and_or",
                   "dist_under_not", "dist_under_bool_eq", "64_nodes"]


def literal_codes(text, nodes, code):
    """Dictionary code of every node (the literal's for StringConst nodes, 0 elsewhere).  The parser emits StringConst
    nodes in textual order."""
    lits = re.findall(r"'([^']*)'", text)
    sc = np.flatnonzero(nodes[:, 0] == NT["StringConst"])
    assert len(sc) == len(lits), text
    out = np.zeros(len(nodes), np.int32)
    out[sc] = [code[s] for s in lits]
    return out


def facet_cases(vals, rng):
    """(group expression, aggregates, id list) triples.  DOUBLE keys only over rows where they are finite: a NaN key
    makes FacetExecutor::Project throw."""
    y = np.array(vals["y"], np.float64)
    x = np.array(vals["x"], np.float32).astype(np.float64)
    every = np.arange(N_ROWS)
    fin_y = np.flatnonzero(np.isfinite(y) & (np.abs(y) < 1e300))
    fin_x = np.flatnonzero(np.isfinite(x))
    perm = rng.permutation(N_ROWS)
    cases = [
        ("a4 / b4", ["COUNT(*)"], np.arange(8)),
        ("a4 % b4", ["COUNT(*)"], np.arange(8)),
        ("a4 / b4", ["COUNT(*)", "SUM(a1)", "MIN(y)", "MAX(x)"], every),
        ("a4 % b4", ["COUNT(*)", "SUM(b4)", "MIN(a8)", "MAX(@distance)"], perm[:100]),
        ("a8 * 2", ["COUNT(*)", "SUM(a1)"], every),
        ("a8 + a8", ["MAX(a2)", "MIN(a2)"], perm),
        ("a1 * 100000000", ["COUNT(*)", "SUM(a4 / b4)"], every),
        ("@distance > 1.5", ["COUNT(*)", "MAX(@distance)", "MIN(a1 + @distance)"], every),
        ("(@distance > 1.5) AND t", ["COUNT(*)", "SUM(@distance)"], every),
        ("t", ["COUNT(*)", "SUM(a2)", "MIN(x)", "MAX(y)"], every),
        ("(t) = (u)", ["COUNT(*)", "MIN(b4)"], perm[:77]),
        ("s", ["COUNT(*)", "SUM(a2)", "MIN(@distance)", "MAX(a1)"], every),
        ("w", ["COUNT(*)", "MAX(a4 % b4)"], perm[:150]),
        ("y", ["COUNT(*)", "SUM(a1)", "MIN(a2)", "MAX(@distance * 2)"], fin_y),
        ("y * 0", ["COUNT(*)", "SUM(x)"], fin_y),
        ("x - 0.25", ["COUNT(*)", "MAX(a1 / b4)"], fin_x),
        ("a2 % 5", ["SUM(x)", "SUM(y)", "MIN(x)", "MAX(y)", "COUNT(*)"], every),
    ]
    return cases


def main():
    L = load_driver()
    rng = np.random.default_rng(20261017)
    vals = column_values(rng)
    ref = build_table(vals)
    stride = ref.stride
    names = (C.c_char_p * len(COLS))(*[n.encode() for n, _ in COLS])
    from oracle.oracle import FIELD_TYPE
    types = (C.c_int * len(COLS))(*[FIELD_TYPE[t] for _, t in COLS])
    offs = np.array([ref.attr_offset(n) for n, _ in COLS], np.int64)
    tab = L.table_new(C.cast(ref.L.ref_attrs(ref.h), C.c_void_p), stride, N_ROWS, len(COLS), names, types, offs.ctypes.data)
    for ci, name in enumerate(STR_COLS):
        assert ref.attr_offset(name) == ci
        for r, v in enumerate(vals[name]):
            L.table_set_string(tab, ci, r, v.encode())
    words = sorted(set(vals["s"]) | set(vals["w"]) | set(STR_LITS) | set(LIKE_PATS))
    code = {w: i for i, w in enumerate(words)}

    gen = Gen(np.random.default_rng(7))
    fd = np.array(FILTER_DISTS, np.float64)
    texts, node_list, codes, bits, fams = [], [], [], [], set()

    def add_filter(text):
        try:
            nodes = ref.filter_nodes(text)
        except ValueError:
            return False     # does not parse, or more than 64 nodes
        out = np.zeros((fd.size, N_ROWS), np.uint8)
        n = L.eval_expr(tab, text.encode(), 1, N_ROWS, fd.ctypes.data, fd.size, out.ctypes.data, None)
        assert n == len(nodes), text
        texts.append(text)
        node_list.append(nodes)
        codes.append(literal_codes(text, nodes, code))
        bits.append(out)
        fams.update(families(nodes))
        return True

    for text in CURATED_FILTERS:
        assert add_filter(text), text
    # programs of exactly 64 nodes: a random program wrapped in NOTs up to the limit
    n64 = 0
    while n64 < 24:
        text = gen.boolean(5)
        try:
            n = len(ref.filter_nodes(text))
        except ValueError:
            continue
        if 30 <= n <= MAX_NODES:
            k = MAX_NODES - n
            n64 += add_filter("NOT (" * k + text + ")" * k)
    while len(texts) < len(CURATED_FILTERS) + 24 + N_RANDOM_FILTERS:
        add_filter(gen.boolean(int(gen.rng.integers(1, 6))))
    missing = [f for f in FILTER_FAMILIES if f not in fams]
    assert not missing, "families without a program: %s" % missing

    vd = np.array(VALUE_DISTS, np.float64)
    vtexts, vnodes, vtypes, vnums = [], [], [], []
    vgen = Gen(np.random.default_rng(8))
    curated_values = ["a4 / b4", "a4 % b4", "-5 % b4", "a8 * 2", "a8 + a8", "a8 - 1", "a8 + 0.5", "x / 0", "y % 0.0",
                      "x * y", "@distance", "1 / @distance", "@distance % 2", "@distance - x", "a1 / 3", "a2 % -3",
                      "y - y", "x + 0.1", "0.1 + 0.25", "a4 * 65536", "a8 / -1"] + [c for c in INT_COLS + REAL_COLS]
    pending = list(curated_values)
    while len(vtexts) < len(curated_values) + N_RANDOM_VALUES:
        text = pending.pop(0) if pending else vgen.value()
        try:
            nodes, vt = ref.value_nodes(text)
        except ValueError:
            assert text not in curated_values, text
            continue
        out = np.zeros((vd.size, N_ROWS), np.float64)
        n = L.eval_expr(tab, text.encode(), 0, N_ROWS, vd.ctypes.data, vd.size, None, out.ctypes.data)
        assert n == len(nodes), text
        vtexts.append(text)
        vnodes.append(nodes)
        vtypes.append(vt)
        vnums.append(out)
    vn = np.array(vnums)
    assert np.isnan(vn).any() and np.isinf(vn).any() and np.any((vn == 0) & np.signbit(vn))

    frng = np.random.default_rng(9)
    fcases = []
    for group, aggs, ids in facet_cases(vals, frng):
        kn, kt = ref.value_nodes(group)
        ids = np.asarray(ids, np.int64)
        ds = np.array(FILTER_DISTS, np.float64)[frng.integers(0, len(FILTER_DISTS), ids.size)]
        fcases.append((group, aggs, ids, ds, kn, kt, json.dumps(ref.facet(group, aggs, ids, ds))))
    kinds = {kt for _, _, _, _, _, kt, _ in fcases}
    assert kinds == {0, 1, 2, 3}, kinds

    def cat(arrs):
        off = np.zeros(len(arrs) + 1, np.int64)
        np.cumsum([len(a) for a in arrs], out=off[1:])
        return off, np.concatenate(arrs)

    f_off, f_nodes = cat(node_list)
    v_off, v_nodes = cat(vnodes)
    out = dict(
        n_rows=np.int64(N_ROWS), stride=np.int64(stride), attrs=ref.attrs[:N_ROWS * stride].copy(),
        col_names=np.array([n for n, _ in COLS]), col_types=np.array([t for _, t in COLS]), col_offsets=offs,
        words=np.array(words), str_codes=np.array([[code[v] for v in vals[c]] for c in STR_COLS], np.int32),
        filter_text=np.array(texts), filter_off=f_off, filter_nodes=f_nodes,
        filter_lit_codes=np.concatenate(codes), filter_dists=fd,
        filter_bits=np.packbits(np.array(bits), axis=2),
        value_text=np.array(vtexts), value_off=v_off, value_nodes=v_nodes, value_type=np.array(vtypes, np.int64),
        value_dists=vd, value_num=vn,
        facet_group=np.array([c[0] for c in fcases]), facet_aggs=np.array([json.dumps(c[1]) for c in fcases]),
        facet_json=np.array([c[6] for c in fcases]), facet_key_type=np.array([c[5] for c in fcases], np.int64))
    for i, c in enumerate(fcases):
        out["facet_ids_%d" % i], out["facet_dists_%d" % i], out["facet_key_nodes_%d" % i] = c[2], c[3], c[4]
        for j, a in enumerate(c[1]):
            inner = "1" if a.upper().startswith("COUNT(") else a[a.index("(") + 1:-1]
            out["facet_agg_nodes_%d_%d" % (i, j)] = ref.value_nodes(inner)[0]
    path = os.path.join(HERE, "exprs.npz")
    # np.savez_compressed stamps the zip members with the current time; write them with a fixed one instead
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(out):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(out[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())
    print("wrote exprs.npz: %d filter programs (%d of 64 nodes), %d value expressions, %d facet cases; %d bytes" % (
        len(texts), sum(len(n) == MAX_NODES for n in node_list), len(vtexts), len(fcases), os.path.getsize(path)))


if __name__ == "__main__":
    main()
