"""Writes tests/golden/like.npz: the reference's own LIKE answers on hand-built expression nodes.

    python tests/golden/make_like_golden.py

Needs oracle/_ref/libepsilla_ref.so (built by __graft_entry__.build() from a reference checkout) and that checkout's
headers ($EPSILLA_REFERENCE or oracle.reference_dir()).  The small driver below is test infrastructure: for every
pattern it builds the nodes StringAttr 's', StringConst <pattern>, LIKE by hand (bypassing the parser's quoting) and
asks ExprEvaluator::LogicalEvaluate for every subject of the column.  The file stores the subjects, the patterns (as
offsets + bytes) and the match matrix [subjects x patterns].

It also stores the reference's VecSearchExecutor::Search answers (oracle.Ref, IntraQueryThreads = 1) for the LIKE
filters of SEARCH_FILTERS, parsed by the reference's own parser, on a seeded integer-valued table (exact distances in
any summation order) with an INT4 column 'a' and STRING columns 'title' and 'tag': the brute-force branch (no graph),
prefilter, and the graph branch over a random CSR of the first 2500 rows (stored) with a 500-row tail.  For every
filter it keeps the parser's node array (the PODs of ref_filter_nodes) and its string literals in textual order, which
is the order of its StringConst nodes.
"""
import ctypes as C
import os
import re
import subprocess
import sys
import tempfile
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

DRIVER = r'''
#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>
#include "db/vector.hpp"
#include "query/expr/expr_evaluator.hpp"
using namespace vectordb;
using namespace vectordb::query::expr;
extern "C" int like_matrix(int64_t ns, const int64_t* soff, const char* sb, int64_t np, const int64_t* poff,
                           const char* pb, uint8_t* out) {
  std::vector<engine::VariableLenAttrColumnContainer> var(1);
  for (int64_t i = 0; i < ns; ++i) var[0].push_back(std::string(sb + soff[i], soff[i + 1] - soff[i]));
  std::unordered_map<std::string, size_t> fmap{{"s", 0}};
  int64_t primitive = 0, n_str = 1;
  for (int64_t p = 0; p < np; ++p) {
    std::vector<ExprNodePtr> nodes(3);
    for (auto& n : nodes) n = std::make_shared<ExprNode>();
    nodes[0]->node_type = NodeType::StringAttr; nodes[0]->value_type = ValueType::STRING; nodes[0]->field_name = "s";
    nodes[1]->node_type = NodeType::StringConst; nodes[1]->value_type = ValueType::STRING;
    nodes[1]->str_value = std::string(pb + poff[p], poff[p + 1] - poff[p]);
    nodes[2]->node_type = NodeType::LIKE; nodes[2]->value_type = ValueType::BOOL; nodes[2]->left = 0; nodes[2]->right = 1;
    ExprEvaluator ev(nodes, fmap, primitive, n_str, nullptr, var);
    for (int64_t i = 0; i < ns; ++i) out[i * np + p] = ev.LogicalEvaluate(2, i) ? 1 : 0;
  }
  return 0;
}
'''


def load_driver():
    from oracle.oracle import reference_dir
    ref = reference_dir()
    so = os.path.join(ROOT, "oracle", "_ref", "libepsilla_ref.so")
    if not ref or not os.path.exists(so):
        sys.exit("make_like_golden: needs a reference checkout and oracle/_ref/libepsilla_ref.so (run build())")
    tmp = tempfile.mkdtemp(prefix="like_ref_")
    src, out = os.path.join(tmp, "like_driver.cpp"), os.path.join(tmp, "liblike_driver.so")
    open(src, "w").write(DRIVER)
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-DNDEBUG", "-fopenmp", "-fPIC", "-w", "-shared",
                           "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ref, "engine"), src, "-o", out,
                           so, "-Wl,-rpath," + os.path.dirname(so)])
    L = C.CDLL(out)
    vp, i64 = C.c_void_p, C.c_int64
    L.like_matrix.argtypes = [i64, vp, vp, i64, vp, vp, vp]
    return L


def pack(strings):
    off = np.zeros(len(strings) + 1, np.int64)
    np.cumsum([len(s) for s in strings], out=off[1:])
    return off, np.frombuffer(b"".join(strings) + b"\0", np.uint8)[:-1].copy()


def unpack(off, buf):
    b = buf.tobytes()
    return [b[off[i]:off[i + 1]] for i in range(off.size - 1)]


META = b".*\\[]()$^|?+{}"


def cases():
    """~200 subjects x ~60 patterns: empty strings, line terminators on either side, every regex metacharacter, '_'
    runs, UTF-8 text, NUL and subjects up to a few hundred bytes.  At most three '%' per pattern: libstdc++'s
    regex_match backtracks through every split of a failing subject, O(n^k) for k '.*' (the device tests hold longer
    chains to tests/like_model.py)."""
    rng = np.random.default_rng(2026)
    subj = [b"", b"a", b"ab", b"abc", b"a\nb", b"a\rb", b"\n", b"\r", b"\r\n", b"ab\n", b"\nab", b"a\n\nb", b"%", b"_",
            b"%%", b"a%b", b"a_b", b"A", b"ABC", b"\0", b"a\0b", "café".encode(), "été".encode(),
            "日本語".encode(), b"\xff\xfe", b"city of sale", b"sale", b"wholesale\nsale", b"x" * 300,
            (b"ab" * 150), b"a" * 299 + b"b", b"a\n" * 100]
    subj += [bytes([c]) for c in META] + [b"a" + bytes([c]) + b"b" for c in META] + [META]
    alphabet = np.frombuffer(b"ab.\n\r%_*\\[\xc3\xa9$", np.uint8)
    while len(subj) < 200:
        n = int(rng.integers(0, 40 if len(subj) % 3 else 300))
        subj.append(alphabet[rng.integers(0, alphabet.size, n)].tobytes())
    pats = [b"", b"%", b"%%", b"%%%", b"_", b"__", b"___", b"a", b"a%", b"%a", b"%a%", b"a%b", b"a_b", b"a\nb", b"a\rb",
            b"%\n%", b"%\r%", b"\n", b"%\n", b"\n%", b"a\n%", b"%\nb", b"_\n_", b"%_%", b"%__%", b"%\0%", b"a\0b",
            "%é%".encode(), "caf_".encode(), "caf__".encode(), "caf%".encode(), b"\xff%", b"A%", b"%sale", b"%sale%",
            b"sale", b"x" * 300, b"%x%x%", b"x%x%", b"%%%b", b"_" * 300, b"_" * 299 + b"%", b"%" + b"_" * 60,
            b"%ab%ab%", b"a%\n%b", b"%\n\n%"]
    pats += [b"%" + bytes([c]) + b"%" for c in META] + [META, b"%" + META]
    while len(pats) < 64:
        n = int(rng.integers(1, 12))
        p = alphabet[rng.integers(0, alphabet.size, n)].tobytes()
        if p.count(b"%") <= 2:  # std::regex_match backtracks O(n^k) over k '.*' on a failing subject
            pats.append(p)
    return subj, pats


SEARCH_FILTERS = [
    "title LIKE '%a%'",
    "title LIKE 'a_b%' AND a < 50",
    "NOT (title LIKE '%b') OR a >= 90",
    "(title LIKE '%a%') AND (NOT (tag LIKE 'x%'))",
    "(NOT (tag LIKE '%y_') AND title LIKE '%ab%') OR title LIKE tag",
    "title LIKE '' OR (tag LIKE '%' AND a < 10)",
    "title LIKE '%.%' OR title LIKE '_x_%'",
    "'ab' LIKE title OR a < 5",
]
SEARCH_SEED, N_ROWS, N_INDEXED, DIM, NQ, LIMIT, GRAPH_L = 31, 3000, 2500, 16, 20, 10, 64


def search_table():
    """The seeded table of the search cases (also redrawn by tests/test_gpu_like.py)."""
    import graph_model as gm
    rng = np.random.default_rng(SEARCH_SEED)
    X = gm.int_table(N_ROWS, DIM, SEARCH_SEED)
    Q = gm.int_table(NQ, DIM, SEARCH_SEED + 1)
    a = rng.integers(0, 100, N_ROWS).astype(np.int32)
    pick = lambda alpha, hi: ["".join(alpha[j] for j in rng.integers(0, len(alpha), int(rng.integers(0, hi))))
                              for _ in range(N_ROWS)]
    title = pick("aab_%.\\\nxy", 9)
    tag = pick("xyz_%\n", 5)
    off, nb = gm.random_csr(N_INDEXED, 4, 24, SEARCH_SEED + 2)
    return X, Q, a, title, tag, off, nb


def search_cases():
    from oracle.oracle import Ref
    X, Q, a, title, tag, off, nb = search_table()
    ref = Ref("l2", DIM, N_ROWS, attr_cols=[("a", "int4"), ("title", "string"), ("tag", "string")])
    ref.set_rows(X)
    ref.set_attr_column("a", a)
    ref.set_string_column("title", title)
    ref.set_string_column("tag", tag)
    out = {"search_attrs": ref.attrs[:N_ROWS * ref.stride].copy(), "search_stride": np.int64(ref.stride),
           "search_offsets": off, "search_nbrs": nb}
    for col, vals in (("title", title), ("tag", tag)):
        o, b = pack([v.encode() for v in vals])
        out["search_%s_off" % col], out["search_%s_bytes" % col] = o, b
    buf = np.zeros(64 * 8, np.int64)
    for i, f in enumerate(SEARCH_FILTERS):
        n = ref.L.ref_filter_nodes(ref.h, f.encode(), buf.ctypes.data, 64)
        assert n > 0, f
        out["search_nodes_%d" % i] = buf[:n * 8].reshape(n, 8).copy()
        lo, lb = pack([t.encode() for t in re.findall(r"'([^']*)'", f)])
        out["search_lits_%d_off" % i], out["search_lits_%d_bytes" % i] = lo, lb
    branches = (("brute", False, None, 500), ("prefilter", True, None, 500), ("graph", False, (off, nb), GRAPH_L))
    for name, pre, graph, L in branches:
        if graph is not None:
            ref.set_graph(N_INDEXED, graph[0], graph[1], 3)
        ref.make_executors(1, T=1, L=L, prefilter=pre)
        for i, f in enumerate(SEARCH_FILTERS):
            ids, ds, cnt = ref.search_batch(Q, LIMIT, f)
            key = "search_%s_%d" % (name, i)
            out[key + "_ids"], out[key + "_dists"], out[key + "_counts"] = ids.astype(np.int32), ds.astype(np.float32), cnt
    out["search_table_crc32"] = np.int64(zlib.crc32(X.tobytes() + Q.tobytes() + a.tobytes()))
    return out


def main():
    L = load_driver()
    subj, pats = cases()
    so, sb = pack(subj)
    po, pb = pack(pats)
    out = np.zeros((len(subj), len(pats)), np.uint8)
    L.like_matrix(len(subj), so.ctypes.data, sb.ctypes.data if sb.size else None, len(pats), po.ctypes.data,
                  pb.ctypes.data, out.ctypes.data)
    searches = search_cases()
    np.savez_compressed(os.path.join(HERE, "like.npz"), subj_off=so, subj_bytes=sb, pat_off=po, pat_bytes=pb, match=out,
                        **searches)
    print("wrote like.npz: %d subjects x %d patterns, %d matches; %d search filters" % (
        len(subj), len(pats), int(out.sum()), len(SEARCH_FILTERS)))
    for name in ("brute", "prefilter", "graph"):
        print(name, [int(searches["search_%s_%d_counts" % (name, i)].sum()) for i in range(len(SEARCH_FILTERS))])


if __name__ == "__main__":
    main()
