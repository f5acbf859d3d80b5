"""Writes tests/golden/sparse.npz: the reference's own VecSearchExecutor::Search answers on a seeded sparse table.

    python tests/golden/make_sparse_golden.py [--time-bruteforce]

Needs oracle/_ref/libepsilla_ref.so (built by __graft_entry__.build() from a reference checkout) and that checkout's
headers ($EPSILLA_REFERENCE or oracle.reference_dir()).  The small driver below is test infrastructure: it only builds
the reference's objects (a TableSegmentMVP with INT4 'a', STRING 's' and SPARSE_VECTOR_FLOAT 'Vec' fields, an empty
ANNGraphSegment, a VecSearchExecutor over the sparse column with GetDistFunc's sparse function) and forwards Search
calls, so the stored ids and distances are the reference's BruteForceSearch / PreFilterBruteForceSearch output.

The table and queries are redrawn by tests/test_gpu_sparse.py (sparse_rows, seeds 11 / 12); the file keeps their
CRC.  --time-bruteforce also times the reference's Search (one thread) per query on a 100k-row SPLADE-like subsample
of tools/sparse_check.py's table, on the host.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

DRIVER = r'''
#include <omp.h>
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <vector>
#include "db/ann_graph_segment.hpp"
#include "db/execution/vec_search_executor.hpp"
#include "db/index/index.hpp"
#include "db/table_segment_mvp.hpp"
#include "db/vector.hpp"
#include "query/expr/expr.hpp"
using namespace vectordb;
using namespace vectordb::engine;
struct Ctx {
  meta::TableSchema schema;
  std::unique_ptr<TableSegmentMVP> seg;
  std::shared_ptr<ANNGraphSegment> ann;
  std::unordered_map<std::string, meta::FieldType> field_map;
  meta::MetricType metric;
  int64_t dim;
};
static SparseVectorPtr make_vec(const int64_t* off, const int64_t* idx, const float* val, int64_t r) {
  auto v = std::make_shared<SparseVector>();
  for (int64_t i = off[r]; i < off[r + 1]; ++i) v->push_back(SparseVectorElement{static_cast<size_t>(idx[i]), val[i]});
  return v;
}
extern "C" {
void* sp_create(int metric, int64_t dim, int64_t n, const int64_t* off, const int64_t* idx, const float* val,
                const int32_t* a, const int32_t* s) {
  auto* c = new Ctx();
  c->metric = static_cast<meta::MetricType>(metric);
  c->dim = dim;
  c->schema.id_ = 0;
  c->schema.name_ = "t";
  const char* names[3] = {"a", "s", "Vec"};
  meta::FieldType types[3] = {meta::FieldType::INT4, meta::FieldType::STRING, meta::FieldType::SPARSE_VECTOR_FLOAT};
  for (int i = 0; i < 3; ++i) {
    meta::FieldSchema f;
    f.id_ = i;
    f.name_ = names[i];
    f.field_type_ = types[i];
    f.is_primary_key_ = false;
    if (i == 2) { f.vector_dimension_ = dim; f.metric_type_ = c->metric; }
    c->schema.fields_.push_back(f);
    if (i < 2) c->field_map[f.name_] = f.field_type_;
  }
  c->field_map["@distance"] = meta::FieldType::DOUBLE;
  c->seg.reset(new TableSegmentMVP(c->schema, n, nullptr));
  const size_t ao = c->seg->field_name_mem_offset_map_["a"], so = c->seg->field_name_mem_offset_map_["s"],
               vo = c->seg->field_name_mem_offset_map_["Vec"];
  for (int64_t r = 0; r < n; ++r) {
    std::memcpy(c->seg->attribute_table_ + r * c->seg->primitive_offset_ + ao, &a[r], 4);
    c->seg->var_len_attr_table_[so][r] = std::string("v") + std::to_string(s[r]);
    c->seg->var_len_attr_table_[vo][r] = make_vec(off, idx, val, r);
  }
  c->seg->record_number_ = n;
  c->ann = std::make_shared<ANNGraphSegment>(true);
  return c;
}
void sp_destroy(void* h) { delete static_cast<Ctx*>(h); }
void sp_set_deleted(void* h, int64_t id) { static_cast<Ctx*>(h)->seg->deleted_->set(id); }
// Search of nq queries, one executor (T = 1): ids / dists [nq x limit], counts [nq]; -1 when the filter does not parse
int sp_search(void* h, int prefilter, int64_t L_local, int64_t nq, const int64_t* off, const int64_t* idx,
              const float* val, int64_t limit, const char* filter, int64_t* ids, double* dists, int64_t* counts) {
  auto* c = static_cast<Ctx*>(h);
  omp_set_num_threads(1);
  const size_t vo = c->seg->field_name_mem_offset_map_["Vec"];
  execution::VecSearchExecutor ex(c->dim, c->ann->navigation_point_, c->ann, c->ann->offset_table_, c->ann->neighbor_list_,
                                  &c->seg->var_len_attr_table_[vo], GetDistFunc(meta::FieldType::SPARSE_VECTOR_FLOAT, c->metric),
                                  nullptr, 1, 500, L_local, 1, prefilter != 0);
  for (int64_t q = 0; q < nq; ++q) {
    std::vector<query::expr::ExprNodePtr> nodes;
    if (filter && filter[0] && !query::expr::Expr::ParseNodeFromStr(filter, nodes, c->field_map).ok()) return -1;
    int64_t rs = 0;
    VectorPtr qv = make_vec(off, idx, val, q);
    if (!ex.Search(qv, c->seg.get(), static_cast<size_t>(limit), nodes, rs).ok()) return -2;
    counts[q] = rs;
    for (int64_t i = 0; i < limit; ++i) {
      ids[q * limit + i] = i < rs ? ex.search_result_[i] : -1;
      dists[q * limit + i] = i < rs ? ex.distance_[i] : INFINITY;
    }
  }
  return 0;
}
}
'''


def load_driver():
    from oracle.oracle import reference_dir
    ref = reference_dir()
    so = os.path.join(ROOT, "oracle", "_ref", "libepsilla_ref.so")
    if not ref or not os.path.exists(so):
        sys.exit("make_sparse_golden: needs a reference checkout and oracle/_ref/libepsilla_ref.so (run build())")
    tmp = tempfile.mkdtemp(prefix="sparse_ref_")
    src, out = os.path.join(tmp, "sparse_driver.cpp"), os.path.join(tmp, "libsparse_driver.so")
    open(src, "w").write(DRIVER)
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-DNDEBUG", "-fopenmp", "-fPIC", "-w", "-shared",
                           "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ref, "engine"), src, "-o", out,
                           so, "-Wl,-rpath," + os.path.dirname(so)])
    L = C.CDLL(out)
    vp, i64 = C.c_void_p, C.c_int64
    L.sp_create.restype = vp
    L.sp_create.argtypes = [C.c_int, i64, i64, vp, vp, vp, vp, vp]
    L.sp_destroy.argtypes = [vp]
    L.sp_set_deleted.argtypes = [vp, i64]
    L.sp_search.argtypes = [vp, C.c_int, i64, i64, vp, vp, vp, i64, C.c_char_p, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def search(L, h, qs, limit, prefilter=False, L_local=500, filt=""):
    off, idx, val = qs
    nq = off.size - 1
    ids = np.empty((nq, limit), np.int64)
    ds = np.empty((nq, limit), np.float64)
    cnt = np.empty(nq, np.int64)
    rc = L.sp_search(h, int(prefilter), L_local, nq, _p(off), _p(idx), _p(val), limit, filt.encode(), _p(ids), _p(ds), _p(cnt))
    assert rc == 0, (rc, filt)
    return ids, ds, cnt


# every case: (name, prefilter, L_local, limit, filter string, deleted rows applied)
CASES = [("brute", False, 500, 10, "", False), ("brute_L7", False, 7, 10, "", False), ("deleted", False, 500, 10, "", True),
         ("numeric", False, 500, 10, "a < 30", True), ("distance", False, 500, 10, "@distance < {thr}", True),
         ("string", False, 500, 10, "s <> 'v3'", True), ("prefilter", True, 500, 50, "a < 10", True)]
THR = {1: 6.0, 2: 0.97, 3: -0.3}


def table(metric=1):
    """Seeded table of the golden cases.  Cosine uses the same draw without empty rows: an empty row is NaN against
    every query, and NaN breaks the strict weak ordering std::sort needs, so the reference's order of the whole list
    (numbers included) would be unspecified.  The device's NaN rule is tested against the restatement instead."""
    from test_gpu_sparse import sparse_rows
    n, vocab, nq = 3000, 2000, 24
    rows = sparse_rows(n, vocab, 11, empty_every=0 if metric == 2 else 97)
    qs = sparse_rows(nq, vocab, 12, max_nnz=40, empty_every=0, dup_every=0)
    qs = (np.concatenate([qs[0], [qs[0][-1]]]), qs[1], qs[2])  # + one empty query
    attr = (np.arange(n) * 7 % 100).astype(np.int32)
    codes = (np.arange(n) % 5).astype(np.int32)
    dead = np.arange(3, n, 41)
    return n, vocab, rows, qs, attr, codes, dead


def crc(*arrays):
    c = 0
    for a in arrays:
        c = zlib.crc32(np.ascontiguousarray(a).tobytes(), c)
    return c


def main():
    L = load_driver()
    out = {}
    for metric in (1, 2, 3):
        n, vocab, rows, qs, attr, codes, dead = table(metric)
        out["m%d_table_crc32" % metric] = np.int64(crc(*rows, *qs))
        h = L.sp_create(metric, vocab, n, _p(rows[0]), _p(rows[1]), _p(rows[2]), _p(attr), _p(codes))
        deleted_on = False
        for name, pre, ll, limit, filt, use_del in CASES:
            if use_del and not deleted_on:
                for d in dead:
                    L.sp_set_deleted(h, int(d))
                deleted_on = True
            ids, ds, cnt = search(L, h, qs, limit, pre, ll, filt.format(thr=THR[metric]))
            key = "m%d_%s" % (metric, name)
            out[key + "_ids"] = ids.astype(np.int32)
            out[key + "_dists"] = ds.astype(np.float32)
            out[key + "_counts"] = cnt.astype(np.int32)
        L.sp_destroy(h)
    np.savez_compressed(os.path.join(HERE, "sparse.npz"), **out)
    print("wrote sparse.npz (%d arrays)" % len(out))
    if "--time-bruteforce" in sys.argv:
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from sparse_check import splade_like
        m = 100_000
        rows = splade_like(m, 100, 140, 1)
        qs = splade_like(8, 30, 40, 2)
        z = np.zeros(m, np.int32)
        h = L.sp_create(3, 30522, m, _p(rows[0]), _p(rows[1]), _p(rows[2]), _p(z), _p(z))
        t = time.perf_counter()
        search(L, h, qs, 10)
        dt = (time.perf_counter() - t) / 8
        print("reference Search (brute-force branch, 1 thread, host CPU): %.1f ms per query on %d rows" % (dt * 1e3, m))
        L.sp_destroy(h)


if __name__ == "__main__":
    main()
