"""Writes tests/golden/sparse_graph.npz: the reference's own sparse graph build and graph-branch Search answers.

    python tests/golden/make_sparse_graph_golden.py

Needs what make_sparse_golden.py needs (oracle/_ref/libepsilla_ref.so and the reference checkout's headers); nothing at
test time does.  Its driver is extended by three calls: ANNGraphSegment::BuildFromVectorTable on the sparse column
(one OpenMP thread), setting the segment's record_number_ (rows visible to Search), and Search at IntraQueryThreads = 1
with a queue length L and a counting wrapper around the SparseVecDistFunc.

For each metric, on the rows of make_sparse_golden.table(metric): the graph over the first 2 000 rows (CSR and
navigation point), and ids, distances, counts and per-query distance calls for L in {64, 200} with and without the
1 000-row tail, L_local < limit, deleted rows, and numeric, @distance and string filters.  The cosine cases drop the
empty query: it is NaN against every row, and the reference's order is then unspecified.
"""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from make_sparse_golden import DRIVER, THR, crc, table  # noqa: E402

GRAPH_DRIVER = r'''
extern "C" {
void sp_set_rows(void* h, int64_t n) { static_cast<Ctx*>(h)->seg->record_number_ = n; }
// ANNGraphSegment::BuildFromVectorTable over rows [0, n) of the sparse column, one thread
int sp_build(void* h, int64_t n) {
  auto* c = static_cast<Ctx*>(h);
  omp_set_num_threads(1);
  const size_t vo = c->seg->field_name_mem_offset_map_["Vec"];
  c->ann = std::make_shared<ANNGraphSegment>(true);
  try {
    c->ann->BuildFromVectorTable(&c->seg->var_len_attr_table_[vo], n, c->dim, c->metric);
  } catch (...) {
    return -1;
  }
  return 0;
}
int64_t sp_graph(void* h, int64_t* offsets, int64_t* nbrs, int64_t* nav) {
  auto* c = static_cast<Ctx*>(h);
  const int64_t n = c->ann->record_number_;
  if (offsets) std::memcpy(offsets, c->ann->offset_table_, (n + 1) * 8);
  if (nbrs) std::memcpy(nbrs, c->ann->neighbor_list_, c->ann->offset_table_[n] * 8);
  if (nav) *nav = c->ann->navigation_point_;
  return nbrs ? n : c->ann->offset_table_[n];
}
// Search of nq queries at T = 1 with L_master = L_local = L; calls[q] = SparseVecDistFunc calls of query q
int sp_search_counted(void* h, int64_t L, int64_t nq, const int64_t* off, const int64_t* idx, const float* val,
                      int64_t limit, const char* filter, int64_t* ids, double* dists, int64_t* counts, int64_t* calls) {
  auto* c = static_cast<Ctx*>(h);
  omp_set_num_threads(1);
  const size_t vo = c->seg->field_name_mem_offset_map_["Vec"];
  SparseVecDistFunc inner = std::get<SparseVecDistFunc>(GetDistFunc(meta::FieldType::SPARSE_VECTOR_FLOAT, c->metric));
  int64_t n_calls = 0;
  SparseVecDistFunc counting = [&inner, &n_calls](const SparseVector& a, const SparseVector& b) {
    ++n_calls;
    return inner(a, b);
  };
  execution::VecSearchExecutor ex(c->dim, c->ann->navigation_point_, c->ann, c->ann->offset_table_, c->ann->neighbor_list_,
                                  &c->seg->var_len_attr_table_[vo], DistFunc(counting), nullptr, 1, L, L, 1, false);
  for (int64_t q = 0; q < nq; ++q) {
    std::vector<query::expr::ExprNodePtr> nodes;
    if (filter && filter[0] && !query::expr::Expr::ParseNodeFromStr(filter, nodes, c->field_map).ok()) return -1;
    int64_t rs = 0;
    VectorPtr qv = make_vec(off, idx, val, q);
    n_calls = 0;
    if (!ex.Search(qv, c->seg.get(), static_cast<size_t>(limit), nodes, rs).ok()) return -2;
    calls[q] = n_calls;
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

N_GRAPH = 2000
# every case: (name, L, limit, rows visible to Search, filter string, deleted rows applied)
CASES = [("L64", 64, 10, N_GRAPH, "", False), ("L200", 200, 10, N_GRAPH, "", False),
         ("L64_tail", 64, 10, None, "", False), ("L200_tail", 200, 10, None, "", False),
         ("Llocal", 16, 50, None, "", False), ("deleted", 64, 10, None, "", True),
         ("numeric", 64, 10, None, "a < 30", True), ("distance", 64, 10, None, "@distance < {thr}", True),
         ("string", 200, 50, None, "s <> 'v3'", True)]


def load_driver():
    from oracle.oracle import reference_dir
    ref = reference_dir()
    so = os.path.join(ROOT, "oracle", "_ref", "libepsilla_ref.so")
    if not ref or not os.path.exists(so):
        sys.exit("make_sparse_graph_golden: needs a reference checkout and oracle/_ref/libepsilla_ref.so (run build())")
    tmp = tempfile.mkdtemp(prefix="sparse_graph_ref_")
    src, out = os.path.join(tmp, "sparse_graph_driver.cpp"), os.path.join(tmp, "libsparse_graph_driver.so")
    open(src, "w").write(DRIVER + GRAPH_DRIVER)
    subprocess.check_call(["/usr/bin/g++", "-std=c++17", "-O3", "-DNDEBUG", "-fopenmp", "-fPIC", "-w", "-shared",
                           "-I", os.path.join(ROOT, "oracle", "shim"), "-I", os.path.join(ref, "engine"), src, "-o", out,
                           so, "-Wl,-rpath," + os.path.dirname(so)])
    L = C.CDLL(out)
    vp, i64 = C.c_void_p, C.c_int64
    L.sp_create.restype = vp
    L.sp_create.argtypes = [C.c_int, i64, i64, vp, vp, vp, vp, vp]
    L.sp_destroy.argtypes = [vp]
    L.sp_set_deleted.argtypes = [vp, i64]
    L.sp_set_rows.argtypes = [vp, i64]
    L.sp_build.argtypes = [vp, i64]
    L.sp_graph.restype = i64
    L.sp_graph.argtypes = [vp, vp, vp, vp]
    L.sp_search_counted.argtypes = [vp, i64, i64, vp, vp, vp, i64, C.c_char_p, vp, vp, vp, vp]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def drop_empty_query(qs):
    off, idx, val = qs
    assert off[-1] == off[-2]
    return off[:-1].copy(), idx, val


def main():
    L = load_driver()
    out = {}
    for metric in (1, 2, 3):
        n, vocab, rows, qs, attr, codes, dead = table(metric)
        out["m%d_table_crc32" % metric] = np.int64(crc(*rows, *qs))
        if metric == 2:
            qs = drop_empty_query(qs)
        h = L.sp_create(metric, vocab, n, _p(rows[0]), _p(rows[1]), _p(rows[2]), _p(attr), _p(codes))
        assert L.sp_build(h, N_GRAPH) == 0
        e = L.sp_graph(h, None, None, None)
        off, nb, nav = np.zeros(N_GRAPH + 1, np.int64), np.zeros(e, np.int64), C.c_int64()
        assert L.sp_graph(h, _p(off), _p(nb), C.byref(nav)) == N_GRAPH
        out["m%d_graph_offsets" % metric] = off
        out["m%d_graph_nbrs" % metric] = nb.astype(np.int32)
        out["m%d_graph_nav" % metric] = np.int64(nav.value)
        deleted_on = False
        nq = qs[0].size - 1
        for name, Lq, limit, visible, filt, use_del in CASES:
            if use_del and not deleted_on:
                for d in dead:
                    L.sp_set_deleted(h, int(d))
                deleted_on = True
            L.sp_set_rows(h, n if visible is None else visible)
            ids = np.empty((nq, limit), np.int64)
            ds = np.empty((nq, limit), np.float64)
            cnt = np.empty(nq, np.int64)
            calls = np.empty(nq, np.int64)
            rc = L.sp_search_counted(h, Lq, nq, _p(qs[0]), _p(qs[1]), _p(qs[2]), limit,
                                     filt.format(thr=THR[metric]).encode(), _p(ids), _p(ds), _p(cnt), _p(calls))
            assert rc == 0, (rc, name)
            key = "m%d_%s" % (metric, name)
            out[key + "_ids"] = ids.astype(np.int32)
            out[key + "_dists"] = ds.astype(np.float32)
            out[key + "_counts"] = cnt.astype(np.int32)
            out[key + "_calls"] = calls.astype(np.int32)
        L.sp_destroy(h)
    np.savez_compressed(os.path.join(HERE, "sparse_graph.npz"), **out)
    print("wrote sparse_graph.npz (%d arrays)" % len(out))


if __name__ == "__main__":
    main()
