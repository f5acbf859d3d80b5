"""Sparse graph search against the sparse exact scan on the SPLADE-like table of tools/sparse_check.py.

In one process: reads the card's name and power limit, builds the graph (eps_index_build on the sparse index) and
times it, runs the exact scan (EPS_SPARSE_SEARCH_SCAN) as ground truth, then sweeps the queue length L in graph mode
(EPS_SPARSE_SEARCH_GRAPH) at batch 1024, k = 10, inner product.  Per L it reports recall@k against the exact scan,
queries/s (end to end and over the graph kernel time, CUDA events), n_dist per query, and the latency of one query per
call.  Prints one JSON line per measurement.

    python tools/sparse_graph_check.py [--rows N] [--batch B] [--L 16,32,...] [--steps K] [--warmup W] [--metric ip]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from sparse_check import VOCAB, card, splade_like  # noqa: E402


def timed(ix, qs, k, steps, warmup):
    for _ in range(warmup):
        ix.search(qs, k)
    wall, kern = [], []
    for _ in range(steps):
        t = time.perf_counter()
        res = ix.search(qs, k)
        wall.append(time.perf_counter() - t)
        kern.append(res[3]["kernel_ms"])
    return res, float(np.median(wall)), float(np.median(kern))


def recall(got, truth, k):
    hit = sum(len(set(g[:k].tolist()) & set(t[:k].tolist())) for g, t in zip(got, truth))
    return hit / float(k * truth.shape[0])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--L", default="16,32,64,128,256,512")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--metric", default="ip")
    ap.add_argument("--out-degree", type=int, default=50)
    a = ap.parse_args()
    import vectordb_b200
    if vectordb_b200.load_library().eps_device_count() <= 0:
        sys.exit("sparse_graph_check: no CUDA device: nothing is measured without the GPU")
    name, power = card()
    head = {"card": name, "power_limit": power, "rows": a.rows, "batch": a.batch, "k": a.k, "metric": a.metric}
    rows = splade_like(a.rows, 100, 140, 1)
    qs = splade_like(a.batch, 30, 40, 2)
    one = (qs[0][:2], qs[1][:qs[0][1]], qs[2][:qs[0][1]])
    ix = vectordb_b200.SparseIndex(a.metric, VOCAB, capacity=a.rows)
    ix.append(rows)
    t = time.perf_counter()
    ix.build(a.rows, out_degree=a.out_degree)
    build_s = time.perf_counter() - t
    n_indexed, off, _, nav = ix.get_graph()
    print(json.dumps(dict(head, what="build", build_s=build_s, out_degree=a.out_degree, n_indexed=n_indexed,
                          edges_per_row=float(off[-1]) / n_indexed, nav_row_length=int(off[nav + 1] - off[nav]))))

    ix.set_search_mode("scan")
    ix.config(500, 500)
    truth, wall, kern = timed(ix, qs, a.k, a.steps, a.warmup)
    _, one_wall, one_kern = timed(ix, one, a.k, a.steps, a.warmup)
    print(json.dumps(dict(head, what="exact scan", qps_end_to_end=a.batch / wall, kernel_ms_median=kern,
                          qps_kernel=a.batch / (kern / 1e3), n_dist_per_query=truth[3]["n_dist"] / a.batch,
                          single_query_ms=one_wall * 1e3, single_query_kernel_ms=one_kern)))

    ix.set_search_mode("graph")
    for L in [int(x) for x in a.L.split(",")]:
        ix.config(L, L)
        res, wall, kern = timed(ix, qs, a.k, a.steps, a.warmup)
        _, one_wall, one_kern = timed(ix, one, a.k, a.steps, a.warmup)
        st = res[3]
        print(json.dumps(dict(head, what="graph", L=L, recall_at_k=recall(res[0], truth[0], a.k),
                              qps_end_to_end=a.batch / wall, kernel_ms_median=kern, qps_kernel=a.batch / (kern / 1e3),
                              n_dist_per_query=st["n_dist"] / a.batch, n_expand_per_query=st["n_expand"] / a.batch,
                              single_query_ms=one_wall * 1e3, single_query_kernel_ms=one_kern)))
    ix.close()


if __name__ == "__main__":
    main()
