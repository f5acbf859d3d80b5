"""Extending a sparse index's posting lists over appended rows against rebuilding them, on the seeded SPLADE-like table
of sparse_check.py (eps_index_extend_sparse_postings).

For each metric (IP: the inverted index, L2: the L2 screen) one index holds the --rows rows, and for each tail m of
--tails the lists cover the first rows - m.  Every round restores that starting state with a build over rows - m, times
the extension over the m rows, restores the start again and times the full rebuild over every row.  Measured:
  * the call's time, from the host clock around the call (both calls synchronise the index's stream);
  * the device memory the call keeps (net), from its formula and from cudaMemGetInfo before and after the call, and
    the memory it holds while it runs (peak, from the formula, without cub's scratch);
  * queries/s at batch --batch and the latency of one query (median of --single calls), with the m rows merged as the
    lists' tail and after the extension, from the host clock around calls that end in a stream synchronise.
The extended and the rebuilt lists must be byte-equal, and every search output (ids, distances, counts; for L2 the count
of re-scored pairs) equal with the tail merged, after the extension and after the rebuild.  Prints one JSON line per
(metric, tail) with the card's name and power limit, read in the same run.

    python tools/sparse_extend_check.py [--rows N] [--tails 10000,100000,500000] [--metrics ip,l2] [--rounds R]
                                        [--batch B] [--steps K] [--warmup W] [--single S]
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
from sparse_inverted_check import assert_equal, timed  # noqa: E402

MIB = 1 << 20


def free_bytes():
    import torch
    return torch.cuda.mem_get_info(0)[0]


def lists_bytes(t, p):
    """Device bytes of lists with t terms and p postings, as the index holds them (the build keeps p + 1 postings)."""
    return max(t, 1) * 4 + (t + 1) * 8 + p * 8


def build(ix, metric, n):
    (ix.build_l2_screen if metric == "l2" else ix.build_inverted)(n)


def call(fn):
    f0 = free_bytes()
    t = time.perf_counter()
    fn()
    s = time.perf_counter() - t
    return s, f0 - free_bytes()


def measure_search(ix, metric, qs, a):
    """Median batch and single-query wall times, the outputs of every call, and the pairs re-scored (L2)."""
    r0 = ix.l2_screen_info()["rescored"] if metric == "l2" else 0
    for _ in range(a.warmup):
        ix.search(qs, a.k)
    outs, wall = [], []
    for _ in range(a.steps):
        o, w = timed(ix, qs, a.k)
        outs.append(o)
        wall.append(w)
    one_wall = []
    for i in range(a.single):
        q = i % a.batch
        one = (np.array([0, qs[0][q + 1] - qs[0][q]]), qs[1][qs[0][q]:qs[0][q + 1]], qs[2][qs[0][q]:qs[0][q + 1]])
        o, w = timed(ix, one, a.k)
        outs.append(o)
        one_wall.append(w)
    rescored = ix.l2_screen_info()["rescored"] - r0 if metric == "l2" else 0
    return float(np.median(wall)), float(np.median(one_wall)), outs, rescored


def same_lists(x, y, what):
    assert x["rows"] == y["rows"], what + ": rows covered"
    for key in ("terms", "ptr", "post_rows", "post_values"):
        assert x[key].tobytes() == y[key].tobytes(), "%s: %s differ" % (what, key)


def run_case(a, ix, metric, m, qs, name, power):
    n, n0 = a.rows, a.rows - m
    build(ix, metric, n0)
    info0 = ix.inverted_info()
    tail_batch, tail_one, tail_outs, tail_rescored = measure_search(ix, metric, qs, a)
    ext_s, reb_s, ext_net, reb_net, ext_after, reb_after = [], [], [], [], None, None
    for rnd in range(a.rounds):
        build(ix, metric, n0)
        s, d = call(lambda: ix.extend_postings(n))
        ext_s.append(s)
        ext_net.append(d)
        ext_lists = ix.postings()
        info1 = ix.inverted_info()
        if rnd == 0:
            ext_after = measure_search(ix, metric, qs, a)
        build(ix, metric, n0)
        s, d = call(lambda: build(ix, metric, n))
        reb_s.append(s)
        reb_net.append(d)
        same_lists(ext_lists, ix.postings(), "%s, tail %d, round %d: extended vs rebuilt" % (metric, m, rnd))
        del ext_lists
        if rnd == 0:
            reb_after = measure_search(ix, metric, qs, a)
    for what, got in (("after the extension", ext_after), ("after the rebuild", reb_after)):
        for i, (x, y) in enumerate(zip(got[2], tail_outs)):
            assert_equal(x, y, "%s, tail %d, call %d: %s vs tail merged" % (metric, m, i, what))
    if metric == "l2":
        assert ext_after[3] == reb_after[3], "%s, tail %d: re-scored pairs differ" % (metric, m)
    t0, p0, t1, p1 = info0["terms"], info0["postings"], info1["terms"], info1["postings"]
    p_new, t_new = p1 - p0, int(np.unique(a.table[1][a.table[0][n0]:a.table[0][n]]).size)
    out = {
        "card": name, "power_limit": power, "metric": metric, "rows": n, "tail_rows": m, "rounds": a.rounds,
        "batch": a.batch, "k": a.k, "steps": a.steps, "warmup": a.warmup, "single_calls": a.single,
        "postings_before": p0, "postings_after": p1, "terms_before": t0, "terms_after": t1, "new_postings": p_new,
        "lists_and_outputs_bitwise_equal": True,
        "extend_s": ext_s, "rebuild_s": reb_s, "extend_s_median": float(np.median(ext_s)),
        "rebuild_s_median": float(np.median(reb_s)),
        "speedup_call": float(np.median(reb_s) / np.median(ext_s)),
        # the lists grow by the same bytes either way; cudaMalloc rounds each of the 3 arrays freed and 3 made to 2 MiB
        "net_bytes_formula": lists_bytes(t1, p1) - lists_bytes(t0, p0 + 1),
        "net_bytes_measured_extend": ext_net, "net_bytes_measured_rebuild": reb_net,
        "extend_peak_bytes_formula": max(24 * p_new + 16 + 12 * t_new + 8,
                                         8 * (p_new + 1) + 28 * t_new + 16 + 8 * t0 + lists_bytes(t1, p1)),
        "rebuild_peak_bytes_formula": 24 * p1 + 16 + 12 * t1 + 8,
        "qps_tail_merged": a.batch / tail_batch, "qps_extended": a.batch / ext_after[0],
        "qps_rebuilt": a.batch / reb_after[0],
        "batch_ms_tail_merged": tail_batch * 1e3, "batch_ms_extended": ext_after[0] * 1e3,
        "single_query_ms_tail_merged": tail_one * 1e3, "single_query_ms_extended": ext_after[1] * 1e3,
        "single_query_ms_rebuilt": reb_after[1] * 1e3,
    }
    if metric == "l2":
        out["rescored_tail_merged"], out["rescored_extended"] = tail_rescored, ext_after[3]
    out["net_bytes_within_alloc_rounding"] = all(abs(d - out["net_bytes_formula"]) <= 8 * MIB for d in ext_net)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--tails", default="10000,100000,500000")
    ap.add_argument("--metrics", default="ip,l2")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--single", type=int, default=50)
    a = ap.parse_args()
    import vectordb_b200
    if vectordb_b200.load_library().eps_device_count() <= 0:
        sys.exit("sparse_extend_check: no CUDA device: nothing is measured without the GPU")
    a.table = splade_like(a.rows, 100, 140, 1)
    qs = splade_like(a.batch, 30, 40, 2)
    name, power = card()
    for metric in a.metrics.split(","):
        ix = vectordb_b200.SparseIndex(metric, VOCAB, capacity=a.rows)
        ix.append(a.table)
        ix.config(500, 500, force_brute=True)
        for m in [int(x) for x in a.tails.split(",")]:
            run_case(a, ix, metric, m, qs, name, power)
        ix.close()


if __name__ == "__main__":
    main()
