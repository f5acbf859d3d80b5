"""The sparse L2 screen against the exact scan it screens, on the seeded SPLADE-like table of sparse_check.py.

Two L2 indexes hold the same 1M rows, one with the L2 screen (SparseIndex.build_l2_screen) and one without.  Measured,
alternating the two in one process: queries/s at batch 1024 (warm-up, then --steps timed calls each) and the latency of
one query (median of --single calls each), from the host clock around calls that end in a stream synchronise and from
the library's CUDA events (eps_stats.total_ms); the share of (query, row) pairs the screen re-scored through the merge.
The outputs of the two must be bitwise equal (ids, distances, counts) at every step.  With --build, the L2 graph build
with and without the screen at --build-rows (default 200k and 500k rows), whose graphs must be identical.  Prints one
JSON line per measurement with the card's name and power limit, read in the same run.

    python tools/sparse_l2_screen_check.py [--rows N] [--batch B] [--steps K] [--warmup W] [--single S]
                                           [--build] [--build-rows 200000,500000] [--out-degree D]
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


def search(a, vdb, rows, name, power):
    qs = splade_like(a.batch, 30, 40, 2)
    plain = vdb.SparseIndex("l2", VOCAB, capacity=a.rows)
    scr = vdb.SparseIndex("l2", VOCAB, capacity=a.rows)
    for ix in (plain, scr):
        ix.append(rows)
        ix.config(500, 500, force_brute=True)
    t = time.perf_counter()
    scr.build_l2_screen()
    build_s = time.perf_counter() - t
    res = {"scan": {"wall": [], "dev": [], "one_wall": [], "one_dev": []}}
    res["screen"] = {k: [] for k in res["scan"]}
    pair = (("scan", plain), ("screen", scr))
    for _ in range(a.warmup):
        for _, ix in pair:
            ix.search(qs, a.k)
    r0 = scr.l2_screen_info()["rescored"]
    for step in range(a.steps):
        outs = {}
        for key, ix in pair:
            outs[key], w = timed(ix, qs, a.k)
            res[key]["wall"].append(w)
            res[key]["dev"].append(outs[key][3]["total_ms"])
        assert_equal(outs["screen"], outs["scan"], "batch %d, step %d" % (a.batch, step))
    rescored_batch = (scr.l2_screen_info()["rescored"] - r0) / (a.steps * a.batch * a.rows)
    r0 = scr.l2_screen_info()["rescored"]
    for i in range(a.single + a.warmup):
        q = i % a.batch
        one = (np.array([0, qs[0][q + 1] - qs[0][q]]), qs[1][qs[0][q]:qs[0][q + 1]], qs[2][qs[0][q]:qs[0][q + 1]])
        outs = {}
        for key, ix in pair:
            outs[key], w = timed(ix, one, a.k)
            if i >= a.warmup:
                res[key]["one_wall"].append(w)
                res[key]["one_dev"].append(outs[key][3]["total_ms"])
        assert_equal(outs["screen"], outs["scan"], "single query %d" % q)
    rescored_single = (scr.l2_screen_info()["rescored"] - r0) / ((a.single + a.warmup) * a.rows)
    med = {key: {k: float(np.median(v)) for k, v in r.items()} for key, r in res.items()}
    info = scr.inverted_info()
    out = {
        "what": "search", "card": name, "power_limit": power, "metric": "l2", "rows": a.rows, "batch": a.batch,
        "k": a.k, "steps": a.steps, "warmup": a.warmup, "single_calls": a.single,
        "nnz_per_row": int(rows[0][-1]) / a.rows, "nnz_per_query": int(qs[0][-1]) / a.batch,
        "outputs_bitwise_equal": True, "build_s": build_s, "postings": info["postings"], "terms": info["terms"],
        "rescored_fraction_batch": rescored_batch, "rescored_fraction_single": rescored_single,
        "rescored_per_query_batch": rescored_batch * a.rows, "rescored_per_query_single": rescored_single * a.rows,
    }
    for key in ("scan", "screen"):
        m = med[key]
        out[key] = {"qps": a.batch / m["wall"], "batch_ms_median": m["wall"] * 1e3, "batch_device_ms_median": m["dev"],
                    "single_query_ms_median": m["one_wall"] * 1e3, "single_query_device_ms_median": m["one_dev"]}
    out["speedup_batch"] = med["scan"]["wall"] / med["screen"]["wall"]
    out["speedup_single_query"] = med["scan"]["one_wall"] / med["screen"]["one_wall"]
    print(json.dumps(out), flush=True)
    plain.close()
    scr.close()


def build(a, vdb, rows_all, name, power):
    for n in [int(x) for x in a.build_rows.split(",")]:
        rows = (rows_all[0][:n + 1], rows_all[1][:rows_all[0][n]], rows_all[2][:rows_all[0][n]])
        ix = vdb.SparseIndex("l2", VOCAB, capacity=n)
        ix.append(rows)
        t = time.perf_counter()
        ix.build(n, out_degree=a.out_degree)
        merge_s = time.perf_counter() - t
        want = ix.get_graph()
        ix.build_l2_screen()
        r0 = ix.l2_screen_info()["rescored"]
        t = time.perf_counter()
        ix.build(n, out_degree=a.out_degree)
        screen_s = time.perf_counter() - t
        got = ix.get_graph()
        for what, x, y in zip(("n_indexed", "offsets", "neighbours", "nav"), got, want):
            assert np.array_equal(x, y), "build of %d rows: %s differ" % (n, what)
        rescored = ix.l2_screen_info()["rescored"] - r0
        print(json.dumps({"what": "build", "card": name, "power_limit": power, "metric": "l2", "rows": n,
                          "out_degree": a.out_degree, "graphs_identical": True, "merge_build_s": merge_s,
                          "screen_build_s": screen_s, "speedup": merge_s / screen_s,
                          "rescored_fraction": rescored / float(n) / n}), flush=True)
        ix.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--single", type=int, default=200)
    ap.add_argument("--build", action="store_true", help="also the L2 graph build with and without the screen")
    ap.add_argument("--build-only", action="store_true", help="only the graph builds")
    ap.add_argument("--build-rows", default="200000,500000")
    ap.add_argument("--out-degree", type=int, default=50)
    a = ap.parse_args()
    import vectordb_b200
    if vectordb_b200.load_library().eps_device_count() <= 0:
        sys.exit("sparse_l2_screen_check: no CUDA device: nothing is measured without the GPU")
    n_rows = max([a.rows] + ([int(x) for x in a.build_rows.split(",")] if a.build or a.build_only else []))
    rows = splade_like(n_rows, 100, 140, 1)
    name, power = card()
    if not a.build_only:
        a.rows = min(a.rows, n_rows)
        search(a, vectordb_b200, (rows[0][:a.rows + 1], rows[1][:rows[0][a.rows]], rows[2][:rows[0][a.rows]]), name, power)
    if a.build or a.build_only:
        build(a, vectordb_b200, rows, name, power)


if __name__ == "__main__":
    main()
