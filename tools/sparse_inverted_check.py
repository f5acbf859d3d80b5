"""The sparse inverted index against the exact scan it replaces, on the seeded SPLADE-like table of sparse_check.py.

For each metric (IP and cosine) two indexes hold the same 1M rows, one with posting lists (SparseIndex.build_inverted)
and one without.  Measured, alternating the two in one process: queries/s at batch 1024 (warm-up, then --steps timed
calls each) and the latency of one query (median of --single calls each), from the host clock around calls that end in
a stream synchronise and from the library's CUDA events (eps_stats.total_ms).  Also the build's time and the index's
device bytes.  The outputs of the two must be bitwise equal (ids, distances, counts).  Prints one JSON line per metric
with the card's name and power limit, read in the same run.

    python tools/sparse_inverted_check.py [--rows N] [--batch B] [--steps K] [--warmup W] [--single S] [--metrics ip,cosine]
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


def timed(ix, qs, k):
    t = time.perf_counter()
    out = ix.search(qs, k)
    return out, time.perf_counter() - t


def assert_equal(a, b, what):
    assert np.array_equal(a[2], b[2]), what + ": counts differ"
    assert np.array_equal(a[0], b[0]), what + ": ids differ"
    assert np.array_equal(a[1].view(np.uint64), b[1].view(np.uint64)), what + ": distances are not bitwise equal"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--single", type=int, default=200)
    ap.add_argument("--metrics", default="ip,cosine")
    a = ap.parse_args()
    import vectordb_b200
    L = vectordb_b200.load_library()
    if L.eps_device_count() <= 0:
        sys.exit("sparse_inverted_check: no CUDA device: nothing is measured without the GPU")
    rows = splade_like(a.rows, 100, 140, 1)
    qs = splade_like(a.batch, 30, 40, 2)
    name, power = card()
    for metric in a.metrics.split(","):
        scan = vectordb_b200.SparseIndex(metric, VOCAB, capacity=a.rows)
        inv = vectordb_b200.SparseIndex(metric, VOCAB, capacity=a.rows)
        for ix in (scan, inv):
            ix.append(rows)
            ix.config(500, 500, force_brute=True)
        t = time.perf_counter()
        inv.build_inverted()
        build_s = time.perf_counter() - t
        info = inv.inverted_info()
        res = {"scan": {"wall": [], "dev": [], "one_wall": [], "one_dev": []}}
        res["inverted"] = {k: [] for k in res["scan"]}
        pair = (("scan", scan), ("inverted", inv))
        for _ in range(a.warmup):
            for _, ix in pair:
                ix.search(qs, a.k)
        for step in range(a.steps):
            outs = {}
            for key, ix in pair:
                outs[key], w = timed(ix, qs, a.k)
                res[key]["wall"].append(w)
                res[key]["dev"].append(outs[key][3]["total_ms"])
            assert_equal(outs["inverted"], outs["scan"], "batch %d, step %d" % (a.batch, step))
        for i in range(a.single + a.warmup):
            q = i % a.batch
            one = (np.array([0, qs[0][q + 1] - qs[0][q]]), qs[1][qs[0][q]:qs[0][q + 1]], qs[2][qs[0][q]:qs[0][q + 1]])
            outs = {}
            for key, ix in pair:
                outs[key], w = timed(ix, one, a.k)
                if i >= a.warmup:
                    res[key]["one_wall"].append(w)
                    res[key]["one_dev"].append(outs[key][3]["total_ms"])
            assert_equal(outs["inverted"], outs["scan"], "single query %d" % q)
        med = {key: {k: float(np.median(v)) for k, v in r.items()} for key, r in res.items()}
        out = {
            "card": name, "power_limit": power, "metric": metric, "rows": a.rows, "batch": a.batch, "k": a.k,
            "steps": a.steps, "warmup": a.warmup, "single_calls": a.single,
            "nnz_per_row": int(rows[0][-1]) / a.rows, "nnz_per_query": int(qs[0][-1]) / a.batch,
            "outputs_bitwise_equal": True,
            "build_s": build_s, "index_terms": info["terms"], "index_postings": info["postings"],
            "index_bytes": info["postings"] * 8 + info["terms"] * 12 + 8,
        }
        for key in ("scan", "inverted"):
            m = med[key]
            out[key] = {"qps": a.batch / m["wall"], "batch_ms_median": m["wall"] * 1e3, "batch_device_ms_median": m["dev"],
                        "single_query_ms_median": m["one_wall"] * 1e3, "single_query_device_ms_median": m["one_dev"]}
        out["speedup_batch"] = med["scan"]["wall"] / med["inverted"]["wall"]
        out["speedup_single_query"] = med["scan"]["one_wall"] / med["inverted"]["one_wall"]
        print(json.dumps(out), flush=True)
        scan.close()
        inv.close()


if __name__ == "__main__":
    main()
