"""Sparse graph build with and without posting lists, on the seeded SPLADE-like table of sparse_check.py.

For each row count, one index holds the table; its graph is built (SparseIndex.build, out_degree 50) once by the
all-pairs merge scan and once with posting lists over every row (SparseIndex.build_inverted first), alternating the two
in one process for --repeats rounds.  The graphs (offsets, neighbours, navigation point) must be identical.  Times come
from the host clock around calls that end in a device synchronise.  Prints one JSON line per row count with the card's
name and power limit, read in the same run.

    python tools/sparse_build_check.py [--rows 500000,1000000] [--repeats R] [--metric ip|cosine] [--out-degree D]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="500000,1000000")
    ap.add_argument("--repeats", type=int, default=1)
    ap.add_argument("--metric", default="ip")
    ap.add_argument("--out-degree", type=int, default=50)
    a = ap.parse_args()
    import vectordb_b200
    L = vectordb_b200.load_library()
    if L.eps_device_count() <= 0:
        sys.exit("sparse_build_check: no CUDA device: nothing is measured without the GPU")
    name, power = card()
    for n in (int(s) for s in a.rows.split(",")):
        rows = splade_like(n, 100, 140, 1)
        ix = vectordb_b200.SparseIndex(a.metric, VOCAB, capacity=n)
        ix.append(rows)
        times = {"merge": [], "postings": []}
        graphs = {}
        inverted_s = []
        for _ in range(a.repeats):
            for mode in ("merge", "postings"):
                if mode == "postings":
                    t = time.perf_counter()
                    ix.build_inverted(n)
                    inverted_s.append(time.perf_counter() - t)
                else:
                    ix.build_inverted(0)   # drops the postings
                t = time.perf_counter()
                ix.build(n, out_degree=a.out_degree)
                times[mode].append(time.perf_counter() - t)
                g = ix.get_graph()
                if mode in graphs:
                    assert all(np.array_equal(x, y) for x, y in zip(g, graphs[mode])), mode + ": graph changed between rounds"
                graphs[mode] = g
        for part, x, y in zip(("n_indexed", "offsets", "neighbours", "nav"), graphs["merge"], graphs["postings"]):
            assert np.array_equal(x, y), "%d rows: %s differ between the merge and the postings build" % (n, part)
        out = {
            "card": name, "power_limit": power, "metric": a.metric, "rows": n, "out_degree": a.out_degree,
            "repeats": a.repeats, "nnz_per_row": int(rows[0][-1]) / n, "graphs_equal": True,
            "build_merge_s": times["merge"], "build_postings_s": times["postings"], "build_inverted_s": inverted_s,
            "speedup": float(np.median(times["merge"]) / np.median(times["postings"])),
        }
        print(json.dumps(out), flush=True)
        ix.close()


if __name__ == "__main__":
    main()
