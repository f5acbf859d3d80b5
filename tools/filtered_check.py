"""Filtered graph search: post-filter against collect mode (eps_index_set_filter_search) on the bench's manifold table.

For each table size, k and selectivity of an uncorrelated INT4 filter ("u < s * 2^20", u uniform in [0, 2^20)), the
modes are alternated in one process over the same batch:
  post          the reference's post-filter of the graph queue (the default);
  collect       collect mode as shipped (threshold kCollectScanRows, capi.cu);
  collect-graph collect mode with the threshold at 0 (the graph search always runs);
  collect-scan  collect mode with the threshold above P (the scan over the passing rows answers every query);
  prefilter     the exact scan of prefilter mode, coarse pass on (the library's default);
and each reports queries/s, recall@k against the exact filtered answer (prefilter mode, coarse pass off), the mean
count per query and the share of queries answered by the scan over the passing rows (n_redone / nq).  The card's name
and power limit are read in the same run.  One JSON line per measurement.

    python tools/filtered_check.py [--rows 1000000,10000000] [--k 10,100] [--batch 1024] [--L 512]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

INT4, INT_CONST, LT, VT_INT, VT_BOOL = 7, 1, 19, 1, 3
U_RANGE = 1 << 20


def u_lt(m):
    return np.array([[INT4, VT_INT, -1, -1, 0, 0, 0, 0], [INT_CONST, VT_INT, -1, -1, m, 0, 0, -1],
                     [LT, VT_BOOL, 0, 1, 0, 0, 0, -1]], np.int64)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rows", default="1000000,10000000")
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--batch", type=int, default=1024)
    p.add_argument("--k", default="10,100")
    p.add_argument("--sel", default="0.0001,0.001,0.01,0.1,0.5")
    p.add_argument("--L", type=int, default=512)
    p.add_argument("--width", type=int, default=6)
    p.add_argument("--reps", type=int, default=3)
    a = p.parse_args()
    import torch
    import bench
    import vectordb_b200 as vdb
    dev = torch.device("cuda:0")
    print(json.dumps({"card": card()}), flush=True)
    for rows in [int(r) for r in a.rows.split(",")]:
        X = bench.gen_table(rows, a.dim, "manifold", 42, dev)
        Q = bench.gen_queries(a.batch, a.dim, "manifold", 43, dev)
        u = np.random.default_rng(7).integers(0, U_RANGE, rows).astype(np.int32)
        ix = vdb.Index("l2", a.dim, capacity=rows)
        ix.adopt_device_rows(X.data_ptr(), rows)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ix.build(rows, knn_k=64, nnd_iters=14)
        print(json.dumps({"rows": rows, "build_s": round(time.perf_counter() - t0, 1)}), flush=True)
        ix.set_attrs(u.view(np.uint8), 4, rows)
        ix.set_search_width(a.width)
        for k in [int(x) for x in a.k.split(",")]:
            ids = torch.empty((a.batch, k), dtype=torch.int64, device=dev)
            ds = torch.empty((a.batch, k), dtype=torch.float32, device=dev)
            cnt = torch.empty((a.batch,), dtype=torch.int64, device=dev)

            def run(nodes):
                t = time.perf_counter()
                st = ix.search_device(Q.data_ptr(), a.batch, k, ids.data_ptr(), ds.data_ptr(), cnt.data_ptr(), filter_nodes=nodes,
                                      want_stats=True, sync=True)
                return time.perf_counter() - t, st

            for sel in [float(s) for s in a.sel.split(",")]:
                nodes = u_lt(int(round(sel * U_RANGE)))
                P = int((u < int(round(sel * U_RANGE))).sum())
                ix.config(a.L, a.L, prefilter=True)
                ix.set_coarse("fp32")
                run(nodes)
                truth = [set(r[:c].tolist()) for r, c in zip(ids.cpu().numpy(), cnt.cpu().numpy())]
                ix.set_coarse("tf32")
                modes = [("post", "post", None, False), ("collect", "collect", None, False),
                         ("collect-graph", "collect", "0", False), ("collect-scan", "collect", str(rows + 1), False),
                         ("prefilter", "post", None, True)]
                res = {m[0]: [] for m in modes}
                for rep in range(a.reps + 1):  # rep 0 warms every mode up
                    for name, mode, env, pre in modes:
                        if env is None:
                            os.environ.pop("EPS_COLLECT_SCAN_ROWS", None)
                        else:
                            os.environ["EPS_COLLECT_SCAN_ROWS"] = env
                        ix.config(a.L, a.L, prefilter=pre)
                        ix.set_filter_search(mode)
                        dt, st = run(nodes)
                        if rep == 0:
                            continue
                        got = ids.cpu().numpy()
                        c = cnt.cpu().numpy()
                        hit = [len(truth[q] & set(got[q, :c[q]].tolist())) for q in range(a.batch)]
                        want = sum(len(t) for t in truth)
                        res[name].append((dt, sum(hit) / max(1, want), float(c.mean()), st["n_redone"] / a.batch))
                os.environ.pop("EPS_COLLECT_SCAN_ROWS", None)
                ix.set_filter_search("post")
                for name, r in res.items():
                    dt = sorted(x[0] for x in r)[len(r) // 2]
                    print(json.dumps({"rows": rows, "k": k, "sel": sel, "P": P, "mode": name, "qps": round(a.batch / dt, 1),
                                      "recall": round(r[-1][1], 4), "mean_count": round(r[-1][2], 2),
                                      "scanned_share": round(r[-1][3], 4)}), flush=True)
        ix.close()
        del X, Q
        torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
