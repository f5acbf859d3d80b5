"""Throughput of the sparse exact scan on a seeded SPLADE-like table (eps_search_sparse_batch).

Table: vocabulary 30 522, Zipf-distributed term ids, about 120 nnz per row and 30-40 per query, float32 values.
Default shape: 1M rows, batch 1024, k = 10, inner product.  Prints one JSON line with queries/s, the scan's kernel time
(CUDA events around the distance + selection launches), the card's name and power limit read in the same process, and
the bytes the scan has to move over kernel time against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).

    python tools/sparse_check.py [--rows N] [--batch B] [--steps K] [--warmup W] [--metric ip|l2|cosine]
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

VOCAB = 30522
HBM_BPS = 3.35e12


def splade_like(n, nnz_lo, nnz_hi, seed):
    """CSR with nnz ~ U[nnz_lo, nnz_hi] distinct Zipf(1.1)-ranked term ids per row (drawn with repeats, deduplicated)."""
    rng = np.random.default_rng(seed)
    ranks = np.arange(1, VOCAB + 1, dtype=np.float64)
    p = ranks ** -1.1
    cdf = np.cumsum(p / p.sum())
    perm = rng.permutation(VOCAB)            # term id of each frequency rank
    want = rng.integers(nnz_lo, nnz_hi + 1, n)
    draw = int(want.max() * 1.6) + 8          # repeats of frequent terms are dropped below
    offs = [np.zeros(1, np.int64)]
    idx_parts, val_parts = [], []
    total = 0
    for r0 in range(0, n, 65536):
        m = min(65536, n - r0)
        ids = perm[np.searchsorted(cdf, rng.random((m, draw)))].astype(np.int64)
        ids.sort(axis=1)
        keep = np.ones_like(ids, bool)
        keep[:, 1:] = ids[:, 1:] != ids[:, :-1]
        # keep the first want[r] distinct ids of each row (in index order)
        keep &= np.cumsum(keep, axis=1) <= want[r0:r0 + m, None]
        cnt = keep.sum(1)
        idx_parts.append(ids[keep])
        val_parts.append(rng.random(int(cnt.sum()), dtype=np.float32) * 2.0)
        offs.append(total + np.cumsum(cnt))
        total += int(cnt.sum())
    return np.concatenate(offs), np.concatenate(idx_parts), np.concatenate(val_parts).astype(np.float32)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, power = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, power
    except Exception as e:  # the numbers below are still labelled with what could be read
        return "unknown (%s)" % e, "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--metric", default="ip")
    a = ap.parse_args()
    import vectordb_b200
    L = vectordb_b200.load_library()
    if L.eps_device_count() <= 0:
        sys.exit("sparse_check: no CUDA device: nothing is measured without the GPU")
    t0 = time.time()
    rows = splade_like(a.rows, 100, 140, 1)
    qs = splade_like(a.batch, 30, 40, 2)
    gen_s = time.time() - t0
    ix = vectordb_b200.SparseIndex(a.metric, VOCAB, capacity=a.rows)
    ix.append(rows)
    ix.config(500, 500, force_brute=True)
    for _ in range(a.warmup):
        ix.search(qs, a.k)
    kern, tot, wall = [], [], []
    for _ in range(a.steps):
        t = time.perf_counter()
        ids, ds, cnt, st = ix.search(qs, a.k)
        wall.append(time.perf_counter() - t)
        kern.append(st["kernel_ms"])
        tot.append(st["total_ms"])
    # single-query latency (one query per call, as a REST search issues it): a CTA holds 32 queries, one per lane,
    # so with nq = 1 a warp still walks every row while 31 of its lanes idle
    one = (qs[0][:2], qs[1][:qs[0][1]], qs[2][:qs[0][1]])
    for _ in range(a.warmup):
        ix.search(one, a.k)
    one_wall, one_kern = [], []
    for _ in range(a.steps):
        t = time.perf_counter()
        st1 = ix.search(one, a.k)[3]
        one_wall.append(time.perf_counter() - t)
        one_kern.append(st1["kernel_ms"])
    name, power = card()
    nnz = int(rows[0][-1])
    csr_bytes = nnz * 8 + (a.rows + 1) * 8 + (a.rows * 4 if a.metric.startswith("cos") else 0)
    tiles = (a.batch + 31) // 32
    tile_bytes = a.batch * a.rows * 4 * 2          # fp32 distance tile written by the scan and read by the selection
    kms = float(np.median(kern))
    out = {
        "card": name, "power_limit": power, "rows": a.rows, "batch": a.batch, "k": a.k, "metric": a.metric,
        "nnz_per_row": nnz / a.rows, "nnz_per_query": int(qs[0][-1]) / a.batch,
        "steps": a.steps, "warmup": a.warmup,
        "qps_end_to_end": a.batch / float(np.median(wall)),
        "kernel_ms_median": kms, "kernel_ms_min": float(np.min(kern)), "total_ms_median": float(np.median(tot)),
        "qps_kernel": a.batch / (kms / 1e3),
        "csr_bytes": csr_bytes, "query_tiles": tiles,
        # one CSR pass from HBM (the query tiles of a row slice run side by side and share it through L2) plus the tile
        "hbm_bytes_min": csr_bytes + tile_bytes,
        "hbm_fraction_of_3.35TBps": (csr_bytes + tile_bytes) / (kms / 1e3) / HBM_BPS,
        # every query tile reads the whole CSR: an upper bound on DRAM traffic if L2 shared nothing
        "bytes_all_tiles": csr_bytes * tiles + tile_bytes,
        "bytes_all_tiles_per_s_over_3.35TBps": (csr_bytes * tiles + tile_bytes) / (kms / 1e3) / HBM_BPS,
        "n_dist_per_query": st["n_dist"] / a.batch,
        "single_query_ms_median": float(np.median(one_wall)) * 1e3,
        "single_query_kernel_ms_median": float(np.median(one_kern)),
        # the reference runs on the host: tests/golden/make_sparse_golden.py --time-bruteforce measures it
        "reference_bruteforce_ms_per_query": "see make_sparse_golden.py --time-bruteforce (host CPU)",
        "table_generation_s": gen_s,
    }
    print(json.dumps(out))
    ix.close()


if __name__ == "__main__":
    main()
