"""Cost of LIKE filters on the device (DESIGN.md §K3).

    python tools/like_check.py [--rows 1000000] [--dim 768]

1. The match kernel alone: a 1-row index whose dictionary holds 1M / 10M distinct synthetic titles (~30 bytes), searched
   with `name LIKE '%x%'` and with `name = 'x'`; the difference of the two calls' device time (CUDA events, eps_stats
   total_ms) is the LIKE pass.  It is set against the dictionary's bytes at 3.35 TB/s.
2. Exact scan and graph search on a rows x dim table at batch 1024 and 1, with `name LIKE '%x%'` against an IN filter
   (an OR of =) that admits the same rows: the rows' names come from 400 titles, 20 of which contain an 'x', and the
   dictionary holds 1M titles in all, so the LIKE pass runs over 1M codes per call.
Prints one JSON line per measurement, with the card's name and power limit read in the same run.
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
import vectordb_b200 as vdb  # noqa: E402

S_CONST, S_ATTR, EQ, OR, LIKE = 2, 9, 21, 26, 29
WORDS = [b"sale", b"city", b"blue", b"river", b"house", b"garden", b"north", b"light", b"stone", b"market", b"paper",
         b"winter", b"gold", b"field", b"tower", b"glass", b"music", b"storm", b"cloud", b"forest"]


def titles(n, seed):
    """n distinct ~30-byte titles without an 'x' (the numbering keeps them distinct)."""
    rng = np.random.default_rng(seed)
    w = rng.integers(0, len(WORDS), (n, 4))
    return [b" ".join(WORDS[j] for j in w[i]) + b" %d" % i for i in range(n)]


def like_nodes(code):
    return np.array([[S_ATTR, 0, -1, -1, 0, 0, 0, 0], [S_CONST, 0, -1, -1, code, 0, 0, -1], [LIKE, 3, 0, 1, 0, 0, 0, -1]], np.int64)


def in_nodes(codes):
    rows = [[S_ATTR, 0, -1, -1, 0, 0, 0, 0]]
    acc = None
    for c in codes:
        rows.append([S_CONST, 0, -1, -1, int(c), 0, 0, -1])
        rows.append([EQ, 3, 0, len(rows) - 1, 0, 0, 0, -1])
        if acc is not None:
            rows.append([OR, 3, acc, len(rows) - 1, 0, 0, 0, -1])
        acc = len(rows) - 1
    return np.array(rows, np.int64)


def device_ms(ix, Q, limit, nodes, reps):
    ix.search(Q, limit, filter_nodes=nodes)
    t = []
    for _ in range(reps):
        t.append(ix.search(Q, limit, filter_nodes=nodes)[3]["total_ms"])
    return float(np.median(t))


def kernel_pass(n, card):
    ix = vdb.Index("l2", 4, host_vectors=np.zeros((1, 4), np.float32))
    ix.sync_rows(1)
    ix.config(10, 10, force_brute=True)
    t0 = time.perf_counter()
    strings = titles(n, 1)
    for i in range(0, n, 1 << 20):
        ix.append_string_dictionary(i, strings[i:i + (1 << 20)])
    nbytes = sum(len(s) for s in strings)
    ix.append_string_dictionary(n, [b"%x%"])
    ix.set_string_codes(0, 0, np.zeros(1, np.int32))
    upload_s = time.perf_counter() - t0
    Q = np.zeros((1, 4), np.float32)
    like = device_ms(ix, Q, 1, like_nodes(n), 20)
    eq = device_ms(ix, Q, 1, in_nodes([n]), 20)
    ix.close()
    print(json.dumps(dict(what="match kernel", card=card, codes=n, dict_bytes=nbytes, like_ms=like, eq_ms=eq,
                          pass_ms=like - eq, bound_ms=(nbytes + 8 * n) / 3.35e12 * 1e3, host_prepare_s=upload_s)))


def searches(rows, dim, card):
    rng = np.random.default_rng(2)
    X = rng.standard_normal((rows, dim), dtype=np.float32)
    dic = titles(1_000_000, 3)
    hits = [b"box " + d for d in dic[:20]]          # the 20 titles with an 'x'
    dic = hits + dic[20:]
    codes = rng.integers(0, 400, rows).astype(np.int32)
    ix = vdb.Index("l2", dim, host_vectors=X)
    ix.sync_rows(rows)
    for i in range(0, len(dic), 1 << 20):
        ix.append_string_dictionary(i, dic[i:i + (1 << 20)])
    ix.append_string_dictionary(len(dic), [b"%x%"])
    ix.set_string_codes(0, 0, codes)
    like, eq = like_nodes(len(dic)), in_nodes(range(20))
    t0 = time.perf_counter()
    ix.build(rows)
    build_s = time.perf_counter() - t0
    for mode, force in (("exact scan", True), ("graph", False)):
        ix.config(256, 256, force_brute=force)
        for nq in (1024, 1):
            Q = rng.standard_normal((nq, dim), dtype=np.float32)
            a = ix.search(Q, 10, filter_nodes=like)
            b = ix.search(Q, 10, filter_nodes=eq)
            same = all(np.array_equal(x, y) for x, y in zip(a[:3], b[:3]))
            reps = 5 if nq > 1 else 50
            t_like, t_in = device_ms(ix, Q, 10, like, reps), device_ms(ix, Q, 10, eq, reps)
            print(json.dumps(dict(what=mode, card=card, rows=rows, dim=dim, nq=nq, like_ms=t_like, in_ms=t_in,
                                  like_minus_in_ms=t_like - t_in, same_answers=same, selectivity=float(np.mean(codes < 20)),
                                  graph_build_s=build_s)))
    ix.close()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rows", type=int, default=1_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--skip-search", action="store_true")
    a = p.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    for n in (1_000_000, 10_000_000):
        kernel_pass(n, card)
    if not a.skip_search:
        searches(a.rows, a.dim, card)


if __name__ == "__main__":
    main()
