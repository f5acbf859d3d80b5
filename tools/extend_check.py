"""Developer tool (GPU): eps_index_extend_graph against a full build on the bench's table.
  python tools/extend_check.py [base_rows appended_rows ...]      (default: 9000000 1000000)
For each (base, appended) pair, on the first base + appended rows of the bench's manifold table (768-d, seed 42) with
the bench's build parameters: a full build over every row; a build over the base rows, searched with the appended rows
as the exact-scan tail; that graph extended to every row.  Prints one JSON line per pair on stdout: build and
extension times, the extension's phase split (EPS_EXTEND_PHASES, which
synchronises at every phase boundary), recall@10 of the three at L = 256, 512, 768 (width 6, batches of 1024) against
an fp32 torch scan, graph-search queries/s of the tail and extended indexes at L = 768 (one batch at a time, CUDA events),
and the card's name and power limit read in the same run."""
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import vectordb_b200
from bench import gen_queries, gen_table

DIM, NQ, K, WIDTH, KNN_K, NND_ITERS = 768, 1024, 10, 6, 64, 14
LS = (256, 512, 768)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def search(ix, Q, L, width):
    ix.config(L, L)
    ix.set_search_width(width)
    dev = Q.device
    ids = torch.empty((NQ, K), dtype=torch.int64, device=dev)
    ds = torch.empty((NQ, K), dtype=torch.float32, device=dev)
    cnt = torch.empty((NQ,), dtype=torch.int64, device=dev)
    ix.search_device(Q.data_ptr(), NQ, K, ids.data_ptr(), ds.data_ptr(), cnt.data_ptr())
    return ids


def exact_truth(X, Q, chunk=1 << 20):
    """Top-K ids by L2 in fp32 (torch, TF32 off): the yardstick, independent of the library."""
    torch.backends.cuda.matmul.allow_tf32 = False
    qn = (Q * Q).sum(1, keepdim=True)
    best_d = best_i = None
    for r0 in range(0, X.shape[0], chunk):
        Xc = X[r0:r0 + chunk]
        d = qn - 2.0 * Q @ Xc.T + (Xc * Xc).sum(1)[None, :]
        dv, di = d.topk(K, dim=1, largest=False)
        di += r0
        if best_d is None:
            best_d, best_i = dv, di
        else:
            dv, sel = torch.cat([best_d, dv], 1).topk(K, dim=1, largest=False)
            best_d, best_i = dv, torch.cat([best_i, di], 1).gather(1, sel)
    return best_i


def recall(ids, truth):
    return float((ids[:, :, None] == truth[:, None, :]).any(-1).sum()) / truth.numel()


def qps(ix, Q, L, reps=10):
    search(ix, Q, L, WIDTH)  # warm-up of this shape
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = 0.0
    for _ in range(reps):
        start.record()
        search(ix, Q, L, WIDTH)
        stop.record()
        stop.synchronize()
        ms += start.elapsed_time(stop)
    return NQ * reps / (ms / 1e3)


def index_over(X, rows):
    ix = vectordb_b200.Index("l2", DIM, capacity=rows)
    ix.adopt_device_rows(X.data_ptr(), rows)
    return ix


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def extend_with_phases(ix, n):
    """extend_graph with EPS_EXTEND_PHASES set; the library's phase line is read from fd 2."""
    os.environ["EPS_EXTEND_PHASES"] = "1"
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            s = timed(lambda: ix.extend_graph(n, knn_k=KNN_K, nnd_iters=NND_ITERS))
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            del os.environ["EPS_EXTEND_PHASES"]
        f.seek(0)
        lines = [l for l in f.read().splitlines() if l.startswith("{")]
    return s, (json.loads(lines[-1]) if lines else None)


def progress(out, key):
    print("%s: %s" % (key, out[key]), file=sys.stderr, flush=True)  # long steps: show that the run is alive


def run(base, appended, dev):
    n = base + appended
    X = gen_table(n, DIM, "manifold", 42, dev)
    Q = gen_queries(NQ, DIM, "manifold", 43, dev)
    out = {"rows": n, "base_rows": base, "appended_rows": appended, "dim": DIM}
    truth = exact_truth(X, Q)
    ix = index_over(X, n)
    out["full_build_s"] = timed(lambda: ix.build(n, knn_k=KNN_K, nnd_iters=NND_ITERS))
    progress(out, "full_build_s")
    out["full_recall"] = {L: recall(search(ix, Q, L, WIDTH), truth) for L in LS}
    ix.close()
    ix = index_over(X, n)
    out["base_build_s"] = timed(lambda: ix.build(base, knn_k=KNN_K, nnd_iters=NND_ITERS))
    progress(out, "base_build_s")
    out["tail_recall"] = {L: recall(search(ix, Q, L, WIDTH), truth) for L in LS}
    out["tail_qps_L768"] = qps(ix, Q, 768)
    progress(out, "tail_qps_L768")
    out["extend_s"], phases = extend_with_phases(ix, n)
    progress(out, "extend_s")
    out.update(phases or {})
    assert ix.get_graph()[0] == n
    out["extended_recall"] = {L: recall(search(ix, Q, L, WIDTH), truth) for L in LS}
    out["extended_qps_L768"] = qps(ix, Q, 768)
    out["extend_over_full_build"] = out["extend_s"] / out["full_build_s"]
    ix.close()
    del X, Q
    torch.cuda.empty_cache()
    return out


def main():
    args = [int(a) for a in sys.argv[1:]] or [9_000_000, 1_000_000]
    dev = torch.device("cuda", 0)
    gpu = card()
    for base, appended in zip(args[0::2], args[1::2]):
        out = run(base, appended, dev)
        out["gpu"] = gpu
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
