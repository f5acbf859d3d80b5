"""Developer tool (GPU): the graph screen on inner-product and cosine indexes, screen off against on, alternated.
  python tools/graph_screen_metric_check.py [--rows 10000000] [--rounds 2] [--L 768] [--metrics ip,cosine]
Builds the bench's manifold table (bench.gen_table, seed 42, 768-d) on the device and, per metric, one graph with the
bench's build parameters (knn_k 64, nnd_iters 14): IP on the raw rows; cosine on rows and queries normalised as the
reference's engine::Normalize does (a sequential fp32 sum of squares, its square root, a division), on the device.  The
graph is installed on a fresh index whose screen is off, so that turning it on times the whole sketch setup
(covariance, basis, row sketches and the dot-product row terms) and measures its device bytes.  Then, alternating the
screen off and on for --rounds rounds, it searches the bench's query batches at the bench's shape (batch 1024, k = 10,
L = 768, width 6, auto geometry): queries/s with one batch at a time and with 3 batches in flight (CUDA events), and
the share of evaluated rows the screen dropped (n_screened / n_dist).  One JSON line per run, with the card's name,
power limit and SM clock read in the same run.  It fails unless ids, distances, counts and the eps_stats counters
(n_dist, n_seed, n_expand, n_edges, n_queries, n_redone) of every batch are bitwise equal between off and on.
With the screen on, it then times the launch rule that prefers a ring leaving 60 KB of L1 (graph_search.cu): 3 batches
in flight under the auto geometry (which asks for the 196 KB shared-memory carve-out when it picks such a ring), against
rings of 10 and 12 rows at 4 CTAs per SM set with set_graph_tuning (the driver's own carve-out: 228 KB for ring 12),
alternated over --rounds rounds."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS, DIM, NQ, K, WIDTH, KNN_K, NND_ITERS, LANES, WARMUP, STEPS = 10_000_000, 768, 1024, 10, 6, 64, 14, 3, 3, 10
COUNTERS = ("n_dist", "n_seed", "n_expand", "n_edges", "n_queries", "n_redone")
OFF, ON = 0, 1


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def normalise_(X, chunk=1 << 16):
    """engine::Normalize on every row of X in place: sum += v[i] * v[i] in order (fp32), then v[i] /= sqrt(sum)."""
    import torch
    for r0 in range(0, X.shape[0], chunk):
        B = X[r0:r0 + chunk]
        T = B.t().contiguous()
        s = torch.zeros(B.shape[0], dtype=torch.float32, device=X.device)
        for i in range(X.shape[1]):
            s += T[i] * T[i]
        B /= torch.sqrt(s)[:, None]


def run_metric(a, metric, X, Qs, vdb, torch):
    dev = X.device
    b = vdb.Index(metric, DIM, capacity=a.rows)
    b.set_graph_screen(OFF)
    b.adopt_device_rows(X.data_ptr(), a.rows)
    t0 = time.perf_counter()
    b.build(a.rows, knn_k=KNN_K, nnd_iters=NND_ITERS)
    build_s = time.perf_counter() - t0
    n, off, nb, nav = b.get_graph()
    b.close()
    ix = vdb.Index(metric, DIM, capacity=a.rows)
    ix.set_graph_screen(OFF)
    ix.adopt_device_rows(X.data_ptr(), a.rows)
    ix.set_graph(n, off, nb, nav)
    del off, nb
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(dev)[0]
    t0 = time.perf_counter()
    ix.set_graph_screen(ON)
    setup_s = time.perf_counter() - t0
    sketch_bytes = free0 - torch.cuda.mem_get_info(dev)[0]
    info = ix.graph_screen_info()
    ix.config(a.L, a.L)
    ix.set_search_width(WIDTH)
    ix.set_graph_tuning(0, 0)
    outs = [[torch.empty((NQ, K), dtype=torch.int64, device=dev), torch.empty((NQ, K), dtype=torch.float32, device=dev),
             torch.empty((NQ,), dtype=torch.int64, device=dev)] for _ in range(LANES)]
    lanes, streams = [], []

    def run(li, s, stats=False):
        o = outs[li]
        return lanes[li].search_device(Qs[s].data_ptr(), NQ, K, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(), want_stats=stats,
                                       sync=stats)

    def one_batch():
        for s in range(WARMUP):
            run(0, s, True)
        scr0 = ix.graph_screen_info()["n_screened"]
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
        st, dumps = [], []
        for s in range(STEPS):
            evs[s][0].record(streams[0])
            st.append(run(0, WARMUP + s, True))
            evs[s][1].record(streams[0])
            dumps.append([t.cpu().numpy() for t in outs[0]])
        torch.cuda.synchronize()
        ms = sum(e0.elapsed_time(e1) for e0, e1 in evs)
        return NQ * STEPS / (ms / 1e3), st, ix.graph_screen_info()["n_screened"] - scr0, dumps

    def in_flight():
        def region(first, cnt):
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record(streams[0])
            for s_ in streams[1:]:
                s_.wait_event(e0)
            for s in range(cnt):
                run(s % LANES, (first + s) % len(Qs))
            ends = []
            for s_ in streams:
                e = torch.cuda.Event(enable_timing=True)
                e.record(s_)
                ends.append(e)
            torch.cuda.synchronize()
            return max(e0.elapsed_time(e) for e in ends)
        region(0, max(WARMUP, LANES))
        return NQ * STEPS / (region(WARMUP, STEPS) / 1e3)

    ref = None
    for rnd in range(a.rounds):
        for mode in (OFF, ON):
            ix.set_graph_screen(mode)  # views copy the mode; the index refuses mode changes while it has views
            lanes[:] = [ix] + [ix.view() for _ in range(LANES - 1)]
            streams[:] = [torch.cuda.ExternalStream(v.stream, device=dev) for v in lanes]
            qps1, st, nscr, dumps = one_batch()
            qps3 = in_flight()
            for v in lanes[1:]:
                v.close()
            ndist = sum(s_["n_dist"] for s_ in st)
            got = (dumps, [{k: s_[k] for k in COUNTERS} for s_ in st])
            if ref is None:
                ref = got
            for s in range(STEPS):
                for i, name in enumerate(("ids", "distances", "counts")):
                    x, y = ref[0][s][i], got[0][s][i]
                    assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), "%s: %s of batch %d differ" % (metric, name, s)
            assert ref[1] == got[1], "%s: eps_stats counters differ: %s vs %s" % (metric, ref[1], got[1])
            r = {"metric": metric, "round": rnd, "screen": "on" if mode == ON else "off", "rows": a.rows, "L": a.L,
                 "qps_one_batch": round(qps1), "qps_in_flight": round(qps3), "n_screened_over_n_dist": nscr / ndist,
                 "n_dist_per_query": ndist / (NQ * STEPS), "variance_share": info["share"], "sketch_setup_s": setup_s,
                 "sketch_device_bytes": sketch_bytes, "build_s": build_s, "outputs_bitwise_equal": True, "card": card()}
            print(json.dumps(r), flush=True)
    ix.set_graph_screen(ON)
    lanes[:] = [ix] + [ix.view() for _ in range(LANES - 1)]
    streams[:] = [torch.cuda.ExternalStream(v.stream, device=dev) for v in lanes]
    geo = {"auto": [], "ring 10, 4 CTAs/SM": [], "ring 12, 4 CTAs/SM": []}
    for rnd in range(a.rounds):
        for name, tuning in (("auto", (0, 0)), ("ring 10, 4 CTAs/SM", (10, 4)), ("ring 12, 4 CTAs/SM", (12, 4))):
            for v in lanes:
                v.set_graph_tuning(*tuning)
            geo[name].append(round(in_flight()))
    for v in lanes[1:]:
        v.close()
    print(json.dumps({"metric": metric, "screen": "on", "launch_geometry_qps_in_flight": geo, "card": card()}), flush=True)
    ix.close()


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rows", type=int, default=ROWS)
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--L", type=int, default=768)
    p.add_argument("--metrics", default="ip,cosine")
    a = p.parse_args()
    import torch
    import vectordb_b200 as vdb
    from bench import gen_queries, gen_table
    dev = torch.device("cuda", 0)
    X = gen_table(a.rows, DIM, "manifold", 42, dev)
    Q = [gen_queries(NQ, DIM, "manifold", 43 + s * 64, dev) for s in range(WARMUP + STEPS)]
    metrics = a.metrics.split(",")
    for metric in sorted(metrics, key=lambda m: m == "cosine"):  # cosine last: it normalises the rows in place
        if metric == "cosine":
            normalise_(X)
            for q in Q:
                normalise_(q)
        torch.cuda.synchronize()
        run_metric(a, metric, X, Q, vdb, torch)


if __name__ == "__main__":
    main()
