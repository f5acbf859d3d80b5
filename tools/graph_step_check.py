"""Developer tool (GPU): two or more builds of the library on one graph of the bench's table, alternated.
  python tools/graph_step_check.py LIB_A.so LIB_B.so [...] [--rounds 2] [--dist manifold] [--L 768] [--sweep]
Builds the bench's table (seed 42, 768-d) and its graph once, with the bench's generators and build parameters
(knn_k 64, nnd_iters 14), and saves the CSR in /dev/shm.  Then, in one child process per (round, library), A B A B,
each library (loaded through EPS_B200_LIB) installs that graph with set_graph and searches the bench's query batches
(1024 queries, top 10, width 6, auto geometry) at queue length L: queries/s with one batch at a time and with 3 batches
in flight (CUDA events), and per query n_dist / n_expand / n_edges / n_screened.  From those counters it models the
DRAM bytes a query reads, and the rate they imply against the 3.35 TB/s data-sheet figure: the rows it fetches (rows
evaluated minus rows screened, 4 * dim bytes each), the sketches the screen reads (128 B + a 32 B sector for the bound,
per fresh id), and the adjacency rows (256 B per expansion).  The ids, distances and counts of every batch must be
bitwise equal across the libraries, or the tool fails.  --sweep also times every ring size {4, 6, 8, 9, 10, 11, 12} x CTAs per
SM {4, 5, 6, 7} (set_graph_tuning) with 3 batches in flight.  A library built with the phase timers (make prof) prints
its [gs-profile] lines; they are passed on.  Prints one JSON line per child and a summary line, with the card's name,
power limit and SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ROWS, DIM, NQ, K, WIDTH, KNN_K, NND_ITERS, LANES, WARMUP, STEPS = 10_000_000, 768, 1024, 10, 6, 64, 14, 3, 3, 10
HBM_PEAK = 3.35e12  # NVIDIA data sheet, H100 SXM


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def table(a):
    import torch
    from bench import gen_table
    X = gen_table(a.rows, DIM, a.dist, 42, torch.device("cuda", 0))
    torch.cuda.synchronize()
    return X


def build_child(a):
    import numpy as np
    import torch
    import vectordb_b200
    X = table(a)
    ix = vectordb_b200.Index("l2", DIM, capacity=a.rows)
    ix.adopt_device_rows(X.data_ptr(), a.rows)
    ix.build(a.rows, knn_k=KNN_K, nnd_iters=NND_ITERS)
    n, off, nb, nav = ix.get_graph()
    np.savez(a.graph, n=n, off=off, nb=nb.astype(np.int32), nav=nav)
    ix.close()
    torch.cuda.synchronize()


def search_child(a):
    import numpy as np
    import torch
    import vectordb_b200
    from bench import gen_queries
    dev = torch.device("cuda", 0)
    X = table(a)
    Qs = [gen_queries(NQ, DIM, a.dist, 43 + s * 64, dev) for s in range(WARMUP + STEPS)]
    g = np.load(a.graph)
    ix = vectordb_b200.Index("l2", DIM, capacity=a.rows)
    ix.adopt_device_rows(X.data_ptr(), a.rows)
    ix.set_graph(int(g["n"]), g["off"], g["nb"], int(g["nav"]))
    lanes = [ix] + [ix.view() for _ in range(LANES - 1)]
    outs = [[torch.empty((NQ, K), dtype=torch.int64, device=dev), torch.empty((NQ, K), dtype=torch.float32, device=dev),
             torch.empty((NQ,), dtype=torch.int64, device=dev)] for _ in lanes]
    streams = [torch.cuda.ExternalStream(v.stream, device=dev) for v in lanes]

    def setup(ring=0, ctas=0):
        for v in lanes:
            v.config(a.L, a.L)
            v.set_search_width(WIDTH)
            v.set_graph_tuning(ring, ctas)

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
        nscr = ix.graph_screen_info()["n_screened"] - scr0
        return NQ * STEPS / (ms / 1e3), st, nscr, dumps

    def in_flight():
        def region(first, n):
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record(streams[0])
            for s_ in streams[1:]:
                s_.wait_event(e0)
            for s in range(n):
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

    setup()
    qps1, st, nscr, dumps = one_batch()
    qps3 = in_flight()
    per = {k: sum(s_[k] for s_ in st) / (NQ * STEPS) for k in ("n_dist", "n_seed", "n_expand", "n_edges")}
    per["n_screened"] = nscr / (NQ * STEPS)
    fresh = per["n_dist"] - per["n_seed"]
    rows = fresh - per["n_screened"]
    sk = fresh if nscr > 0 else 0.0
    dram = rows * 4 * DIM + sk * (128 + 32) + per["n_expand"] * 256
    r = {"lib": a.lib, "card": card(), "qps_one_batch": qps1, "qps_in_flight": qps3, "per_query": per,
         "dram_bytes_per_query": dram, "dram_GBps_in_flight": dram * qps3 / 1e9, "share_of_3.35TBps": dram * qps3 / HBM_PEAK}
    if a.sweep:
        sw = {}
        for ring in (4, 6, 8, 9, 10, 11, 12):
            for ctas in (4, 5, 6, 7):
                setup(ring, ctas)
                sw["%d,%d" % (ring, ctas)] = in_flight()
        r["sweep_in_flight"] = sw
        setup()
    np.savez(a.dump, **{"%s_%d" % (n_, s): d[i] for s, d in enumerate(dumps) for i, n_ in enumerate(("ids", "distances", "counts"))})
    for v in lanes[1:]:
        v.close()
    ix.close()
    print("RESULT " + json.dumps(r), flush=True)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("libs", nargs="*")
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--rows", type=int, default=ROWS)
    p.add_argument("--dist", default="manifold", choices=["manifold", "cluster"])
    p.add_argument("--L", type=int, default=768)
    p.add_argument("--sweep", action="store_true")
    p.add_argument("--child", default="", choices=["", "build", "search"])
    p.add_argument("--graph", default="")
    p.add_argument("--lib", default="")
    p.add_argument("--dump", default="")
    a = p.parse_args()
    if a.child == "build":
        return build_child(a)
    if a.child == "search":
        return search_child(a)
    import numpy as np
    assert len(a.libs) >= 2, "give at least two libraries"
    shm = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    tmp = tempfile.mkdtemp(prefix="graph_step_check_", dir=shm)
    graph = os.path.join(tmp, "graph.npz")
    base = [sys.executable, os.path.abspath(__file__), "--rows", str(a.rows), "--dist", a.dist, "--L", str(a.L), "--graph", graph]
    results = {lib: [] for lib in a.libs}
    try:
        subprocess.check_call(base + ["--child", "build"])
        for rnd in range(a.rounds):
            for li, lib in enumerate(a.libs):
                dump = os.path.join(tmp, "out_%d_%d.npz" % (rnd, li))
                env = dict(os.environ, EPS_B200_LIB=os.path.abspath(lib))
                pr = subprocess.run(base + ["--child", "search", "--lib", lib, "--dump", dump] + (["--sweep"] if a.sweep else []),
                                    env=env, capture_output=True, text=True)
                prof = {}  # the last [gs-profile] line of each kind: those of the last timed one-batch step
                for line in pr.stderr.splitlines():
                    if line.startswith("[gs-profile]"):
                        prof[line[13:30]] = line
                for line in prof.values():
                    print("  %s: %s" % (os.path.basename(lib), line), flush=True)
                if pr.returncode != 0:
                    sys.stderr.write(pr.stderr[-4000:])
                    raise SystemExit("child failed for %s" % lib)
                r = json.loads([ln for ln in pr.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
                print(json.dumps(r), flush=True)
                results[lib].append(r)
                ref = np.load(os.path.join(tmp, "out_0_0.npz"))
                got = np.load(dump)
                for key in ref.files:
                    assert np.array_equal(ref[key], got[key]), "%s differs between %s and %s" % (key, a.libs[0], lib)
        summary = {"card": card(), "dist": a.dist, "L": a.L, "outputs_bitwise_equal": True}
        for lib, rs in results.items():
            summary[os.path.basename(lib)] = {
                "qps_in_flight": sorted(round(r["qps_in_flight"]) for r in rs),
                "qps_one_batch": sorted(round(r["qps_one_batch"]) for r in rs),
                "dram_GBps_in_flight": sorted(round(r["dram_GBps_in_flight"]) for r in rs)}
        print("SUMMARY " + json.dumps(summary), flush=True)
    finally:
        for f in os.listdir(tmp):
            os.remove(os.path.join(tmp, f))
        os.rmdir(tmp)


if __name__ == "__main__":
    main()
