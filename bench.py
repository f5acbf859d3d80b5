#!/usr/bin/env python
"""bench.py — headline benchmark of the H100-native Epsilla vector-search hot path.

Metric (BASELINE.json): QPS at recall@10 >= 0.99 on 10M x 768 float32, batch = 1024, top-10, reported with the
roofline fraction of the dominant kernel and with the reference's own CPU path timed on the same box.

  python bench.py [--gpus N --steps K --warmup W] [--impl reference] [--dump-outputs DIR]
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...

Workload.  Three synthetic 10M x 768 tables (random floats, seeded, generated on the device):
  * "manifold" (headline, --dist): SURVEY.md §8d's clustered variant — 1024 Gaussian centres, sigma = 0.1, seed 44 —
    with the blobs living in a 32-d latent space (centres N(0, 0.15^2) there, so neighbouring blobs overlap) that a
    fixed orthonormal map embeds in R^768, plus isotropic noise of sigma 0.005: clustered data of low intrinsic
    dimension, the structure embedding tables have and the case a graph index exists for (a queue length L of a
    few hundred reaches recall 0.99).  (Logs made before this scaling describe the same table with unit blobs: every
    length is 10x larger, every ranking identical.)
  * "cluster": the same variant read the other way, centres uniform in the unit cube with ISOTROPIC sigma = 0.1 blobs in
    all 768 dimensions.
    Distances inside a blob concentrate, so recall 0.99 means visiting the query's whole 9.8k-row blob, and the 1024
    blobs are separate graph components that the search can only enter through the navigation point's > 1000
    out-neighbours: L >= 1536 (PrepareInitIds seeds exactly L of them).  Graph search still beats the exact scan;
  * "uniform": SURVEY.md §8d's iid uniform[0,1) table.  No neighbourhood structure at all (the reference itself
    touches 75-95 % of the table for recall 0.99; graph search at L = 2048 finds 30 % of the neighbours): measured
    with the exact scan.
`value` is the fastest mode (graph at the smallest L of the sweep that reaches the target, or the exact scan) with
recall@10 >= 0.99 on the --dist table; --extra-tables measures the other tables in the same run (N = 1) and prints
them as "uniform" / "cluster" records with their own recall, QPS and rooflines.  The default run carries the uniform
record; `--extra-tables cluster,uniform` (one more graph build) adds the isotropic one.

One "step" = one pass of the hot path over one batch of 1024 queries per GPU.  A step is timed with CUDA events on
the index's launch stream, bracketed by barrier + synchronize, MAX over ranks.  `value` has the queries already
resident in HBM; `e2e` goes through the host-buffer C-ABI call (eps_search_batch: H2D of the queries and D2H of
ids / distances / counts inside the timed region).  --dump-outputs DIR writes what the last timed step of `value`
returned (ids and counts as float64, distances as float32) to DIR/<name>.npy; the inputs are seeded, so two builds run
with the same arguments can be compared output for output.

Reference arm (--impl reference) and `cpu_baseline`: the reference's own VecSearchExecutor (oracle/_ref = its
sources compiled unmodified) searching THE SAME CSR graph at the same queue length on the host cores, in the two
modes of SURVEY.md §8d: (i) the reference defaults, NumExecutorPerField = 16 executors x IntraQueryThreads = 4, and
(ii) throughput-optimal, one executor per core at IntraQueryThreads = 1.  The graph is built on the device
beforehand (untimed set-up: the reference's own build needs days at 10M rows); the timed region is the reference's
code only.  It runs in a child process under a timeout (a starved OpenMP team hangs the reference, SURVEY.md Q9).

Multi-GPU (N > 1): the 10M x 768 table (30.7 GB) fits one GPU, so ranks hold replicas and the query stream is
partitioned (independent units, no data-path collective, scaling "weak").  --shard-rows instead partitions the
ROWS (config C5 shape): every rank searches the same batch over its shard and the per-shard top-k are exchanged by
the library itself (eps_search_batch_sharded: ncclAllGather + merge kernel on the index stream).
"""
import argparse
import atexit
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "QPS @ recall@10>=0.99, 10Mx768 f32, batch=1024"


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", default="ours", choices=["ours", "reference", "reference-child"])
    p.add_argument("--rows", type=int, default=10_000_000)
    p.add_argument("--dim", type=int, default=768)
    p.add_argument("--batch", type=int, default=1024)
    p.add_argument("--k", type=int, default=10)
    p.add_argument("--metric", default="l2")
    p.add_argument("--dist", default="manifold", choices=["uniform", "cluster", "manifold"])
    p.add_argument("--centers", type=int, default=1024)
    p.add_argument("--modes", default="graph,brute-bf16", help="candidate modes: graph, brute-bf16, brute-tf32, brute-fp32")
    p.add_argument("--L-sweep", default="128,192,256,384,512,768,1024,1536,2048,3072,4096", help="graph queue lengths, ascending; stops at the first that reaches the recall target")
    p.add_argument("--width", type=int, default=6, help="graph search width (1 = the reference's sequential order)")
    p.add_argument("--lanes", type=int, default=3, help="concurrent batches in flight: the index + (lanes-1) read-only views, "
                   "steps issued round-robin (1 = strictly one batch at a time)")
    p.add_argument("--ring", type=int, default=0, help="graph kernel: TMA row-ring slots per CTA (0 = auto)")
    p.add_argument("--ctas", type=int, default=0, help="graph kernel: resident CTAs per SM (0 = auto)")
    p.add_argument("--knn-k", type=int, default=64)
    p.add_argument("--nnd-iters", type=int, default=14)
    p.add_argument("--extra-tables", default="uniform", help="other SURVEY 8d tables measured in the same run at N=1 "
                   "(uniform: exact scan, + graph with --uniform-graph; cluster: graph build + graph + exact scan); '' = none")
    p.add_argument("--uniform-graph", action="store_true", help="also build + search a graph on the iid-uniform table")
    p.add_argument("--shard-rows", action="store_true")
    p.add_argument("--recall-target", type=float, default=0.99)
    p.add_argument("--cpu-queries", type=int, default=256)
    p.add_argument("--cpu-timeout", type=int, default=420)
    p.add_argument("--no-cpu", action="store_true")
    p.add_argument("--graph-file", default="", help="(reference-child) npz with the CSR to search")
    p.add_argument("--L", type=int, default=0, help="(reference arm) queue length; 0 = take it from the graph file / 512")
    p.add_argument("--filter", default="", help="(reference-child) filter string for the reference's parser")
    p.add_argument("--attr-mod", type=int, default=0, help="(reference-child) INT4 column ID = row %% this")
    p.add_argument("--seed-shift", type=int, default=0, help="(reference-child) table seed = 42 + this (row shards)")
    p.add_argument("--dump-outputs", default="", metavar="DIR", help="write the outputs of the last timed step to DIR/<name>.npy")
    return p.parse_args()


# ------------------------------------------------------------------------------------------------------
# synthetic data (identical bits on every rank and in the reference arm: generated on device in 1M-row chunks from
# a seeded Philox stream; the CPU generator of the same seed is a different stream and is only used when no GPU
# is present, i.e. in the CPU contract test)
# ------------------------------------------------------------------------------------------------------
LATENT_DIM = int(os.environ.get("EPS_BENCH_LATENT", "32"))       # "manifold" tables: dimension of the latent space
LATENT_SIGMA = float(os.environ.get("EPS_BENCH_SIGMA", "0.1"))     # std of every Gaussian blob (SURVEY 8d: sigma = 0.1)
LATENT_SPREAD = float(os.environ.get("EPS_BENCH_SPREAD", "1.5"))   # std of the mixture centres, in units of the blob std
LATENT_NOISE = float(os.environ.get("EPS_BENCH_NOISE", "0.05"))    # isotropic noise in the full space, in units of the blob std


def _mixture(dim, dist, device, centers_n):
    """Fixed (seed 44) parameters of the synthetic tables.  "cluster": centres uniform in the unit cube, isotropic blobs
    of std 0.1 in all `dim` dimensions (distances concentrate: the hardest case for any graph index).  "manifold": a
    mixture of overlapping unit Gaussians in a LATENT_DIM-dimensional latent space, mapped into R^dim by a fixed linear
    map with orthonormal rows, plus small isotropic noise — low intrinsic dimension, as embedding tables have."""
    import torch
    gc = torch.Generator(device=device)
    gc.manual_seed(44)
    if dist == "cluster":
        return torch.rand((centers_n, dim), generator=gc, device=device), None
    lat = torch.randn((centers_n, LATENT_DIM), generator=gc, device=device) * (LATENT_SPREAD * LATENT_SIGMA)
    a = torch.randn((dim, LATENT_DIM), generator=gc, device=device)
    q, _ = torch.linalg.qr(a)  # dim x LATENT_DIM, orthonormal columns
    return lat, q.T.contiguous()


def _draw(out, dist, g, device, centers, umap):
    import torch
    n, dim = out.shape
    if dist == "uniform":
        out.uniform_(0.0, 1.0, generator=g)
        return
    lab = torch.randint(0, centers.shape[0], (n,), generator=g, device=device)
    if dist == "cluster":
        out.normal_(0.0, 0.1, generator=g)
        out += centers[lab]
        return
    z = torch.randn((n, LATENT_DIM), generator=g, device=device) * LATENT_SIGMA
    z += centers[lab]
    out.normal_(0.0, LATENT_NOISE * LATENT_SIGMA, generator=g)
    out.addmm_(z, umap)


def table_chunks(rows, dim, dist, seed, device, centers_n=1024, out=None):
    """The rows of the seeded table in 1M-row chunks, drawn in order (into `out` when given): (first row, chunk)."""
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    centers, umap = (None, None) if dist == "uniform" else _mixture(dim, dist, device, centers_n)
    step = 1_000_000
    for r0 in range(0, rows, step):
        n = min(rows, r0 + step) - r0
        buf = out[r0:r0 + n] if out is not None else torch.empty((n, dim), dtype=torch.float32, device=device)
        _draw(buf, dist, g, device, centers, umap)
        yield r0, buf


def gen_table(rows, dim, dist, seed, device, centers_n=1024):
    import torch
    X = torch.empty((rows, dim), dtype=torch.float32, device=device)
    for _ in table_chunks(rows, dim, dist, seed, device, centers_n, out=X):
        pass
    return X


def gen_queries(n, dim, dist, seed, device, centers_n=1024):
    import torch
    g = torch.Generator(device=device)
    g.manual_seed(seed)
    Q = torch.empty((n, dim), dtype=torch.float32, device=device)
    centers, umap = (None, None) if dist == "uniform" else _mixture(dim, dist, device, centers_n)
    _draw(Q, dist, g, device, centers, umap)
    return Q


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region (read only; the sampler is stopped at exit)."""

    def __init__(self, index):
        self.index = index
        self.samples = []
        self.proc = None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            atexit.register(self.proc.kill)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.samples.append(line.strip())

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        sm, mx, reasons = [], [], set()
        for s in self.samples:
            f = [x.strip() for x in s.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def measured_peaks():
    """HBM GB/s and dense BF16 TFLOP/s to state rooflines against: MEASURED_PEAKS.json when present, else the H100 SXM
    data sheet (3.35 TB/s, 989 TFLOP/s at 700 W; a card with a lower power limit does not reach them)."""
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            d = json.load(open(p))
            return float(d["hbm_gbs"]), float(d.get("bf16_tflops_sustained", d.get("bf16_tflops", 989.0))), "measured"
        except Exception:
            pass
    return 3350.0, 989.0, "H100 SXM data sheet"


def workload_name(a, extra=""):
    data = {"uniform": "iid-uniform[0,1)",
            "cluster": "clustered, isotropic (%d Gaussian centres in the unit cube, sigma=0.1 in all %d dimensions)" % (a.centers, a.dim),
            "manifold": "clustered, low intrinsic dimension (%d Gaussian centres, sigma=%.2f, centre std %.3f, in a %d-d latent "
                        "space mapped to R^%d by a fixed orthonormal map, + isotropic noise sigma=%.4f)" % (
                            a.centers, LATENT_SIGMA, LATENT_SPREAD * LATENT_SIGMA, LATENT_DIM, a.dim, LATENT_NOISE * LATENT_SIGMA)}[a.dist]
    return "%dx%d f32 %s %s (seed 42), batch=%d, top-%d%s" % (a.rows, a.dim, a.metric, data, a.batch, a.k, extra)


# ------------------------------------------------------------------------------------------------------
# the reference's CPU path (oracle/_ref = the reference's own sources compiled unmodified)
# ------------------------------------------------------------------------------------------------------
def reference_child(a):
    """Child process: load the table (regenerated with the same seed on the device when there is one) and the CSR
    from --graph-file, then time VecSearchExecutor::Search on the host cores.  Prints one JSON object."""
    import torch
    from oracle import oracle
    g = np.load(a.graph_file, allow_pickle=False)
    dev = "cuda:0" if torch.cuda.is_available() else "cpu"

    def host_table(dst):
        # chunk by chunk: the parent's table and index stay resident on the same GPU meanwhile
        for r0, c in table_chunks(a.rows, a.dim, a.dist, 42 + a.seed_shift, dev, a.centers):
            if a.metric == "cosine":
                c /= c.norm(dim=1, keepdim=True)
            dst[r0:r0 + c.shape[0]] = c.cpu().numpy()
    cores = os.cpu_count() or 1
    kind = "reference" if oracle.have_ref() else "port"
    n_indexed = int(g["n_indexed"])
    L = int(a.L or g["L"])
    out = {"kind": kind, "cores": cores, "L": L, "graph": n_indexed > 0, "modes": {}}
    queries = g["queries"]  # [steps_total, nq, dim]
    if kind != "reference":
        Xh = np.empty((a.rows, a.dim), np.float32)
        host_table(Xh)
        port = oracle.Port()
        vals = []
        for s in range(queries.shape[0]):
            t0 = time.perf_counter()
            kw = dict(metric=a.metric, vectors=Xh, queries=queries[s], limit=a.k, L=L)
            if n_indexed > 0:
                kw.update(n_indexed=n_indexed, offsets=g["offsets"], nbrs=g["nbrs"].astype(np.int64), nav=int(g["nav"]))
            port.search_batch(**kw)
            vals.append(queries.shape[1] / (time.perf_counter() - t0))
        out["modes"]["port_T1"] = {"qps": vals, "n_exec": 1, "T": 1}
        print(json.dumps(out))
        return
    r = oracle.Ref(a.metric, a.dim, a.rows, [("ID", "int4")])
    host_table(r.vectors)  # straight into the reference's own table (no second host copy)
    r.set_row_count(a.rows)
    if a.attr_mod > 0:
        r.set_attr_column("ID", (np.arange(a.rows) % a.attr_mod).astype(np.int32))
    if n_indexed > 0:
        r.set_graph(n_indexed, g["offsets"], g["nbrs"].astype(np.int64), int(g["nav"]))
        plans = [("i_defaults_16x4", min(16, max(1, cores // 4)), 4), ("ii_one_executor_per_core", cores, 1)]
    else:
        n_exec = min(16, cores)
        plans = [("brute_force_branch", n_exec, max(1, cores // n_exec))]
    for name, n_exec, T in plans:
        r.make_executors(n_exec, T, L)
        vals = []
        for s in range(queries.shape[0]):
            t0 = time.perf_counter()
            r.search_batch(queries[s], a.k, a.filter)
            vals.append(queries.shape[1] / (time.perf_counter() - t0))
        out["modes"][name] = {"qps": vals, "n_exec": n_exec, "T": T}
    # sequential-order results (IntraQueryThreads = 1, one executor) of the first 32 queries of step 0: parity sample
    if n_indexed > 0:
        r.make_executors(1, 1, L)
        ids, _, _ = r.search_batch(queries[0][:32], a.k, a.filter)
        out["ids_T1_step0"] = ids.tolist()
    print(json.dumps(out))


def run_reference_child(a, graph, L, queries, timeout, filter_str="", attr_mod=0, seed_shift=0):
    """Spawn the child on `graph` = (n_indexed, offsets, nbrs, nav) or None; queries [steps, nq, dim] float32."""
    tmpdir = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    path = os.path.join(tmpdir, "eps_bench_graph_%d.npz" % os.getpid())
    try:
        if graph is None:
            np.savez(path, n_indexed=0, offsets=np.zeros(1, np.int64), nbrs=np.zeros(0, np.int32), nav=0, L=L, queries=queries)
        else:
            np.savez(path, n_indexed=graph[0], offsets=graph[1], nbrs=np.asarray(graph[2], np.int32), nav=graph[3], L=L,
                     queries=queries)
        cmd = [sys.executable, os.path.abspath(__file__), "--impl", "reference-child", "--graph-file", path, "--rows", str(a.rows),
               "--dim", str(a.dim), "--dist", a.dist, "--centers", str(a.centers), "--metric", a.metric, "--k", str(a.k), "--L", str(L),
               "--filter", filter_str, "--attr-mod", str(attr_mod), "--seed-shift", str(seed_shift)]
        env = dict(os.environ)
        for k in ("RANK", "LOCAL_RANK", "WORLD_SIZE", "OMP_NUM_THREADS", "OMP_THREAD_LIMIT"):
            env.pop(k, None)  # torchrun sets OMP_NUM_THREADS=1 for its workers; the reference sizes its own teams
        p = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
        lines = [l for l in p.stdout.splitlines() if l.startswith("{")]
        if p.returncode != 0 or not lines:
            raise RuntimeError("reference child failed rc=%d: %s" % (p.returncode, p.stderr[-400:]))
        return json.loads(lines[-1])
    finally:
        try:
            os.remove(path)
        except OSError:
            pass


def build_graph_for_reference(a, dev):
    """Set-up of the reference arm: a CSR over the table and the queue length to search it at.  On a GPU box the graph
    is built on the device by the library (the reference's own build is infeasible at 10M rows) and L is found by the
    same rule as in the GPU arm — the smallest L of --L-sweep whose recall@k against the exact scan reaches the
    target — so both arms sit at the same operating point; without a GPU (CPU contract test) the reference builds the
    graph itself when the table is small; otherwise there is no graph and the reference takes its brute-force branch."""
    import torch
    if torch.cuda.is_available():
        t0 = time.perf_counter()
        A = Arena(a, a.dist, torch.device("cuda", 0), 0, 0, 1)
        A.ground_truth()
        A.ix.build(a.rows, knn_k=a.knn_k, nnd_iters=a.nnd_iters)
        torch.cuda.synchronize()
        L = a.L
        if not L:
            for cand in [int(x) for x in a.L_sweep.split(",")]:
                if cand > a.rows:
                    break
                L = cand
                A.set_mode(("graph", cand, ""))
                rec = 1.0
                for _ in range(2 if a.width > 1 else 1):  # same gate as the GPU arm: the worse of two passes of the wide mode
                    A.search(A.Qpool[0])
                    rec = min(rec, recall_of(A.truth, A.out_ids, a.k))
                if rec >= a.recall_target:
                    break
        g = A.ix.get_graph()
        A.close()
        torch.cuda.empty_cache()
        return g, L, "built on device by libepsilla_b200 (set-up, untimed, %.0f s incl. the L sweep)" % (time.perf_counter() - t0)
    if a.rows <= 200_000:
        from oracle import oracle
        if oracle.have_ref():
            X = gen_table(a.rows, a.dim, a.dist, 42, "cpu", a.centers).numpy()
            r = oracle.Ref(a.metric, a.dim, a.rows, [("ID", "int4")])
            r.set_rows(X)
            g = r.build(a.rows, threads=os.cpu_count() or 1)
            return g, a.L or 512, "built by the reference itself (RebuildThreads = %d)" % (os.cpu_count() or 1)
    return None, a.L or 512, "no graph: the reference's brute-force branch"


def run_reference_arm(a):
    """--impl reference: the reference's own CPU implementation of the path on the host cores, searching the same
    kind of CSR at the queue length the GPU arm operates at (--L, default 512).  Rank 0 only."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    import torch
    dev = "cuda:0" if torch.cuda.is_available() else "cpu"
    graph, L, how = build_graph_for_reference(a, dev)
    n_steps = a.warmup + a.steps
    Q = np.stack([gen_queries(a.batch, a.dim, a.dist, 43 + s * 64, dev, a.centers).cpu().numpy() for s in range(n_steps)])
    if a.metric == "cosine":
        Q /= np.linalg.norm(Q, axis=2, keepdims=True)
    res = run_reference_child(a, graph, L, Q.astype(np.float32), timeout=max(600, a.cpu_timeout * 3))
    best_name = max(res["modes"], key=lambda m: float(np.mean(res["modes"][m]["qps"][a.warmup:])))
    best = res["modes"][best_name]
    v = float(np.mean(best["qps"][a.warmup:]))
    sample = "every step = the full batch of %d queries, %s, L=%d, %d executors x %d threads; graph %s" % (
        a.batch, best_name, res["L"], best["n_exec"], best["T"], how)
    print(json.dumps({
        "impl": "reference", "metric": METRIC, "value": v, "unit": "queries/s", "n_gpus": a.gpus, "steps": a.steps,
        "warmup": a.warmup, "ms_per_step": 1000.0 * a.batch / v, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_name(a, ", reference VecSearchExecutor on the host cores (%s)" % (
            "graph search L=%d on the same CSR" % res["L"] if res["graph"] else "BruteForceSearch branch"))},
        "cpu_baseline": {"value": v, "unit": "queries/s", "cores": best["n_exec"] * best["T"], "kind": res["kind"], "sample": sample,
                         "modes": {m: float(np.mean(x["qps"][a.warmup:])) for m, x in res["modes"].items()}},
        "e2e": {"value": v, "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }))


# ------------------------------------------------------------------------------------------------------
def recall_of(truth, ids, k):
    t, g = truth.cpu().numpy(), ids.cpu().numpy()
    return float(np.mean([len(set(g[i].tolist()) & set(t[i].tolist())) / k for i in range(t.shape[0])]))


def classify_misses(truth_i, truth_d, got_i, got_d, k, tol=1e-4):
    """Misses of `got` against the exact fp32 scan: a 'tie' is an id swapped for one at the same distance (within
    `tol` relative of the k-th exact distance), anything else is a real loss."""
    ties = real = 0
    for q in range(truth_i.shape[0]):
        tset = set(truth_i[q].tolist())
        missing = tset - set(got_i[q].tolist())
        if not missing:
            continue
        kth = float(truth_d[q, k - 1])
        extra = [j for j in range(k) if int(got_i[q, j]) not in tset]
        for _, j in zip(missing, extra):
            if abs(float(got_d[q, j]) - kth) <= tol * max(abs(kth), 1e-30):
                ties += 1
            else:
                real += 1
        real += max(0, len(missing) - len(extra))
    return {"ties": ties, "real": real}


class Arena:
    """One table on the device with its index, query pool and exact ground truth."""

    def __init__(self, a, dist_name, dev, local, rank, world, seed_shift=0):
        import torch
        import vectordb_b200
        self.a, self.dev, self.dist_name = a, dev, dist_name
        self.rows = a.rows
        self.X = gen_table(a.rows, a.dim, dist_name, 42 + seed_shift, dev, a.centers)
        n_pool = a.warmup + a.steps
        qseed = lambda s: 43 + s * 64 + (0 if a.shard_rows else rank)
        self.Qpool = [gen_queries(a.batch, a.dim, dist_name, qseed(s), dev, a.centers) for s in range(n_pool)]
        if a.metric == "cosine":
            self.X /= self.X.norm(dim=1, keepdim=True)
            self.Qpool = [q / q.norm(dim=1, keepdim=True) for q in self.Qpool]
        self.ix = vectordb_b200.Index(a.metric, a.dim, capacity=a.rows, device=local)
        self.ix.adopt_device_rows(self.X.data_ptr(), a.rows)
        self.out_ids = torch.empty((a.batch, a.k), dtype=torch.int64, device=dev)
        self.out_d = torch.empty((a.batch, a.k), dtype=torch.float32, device=dev)
        self.out_c = torch.empty((a.batch,), dtype=torch.int64, device=dev)
        self.stream = torch.cuda.ExternalStream(self.ix.stream, device=dev)
        torch.cuda.synchronize()  # the library launches on its own non-blocking stream: the generators must be done

    def search(self, q, **kw):
        return self.ix.search_device(q.data_ptr(), self.a.batch, self.a.k, self.out_ids.data_ptr(), self.out_d.data_ptr(),
                                     self.out_c.data_ptr(), **kw)

    def ground_truth(self):
        """fp32 SIMT exact scan (no tensor-core coarse pass) of Qpool[0], cross-checked in fp64 on 4 queries."""
        import torch
        a, dev = self.a, self.dev
        self.ix.config(512, 512, force_brute=True)
        self.ix.set_coarse("fp32")
        self.search(self.Qpool[0])
        self.truth, self.truth_d = self.out_ids.clone(), self.out_d.clone()
        with torch.no_grad():
            qs = self.Qpool[0][:4].double()
            best = torch.full((4, a.k), float("inf"), device=dev, dtype=torch.float64)
            bid = torch.zeros((4, a.k), dtype=torch.int64, device=dev)
            for r0 in range(0, self.rows, 500_000):
                xb = self.X[r0:r0 + 500_000].double()
                if a.metric == "l2":
                    dd = (qs * qs).sum(1)[:, None] - 2 * qs @ xb.T + (xb * xb).sum(1)[None, :]
                elif a.metric == "ip":
                    dd = -(qs @ xb.T)
                else:
                    dd = 1 - qs @ xb.T
                cat_d = torch.cat([best, dd], 1)
                cat_i = torch.cat([bid, torch.arange(r0, r0 + xb.shape[0], device=dev)[None, :].expand(4, -1)], 1)
                best, sel = torch.topk(cat_d, a.k, dim=1, largest=False)
                bid = torch.gather(cat_i, 1, sel)
                del xb, dd
            chk = float(np.mean([len(set(bid[i].tolist()) & set(self.truth[i].tolist())) / a.k for i in range(4)]))
        assert chk >= 0.99, "exact-scan ground truth disagrees with the fp64 check: %.3f" % chk
        return chk

    def set_mode(self, m):
        a = self.a
        for ix in [self.ix] + [ln["ix"] for ln in getattr(self, "lanes", [])[1:]]:
            if m[0] == "graph":
                ix.config(m[1], m[1], force_brute=False)
                ix.set_search_width(a.width)
                ix.set_graph_tuning(a.ring, a.ctas)
            else:
                ix.config(512, 512, force_brute=True)
                ix.set_coarse(m[2])

    def open_lanes(self, n):
        """Lane 0 = the index itself; lanes 1.. = read-only views (own stream + scratch) with their own result buffers."""
        import torch
        a, dev = self.a, self.dev
        self.lanes = [{"ix": self.ix, "stream": self.stream, "ids": self.out_ids, "d": self.out_d, "c": self.out_c}]
        for _ in range(1, n):
            v = self.ix.view()
            self.lanes.append({"ix": v, "stream": torch.cuda.ExternalStream(v.stream, device=dev),
                               "ids": torch.empty_like(self.out_ids), "d": torch.empty_like(self.out_d), "c": torch.empty_like(self.out_c)})

    def close_lanes(self):
        for ln in getattr(self, "lanes", [])[1:]:
            ln["ix"].close()
        self.lanes = []

    def close(self):
        self.close_lanes()
        self.ix.close()
        del self.X, self.Qpool


def main():
    a = parse()
    if a.impl == "reference":
        run_reference_arm(a)
        return
    if a.impl == "reference-child":
        reference_child(a)
        return
    import torch
    import torch.distributed as dist
    import vectordb_b200  # noqa: F401  (fails loudly when libepsilla_b200.so is missing)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)

    def barrier():
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    def min_over_ranks(x):
        t = torch.tensor([x], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MIN)
        return float(t.item())

    hbm_peak, tf_peak, peak_src = measured_peaks()
    n_pool = a.warmup + a.steps
    A = Arena(a, a.dist, dev, local, rank, world, seed_shift=(rank if a.shard_rows else 0))
    ix, rows = A.ix, a.rows
    chk = A.ground_truth()

    # row shards: the exchange lives in the library (ncclAllGather + merge kernel on the index stream)
    group = None
    if a.shard_rows and world > 1:
        from vectordb_b200.sharded import ShardGroup
        uid = [ShardGroup.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        group = ShardGroup(uid[0], rank, world, local)
        m_ids = torch.empty((a.batch, a.k), dtype=torch.int64, device=dev)
        m_d = torch.empty((a.batch, a.k), dtype=torch.float32, device=dev)

    def timed_device_steps(m, n_steps, first, want_stats=True):
        """Device-resident inputs: CUDA events on the launch stream; max over ranks."""
        A.set_mode(m)
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n_steps)]
        stats = []
        barrier()
        for s in range(n_steps):
            q = A.Qpool[(first + s) % n_pool]
            evs[s][0].record(A.stream)
            if group is not None:
                group.search(A.ix, rank * rows, q.data_ptr(), a.batch, a.k, m_ids.data_ptr(), m_d.data_ptr(), sync=True)
                stats.append(None)
            else:
                stats.append(A.search(q, want_stats=want_stats, sync=True))
            evs[s][1].record(A.stream)
        barrier()
        return max_over_ranks(sum(e0.elapsed_time(e1) for e0, e1 in evs)), stats

    def timed_overlapped(m, n_steps, first):
        """Same steps issued round-robin over the lanes without waiting for each other: one start event, one end event
        per lane, region time = latest end - start (device clock), max over ranks."""
        A.set_mode(m)
        lanes = A.lanes
        barrier()
        e0 = torch.cuda.Event(enable_timing=True)
        e0.record(lanes[0]["stream"])
        for ln in lanes[1:]:
            ln["stream"].wait_event(e0)
        for s in range(n_steps):
            ln = lanes[s % len(lanes)]
            q = A.Qpool[(first + s) % n_pool]
            ln["ix"].search_device(q.data_ptr(), a.batch, a.k, ln["ids"].data_ptr(), ln["d"].data_ptr(), ln["c"].data_ptr(), sync=False)
        ends = []
        for ln in lanes:
            e = torch.cuda.Event(enable_timing=True)
            e.record(ln["stream"])
            ends.append(e)
        barrier()
        return max_over_ranks(max(e0.elapsed_time(e) for e in ends))

    # ---- candidate modes: graph at the smallest L reaching the recall target, exact scan ----
    want = [m.strip() for m in a.modes.split(",") if m.strip()]
    report, build_s = [], None
    key_rec = "recall_at_%d" % a.k

    def probe(m):
        A.set_mode(m)
        A.search(A.Qpool[0])
        rec = recall_of(A.truth, A.out_ids, a.k)
        if m[0] == "graph" and a.width > 1:  # the gate is the worse of two passes
            A.search(A.Qpool[0])
            rec = min(rec, recall_of(A.truth, A.out_ids, a.k))
        # every rank builds its own graph (NN-descent is not deterministic): the gate is the worst rank's recall, so that
        # all ranks stop the sweep at the same L and pick the same mode (their barriers must match)
        rec = min_over_ranks(rec)
        timed_device_steps(m, a.warmup, 0)
        ms, stats = timed_device_steps(m, max(2, min(a.steps, 3)), a.warmup)
        qps = (1 if a.shard_rows else world) * a.batch * len(stats) / (ms / 1000.0)
        r = {"mode": m[0], "L": m[1], "coarse": m[2], key_rec: rec, "qps_probe": qps}
        if stats[0] is not None:
            r["n_dist_per_query"] = float(np.mean([s["n_dist"] for s in stats])) / a.batch
            if m[0] == "brute":
                r["queries_redone_by_guard_per_step"] = float(np.mean([s["n_redone"] for s in stats]))
        report.append(r)
        return r

    if "graph" in want:
        t0 = time.perf_counter()
        ix.build(rows, knn_k=a.knn_k, nnd_iters=a.nnd_iters)
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        for L in [int(x) for x in a.L_sweep.split(",")]:
            if L > rows:
                break
            if probe(("graph", L, ""))[key_rec] >= a.recall_target:
                break
    for w in want:
        if w.startswith("brute"):
            probe(("brute", 0, w.split("-")[1] if "-" in w else "tf32"))
    ok = [r for r in report if r[key_rec] >= a.recall_target]
    chosen = max(ok, key=lambda r: r["qps_probe"]) if ok else max(report, key=lambda r: r[key_rec])
    mode = (chosen["mode"], chosen["L"], chosen["coarse"])

    # ---- timed region: `value` (inputs resident in HBM) ----
    # One batch at a time first (per-step kernel times and counters), then — graph mode, --lanes > 1 — the same steps
    # with `lanes` batches in flight: a batch is one wave of persistent CTAs whose duration is set by its longest query
    # (2x the median at 10M rows), so with a single batch in flight the SMs idle behind the stragglers; a second
    # batch on a view of the index fills them.  `value` is the in-flight figure, the serial one is printed beside it.
    clocks = ClockSampler(local)
    timed_device_steps(mode, a.warmup, 0)
    clocks.start()
    prof_region = bool(os.environ.get("EPS_BENCH_PROFILE_REGION"))  # ncu --profile-from-start off: only these steps are captured
    if prof_region:
        torch.cuda.profiler.start()
    ms_serial, stats = timed_device_steps(mode, a.steps, a.warmup)
    if prof_region:
        torch.cuda.profiler.stop()
    if group is not None:
        last_out = {"ids": m_ids.cpu().numpy(), "distances": m_d.cpu().numpy()}
    else:
        last_out = {"ids": A.out_ids.cpu().numpy(), "distances": A.out_d.cpu().numpy(), "counts": A.out_c.cpu().numpy()}
    if stats[0] is None:  # row shards: the sharded call returns no counters; the local search of the same steps does
        stats = [A.search(A.Qpool[(a.warmup + s_) % n_pool], want_stats=True) for s_ in range(a.steps)]
        for st_ in stats:
            st_["kernel_ms"] = ms_serial / a.steps  # step time of the sharded call (local search + exchange + merge)
    have_stats = stats[0] is not None
    launches = int(sum(s["kernel_launches"] for s in stats)) if have_stats else None
    if launches is not None and group is not None:
        launches += 2 * a.steps  # pack_shard_block_kernel + merge_shards_kernel around the ncclAllGather
    kernel_ms = float(sum(s["kernel_ms"] for s in stats)) if have_stats else ms_serial
    agg = {k: float(sum(s[k] for s in stats)) if have_stats else 0.0 for k in ("n_dist", "n_seed", "n_expand", "n_edges")}
    ms_dev, n_lanes, lanes_recall = ms_serial, 1, None
    if mode[0] == "graph" and a.lanes > 1 and group is None:
        A.open_lanes(a.lanes)
        A.set_mode(mode)
        for ln in A.lanes:  # every lane answers the ground-truth batch like the index itself
            ln["ix"].search_device(A.Qpool[0].data_ptr(), a.batch, a.k, ln["ids"].data_ptr(), ln["d"].data_ptr(), ln["c"].data_ptr())
        lanes_recall = [recall_of(A.truth, ln["ids"], a.k) for ln in A.lanes]
        timed_overlapped(mode, max(a.warmup, len(A.lanes)), 0)
        ms_dev = timed_overlapped(mode, a.steps, a.warmup)
        n_lanes = len(A.lanes)
        ln = A.lanes[(a.steps - 1) % n_lanes]  # the lane that ran the last step
        last_out = {"ids": ln["ids"].cpu().numpy(), "distances": ln["d"].cpu().numpy(), "counts": ln["c"].cpu().numpy()}
        kernel_ms = ms_dev  # region time: the launches of different lanes overlap, per-launch times do not add up

    # ---- e2e: host buffers through the public C-ABI call, H2D + D2H inside the timed region ----
    import ctypes as C
    from vectordb_b200.lib import check
    A.set_mode(mode)
    Qhost = [torch.empty((a.batch, a.dim), dtype=torch.float32).pin_memory().copy_(q.cpu()) for q in A.Qpool]
    e_out = [(np.empty((a.batch, a.k), np.int64), np.empty((a.batch, a.k), np.float64), np.empty(a.batch, np.int64)) for _ in range(n_lanes)]
    h_ids = torch.empty((a.batch, a.k), dtype=torch.int64).pin_memory()
    h_d = torch.empty((a.batch, a.k), dtype=torch.float32).pin_memory()
    d_q = torch.empty((a.batch, a.dim), dtype=torch.float32, device=dev)

    def e2e_step(s, lane=0):
        q = Qhost[s % n_pool]
        if group is None:
            h = A.lanes[lane]["ix"].h if n_lanes > 1 else ix.h
            e_ids, e_d, e_c = e_out[lane]
            check(ix.L.eps_search_batch(h, C.c_void_p(q.data_ptr()), a.batch, a.k, None, 0, e_ids.ctypes.data_as(C.c_void_p),
                                        e_d.ctypes.data_as(C.c_void_p), e_c.ctypes.data_as(C.c_void_p), None))
        else:  # row shards: H2D of the replicated batch, sharded search + exchange, D2H of the merged result
            with torch.cuda.stream(A.stream):
                d_q.copy_(q, non_blocking=True)
                group.search(ix, rank * rows, d_q.data_ptr(), a.batch, a.k, m_ids.data_ptr(), m_d.data_ptr(), sync=False)
                h_ids.copy_(m_ids, non_blocking=True)
                h_d.copy_(m_d, non_blocking=True)
            A.stream.synchronize()

    def e2e_run(first, n_steps):
        """n_steps calls of the blocking host-buffer entry point; with lanes, one caller thread per lane (the call
        releases the GIL), steps dealt round-robin."""
        if n_lanes == 1:
            for s in range(n_steps):
                e2e_step(first + s)
            return
        errs = []

        def worker(li):
            try:
                for s in range(li, n_steps, n_lanes):
                    e2e_step(first + s, li)
            except Exception as e:  # surfaced below
                errs.append(e)
        ts = [threading.Thread(target=worker, args=(li,)) for li in range(n_lanes)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        if errs:
            raise errs[0]

    e2e_run(0, max(a.warmup, n_lanes))
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(A.stream)
    e2e_run(a.warmup, a.steps)
    e1.record(A.stream)  # every call has synchronised its own lane before returning
    barrier()
    ms_e2e = max_over_ranks(e0.elapsed_time(e1))
    clk = clocks.stop()

    units = a.batch * a.steps * (1 if a.shard_rows else world)
    value = units / (ms_dev / 1000.0)
    e2e_value = units / (ms_e2e / 1000.0)

    # ---- roofline of the dominant kernel (algorithmic bytes per SURVEY.md §8d / DESIGN.md) ----
    def graph_roofline(agg_, L_, k_ms, n_steps):
        bytes_alg = (agg_["n_dist"] - agg_["n_seed"]) * a.dim * 4.0 + agg_["n_edges"] * 4.0 + agg_["n_expand"] * 16.0 + \
            n_steps * (L_ * a.dim * 4.0) + n_steps * a.batch * (a.dim * 4.0 + a.k * 12.0)
        ach = bytes_alg / (k_ms / 1000.0) / 1e9 if k_ms > 0 else 0.0
        return {"bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "traffic": None,
                "kernel": "graph_search_kernel (persistent CTAs, cp.async.bulk row ring)", "peak_source": peak_src,
                "kernel_ms_per_step": k_ms / n_steps, "algorithmic_bytes_per_step": bytes_alg / n_steps,
                "n_dist_per_query": agg_["n_dist"] / (n_steps * a.batch)}

    def scan_roofline(coarse, k_ms, n_steps):
        bytes_alg = n_steps * (rows * a.dim * 4.0 + a.batch * a.dim * 4.0 + a.batch * a.k * 12.0)
        if coarse == "fp32":
            ach = bytes_alg / (k_ms / 1000.0) / 1e9 if k_ms > 0 else 0.0
            return {"bound": "hbm", "achieved": ach, "peak": hbm_peak, "unit": "GB/s", "frac": ach / hbm_peak, "traffic": None,
                    "kernel": "bf_dist_tile_kernel + bf_select_kernel", "peak_source": peak_src, "kernel_ms_per_step": k_ms / n_steps}
        flop = n_steps * rows * float(a.batch) * a.dim * 2.0
        ach = flop / (k_ms / 1000.0) / 1e12 if k_ms > 0 else 0.0
        peak = tf_peak / 2.0 if coarse == "tf32" else tf_peak  # wgmma TF32 runs at half the BF16 rate
        return {"bound": "tensor", "achieved": ach, "peak": peak, "unit": "TFLOP/s", "frac": ach / peak, "traffic": None,
                "kernel": "tc_dist_kernel (wgmma %s, fused threshold select) + bf_select_kernel + rescore_kernel" % (
                    "tf32" if coarse == "tf32" else "bf16"),
                "peak_source": "%s bf16 (%.0f TF/s)%s" % (peak_src, tf_peak, " / 2 for TF32" if coarse == "tf32" else ""),
                "kernel_ms_per_step": k_ms / n_steps,
                "hbm_algorithmic_GBps": bytes_alg / (k_ms / 1000.0) / 1e9 if k_ms > 0 else 0.0}

    roof = graph_roofline(agg, mode[1], kernel_ms, a.steps) if mode[0] == "graph" else scan_roofline(mode[2], kernel_ms, a.steps)

    # ---- secondary records of the non-chosen modes, each with its own roofline ----
    extra = {}
    for r in report:
        m = (r["mode"], r["L"], r["coarse"])
        if m == mode or r[key_rec] < a.recall_target or group is not None:
            continue
        tag = "graph" if m[0] == "graph" else "exact_scan_" + m[2]
        if tag in extra:
            continue
        ms, st = timed_device_steps(m, min(a.steps, 5), a.warmup)
        k_ms = float(sum(s["kernel_ms"] for s in st))
        ag = {k: float(sum(s[k] for s in st)) for k in ("n_dist", "n_seed", "n_expand", "n_edges")}
        extra[tag] = {"value": world * a.batch * len(st) / (ms / 1000.0), "unit": "queries/s", key_rec: r[key_rec], "L": m[1],
                      "roofline": graph_roofline(ag, m[1], k_ms, len(st)) if m[0] == "graph" else scan_roofline(m[2], k_ms, len(st))}

    # ---- exactness accounting of the exact-scan mode against the fp32 scan (ties vs real losses) ----
    misses = None
    bf = [r for r in report if r["mode"] == "brute" and r["coarse"] != "fp32"]
    if bf and group is None:
        A.set_mode(("brute", 0, bf[0]["coarse"]))
        A.search(A.Qpool[0])
        misses = classify_misses(A.truth.cpu().numpy(), A.truth_d.cpu().numpy(), A.out_ids.cpu().numpy(), A.out_d.cpu().numpy(), a.k)
        misses["queries"] = a.batch
        misses["mode"] = "exact scan, %s coarse pass" % bf[0]["coarse"]

    out = {
        "metric": METRIC, "value": value, "unit": "queries/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
        "ms_per_step": ms_dev / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        "config": {"workload": workload_name(a, ", mode=%s; %s" % (
            ("graph search L=%d width=%d" % (mode[1], a.width)) if mode[0] == "graph" else
            "exact scan (wgmma %s coarse pass + fp32 re-score)" % mode[2],
            "row shards + in-library ncclAllGather + merge" if a.shard_rows else "replicated table, query stream partitioned over ranks")),
            key_rec: chosen[key_rec], "l2_flush": "inputs (%.1f GB table) larger than L2" % (rows * a.dim * 4 / 1e9),
            "fp64_groundtruth_check": chk, "batches_in_flight": n_lanes},
        "e2e": {"value": e2e_value, "unit": "queries/s", "h2d_bytes_per_step": a.batch * a.dim * 4,
                "d2h_bytes_per_step": a.batch * a.k * 12 + (0 if group is not None else a.batch * 8)},
        "gpu_launches": launches, "clocks": clk, "roofline": roof, "modes": report,
    }
    if n_lanes > 1:
        out["one_batch_at_a_time"] = {"value": units / (ms_serial / 1000.0), "unit": "queries/s", "ms_per_step": ms_serial / a.steps,
                                      "roofline_frac": roof["achieved"] * ms_dev / ms_serial / roof["peak"]}
        out["config"]["recall_per_lane"] = lanes_recall
        out["config"][key_rec] = min([chosen[key_rec]] + lanes_recall)
        roof["timing"] = "%d steps over %d lanes (index + views); achieved = algorithmic bytes of the steps / region time" % (a.steps, n_lanes)
    out.update(extra)
    if misses is not None:
        out["exact_scan_misses_vs_fp32"] = misses
    if build_s is not None:
        out["graph_build_s"] = build_s

    # ---- the reference's CPU path on this box's host cores, searching the SAME CSR (rank 0) ----
    good_graph = [r for r in report if r["mode"] == "graph" and r[key_rec] >= a.recall_target]
    if rank == 0 and not a.no_cpu:
        try:
            graph, L = None, 500
            if good_graph:
                graph = ix.get_graph()
                L = mode[1] if mode[0] == "graph" else good_graph[0]["L"]
                deg = np.diff(graph[1])
                out["graph_stats"] = {"edges": int(graph[1][-1]), "avg_degree": float(deg.mean()), "nav_degree": int(deg[graph[3]]),
                                      "max_degree_other": int(np.delete(deg, graph[3]).max())}
            nqc = min(a.cpu_queries, a.batch) if graph is not None else min(8, a.batch)  # the reference's brute-force branch is slow
            Qc = np.stack([A.Qpool[0][:nqc].cpu().numpy(), A.Qpool[1 % n_pool][:nqc].cpu().numpy()]).astype(np.float32)
            res = run_reference_child(a, graph, L, Qc, timeout=a.cpu_timeout)
            modes_qps = {m: float(x["qps"][-1]) for m, x in res["modes"].items()}
            best_name = max(modes_qps, key=modes_qps.get)
            best = res["modes"][best_name]
            cb = {"value": modes_qps[best_name], "unit": "queries/s", "cores": best["n_exec"] * best["T"], "kind": res["kind"],
                  "sample": "%d queries of a step's batch, %s on the same CSR at L=%d (%d executors x %d threads, %d host cores)" % (
                      nqc, best_name, res["L"], best["n_exec"], best["T"], res["cores"]),
                  "modes": modes_qps}
            if "ids_T1_step0" in res and graph is not None:
                # parity sample: width 1 on the device vs the reference at IntraQueryThreads = 1, same CSR, same L
                ref_ids = np.asarray(res["ids_T1_step0"], np.int64)
                A.set_mode(("graph", L, ""))
                ix.set_search_width(1)
                A.search(A.Qpool[0])
                g1 = A.out_ids.cpu().numpy()[:ref_ids.shape[0]]
                cb["parity_sample"] = {"queries": int(ref_ids.shape[0]),
                                       "ids_identical_width1_vs_reference_T1": float(np.mean(g1 == ref_ids)),
                                       "queries_identical": float(np.mean(np.all(g1 == ref_ids, axis=1)))}
                ix.set_search_width(a.width)
            out["cpu_baseline"] = cb
        except Exception as e:  # the bench line must still print
            out["cpu_baseline"] = {"value": None, "unit": "queries/s", "cores": os.cpu_count(), "kind": "reference",
                                   "sample": "failed: %r" % (e,)}

    # ---- the other tables of SURVEY.md §8d in the same run (N = 1: replicas would only repeat them) ----
    for t in [x.strip() for x in a.extra_tables.split(",") if x.strip()]:
        if t == a.dist or group is not None or world > 1:
            continue
        try:
            A.close()
            torch.cuda.empty_cache()
            au = argparse.Namespace(**vars(a))
            au.dist = t
            A = Arena(au, t, dev, local, rank, world)
            A.ground_truth()
            trep = {"workload": workload_name(au)}
            if t != "uniform" or a.uniform_graph:
                t0 = time.perf_counter()
                A.ix.build(rows, knn_k=a.knn_k, nnd_iters=a.nnd_iters)
                torch.cuda.synchronize()
                trep["graph_build_s"] = time.perf_counter() - t0
                sweep = []
                for L in [int(x) for x in a.L_sweep.split(",")]:
                    if L < 1024 and t == "cluster":  # the navigation point alone has > 1000 out-neighbours there
                        continue
                    gm = ("graph", L, "")
                    A.set_mode(gm)
                    A.search(A.Qpool[0])
                    grec = recall_of(A.truth, A.out_ids, a.k)
                    sweep.append({"L": L, key_rec: grec})
                    if grec >= a.recall_target or L >= 2048:
                        break
                timed_device_steps(gm, a.warmup, 0)
                ms, st = timed_device_steps(gm, min(a.steps, 5), a.warmup)
                k_ms = float(sum(x["kernel_ms"] for x in st))
                ag = {k: float(sum(x[k] for x in st)) for k in ("n_dist", "n_seed", "n_expand", "n_edges")}
                trep["graph"] = {"value": a.batch * len(st) / (ms / 1000.0), "unit": "queries/s", "L": gm[1], "width": a.width,
                                 key_rec: grec, "roofline": graph_roofline(ag, gm[1], k_ms, len(st)), "L_sweep": sweep}
                if a.lanes > 1:  # the same steps with `lanes` batches in flight (see the headline record)
                    A.open_lanes(a.lanes)
                    timed_overlapped(gm, max(a.warmup, a.lanes), 0)
                    ms_o = timed_overlapped(gm, len(st), a.warmup)
                    trep["graph"] = {"value": a.batch * len(st) / (ms_o / 1000.0), "unit": "queries/s", "L": gm[1], "width": a.width,
                                     key_rec: grec, "batches_in_flight": a.lanes, "roofline": graph_roofline(ag, gm[1], ms_o, len(st)),
                                     "one_batch_at_a_time": trep["graph"], "L_sweep": sweep}
                    A.close_lanes()
            m = ("brute", 0, "bf16")
            A.set_mode(m)
            A.search(A.Qpool[0])
            urec = recall_of(A.truth, A.out_ids, a.k)
            umiss = classify_misses(A.truth.cpu().numpy(), A.truth_d.cpu().numpy(), A.out_ids.cpu().numpy(), A.out_d.cpu().numpy(), a.k)
            timed_device_steps(m, a.warmup, 0)
            ms, st = timed_device_steps(m, min(a.steps, 5), a.warmup)
            k_ms = float(sum(x["kernel_ms"] for x in st))
            trep["exact_scan_bf16"] = {"value": a.batch * len(st) / (ms / 1000.0), "unit": "queries/s", key_rec: urec,
                                       "roofline": scan_roofline("bf16", k_ms, len(st)), "misses_vs_fp32": umiss,
                                       "queries_redone_by_guard_per_step": float(np.mean([x["n_redone"] for x in st]))}
            out[t] = trep
        except Exception as e:
            out[t] = {"failed": repr(e)}
    if rank == 0:
        if a.dump_outputs:
            os.makedirs(a.dump_outputs, exist_ok=True)
            for name, arr in last_out.items():
                np.save(os.path.join(a.dump_outputs, name + ".npy"), arr.astype(np.float32 if name == "distances" else np.float64))
        print(json.dumps(out))
    if group is not None:
        group.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
