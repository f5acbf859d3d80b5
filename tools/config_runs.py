"""Runs the BASELINE.json configs as they are stated and prints ONE JSON line per run (kept under profiles/).

  C1  brute-force L2 top-10, 10k x 128, batch = 1 (host-buffer call per query) next to the reference CPU path
  C2  1M x 768 cosine, graph index, batch = 1024, top-10
  C3  10M x 768 L2, graph index, batch = 4096, top-100 + metadata filter (attr = row % 100, "ID < 10", post-filter)
  C4  5M x 1536 IP, index build + search (batch 1024, top-10; 31 GB of rows on an 80 GB H100)
  C5  100M x 768 L2 sharded across 8 GPUs (12.5M rows per rank, own graph per shard), batch = 8192, top-10,
      NCCL candidate all-gather inside the library — launch with torchrun --nproc-per-node 8

Every graph run sweeps L up to the first recall >= 0.99 against the fp32 exact scan, reports QPS, distance
evaluations per query and the HBM-roofline fraction of graph_search_kernel (SURVEY.md §8d bytes), times the exact scan
beside it, and — through bench.run_reference_child — searches THE SAME CSR with the reference's own executor on the
host cores (throughput modes + an ids-identical sample at IntraQueryThreads = 1 / search width 1).

Usage: python tools/config_runs.py c1|c2|c3|c4|c5 [--rows N] [--dist cluster|uniform] [--width W] [--no-cpu]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

P = argparse.ArgumentParser()
P.add_argument("which", choices=["c1", "c2", "c3", "c4", "c5"])
P.add_argument("--rows", type=int, default=0)
P.add_argument("--dist", default="manifold", choices=["manifold", "cluster", "uniform"])
P.add_argument("--centers", type=int, default=1024)
P.add_argument("--width", type=int, default=8)
P.add_argument("--ring", type=int, default=0)
P.add_argument("--ctas", type=int, default=0)
P.add_argument("--L-sweep", default="128,192,256,384,512,768,1024,1536,2048,3072,4096")
P.add_argument("--nnd-iters", type=int, default=14)
P.add_argument("--no-cpu", action="store_true")
P.add_argument("--cpu-timeout", type=int, default=600)
A = P.parse_args()


def c1():
    import vectordb_b200
    from oracle.oracle import Ref
    rows, dim, k = 10_000, 128, 10
    rng = np.random.default_rng(42)
    X = rng.random((rows, dim), dtype=np.float32)
    Q = rng.random((512, dim), dtype=np.float32)
    ix = vectordb_b200.Index("l2", dim, host_vectors=X)
    ix.sync_rows(rows)
    for q in Q[:32]:
        ix.search(q, k, want_stats=False)
    t0 = time.perf_counter()
    got = [ix.search(q, k, want_stats=False)[0][0] for q in Q]
    gpu_qps = len(Q) / (time.perf_counter() - t0)
    out = {"config": "C1 10000x128 L2 brute force, batch=1, top-10 (one eps_search_batch call per query, host buffers)",
           "gpu_qps_sequential_calls": gpu_qps, "gpu_latency_us": 1e6 / gpu_qps}
    try:
        r = Ref("l2", dim, rows, [("ID", "int4")])
        r.set_rows(X)
        for T in (1, 8):
            r.make_executors(1, T, 500)
            for q in Q[:8]:
                r.search(q, k)
            t0 = time.perf_counter()
            ref = [r.search(q, k)[0] for q in Q]
            out["reference_cpu_qps_T%d" % T] = len(Q) / (time.perf_counter() - t0)
        out["ids_identical"] = float(np.mean([np.array_equal(a, b) for a, b in zip(got, ref)]))
    except Exception as e:
        out["reference"] = "unavailable: %r" % (e,)
    print(json.dumps(out))


def graph_config(name, rows, dim, metric, nq, k, filt=None, local=0, rank=0, world=1, group=None):
    """Shared body of C2-C5.  filt = (filter string for the reference parser, POD nodes for the C ABI, attr modulus)."""
    import torch
    import vectordb_b200
    dev = torch.device("cuda", local)
    hbm_peak, tf_peak, peak_src = bench.measured_peaks()
    ns = argparse.Namespace(rows=rows, dim=dim, dist=A.dist, centers=A.centers, metric=metric, k=k, batch=nq)
    X = bench.gen_table(rows, dim, A.dist, 42 + rank, dev, A.centers)
    Q = bench.gen_queries(nq, dim, A.dist, 43, dev, A.centers)
    if metric == "cosine":
        X /= X.norm(dim=1, keepdim=True)
        Q /= Q.norm(dim=1, keepdim=True)
    ix = vectordb_b200.Index(metric, dim, capacity=rows, device=local)
    ix.adopt_device_rows(X.data_ptr(), rows)
    torch.cuda.synchronize()  # generators done before the library stream reads
    nodes = None
    if filt:
        attr = (np.arange(rows) % filt[2]).astype(np.int32)
        ix.set_attrs(attr.view(np.uint8), 4, rows)
        nodes = filt[1]
    oi = torch.empty((nq, k), dtype=torch.int64, device=dev)
    od = torch.empty((nq, k), dtype=torch.float32, device=dev)
    oc = torch.empty((nq,), dtype=torch.int64, device=dev)

    def search(stats=True):
        return ix.search_device(Q.data_ptr(), nq, k, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), filter_nodes=nodes, want_stats=stats)

    def timed(reps=3):
        search()
        torch.cuda.synchronize()
        ms, st = 0.0, None
        for _ in range(reps):
            st = search()
            ms += st["total_ms"]
        return ms / reps, st

    out = {"config": "%s %s, rank %d of %d" % (name, bench.workload_name(ns), rank, world)}
    # exact ground truth: fp32 SIMT scan of the (filtered) table — for a filter, the prefilter branch semantics
    ix.config(512, 512, force_brute=True)
    ix.set_coarse("fp32")
    search(False)
    truth, truth_d = oi.cpu().numpy().copy(), od.cpu().numpy().copy()
    truth_c = oc.cpu().numpy().copy()
    rec = lambda g: float(np.mean([len(set(g[i][g[i] >= 0].tolist()) & set(truth[i][:truth_c[i]].tolist())) / max(1, truth_c[i])
                                   for i in range(nq)]))
    ix.set_coarse("bf16")
    ms, st = timed()
    g = oi.cpu().numpy()
    out["exact_scan_bf16"] = {"qps": nq / (ms / 1e3), "ms_per_batch": ms, "recall": rec(g),
                              "misses_vs_fp32": bench.classify_misses(truth, truth_d, g, od.cpu().numpy(), k) if not filt else None,
                              "tensor_TFLOPs": 2.0 * rows * nq * dim / (st["kernel_ms"] / 1e3) / 1e12}
    t0 = time.perf_counter()
    ix.build(rows, knn_k=64, nnd_iters=A.nnd_iters)
    torch.cuda.synchronize()
    out["graph_build_s"] = time.perf_counter() - t0
    n, off, nb, nav = ix.get_graph()
    deg = np.diff(off)
    out["graph"] = {"edges": int(off[-1]), "avg_degree": float(deg.mean()), "max_degree": int(deg.max())}
    ix.set_search_width(A.width)
    ix.set_graph_tuning(A.ring, A.ctas)
    sweep, chosen = [], None
    for L in [int(x) for x in A.L_sweep.split(",")]:
        if L < k or L > rows:
            continue
        ix.config(L, L)
        ms, st = timed()
        g = oi.cpu().numpy()
        byt = (st["n_dist"] - st["n_seed"]) * dim * 4.0 + st["n_edges"] * 4.0 + st["n_expand"] * 16.0 + L * dim * 4.0 + nq * (dim * 4.0 + k * 12.0)
        r = {"L": L, "recall": rec(g), "qps": nq / (ms / 1e3), "ms_per_batch": ms, "kernel_ms": st["kernel_ms"],
             "n_dist_per_query": st["n_dist"] / nq, "mean_results": float(oc.cpu().numpy().mean()),
             "hbm_GBps": byt / (st["kernel_ms"] / 1e3) / 1e9, "hbm_frac_of_%s_peak" % peak_src: byt / (st["kernel_ms"] / 1e3) / 1e9 / hbm_peak}
        if filt:
            r["all_pass_filter"] = bool(np.all(attr[g[g >= 0]] < 10))
        sweep.append(r)
        if r["recall"] >= 0.99:
            chosen = r
            break
    out["graph_sweep"] = sweep
    out["graph_operating_point"] = chosen
    if chosen is not None and group is None:
        # the same batch with two batches in flight (the index + one read-only view, see bench.py --lanes)
        v = ix.view()
        lanes = [(ix, oi, od, oc), (v, torch.empty_like(oi), torch.empty_like(od), torch.empty_like(oc))]
        streams = [torch.cuda.ExternalStream(h.stream, device=dev) for h, _, _, _ in lanes]

        def region(n_steps):
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True)
            e0.record(streams[0])
            streams[1].wait_event(e0)
            for s in range(n_steps):
                h, a_i, a_d, a_c = lanes[s % 2]
                h.search_device(Q.data_ptr(), nq, k, a_i.data_ptr(), a_d.data_ptr(), a_c.data_ptr(), filter_nodes=nodes, sync=False)
            ends = []
            for st_ in streams:
                e = torch.cuda.Event(enable_timing=True)
                e.record(st_)
                ends.append(e)
            torch.cuda.synchronize()
            return max(e0.elapsed_time(e) for e in ends) / n_steps
        region(4)
        ms2 = region(8)
        byt = chosen["hbm_GBps"] * 1e9 * chosen["kernel_ms"] / 1e3
        chosen["two_batches_in_flight"] = {"qps": nq / (ms2 / 1e3), "ms_per_batch": ms2, "hbm_GBps": byt / (ms2 / 1e3) / 1e9,
                                           "hbm_frac": byt / (ms2 / 1e3) / 1e9 / hbm_peak,
                                           "view_ids_identical_to_base_sample": bool(np.array_equal(lanes[1][1].cpu().numpy()[:8] >= 0, oi.cpu().numpy()[:8] >= 0))}
        v.close()
    if group is not None:  # C5: the sharded search with the in-library exchange, merged recall against merged truth
        import torch.distributed as dist
        L = (chosen or sweep[-1])["L"]
        ix.config(L, L)
        mi = torch.empty((nq, k), dtype=torch.int64, device=dev)
        md = torch.empty((nq, k), dtype=torch.float32, device=dev)
        group.search(ix, rank * rows, Q.data_ptr(), nq, k, mi.data_ptr(), md.data_ptr())
        stream = torch.cuda.ExternalStream(ix.stream, device=dev)
        torch.cuda.synchronize(); dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(3):
            group.search(ix, rank * rows, Q.data_ptr(), nq, k, mi.data_ptr(), md.data_ptr())
        e1.record(stream)
        torch.cuda.synchronize(); dist.barrier()
        t = torch.tensor([e0.elapsed_time(e1) / 3], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        # merged exact truth: all-gather the per-shard fp32 truths and merge on the host
        ti = torch.from_numpy(truth + rank * rows).to(dev)
        td = torch.from_numpy(truth_d).to(dev)
        all_i = [torch.empty_like(ti) for _ in range(world)]
        all_d = [torch.empty_like(td) for _ in range(world)]
        dist.all_gather(all_i, ti); dist.all_gather(all_d, td)
        from vectordb_b200.sharded import numpy_merge
        wi, _ = numpy_merge(np.stack([x.cpu().numpy() for x in all_i]), np.stack([x.cpu().numpy() for x in all_d]), k)
        gi = mi.cpu().numpy()
        out["sharded"] = {"L": L, "qps": nq / (float(t.item()) / 1e3), "ms_per_batch_max_over_ranks": float(t.item()),
                          "merged_recall": float(np.mean([len(set(gi[i].tolist()) & set(wi[i].tolist())) / k for i in range(nq)]))}
    if not A.no_cpu and rank == 0 and chosen is not None:
        try:
            nqc = min(128, nq)
            Qc = np.stack([Q[:nqc].cpu().numpy()] * 2).astype(np.float32)
            ns2 = argparse.Namespace(**vars(ns))
            res = bench.run_reference_child(ns2, (n, off, nb, nav), chosen["L"], Qc, timeout=A.cpu_timeout,
                                            filter_str=filt[0] if filt else "", attr_mod=filt[2] if filt else 0, seed_shift=rank)
            cpu = {m: float(x["qps"][-1]) for m, x in res["modes"].items()}
            cpu["cores"] = res["cores"]
            if "ids_T1_step0" in res:
                ix.config(chosen["L"], chosen["L"])
                ix.set_search_width(1)
                search(False)
                ref_ids = np.asarray(res["ids_T1_step0"], np.int64)
                g1 = oi.cpu().numpy()[:ref_ids.shape[0]]
                cpu["ids_identical_width1_vs_reference_T1"] = float(np.mean(g1 == ref_ids))
                cpu["queries_identical"] = float(np.mean(np.all(g1 == ref_ids, axis=1)))
            out["reference_cpu_same_csr"] = cpu
        except Exception as e:
            out["reference_cpu_same_csr"] = "failed: %r" % (e,)
    return out


def main():
    which = A.which
    if which == "c1":
        c1()
        return
    import torch
    if which == "c2":
        print(json.dumps(graph_config("C2", A.rows or 1_000_000, 768, "cosine", 1024, 10)))
    elif which == "c3":
        nodes = np.array([[7, 1, -1, -1, 0, 0, 0, 0], [1, 1, -1, -1, 10, 0, 0, -1], [19, 3, 0, 1, 0, 0, 0, -1]], np.int64)  # Int4Attr@0 < 10
        print(json.dumps(graph_config("C3", A.rows or 10_000_000, 768, "l2", 4096, 100, filt=("ID < 10", nodes, 100))))
    elif which == "c4":
        print(json.dumps(graph_config("C4", A.rows or 5_000_000, 1536, "ip", 1024, 10)))
    else:
        import torch.distributed as dist
        from vectordb_b200.sharded import ShardGroup
        world = int(os.environ.get("WORLD_SIZE", "1"))
        rank = int(os.environ.get("RANK", "0"))
        local = int(os.environ.get("LOCAL_RANK", "0"))
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        uid = [ShardGroup.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        group = ShardGroup(uid[0], rank, world, local)
        out = graph_config("C5", A.rows or 100_000_000 // max(world, 1), 768, "l2", 8192, 10, local=local, rank=rank, world=world, group=group)
        if rank == 0:
            print(json.dumps(out))
        group.close()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
