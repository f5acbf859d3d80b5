"""Developer tool: exact-scan results with the wgmma coarse pass vs the fp32 SIMT path (EPS_NO_TC=1), same data."""
import os, sys, subprocess, json, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

def run(rows, dim, nq, k, metric):
    import torch, vectordb_b200
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev); g.manual_seed(1)
    X = torch.rand((rows, dim), generator=g, device=dev)
    Q = torch.rand((nq, dim), generator=g, device=dev)
    if metric == "cosine":
        X /= X.norm(dim=1, keepdim=True); Q /= Q.norm(dim=1, keepdim=True)
    ix = vectordb_b200.Index(metric, dim, capacity=rows)
    ix.adopt_device_rows(X.data_ptr(), rows)
    ix.config(512, 512, force_brute=True)
    ix.set_coarse(os.environ.get("EPS_COARSE", "tf32"))
    oi = torch.empty((nq, k), dtype=torch.int64, device=dev); od = torch.empty((nq, k), dtype=torch.float32, device=dev)
    oc = torch.empty((nq,), dtype=torch.int64, device=dev)
    for _ in range(2):
        st = ix.search_device(Q.data_ptr(), nq, k, oi.data_ptr(), od.data_ptr(), oc.data_ptr(), want_stats=True)
    return oi.cpu().numpy(), od.cpu().numpy(), st["kernel_ms"]

if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "child":
        rows, dim, nq, k = map(int, sys.argv[2:6]); metric = sys.argv[6]
        ids, ds, ms = run(rows, dim, nq, k, metric)
        np.savez(sys.argv[7], ids=ids, ds=ds, ms=ms)
        sys.exit(0)
    cases = [(300000, 96, 300, 100, "ip"), (1000000, 768, 1024, 10, "l2"), (4000000, 768, 1024, 10, "l2")]
    if len(sys.argv) > 1 and sys.argv[1] == "all":
        cases = [(20000, 64, 256, 10, "l2"), (50000, 768, 1024, 10, "l2"), (33333, 100, 300, 100, "ip"),
                 (40000, 128, 512, 10, "cosine")] + cases
    for c in cases:
        out = {}
        for tag, env in (("tc", {"EPS_COARSE": "tf32"}), ("bf16", {"EPS_COARSE": "bf16"}), ("bf16_2cta", {"EPS_COARSE": "bf16", "EPS_TC_2CTA": "1"}),
                         ("tf32_2cta", {"EPS_COARSE": "tf32", "EPS_TC_2CTA": "1"}), ("simt", {"EPS_COARSE": "fp32"})):
            f = "/tmp/tc_%s.npz" % tag
            e = dict(os.environ); e.update(env)
            r = subprocess.run(["timeout", "90", sys.executable, __file__, "child"] + [str(x) for x in c] + [f], env=e,
                               capture_output=True, text=True)
            if r.returncode != 0:
                print("case", c, tag, "FAILED rc", r.returncode, r.stderr[-300:]); continue
            out[tag] = np.load(f)
        if "simt" not in out:
            continue
        res = {"case": c, "simt_ms": round(float(out["simt"]["ms"]), 3)}
        for t in ("tc", "bf16", "bf16_2cta", "tf32_2cta"):
            if t not in out:
                continue
            res[t + "_ids_equal"] = float((out[t]["ids"] == out["simt"]["ids"]).mean())
            res[t + "_set_recall"] = float(np.mean([len(set(a) & set(b)) / len(b) for a, b in zip(out[t]["ids"], out["simt"]["ids"])]))
            res[t + "_ms"] = round(float(out[t]["ms"]), 3)
        print(json.dumps(res))
