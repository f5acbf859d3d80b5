"""CPU test of the bench contract: `bench.py --impl reference` (the reference's own CPU path through
oracle/_ref, or the C port when that library is absent) prints ONE JSON line with the agreed keys."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reference_arm_prints_contract_line():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--rows", "20000", "--dim", "32",
                          "--batch", "64", "--steps", "2", "--warmup", "1", "--cpu-queries", "16"], capture_output=True,
                         text=True, env=env, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "queries/s" and d["higher_is_better"] is True
    assert d["metric"].startswith("QPS @ recall@10") and d["value"] > 0 and d["steps"] == 2 and d["warmup"] == 1
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"] == {"value": d["value"], "unit": "queries/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
    assert "workload" in d["config"]


def test_synthetic_tables_are_seeded_and_the_manifold_table_has_low_rank():
    """bench.gen_table: same seed -> same bits; the "manifold" table = Gaussian blobs of sigma 0.1 in a 32-d latent
    space embedded in R^d (+ small isotropic noise), i.e. its singular values collapse after the 32nd; the
    "cluster" table is isotropic."""
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    import bench
    dev = torch.device("cpu")
    a = bench.gen_table(3000, 96, "manifold", 42, dev, 16)
    b = bench.gen_table(3000, 96, "manifold", 42, dev, 16)
    assert torch.equal(a, b) and a.dtype == torch.float32 and tuple(a.shape) == (3000, 96)
    s = np.linalg.svd((a - a.mean(0)).numpy(), compute_uv=False)
    assert s[bench.LATENT_DIM - 1] > 10 * s[bench.LATENT_DIM], s[28:36]          # 32 directions carry the blobs
    assert abs(s[-1] / np.sqrt(3000) - bench.LATENT_NOISE * bench.LATENT_SIGMA) < 2e-3  # the rest is the noise floor
    c = bench.gen_table(3000, 96, "cluster", 42, dev, 16)
    sc = np.linalg.svd((c - c.mean(0)).numpy(), compute_uv=False)
    assert sc[40] > 0.5 * sc[20]                                                   # no low-rank structure beyond the 16 centres
    q = bench.gen_queries(8, 96, "manifold", 43, dev, 16)
    assert tuple(q.shape) == (8, 96) and float(torch.cdist(q, a).min(1).values.max()) < 1.5


def test_classify_misses_separates_ties_from_real_losses():
    sys.path.insert(0, ROOT)
    import numpy as np
    import bench
    ti = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9]])
    td = np.array([[0.1, 0.2, 0.3], [0.1, 0.2, 0.3], [0.1, 0.2, 0.3]], np.float32)
    gi = np.array([[1, 2, 3], [4, 5, 60], [7, 8, 90]])
    gd = np.array([[0.1, 0.2, 0.3], [0.1, 0.2, 0.3], [0.1, 0.2, 0.35]], np.float32)  # q1: same distance (tie), q2: worse
    assert bench.classify_misses(ti, td, gi, gd, 3) == {"ties": 1, "real": 1}


def test_reference_arm_under_torchrun_prints_once():
    """N > 1: the reference arm is launched with torchrun like the GPU arm; rank 0 alone runs and prints the
    line, the other ranks exit 0 without work."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                          "--master-port", "29577", os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--rows", "20000",
                          "--dim", "32", "--batch", "64", "--steps", "2", "--warmup", "1", "--cpu-queries", "16"],
                         capture_output=True, text=True, env=env, timeout=900)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.splitlines() if l.startswith("{")]
    assert len(lines) == 1, out.stdout[-2000:]
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 2 and d["value"] > 0
