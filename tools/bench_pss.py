"""Pose Structure Score cost on the device (csrc/pss.cu): k-means fit time (10 restarts of
k-means++ and Lloyd) at k = 50, 100 on 1e5 and 1.5e6 synthetic skeleton-like poses (d = 51),
assignment throughput, the cost PSS adds to H36M evaluation of 1e5 samples, and scikit-learn's
KMeans on the host cores as a CPU baseline when it is importable.  One JSON line per number; the
card name and power limit are read in the same run.  The algorithmic work of one Lloyd pass is
3*N*k*d float64 operations (difference, square, add per coordinate).

    python tools/bench_pss.py
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "epipolarpose_b200"))
from epipolarpose_b200 import ops  # noqa: E402
from tests.pss_cases import skeleton_poses  # noqa: E402  (input synthesis only)

dev = torch.device("cuda:0")
ops.device_check()


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


emit(card=card(), torch_device=torch.cuda.get_device_name())


def fit(x, k, n_init=10, max_iter=300):
    """fit_pose_clusters' loop, timed, with the updates of each restart."""
    N, d = x.shape
    ws = torch.empty(ops.kmeans_workspace(N, d, k), dtype=torch.uint8, device=dev)
    cen = torch.empty(k, d, dtype=torch.float64, device=dev)
    lab = torch.empty(N, dtype=torch.int32, device=dev)
    idx = torch.empty(k, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    iters = []
    for r in range(n_init):
        _, n = ops.kmeans_fit(x, N, d, k, 0, r, max_iter, cen, lab, idx, None, ws)
        iters.append(n)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, iters


d = 51
data = {}
for N in (100_000, 1_500_000):
    xn = skeleton_poses(np.random.default_rng(N), N, d // 3, k_true=64)
    data[N] = xn
    x = torch.from_numpy(xn).to(dev)
    fit(x, 3, n_init=1, max_iter=2)                                       # module load, smem attributes
    for k in (50, 100):
        t, iters = fit(x, k)
        passes = sum(iters) + 10                                          # assignment passes incl. pass 0
        flops = 3.0 * N * k * d * passes
        emit(measure="kmeans_fit", N=N, k=k, d=d, n_init=10, seconds=round(t, 4), updates=iters,
             lloyd_gflop=round(flops / 1e9, 1), gflops=round(flops / t / 1e9, 1))

# assignment throughput (includes the finiteness check and its 4-byte read-back)
N, k = 1_500_000, 100
x = torch.from_numpy(data[N]).to(dev)
c = x[torch.randperm(N, generator=torch.Generator().manual_seed(0))[:k].to(dev)].contiguous()
lab = torch.empty(N, dtype=torch.int32, device=dev)
d2 = torch.empty(N, dtype=torch.float64, device=dev)
for _ in range(2):
    ops.kmeans_assign(x, N, d, c, k, lab, d2)
ts = []
for _ in range(9):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ops.kmeans_assign(x, N, d, c, k, lab, d2)
    e1.record()
    torch.cuda.synchronize()
    ts.append(e0.elapsed_time(e1) * 1e-3)
t = sorted(ts)[len(ts) // 2]
emit(measure="kmeans_assign", N=N, k=k, d=d, ms=round(t * 1e3, 3), points_per_s=round(N / t, 1),
     gflops=round(3.0 * N * k * d / t / 1e9, 1))

# added cost inside evaluation: 1e5 samples, 17 joints, centroids given (fitting is once per process)
from lib.dataset.h36m_eval import evaluate_h36m  # noqa: E402
from lib.core.pss import h36m_pss  # noqa: E402
S, J = 100_000, 17
rng = np.random.default_rng(3)
gt = np.concatenate([rng.uniform(100, 900, (S, J, 2)), rng.normal(0, 300, (S, J, 1))], axis=2)
gt[:, 0, 2] = 0
pred = gt + rng.normal(0, 20, gt.shape)
pelvis = np.stack([np.zeros(S), np.zeros(S), rng.uniform(3000, 6000, S)], 1)
fl = rng.uniform(1100, 1200, (S, 2))
c_p = rng.uniform(480, 540, (S, 2))
with tempfile.TemporaryDirectory() as tmp:
    cf = os.path.join(tmp, "c.npz")
    np.savez(cf, k50=data[100_000][:50], k100=data[100_000][:100])

    def timed(fn, reps=5):
        fn()
        ts = []
        for _ in range(reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
        return sorted(ts)[len(ts) // 2]
    t_eval = timed(lambda: evaluate_h36m(pred, gt, pelvis, fl, c_p))
    t_pss = timed(lambda: h36m_pss(pred, gt, pelvis, fl, c_p, False, [50, 100], "", cf))
emit(measure="evaluate_h36m", S=S, ms=round(t_eval * 1e3, 2))
emit(measure="pss_added", S=S, ks=[50, 100], ms=round(t_pss * 1e3, 2),
     note="host-to-device copies, normalisation and two assignments per k; fitting excluded")

try:
    from sklearn.cluster import KMeans
except ImportError:
    KMeans = None
if KMeans is None:
    emit(measure="sklearn_kmeans", skipped="scikit-learn not importable")
else:
    for k in (50, 100):
        t0 = time.perf_counter()
        km = KMeans(n_clusters=k, n_init=10, algorithm="lloyd", max_iter=300, tol=0, random_state=0)
        km.fit(data[100_000])
        emit(measure="sklearn_kmeans", N=100_000, k=k, d=d, n_init=10, host_cores=os.cpu_count(),
             seconds=round(time.perf_counter() - t0, 3))
