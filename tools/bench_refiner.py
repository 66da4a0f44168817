"""Refiner inference cost on the device: epb_refiner_forward (refiner.model.Refiner, one call per
8192 rows) against the training engine's eval forward (LinearModelPG.eval()) at N = 1, 64, 4096 and
1e5 rows (linear_size 1024, 45 -> 45), as device-event times and rows/s, with the libepb launches
of one call at N = 1; the refiner's evaluate of 1e5 poses: the reference-style numpy loop
(oracle compute_similarity_transform per sample) against epb_pose_errors; the time TEST.REFINER adds
to a 1e5-sample evaluation; RefinedPosePredictor against PosePredictor at N = 1 and 32.  The card name, power
limit and max SM clock are read in the same run; one JSON line per number.

    python tools/bench_refiner.py
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "epipolarpose_b200"))
from epipolarpose_b200 import ops  # noqa: E402
from oracle import restate_refiner as rr  # noqa: E402
from refiner import data as rdata, model as rmodel  # noqa: E402
from tests import refiner_cases as rc  # noqa: E402  (input synthesis and the numpy restatement)

dev = torch.device("cuda:0")
ops.device_check()


def emit(**kw):
    print(json.dumps(kw), flush=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn, reps):
    """Median device-event time (ms) of fn() over reps calls, after 3 warm-up calls."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


emit(card=card(), torch_device=torch.cuda.get_device_name())
sd = rr.init_state(rr.param_shapes(1024, 45, 45), 23)
model = rmodel.LinearModelPG(linear_size=1024, p_dropout=0.5, input_size=45, output_size=45)
model.load_state_dict(sd)
model = model.to(dev).eval()
ref = rmodel.Refiner(model, None)

for N in (1, 64, 4096, 100000):
    x = torch.randn((N, 45), device=dev)
    out = torch.empty((N, 45), device=dev)
    reps = 200 if N <= 4096 else 20
    t_k = timed(lambda: ref.forward(x, out=out, normalize=False, denormalize=False), reps)
    with torch.no_grad():
        t_e = timed(lambda: model(x), reps if N <= 4096 else 5)
    row = dict(what="refiner_forward", N=N, kernel_ms=t_k, kernel_rows_per_s=N / t_k * 1e3,
               eval_engine_ms=t_e, eval_engine_rows_per_s=N / t_e * 1e3)
    if N == 1:
        l0 = ops.launches
        ref.forward(x, out=out, normalize=False, denormalize=False)
        l1 = ops.launches
        with torch.no_grad():
            model(x)
        row.update(kernel_launches=l1 - l0, eval_engine_libepb_launches=ops.launches - l1)
    emit(**row)

# graph replay of the refiner alone at N = 1 and 32 (what a per-frame refinement costs)
for N in (1, 32):
    xs = torch.randn((N, 45), device=dev)
    out = torch.empty((N, 45), device=dev)
    ref.forward(xs, out=out)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ref.forward(xs, out=out)
    emit(what="refiner_graph_replay", N=N, ms=timed(g.replay, 500))

# evaluate of 1e5 refined poses: numpy per-sample loop against the device kernel
S = 100000
rng = np.random.default_rng(1)
gt = rc.poses(rng, S, 15)
pred = gt + rng.normal(0, 30, gt.shape)
rdata.pose_errors(pred[:10], gt[:10])
torch.cuda.synchronize()
t0 = time.perf_counter()
m_dev, _ = rdata.pose_errors(pred, gt)
t_dev = time.perf_counter() - t0
n_host = 10000
t0 = time.perf_counter()
m_host, _ = rc.pose_errors(pred[:n_host], gt[:n_host])
t_host = (time.perf_counter() - t0) * S / n_host
emit(what="pose_errors", S=S, device_s_host_to_host=t_dev, numpy_s_extrapolated_from=n_host, numpy_s=t_host,
     max_diff_mm=float(np.max(np.abs(m_dev[:n_host] - m_host))))

# what TEST.REFINER adds to a 1e5-sample H36M evaluation: refine the pred column, score against gt
import pickle  # noqa: E402
import tempfile  # noqa: E402
from lib.core import refine  # noqa: E402
with tempfile.TemporaryDirectory() as tmp:
    ck, nm = os.path.join(tmp, "r.pth.tar"), os.path.join(tmp, "norm.pkl")
    torch.save({"state_dict": sd}, ck)
    with open(nm, "wb") as f:
        pickle.dump((np.zeros(45, np.float32), np.full(45, 100, np.float32), np.zeros(45, np.float32),
                     np.full(45, 100, np.float32)), f)
    poses = np.zeros((S, 16, 9))
    poses[:, :, 0:3] = np.insert(pred, 6, 0.0, axis=1)
    poses[:, :, 6:9] = np.insert(gt, 6, 0.0, axis=1)
    refine.h36m_refined(poses[:100], ck, nm)             # loads the refiner once, as evaluate does
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    refine.h36m_refined(poses, ck, nm)
    emit(what="test_refiner_cost", S=S, s_host_to_host=time.perf_counter() - t0)

# RefinedPosePredictor against PosePredictor (R50, J16, D64, 256x256 images, random init)
from lib.core.inference import PosePredictor, RefinedPosePredictor  # noqa: E402
from tests import golden_inputs as gi  # noqa: E402
from tests.golden_inputs import _model  # noqa: E402
net = _model(dev, gi.SIZE_CASES["c1"], "f16x3", train=False)
rp = RefinedPosePredictor(net, model, None, flip_test=False)
pp = PosePredictor(net, flip_test=False)
for N in (1, 32):
    x = np.random.default_rng(N).standard_normal((N, 3, 256, 256)).astype(np.float32)
    boxes = {"center_x": np.full(N, 500.0), "center_y": np.full(N, 500.0), "width": np.full(N, 400.0),
             "height": np.full(N, 400.0)}
    cams = {"fl": np.full((N, 2), 1150.0), "c_p": np.full((N, 2), 512.0), "depth": np.full(N, 4500.0)}
    row = dict(what="refined_predictor", N=N)
    for name, fn in (("refined_predictor", lambda: rp(x, boxes, cams)), ("pose_predictor", lambda: pp(x, boxes=boxes))):
        fn()
        ts = []
        for _ in range(50):
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        row[name + "_ms"] = float(np.median(ts) * 1e3)
    row["refined_graph_replay_ms"] = timed(rp.graphs[(N, 256, 256)]["graph"].replay, 100)
    row["pose_graph_replay_ms"] = timed(pp.graphs[(N, 256, 256)]["graph"].replay, 100)
    emit(**row)
