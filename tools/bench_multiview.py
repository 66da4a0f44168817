"""Latency of multi-view inference: MultiViewPredictor (PoseResNet-50, J 17, D 64, 256x256 images,
random init, split-fp16 engine) against what a user had to do without it, and the robust
triangulation kernel on its own.

    python tools/bench_multiview.py [--shapes 1x4,8x4,32x4,1x8] [--reps 100]

Prints ONE JSON line with the GPU name, its power limit and max SM clock (read in the same run,
before and after) and, per (T, V):
  multiview    host clock around mv(images, boxes, P): HOST images in, numpy out, one graph replay
  replay       device events around that graph replay alone
  single_view  device events around the PosePredictor graph of the same T*V images: what the
               geometry adds inside the graph is replay - single_view
  composed_numpy   host clock around PosePredictor(images, boxes) + the numpy restatement of the
               triangulation on its 2-D output (tests/multiview_cases.py)
  composed_device  host clock around PosePredictor(images, boxes) + one eager epb_triangulate_robust
               on its 2-D output (host -> device -> host)
(median and p90 in ms; the host-clocked variants alternate in one loop; reps = max(20, reps / T)),
and for the kernel alone, at V = 4 and 8 and NT*J = 17, 17*64 and 2^20 joints (3 px noise, one
80 px outlier per joint): microseconds per launch from device events around 20 back-to-back
launches, median over 15 rounds.  Needs a GPU: there is no CPU timing."""
import argparse
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
from oracle import refshim, restate  # noqa: E402
from epipolarpose_b200 import ops  # noqa: E402
import lib.models as models  # noqa: E402
import lib.utils.triangulation as tri  # noqa: E402
from lib.core.inference import MultiViewPredictor, PosePredictor  # noqa: E402
from tests import multiview_cases as mc  # noqa: E402

J, D, HW = 17, 64, 256
THR = 15.0


def stats(ts, scale=1e3):
    a = np.asarray(ts) * scale
    return {"median_ms": float(np.median(a)), "p90_ms": float(np.percentile(a, 90)), "n": len(a)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl, clk = [v.strip() for v in q.stdout.strip().split(",")] if q.returncode == 0 else ("?", "?", "?")
    return {"gpu": torch.cuda.get_device_name(0), "smi_name": name, "power_limit_w": pl,
            "max_sm_clock_mhz": clk}


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def replay_times(graph, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ts = []
    for _ in range(reps):
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    return ts


def shape_row(model, T, V, reps):
    rng = np.random.default_rng(10 * T + V)
    _, _, _, _, P = restate.synthetic_cameras(rng, T, V)
    x = rng.standard_normal((T, V, 3, HW, HW)).astype(np.float32)
    n = T * V
    boxes = {"center_x": 512 + rng.uniform(-20, 20, n), "center_y": 515 + rng.uniform(-20, 20, n),
             "width": rng.uniform(150, 400, n), "height": rng.uniform(150, 400, n)}
    mv = MultiViewPredictor(model, flip_test=False, threshold_px=THR)
    pp = PosePredictor(model, flip_test=False)
    xf = x.reshape(n, 3, HW, HW)

    def composed_numpy():
        k = pp(xf, boxes=boxes).reshape(T, V, J, 4)
        return [mc.robust_nview_triangulation(k[t], P[t], None, THR) for t in range(T)]

    def composed_device():
        k = torch.from_numpy(pp(xf, boxes=boxes).reshape(T, V, J, 4)).cuda()
        return [o.cpu() for o in tri.triangulate_views_robust(k, torch.from_numpy(P).cuda(), None, THR)]

    fns = {"multiview": lambda: mv(x, boxes, P), "composed_numpy": composed_numpy,
           "composed_device": composed_device}
    for _ in range(3):
        for f in fns.values():
            f()
    r = max(20, reps // T)
    ts = {k: [] for k in fns}
    for _ in range(r):                              # alternate the variants in one loop
        for k, f in fns.items():
            ts[k].append(clock(f))
    row = {"T": T, "V": V, "reps": r}
    row.update({k: stats(v) for k, v in ts.items()})
    a, b = [], []
    for _ in range(3):                              # alternate the two graphs in blocks
        a += replay_times(mv.graphs[(T, V, HW, HW)]["graph"], r)
        b += replay_times(pp.graphs[(n, HW, HW)]["graph"], r)
    row["replay"], row["single_view"] = stats(a), stats(b)
    row["geometry_in_graph_ms"] = row["replay"]["median_ms"] - row["single_view"]["median_ms"]
    out = mv(x, boxes, P)
    row["status_share"] = float(out["status"].mean())
    return row


CALLS, ROUNDS = 20, 15


def kernel_row(V, NT, Jk):
    P, X, ue, un = mc.rig(V + NT % 11, min(NT, 256), V, Jk)
    uo, _ = mc.plant_outliers(un, V)
    k = (NT + len(P) - 1) // len(P)
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(np.tile(a, (k,) + (1,) * (a.ndim - 1))[:NT])).cuda()
    u, Pd = t64(uo), t64(P)
    out = tri.triangulate_views_robust(u, Pd, None, THR)
    torch.cuda.synchronize()
    ts = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(CALLS):
            tri.triangulate_views_robust(u, Pd, None, THR, out=out)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / CALLS)
    return {"V": V, "NT": NT, "J": Jk, "joints": NT * Jk, "us_per_launch_median": float(np.median(ts)),
            "us_per_launch_p90": float(np.percentile(ts, 90)), "status_share": float(out[1].double().mean())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1x4,8x4,32x4,1x8")
    ap.add_argument("--reps", type=int, default=100)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiview needs a GPU: a latency measured elsewhere says nothing about it")
    ops.device_check()
    res = gpu_info()
    torch.manual_seed(0)
    cfg = refshim.make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    model = models.pose3d_resnet.get_pose_net(cfg, False).cuda().eval()
    res["latency"] = [shape_row(model, *[int(v) for v in s.split("x")], args.reps) for s in args.shapes.split(",")]
    res["kernel"] = [kernel_row(V, NT, Jk) for V in (4, 8) for NT, Jk in ((1, 17), (64, 17), (65536, 16))]
    res.update({k + "_after": v for k, v in gpu_info().items() if k in ("power_limit_w", "max_sm_clock_mhz")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
