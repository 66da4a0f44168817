"""Inference latency of PoseResNet-50 (J 16, D 64, 256x256 images) on the split-fp16 engine:
eager `model.eval()(x)` + get_joint_location_result against PosePredictor (one CUDA-graph replay,
split-K convs), per batch size, and a per-layer table of the split-K entry.

    python tools/bench_infer.py [--sizes 1,2,4,8,32] [--reps 200] [--layer-sizes 1,32]

Prints ONE JSON line with the GPU name, its power limit and max SM clock (read in the same run)
and, per N:
  eager      host clock around model(x) on a device batch + get_joint_location_result (it ends in
             a device-to-host copy, so the call is synchronised), after warm-up
  predictor  host clock around pred(images) with HOST images in and numpy out
  replay     device events around the graph replay alone
  s1         the predictor with the split planner patched to S = 1 (a tool-side patch, like
             tools/conv_table.py): what the graph alone gives, without split-K
(median and p90 in ms, images/s from the predictor median; reps = max(30, reps / N)), and the
largest coordinate difference predictor vs eager.  The layer table gives, for each distinct
conv16 shape of the predictor's forward at N in --layer-sizes: calls per forward, tiles, K/64, the
planner's S, and the median time per call (CUDA events, alternating) at S = 1, at the planner's
S and at the other powers of two up to K/64 -- each from a CUDA graph of 20 back-to-back calls, so the
time is the device's, not the host's launch cost."""
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
from oracle import refshim  # noqa: E402
from epipolarpose_b200 import ops  # noqa: E402
import lib.models as models  # noqa: E402
import lib.core.integral_loss as il  # noqa: E402
from lib.core.inference import PosePredictor  # noqa: E402
from tests import emul_splitk as es  # noqa: E402

J, D, HW = 16, 64, 256


def stats(ts):
    a = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(a)), "p90_ms": float(np.percentile(a, 90)), "n": len(a)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl, clk = [v.strip() for v in q.stdout.strip().split(",")] if q.returncode == 0 else ("?", "?", "?")
    return {"gpu": torch.cuda.get_device_name(0), "smi_name": name, "power_limit_w": pl,
            "max_sm_clock_mhz": clk}


def host_times(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return ts


def latency_rows(model, sizes, reps):
    pred = PosePredictor(model, flip_test=False)
    planner = ops.conv16_splits
    ops.conv16_splits = lambda g: (1, 0)          # graphs captured under the patch never split
    try:
        pred1 = PosePredictor(model, flip_test=False)
        for N in sizes:
            pred1(np.zeros((N, 3, HW, HW), np.float32))
    finally:
        ops.conv16_splits = planner
    rows = []
    for N in sizes:
        r = max(30, reps // N)
        g = torch.Generator().manual_seed(N)
        xh = torch.randn(N, 3, HW, HW, generator=g)
        xd = xh.cuda()

        def eager():
            with torch.no_grad():
                return il.get_joint_location_result(HW, HW, model(xd))

        for _ in range(5):
            eager()
            pred(xh)
            pred1(xh)
        d = float(np.abs(pred(xh) - eager()).max())
        te, tp, t1 = [], [], []
        for _ in range(r):                         # alternate the three in one loop
            te += host_times(eager, 1)
            tp += host_times(lambda: pred(xh), 1)
            t1 += host_times(lambda: pred1(xh), 1)
        ent = pred.graphs[(N, HW, HW)]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        tr = []
        for _ in range(r):
            e0.record()
            ent["graph"].replay()
            e1.record()
            torch.cuda.synchronize()
            tr.append(e0.elapsed_time(e1) * 1e-3)
        row = {"N": N, "eager": stats(te), "predictor": stats(tp), "replay": stats(tr), "s1": stats(t1),
               "max_abs_diff_vs_eager": d}
        for k in ("eager", "predictor", "s1"):
            row[k]["images_per_s"] = N / (row[k]["median_ms"] * 1e-3)
        rows.append(row)
    return rows


CALLS = 20


def layer_table(model, N, reps=15):
    """Distinct conv16 calls of the predictor's forward at batch N, each timed at several S."""
    pred = PosePredictor(model, flip_test=False)
    rec, orig = {}, ops.conv16_fprop_splitk

    def record(g, *a):
        key = (g.N * g.Hp * g.Wp, g.Cin, g.Cout, g.T, g.os, g.is_)
        if key in rec:
            rec[key]["calls"] += 1
        else:
            a = list(a)
            a[6] = None if a[6] is None else a[6].clone()     # stats: keep the forward's untouched
            rec[key] = {"g": g, "args": a, "calls": 1}
        return orig(g, *a)

    x = torch.randn(N, 3, HW, HW, device="cuda")
    ops.conv16_fprop_splitk = record
    try:
        with torch.no_grad():
            pred.eng.forward(x, None, training=False, save=False, prepared=pred.state)
    finally:
        ops.conv16_fprop_splitk = orig
    torch.cuda.synchronize()
    out = []
    for key, r in rec.items():
        g, (x_, xs, w, wsc, o, b, st, s_plan, _) = r["g"], r["args"]
        kb = es.kblocks(g)
        cand = sorted({1, s_plan} | {s for s in (2, 4, 8, 16, 32, 64) if s <= kb})
        ws = torch.empty(max(cand) * es.phase_tiles(g) * 128 * g.Cout, device="cuda")
        graphs = {}
        for s in cand:                             # CALLS back-to-back calls per replay: device time
            orig(g, x_, xs, w, wsc, o, b, st, s, ws)
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            graphs[s] = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graphs[s], stream=side):
                for _ in range(CALLS):
                    orig(g, x_, xs, w, wsc, o, b, st, s, ws)
        ev = {s: [] for s in cand}
        for _ in range(reps):
            for s in cand:                         # alternate the split counts
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                graphs[s].replay()
                e1.record()
                ev[s].append((e0, e1))
        torch.cuda.synchronize()
        us = {s: float(np.median([a.elapsed_time(b_) for a, b_ in ev[s]])) * 1e3 / CALLS for s in cand}
        out.append({"M": key[0], "Cin": key[1], "Cout": key[2], "T": key[3], "os": key[4], "is": key[5],
                    "calls": r["calls"], "tiles": es.phase_tiles(g) * es.n_tiles(g), "kb": kb,
                    "S": s_plan, "us_S1": us[1], "us_planned": us[s_plan],
                    "us_by_S": {str(s): round(t, 2) for s, t in us.items()}})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,2,4,8,32")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--layer-sizes", default="1,32")
    args = ap.parse_args()
    ops.device_check()
    info = gpu_info()
    torch.manual_seed(0)
    cfg = refshim.make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    model = models.pose3d_resnet.get_pose_net(cfg, False).cuda().eval()
    res = dict(info)
    res["latency"] = latency_rows(model, [int(v) for v in args.sizes.split(",")], args.reps)
    res["layers"] = {n: layer_table(model, int(n)) for n in args.layer_sizes.split(",")}
    res.update({k + "_after": v for k, v in gpu_info().items() if k in ("power_limit_w", "max_sm_clock_mhz")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
