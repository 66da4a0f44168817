"""Inference of the MODEL.VOLUME = false head, PoseResNet-50 (J 16, D 64, 256x256 images) on the
split-fp16 engine: HeatmapPredictor (one CUDA-graph replay: network + epb_heatmap_decode) against
eager `model.eval()(x)` + the numpy decode (get_final_preds' argmax / refinement and get_depth_preds,
restated in tests/heatmap_cases.py), and the decode kernel alone.

    python tools/bench_heatmap.py [--sizes 1,32] [--reps 200]

Prints ONE JSON line with the GPU name, its power limit and max SM clock (read in the same run,
before and after) and:
  latency   per N and flip test off / on: host clock around pred(images) with HOST images in and
            numpy out, device events around the graph replay alone, and the eager baseline (host
            clock around model(x) on a device batch, the copy to the host and the numpy decode);
            median / p90 ms and images/s from the medians; reps = max(30, reps / N), alternated
  decode    epb_heatmap_decode alone at N = 1 and 32 on both layouts (NCHW, and the channels-last
            [N, 64, 64, 16] buffer the final conv writes), with and without flip: device events
            around a CUDA graph of 50 back-to-back launches, and the bytes the decode must read
            (heat-maps + depth logits) over that time against the 3.35 TB/s HBM3 data-sheet peak."""
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
from epipolarpose_b200 import ops  # noqa: E402
import lib.models as models  # noqa: E402
from lib.core.inference import HeatmapPredictor, heatmap_decode_device  # noqa: E402
from tests import heatmap_cases as hc  # noqa: E402
from tools.bench_cfg import make_cfg  # noqa: E402

J, D, HW = 16, 64, 256
HBM_PEAK = 3.35e12
CALLS = 50


def stats(ts):
    a = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(a)), "p90_ms": float(np.percentile(a, 90)), "n": len(a)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits", "-i", "0"], capture_output=True, text=True)
    name, pl, clk = [v.strip() for v in q.stdout.strip().split(",")] if q.returncode == 0 else ("?", "?", "?")
    return {"gpu": torch.cuda.get_device_name(0), "smi_name": name, "power_limit_w": pl,
            "max_sm_clock_mhz": clk}


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def numpy_decode(hm, depth, pairs):
    """the eager baseline's host decode: [flip merge,] get_final_preds' argmax + refinement and
    get_depth_preds, rows in patch px"""
    if pairs is not None:
        hm, depth = hc.flip_merge(hm, depth, pairs, True)
    _, maxvals, d, px = hc.decode_ref(hm, depth, D, HW, HW, 2000.0)
    return np.concatenate([px, (d / 2000.0 * HW)[..., None], maxvals[..., None]], axis=2)


def latency_rows(model, sizes, reps):
    rows = []
    for flip in (False, True):
        pairs = hc.MPII_PAIRS if flip else None
        pred = HeatmapPredictor(model, flip_test=flip, shift_heatmap=True, flip_pairs=pairs)
        for N in sizes:
            r = max(30, reps // N)
            xh = torch.randn(N, 3, HW, HW, generator=torch.Generator().manual_seed(N))
            xd = xh.cuda()

            def eager():
                with torch.no_grad():
                    x = torch.cat([xd, torch.flip(xd, [3])]) if flip else xd
                    hm, d = model(x)
                    return numpy_decode(hm.cpu().numpy(), d.cpu().numpy(), pairs)

            for _ in range(3):
                eager()
                pred(xh)
            diff = np.abs(pred(xh)[..., :2] - eager()[..., :2])
            te, tp = [], []
            for _ in range(r):
                te.append(timed(eager))
                tp.append(timed(lambda: pred(xh)))
            ent = pred.graphs[(N, HW, HW)]
            ev = []
            for _ in range(r):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                ent["graph"].replay()
                e1.record()
                ev.append((e0, e1))
            torch.cuda.synchronize()
            row = {"N": N, "flip": flip, "predictor": stats(tp), "eager_numpy": stats(te),
                   "replay": stats([a.elapsed_time(b) * 1e-3 for a, b in ev]),
                   "joints_equal_vs_eager": float(np.mean(diff == 0))}
            for k in ("predictor", "eager_numpy", "replay"):
                row[k]["images_per_s"] = N / (row[k]["median_ms"] * 1e-3)
            rows.append(row)
    return rows


def decode_rows(reps=20):
    out = []
    h = HW // 4
    for N in (1, 32):
        for flip in (False, True):
            B = 2 * N if flip else N
            pairs = hc.MPII_PAIRS if flip else None
            hm, depth = hc.seeded(N, J, h, h, D, 1, B=B)
            nchw = torch.from_numpy(hm).cuda()
            cl = nchw.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
            dd = torch.from_numpy(depth).cuda()
            kps = torch.empty((N, J, 4), device="cuda", dtype=torch.float64)
            res = {}
            for name, t in (("nchw", nchw), ("channels_last", cl)):
                heatmap_decode_device(t, dd, D, None, HW, HW, 2000.0, True, pairs, True, out=kps)
                side = torch.cuda.Stream()
                side.wait_stream(torch.cuda.current_stream())
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=side):
                    for _ in range(CALLS):
                        heatmap_decode_device(t, dd, D, None, HW, HW, 2000.0, True, pairs, True, out=kps)
                ev = []
                for _ in range(reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    g.replay()
                    e1.record()
                    ev.append((e0, e1))
                torch.cuda.synchronize()
                us = float(np.median([a.elapsed_time(b) for a, b in ev])) * 1e3 / CALLS
                nbytes = 4 * (B * J * h * h + B * J * D)
                res[name] = {"us": us, "bytes": nbytes, "GB_per_s": nbytes / (us * 1e-6) / 1e9,
                             "share_of_hbm_peak": nbytes / (us * 1e-6) / HBM_PEAK}
            out.append({"N": N, "flip": flip, **res})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,32")
    ap.add_argument("--reps", type=int, default=200)
    args = ap.parse_args()
    ops.device_check()
    res = dict(gpu_info())
    torch.manual_seed(0)
    cfg = make_cfg(num_layers=50, num_joints=J, volume=False, depth_res=D, image_size=(HW, HW))
    model = models.pose3d_resnet.get_pose_net(cfg, False).cuda().eval()
    res["latency"] = latency_rows(model, [int(v) for v in args.sizes.split(",")], args.reps)
    res["decode"] = decode_rows()
    res.update({k + "_after": v for k, v in gpu_info().items() if k in ("power_limit_w", "max_sm_clock_mhz")})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
