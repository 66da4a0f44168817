"""Cost of self-supervision without camera extrinsics (TRAIN.ESTIMATE_EXTRINSICS) on one GPU.
Prints one JSON line: GPU name and power limit; relative_pose_kernel time (CUDA events) at
NP = 64 pairs (the C4 step: 32 tuples x 2 pairs) and NP = 65536; the C4 self-supervised graphed
training step (bench.py's workload: R50, 4 x 32 views of 256x256, J = 16, D = 64, f16x3) with
known and with estimated extrinsics, alternated over several rounds, in ms per step.
    python tools/bench_relpose.py [--rounds 3] [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def power_limit_w():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def kernel_ms(NP, reps, dev):
    from lib.utils import triangulation as tri
    from tests import relpose_cases as rc
    d = rc.rig_pairs(64, 7)
    k = -(-NP // 64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(np.tile(a, (k,) + (1,) * (a.ndim - 1))[:NP])).to(dev)
    kps = torch.cat([t(d["ua"]), t(d["ub"])])
    intr = torch.cat([t(d["intr_a"]), t(d["intr_b"])])
    box = torch.cat([t(d["box_a"]), t(d["box_b"])])
    tri.relative_pose_pairs(kps, intr, box)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        tri.relative_pose_pairs(kps, intr, box)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def step_ms(estimate, steps, dev, state):
    import lib.core.function as fn
    import lib.core.integral_loss as il
    import lib.models as models
    import lib.utils.utils as U
    from tools.bench_cfg import make_cfg
    from lib.dataset.synthetic import ring_camera
    TUPLES, VIEWS, HW, J, D = 32, 4, 256, 16, 64
    n_img = TUPLES * VIEWS
    if "model" not in state:
        cfg = make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
        torch.manual_seed(0)
        state["model"] = models.pose3d_resnet.get_pose_net(cfg, False, precision="f16x3").to(dev).train()
        state["crit"] = il.SmoothL1JointLocationLoss(J).to(dev)
        state["opt"] = U.FusedAdam(list(state["model"].parameters()), lr=1e-3)
        rng = np.random.default_rng(1000)
        order = [(t, 0) for t in range(TUPLES)] + [(t, 3) for t in range(TUPLES)] + \
                [(t, 1) for t in range(TUPLES)] + [(t, 2) for t in range(TUPLES)]
        cams = {(t, v): ring_camera(rng, v) for t in range(TUPLES) for v in range(VIEWS)}
        meta = {"center_x": torch.tensor(500 + rng.uniform(-50, 50, n_img)),
                "center_y": torch.tensor(500 + rng.uniform(-50, 50, n_img)),
                "width": torch.tensor(800 + rng.uniform(-100, 100, n_img)),
                "height": torch.tensor(800 + rng.uniform(-100, 100, n_img)),
                "scale": torch.ones(n_img, dtype=torch.float64), "rot": torch.zeros(n_img, dtype=torch.float64),
                "R": torch.tensor(np.stack([cams[o][0] for o in order])),
                "T": torch.tensor(np.stack([cams[o][1] for o in order])),
                "f": torch.tensor(np.stack([cams[o][2] for o in order])),
                "c": torch.tensor(np.stack([cams[o][3] for o in order])),
                "projection_matrix": torch.tensor(np.stack([cams[o][4] for o in order]))}
        state["meta"] = {k: v.to(dev) for k, v in meta.items()}
        g = torch.Generator().manual_seed(1000)
        state["x"] = [torch.randn(n_img, 3, HW, HW, generator=g).to(dev) for _ in range(2)]
    stepper = fn.GraphedTrainStep(state["model"], state["crit"], state["opt"], online=True,
                                  method="iterative", estimate_extrinsics=estimate)
    for i in range(3):                       # eager, capture, replay
        stepper(state["x"][i % 2], meta=state["meta"])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = stepper(state["x"][i % 2], meta=state["meta"])
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item()
    del stepper
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    from epipolarpose_b200 import ops
    dev = torch.device("cuda")
    ops.device_check()
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w(),
           "relative_pose_kernel_ms": {"np64": round(kernel_ms(64, 50, dev), 4),
                                       "np65536": round(kernel_ms(65536, 3, dev), 3)}}
    state, known, est = {}, [], []
    for _ in range(args.rounds):
        known.append(step_ms(False, args.steps, dev, state))
        est.append(step_ms(True, args.steps, dev, state))
    out["step_ms_known_extrinsics"] = [round(v, 2) for v in known]
    out["step_ms_estimated_extrinsics"] = [round(v, 2) for v in est]
    out["step_ms_difference_median"] = round(float(np.median(np.array(est) - np.array(known))), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
