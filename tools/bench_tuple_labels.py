"""Cost of the robust online labels of whole camera tuples (TRAIN.TRIANGULATION_METHOD: robust) on
one GPU.  Prints one JSON line: GPU name, power limit and max SM clock; then
  (a) the label stage alone at 32 tuples x 4 views, J in {16, 17}: epb_tuple_labels against the
      pair path's label stage on the same batch (epb_patch_to_image + epb_triangulate iterative +
      epb_project_labels), each captured in a CUDA graph and timed with CUDA events over --reps
      replays (us per batch);
  (b) the C4 self-supervised graphed training step (R50, J = 16, D = 64, 32 tuples x 4 views of
      256 x 256, f16x3): pairs / iterative (bench.py's layout) against robust / V = 4 (view-major),
      alternated over --rounds rounds of --steps replays, ms per step and the medians.
    python tools/bench_tuple_labels.py [--reps 500] [--rounds 5] [--steps 10]"""
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

TUPLES, VIEWS = 32, 4


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        w, mhz = r.stdout.strip().splitlines()[0].split(",")
        return float(w), float(mhz)
    except Exception:
        return None, None


def graph_us(fn, reps):
    """fn captured in a CUDA graph, replayed `reps` times: us per replay (CUDA events)"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        fn()
    for _ in range(20):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return 1000.0 * e0.elapsed_time(e1) / reps


def label_stage(J, reps, dev):
    import lib.utils.img_utils as iu
    from tests import tuple_label_cases as tc
    coords, lse, meta, _, _ = tc.case(40 + J, TUPLES, VIEWS, J, outliers=0.25, lse=True)
    B = TUPLES * VIEWS
    mt = {k: torch.as_tensor(np.asarray(v, dtype=np.float64)).to(dev) for k, v in meta.items()}
    geom = {"_packed": iu.pack_meta(mt, B, dev)}
    c, ls = torch.from_numpy(coords).to(dev), torch.from_numpy(lse).to(dev)

    def robust():
        iu.tuple_labels_device(c, ls, geom, VIEWS, 15.0)

    def pairs():
        kps = iu.patch_to_image_device(c, geom)
        iu.labels_from_global_coords_device(iu.triangulate_device(kps, geom, "iterative"), geom)
    return {"robust_v4_us": round(graph_us(robust, reps), 2), "pairs_iterative_us": round(graph_us(pairs, reps), 2)}


def _meta(order, dev):
    from lib.dataset.synthetic import ring_camera
    rng = np.random.default_rng(1000)
    n = len(order)
    cams = {(t, v): ring_camera(rng, v) for t in range(TUPLES) for v in range(VIEWS)}
    meta = {"center_x": torch.tensor(500 + rng.uniform(-50, 50, n)), "center_y": torch.tensor(500 + rng.uniform(-50, 50, n)),
            "width": torch.tensor(800 + rng.uniform(-100, 100, n)), "height": torch.tensor(800 + rng.uniform(-100, 100, n)),
            "scale": torch.ones(n, dtype=torch.float64), "rot": torch.zeros(n, dtype=torch.float64)}
    for i, k in enumerate(("R", "T", "f", "c", "projection_matrix")):
        meta[k] = torch.tensor(np.stack([cams[o][i] for o in order]))
    return {k: v.to(dev) for k, v in meta.items()}


def step_ms(robust, steps, dev, state):
    import lib.core.function as fn
    import lib.core.integral_loss as il
    import lib.models as models
    import lib.utils.utils as U
    from tools.bench_cfg import make_cfg
    HW, J, D = 256, 16, 64
    if "model" not in state:
        cfg = make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
        torch.manual_seed(0)
        state["model"] = models.pose3d_resnet.get_pose_net(cfg, False, precision="f16x3").to(dev).train()
        state["crit"] = il.SmoothL1JointLocationLoss(J).to(dev)
        state["opt"] = U.FusedAdam(list(state["model"].parameters()), lr=1e-3)
        pair_order = [(t, v) for v in (0, 3, 1, 2) for t in range(TUPLES)]       # bench.py's pair layout
        state["meta_pairs"] = _meta(pair_order, dev)
        state["meta_robust"] = _meta([(t, v) for v in range(VIEWS) for t in range(TUPLES)], dev)
        g = torch.Generator().manual_seed(1000)
        state["x"] = [torch.randn(TUPLES * VIEWS, 3, HW, HW, generator=g).to(dev) for _ in range(2)]
    if robust:
        stepper = fn.GraphedTrainStep(state["model"], state["crit"], state["opt"], online=True, method="robust",
                                      views=VIEWS)
        meta = state["meta_robust"]
    else:
        stepper = fn.GraphedTrainStep(state["model"], state["crit"], state["opt"], online=True, method="iterative")
        meta = state["meta_pairs"]
    for i in range(3):                       # eager, capture, replay
        stepper(state["x"][i % 2], meta=meta)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        loss = stepper(state["x"][i % 2], meta=meta)
    e1.record()
    torch.cuda.synchronize()
    assert torch.isfinite(loss).item()
    del stepper
    torch.cuda.empty_cache()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=500)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if args.reps < 200:
        raise SystemExit("--reps must be at least 200")
    from epipolarpose_b200 import ops
    dev = torch.device("cuda")
    ops.device_check()
    w, mhz = card()
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": w, "max_sm_clock_mhz": mhz,
           "label_stage_32x4": {"J%d" % J: label_stage(J, args.reps, dev) for J in (16, 17)}}
    state, pairs, robust = {}, [], []
    for _ in range(args.rounds):
        pairs.append(step_ms(False, args.steps, dev, state))
        robust.append(step_ms(True, args.steps, dev, state))
    out["step_ms_pairs_iterative"] = [round(v, 2) for v in pairs]
    out["step_ms_robust_v4"] = [round(v, 2) for v in robust]
    out["step_ms_median"] = {"pairs_iterative": round(float(np.median(pairs)), 2),
                             "robust_v4": round(float(np.median(robust)), 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
