"""Data-loading throughput of the h36m dataset on one GPU.  Builds an H36M-shaped tree in a
temporary directory (dict-form annotation pickle, 4 cameras) whose records point at the two
1000x1002 q90 4:2:0 frames of tests/golden/jpeg.npz, and prints JSON lines, each with the card
name, power limit and max SM clock:
  loader     (a) frames/s of DataLoader(num_workers=8) batches assembled on the device
             (lib.dataset.assemble_batch: device JPEG decode + 256x256 crop + labels), 128 frames
             per batch (TRI: 64 frame pairs);
  step       (b) the R50 self-supervised training step (train_integral, graphed, TRI +
             ONLINE_TRIANGULATION) fed by that loader, against the same loop on a resident batch;
  host_path  (c) the reference-style host pipeline (cv2.imread + cv2.warpAffine + normalisation
             in the workers) in 8 and 16 workers, frames/s (a CPU number).
Two distinct files are read over and over, so file reads come from the page cache.
    python tools/bench_data.py [--frames 2048] [--batches 12]"""
import argparse
import json
import os
import pickle
import random
import sys
import tempfile
import time

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.bench_jpeg import card  # noqa: E402

PAIRS = 64                    # 128 frames per step, as bench.py's 32 tuples x 4 views


def make_tree(tmp, frames):
    from lib.utils.cameras import Camera
    from lib.dataset.synthetic import ring_camera
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
    names = list(g["names"])
    os.makedirs(os.path.join(tmp, "images"))
    os.makedirs(os.path.join(tmp, "annot"))
    for tag in ("a", "b"):
        i = names.index("frame1000_" + tag)
        with open(os.path.join(tmp, "images", tag + ".jpg"), "wb") as f:
            f.write(g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes())
    rng = np.random.default_rng(0)
    anno = {v + 1: [] for v in range(4)}
    for t in range(frames // 4):
        X = rng.normal(0.0, 400.0, size=(17, 3))
        for v in range(4):
            R, T, f, c, _ = ring_camera(rng, v)
            cam = Camera((R, T, f, c, np.zeros((3, 1)), np.zeros((2, 1)), "cam%d" % v))
            Xc = (R @ (X.T - T)).T
            j3d = np.stack([Xc[:, 0] / Xc[:, 2] * f[0] + c[0], Xc[:, 1] / Xc[:, 2] * f[1] + c[1],
                            Xc[:, 2] - Xc[0, 2]], axis=1)
            anno[v + 1].append(dict(image="images/%s.jpg" % "ab"[(t + v) % 2], joints_3d=j3d,
                                    joints_3d_vis=np.ones((17, 3)), pelvis=Xc[0], fl=f, c_p=c, cam=cam,
                                    center_x=500.0 + rng.uniform(-50, 50), center_y=500.0 + rng.uniform(-50, 50),
                                    width=800.0, height=800.0, flip_pairs=[], parent_ids=np.zeros(17, np.int64),
                                    action="Walking"))
    with open(os.path.join(tmp, "annot", "train.pkl"), "wb") as f:
        pickle.dump(anno, f)


def config(tmp, layers, precision):
    from lib.core.config import config as cfg, reset_config
    reset_config()
    cfg.WORKERS = 8
    cfg.PRINT_FREQ = 10 ** 9
    cfg.MODEL.EXTRA.NUM_LAYERS = layers
    cfg.MODEL.INIT_WEIGHTS = False
    cfg.MODEL.PRECISION = precision
    cfg.MODEL.IMAGE_SIZE = np.array([256, 256])
    cfg.LOSS.FN = "SmoothL1JointLocationLoss"
    cfg.DATASET.ROOT = tmp
    cfg.DATASET.TRI = True
    cfg.TRAIN.ONLINE_TRIANGULATION = True
    cfg.TRAIN.BATCH_SIZE = PAIRS
    return cfg


def bench_loader(ds, batches, workers):
    from lib.dataset import assemble_batch
    dl = DataLoader(ds, batch_size=PAIRS, shuffle=True, num_workers=workers, pin_memory=True, drop_last=True)
    n, t0 = 0, None
    for i, b in enumerate(dl):
        x = assemble_batch(b)[0]
        if i == 1:                   # the first batch pays for worker start-up
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        elif i > 1:
            n += x.shape[0]
        if i == batches + 1:
            break
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def bench_step(cfg, ds, precision, steps):
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.utils.utils as U
    from lib.core.function import train_integral, loader_batch
    from lib.dataset import assemble_batch  # noqa: F401
    torch.manual_seed(0)
    model = models.pose3d_resnet.get_pose_net(cfg, False, precision=precision).cuda().train()
    crit = il.SmoothL1JointLocationLoss(17).cuda()
    opt = U.FusedAdam(list(model.parameters()), lr=1e-3)
    dl = DataLoader(ds, batch_size=PAIRS, shuffle=True, num_workers=cfg.WORKERS, pin_memory=True, drop_last=True)
    first = loader_batch(next(iter(dl)))
    resident = [first] * steps
    train_integral(cfg, resident[:3], model, crit, opt, 0)              # warm-up + capture
    out = {}
    for name, src in (("resident", resident), ("loader", dl), ("resident", resident), ("loader", dl)):
        it = list(src) if name == "resident" else src
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        train_integral(cfg, it, model, crit, opt, 1)
        torch.cuda.synchronize()
        n = len(it) if name == "resident" else len(dl)
        out.setdefault(name, []).append((time.perf_counter() - t0) / n * 1e3)
    return {k: min(v) for k, v in out.items()}, len(dl)


class HostPath(Dataset):
    """Reference-style sample on the host: cv2.imread, the augmentation draws, cv2.warpAffine
    of the box to 256x256, BGR->RGB, colour scale, clip, normalisation (float32 CHW)."""

    def __init__(self, ds):
        self.recs = [r for d in ds.db for r in d]
        self.root = ds.root
        self.mean, self.std = ds.mean, ds.std

    def __len__(self):
        return len(self.recs)

    def __getitem__(self, i):
        import cv2
        from lib.utils.img_utils import do_augmentation
        r = self.recs[i]
        img = cv2.imread(os.path.join(self.root, r["image"]), cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
        scale, rot, _, color = do_augmentation()
        a = np.deg2rad(rot)
        w, h = r["width"] * scale, r["height"] * scale
        c = np.array([r["center_x"], r["center_y"]])
        down = np.array([-np.sin(a), np.cos(a)]) * h * 0.5
        right = np.array([np.cos(a), np.sin(a)]) * w * 0.5
        src = np.float32([c, c + down, c + right])
        dst = np.float32([[128, 128], [128, 256], [256, 128]])
        patch = cv2.warpAffine(img, cv2.getAffineTransform(src, dst), (256, 256), flags=cv2.INTER_LINEAR)
        x = patch[:, :, ::-1].transpose(2, 0, 1).astype(np.float32)
        for k in range(3):
            x[k] = (np.clip(x[k] * color[k], 0, 255) - self.mean[k]) / self.std[k]
        return torch.from_numpy(x)


def bench_host(ds, workers, batches):
    dl = DataLoader(HostPath(ds), batch_size=2 * PAIRS, shuffle=True, num_workers=workers, drop_last=True)
    n, t0 = 0, None
    for i, x in enumerate(dl):
        if i == 1:
            t0 = time.perf_counter()
        elif i > 1:
            n += x.shape[0]
        if i == batches + 1:
            break
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4096)
    ap.add_argument("--batches", type=int, default=12)
    ap.add_argument("--layers", type=int, default=50)
    ap.add_argument("--precision", default=os.environ.get("EPB_PRECISION", "f16x3"))
    args = ap.parse_args()
    from epipolarpose_b200 import ops
    import lib.dataset as dataset
    ops.device_check()
    info = card()
    info["host_cpus"] = os.cpu_count()
    with tempfile.TemporaryDirectory() as tmp:
        make_tree(tmp, args.frames)
        cfg = config(tmp, args.layers, args.precision)
        np.random.seed(0)
        random.seed(0)
        ds = dataset.h36m(cfg, tmp, "train", True)
        fps = bench_loader(ds, args.batches, 8)
        print(json.dumps(dict(info, bench="loader", workers=8, frames_per_batch=2 * PAIRS,
                              frames_per_s=round(fps, 1))), flush=True)
        ms, n = bench_step(cfg, ds, args.precision, args.batches)
        print(json.dumps(dict(info, bench="step", layers=args.layers, precision=args.precision,
                              frames_per_step=2 * PAIRS, steps_per_epoch=n,
                              resident_ms_per_step=round(ms["resident"], 2),
                              loader_ms_per_step=round(ms["loader"], 2))), flush=True)
        for w in (8, 16):
            print(json.dumps(dict(info, bench="host_path", workers=w,
                                  frames_per_s=round(bench_host(ds, w, args.batches), 1))), flush=True)


if __name__ == "__main__":
    main()
