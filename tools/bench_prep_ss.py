"""Throughput of save_triangulations (lib/utils/prep_h36m.py): writing a self-supervised annotation
file from a network's predictions, end to end.

Writes a seeded synthetic dict-form tree under --out (images/ and annot/src.pkl): `--tuples` frames
of 4 ring cameras, 17 joints, whose records point at `--files` distinct 1000x1000 q90 JPEG frames
(seeded smooth noise, transcoded to short restart intervals as tools/prep_frames.py prepares a
frame tree for the device decoder, read over and over, so file reads come from the page cache).  Then times
save_triangulations on it, PoseResNet-50 (random init, split-fp16 engine), J 16 from the 17-joint
source (MPII order), 256x256 crops, `--batch` tuples per batch, `--workers` loader workers, after a
warm-up run on the first 2 batches (graph capture of both batch sizes).  Prints ONE JSON line: the
GPU name, power limit and max SM clock (read in the same run), and per method: tuples/s, seconds,
the shares of the wall time spent waiting for the loader's workers, assembling the batches on the
device (JPEG decode, crop) and in the predictor's calls (its graph replays, host -> device copies
of the boxes and cameras, results to the host), and the report.  Needs a GPU.

    python tools/bench_prep_ss.py --out DIR [--tuples 2048] [--methods robust,iterative]"""
import argparse
import json
import os
import pickle
import sys
import time

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.bench_jpeg import card  # noqa: E402


def make_tree(out, tuples, files, seed=0):
    import cv2
    from lib.utils.cameras import Camera
    from lib.dataset.synthetic import ring_camera
    from lib.utils.img_utils import transcode_jpeg_batch_device
    rng = np.random.default_rng(seed)
    blobs = []
    os.makedirs(os.path.join(out, "images"), exist_ok=True)
    os.makedirs(os.path.join(out, "annot"), exist_ok=True)
    for i in range(files):
        low = rng.uniform(0, 255, (25, 25, 3)).astype(np.float32)
        img = cv2.resize(low, (1000, 1000), interpolation=cv2.INTER_CUBIC) + rng.normal(0, 3, (1000, 1000, 3))
        ok, blob = cv2.imencode(".jpg", np.clip(img, 0, 255).astype(np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 90])
        assert ok
        blobs.append(blob.tobytes())
    # as tools/prep_frames.py prepares a frame tree: lossless re-coding with short restart intervals
    blobs, status = transcode_jpeg_batch_device(blobs)
    assert not np.any(status), status
    for i, blob in enumerate(blobs):
        with open(os.path.join(out, "images", "f%03d.jpg" % i), "wb") as f:
            f.write(blob)
    parents = np.array([0, 0, 1, 2, 0, 4, 5, 0, 8, 8, 9, 8, 11, 12, 8, 14, 15], dtype=np.int64)
    pairs = [[1, 4], [2, 5], [3, 6], [14, 11], [15, 12], [16, 13]]
    anno = {v + 1: [] for v in range(4)}
    for t in range(tuples):
        X = rng.normal(0.0, 400.0, size=(17, 3))
        for v in range(4):
            R, T, f, c, _ = ring_camera(rng, v)
            cam = Camera((R, T, f, c, np.zeros((3, 1)), np.zeros((2, 1)), "cam%d" % v))
            Xc = (R @ (X.T - T)).T
            j3d = np.stack([Xc[:, 0] / Xc[:, 2] * f[0] + c[0], Xc[:, 1] / Xc[:, 2] * f[1] + c[1],
                            Xc[:, 2] - Xc[0, 2]], axis=1)
            anno[v + 1].append(dict(image="images/f%03d.jpg" % ((4 * t + v) % files), joints_3d=j3d,
                                    joints_3d_vis=np.ones((17, 3)), pelvis=Xc[0], fl=np.asarray(f).reshape(2),
                                    c_p=np.asarray(c).reshape(2), cam=cam,
                                    center_x=500.0 + rng.uniform(-50, 50), center_y=500.0 + rng.uniform(-50, 50),
                                    width=800.0, height=800.0, flip_pairs=pairs, parent_ids=parents,
                                    action="Walking"))
    make_tree.mean_bytes = float(np.mean([len(b) for b in blobs]))
    path = os.path.join(out, "annot", "src.pkl")
    with open(path, "wb") as f:
        pickle.dump(anno, f, protocol=4)
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--tuples", type=int, default=2048)
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--methods", default="robust,iterative")
    a = ap.parse_args()
    import lib.dataset as dataset
    from lib.dataset.JointIntegralDataset import load_pickle
    from lib.utils.prep_h36m import save_triangulations, _make_predictor, joint_layout
    from tests import golden_inputs as gi
    from tests.golden_inputs import _model
    from tests import dataset_cases as dc
    from epipolarpose_b200 import ops
    ops.device_check()
    dev = torch.device("cuda:0")
    src = make_tree(a.out, a.tuples, a.files)
    anno = load_pickle(src)
    model = _model(dev, gi.SIZE_CASES["c1"], "f16x3", train=False)          # R50, J 16, D 64, 256x256
    cfg = dc.cfg()
    cfg.MODEL.IMAGE_SIZE = [256, 256]
    ds = dataset.h36m(cfg, a.out, "src", False)
    layout = joint_layout(16, 17, anno[1][0]["flip_pairs"], anno[1][0]["parent_ids"])
    res = {"card_before": card()}
    for method in a.methods.split(","):
        pred = _make_predictor(model, method, False, layout[2], 15.0)
        warm = {c: anno[c][:2 * a.batch + 1] for c in anno}
        save_triangulations(model, ds, warm, os.path.join(a.out, "warm.pkl"), method=method,
                            tuples_per_batch=a.batch, workers=a.workers, predictor=pred)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        rep = save_triangulations(model, ds, src, os.path.join(a.out, "ss-%s.pkl" % method), method=method,
                                  tuples_per_batch=a.batch, workers=a.workers, predictor=pred)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        res[method] = {"tuples_per_s": a.tuples / dt, "seconds": dt,
                       "predictor_share": rep["predictor_seconds"] / dt,
                       "loader_wait_share": rep["loader_wait_seconds"] / dt,
                       "assemble_share": rep["assemble_seconds"] / dt, "report": rep}
    res["card_after"] = card()
    res.update(tuples=a.tuples, batch=a.batch, workers=a.workers, network="R50 J16 D64 256x256 f16x3 random init",
               frame="1000x1000 q90 JPEG", frame_mean_bytes=make_tree.mean_bytes)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
