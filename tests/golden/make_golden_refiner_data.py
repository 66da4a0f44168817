"""Writes the refiner dataset fixture and its goldens (build container only: it runs the unmodified
reference refiner/data.py under oracle/refshim.py).

  tests/golden/refiner_data/{train,valid}.pkl  {'inp', 'out'} float32 skeleton-like poses in mm, MPII
                                               order, root (hip, joint 6) at the origin; train as
                                               [S,16,3], valid as [S,48] (both forms the class reads)
  tests/golden/refiner_data.npz                what the reference class made of them with
                                               np.random.seed(SEED): normalised train data / labels,
                                               the four norm arrays, the permutation, the valid data /
                                               labels, and evaluate()'s return value, seven results and
                                               per-joint errors for fixed predictions (float32 arithmetic)
"""
import importlib
import logging
import os
import pickle
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import refshim  # noqa: E402

SEED = 7
OUT = os.path.join(ROOT, "tests", "golden")

# a standing skeleton in MPII order (mm, camera-like axes: x right, y down, z forward), hip at 0
SKELETON = np.array([
    [-120, 850, 30], [-110, 450, 10], [-130, 0, 0], [130, 0, 0], [110, 450, 10], [120, 850, 30],
    [0, 0, 0], [0, -480, 10], [0, -580, 0], [0, -720, -20], [-420, -120, 40], [-330, -280, 30],
    [-180, -480, 10], [180, -480, 10], [330, -280, 30], [420, -120, 40]], dtype=np.float64)


def _poses(rng, S):
    out = np.empty((S, 16, 3))
    for s in range(S):
        a = rng.uniform(-np.pi, np.pi)
        R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        p = (SKELETON + rng.normal(0, 40, SKELETON.shape)) @ R.T
        out[s] = p - p[6]
    return out


def make(rng):
    gt_tr, gt_va = _poses(rng, 96), _poses(rng, 40)
    inp_tr = gt_tr + rng.normal(0, 30, gt_tr.shape)
    inp_va = gt_va + rng.normal(0, 30, gt_va.shape)
    for a in (inp_tr, inp_va):
        a[:, 6] = 0.0
    return ({"inp": inp_tr.astype(np.float32), "out": gt_tr.astype(np.float32)},
            {"inp": inp_va.reshape(-1, 48).astype(np.float32), "out": gt_va.reshape(-1, 48).astype(np.float32)})


class _Capture(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def main():
    rng = np.random.default_rng(20261017)
    train, valid = make(rng)
    fix = os.path.join(OUT, "refiner_data")
    os.makedirs(fix, exist_ok=True)
    for name, d in (("train", train), ("valid", valid)):
        with open(os.path.join(fix, name + ".pkl"), "wb") as f:
            pickle.dump(d, f, protocol=4)

    refshim.install()
    mod = importlib.import_module("refiner.data")
    cwd = os.getcwd()
    tmp = tempfile.mkdtemp()
    try:
        os.makedirs(os.path.join(tmp, "refiner", "data"))
        for name in ("train", "valid"):
            shutil.copy(os.path.join(fix, name + ".pkl"), os.path.join(tmp, "refiner", "data"))
        os.chdir(tmp)
        np.random.seed(SEED)
        tr = mod.Human36M(is_train=True)
        np.random.seed(SEED)
        perm = np.random.permutation(len(tr))
        va = mod.Human36M(is_train=False)
        prng = np.random.default_rng(5)
        preds = ((va.labels + prng.normal(0, 25, va.labels.shape).astype(np.float32) - va.labels_mean)
                 / va.labels_std).astype(np.float32)
        cap = _Capture()
        mod.logger.addHandler(cap)
        mod.logger.setLevel(logging.INFO)
        ret = va.evaluate(preds)
        mod.logger.removeHandler(cap)
    finally:
        os.chdir(cwd)
        shutil.rmtree(tmp)
    vals = dict(line.split(" : ") for line in cap.lines if " : " in line)
    per_joint = np.array([float(vals[n]) for n in mod.MPII_NAMES])
    results = np.array([float(vals[k]) for k in ("hm36_17j", "hm36_17j_align", "hm36_17j_14", "hm36_17j_14_al",
                                                 "hm36_17j_x", "hm36_17j_y", "hm36_17j_z")])
    np.savez_compressed(os.path.join(OUT, "refiner_data.npz"), seed=SEED,
                        train_data=tr.data, train_labels=tr.labels, perm=perm,
                        data_mean=tr.data_mean, data_std=tr.data_std,
                        labels_mean=tr.labels_mean, labels_std=tr.labels_std,
                        valid_data=va.data, valid_labels=va.labels, eval_preds=preds,
                        eval_return=np.float64(ret), eval_results=results, eval_per_joint=per_joint)
    print("wrote", fix, "and refiner_data.npz; evaluate ->", ret)


if __name__ == "__main__":
    main()
