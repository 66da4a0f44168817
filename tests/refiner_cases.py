"""TEST INFRASTRUCTURE: float64 numpy restatements for the refiner tests.

  pose_errors(pred, gt, subset)  the per-sample body of the reference refiner's evaluate
                                 (refiner/data.py:78-160) in float64, on oracle.restate's
                                 compute_similarity_transform -> (metrics [S,7], per_joint [S,J])
  pose_to_camera(joints, cam, root)  CamBackProj of every joint minus the root's ([N,J,3] mm)
  poses(rng, S, J)               skeleton-like camera-frame poses with the hip at the origin
Plus the fixture paths of tests/golden/refiner_data."""
import os

import numpy as np

from oracle import restate

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = os.path.join(HERE, "golden", "refiner_data")
GOLDEN = os.path.join(HERE, "golden", "refiner_data.npz")
J14 = [0, 1, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14]


def pose_errors(pred, gt, subset=J14):
    pred, gt = np.asarray(pred, np.float64), np.asarray(gt, np.float64)
    S, J, _ = pred.shape
    metrics, per_joint = np.zeros((S, 7)), np.zeros((S, J))
    for s in range(S):
        _, _, T, b, c = restate.compute_similarity_transform(gt[s], pred[s], compute_optimal_scale=True)
        d = gt[s] - pred[s]
        da = gt[s] - (b * pred[s].dot(T) + c)
        e, ea = np.linalg.norm(d, axis=1), np.linalg.norm(da, axis=1)
        metrics[s] = [e.mean(), ea.mean(), e[subset].mean(), ea[subset].mean(),
                      np.abs(d[:, 0]).mean(), np.abs(d[:, 1]).mean(), np.abs(d[:, 2]).mean()]
        per_joint[s] = e
    return metrics, per_joint


def pose_to_camera(joints, cam, root):
    joints, cam = np.asarray(joints, np.float64), np.asarray(cam, np.float64)
    d = joints[:, :, 2] + cam[:, 4:5]
    X = np.stack([(joints[:, :, 0] - cam[:, 2:3]) / cam[:, 0:1] * d,
                  (joints[:, :, 1] - cam[:, 3:4]) / cam[:, 1:2] * d, d], axis=2)
    return X - X[:, root:root + 1]


def poses(rng, S, J=16, hip=6):
    base = rng.normal(0, 300, (J, 3))
    p = base[None] + rng.normal(0, 40, (S, J, 3))
    return p - p[:, hip:hip + 1]
