"""Pose Structure Score (PSS@k), the paper's third metric next to MPJPE / N-MPJPE / P-MPJPE.
The reference release does not contain it, so this module fixes the definition:

1. Pose vector: every joint back-projected to camera-frame mm with the arithmetic of
   epb_h36m_eval (CamBackProj with fl, c_p and the pelvis depth), minus the root joint (0 in H36M
   order, 6 with DATASET.MPII_ORDER), divided by the Frobenius norm of the root-relative pose (PSS
   is scale-invariant; a zero pose stays zero).  Ground truth is `joints_3d` (permuted by
   H36M_TO_MPII_PERM under MPII_ORDER); predictions are the `preds` given to `evaluate`, not
   Procrustes-aligned.
2. Clusters: k-means of the ground truth of `<DATASET.ROOT>/annot/train-fs.pkl` (all cameras of
   the dict form, in camera-key order), in the evaluation's joint order.
3. k-means++, one candidate per step: uniform draws from splitmix64 seeded by (seed, restart),
   top 53 bits; centre 0 = floor(u N); centre j = the first point whose inclusive prefix of D^2
   exceeds u * sum(D^2).  Prefix sums: chunks of 1024 points summed in index order, chunk totals
   in chunk order.  sum(D^2) = 0 (fewer than k distinct poses) is an error.
4. Lloyd: exact squared distances summed in coordinate order without FMA, ties to the lowest
   centre; centroid = member sum (same two-level order) / count; an empty cluster, in cluster
   order, takes the point farthest from its current centre (lowest index on ties, no point
   twice); stop when a pass changes no label or after max_iter = 300 updates; n_init = 10
   restarts, lowest inertia wins (ties to the lowest restart).
5. PSS@k = (samples whose prediction and ground truth fall in the same cluster) / S.

Every floating-point order is fixed (csrc/pss.cu), so tests/pss_cases.py reproduces the device
bit for bit.  numpy in, numpy out; the work runs on the device (`_backend`, a test hook like
h36m_eval's)."""
import os

import numpy as np
import torch

from epipolarpose_b200 import ops as _ops

_backend = [_ops]
_CLUSTERS = {}        # (k, mpii_order, annotation path) -> centroids, fitted once per process


def _device():
    return torch.device("cuda") if _backend[0] is _ops else torch.device("cpu")


def _t(a, dtype=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(_device())


def normalize_poses(img_joints, fl, c_p, pelvis, root):
    """img_joints [S,J,>=3] (x px, y px, root-relative depth mm), fl / c_p [S,>=2], pelvis [S,3]
    or [S] (depth) -> [S, 3J] scale-normalised root-relative camera-frame poses."""
    p = np.asarray(img_joints, dtype=np.float64)
    if p.ndim != 3 or p.shape[2] < 3:
        raise ValueError("joints must be [S, J, >=3]")
    p = p[:, :, 0:3]
    S, J = p.shape[:2]
    pz = np.asarray(pelvis, dtype=np.float64)
    pz = pz[:, 2] if pz.ndim == 2 else pz
    cam = np.concatenate([np.asarray(fl, dtype=np.float64)[:, 0:2], np.asarray(c_p, dtype=np.float64)[:, 0:2],
                          pz.reshape(S, 1)], axis=1)
    out = torch.empty((S, J * 3), dtype=torch.float64, device=_device())
    if S:
        _backend[0].pose_normalize(_t(p), _t(cam), S, J, int(root), out)
    return out.cpu().numpy()


def fit_pose_clusters(poses, k, seed=0, n_init=10, max_iter=300):
    """k-means of poses [N, d] (the definition above): the centroids [k, d] of the restart with
    the lowest inertia."""
    ops = _backend[0]
    x = np.asarray(poses, dtype=np.float64)
    if x.ndim != 2 or n_init < 1:
        raise ValueError("poses must be [N, d] and n_init >= 1")
    N, d = x.shape
    ws = torch.empty(ops.kmeans_workspace(N, d, int(k)), dtype=torch.uint8, device=_device())
    xt = _t(x)
    cen = torch.empty((k, d), dtype=torch.float64, device=_device())
    labels = torch.empty(N, dtype=torch.int32, device=_device())
    idx = torch.empty(k, dtype=torch.int32, device=_device())
    best, best_c = None, None
    for r in range(n_init):
        inertia, _ = ops.kmeans_fit(xt, N, d, int(k), seed, r, max_iter, cen, labels, idx, None, ws)
        if best is None or inertia < best:
            best, best_c = inertia, cen.clone()
    return best_c.cpu().numpy()


def assign_clusters(poses, centroids):
    """Nearest centroid of each pose (lowest index on ties): int32 [N]."""
    x = np.asarray(poses, dtype=np.float64)
    c = np.asarray(centroids, dtype=np.float64)
    if x.ndim != 2 or c.ndim != 2 or x.shape[1] != c.shape[1]:
        raise ValueError("poses [N, d] and centroids [k, d] must share d")
    labels = torch.empty(len(x), dtype=torch.int32, device=_device())
    _backend[0].kmeans_assign(_t(x), len(x), x.shape[1], _t(c), len(c), labels, None)
    return labels.cpu().numpy()


def pose_structure_score(pred, gt, centroids):
    """Fraction of samples whose normalised prediction and ground truth share a cluster."""
    if len(pred) != len(gt):
        raise ValueError("pred and gt differ in length")
    if len(pred) == 0:
        return 0.0
    return np.count_nonzero(assign_clusters(pred, centroids) == assign_clusters(gt, centroids)) / len(pred)


def _train_poses(anno_path, mpii_order):
    from ..dataset.JointIntegralDataset import load_pickle
    from ..dataset.h36m_eval import H36M_TO_MPII_PERM
    anno = load_pickle(anno_path)
    recs = [r for key in sorted(anno) for r in anno[key]] if isinstance(anno, dict) else list(anno)
    get = lambda key: np.stack([np.asarray(r[key], dtype=np.float64) for r in recs])
    gt = get('joints_3d')
    if mpii_order:
        gt = gt[:, H36M_TO_MPII_PERM, :]
    return normalize_poses(gt, get('fl'), get('c_p'), get('pelvis'), 6 if mpii_order else 0)


def train_clusters(anno_path, ks, mpii_order):
    """{k: centroids} of the training ground truth, fitted once per process for each key."""
    keys = {k: (int(k), bool(mpii_order), os.path.abspath(anno_path)) for k in ks}
    missing = [k for k in ks if keys[k] not in _CLUSTERS]
    if missing:
        x = _train_poses(anno_path, mpii_order)
        for k in missing:
            _CLUSTERS[keys[k]] = fit_pose_clusters(x, int(k))
    return {k: _CLUSTERS[keys[k]] for k in ks}


def h36m_pss(preds, gt_joints_3d, pelvis, fl, c_p, mpii_order, ks, anno_path, centroids_file=''):
    """[('PSS@<k>', value)] for each k: preds [S,J,>=3] in the evaluation's joint order,
    gt_joints_3d [S,17,3] in H36M order.  Centroids come from `centroids_file` (an .npz with one
    array `k<k>` [k, 3J] per k) when given, else from train_clusters(anno_path, ...)."""
    from ..dataset.h36m_eval import H36M_TO_MPII_PERM
    gt = np.asarray(gt_joints_3d, dtype=np.float64)
    if mpii_order:
        gt = gt[:, H36M_TO_MPII_PERM, :]
    root = 6 if mpii_order else 0
    P = normalize_poses(preds, fl, c_p, pelvis, root)
    G = normalize_poses(gt, fl, c_p, pelvis, root)
    if centroids_file:
        with np.load(centroids_file) as f:
            cents = {k: np.asarray(f['k%d' % k], dtype=np.float64) for k in ks}
        for k, c in cents.items():
            if c.shape != (k, P.shape[1]):
                raise ValueError("%s: k%d has shape %s, expected %s" % (centroids_file, k, c.shape, (k, P.shape[1])))
    else:
        cents = train_clusters(anno_path, ks, mpii_order)
    return [('PSS@%d' % k, float(pose_structure_score(P, G, cents[k]))) for k in ks]
