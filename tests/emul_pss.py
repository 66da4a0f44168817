"""TEST INFRASTRUCTURE: CPU emulation of the Pose Structure Score entry points of libepb.so
(epb_pose_normalize, epb_kmeans_workspace, epb_kmeans_fit, epb_kmeans_assign) with the SAME
signatures as epipolarpose_b200.ops, on torch CPU tensors.  It runs the numpy restatement of
tests/pss_cases.py and raises EpbError where the C ABI returns EPB_EINVAL, so that host tests can
swap it in as lib/core/pss.py's backend (`pss._backend[0]`).  Never imported by the product path."""
import numpy as np
import torch

from epipolarpose_b200._lib import EpbError
from tests import pss_cases as pc


def _error(e):
    return EpbError("libepb call failed (-1): %s" % e)


def pose_normalize(pose, cam, S, J, root, out):
    out.view(S, J * 3).copy_(torch.from_numpy(pc.normalize(pose.reshape(S, J, 3).numpy(), cam.reshape(S, 5).numpy(),
                                                           root)))


def kmeans_workspace(N, d, k):
    if k < 1 or k > N or d < 1:
        raise _error("k = %d outside [1, N = %d]" % (k, N))
    return 1


def kmeans_fit(x, N, d, k, seed, restart, max_iter, centroids, labels, init_idx, trace, ws):
    """One restart of the restatement; returns (inertia, updates done)."""
    try:
        f = pc.fit_restart(x.reshape(N, d).numpy(), k, int(seed), restart, max_iter)
    except ValueError as e:
        raise _error(e)
    centroids.view(k, d).copy_(torch.from_numpy(f["centroids"]))
    labels.copy_(torch.from_numpy(f["labels"]))
    init_idx.copy_(torch.from_numpy(f["init_idx"]))
    if trace is not None:
        trace.view(-1, N)[:len(f["trace"])].copy_(torch.from_numpy(f["trace"]))
    return f["inertia"], f["n_iter"]


def kmeans_assign(x, N, d, centroids, k, labels, dist2):
    xs, cs = x.reshape(N, d).numpy(), centroids.reshape(k, d).numpy()
    if not (np.isfinite(xs).all() and np.isfinite(cs).all()):
        raise _error("k-means assign: non-finite point or centroid")
    lab, d2 = pc.assign(xs, cs)
    labels.copy_(torch.from_numpy(lab))
    if dist2 is not None:
        dist2.copy_(torch.from_numpy(d2))
