"""Two-view triangulation -- host-side mirror of the reference
lib/utils/triangulation.py function surface:
    f(u1[J,2], P1[>=3,4], u2[J,2], P2[>=3,4]) -> (x[J,3] of output_dtype, status[J])
for linear_eigen_triangulation (:8-27, homogeneous DLT = cv2.triangulatePoints),
linear_LS_triangulation (:34-97) and iterative_LS_triangulation (:104-181), plus
set_triangl_output_dtype (:226-232).  The arithmetic (float64 one-sided Jacobi
SVD per joint) runs in the sm_90a kernel epb_triangulate; numpy in / numpy out
like the reference.  `triangulate_pairs` is the batched tensor API the training
loop uses (no host round trip).  polynomial_triangulation (:184-220: fundamental matrix
from the projection matrices, cv2.correctMatches = Hartley-Sturm optimal correction, then
the homogeneous DLT) runs as method "polynomial" of the same kernel, including the reference's
8-point fallback (:215-217): when the correction is NaN for every joint of a pair, F is
re-estimated from the matches (cv2.findFundamentalMat FM_8POINT) on the device and the
correction repeated; "polynomial_8point" runs that branch unconditionally.
`relative_pose_pairs` estimates each pair's projection matrices from the 2-D joints alone
(self-supervision without camera extrinsics).
`triangulate_views_robust` / `robust_nview_triangulation` (not in the reference) triangulate each
joint of a calibrated rig of 2..8 views by consensus over the view pairs, leaving out and reporting
the views that disagree (epb_triangulate_robust)."""
import numpy as np
import torch

from epipolarpose_b200 import ops as _ops

_backend = [_ops]
METHODS = {"linear_eigen": 0, "linear_LS": 1, "iterative_LS": 2, "polynomial": 3,
           "polynomial_8point": 4,
           "eigen": 0, "ls": 1, "iterative": 2}

output_dtype = float


def set_triangl_output_dtype(output_dtype_):
    global output_dtype
    output_dtype = output_dtype_


def triangulate_pairs(u1, u2, P1, P2, method="iterative", tolerance=3.e-5, stride_u=None):
    """u1,u2 [NP,J,S>=2] float64 (first two columns used), P1,P2 [NP,3,4] float64,
    all on the device -> (X [NP,J,3] float64, status [NP,J] int32)."""
    ops = _backend[0]
    NP, J = u1.shape[0], u1.shape[1]
    S = u1.shape[2] if stride_u is None else stride_u
    X = torch.empty((NP, J, 3), device=u1.device, dtype=torch.float64)
    status = torch.empty((NP, J), device=u1.device, dtype=torch.int32)
    if NP * J:
        ops.triangulate(u1.contiguous(), u2.contiguous(), S, P1.contiguous(), P2.contiguous(),
                        NP, J, METHODS[method], tolerance, X, status)
    return X, status


def triangulate_views(u, P):
    """V-view homogeneous DLT (2 <= V <= 4; not in the reference, SURVEY 8(f) row 3):
    u [NT,V,J,S>=2] float64, P [NT,V,3,4] float64 on the device -> (X [NT,J,3], status [NT,J])."""
    ops = _backend[0]
    NT, V, J = u.shape[0], u.shape[1], u.shape[2]
    if not 2 <= V <= 4:
        raise ValueError("triangulate_views handles 2..4 views per tuple, got %d" % V)
    X = torch.empty((NT, J, 3), device=u.device, dtype=torch.float64)
    status = torch.empty((NT, J), device=u.device, dtype=torch.int32)
    if NT * J:
        ops.triangulate_nview(u.contiguous(), u.shape[3], P.reshape(NT, V, 12).contiguous(), NT, V, J, X, status)
    return X, status


DEFAULT_THRESHOLD_PX = 15.0


def triangulate_views_robust(u, P, weights=None, threshold_px=DEFAULT_THRESHOLD_PX, out=None):
    """Robust V-view triangulation (2 <= V <= 8; epb_triangulate_robust, see include/epb.h):
    u [NT,V,J,S>=2] float64 image px, P [NT,V,3,4] float64, weights [NT,V,J] float64 >= 0 or None
    (ones; 0 = the view is absent for that joint), all on the device -> (X [NT,J,3] float64,
    status [NT,J] int32, inliers [NT,J] int32 bit mask over the views, resid [NT,J] float64 RMS
    reprojection error in px over the inlier views).  Joints with status 0 have X = 0, inliers = 0
    and resid = 0.  `out`: the four result tensors to write into (for graph capture)."""
    ops = _backend[0]
    NT, V, J = u.shape[0], u.shape[1], u.shape[2]
    if not 2 <= V <= 8:
        raise ValueError("triangulate_views_robust handles 2..8 views per tuple, got %d" % V)
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError("threshold_px must be a positive number of pixels, got %r" % (threshold_px,))
    if weights is not None and tuple(weights.shape) != (NT, V, J):
        raise ValueError("weights must be [NT, V, J] = %s, got %s" % ((NT, V, J), tuple(weights.shape)))
    if out is None:
        out = (torch.empty((NT, J, 3), device=u.device, dtype=torch.float64),
               torch.empty((NT, J), device=u.device, dtype=torch.int32),
               torch.empty((NT, J), device=u.device, dtype=torch.int32),
               torch.empty((NT, J), device=u.device, dtype=torch.float64))
    X, status, inliers, resid = out
    if NT * J:
        ops.triangulate_robust(u.contiguous(), u.shape[3], P.reshape(NT, V, 12).contiguous(),
                               None if weights is None else weights.contiguous(), NT, V, J,
                               threshold_px, X, inliers, resid, status)
    return X, status, inliers, resid


def relative_pose_pairs(kps, intr, box, rect3d_w=2000.0, diag=False):
    """Camera geometry of each view pair from its own 2-D joints (no extrinsics; epb_relative_pose):
    sample i pairs with i + B/2.  kps [B,J,S>=2] image px, intr [B,4] f(2) c(2), box [B,6], all
    float64 on the device (B even, 8 <= J <= 32) -> (P_a [NP,3,4], P_b [NP,3,4], cam [B,16],
    inliers [NP,J] int32, status [NP] int32), NP = B/2; with diag=True also diag [NP,3] int32
    (chosen hypothesis, chosen candidate, inlier count).  P_a = K_a[I|0], P_b = K_b[R|t] with t
    scaled so that each box spans rect3d_w mm at the root joint's depth; failed pairs have
    status 0, R = I and t = 0."""
    ops = _backend[0]
    B, J = kps.shape[0], kps.shape[1]
    if B % 2:
        raise ValueError("relative_pose_pairs pairs sample i with i + B/2: B must be even, got %d" % B)
    if not 8 <= J <= 32:
        raise ValueError("relative_pose_pairs needs 8 <= J <= 32 joints, got %d" % J)
    NP, dev = B // 2, kps.device
    Pa = torch.empty((NP, 3, 4), device=dev, dtype=torch.float64)
    Pb = torch.empty((NP, 3, 4), device=dev, dtype=torch.float64)
    cam = torch.empty((B, 16), device=dev, dtype=torch.float64)
    inliers = torch.empty((NP, J), device=dev, dtype=torch.int32)
    status = torch.empty((NP,), device=dev, dtype=torch.int32)
    dg = torch.empty((NP, 3), device=dev, dtype=torch.int32) if diag else None
    if NP:
        ops.relative_pose(kps.contiguous(), kps.shape[2], intr.contiguous(), box.contiguous(), B, J,
                          rect3d_w, Pa, Pb, cam, inliers, status, dg)
    out = (Pa, Pb, cam, inliers, status)
    return out + (dg,) if diag else out


def _device():
    return torch.device("cuda") if _backend[0] is _ops else torch.device("cpu")


def _run(u1, P1, u2, P2, method, tolerance=3.e-5):
    u1 = np.ascontiguousarray(u1, dtype=np.float64)
    u2 = np.ascontiguousarray(u2, dtype=np.float64)
    assert u1.ndim == 2 and u1.shape == u2.shape and u1.shape[1] >= 2
    dev = _device()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    X, st = triangulate_pairs(t(u1)[None], t(u2)[None], t(np.asarray(P1)[0:3, 0:4])[None],
                              t(np.asarray(P2)[0:3, 0:4])[None], method, tolerance)
    return X[0].cpu().numpy(), st[0].cpu().numpy()


def linear_eigen_triangulation(u1, P1, u2, P2, max_coordinate_value=1.e16):
    x, st = _run(u1, P1, u2, P2, "linear_eigen")
    if max_coordinate_value != 1.e16:
        with np.errstate(invalid="ignore"):
            st = np.max(np.abs(x), axis=1) <= max_coordinate_value
    return x.astype(output_dtype), st.astype(bool)


def linear_LS_triangulation(u1, P1, u2, P2):
    x, _ = _run(u1, P1, u2, P2, "linear_LS")
    return x.astype(output_dtype), np.ones(len(u1), dtype=bool)


def iterative_LS_triangulation(u1, P1, u2, P2, tolerance=3.e-5):
    x, st = _run(u1, P1, u2, P2, "iterative_LS", tolerance)
    return x.astype(output_dtype), st.astype(int)


def polynomial_triangulation(u1, P1, u2, P2):
    x, st = _run(u1, P1, u2, P2, "polynomial")
    return x.astype(output_dtype), st.astype(bool)


def robust_nview_triangulation(us, Ps, weights=None, threshold_px=DEFAULT_THRESHOLD_PX):
    """One tuple of a calibrated rig, numpy in / numpy out: us [V,J,>=2], Ps [V,>=3,4], weights [V,J]
    or None -> (x [J,3] of output_dtype, status [J] bool, inliers [J] int bit mask over the views,
    resid [J] px).  See triangulate_views_robust.  The default threshold, in original-image pixels,
    is a guess: it has not been tuned on real predictions."""
    us = np.ascontiguousarray(us, dtype=np.float64)
    assert us.ndim == 3 and us.shape[2] >= 2
    dev = _device()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    P = np.stack([np.asarray(p, dtype=np.float64)[0:3, 0:4] for p in Ps])
    X, st, inl, res = triangulate_views_robust(t(us)[None], t(P)[None],
                                               None if weights is None else t(weights)[None], threshold_px)
    return (X[0].cpu().numpy().astype(output_dtype), st[0].cpu().numpy().astype(bool),
            inl[0].cpu().numpy().astype(int), res[0].cpu().numpy())
