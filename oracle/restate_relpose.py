"""TEST INFRASTRUCTURE ONLY -- numpy float64 restatement of the relative-pose estimator
(csrc/geometry.cu relative_pose_kernel, include/epb.h epb_relative_pose): self-supervision
without camera extrinsics.  The reference only sketches this step (lib/utils/cameras.py:133-143,
Camera.get_essential_matrix / get_fundamental_matrix with cv2.FM_LMEDS, no caller); the rules
below are this project's, restated independently of the CUDA code with numpy.linalg:

  1. LMedS F: hypothesis h (0..255) fits oracle.restate.fundamental_8point to the first 8 entries
     of a Fisher-Yates shuffle of 0..J-1 driven by splitmix64 seeded with h; score = lower median
     over all J joints of the squared Sampson distance (px^2, non-finite -> inf); invalid: a
     non-finite scheduled joint, no 8-point F, or an infinite score.  Best = lowest score, ties to
     the lowest h.  Inliers: r^2 <= max((2.5 sigma)^2, 1e-6), sigma = 1.4826 (1 + 5/(J-8))
     sqrt(score) (every finite joint when J = 8); refit on the inliers.
  2. E = K_b^T F K_a; SVD (numpy), u3 = u1 x u2, v3 = v1 x v2, (u1, v1, u3, v3) negated when the
     largest-magnitude entry of u3 is negative; candidates (UWV^T, u3), (UWV^T, -u3),
     (UW^TV^T, u3), (UW^TV^T, -u3); most inliers in front of both cameras (homogeneous DLT with
     K_a[I|0], K_b[R|t]) wins, ties to the first.
  3. |t| = 1 root (joint 0) depths Z_a, Z_b; s_v = f_x,v rect3d_w / (bb_w,v scale_v Z_v);
     t <- sqrt(s_a s_b) t.
  4. P_a = K_a[I|0], P_b = K_b[R|t]; cam rows R(9) T(3) f(2) c(2): a = (I, 0), b = (R, -R^T t).
"""
import numpy as np

from oracle import restate

N_HYP = 256
_M64 = (1 << 64) - 1


def splitmix64_stream(seed):
    s = seed & _M64
    while True:
        s = (s + 0x9E3779B97F4A7C15) & _M64
        z = s
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
        yield z ^ (z >> 31)


def hypothesis_joints(h, J):
    """The 8 joints of hypothesis h: partial Fisher-Yates over 0..J-1 driven by splitmix64(h)."""
    perm = list(range(J))
    g = splitmix64_stream(h)
    for k in range(8):
        r = k + next(g) % (J - k)
        perm[k], perm[r] = perm[r], perm[k]
    return perm[:8]


def sampson2(F, ua, ub):
    """Squared Sampson distance (px^2) of each match, +inf where not finite."""
    x1, y1, x2, y2 = ua[:, 0], ua[:, 1], ub[:, 0], ub[:, 1]
    with np.errstate(all="ignore"):
        f0 = F[0, 0] * x1 + F[0, 1] * y1 + F[0, 2]
        f1 = F[1, 0] * x1 + F[1, 1] * y1 + F[1, 2]
        f2 = F[2, 0] * x1 + F[2, 1] * y1 + F[2, 2]
        g0 = F[0, 0] * x2 + F[1, 0] * y2 + F[2, 0]
        g1 = F[0, 1] * x2 + F[1, 1] * y2 + F[2, 1]
        e = x2 * f0 + y2 * f1 + f2
        r = e * e / (f0 * f0 + f1 * f1 + g0 * g0 + g1 * g1)
    return np.where(np.isfinite(r), r, np.inf)


_SCHEDULE = {}


def schedule(J):
    if J not in _SCHEDULE:
        _SCHEDULE[J] = np.array([hypothesis_joints(h, J) for h in range(N_HYP)])
    return _SCHEDULE[J]


def fundamental_8point_batch(a, b):
    """oracle.restate.fundamental_8point over a batch of point sets a, b [H,n,2] -> (F [H,3,3],
    valid [H]); the same steps, batched through numpy.linalg."""
    a = a.astype(np.float32).astype(np.float64)
    b = b.astype(np.float32).astype(np.float64)
    c1, c2 = a.mean(1, keepdims=True), b.mean(1, keepdims=True)
    s1 = np.sqrt(((a - c1) ** 2).sum(2)).mean(1)
    s2 = np.sqrt(((b - c2) ** 2).sum(2)).mean(1)
    eps32 = np.finfo(np.float32).eps
    valid = (s1 >= eps32) & (s2 >= eps32)
    with np.errstate(all="ignore"):
        s1, s2 = np.sqrt(2.0) / s1, np.sqrt(2.0) / s2
        p, q = (a - c1) * s1[:, None, None], (b - c2) * s2[:, None, None]
    p = np.where(valid[:, None, None], p, 0.0)
    q = np.where(valid[:, None, None], q, 0.0)
    r = np.stack([q[..., 0] * p[..., 0], q[..., 0] * p[..., 1], q[..., 0], q[..., 1] * p[..., 0],
                  q[..., 1] * p[..., 1], q[..., 1], p[..., 0], p[..., 1], np.ones(p.shape[:2])], axis=2)
    w, v = np.linalg.eigh(np.einsum("hia,hib->hab", r, r))
    valid &= (np.abs(w) >= np.finfo(np.float64).eps).sum(1) >= 8
    F0 = v[:, :, 0].reshape(-1, 3, 3)
    U, sv, Vt = np.linalg.svd(F0)
    sv[:, 2] = 0.0
    F0 = U @ (sv[:, :, None] * Vt)
    z = np.zeros_like(s1)
    with np.errstate(all="ignore"):
        return _denormalise(F0, s1, s2, c1, c2, z, eps32), valid


def _denormalise(F0, s1, s2, c1, c2, z, eps32):
    T1 = np.stack([np.stack([s1, z, -s1 * c1[:, 0, 0]], 1), np.stack([z, s1, -s1 * c1[:, 0, 1]], 1),
                   np.stack([z, z, z + 1], 1)], 1)
    T2 = np.stack([np.stack([s2, z, -s2 * c2[:, 0, 0]], 1), np.stack([z, s2, -s2 * c2[:, 0, 1]], 1),
                   np.stack([z, z, z + 1], 1)], 1)
    F = np.transpose(T2, (0, 2, 1)) @ F0 @ T1
    big = np.abs(F[:, 2, 2]) > eps32
    F[big] = F[big] / F[big, 2, 2][:, None, None]
    return F


def hypothesis_scores(ua, ub):
    """[N_HYP] LMedS scores (NaN: invalid hypothesis) and the hypotheses' F [N_HYP,3,3]."""
    J = len(ua)
    idx = schedule(J)
    a, b = ua[idx], ub[idx]
    fin = np.isfinite(a).all((1, 2)) & np.isfinite(b).all((1, 2))
    F, valid = fundamental_8point_batch(np.where(fin[:, None, None], a, 0.0),
                                        np.where(fin[:, None, None], b, 0.0))
    valid &= fin
    scores = np.full(N_HYP, np.nan)
    for h in np.nonzero(valid)[0]:
        s = np.sort(sampson2(F[h], ua, ub))[(J - 1) // 2]
        if np.isfinite(s):
            scores[h] = s
    return scores, F


def _K(intr):
    return np.array([[intr[0], 0.0, intr[2]], [0.0, intr[1], intr[3]], [0.0, 0.0, 1.0]])


def candidates(E):
    """The four (R, unit t) of E, in the fixed order of the kernel."""
    U, _, Vt = np.linalg.svd(E)
    u1, u2, v1, v2 = U[:, 0].copy(), U[:, 1].copy(), Vt[0].copy(), Vt[1].copy()
    u3, v3 = np.cross(u1, u2), np.cross(v1, v2)
    if u3[np.argmax(np.abs(u3))] < 0:
        u1, v1, u3, v3 = -u1, -v1, -u3, -v3
    p = np.outer(u2, v1) - np.outer(u1, v2)
    q = np.outer(u3, v3)
    R1, R2 = p + q, q - p
    return [(R1, u3), (R1, -u3), (R2, u3), (R2, -u3)]


def _P(intr, R, t):
    return _K(intr) @ np.concatenate([R, np.asarray(t).reshape(3, 1)], axis=1)


def _depths(ua, ub, Pa, Pb, R, t):
    """Homogeneous DLT of each match -> (finite, depth in a, depth in b)."""
    X, ok = restate.linear_eigen_triangulation(ua, Pa, ub, Pb)
    with np.errstate(all="ignore"):
        return ok, X[:, 2], X @ R[2] + t[2]


def relative_pose(ua, ub, intr_a, intr_b, box_a, box_b, rect3d_w=2000.0):
    """One view pair: ua, ub [J,>=2] image px; intr f(2) c(2); box c_x c_y w h scale rot.
    Returns a dict with P_a, P_b [3,4], cam_a, cam_b [16], inliers [J] bool, status (0/1),
    best_h / cand (-1: not reached), n_inl, scores [N_HYP], F (refit), counts [4]."""
    ua = np.asarray(ua, dtype=np.float64)[:, :2]
    ub = np.asarray(ub, dtype=np.float64)[:, :2]
    intr_a = np.asarray(intr_a, dtype=np.float64)
    intr_b = np.asarray(intr_b, dtype=np.float64)
    J = len(ua)
    scores, Fs = hypothesis_scores(ua, ub)
    out = dict(scores=scores, best_h=-1, cand=-1, n_inl=0, inliers=np.zeros(J, bool), status=0,
               F=None, counts=np.zeros(4, int))
    R, t = np.eye(3), np.zeros(3)
    ok = bool(np.isfinite(scores).any())
    if ok:
        h = int(np.nanargmin(scores))                  # first occurrence of the minimum
        out["best_h"] = h
        if J > 8:
            sig = 1.4826 * (1.0 + 5.0 / (J - 8)) * np.sqrt(scores[h])
            thr = max((2.5 * sig) * (2.5 * sig), 1e-6)
        else:
            thr = np.finfo(np.float64).max
        inl = sampson2(Fs[h], ua, ub) <= thr
        out["inliers"], out["n_inl"] = inl, int(inl.sum())
        ok = out["n_inl"] >= 8
    if ok:
        F = restate.fundamental_8point(ua[out["inliers"]], ub[out["inliers"]])
        ok = F is not None
        out["F"] = F
    if ok:
        E = _K(intr_b).T @ F @ _K(intr_a)
        out["E"] = E
        ok = bool(np.isfinite(E).all())
    if ok:
        cands = candidates(E)
        ok = all(np.isfinite(Rc).all() for Rc, _ in cands)
    if ok:
        Pa = _P(intr_a, np.eye(3), np.zeros(3))
        inl = out["inliers"]
        for c, (Rc, tc) in enumerate(cands):
            fin, za, zb = _depths(ua[inl], ub[inl], Pa, _P(intr_b, Rc, tc), Rc, tc)
            out["counts"][c] = int((fin & (za > 0) & (zb > 0)).sum())
        win = int(np.argmax(out["counts"]))
        out["cand"] = win
        n = out["counts"][win]
        ok = n >= (out["n_inl"] + 1) // 2 and n >= 8
        R, t = cands[win]
    if ok:
        fin, za, zb = _depths(ua[:1], ub[:1], Pa, _P(intr_b, R, t), R, t)
        ok = bool(fin[0] and za[0] > 0 and zb[0] > 0)
        if ok:
            sa = intr_a[0] * rect3d_w / (box_a[2] * box_a[4] * za[0])
            sb = intr_b[0] * rect3d_w / (box_b[2] * box_b[4] * zb[0])
            t = np.sqrt(sa * sb) * t
    if ok:
        T = -(R.T @ t)
        ok = bool(np.isfinite(_P(intr_b, R, t)).all() and np.isfinite(T).all())
    if not ok:
        R, t = np.eye(3), np.zeros(3)
    T = -(R.T @ t) if ok else np.zeros(3)
    out["status"] = int(ok)
    out["R"], out["t"] = R, t
    out["P_a"] = _P(intr_a, np.eye(3), np.zeros(3))
    out["P_b"] = _P(intr_b, R, t)
    out["cam_a"] = np.concatenate([np.eye(3).reshape(9), np.zeros(3), intr_a])
    out["cam_b"] = np.concatenate([R.reshape(9), T, intr_b])
    return out
