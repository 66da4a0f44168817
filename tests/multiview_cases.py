"""Shared by tests/test_multiview_host.py and tests/test_gpu_multiview.py: the numpy restatement of
epb_triangulate_robust (written from its contract in include/epb.h on top of the oracle's
linear_eigen_triangulation_nview, numpy SVD instead of the kernel's one-sided Jacobi) and seeded
multi-view cases."""
import numpy as np

from oracle import restate

MAX_V = 8


def pairs(V):
    """hypothesis order: (0,1), (0,2), .., (V-2,V-1)"""
    return [(a, b) for a in range(V) for b in range(a + 1, V)]


def _reproj2(u, P, x):
    """(squared reprojection error, in front and finite) of x in one view"""
    with np.errstate(all="ignore"):
        h = P @ np.append(x, 1.0)
        d = h[:2] / h[2] - u
        e2 = float(d @ d)
    return e2, bool(h[2] > 0 and np.isfinite(e2))


def _inliers(us, Ps, usable, x, thr2):
    mask, cost = 0, 0.0
    for v in usable:
        e2, ok = _reproj2(us[v], Ps[v], x)
        ok = ok and e2 <= thr2
        mask |= int(ok) << v
        cost += e2 if ok else thr2
    return mask, cost


def _views(mask):
    return [v for v in range(MAX_V) if (mask >> v) & 1]


def _weighted_dlt(us, Ps, w, views):
    A = []
    for v in views:
        A.append(w[v] * (us[v, 0] * Ps[v, 2] - Ps[v, 0]))
        A.append(w[v] * (us[v, 1] * Ps[v, 2] - Ps[v, 1]))
    A = np.asarray(A)
    if not np.isfinite(A).all():
        return None
    with np.errstate(all="ignore"):
        _, sv, vt = np.linalg.svd(A)
        if not sv[2] > 1e-10 * sv[0]:         # rank < 3: the rays are one line
            return None
        h = vt[-1]
        x = h[:3] / h[3]
    return x if np.isfinite(x).all() and np.max(np.abs(x)) <= 1e16 else None


def robust_point(us, Ps, w, thr):
    """one joint: us [V,2], Ps [V,3,4], w [V] -> (x [3], inlier mask, resid, status)"""
    V, thr2 = len(us), thr * thr
    fail = (np.zeros(3), 0, 0.0, 0)
    usable = [v for v in range(V) if w[v] > 0 and np.isfinite(w[v]) and np.isfinite(us[v]).all()]
    best = None
    for h, (a, b) in enumerate(pairs(V)):
        if a not in usable or b not in usable:
            continue
        with np.errstate(all="ignore"):
            try:
                x, st = restate.linear_eigen_triangulation_nview(us[[a, b]][:, None], Ps[[a, b]])
            except np.linalg.LinAlgError:
                continue
        if not st[0]:
            continue
        mask, cost = _inliers(us, Ps, usable, x[0], thr2)
        key = (-bin(mask).count("1"), cost, h)
        if best is None or key < best[0]:
            best = (key, mask)
    if best is None or -best[0][0] < 2:
        return fail
    mask = best[1]
    x = _weighted_dlt(us, Ps, w, _views(mask))
    if x is None:
        return fail
    m1, _ = _inliers(us, Ps, usable, x, thr2)
    if m1 != mask:
        mask = m1
        if bin(m1).count("1") < 2:
            return fail
        x = _weighted_dlt(us, Ps, w, _views(mask))
        if x is None:
            return fail
    e2 = [_reproj2(us[v], Ps[v], x)[0] for v in _views(mask)]
    r = float(np.sqrt(np.sum(e2) / len(e2)))
    if not np.isfinite(r):
        return fail
    return x, mask, r, 1


def robust_nview_triangulation(us, Ps, weights=None, threshold_px=15.0):
    """us [V,J,>=2], Ps [V,3,4], weights [V,J] or None -> (x [J,3], status [J] int, inliers [J]
    int bit mask over the views, resid [J] px)."""
    us = np.asarray(us, dtype=np.float64)[:, :, :2]
    Ps = np.asarray(Ps, dtype=np.float64)[:, :3, :4]
    V, J = us.shape[0], us.shape[1]
    assert 2 <= V <= MAX_V
    w = np.ones((V, J)) if weights is None else np.asarray(weights, dtype=np.float64)
    x, st = np.zeros((J, 3)), np.zeros(J, dtype=np.int32)
    inl, res = np.zeros(J, dtype=np.int32), np.zeros(J)
    for j in range(J):
        x[j], inl[j], res[j], st[j] = robust_point(us[:, j], Ps, w[:, j], threshold_px)
    return x, st, inl, res


def rig(seed, NT, V, J, noise_px=3.0):
    """NT tuples of V ring cameras looking at J joints: (P [NT,V,3,4], X [NT,J,3] mm, exact
    projections [NT,V,J,2], noisy projections)"""
    rng = np.random.default_rng(seed)
    _, _, _, _, P = restate.synthetic_cameras(rng, NT, V)
    X = rng.normal(0, 400, (NT, J, 3))
    ue = np.stack([[restate.project(P[t, v], X[t]) for v in range(V)] for t in range(NT)])
    return P, X, ue, ue + rng.normal(0, noise_px, ue.shape)


def even_rig(seed, NT, V, J):
    """rig() with the V cameras spread evenly over the ring (360 / V degrees apart, +-10) at heights
    1.5 m +- 1 m: for odd V no two cameras face each other, so a point moved in one view cannot
    slide along a ray the other two share.  (P, X, exact projections)"""
    rng = np.random.default_rng(seed)
    P = np.zeros((NT, V, 3, 4))
    for t in range(NT):
        for v in range(V):
            az = np.deg2rad(20.0 + 360.0 * v / V + rng.uniform(-10, 10))
            C = np.array([4500.0 * np.cos(az), 4500.0 * np.sin(az), 1500.0 + rng.uniform(-1000, 1000)])
            zc = -C / np.linalg.norm(C)
            xc = np.cross(zc, [0.0, 0.0, 1.0])
            xc /= np.linalg.norm(xc)
            P[t, v] = restate.projection_matrix(np.stack([xc, np.cross(zc, xc), zc]), C, (1145.0, 1144.0),
                                                (512.0, 515.0))
    X = rng.normal(0, 400, (NT, J, 3))
    ue = np.stack([[restate.project(P[t, v], X[t]) for v in range(V)] for t in range(NT)])
    return P, X, ue


def plant_outliers(u, seed, px=80.0):
    """moves, for every (tuple, joint), the point of one view by px: (u', view index [NT,J])"""
    rng = np.random.default_rng(seed)
    NT, V, J = u.shape[:3]
    which = rng.integers(0, V, (NT, J))
    ang = rng.uniform(0, 2 * np.pi, (NT, J))
    out = u.copy()
    for t in range(NT):
        for j in range(J):
            out[t, which[t, j], j] += px * np.array([np.cos(ang[t, j]), np.sin(ang[t, j])])
    return out, which


def rig_inputs(T, V, seed, HW=256):
    """images [T, V, 3, HW, HW], boxes and projection matrices [T, V, 3, 4] of T synthetic rigs,
    the inputs of MultiViewPredictor"""
    rng = np.random.default_rng(seed)
    _, _, _, _, P = restate.synthetic_cameras(rng, T, V)
    x = rng.standard_normal((T, V, 3, HW, HW)).astype(np.float32)
    n = T * V
    boxes = {"center_x": 512 + rng.uniform(-20, 20, n), "center_y": 515 + rng.uniform(-20, 20, n),
             "width": rng.uniform(40, 80, n), "height": rng.uniform(40, 80, n)}
    return x, boxes, P
