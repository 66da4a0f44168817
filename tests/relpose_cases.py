"""Inputs for the relative-pose tests (CPU harness, golden fixture, GPU kernel): view pairs of the
synthetic ring rigs (oracle.restate.synthetic_cameras) looking at a 17-joint pose, with pixel
noise and joints replaced by random points (outliers)."""
import numpy as np

from oracle import restate


def rig_pairs(n, seed, J=17, noise_px=(0.0, 3.0), n_out=(0, 3), box_consistent=False, rect3d_w=2000.0,
              spread=300.0):
    """n view pairs.  Returns dict: ua, ub [n,J,2] px, intr_a, intr_b [n,4] f(2) c(2), box_a, box_b
    [n,6], R_ab [n,3,3] and t_dir [n,3] (true relative pose, unit t: X_b = R_ab X_a + t),
    X [n,J,3] world, cams (R, T, f, c, P) per view [n,2,...], outliers [n,J] bool, zroot [n,2].
    spread: std of the joints around the origin (mm).  box_consistent: boxes with bb_w scale Z_root / f_x = rect3d_w in both views."""
    rng = np.random.default_rng(seed)
    R, T, f, c, P = restate.synthetic_cameras(rng, n, 4)
    out = {k: [] for k in ("ua", "ub", "intr_a", "intr_b", "box_a", "box_b", "R_ab", "t_dir", "X",
                           "R", "T", "f", "c", "P", "outliers", "zroot")}
    for i in range(n):
        va, vb = rng.choice(4, size=2, replace=False)
        X = rng.normal(0.0, spread, size=(J, 3))
        X[0] = rng.normal(0.0, 100.0, size=3)               # root near the rig's centre
        sigma = rng.uniform(*noise_px)
        k_out = int(rng.integers(n_out[0], n_out[1] + 1))
        bad = np.zeros(J, bool)
        if k_out:
            bad[rng.choice(np.arange(1, J), size=k_out, replace=False)] = True
        uv, boxes, zr = [], [], []
        for v in (va, vb):
            u = restate.project(P[i, v], X) + rng.normal(0.0, 1.0, (J, 2)) * sigma
            u[bad] = rng.uniform(0.0, 1024.0, (k_out, 2))
            z0 = (R[i, v] @ (X[0] - T[i, v]))[2]
            scale = rng.uniform(0.8, 1.25)
            w = f[i, v, 0] * rect3d_w / (scale * z0) if box_consistent else rng.uniform(600.0, 1000.0)
            boxes.append([u[0, 0] + rng.uniform(-30, 30), u[0, 1] + rng.uniform(-30, 30), w, w, scale,
                          rng.uniform(-20, 20) if not box_consistent else 0.0])
            uv.append(u)
            zr.append(z0)
        Ra, Rb = R[i, va], R[i, vb]
        Rab = Rb @ Ra.T
        tab = Rb @ (T[i, va] - T[i, vb])
        out["ua"].append(uv[0]); out["ub"].append(uv[1])
        out["intr_a"].append(np.concatenate([f[i, va], c[i, va]]))
        out["intr_b"].append(np.concatenate([f[i, vb], c[i, vb]]))
        out["box_a"].append(boxes[0]); out["box_b"].append(boxes[1])
        out["R_ab"].append(Rab); out["t_dir"].append(tab / np.linalg.norm(tab))
        out["X"].append(X); out["outliers"].append(bad); out["zroot"].append(zr)
        for k, a in (("R", R), ("T", T), ("f", f), ("c", c), ("P", P)):
            out[k].append(np.stack([a[i, va], a[i, vb]]))
    return {k: np.asarray(v) for k, v in out.items()}
