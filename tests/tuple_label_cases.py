"""Shared by tests/test_tuple_labels_host.py and tests/test_gpu_tuple_labels.py: a float64 numpy
restatement of epb_tuple_labels (written from its contract in include/epb.h on top of the oracle's
trans_coords_from_patch_to_org_3d for patch -> image, tests/multiview_cases.py::robust_point for
the robust fit and the oracle's labels_from_global_coords for the projection, plus the weight rule),
seeded view-major batches of ring-camera tuples with known joints, and the small robust-step model
and SyntheticH36M batch that test_gpu_tuple_labels and the coverage gate of tests/test_step_coverage.py
train on."""
import numpy as np

from oracle import restate
from tests import multiview_cases as mc

PATCH, RECT = 256, 2000
BOX_KEYS = ("center_x", "center_y", "width", "height", "scale", "rot")


def image_points(coords, meta):
    """coords [B, J*3] float32 soft-argmax output -> image points [B, J, 2] (px)"""
    res = restate.joint_location_result(PATCH, PATCH, np.asarray(coords, dtype=np.float32))
    return np.stack([restate.trans_coords_from_patch_to_org_3d(
        res[i], *(float(meta[k][i]) for k in BOX_KEYS[:4]), PATCH, PATCH, RECT, RECT,
        scale=float(meta["scale"][i]), rot=float(meta["rot"][i]))[:, :2] for i in range(len(res))])


def tuple_labels(coords, lse, meta, V, thr=15.0, tuples=None):
    """The restatement: coords [B, J*3] float32 (row v*T + t is view v of tuple t), lse [B, J, 2] or
    None, meta (numpy: the box keys, R [B,3,3], T [B,3(,1)], f, c [B,2], projection_matrix [B,3,4])
    -> (label [B, J*3] float32, weight [B, J*3] float32, X [T,J,3], status, inliers [T,J] int32,
    resid [T,J]).  `tuples`: restate only these tuples (the other rows and tuples stay 0)."""
    coords = np.asarray(coords, dtype=np.float32)
    B, J = coords.shape[0], coords.shape[1] // 3
    T = B // V
    ts = range(T) if tuples is None else tuples
    rows = np.array([v * T + t for v in range(V) for t in ts], dtype=np.int64)
    sub = {k: np.asarray(meta[k])[rows] for k in BOX_KEYS}
    u = np.zeros((B, J, 2))
    u[rows] = image_points(coords[rows], sub)
    P = np.asarray(meta["projection_matrix"], dtype=np.float64)[:, :3, :4]
    w = np.ones((B, J)) if lse is None else \
        np.asarray(lse, dtype=np.float32).reshape(B, J, 2)[:, :, 1].astype(np.float64)
    X, st = np.zeros((T, J, 3)), np.zeros((T, J), dtype=np.int32)
    inl, res = np.zeros((T, J), dtype=np.int32), np.zeros((T, J))
    for t in ts:
        r = [v * T + t for v in range(V)]
        for j in range(J):
            X[t, j], inl[t, j], res[t, j], st[t, j] = mc.robust_point(u[r, j], P[r], w[r, j], thr)
    tr = rows % T
    Xr = X[tr]
    m = {k: np.asarray(meta[k])[rows] for k in BOX_KEYS + ("R", "T", "f", "c")}
    with np.errstate(all="ignore"):
        lab, _ = restate.labels_from_global_coords(Xr, m)
        Rm = np.asarray(m["R"], dtype=np.float64).reshape(-1, 3, 3)
        Tm = np.asarray(m["T"], dtype=np.float64).reshape(-1, 1, 3)
        cz = np.einsum("bjk,bk->bj", Xr - Tm, Rm[:, 2])           # camera-frame depth, X_cam = R (X - T)
    lab = lab.reshape(len(rows), J, 3)
    ok = (st[tr] == 1) & (st[tr, :1] == 1) & (cz > 0) & np.isfinite(cz) & (cz[:, :1] > 0) & \
        np.isfinite(cz[:, :1]) & np.isfinite(lab).all(axis=2)
    label, weight = np.zeros((B, J, 3), np.float32), np.zeros((B, J, 3), np.float32)
    label[rows] = np.where(ok[:, :, None], lab, 0.0)
    weight[rows] = np.repeat(ok[:, :, None], 3, axis=2)
    return label.reshape(B, J * 3), weight.reshape(B, J * 3), X, st, inl, res


def case(seed, T, V, J, noise_px=3.0, outliers=0.0, lse=False):
    """T tuples of V ring cameras (restate.synthetic_cameras) looking at J joints, laid out
    view-major.  The 2-D joints are the exact projections plus noise_px of noise; in a share
    `outliers` of the (tuple, joint)s one view is moved by 80 px (multiview_cases.plant_outliers).
    Boxes around the image centre, scale 0.8..1.2, rotation -30..30 degrees.  -> (coords [B, J*3]
    float32, lse [B, J, 2] float32 or None, meta (numpy), world joints [T,J,3], outlier mask [T,J])"""
    rng = np.random.default_rng(seed)
    R, C, f, c, P = restate.synthetic_cameras(rng, T, V)
    Xw = rng.normal(0, 400, (T, J, 3))
    u = np.stack([[restate.project(P[t, v], Xw[t]) for v in range(V)] for t in range(T)])
    u = u + rng.normal(0, noise_px, u.shape)
    hit = np.zeros((T, J), dtype=bool)
    if outliers:
        uo, _ = mc.plant_outliers(u, seed + 1)
        hit = rng.uniform(size=(T, J)) < outliers
        u = np.where(hit[:, None, :, None], uo, u)
    B = V * T
    order = [(t, v) for v in range(V) for t in range(T)]
    meta = {"center_x": 512 + rng.uniform(-40, 40, B), "center_y": 515 + rng.uniform(-40, 40, B),
            "width": 1000 + rng.uniform(-100, 100, B), "height": 1000 + rng.uniform(-100, 100, B),
            "scale": rng.uniform(0.8, 1.2, B), "rot": rng.uniform(-30, 30, B),
            "R": np.stack([R[o] for o in order]), "T": np.stack([C[o].reshape(3, 1) for o in order]),
            "f": np.stack([f[o] for o in order]), "c": np.stack([c[o] for o in order]),
            "projection_matrix": np.stack([P[o] for o in order])}
    coords = np.zeros((B, J, 3))
    for i, (t, v) in enumerate(order):
        tr = restate.gen_trans_from_patch(meta["center_x"][i], meta["center_y"][i], meta["width"][i],
                                          meta["height"][i], PATCH, PATCH, meta["scale"][i], meta["rot"][i],
                                          inv=False)
        p = np.concatenate([u[t, v], np.ones((J, 1))], axis=1) @ tr.T
        coords[i, :, 0] = p[:, 0] / PATCH - 0.5
        coords[i, :, 1] = p[:, 1] / PATCH - 0.5
        coords[i, :, 2] = rng.uniform(-0.3, 0.3, J)
    ls = None
    if lse:
        ls = np.stack([rng.uniform(0, 20, (B, J)), rng.uniform(0.02, 1.0, (B, J))], axis=2).astype(np.float32)
    return coords.reshape(B, J * 3).astype(np.float32), ls, meta, Xw, hit


def packed(meta):
    """meta -> (box [B,6], P [B,12], cam [B,16]) float64 in the kernel layouts"""
    B = len(meta["center_x"])
    box = np.stack([np.asarray(meta[k], dtype=np.float64) for k in BOX_KEYS], axis=1)
    P = np.asarray(meta["projection_matrix"], dtype=np.float64)[:, :3, :4].reshape(B, 12)
    cam = np.concatenate([np.asarray(meta["R"], np.float64).reshape(B, 9), np.asarray(meta["T"], np.float64).reshape(B, 3),
                          np.asarray(meta["f"], np.float64).reshape(B, 2), np.asarray(meta["c"], np.float64).reshape(B, 2)],
                         axis=1)
    return box, P, cam


def r18(dev, J, D, HW, seed=0):
    """R18 (f16x3) of J joints, D depth bins, HW x HW images in train mode, with FusedAdam"""
    import torch
    import lib.models as models
    import lib.utils.utils as U
    from oracle import refshim
    torch.manual_seed(seed)
    cfg = refshim.make_cfg(num_layers=18, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    m = models.pose3d_resnet.get_pose_net(cfg, False, precision="f16x3").to(dev).train()
    return m, U.FusedAdam(list(m.parameters()), lr=1e-4)


def synthetic_batch(J, HW, tuples, views=4):
    """one view-major batch of SyntheticH36M through tuple_batch_sampler and loader_batch"""
    from torch.utils.data import default_collate
    from lib.core.config import AttrDict, _DEFAULTS
    from lib.core.function import loader_batch
    from lib.dataset.synthetic import SyntheticH36M
    c = AttrDict(_DEFAULTS)
    c.MODEL.NUM_JOINTS, c.MODEL.IMAGE_SIZE, c.DATASET.SYNTHETIC_LEN = J, [HW, HW], 4 * tuples
    ds = SyntheticH36M(c)
    idx = next(iter(ds.tuple_batch_sampler(tuples, views)))
    return loader_batch(default_collate([ds[i] for i in idx]))
