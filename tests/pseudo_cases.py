"""Shared by tests/test_pseudo_labels_host.py and tests/test_gpu_pseudo_labels.py: a float64 numpy
restatement of epb_pseudo_records (from_worldjt_to_imagejt, reference lib/utils/prep_h36m.py:176-204,
on the projection of oracle/restate.py::labels_from_global_coords), seeded cases, and a torch-CPU
emulation of the two entry points lib/utils/prep_h36m.py calls (same signatures as
epipolarpose_b200.ops)."""
import numpy as np
import torch

from oracle import restate


def restated(X, status, cam, root):
    """X [T,S,J,3], status [T,S,J], cam [T,V,16] -> (joints_3d [T,V,J,3], vis, pelvis [T,V,3], ok [T,V])."""
    X, cam = np.asarray(X, np.float64), np.asarray(cam, np.float64)
    T, S, J = X.shape[:3]
    V = cam.shape[1]
    jt, vis = np.zeros((T, V, J, 3)), np.zeros((T, V, J, 3))
    pel, ok = np.zeros((T, V, 3)), np.zeros((T, V), np.int32)
    for t in range(T):
        for v in range(V):
            s = 0 if S == 1 else v
            R, Tc, f, c = cam[t, v, :9].reshape(3, 3), cam[t, v, 9:12], cam[t, v, 12:14], cam[t, v, 14:16]
            with np.errstate(all="ignore"):
                pc = (X[t, s] - Tc) @ R.T                           # prep_h36m.py:186
                u = pc[:, 0] / pc[:, 2] * f[0] + c[0]              # CamProj :170-175
                w = pc[:, 1] / pc[:, 2] * f[1] + c[1]
                z = pc[:, 2] - pc[root, 2]                         # :199
            r = pc[root]
            ok[t, v] = int(status[t, s, root] == 1 and np.isfinite(r).all() and r[2] > 0)
            if not ok[t, v]:
                continue
            pel[t, v] = r
            on = (np.asarray(status[t, s]) == 1) & (pc[:, 2] > 0) & np.isfinite(u) & np.isfinite(w) & np.isfinite(z)
            jt[t, v, on] = np.stack([u, w, z], axis=1)[on]
            vis[t, v, on] = 1.0
    return jt, vis, pel, ok


def case(seed, T, S, V, J, root=0):
    """T frames of V ring cameras (restate.synthetic_cameras) around J joints near the origin:
    (X [T,S,J,3], status [T,S,J] int32, cam [T,V,16]).  Planted: joints with status 0, a frame
    whose root failed, a joint behind one camera, a joint on a camera's focal plane."""
    rng = np.random.default_rng(seed)
    Rm, Tm, f, c, _ = restate.synthetic_cameras(rng, T, V)
    cam = np.concatenate([Rm.reshape(T, V, 9), Tm, f, c], axis=2)
    X = rng.normal(0, 400, (T, S, J, 3))
    status = (rng.uniform(size=(T, S, J)) > 0.1).astype(np.int32)
    status[:, :, root] = 1
    if T > 1:
        status[1, :, root] = 0                                    # root failed
    if T > 2:
        s = 0
        X[2, s, (root + 1) % J] = Tm[2, 0] * 1.5                  # behind camera 0 (past its centre)
        status[2, s, (root + 1) % J] = 1
    if T > 3:
        X[3, 0, (root + 2) % J] = Tm[3, 0]                        # at camera 0's centre: depth 0
        status[3, 0, (root + 2) % J] = 1
    if T > 4:
        status[4, :, (root + 3) % J] = -1                         # the pair triangulator's negative codes
    return X, status, cam


def assert_same(got, want, rel=1e-9):
    jt, vis, pel, ok = (np.asarray(a) for a in got)
    wjt, wvis, wpel, wok = want
    assert np.array_equal(ok, wok) and np.array_equal(vis, wvis)
    assert np.isfinite(jt).all() and np.isfinite(pel).all()
    for a, b in ((jt, wjt), (pel, wpel)):
        scale = np.maximum(np.abs(b), 1.0)
        assert np.max(np.abs(a - b) / scale) <= rel, np.max(np.abs(a - b) / scale)


class Emulated:
    """epb_pseudo_records and epb_pose_to_camera on torch CPU tensors, from include/epb.h."""

    @staticmethod
    def pseudo_records(X, status, cam, T, S, V, J, root, joints_3d, vis, pelvis, ok):
        assert X.shape == (T, S, J, 3) and status.shape == (T, S, J) and cam.shape == (T, V, 16)
        for dst, src in zip((joints_3d, vis, pelvis, ok), restated(X.numpy(), status.numpy(), cam.numpy(), root)):
            dst.copy_(torch.from_numpy(np.ascontiguousarray(src)).to(dst.dtype))

    @staticmethod
    def pose_to_camera(joints, cam, N, J, root, out):
        a = joints.numpy().reshape(N, J, 3)
        c = cam.numpy().reshape(N, 5)
        d = a[:, :, 2] + c[:, 4:5]
        y = np.stack([(a[:, :, 0] - c[:, 2:3]) / c[:, 0:1] * d, (a[:, :, 1] - c[:, 3:4]) / c[:, 1:2] * d, d], axis=2)
        out.copy_(torch.from_numpy(y - y[:, root:root + 1]).reshape(out.shape))
