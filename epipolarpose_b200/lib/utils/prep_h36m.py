"""Self-supervised Human3.6M annotations from a pretrained network: `save_triangulations`, which the
reference names in lib/utils/prep_h36m.py:211-213 and leaves unimplemented.

The released reference trains its self-supervised model on `train-ss.pkl`: Human3.6M frames whose
`joints_3d` are pseudo-labels, a pretrained 2-D network's predictions triangulated across the
frame's cameras and projected back into each camera.  `save_triangulations` writes such a file
from any network and any dict-form annotation pickle (`{1..V: per-camera lists}`, the form of
`train-ss.pkl` and `valid.pkl`):

  * frame k is the tuple [src[c + 1][k] for c in range(V)];
  * DataLoader workers read the tuples as deferred samples (the dataset's get_data with augmentation
    off), and the main process assembles each batch on the device (lib.dataset.assemble_batch);
  * method 'robust': MultiViewPredictor (network, soft-argmax, patch -> image and the robust V-view
    triangulation in one graph replay) gives one world pose per frame; methods 'iterative' /
    'polynomial': PosePredictor's 2-D joints, camera c triangulated with its first neighbour in
    dataset.cam_config by epb_triangulate (the reference's img_utils.triangulate for 'iterative'),
    one world pose per camera;
  * epb_pseudo_records projects the world joints into every camera (from_worldjt_to_imagejt,
    :176-204): joints_3d, joints_3d_vis and pelvis of each record are replaced, everything else is
    the source record's.  A frame whose root is not triangulated, or lies behind one of its cameras,
    is dropped from every camera's list, so the lists stay frame-aligned.

The network decides the joint layout: the source's when the counts agree; 16 joints from a 17-joint
source (experiments/h36m/train-ss.yaml: NUM_JOINTS 16, MPII_ORDER true) are written in MPII order
through H36M_TO_MPII_PERM with the root at Hip (6)."""
import copy
import os
import pickle
import time

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset
from torch.utils.data.dataloader import default_collate

from epipolarpose_b200 import ops as _ops
from ..dataset.JointIntegralDataset import load_pickle
from ..dataset.h36m_eval import H36M_TO_MPII_PERM
from ..dataset.deferred import assemble_batch, is_deferred

_backend = [_ops]
PAIR_METHODS = {'iterative': 'iterative_LS', 'polynomial': 'polynomial'}
METHODS = ('robust',) + tuple(PAIR_METHODS)


def _device():
    return torch.device('cuda') if _backend[0] is _ops else torch.device('cpu')


def pseudo_records(X, status, cam, root):
    """epb_pseudo_records (include/epb.h): X [T,S,J,3] float64 world joints, status [T,S,J] int32,
    cam [T,V,16] float64 (R, T, f, c), all on the device, S = 1 or V -> (joints_3d [T,V,J,3],
    vis [T,V,J,3], pelvis [T,V,3], ok [T,V] int32)."""
    T, S, J = X.shape[0], X.shape[1], X.shape[2]
    V = cam.shape[1]
    if tuple(status.shape) != (T, S, J) or tuple(cam.shape) != (T, V, 16):
        raise ValueError("pseudo_records: X %s, status %s and cam %s do not agree"
                         % (tuple(X.shape), tuple(status.shape), tuple(cam.shape)))
    dev = X.device
    jt = torch.empty((T, V, J, 3), device=dev, dtype=torch.float64)
    vis = torch.empty((T, V, J, 3), device=dev, dtype=torch.float64)
    pelvis = torch.empty((T, V, 3), device=dev, dtype=torch.float64)
    ok = torch.empty((T, V), device=dev, dtype=torch.int32)
    if T:
        _backend[0].pseudo_records(X.contiguous(), status.contiguous(), cam.contiguous(), T, S, V, J, root, jt, vis,
                                   pelvis, ok)
    return jt, vis, pelvis, ok


def joint_layout(J, J_src, flip_pairs, parent_ids):
    """Layout of the written records for a network of J joints and a source of J_src:
    (perm or None, root, flip_pairs, parent_ids).  perm [J] picks the source joints in the written
    order (H36M_TO_MPII_PERM for 16 from 17); flip_pairs and parent_ids are mapped through it."""
    if J == J_src:
        return None, 6 if J == 16 else 0, flip_pairs, parent_ids
    if not (J == 16 and J_src == 17):
        raise ValueError("the network predicts %d joints and the source records hold %d: only the same "
                         "count, or 16 (MPII order) from 17 (Human3.6M order), can be written" % (J, J_src))
    perm = np.asarray(H36M_TO_MPII_PERM, dtype=np.int64)
    inv = {int(h): i for i, h in enumerate(perm)}
    pairs = [[inv[int(a)], inv[int(b)]] for a, b in flip_pairs if int(a) in inv and int(b) in inv]
    if len(pairs) != sum(1 for a, b in flip_pairs if int(a) in inv or int(b) in inv):
        raise ValueError("a flip pair of the source joins a joint the MPII order drops")
    par = np.asarray(parent_ids)
    if any(int(par[h]) not in inv for h in perm):
        raise ValueError("a joint of the MPII order has its parent among the dropped joints")
    parents = np.array([inv[int(par[h])] for h in perm], dtype=par.dtype)
    return perm, 6, pairs, parents


def _cam16(rec):
    c = rec['cam']
    return np.concatenate([np.asarray(c.R, np.float64).reshape(9), np.asarray(c.T, np.float64).reshape(3),
                           np.asarray(c.f, np.float64).reshape(2), np.asarray(c.c, np.float64).reshape(2)])


class _Tuples(Dataset):
    """Frame k of a dict-form source -> its V views through dataset.get_data (deferred samples in a
    DataLoader worker)."""

    def __init__(self, dataset, src, V):
        self.ds, self.src, self.V = dataset, src, V

    def __len__(self):
        return len(self.src[1])

    def __getitem__(self, k):
        return [self.ds.get_data(copy.deepcopy(self.src[c + 1][k])) for c in range(self.V)]


def _collate_tuples(items):
    """A batch of tuples -> one batch of their views, tuple-major."""
    return default_collate([v for tup in items for v in tup])


def _assemble(batch, dev):
    """Loader batch -> images float32 [T*V, 3, H, W] on the device."""
    x = assemble_batch(batch)[0] if is_deferred(batch) else batch[0]
    return x.to(dev, non_blocking=True)


def _load_source(src):
    anno = load_pickle(src) if isinstance(src, (str, os.PathLike)) else src
    if not isinstance(anno, dict):
        raise ValueError("save_triangulations needs frame-aligned cameras: a dict-form annotation pickle "
                         "({1..V: one list per camera}); a list-form pickle does not say which records "
                         "show the same frame")
    V = len(anno)
    if sorted(anno) != list(range(1, V + 1)) or not 2 <= V <= 8:
        raise ValueError("a dict-form annotation pickle is keyed 1..V with 2 <= V <= 8, got keys %s"
                         % sorted(anno))
    if len({len(anno[c]) for c in anno}) != 1:
        raise ValueError("the cameras' lists of a dict-form annotation pickle differ in length: %s"
                         % {c: len(anno[c]) for c in anno})
    return anno, V


def _make_predictor(model, method, flip_test, flip_pairs, threshold_px):
    from ..core.inference import MultiViewPredictor, PosePredictor
    if method == 'robust':
        return MultiViewPredictor(model, flip_test=flip_test, flip_pairs=flip_pairs, threshold_px=threshold_px)
    return PosePredictor(model, flip_test=flip_test, flip_pairs=flip_pairs)


def _agreement(jt, pelvis, cam, recs, perm, root, vis):
    """Root-relative camera-frame MPJPE (mm) of the written joints against the source's joints_3d,
    both through epb_pose_to_camera, over the joints with vis 1 in both: (sum, count)."""
    F, V, J = jt.shape[:3]
    if F == 0:
        return 0.0, 0
    ops = _backend[0]
    dev = _device()
    gt = np.stack([np.stack([np.asarray(r['joints_3d'], np.float64)[:, :3] for r in tup]) for tup in recs])
    gvis = np.stack([np.stack([np.asarray(r['joints_3d_vis'], np.float64)[:, 0] for r in tup]) for tup in recs])
    if perm is not None:
        gt, gvis = gt[:, :, perm], gvis[:, :, perm]
    gcam = np.stack([np.stack([np.concatenate([np.asarray(r['fl'], np.float64).reshape(2),
                                               np.asarray(r['c_p'], np.float64).reshape(2),
                                               np.asarray(r['pelvis'], np.float64).reshape(3)[2:]])
                               for r in tup]) for tup in recs])
    pcam = np.concatenate([cam[:, :, 12:16], pelvis[:, :, 2:3]], axis=2)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64).reshape(F * V, -1)).to(dev)
    out = []
    for a, c in ((jt, pcam), (gt, gcam)):
        o = torch.empty((F * V, J, 3), device=dev, dtype=torch.float64)
        ops.pose_to_camera(t(a), t(c), F * V, J, root, o)
        out.append(o.cpu().numpy().reshape(F, V, J, 3))
    both = (vis[..., 0] > 0) & (gvis > 0)
    e = np.linalg.norm(out[0] - out[1], axis=3)
    return float(e[both].sum()), int(both.sum())


def save_triangulations(model, dataset, src, dst, method='robust', flip_test=None, threshold_px=15.0,
                        tuples_per_batch=32, workers=8, predictor=None):
    """Write `dst`, a dict-form annotation pickle of pseudo-labels for the frames of `src` (a path or
    an already loaded dict-form annotation), from `model`'s predictions on them; see the module
    docstring.  `dataset` (an H36M_Integral) supplies the image root, the crop geometry, get_data and
    cam_config; it is read with augmentation and occluders off.  `predictor` replaces the predictor
    built from `model` (a MultiViewPredictor for 'robust', else a PosePredictor); it must have that
    class's call interface.

    Returns a report dict: frames (written), dropped, failed (share of triangulated joints whose
    status is not 1), inlier_views (mean inlier views per joint, failed joints counting 0; 'robust' only,
    else None), agreement_mm (root-relative camera-frame MPJPE of the written labels against the
    source's joints_3d over the joints visible in both, NaN when there are none: a label-quality
    figure when the source holds ground truth), and host-clock seconds: in all, waiting for the loader's
    workers, assembling the batches on the device, and in the predictor's calls."""
    if method not in METHODS:
        raise ValueError("method must be one of %s, got %r" % (METHODS, method))
    t0 = time.perf_counter()
    anno, V = _load_source(src)
    T_all = len(anno[1])
    J_src = len(np.asarray(anno[1][0]['joints_3d'])) if T_all else 0
    nb = None
    if method in PAIR_METHODS:
        cc = list(getattr(dataset, 'cam_config', []) or [])
        if len(cc) != V:
            raise ValueError("the pair methods triangulate each camera with its first neighbour in "
                             "dataset.cam_config, which lists %d cameras for %d" % (len(cc), V))
        nb = np.array([int(c[0]) for c in cc], dtype=np.int64)
        if np.any(nb < 0) or np.any(nb >= V) or np.any(nb == np.arange(V)):
            raise ValueError("dataset.cam_config %s does not name another camera of 0..%d" % (cc, V - 1))
    layout = None
    if T_all and model is not None:
        net = getattr(model, 'module', model)
        layout = joint_layout(int(net._plan.num_joints), J_src, anno[1][0]['flip_pairs'], anno[1][0]['parent_ids'])
    if predictor is None:
        predictor = _make_predictor(model, method, flip_test, layout[2] if layout else None, threshold_px)

    ds = copy.copy(dataset)                     # shallow: the same db, read without augmentation
    ds.is_train, ds.occluders = False, None
    tpb = max(1, int(tuples_per_batch))
    loader = DataLoader(_Tuples(ds, anno, V), batch_size=tpb, shuffle=False, num_workers=int(workers),
                        collate_fn=_collate_tuples)
    dev = _device()
    out = {c + 1: [] for c in range(V)}
    n_fail = n_joint = n_kept = 0
    inl_sum, agree = 0, [0.0, 0]
    t_pred = t_wait = t_asm = 0.0
    k0 = 0
    it = iter(loader)
    while True:
        ts = time.perf_counter()
        batch = next(it, None)
        t_wait += time.perf_counter() - ts
        if batch is None:
            break
        recs = [[anno[c + 1][k] for c in range(V)] for k in range(k0, k0 + tpb) if k < T_all]
        T = len(recs)
        k0 += T
        ts = time.perf_counter()
        x = _assemble(batch, dev)
        if x.is_cuda:
            torch.cuda.synchronize(x.device)        # attributes the decode and crop to this stage
        t_asm += time.perf_counter() - ts
        H, W = x.shape[2], x.shape[3]
        flat = [r for tup in recs for r in tup]
        boxes = {k: np.array([float(r[k]) for r in flat]) for k in ('center_x', 'center_y', 'width', 'height')}
        boxes['scale'], boxes['rot'] = np.ones(T * V), np.zeros(T * V)
        P = np.stack([np.asarray(r['cam'].projection_matrix, np.float64)[0:3, 0:4] for r in flat]).reshape(T, V, 3, 4)
        cam = np.stack([_cam16(r) for r in flat]).reshape(T, V, 16)
        ts = time.perf_counter()
        if method == 'robust':
            res = predictor(x.reshape(T, V, 3, H, W), boxes, P)
            t_pred += time.perf_counter() - ts
            X = torch.from_numpy(np.ascontiguousarray(res['world'], np.float64)).to(dev)[:, None]
            st = torch.from_numpy(np.ascontiguousarray(res['status'], np.int32)).to(dev)[:, None]
            inl_sum += int(sum(bin(int(m)).count('1') for m in np.asarray(res['inliers']).ravel()))
        else:
            from .triangulation import triangulate_pairs
            kps = np.asarray(predictor(x, boxes), np.float64)
            t_pred += time.perf_counter() - ts
            J = kps.shape[1]
            k4 = torch.from_numpy(np.ascontiguousarray(kps.reshape(T, V, J, 4))).to(dev)
            Pd = torch.from_numpy(np.ascontiguousarray(P)).to(dev)
            nbt = torch.from_numpy(nb).to(dev)
            X, st = triangulate_pairs(k4.reshape(T * V, J, 4), k4[:, nbt].reshape(T * V, J, 4),
                                      Pd.reshape(T * V, 3, 4), Pd[:, nbt].reshape(T * V, 3, 4), PAIR_METHODS[method])
            X, st = X.view(T, V, J, 3), st.view(T, V, J)
        J = X.shape[2]
        if layout is None:
            layout = joint_layout(J, J_src, anno[1][0]['flip_pairs'], anno[1][0]['parent_ids'])
        perm, root, pairs, parents = layout
        want = len(perm) if perm is not None else J_src
        if J != want:
            raise ValueError("the predictor returned %d joints, the layout expects %d" % (J, want))
        jt, vis, pel, ok = (a.cpu().numpy() for a in pseudo_records(X, st, torch.from_numpy(cam).to(dev), root))
        stn = st.cpu().numpy()
        n_fail += int((stn != 1).sum())
        n_joint += stn.size
        keep = np.flatnonzero(ok.all(axis=1))
        n_kept += len(keep)
        s, n = _agreement(jt[keep], pel[keep], cam[keep], [recs[i] for i in keep], perm, root, vis[keep])
        agree[0] += s
        agree[1] += n
        for i in keep:
            for c in range(V):
                r = copy.copy(recs[i][c])
                r['joints_3d'] = np.ascontiguousarray(jt[i, c])
                r['joints_3d_vis'] = np.ascontiguousarray(vis[i, c])
                r['pelvis'] = np.ascontiguousarray(pel[i, c])
                if perm is not None:
                    r['flip_pairs'] = [list(p) for p in pairs]
                    r['parent_ids'] = parents.copy()
                out[c + 1].append(r)
    if k0 != T_all:
        raise RuntimeError("the loader returned %d of %d frames" % (k0, T_all))
    d = os.path.dirname(os.path.abspath(dst))
    os.makedirs(d, exist_ok=True)
    with open(dst, 'wb') as f:
        pickle.dump(out, f, protocol=4)
    return {'frames': n_kept, 'dropped': T_all - n_kept,
            'failed': float(n_fail / n_joint) if n_joint else float('nan'),
            'inlier_views': (float(inl_sum / n_joint) if n_joint else float('nan')) if method == 'robust' else None,
            'agreement_mm': float(agree[0] / agree[1]) if agree[1] else float('nan'),
            'seconds': time.perf_counter() - t0, 'loader_wait_seconds': t_wait, 'assemble_seconds': t_asm,
            'predictor_seconds': t_pred}
