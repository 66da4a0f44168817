"""Self-supervision glue and patch<->image geometry -- host-side mirror of the
hot-path part of the reference lib/utils/img_utils.py:
  trans_coords_from_patch_to_org_3d (:150-155), self_supervision (:166-190),
  triangulate (:193-209), get_batch_labels_from_global_coords (:212-243).
Everything downstream of the network output runs on the device in float64
kernels (epb_patch_to_image -> epb_triangulate -> epb_project_labels); the
reference's per-sample / per-joint Python loops disappear.  `meta` follows the
dataset contract of reference lib/dataset/h36m.py:73-86 (collated: tensors or
lists of length B).  numpy in / numpy out like the reference;
`self_supervision_device` returns CUDA tensors for the training loop.

Input pipeline (SURVEY.md section 8(f) row 1): get_single_patch_sample (:246-298),
do_augmentation (:28-39), fliplr_joints (:42-60) with the same names and return values; the crop
(cv2.warpAffine), BGR->RGB, colour scale, clip and normalisation run in ONE kernel for the whole
batch (epb_patch_sample, bit-exact against OpenCV) and the joints -> label half in
epb_patch_joints; `generate_patch_batch_device` is the batched entry point a GPU data loader
calls with already decoded frames.  `flip(tensor, dims)` (:319-331) mirrors the input batch of the
flip test.  The occluder paste (lib/utils/augmentation.py) is not built:
`occluder` must be None."""
import random

import numpy as np
import torch

from epipolarpose_b200 import ops as _ops
from . import triangulation as _tri
from ..core.integral_loss import get_joint_location_coords

_backend = [_ops]


def _dev():
    return torch.device("cuda") if _backend[0] is _ops else torch.device("cpu")


def _t64(v, dev):
    if isinstance(v, torch.Tensor):
        return v.to(device=dev, dtype=torch.float64)
    return torch.as_tensor(np.asarray(v, dtype=np.float64), device=dev)


def _boxes(meta, B, dev):
    """[B,6] float64: c_x, c_y, width, height, scale, rot."""
    cols = [_t64(meta[k], dev).reshape(-1)[:B]
            for k in ('center_x', 'center_y', 'width', 'height', 'scale', 'rot')]
    return torch.stack(cols, dim=1).contiguous()


def _cams(meta, B, dev):
    """[B,16] float64: R(9) T(3) f(2) c(2)."""
    return torch.cat([_t64(meta['R'], dev).reshape(B, 9), _t64(meta['T'], dev).reshape(B, 3),
                      _t64(meta['f'], dev).reshape(B, 2), _t64(meta['c'], dev).reshape(B, 2)],
                     dim=1).contiguous()


def _intrinsics(meta, B, dev):
    """[B,4] float64: f(2) c(2)."""
    return torch.cat([_t64(meta['f'], dev).reshape(B, 2), _t64(meta['c'], dev).reshape(B, 2)],
                     dim=1).contiguous()


def pack_meta(meta, B, dev, estimate_extrinsics=False):
    """Collated `meta` -> device float64 tensors {box [B,6], cam [B,16], P [B,3,4]} (the
    form the kernels consume; static-shaped, so a CUDA graph can re-read them).  Meta with
    intrinsics `f`, `c` but no `R` -- and every meta when estimate_extrinsics is set, which
    ignores `R`, `T` and `projection_matrix` -- gives {box, intr [B,4] = f(2) c(2)}."""
    if isinstance(meta, dict) and "_packed" in meta:
        return meta["_packed"]
    out = {"box": _boxes(meta, B, dev)}
    if estimate_extrinsics or ('R' not in meta and 'f' in meta and 'c' in meta):
        out["intr"] = _intrinsics(meta, B, dev)
        if estimate_extrinsics:
            return out
    if 'R' in meta:
        out["cam"] = _cams(meta, B, dev)
    if 'projection_matrix' in meta:
        out["P"] = _t64(meta['projection_matrix'], dev).reshape(B, -1, 4)[:, 0:3, :].contiguous()
    return out


def patch_to_image_device(coords_norm, meta, patch_w=256, patch_h=256, rect_3d_w=2000):
    """coords_norm [B, J*3] float32 (soft-argmax output) -> kps [B,J,4] float64."""
    ops = _backend[0]
    B = coords_norm.shape[0]
    J = coords_norm.shape[1] // 3
    dev = coords_norm.device
    kps = torch.empty((B, J, 4), device=dev, dtype=torch.float64)
    ops.patch_to_image(coords_norm.contiguous(), pack_meta(meta, B, dev)["box"], B, J, patch_w,
                       patch_h, rect_3d_w, kps)
    return kps


def triangulate_device(kps, meta, method="iterative"):
    """reference :193-209: sample i pairs with i + B/2; both halves receive the
    same world-frame result."""
    B, J = kps.shape[0], kps.shape[1]
    half = B // 2
    P = pack_meta(meta, B, kps.device)["P"]
    X, _ = _tri.triangulate_pairs(kps[:half], kps[half:2 * half], P[:half], P[half:2 * half],
                                  method=method, stride_u=kps.shape[2])
    return torch.cat([X, X], dim=0)


def labels_from_global_coords_device(X, meta, patch_w=256., patch_h=256., rect_3d_w=2000.):
    ops = _backend[0]
    B, J = X.shape[0], X.shape[1]
    dev = X.device
    label = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    weight = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    pm = pack_meta(meta, B, dev)
    ops.project_labels(X.contiguous(), pm["cam"], pm["box"], B, J, patch_w, patch_h, rect_3d_w,
                       label, weight)
    return label, weight


def labels_estimated_extrinsics_device(kps, meta, method="iterative", patch_w=256., patch_h=256.,
                                       rect_3d_w=2000.):
    """Self-supervision without camera extrinsics: kps [B,J,4] image px -> (label, weight) f32
    [B, J*3].  Each pair's projection matrices come from its own 2-D joints
    (triangulation.relative_pose_pairs; only the box and the intrinsics f, c are read), the pair
    is triangulated with them by `method` -- after the pose has been scaled, so the iterative
    method's absolute depth tolerance keeps its meaning -- and re-projected with the estimated
    cameras.  Pairs whose pose could not be estimated get weight 0 (and label 0) in both views.
    Static shapes, no host synchronisation: capturable in a CUDA graph."""
    ops = _backend[0]
    B, J = kps.shape[0], kps.shape[1]
    half = B // 2
    dev = kps.device
    pm = pack_meta(meta, B, dev, estimate_extrinsics=True)
    Pa, Pb, cam, _, status = _tri.relative_pose_pairs(kps, pm["intr"], pm["box"], rect_3d_w)
    X, _ = _tri.triangulate_pairs(kps[:half], kps[half:], Pa, Pb, method=method, stride_u=kps.shape[2])
    X = torch.cat([X, X], dim=0)
    label = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    weight = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    ops.project_labels(X, cam, pm["box"], B, J, patch_w, patch_h, rect_3d_w, label, weight)
    ok = torch.cat([status, status], dim=0).reshape(B, 1) != 0
    return torch.where(ok, label, 0.0), weight * ok


def self_supervision_device(preds, meta, method="iterative", estimate_extrinsics=False):
    """preds: network output [B, J*D, H, W] (CUDA) -> (label, weight) CUDA f32
    [B, J*3]; labels carry no gradient (reference integral_loss.py:88-91).  With
    estimate_extrinsics the cameras come from the predicted 2-D joints themselves
    (labels_estimated_extrinsics_device; meta needs only the box and f, c)."""
    coords = get_joint_location_coords(preds)
    kps = patch_to_image_device(coords, meta)
    if estimate_extrinsics:
        return labels_estimated_extrinsics_device(kps, meta, method)
    X = triangulate_device(kps, meta, method)
    return labels_from_global_coords_device(X, meta)


def self_supervision(preds, meta):
    """reference :166-190 -> numpy float32 (label, weight)."""
    label, weight = self_supervision_device(preds, meta)
    return label.cpu().numpy(), weight.cpu().numpy()


def triangulate(kps, meta):
    """reference :193-209, numpy [B,J,>=2] -> numpy [B,J,3] float64."""
    k = torch.as_tensor(np.ascontiguousarray(kps, dtype=np.float64), device=_dev())
    return triangulate_device(k, meta).cpu().numpy()


def get_batch_labels_from_global_coords(coords_3d_in_global_frame, meta):
    """reference :212-243 -> numpy float32 (label, weight)."""
    X = torch.as_tensor(np.ascontiguousarray(coords_3d_in_global_frame, dtype=np.float64),
                        device=_dev())
    label, weight = labels_from_global_coords_device(X, meta)
    return label.cpu().numpy(), weight.cpu().numpy()


def trans_coords_from_patch_to_org_3d(coords_in_patch, c_x, c_y, bb_width, bb_height,
                                      patch_width, patch_height, rect_3d_width, rect_3d_height,
                                      scale=1.0, rot=0):
    """reference :150-155 for ONE sample: [J,>=3] patch px -> image px (+ z in mm)."""
    return trans_coords_from_patch_to_org_3d_batch(
        np.asarray(coords_in_patch)[None], [c_x], [c_y], [bb_width], [bb_height], patch_width,
        patch_height, rect_3d_width, [scale], [rot])[0]


def trans_coords_from_patch_to_org_3d_batch(coords, c_x, c_y, bb_w, bb_h, patch_w, patch_h,
                                            rect_3d_w, scale=None, rot=None):
    """Batched form used by eval_integral: coords [B,J,>=3] (x,y,z in patch px)."""
    ops = _backend[0]
    coords = np.asarray(coords, dtype=np.float64)
    B, J = coords.shape[0], coords.shape[1]
    dev = _dev()
    # back to the normalised soft-argmax units the kernel consumes
    norm = np.empty((B, J, 3), dtype=np.float32)
    norm[:, :, 0] = coords[:, :, 0] / patch_w - 0.5
    norm[:, :, 1] = coords[:, :, 1] / patch_h - 0.5
    norm[:, :, 2] = coords[:, :, 2] / patch_w
    meta = {'center_x': c_x, 'center_y': c_y, 'width': bb_w, 'height': bb_h,
            'scale': scale if scale is not None else np.ones(B),
            'rot': rot if rot is not None else np.zeros(B)}
    kps = torch.empty((B, J, 4), device=dev, dtype=torch.float64)
    ops.patch_to_image(torch.from_numpy(norm.reshape(B, J * 3)).to(dev), _boxes(meta, B, dev), B, J,
                       float(patch_w), float(patch_h), float(rect_3d_w), kps)
    out = coords.copy()
    res = kps.cpu().numpy()
    out[:, :, 0:3] = res[:, :, 0:3]
    return out


# ---------------------------------------------------------------------- input pipeline
def flip(tensor, dims):
    """reference :319-331: a copy of `tensor` reversed along `dims` (an int or a sequence), on the
    tensor's device.  The reference's index meshgrid selects exactly what torch.flip returns."""
    if not isinstance(dims, (tuple, list)):
        dims = [dims]
    return torch.flip(tensor, list(dims))


def do_augmentation():
    """reference :28-39 (scale_factor 0.25, rot_factor 30, color_factor 0.2, rot_aug_rate 0.6,
    do_flip_aug False) -- the same draws from np.random / random in the same order."""
    scale = np.clip(np.random.randn(), -1.0, 1.0) * 0.25 + 1.0
    rot = np.clip(np.random.randn(), -2.0, 2.0) * 30 if random.random() <= 0.6 else 0
    do_flip = False and random.random() <= 0.5
    c_up, c_low = 1.0 + 0.2, 1.0 - 0.2
    color_scale = [random.uniform(c_low, c_up), random.uniform(c_low, c_up), random.uniform(c_low, c_up)]
    return scale, rot, do_flip, color_scale


def fliplr_joints(_joints, _joints_vis, width, matched_parts):
    """reference :42-60."""
    joints = _joints.copy()
    joints_vis = _joints_vis.copy()
    joints[:, 0] = width - joints[:, 0] - 1
    for pair in matched_parts:
        joints[pair[0], :], joints[pair[1], :] = joints[pair[1], :], joints[pair[0], :].copy()
        joints_vis[pair[0], :], joints_vis[pair[1], :] = joints_vis[pair[1], :], joints_vis[pair[0], :].copy()
    return joints, joints_vis


def generate_patch_batch_device(images, center_x, center_y, width, height, patch_width, patch_height,
                                scale=None, rot=None, do_flip=None, color_scale=None, mean=None, std=None,
                                occluders=None):
    """B decoded BGR frames (uint8 [H,W,3] numpy arrays or tensors, sizes may differ) ->
    (patches float32 [B,3,ph,pw] on the device, trans float64 [B,2,3], box float64 [B,6]).
    occluders: per sample a list of (rgba uint8 [h,w,4], (cx, cy)) pasted onto the uint8 patch
    in order (augmentation.draw_occluders), or None."""
    ops = _backend[0]
    dev = _dev()
    B = len(images)
    offs, hwp, chunks, pos = [], [], [], 0
    for im in images:
        t = im if isinstance(im, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(im))
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
            raise ValueError("frames must be uint8 [H, W, 3] (cv2.imread layout)")
        t = t.contiguous()
        offs.append(pos)
        hwp.append([t.shape[0], t.shape[1], t.shape[1] * 3])
        chunks.append(t.reshape(-1))
        pos += (t.numel() + 15) // 16 * 16
    base = torch.zeros(max(pos, 16), dtype=torch.uint8)
    for o, c in zip(offs, chunks):
        base[o:o + c.numel()] = c.cpu()
    ones, zeros = np.ones(B), np.zeros(B)
    box = np.stack([np.asarray(center_x, dtype=np.float64).reshape(B), np.asarray(center_y, dtype=np.float64).reshape(B),
                    np.asarray(width, dtype=np.float64).reshape(B), np.asarray(height, dtype=np.float64).reshape(B),
                    np.asarray(ones if scale is None else scale, dtype=np.float64).reshape(B),
                    np.asarray(zeros if rot is None else rot, dtype=np.float64).reshape(B)], axis=1)
    t_box = torch.from_numpy(np.ascontiguousarray(box)).to(dev)
    t_flip = None if do_flip is None else torch.as_tensor(np.asarray(do_flip).astype(np.int32).reshape(B)).to(dev)
    t_col = None if color_scale is None else \
        torch.as_tensor(np.asarray(color_scale, dtype=np.float32).reshape(B, 3)).to(dev)
    ms = None
    if mean is not None and std is not None:
        ms = [float(v) for v in np.asarray(mean).reshape(3)] + [float(v) for v in np.asarray(std).reshape(3)]
    out = torch.empty((B, 3, int(patch_height), int(patch_width)), device=dev, dtype=torch.float32)
    trans = torch.empty((B, 6), device=dev, dtype=torch.float64)
    if occluders is not None:
        from .augmentation import pack_occluders
        ob, od, oc = pack_occluders(occluders, dev)
        ops.patch_sample_occ(base.to(dev), torch.tensor(offs, dtype=torch.int64, device=dev),
                             torch.tensor(hwp, dtype=torch.int32, device=dev), t_box, t_flip, t_col, ms,
                             B, int(patch_width), int(patch_height), ob, od, oc, out, trans)
    else:
        ops.patch_sample(base.to(dev), torch.tensor(offs, dtype=torch.int64, device=dev),
                         torch.tensor(hwp, dtype=torch.int32, device=dev), t_box, t_flip, t_col, ms, B,
                         int(patch_width), int(patch_height), out, trans)
    return out, trans.reshape(B, 2, 3), t_box


def patch_labels_device(joints, box, trans, patch_width, patch_height, rect_3d_width, depth_in_image=False):
    """joints [B,J,3] (image px, depth mm) -> label float64 [B, J*3] (reference :283-296 +
    generate_joint_location_label)."""
    ops = _backend[0]
    dev = _dev()
    jt = torch.as_tensor(np.ascontiguousarray(joints, dtype=np.float64)).to(dev)
    B, J = jt.shape[0], jt.shape[1]
    label = torch.empty((B, J * 3), device=dev, dtype=torch.float64)
    ops.patch_joints(jt.contiguous(), box, trans.reshape(B, 6).contiguous(), B, J, patch_width, patch_height,
                     rect_3d_width, bool(depth_in_image), label)
    return label


def get_single_patch_sample(img_path, center_x, center_y, width, height,
                            joints, joints_vis, flip_pairs, parent_ids,
                            patch_width, patch_height, rect_3d_width, rect_3d_height, mean, std,
                            do_augment, label_func, depth_in_image=False, occluder=None, DEBUG=False):
    """reference :246-298, same arguments and return tuple (img_patch f32 [3,ph,pw] numpy, label,
    label_weight, scale, rot).  `img_path` may also be an already decoded BGR uint8 array.
    `label_func` is honoured when it is not the default generate_joint_location_label."""
    if isinstance(img_path, np.ndarray):
        cvimg = img_path
    else:
        import cv2
        cvimg = cv2.imread(img_path, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
        if not isinstance(cvimg, np.ndarray):
            raise IOError("Fail to read %s" % img_path)
    img_width = cvimg.shape[1]
    if do_augment:
        scale, rot, do_flip, color_scale = do_augmentation()
    else:
        scale, rot, do_flip, color_scale = 1.0, 0, False, [1.0, 1.0, 1.0]
    occ = None
    if occluder:                      # :269-270: drawn after do_augmentation(), pasted on the patch
        from .augmentation import draw_occluders
        occ = [draw_occluders(int(patch_width), int(patch_height), occluder)]
    patches, trans, box = generate_patch_batch_device(
        [cvimg], [center_x], [center_y], [width], [height], patch_width, patch_height, [scale], [rot],
        [do_flip], [color_scale], mean, std, occluders=occ)
    joints = np.array(joints, dtype=np.float64, copy=True)
    joints_vis = np.array(joints_vis, copy=True)
    if do_flip:
        joints, joints_vis = fliplr_joints(joints, joints_vis, img_width, flip_pairs)
    from ..core.integral_loss import generate_joint_location_label
    if label_func is None or label_func is generate_joint_location_label or \
            getattr(label_func, "__name__", "") == "generate_joint_location_label":
        label = patch_labels_device(joints[None], box, trans, patch_width, patch_height, rect_3d_width,
                                    depth_in_image)[0].cpu().numpy()
        label_weight = joints_vis.reshape((-1))
    else:
        tr = trans[0].cpu().numpy()
        for n_jt in range(len(joints)):
            joints[n_jt, 0:2] = np.dot(tr, np.array([joints[n_jt, 0], joints[n_jt, 1], 1.]).T)[0:2]
            den = (width * scale) if depth_in_image else (rect_3d_width * scale)
            joints[n_jt, 2] = joints[n_jt, 2] / den * patch_width
        label, label_weight = label_func(patch_width, patch_height, joints, joints_vis)
    return patches[0].cpu().numpy(), label, label_weight, scale, rot
