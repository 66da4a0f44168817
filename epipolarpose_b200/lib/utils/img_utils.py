"""Self-supervision glue and patch<->image geometry -- host-side mirror of the
hot-path part of the reference lib/utils/img_utils.py:
  trans_coords_from_patch_to_org_3d (:150-155), self_supervision (:166-190),
  triangulate (:193-209), get_batch_labels_from_global_coords (:212-243).
Everything downstream of the network output runs on the device in float64
kernels (epb_patch_to_image -> epb_triangulate -> epb_project_labels); the
reference's per-sample / per-joint Python loops disappear.  `tuple_labels_device` (not in the
reference) labels whole camera tuples from one robust V-view triangulation (epb_tuple_labels).  `meta` follows the
dataset contract of reference lib/dataset/h36m.py:73-86 (collated: tensors or
lists of length B).  numpy in / numpy out like the reference;
`self_supervision_device` returns CUDA tensors for the training loop.

Input pipeline (SURVEY.md section 8(f) row 1): get_single_patch_sample (:246-298),
do_augmentation (:28-39), fliplr_joints (:42-60) with the same names and return values; the crop
(cv2.warpAffine), BGR->RGB, colour scale, clip and normalisation run in ONE kernel for the whole
batch (epb_patch_sample, bit-exact against OpenCV) and the joints -> label half in
epb_patch_joints; `generate_patch_batch_device` is the batched entry point a GPU data loader
calls with decoded frames (host arrays, or the device frames of `decode_jpeg_batch_device`, the JPEG decode of
:251-252 on the GPU; `get_patch_batch_device` is the batched form of the whole sample).  `flip(tensor, dims)` (:319-331) mirrors the input batch of the
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


def tuple_labels_device(coords, lse, meta, views, threshold_px=_tri.DEFAULT_THRESHOLD_PX, patch_w=256.,
                        patch_h=256., rect_3d_w=2000., full=False):
    """Online labels of whole camera tuples (epb_tuple_labels, see include/epb.h): coords [B, J*3]
    float32 soft-argmax output of a view-major batch (B = views * T, row v*T + t is view v of tuple
    t), lse the soft-argmax's workspace ([B, J, 2] or [B*J*2]; its peak probability weights each view
    in the robust refit) or None (weights 1) -> (label, weight) float32 [B, J*3]: the robust V-view
    triangulation of each (tuple, joint) projected into every view of the tuple; weight 0 (and label
    0) where the joint or the tuple's root failed or lies behind the camera.  full=True also returns
    X [T,J,3], status [T,J], inliers [T,J] (bit v: view v) and resid [T,J] (px).  Static shapes, no
    host synchronisation: capturable in a CUDA graph."""
    ops = _backend[0]
    B, J = coords.shape[0], coords.shape[1] // 3
    V = int(views)
    if not 2 <= V <= 8:
        raise ValueError("tuple labels take 2..8 views per tuple, got %d" % V)
    if B % V:
        raise ValueError("a batch of %d rows is not whole tuples of %d views" % (B, V))
    if not (np.isfinite(threshold_px) and threshold_px > 0):
        raise ValueError("threshold_px must be a positive number of pixels, got %r" % (threshold_px,))
    if lse is not None and lse.numel() != B * J * 2:
        raise ValueError("lse must hold B*J*2 = %d values, got %d" % (B * J * 2, lse.numel()))
    T, dev = B // V, coords.device
    pm = pack_meta(meta, B, dev)
    label = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    weight = torch.empty((B, J * 3), device=dev, dtype=torch.float32)
    X = torch.empty((T, J, 3), device=dev, dtype=torch.float64)
    status = torch.empty((T, J), device=dev, dtype=torch.int32)
    inliers = torch.empty((T, J), device=dev, dtype=torch.int32)
    resid = torch.empty((T, J), device=dev, dtype=torch.float64)
    ops.tuple_labels(coords.detach().contiguous(), None if lse is None else lse.detach().reshape(-1).contiguous(),
                     pm["box"], pm["P"].reshape(B, 12).contiguous(), pm["cam"], T, V, J, patch_w, patch_h,
                     rect_3d_w, threshold_px, label, weight, X, inliers, resid, status)
    if full:
        return label, weight, X, status, inliers, resid
    return label, weight


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


_IMREAD_FLAGS = 1 | 128                      # cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION
_JPEG_STATUS = {1: "unsupported", 2: "malformed"}


class JpegFrames:
    """B decoded BGR frames on the device in the layout epb_patch_sample reads: frame i is
    base[offs[i]:] with (H, W, row pitch) = hwp[i]; sizes[i] = (H, W).  status[i] is the device
    decoder's verdict (0 ok, 1 unsupported, 2 malformed; those frames came from cv2)."""

    def __init__(self, base, offs, hwp, sizes, status):
        self.base, self.offs, self.hwp, self.sizes, self.status = base, offs, hwp, sizes, status

    def __len__(self):
        return len(self.sizes)

    def frame(self, i):
        """Frame i as a uint8 [H, W, 3] device tensor (a view)."""
        H, W = self.sizes[i]
        o = int(self._offs_host[i])
        return self.base[o:o + H * W * 3].view(H, W, 3)


def _host_decode(buf, i, why):
    """The reference's own decode (cv2.imread flags) of blob i, for what the device does not decode."""
    try:
        import cv2
    except ImportError:
        raise IOError("JPEG blob %d is %s and cv2 is not importable" % (i, why))
    img = cv2.imdecode(buf, _IMREAD_FLAGS)
    if not isinstance(img, np.ndarray):
        raise IOError("Fail to read JPEG blob %d (%s)" % (i, why))
    return img


def _frame_offsets(hw):
    offs, pos = [], 0
    for H, W in hw:
        offs.append(pos)
        pos += (int(H) * int(W) * 3 + 15) // 16 * 16
    return np.array(offs, dtype=np.int64), pos


def decode_jpeg_batch_device(blobs, stats=None, events=None):
    """B JPEG files (bytes or 1-D uint8 arrays) -> JpegFrames, decoded on the device bit-exact
    against cv2.imread(IMREAD_COLOR | IMREAD_IGNORE_ORIENTATION).  One host->device copy carries the
    compressed bytes and the parsed headers; one epb_jpeg_decode call decodes every image the
    parser accepts.  Images the parser or the device reports as unsupported or malformed
    (progressive, 4:1:1, CMYK, truncated, ...) are decoded with cv2.imdecode on the host and copied
    into their slot; a blob cv2 cannot read either raises IOError naming its index.
    stats / events: optional int32 [EPB_JPEG_STATS] device tensor and EPB_JPEG_EVENTS recorded
    torch.cuda.Events (tools/bench_jpeg.py)."""
    ops = _backend[0]
    dev = _dev()
    bufs = [np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray, memoryview))
            else np.ascontiguousarray(np.asarray(b, dtype=np.uint8).reshape(-1)) for b in blobs]
    B = len(bufs)
    desc, status, hw, out_off, plan = ops.jpeg_parse(bufs)
    host = {i: _host_decode(bufs[i], i, _JPEG_STATUS[int(s)]) for i, s in enumerate(status) if s != 0}
    for i, img in host.items():
        hw[i] = img.shape[:2]
    out_off, out_bytes = _frame_offsets(hw)
    hwp = np.stack([hw[:, 0], hw[:, 1], hw[:, 1] * 3], axis=1).astype(np.int32) if B else np.zeros((0, 3), np.int32)
    # one pinned staging buffer -> one copy: blobs | descriptors | blob offsets | frame offsets | hwp | status
    blob_off = np.zeros(B, dtype=np.int64)
    pos = 0
    for i, b in enumerate(bufs):
        blob_off[i] = pos
        pos += (b.size + 16 + 15) // 16 * 16
    parts = [("desc", desc.reshape(-1)), ("blob_off", blob_off.view(np.uint8)), ("out_off", out_off.view(np.uint8)),
             ("hwp", hwp.reshape(-1).view(np.uint8)), ("status", status.view(np.uint8))]
    where, p = {}, pos
    for name, a in parts:
        where[name] = (p, a.size)
        p = (p + a.size + 15) // 16 * 16
    stage = torch.empty(max(p, 16), dtype=torch.uint8).pin_memory()
    sn = stage.numpy()
    for i, b in enumerate(bufs):
        sn[blob_off[i]:blob_off[i] + b.size] = b
    for name, a in parts:
        sn[where[name][0]:where[name][0] + a.size] = a
    d_stage = stage.to(dev, non_blocking=True)

    def view(name, dtype):
        o, n = where[name]
        return d_stage[o:o + n].view(dtype)
    d_off, d_hwp, d_status = view("out_off", torch.int64), view("hwp", torch.int32), view("status", torch.int32)
    out = torch.empty(max(out_bytes, 16), dtype=torch.uint8, device=dev)
    if int(plan[7]):
        ws = torch.empty(int(plan[0]), dtype=torch.uint8, device=dev)
        ops.jpeg_decode(d_stage, view("blob_off", torch.int64), view("desc", torch.uint8), B, plan, ws, out,
                        d_off, d_hwp, d_status, stats, events)
    dev_status = d_status.cpu().numpy()
    for i, s in enumerate(dev_status):
        if s != 0 and i not in host:
            img = _host_decode(bufs[i], i, _JPEG_STATUS[int(s)])
            if img.shape[:2] != tuple(hw[i]):
                raise IOError("JPEG blob %d: cv2 decodes %s, the header says %s" % (i, img.shape[:2], tuple(hw[i])))
            host[i] = img
    for i, img in host.items():
        out[int(out_off[i]):int(out_off[i]) + img.size].copy_(torch.from_numpy(img.reshape(-1)))
    frames = JpegFrames(out, d_off, d_hwp, [(int(h), int(w)) for h, w in hw], dev_status)
    frames._offs_host = out_off
    return frames


JPEG_TC_MISMATCH = 3          # transcode status: the verify decode differed from the source's


def transcode_jpeg_batch_device(blobs, interval='auto', verify=True):
    """B JPEG files (bytes or 1-D uint8 arrays) -> (list of B bytes, status int32 [B]): each file
    losslessly re-coded on the device with a restart interval of `interval` MCUs ('auto': per image
    the largest whose mean interval is at most 768 bits, so that the device decoder starts most
    1024-bit subsequences at a restart marker) and regenerated Huffman tables.  The quantised
    coefficients are kept, so every decoder gives the source's pixels.  The header keeps every
    segment before SOS except DHT and DRI; bytes after the source's EOI are dropped.
    Status 0: transcoded.  Blobs the device does not decode (1 unsupported, 2 malformed) come back
    unchanged.  verify: decode the outputs and the sources on the device and compare the frames;
    a difference returns the source unchanged with status JPEG_TC_MISMATCH (3)."""
    ops = _backend[0]
    dev = _dev()
    bufs = [np.frombuffer(b, dtype=np.uint8) if isinstance(b, (bytes, bytearray, memoryview))
            else np.ascontiguousarray(np.asarray(b, dtype=np.uint8).reshape(-1)) for b in blobs]
    B = len(bufs)
    if interval == 'auto':
        r = 0
    else:
        r = int(interval)
        if not 1 <= r <= 65535:
            raise ValueError("interval must be 'auto' or 1..65535 MCUs, got %r" % (interval,))
    if B == 0:
        return [], np.zeros(0, np.int32)
    desc, status, _, _, plan = ops.jpeg_parse(bufs)
    tdesc, tplan = ops.jpeg_transcode_plan(desc, B, np.full(B, r, np.int32), plan)
    blob_off = np.zeros(B, dtype=np.int64)
    pos = 0
    for i, b in enumerate(bufs):
        blob_off[i] = pos
        pos += (b.size + 16 + 15) // 16 * 16
    parts = [("desc", desc.reshape(-1)), ("tdesc", tdesc.reshape(-1)), ("blob_off", blob_off.view(np.uint8)),
             ("status", status.view(np.uint8))]
    where, p = {}, pos
    for name, a in parts:
        where[name] = (p, a.size)
        p = (p + a.size + 15) // 16 * 16
    stage = torch.empty(p, dtype=torch.uint8).pin_memory()
    sn = stage.numpy()
    for i, b in enumerate(bufs):
        sn[blob_off[i]:blob_off[i] + b.size] = b
    for name, a in parts:
        sn[where[name][0]:where[name][0] + a.size] = a
    d_stage = stage.to(dev, non_blocking=True)

    def view(name, dtype):
        o, n = where[name]
        return d_stage[o:o + n].view(dtype)
    args = (d_stage, view("blob_off", torch.int64), view("desc", torch.uint8), view("tdesc", torch.uint8), B, plan,
            tplan)
    ws = torch.empty(int(tplan[0]), dtype=torch.uint8, device=dev)
    hdr_off = np.zeros(B + 1, dtype=np.int64)
    hdr_off[1:] = np.cumsum([b.size + int(tplan[3]) for b in bufs])
    hdr = np.zeros(int(hdr_off[-1]), dtype=np.uint8)
    info = ops.jpeg_transcode(*args, ws, view("status", torch.int32), bufs, hdr, hdr_off)
    ok = info["status"] == 0
    ent = torch.empty(max(int((info["bytes"] * ok).sum()), 16), dtype=torch.uint8, device=dev)
    ops.jpeg_transcode_write(*args, ws, view("status", torch.int32), info, ent)
    ent_h = ent.cpu().numpy()
    out, st = [], info["status"].astype(np.int32)
    for i, b in enumerate(bufs):
        if not ok[i]:
            out.append(b.tobytes())
            continue
        h0, o = int(hdr_off[i]), int(info["off"][i])
        out.append(hdr[h0:h0 + int(info["hdr_bytes"][i])].tobytes() + ent_h[o:o + int(info["bytes"][i])].tobytes() +
                   b"\xff\xd9")
    if verify and ok.any():
        idx = [i for i in range(B) if ok[i]]
        src = decode_jpeg_batch_device([bufs[i] for i in idx])
        try:
            both = decode_jpeg_batch_device([out[i] for i in idx])
            new = [(both, k) for k in range(len(idx))]
        except IOError:                     # an output no decoder reads: check them one by one
            new = []
            for i in idx:
                try:
                    new.append((decode_jpeg_batch_device([out[i]]), 0))
                except IOError:
                    new.append((None, 0))
        for k, i in enumerate(idx):
            f, j = new[k]
            if src.status[k] != 0 or f is None or f.status[j] != 0 or not torch.equal(src.frame(k), f.frame(j)):
                out[i] = bufs[i].tobytes()
                st[i] = JPEG_TC_MISMATCH
    return out, st


def read_jpeg_batch_device(paths):
    """decode_jpeg_batch_device of the files at `paths`."""
    blobs = []
    for p in paths:
        with open(p, "rb") as f:
            blobs.append(f.read())
    return decode_jpeg_batch_device(blobs)


def generate_patch_batch_device(images, center_x, center_y, width, height, patch_width, patch_height,
                                scale=None, rot=None, do_flip=None, color_scale=None, mean=None, std=None,
                                occluders=None):
    """B decoded BGR frames (uint8 [H,W,3] numpy arrays or tensors, sizes may differ, or the
    JpegFrames of decode_jpeg_batch_device, read where they are) ->
    (patches float32 [B,3,ph,pw] on the device, trans float64 [B,2,3], box float64 [B,6]).
    occluders: per sample a list of (rgba uint8 [h,w,4], (cx, cy)) pasted onto the uint8 patch
    in order (augmentation.draw_occluders), or None."""
    ops = _backend[0]
    dev = _dev()
    B = len(images)
    if isinstance(images, JpegFrames):          # decoded on the device: no host round trip
        d_base, d_offs, d_hwp = images.base, images.offs, images.hwp
    else:
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
        d_base = base.to(dev)
        d_offs = torch.tensor(offs, dtype=torch.int64, device=dev)
        d_hwp = torch.tensor(hwp, dtype=torch.int32, device=dev)
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
        ops.patch_sample_occ(d_base, d_offs, d_hwp, t_box, t_flip, t_col, ms,
                             B, int(patch_width), int(patch_height), ob, od, oc, out, trans)
    else:
        ops.patch_sample(d_base, d_offs, d_hwp, t_box, t_flip, t_col, ms, B,
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


def get_patch_batch_device(img_paths, center_x, center_y, width, height, joints, joints_vis, flip_pairs,
                           parent_ids, patch_width, patch_height, rect_3d_width, rect_3d_height, mean, std,
                           do_augment, label_func, depth_in_image=False, occluder=None):
    """Batched, device-decoded get_single_patch_sample: B image files (or JPEG blobs) and per-sample
    boxes / joints [B,J,3] / joints_vis [B,J,3] -> (patches float32 [B,3,ph,pw] on the device, label
    [B,...], label_weight [B,...], scale [B], rot [B]) -- the stack of B sequential
    get_single_patch_sample calls, with the same np.random / random draws in the same order
    (do_augmentation(), then draw_occluders, per sample)."""
    B = len(img_paths)
    blobs = []
    for p in img_paths:
        if isinstance(p, (bytes, bytearray, memoryview, np.ndarray)):
            blobs.append(p)
        else:
            with open(p, "rb") as f:
                blobs.append(f.read())
    frames = decode_jpeg_batch_device(blobs)
    aug, occ = [], [] if occluder else None
    for _ in range(B):
        aug.append(do_augmentation() if do_augment else (1.0, 0, False, [1.0, 1.0, 1.0]))
        if occluder:
            from .augmentation import draw_occluders
            occ.append(draw_occluders(int(patch_width), int(patch_height), occluder))
    scale = np.array([a[0] for a in aug], dtype=np.float64)
    rot = np.array([a[1] for a in aug], dtype=np.float64)
    do_flip = [a[2] for a in aug]
    cx = np.asarray(center_x, dtype=np.float64).reshape(B)
    cy = np.asarray(center_y, dtype=np.float64).reshape(B)
    bw = np.asarray(width, dtype=np.float64).reshape(B)
    bh = np.asarray(height, dtype=np.float64).reshape(B)
    patches, trans, box = generate_patch_batch_device(frames, cx, cy, bw, bh, patch_width, patch_height, scale, rot,
                                                      do_flip, [a[3] for a in aug], mean, std, occluders=occ)
    jts, vis = [], []
    for i in range(B):
        j = np.array(joints[i], dtype=np.float64, copy=True)
        v = np.array(joints_vis[i], copy=True)
        if do_flip[i]:
            j, v = fliplr_joints(j, v, frames.sizes[i][1], flip_pairs)
        jts.append(j)
        vis.append(v)
    from ..core.integral_loss import generate_joint_location_label
    if label_func is None or label_func is generate_joint_location_label or \
            getattr(label_func, "__name__", "") == "generate_joint_location_label":
        label = patch_labels_device(np.stack(jts), box, trans, patch_width, patch_height, rect_3d_width,
                                    depth_in_image).cpu().numpy()
        label_weight = np.stack([v.reshape(-1) for v in vis])
    else:
        tr = trans.cpu().numpy()
        labels, weights = [], []
        for i in range(B):
            j = jts[i]
            for n_jt in range(len(j)):
                j[n_jt, 0:2] = np.dot(tr[i], np.array([j[n_jt, 0], j[n_jt, 1], 1.]).T)[0:2]
                den = (bw[i] * scale[i]) if depth_in_image else (rect_3d_width * scale[i])
                j[n_jt, 2] = j[n_jt, 2] / den * patch_width
            lab, w = label_func(patch_width, patch_height, j, vis[i])
            labels.append(lab)
            weights.append(w)
        label, label_weight = np.stack(labels), np.stack(weights)
    return patches, label, label_weight, scale, rot
