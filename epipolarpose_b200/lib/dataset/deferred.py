"""Deferred samples: the host half of get_single_patch_sample (reference
lib/utils/img_utils.py:246-298) in a DataLoader worker, the device half batched in the main
process.

A worker cannot use CUDA once its parent has initialised it, and the reference's scripts build
their loaders with num_workers=config.WORKERS.  So a dataset indexed in a worker returns
`make_deferred(...)`: a dict that holds the file's bytes, the box, the joints (flipped as
get_single_patch_sample would flip them), the do_augmentation() draws and the occluder draws, in
the reference's order (augmentation, then occluders, :260-272).  torch's default_collate batches
it unchanged: numbers and arrays become tensors, `bytes` become lists, so occluders of different
sizes travel packed as bytes.  `assemble_batch` then builds the batch on the device with one
decode_jpeg_batch_device, one generate_patch_batch_device and one patch_labels_device call;
frames the device decoder rejects (progressive, ...) are decoded by cv2 on the host there."""
import struct

import numpy as np
import torch

from ..utils import img_utils as _iu

KEY = 'epb_deferred'

_SOF = {0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC6, 0xC7, 0xC9, 0xCA, 0xCB, 0xCD, 0xCE, 0xCF}


def jpeg_width(blob):
    """Image width from the frame header of a JPEG file (what the reference's fliplr_joints
    reads from the decoded frame), without decoding it."""
    pos, n = 2, len(blob)
    while pos + 4 <= n:
        if blob[pos] != 0xFF:
            pos += 1
            continue
        marker = blob[pos + 1]
        if marker == 0xFF or 0xD0 <= marker <= 0xD8 or marker == 0x01:
            pos += 2 if marker != 0xFF else 1
            continue
        length = struct.unpack('>H', blob[pos + 2:pos + 4])[0]
        if marker in _SOF and pos + 9 <= n:
            return struct.unpack('>H', blob[pos + 7:pos + 9])[0]
        pos += 2 + length
    raise IOError("no JPEG frame header found")


def pack_occluders(lst):
    """[(rgba uint8 [h, w, 4], (cx, cy)), ...] (augmentation.draw_occluders) -> bytes."""
    out = [struct.pack('<i', len(lst))]
    for rgba, (cx, cy) in lst:
        rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
        out.append(struct.pack('<4i', rgba.shape[0], rgba.shape[1], int(cx), int(cy)))
        out.append(rgba.tobytes())
    return b''.join(out)


def unpack_occluders(buf):
    """Inverse of pack_occluders."""
    (count,), pos, out = struct.unpack_from('<i', buf, 0), 4, []
    for _ in range(count):
        h, w, cx, cy = struct.unpack_from('<4i', buf, pos)
        pos += 16
        rgba = np.frombuffer(buf, dtype=np.uint8, count=h * w * 4, offset=pos).reshape(h, w, 4)
        pos += h * w * 4
        out.append((rgba, (cx, cy)))
    return out


def make_deferred(blob, box, joints, joints_vis, flip_pairs, do_augment, occluders, geometry, mean, std,
                  meta):
    """One view, drawn as get_single_patch_sample draws it.  geometry = (patch_width,
    patch_height, rect_3d_width); `meta` gets the drawn scale / rot when it has those keys."""
    pw, ph, rect = geometry
    if do_augment:
        scale, rot, do_flip, color_scale = _iu.do_augmentation()
    else:
        scale, rot, do_flip, color_scale = 1.0, 0, False, [1.0, 1.0, 1.0]
    occ = []
    if occluders:
        from ..utils.augmentation import draw_occluders
        occ = draw_occluders(int(pw), int(ph), occluders)
    joints = np.array(joints, dtype=np.float64, copy=True)
    joints_vis = np.array(joints_vis, dtype=np.float64, copy=True)
    if do_flip:
        joints, joints_vis = _iu.fliplr_joints(joints, joints_vis, jpeg_width(blob), flip_pairs)
    if 'scale' in meta:
        meta['scale'], meta['rot'] = float(scale), float(rot)
    return {KEY: 1, 'jpeg': bytes(blob), 'box': np.array(box, dtype=np.float64),
            'joints': joints, 'joints_vis': joints_vis,
            'aug': np.array([scale, rot, float(bool(do_flip))] + list(color_scale), dtype=np.float64),
            'occluders': pack_occluders(occ),
            'geometry': np.array([pw, ph, rect], dtype=np.float64),
            'mean_std': np.concatenate([np.asarray(mean, np.float64), np.asarray(std, np.float64)]),
            'meta': meta}


def view_keys(batch):
    """['cam_1', .., 'cam_V'] of a TRI batch (a dict with at least 'cam_1' and 'cam_2'), else []."""
    if not (isinstance(batch, dict) and 'cam_1' in batch and 'cam_2' in batch):
        return []
    keys = []
    while 'cam_%d' % (len(keys) + 1) in batch:
        keys.append('cam_%d' % (len(keys) + 1))
    return keys


def is_deferred(batch):
    """A collated batch of deferred samples, or of TRI tuples {'cam_1', .., 'cam_V'} of them."""
    keys = view_keys(batch)
    if keys:
        return is_deferred(batch[keys[0]])
    return isinstance(batch, dict) and KEY in batch


def _np(v):
    return v.numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def cat_meta(*metas):
    """Collated meta of batches a, b, .. -> the meta of [a ; b ; ..]."""
    a = metas[0]
    out = {}
    for k in a:
        x = a[k]
        if isinstance(x, torch.Tensor):
            out[k] = torch.cat([x] + [m[k].to(x.device) for m in metas[1:]], dim=0)
        elif isinstance(x, (list, tuple)):
            out[k] = [e for m in metas for e in m[k]]
        else:
            out[k] = np.concatenate([_np(m[k]) for m in metas], axis=0)
    return out


def assemble_batch(batch):
    """Collated deferred batch -> device (images f32 [B,3,H,W], label f32 [B,J*3], weight f32
    [B,J*3], meta) -- each sample identical to get_single_patch_sample with that sample's draws,
    meta carrying the drawn scale / rot.  A TRI batch {'cam_1', .., 'cam_V'} becomes one batch of VB,
    [cam_1 ; .. ; cam_V]: row v*B + t is view v of tuple t (for V = 2 the pairing of sample i with
    sample i + B, reference img_utils.py:194-199)."""
    keys = view_keys(batch)
    if keys:
        parts = [assemble_batch(batch[k]) for k in keys]
        return (torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]), torch.cat([p[2] for p in parts]),
                cat_meta(*[p[3] for p in parts]))
    if KEY not in batch:
        raise ValueError("not a batch of deferred samples")
    blobs = list(batch['jpeg'])
    B = len(blobs)
    box, aug = _np(batch['box']).reshape(B, 4), _np(batch['aug']).reshape(B, 6)
    pw, ph, rect = (float(v) for v in _np(batch['geometry']).reshape(B, 3)[0])
    ms = _np(batch['mean_std']).reshape(B, 6)[0]
    occ = [unpack_occluders(b) for b in batch['occluders']]
    frames = _iu.decode_jpeg_batch_device(blobs)
    patches, trans, tbox = _iu.generate_patch_batch_device(
        frames, box[:, 0], box[:, 1], box[:, 2], box[:, 3], int(pw), int(ph), scale=aug[:, 0], rot=aug[:, 1],
        do_flip=aug[:, 2] != 0, color_scale=aug[:, 3:6], mean=ms[0:3], std=ms[3:6],
        occluders=occ if any(occ) else None)
    joints = _np(batch['joints'])
    label = _iu.patch_labels_device(joints, tbox, trans, pw, ph, rect).to(torch.float32)
    weight = torch.as_tensor(_np(batch['joints_vis']).reshape(B, -1)).to(patches.device, torch.float32)
    return patches, label, weight, batch['meta']
