"""Centre/scale affine helpers used by get_final_preds -- mirror of the
subset of reference lib/utils/transforms.py (:38-94) on the decode path, and
flip_back (:5-19) of the flip test.
The three-point affine that the reference obtains from cv2.getAffineTransform
is solved directly in float64 numpy (tiny host-side arithmetic; image warps
and flips belong to the data-loader, which is out of the hot path)."""
import numpy as np


def flip_back(output_flipped, matched_parts):
    """reference :5-19: mirror a [batch, joints, height, width] array along width and swap each
    left/right pair of joints, pairs in order.  Like the reference, the result is a reversed view
    of the input and the swaps write through it."""
    assert output_flipped.ndim == 4, 'flip_back expects [batch, joints, height, width]'
    out = output_flipped[..., ::-1]
    for a, b in matched_parts:
        out[:, [a, b]] = out[:, [b, a]]          # the right-hand side is a copy
    return out


def _affine_from_points(src, dst):
    a = np.concatenate([np.asarray(src, np.float32).astype(np.float64), np.ones((3, 1))], axis=1)
    return np.linalg.solve(a, np.asarray(dst, np.float32).astype(np.float64)).T.copy()


def get_dir(src_point, rot_rad):
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    return [src_point[0] * cs - src_point[1] * sn, src_point[0] * sn + src_point[1] * cs]


def get_3rd_point(a, b):
    d = a - b
    return b + np.array([-d[1], d[0]], dtype=np.float32)


def get_affine_transform(center, scale, rot, output_size,
                         shift=np.array([0, 0], dtype=np.float32), inv=0):
    if not isinstance(scale, (np.ndarray, list)):
        scale = np.array([scale, scale])
    scale_tmp = np.asarray(scale) * 200.0
    src_w, dst_w, dst_h = scale_tmp[0], output_size[0], output_size[1]
    src_dir = get_dir([0, src_w * -0.5], np.pi * rot / 180)
    dst_dir = np.array([0, dst_w * -0.5], np.float32)
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0, :] = center + scale_tmp * shift
    src[1, :] = center + src_dir + scale_tmp * shift
    dst[0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[1, :] = np.array([dst_w * 0.5, dst_h * 0.5]) + dst_dir
    src[2:, :] = get_3rd_point(src[0, :], src[1, :])
    dst[2:, :] = get_3rd_point(dst[0, :], dst[1, :])
    return _affine_from_points(dst, src) if inv else _affine_from_points(src, dst)


def affine_transform(pt, t):
    return np.dot(t, np.array([pt[0], pt[1], 1.]).T)[:2]


def transform_preds(coords, center, scale, output_size):
    out = np.zeros(coords.shape)
    trans = get_affine_transform(center, scale, 0, output_size, inv=1)
    for p in range(coords.shape[0]):
        out[p, 0:2] = affine_transform(coords[p, 0:2], trans)
    return out
