"""Seeded inputs of the flip-test golden vectors (tests/golden/make_golden_flip.py) and of the tests
that read them (tests/test_flip_host.py): logits of a 2N batch [x; flip(x)], the joint pairs the
synthetic dataset uses, and index arrays that record where flip / flip_back move each element.
Also the float64 oracle of the flip-test merge, flip_merge_softargmax, pinned to the reference by
flip_test.npz (tests/test_flip_host.py) and the yardstick of the GPU tests (tests/test_gpu_flip.py)."""
import numpy as np

from tests import golden_inputs as gi

MPII_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
H36M_PAIRS = [[1, 4], [2, 5], [3, 6], [14, 11], [15, 12], [16, 13]]

# tag -> (N, J, D, H, W, seed, logit scale, pairs)
CASES = {
    "j16": (2, 16, 8, 16, 16, 41, 3.0, MPII_PAIRS),
    "j17": (2, 17, 8, 16, 16, 42, 3.0, H36M_PAIRS),
}


def logits2N(tag):
    N, J, D, H, W, seed, scale, _ = CASES[tag]
    return gi.logits(2 * N, J, D, H, W, seed, scale)


def index_volume(tag, rows=3):
    """[N, J, rows, W] int32 element indices: flip_back of it is its index map (flip_back moves
    nothing along the row axis, so a few rows pin it as well as D*H of them)."""
    N, J, D, H, W = CASES[tag][:5]
    return np.arange(N * J * rows * W, dtype=np.int32).reshape(N, J, rows, W)


def index_images(N=2, C=3, H=16, W=16):
    return np.arange(N * C * H * W, dtype=np.int64).reshape(N, C, H, W)


def flip_merge_softargmax(preds2N, num_joints, hm_width, hm_height, hm_depth, flip_pairs, shift_heatmap):
    """preds2N [2N, J*D, H, W]: logits of [x; flip(x, 3)] (img_utils.py:319-331) -> [N, J*3]
    float64 soft-argmax of the flip-test merge, everything in float64:
      Fb = flip_back(L[N:] viewed as [N, J, D*H, W], flip_pairs)      transforms.py:5-19
      shift_heatmap: Fb[..., 1:] = Fb[..., :-1]  (column 0 keeps its value; config.py:120)
      merged = 0.5 * (L[:N] + Fb),  then softmax_integral_tensor (integral_loss.py:71-86)."""
    J, D, H, W = num_joints, hm_depth, hm_height, hm_width
    p = np.asarray(preds2N, dtype=np.float64)
    n = p.shape[0] // 2
    fb = p[n:].reshape(n, J, D * H, W)[:, :, :, ::-1].copy()
    for a, b in flip_pairs:
        fb[:, [a, b]] = fb[:, [b, a]]
    if shift_heatmap:
        fb[..., 1:] = fb[..., :-1].copy()
    merged = 0.5 * (p[:n] + fb.reshape(n, J * D, H, W))
    v = merged.reshape(n, J, -1)
    e = np.exp(v - v.max(axis=2, keepdims=True))
    sm = (e / e.sum(axis=2, keepdims=True)).reshape(n, J, D, H, W)
    x = sm.sum(axis=(2, 3)) @ np.arange(W, dtype=np.float64) / W - 0.5
    y = sm.sum(axis=(2, 4)) @ np.arange(H, dtype=np.float64) / H - 0.5
    z = sm.sum(axis=(3, 4)) @ np.arange(D, dtype=np.float64) / D - 0.5
    return np.stack([x, y, z], axis=2).reshape(n, J * 3)
