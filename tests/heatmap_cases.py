"""Shared by the heat-map decode tests: the numpy restatement of the reference decode
(lib/core/inference.py get_max_preds / get_final_preds / get_depth_preds) with the Simple Baselines
flip merge, the crafted and seeded inputs, and the CPU build of the kernel body
(tests/harness/host_heatmap_decode.cu)."""
import os
import shutil
import subprocess

import numpy as np

from oracle import restate
from tests.conftest import ROOT

H36M_PAIRS = ((1, 4), (2, 5), (3, 6), (14, 11), (15, 12), (16, 13))
MPII_PAIRS = ((0, 5), (1, 4), (2, 3), (10, 15), (11, 14), (12, 13))


def pairs_of(J):
    """The dataset's pairs for J = 16 / 17, an arbitrary involution otherwise."""
    if J == 16:
        return MPII_PAIRS
    if J == 17:
        return H36M_PAIRS
    return tuple((2 * k, 2 * k + 1) for k in range(J // 2) if k % 2 == 0)


def perm_of(pairs, J):
    perm = list(range(J))
    for a, b in pairs:
        perm[a], perm[b] = perm[b], perm[a]
    return perm


def flip_merge(hm2N, depth2N, pairs, shift):
    """Simple Baselines' merge on the 2N batch [x; flip(x)] (float32, as the network's outputs)."""
    N = hm2N.shape[0] // 2
    J = hm2N.shape[1]
    perm = perm_of(pairs, J)
    fb = hm2N[N:][:, perm, :, ::-1].copy()                  # flip_back: mirror columns, swap pairs
    if shift:
        fb[:, :, :, 1:] = fb.copy()[:, :, :, 0:-1]
    D = depth2N.shape[1] // J
    db = depth2N[N:].reshape(N, J, D)[:, perm].reshape(N, J * D)
    return ((hm2N[:N] + fb) * np.float32(0.5)).astype(np.float32), \
        ((depth2N[:N] + db) * np.float32(0.5)).astype(np.float32)


def depth_preds64(depth, J, D, depth_range):
    """get_depth_preds in float64 with the maximum subtracted -> [N, J]."""
    v = np.asarray(depth, dtype=np.float64).reshape(-1, J, D)
    e = np.exp(v - v.max(axis=2, keepdims=True))
    s = (e * np.arange(D)).sum(axis=2) / e.sum(axis=2)
    return (s / D - 0.5) * depth_range


def decode_ref(hm, depth, D, patch_w, patch_h, depth_range, post_process=True):
    """The reference decode of (hm [N, J, H, W] f32, depth [N, J*D]) in the patch frame ->
    ([N, J, 2] float32 heat-map coordinates, maxvals [N, J], depth [N, J] float64 mm,
    [N, J, 2] float64 patch pixels)."""
    N, J, H, W = hm.shape
    coords, maxvals, _ = restate.get_max_preds(hm)
    if post_process:
        coords = restate.final_preds_refine(hm, coords)
    px = np.stack([coords[..., 0].astype(np.float64) * (patch_w / W),
                   coords[..., 1].astype(np.float64) * (patch_h / H)], axis=-1)
    return coords, maxvals.reshape(N, J), depth_preds64(depth, J, D, depth_range), px


def ulps32(got, ref):
    """|got - ref| in float32 ulps of ref."""
    ref = np.asarray(ref, dtype=np.float64)
    u = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    return np.abs(np.asarray(got, dtype=np.float64) - ref) / u


def seeded(N, J, H, W, D, seed, B=None):
    """Peaked seeded maps (one Gaussian per joint plus noise) and depth logits for B (default N) rows."""
    B = N if B is None else B
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:H, 0:W]
    hm = 0.02 * rng.standard_normal((B, J, H, W))
    cy = rng.uniform(0, H - 1, (B, J, 1, 1))
    cx = rng.uniform(0, W - 1, (B, J, 1, 1))
    hm += np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / 6.0)
    depth = 4.0 * rng.standard_normal((B, J * D))
    return hm.astype(np.float32), depth.astype(np.float32)


def crafted(J=6, H=48, W=64, D=16):
    """One image of the edge cases: ties, maxima on each border row and column, maxval <= 0,
    equal neighbours, a refinement in both directions."""
    hm, depth = seeded(1, J, H, W, D, 5)
    hm[0, :] *= 0.1
    hm[0, 0, 10, 20] = hm[0, 0, 30, 5] = 2.0              # tie
    hm[0, 1, 0, 33] = 3.0                                 # top row
    hm[0, 2, H - 1, 7] = 3.0                              # bottom row
    hm[0, 3, 17, 0] = 3.0                                 # left column
    hm[0, 3, 18, W - 1] = 3.0                             #   tie with the right column: left wins
    hm[0, 4] = -np.abs(hm[0, 4]) - 0.25                   # maxval <= 0
    hm[0, 5] = 0.0
    hm[0, 5, 20, 30] = 4.0                                # equal neighbours
    hm[0, 5, 20, 29] = hm[0, 5, 20, 31] = hm[0, 5, 19, 30] = hm[0, 5, 21, 30] = 1.0
    return hm, depth


def harness():
    """Build tests/harness/host_heatmap_decode.cu (None without nvcc) and return its runner."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        return None
    import tempfile
    exe = os.path.join(tempfile.mkdtemp(prefix="hm_harness_"), "host_heatmap_decode")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1", "-std=c++17",
                        "-o", exe, os.path.join(ROOT, "tests", "harness", "host_heatmap_decode.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def decode(hm, depth, D, box=None, patch_w=256.0, patch_h=256.0, depth_range=2000.0, post_process=True,
               pairs=None, shift=False, layout=0, C=None):
        """hm [B, J, H, W] float32 (laid out as `layout` for the run), depth [B, J*D] -> kps [N, J, 4]."""
        B, J, H, W = hm.shape
        N = B // 2 if pairs is not None else B
        C = J if C is None else C
        if layout == 1:
            buf = np.full((B, H, W, C), np.nan, dtype=np.float32)
            buf[..., :J] = hm.transpose(0, 2, 3, 1)
        else:
            buf = np.ascontiguousarray(hm, dtype=np.float32)
        inp = buf.tobytes() + np.ascontiguousarray(depth, dtype=np.float32).tobytes()
        if box is not None:
            inp += np.ascontiguousarray(box, dtype=np.float64).tobytes()
        if pairs is not None:
            inp += np.asarray(perm_of(pairs, J), dtype=np.int32).tobytes()
        args = [exe, "decode", layout, C, N, J, H, W, D, repr(float(patch_w)), repr(float(patch_h)),
                repr(float(depth_range)), int(post_process), int(pairs is not None), int(shift), int(box is not None)]
        out = subprocess.run([str(a) for a in args], input=inp, capture_output=True)
        assert out.returncode == 0, out.stderr
        return np.frombuffer(out.stdout, dtype=np.float64).reshape(N, J, 4)

    def p2i(coords, box, patch_w=256.0, patch_h=256.0):
        """patch_to_image_point (epb_patch_to_image's body): coords [B, 3] f32, box [B, 6] -> [B, 4]."""
        B = len(coords)
        inp = np.ascontiguousarray(coords, dtype=np.float32).tobytes() + \
            np.ascontiguousarray(box, dtype=np.float64).tobytes()
        out = subprocess.run([exe, "p2i", str(B), repr(float(patch_w)), repr(float(patch_h))], input=inp,
                             capture_output=True)
        assert out.returncode == 0, out.stderr
        return np.frombuffer(out.stdout, dtype=np.float64).reshape(B, 4)

    decode.p2i = p2i
    return decode


def boxes(N, seed):
    rng = np.random.default_rng(seed)
    return np.stack([rng.uniform(200, 800, N), rng.uniform(200, 600, N), rng.uniform(150, 400, N),
                     rng.uniform(150, 400, N), rng.uniform(0.8, 1.2, N), rng.uniform(-30, 30, N)], axis=1)


def exact_patch_coords(px, py, patch_w, patch_h):
    """Normalised soft-argmax coordinates c with (c + 0.5) * patch = (px, py) exactly (px, py dyadic)."""
    c = np.zeros((px.size, 3), dtype=np.float32)
    c[:, 0] = (px.reshape(-1) / patch_w - 0.5).astype(np.float32)
    c[:, 1] = (py.reshape(-1) / patch_h - 0.5).astype(np.float32)
    assert np.array_equal((c[:, 0].astype(np.float64) + 0.5) * patch_w, px.reshape(-1))
    assert np.array_equal((c[:, 1].astype(np.float64) + 0.5) * patch_h, py.reshape(-1))
    return c


def check_against_ref(kps, hm, depth, D, patch_w, patch_h, depth_range, post_process=True):
    """x, y, maxval bit-exact and depth within 4 float32 ulps of the float64 restatement (patch frame)."""
    coords, maxvals, dref, px = decode_ref(hm, depth, D, patch_w, patch_h, depth_range, post_process)
    assert np.array_equal(kps[..., :2], px), np.argwhere(kps[..., :2] != px)[:5]
    assert np.array_equal(kps[..., 3], maxvals.astype(np.float64))
    worst = float(np.max(ulps32(kps[..., 2], dref)))
    assert worst <= 4.0, worst
    return worst

