"""CPU: the heat-map decode (epb_heatmap_decode, csrc/geometry.cu) through its __host__ __device__ body
built for the CPU (tests/harness/host_heatmap_decode.cu), against the numpy restatement of the
reference's get_max_preds / get_final_preds refinement / get_depth_preds (tests/heatmap_cases.py)
and against the unmodified reference on one pinned set (tests/golden/heatmap_decode.npz); the
refusals of validate_integral's VOLUME = false path."""
import numpy as np
import pytest
import torch

from oracle import refshim
from tests import heatmap_cases as hc


@pytest.fixture(scope="module")
def decode():
    run = hc.harness()
    if run is None:
        pytest.skip("nvcc not available")
    return run


def test_restatement_matches_the_reference(golden):
    """The restatement the tests below use equals the unmodified reference on the pinned set."""
    g = golden("heatmap_decode")
    hm, depth = g["hm"], g["depth"]
    N, J = hm.shape[:2]
    coords, maxvals, _ = hc.restate.get_max_preds(hm)
    assert np.array_equal(coords, g["preds"]) and np.array_equal(maxvals.reshape(N, J), g["maxvals"].reshape(N, J))
    refined = hc.restate.final_preds_refine(hm, coords)
    assert np.array_equal(refined, g["refined"])
    d = hc.depth_preds64(depth, J, 16, 2000.0)
    assert np.max(hc.ulps32(g["depth_mm"], d)) <= 4.0


@pytest.mark.parametrize("layout", [0, 1])
def test_kernel_body_matches_the_reference_golden(decode, golden, layout):
    g = golden("heatmap_decode")
    hm, depth = g["hm"], g["depth"]
    N, J, H, W = hm.shape
    kps = decode(hm, depth, 16, patch_w=float(W), patch_h=float(H), layout=layout, C=J + 3 * layout)
    assert np.array_equal(kps[..., :2].astype(np.float32), g["refined"])
    assert np.array_equal(kps[..., 3], g["maxvals"].reshape(N, J).astype(np.float64))
    assert np.max(hc.ulps32(kps[..., 2], hc.depth_preds64(depth, J, 16, 2000.0))) <= 4.0
    # the reference's own float32 arithmetic (np.exp without the maximum) agrees to its rounding
    assert np.max(np.abs(kps[..., 2] - g["depth_mm"])) <= 2000.0 * 1e-5
    unref = decode(hm, depth, 16, patch_w=float(W), patch_h=float(H), post_process=False, layout=layout,
                   C=J + 3 * layout)
    assert np.array_equal(unref[..., :2].astype(np.float32), g["preds"])


@pytest.mark.parametrize("post_process", [True, False])
@pytest.mark.parametrize("layout", [0, 1])
def test_crafted_maps(decode, layout, post_process):
    """Ties (first index), maxima on each border row / column (refinement skipped), maxval <= 0
    (coordinates zeroed), equal neighbours (sign 0), 48 x 64 maps; padding channels hold NaN."""
    hm, depth = hc.crafted()
    J, H, W = hm.shape[1:]
    kps = decode(hm, depth, 16, post_process=post_process, layout=layout, C=J + 2 * layout)
    hc.check_against_ref(kps, hm, depth, 16, 256.0, 256.0, 2000.0, post_process)
    sx, sy = 256.0 / W, 256.0 / H
    assert tuple(np.round(kps[0, 0, :2] / (sx, sy))) == (20, 10)  # tie: the first index (then refined)
    assert tuple(kps[0, 1, :2]) == (33 * sx, 0.0)               # top row: no refinement
    assert tuple(kps[0, 2, :2]) == (7 * sx, (H - 1) * sy)
    assert tuple(kps[0, 3, :2]) == (0.0, 17 * sy)
    assert tuple(kps[0, 4, :2]) == (0.0, 0.0) and kps[0, 4, 3] < 0
    assert tuple(kps[0, 5, :2]) == (30 * sx, 20 * sy)           # equal neighbours: sign 0


@pytest.mark.parametrize("J,D,shape", [(16, 64, (64, 64)), (17, 16, (48, 64)), (17, 64, (64, 48)),
                                       (16, 16, (48, 64))])
def test_seeded_maps(decode, J, D, shape):
    H, W = shape
    hm, depth = hc.seeded(3, J, H, W, D, 100 + J + D)
    C = (J + 3) // 4 * 4
    a = decode(hm, depth, D, layout=0)
    b = decode(hm, depth, D, layout=1, C=C)
    assert np.array_equal(a, b)
    worst = hc.check_against_ref(a, hm, depth, D, 256.0, 256.0, 2000.0)
    print("J %d D %d %dx%d: depth %.2f float32 ulps of float64" % (J, D, H, W, worst))


def test_depth_for_logits_beyond_the_references_exp(decode):
    """Logits above ~88 overflow the reference's float32 exp; the max-subtracted form decodes them."""
    J, D = 4, 16
    hm, depth = hc.seeded(2, J, 8, 8, D, 3)
    depth = (depth + 500.0).astype(np.float32)
    kps = decode(hm, depth, D)
    assert np.isfinite(kps).all()
    assert np.max(hc.ulps32(kps[..., 2], hc.depth_preds64(depth, J, D, 2000.0))) <= 4.0


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("J", [16, 17])
def test_flip_merge(decode, J, shift):
    """The batch [x; flip(x)]: the decode of the merged maps and depth rows, never written."""
    N, D, H, W = 3, 16, 48, 64
    pairs = hc.pairs_of(J)
    hm2, d2 = hc.seeded(N, J, H, W, D, 40 + J, B=2 * N)
    mh, md = hc.flip_merge(hm2, d2, pairs, shift)
    want = decode(mh, md, D)
    for layout in (0, 1):
        got = decode(hm2, d2, D, pairs=pairs, shift=shift, layout=layout, C=(J + 3) // 4 * 4 + 4 * layout)
        assert np.array_equal(got, want)
    hc.check_against_ref(want, mh, md, D, 256.0, 256.0, 2000.0)


def test_affine_is_patch_to_images(decode):
    """With boxes, x and y are epb_patch_to_image's image points of the decoded patch pixels, bit for bit."""
    N, J, D, H, W = 4, 17, 16, 64, 64
    hm, depth = hc.seeded(N, J, H, W, D, 9)
    box = hc.boxes(N, 10)
    patch = decode(hm, depth, D)
    img = decode(hm, depth, D, box=box)
    assert np.array_equal(img[..., 2:], patch[..., 2:])
    c = hc.exact_patch_coords(patch[..., 0], patch[..., 1], 256.0, 256.0)
    k = decode.p2i(c, np.repeat(box, J, axis=0)).reshape(N, J, 4)
    assert np.array_equal(img[..., :2], k[..., :2])


def test_flat_validation_refusals():
    """Validation of a VOLUME = false network refuses a trunk that cannot feed depth_fc (ResNet-18:
    512 channels, depth_fc reads 2048) with or without flip test, and flip test without the dataset's
    joint pairs; both before any forward."""
    import lib.models as models
    from lib.core.config import reset_config
    from lib.core.function import validate_integral
    from tests import emul_ops
    from tests.test_flip_host import _setup
    try:
        config, r18, ds, loader = _setup(16, volume=False, n=4)
        for flip in (False, True):
            with pytest.raises(ValueError, match="2048-channel trunk"):
                validate_integral(loader, r18, flip_test=flip)
        cfg = refshim.make_cfg(num_layers=50, num_joints=16, volume=False, depth_res=8, image_size=(64, 64))
        r50 = models.pose3d_resnet.get_pose_net(cfg, False, ops=emul_ops)

        class NoPairs(torch.utils.data.Dataset):
            db = [{"image": "x"}]

            def __len__(self):
                return len(ds)

            def __getitem__(self, i):
                return ds[i]
        with pytest.raises(ValueError, match="pairs"):
            validate_integral(torch.utils.data.DataLoader(NoPairs(), batch_size=4), r50, flip_test=True)
    finally:
        reset_config()
