"""GPU (-m gpu): flip test.  epb_softargmax_flip_fwd against the float64 oracle of the merge at the
validation size (N=32, J16 / J17, D64, 64x64) with the shift on and off, the torch-op fallback,
argument errors, the 2N-batch forward, the mirror symmetry of the fused index mapping, and
validate_integral + eval_integral end to end.  Soft-argmax bar as the existing forward: 1e-5 abs in
normalised coordinates."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import refshim, restate_net
from tests import flip_cases as fc
from tests.conftest import relerr

pytestmark = pytest.mark.gpu
EPB_EINVAL = -1                   # include/epb.h


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _logits(dev, N2, J, D, H, W, seed):
    """Random logits (scale 3) with a few peaked joints, channels_last view [N2, J*D, H, W]."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = 3.0 * torch.randn((N2, H, W, J * D), device=dev, generator=g)
    rng = np.random.default_rng(seed)
    for n in range(0, N2, 3):
        for j in rng.choice(J, 4, replace=False):
            h, w, d = rng.integers(0, H), rng.integers(0, W), rng.integers(0, D)
            x[n, h, w, j * D + d] += 14.0
    return x.permute(0, 3, 1, 2)


def _oracle(L2, J, D, H, W, pairs, shift):
    """Per-sample float64 oracle (keeps host memory small at N=32)."""
    N = L2.shape[0] // 2
    return np.concatenate([fc.flip_merge_softargmax(np.concatenate([L2[n:n + 1], L2[N + n:N + n + 1]]),
                                                    J, W, H, D, pairs, shift) for n in range(N)])


def _pairs(J):
    return fc.MPII_PAIRS if J == 16 else fc.H36M_PAIRS


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("J", [16, 17])
def test_flip_kernel_vs_float64(dev, J, shift):
    from epipolarpose_b200 import ops
    import lib.core.integral_loss as il
    N, D, H, W = 32, 64, 64, 64
    x = _logits(dev, 2 * N, J, D, H, W, 100 + J + int(shift))
    perm = il.flip_permutation(_pairs(J), J)
    coords = torch.empty((N, J * 3), device=dev)
    ops.softargmax_flip_fwd(x.permute(0, 2, 3, 1), N, J, D, H, W, perm, int(shift), coords)
    ref = _oracle(x.cpu().numpy(), J, D, H, W, _pairs(J), shift)
    err = np.max(np.abs(coords.cpu().numpy() - ref))
    assert err <= 1e-5, err
    c2 = il.softmax_integral_flip(x, J, W, H, D, _pairs(J), shift)           # the Python surface
    assert torch.equal(c2, coords)


class _Recorder:
    def __init__(self, ops):
        self.ops, self.calls = ops, []

    def __getattr__(self, name):
        fn = getattr(self.ops, name)

        def rec(*a, **k):
            self.calls.append(name)
            return fn(*a, **k)
        return rec


@pytest.mark.parametrize("case", ["d6_channels_last", "nchw"])
def test_flip_fallback_vs_float64(dev, case):
    """D % 4 != 0 and contiguous NCHW logits take the torch-op merge + epb_softargmax_fwd."""
    import lib.core.integral_loss as il
    N, J, H, W = 4, 16, 32, 32
    D = 6 if case == "d6_channels_last" else 32
    x = _logits(dev, 2 * N, J, D, H, W, 7)
    if case == "nchw":
        x = x.contiguous()
    rec = _Recorder(il._backend[0])
    il._backend[0] = rec
    try:
        for shift in (False, True):
            c = il.softmax_integral_flip(x, J, W, H, D, _pairs(J), shift)
            ref = _oracle(x.cpu().numpy(), J, D, H, W, _pairs(J), shift)
            assert np.max(np.abs(c.cpu().numpy() - ref)) <= 1e-5
    finally:
        il._backend[0] = rec.ops
    assert "softargmax_flip_fwd" not in rec.calls and "softargmax_fwd" in rec.calls


def test_flip_entry_point_rejects_bad_arguments(dev):
    from epipolarpose_b200 import _lib
    L = _lib.lib()
    N, J, D, H, W = 2, 4, 8, 8, 8
    x = torch.zeros((2 * N, H, W, J * D), device=dev)
    coords = torch.full((N, J * 3), 7.0, device=dev)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(perm, J=J, D=D, shift=0):
        return L.epb_softargmax_flip_fwd(ctypes.c_void_p(x.data_ptr()), N, J, D, H, W,
                                         (ctypes.c_int * len(perm))(*perm), shift,
                                         ctypes.c_void_p(coords.data_ptr()), st)
    for perm in ([0, 1, 2, 4], [0, 1, 2, -1], [1, 2, 0, 3], [1, 1, 2, 3]):
        assert call(perm) == EPB_EINVAL
        assert "perm" in L.epb_last_error().decode()
    assert call([0, 1, 2, 3], shift=2) == EPB_EINVAL
    assert call([0, 1, 2], J=3, D=6) == EPB_EINVAL                   # D % 4 != 0
    assert call(list(range(129)), J=129, D=32) == EPB_EINVAL         # J*D/4 > 1024
    torch.cuda.synchronize()
    assert bool((coords == 7.0).all())                        # nothing was launched
    assert call([1, 0, 2, 3]) == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(coords).all()) and not bool((coords == 7.0).any())


def test_flip_batch_composition_r50(dev):
    """One forward of [x; flip(x)] equals the two separate forwards (eval BatchNorm)."""
    import lib.models as models
    from tests import golden_inputs as gi
    J, D, HW, N = 16, 64, 256, 4
    cfg = refshim.make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    model = models.pose3d_resnet.get_pose_net(cfg, False)
    model.load_state_dict(restate_net.init_state(restate_net.param_shapes(50, J, True, D), 23))
    model = model.to(dev).eval()
    x = torch.from_numpy(gi.images(N, HW, 24)).to(dev)
    buf = torch.empty((2 * N, 3, HW, HW), device=dev)
    buf[:N] = x
    buf[N:] = torch.flip(buf[:N], [3])
    with torch.no_grad():
        both = model(buf)
        a = model(x)
        b = model(torch.flip(x, [3]))
    assert relerr(both[:N].cpu().numpy(), a.cpu().numpy()) <= 1e-3
    assert relerr(both[N:].cpu().numpy(), b.cpu().numpy()) <= 1e-3


def test_flip_mirror_symmetry(dev):
    """Without the shift the merge of [flip(x); x] is flip_back of the merge of [x; flip(x)]: joint j
    of the first decodes to the mirror of joint pi(j) of the second, x' = -x - 1/W."""
    import lib.core.integral_loss as il
    N, J, D, H, W = 8, 16, 64, 64, 64
    x = _logits(dev, 2 * N, J, D, H, W, 55)
    swapped = torch.cat([x[N:], x[:N]]).contiguous(memory_format=torch.channels_last)
    a = il.softmax_integral_flip(x, J, W, H, D, _pairs(J), False).cpu().numpy().reshape(N, J, 3)
    b = il.softmax_integral_flip(swapped, J, W, H, D, _pairs(J), False).cpu().numpy().reshape(N, J, 3)
    perm = il.flip_permutation(_pairs(J), J)
    m = a[:, perm].copy()
    m[:, :, 0] = -m[:, :, 0] - 1.0 / W
    assert np.max(np.abs(b - m)) <= 1e-5
    # in patch pixels at 256 / 64: x_px' = 252 - x_px
    pa = il.joint_location_result_from_coords(256, 256, a.reshape(N, -1))
    pb = il.joint_location_result_from_coords(256, 256, b.reshape(N, -1))
    assert np.max(np.abs(pb[:, :, 0] - (252.0 - pa[:, perm, 0]))) <= 256 * 1e-5


@pytest.mark.parametrize("J", [16, 17])
def test_validate_integral_flip_end_to_end(dev, tmp_path, J):
    import torch.utils.data
    import lib.dataset as dataset
    import lib.models as models
    import lib.core.integral_loss as il
    from lib.core.config import config, reset_config
    from lib.core.function import validate_integral, eval_integral
    reset_config()
    config.MODEL.NUM_JOINTS = J
    config.MODEL.DEPTH_RES = 16
    config.MODEL.IMAGE_SIZE = [64, 64]
    config.MODEL.EXTRA.NUM_LAYERS = 18
    config.MODEL.INIT_WEIGHTS = False
    config.DATASET.DATASET = "synthetic_h36m"
    config.DATASET.SYNTHETIC_LEN = 20
    config.TEST.FLIP_TEST = True
    model = models.pose3d_resnet.get_pose_net(config, is_train=False).cuda()
    ds = dataset.synthetic_h36m(cfg=config, root="", image_set="valid", is_train=False)
    loader = torch.utils.data.DataLoader(ds, batch_size=8, shuffle=False, num_workers=0)
    preds = validate_integral(loader, model)
    assert preds.shape == (len(ds), J, 4) and np.isfinite(preds).all()
    assert np.isfinite(eval_integral(0, preds, loader, str(tmp_path)))
    ref = []
    with torch.no_grad():
        for d in loader:
            x = d[0].to(dev)
            ref.append(il.get_joint_location_result_flip(256, 256, model(torch.cat([x, torch.flip(x, [3])])),
                                                         ds.flip_pairs, config.TEST.SHIFT_HEATMAP))
    assert np.max(np.abs(preds - np.concatenate(ref))) <= 256 * 1e-5
    reset_config()
