"""CPU: flip test (TEST.FLIP_TEST / TEST.SHIFT_HEATMAP).  The mirror's flip / flip_back and the float64
oracle of the merge (tests/flip_cases.py) against the unmodified reference (tests/golden/flip_test.npz); validate_integral's
flip path through a CPU emulation of epb_softargmax_flip_fwd, written from its contract in
include/epb.h, against the oracle applied to the same 2N logits."""
import types

import numpy as np
import pytest
import torch

from oracle import refshim, restate, restate_net
from tests import emul_ops, flip_cases as fc


class _EmulFlip(types.SimpleNamespace):
    """emul_ops plus epb_softargmax_flip_fwd."""

    def __getattr__(self, name):
        return getattr(emul_ops, name)

    @staticmethod
    def softargmax_flip_fwd(logits2N, N, J, D, H, W, perm, shift, coords):
        from epipolarpose_b200._lib import EpbError
        perm = [int(v) for v in perm]
        if len(perm) != J or any(not 0 <= q < J for q in perm) or any(perm[q] != j for j, q in enumerate(perm)):
            raise EpbError("perm is not an involution of [0, J)")
        if D % 4 or J * D // 4 > 1024 or shift not in (0, 1):
            raise EpbError("unsupported shape")
        v = logits2N.reshape(2 * N, H, W, J, D).permute(0, 3, 4, 1, 2).double()   # [2N, J, D, H, W]
        w = torch.arange(W)
        src = torch.where(w == 0, W - 1, W - w) if shift else W - 1 - w
        merged = 0.5 * (v[:N] + v[N:][:, perm][..., src])
        c = torch.empty(N * J * 3)
        emul_ops.softargmax_fwd(merged.reshape(N, J * D, H, W), 0, N, J, D, H, W, c, torch.empty(N * J * 2,
                                                                                                   dtype=torch.float64))
        coords.view(-1).copy_(c)


EMUL = _EmulFlip()


@pytest.fixture
def emulated():
    import lib.core.integral_loss as il
    prev = il._backend[0]
    il._backend[0] = EMUL
    try:
        yield il
    finally:
        il._backend[0] = prev


def test_flip_and_flip_back_match_reference(golden):
    from lib.utils.img_utils import flip
    from lib.utils.transforms import flip_back
    g = golden("flip_test")
    img = torch.from_numpy(fc.index_images())
    assert np.array_equal(flip(img, 3).numpy(), g["flip_images"])
    assert np.array_equal(flip(img, [3]).numpy(), g["flip_images"])
    for tag in fc.CASES:
        pairs = fc.CASES[tag][-1]
        assert np.array_equal(flip_back(fc.index_volume(tag), pairs), g["flip_back_" + tag])


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("tag", list(fc.CASES))
def test_oracle_flip_merge_matches_reference(golden, tag, shift):
    N, J, D, H, W, seed, scale, pairs = fc.CASES[tag]
    c = fc.flip_merge_softargmax(fc.logits2N(tag), J, W, H, D, pairs, bool(shift))
    assert np.max(np.abs(c - golden("flip_test")["coords_%s_shift%d" % (tag, shift)])) <= 2e-6


@pytest.mark.parametrize("shift", [0, 1])
@pytest.mark.parametrize("memory", ["channels_last", "nchw"])
def test_flip_decode_surface_emulated(emulated, memory, shift):
    """softmax_integral_flip: channels_last logits take the fused entry point, NCHW logits the
    torch-op composition; both equal the oracle."""
    il = emulated
    N, J, D, H, W, seed, scale, pairs = fc.CASES["j17"]
    L2 = fc.logits2N("j17")
    x = torch.from_numpy(L2)
    if memory == "channels_last":
        x = x.permute(0, 2, 3, 1).contiguous().permute(0, 3, 1, 2)
    c = il.softmax_integral_flip(x, J, W, H, D, pairs, shift).numpy()
    ref = fc.flip_merge_softargmax(L2, J, W, H, D, pairs, bool(shift))
    assert np.max(np.abs(c - ref)) <= 2e-6


def test_flip_permutation_errors():
    import lib.core.integral_loss as il
    assert il.flip_permutation(fc.H36M_PAIRS, 17)[14] == 11
    assert il.flip_permutation([], 4) == [0, 1, 2, 3]
    with pytest.raises(ValueError):
        il.flip_permutation([[0, 17]], 17)
    with pytest.raises(ValueError):
        il.flip_permutation([[-1, 2]], 17)
    with pytest.raises(ValueError):
        il.flip_permutation([[0, 1], [1, 2]], 17)            # joint 1 in two pairs


def _setup(J, volume=True, n=12):
    import lib.dataset as dataset
    import lib.models as models
    from lib.core.config import config, reset_config
    reset_config()
    config.MODEL.NUM_JOINTS = J
    config.MODEL.DEPTH_RES = 8
    config.MODEL.IMAGE_SIZE = [32, 32]
    config.MODEL.VOLUME = volume
    config.MODEL.EXTRA.NUM_LAYERS = 18
    config.DATASET.SYNTHETIC_LEN = n
    cfg = refshim.make_cfg(num_layers=18, num_joints=J, volume=volume, depth_res=8, image_size=(32, 32))
    model = models.pose3d_resnet.get_pose_net(cfg, False, ops=emul_ops)
    model.load_state_dict(restate_net.init_state(restate_net.param_shapes(18, J, volume, 8), 5))
    ds = dataset.synthetic_h36m(cfg=config, root="", image_set="valid", is_train=False)
    loader = torch.utils.data.DataLoader(ds, batch_size=5, shuffle=False, num_workers=0)
    return config, model, ds, loader


@pytest.mark.parametrize("J,shift", [(16, True), (17, False)])
def test_validate_integral_flip_emulated(emulated, J, shift):
    """J=16 / 17 synthetic_h36m, 12 samples in batches of 5 (ragged last batch): the result equals
    the oracle merge of the same 2N logits."""
    from lib.core.config import reset_config
    from lib.core.function import validate_integral
    config, model, ds, loader = _setup(J)
    assert ds.flip_pairs == (fc.MPII_PAIRS if J == 16 else fc.H36M_PAIRS)
    out = validate_integral(loader, model, flip_test=True, shift_heatmap=shift)
    assert out.shape == (len(ds), J, 4)
    refs = []
    with torch.no_grad():
        for data in loader:
            x = data[0]
            logits = model(torch.cat([x, torch.flip(x, [3])])).numpy()
            refs.append(restate.joint_location_result(
                256, 256, fc.flip_merge_softargmax(logits, J, 8, 8, 8, ds.flip_pairs, shift)))
    ref = np.concatenate(refs)
    assert np.max(np.abs(out - ref)) <= 256 * 2e-6
    # the keywords default to the module-global config
    config.TEST.FLIP_TEST, config.TEST.SHIFT_HEATMAP = True, shift
    assert np.array_equal(validate_integral(loader, model), out)
    reset_config()


def test_validate_integral_flip_off_is_the_plain_path(emulated, monkeypatch):
    from lib.core.config import reset_config
    from lib.core.function import validate_integral
    import lib.core.integral_loss as il
    monkeypatch.setattr(torch.Tensor, "cuda", lambda self, *a, **k: self)   # the plain path moves batches with .cuda()
    config, model, ds, loader = _setup(16)
    out = validate_integral(loader, model, flip_test=False)
    with torch.no_grad():
        ref = np.concatenate([il.get_joint_location_result(256, 256, model(d[0])) for d in loader])
    assert np.array_equal(out, ref)
    assert np.array_equal(validate_integral(loader, model), out)         # config.TEST.FLIP_TEST: false
    reset_config()


def test_validate_integral_flip_errors(emulated):
    from lib.core.config import reset_config
    from lib.core.function import validate_integral
    config, model, ds, loader = _setup(16, n=4)

    class NoPairs(torch.utils.data.Dataset):
        db = [{"image": "x"}]

        def __len__(self):
            return len(ds)

        def __getitem__(self, i):
            return ds[i]
    with pytest.raises(ValueError, match="pairs"):
        validate_integral(torch.utils.data.DataLoader(NoPairs(), batch_size=4), model, flip_test=True)

    class DbPairs(NoPairs):
        db = [{"flip_pairs": fc.MPII_PAIRS}]
    out = validate_integral(torch.utils.data.DataLoader(DbPairs(), batch_size=4), model, flip_test=True)
    assert np.array_equal(out, validate_integral(loader, model, flip_test=True))
    config, flat, ds, loader = _setup(16, volume=False, n=4)
    with pytest.raises(ValueError, match="VOLUME"):
        validate_integral(loader, flat, flip_test=True)
    reset_config()
