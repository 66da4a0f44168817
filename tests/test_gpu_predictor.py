"""GPU (-m gpu): the split-K conv16 entry (epb_conv16_fprop_splitk) and PosePredictor.

- Split-K against torch float64 at every layer shape of the bench (step_cases.C4_LAYERS_SPLIT16) for
  N = 1 and 32, at the planner's split count and at forced counts 2, 3 and K/64, with a bias so
  that a bias applied twice, or statistics that count the rows past the output view of a ragged
  tile, show.  Float64 uses the exact values the fp16 planes hold, so the bars are the fp32
  accumulation noise of test_gpu_split16 (5e-5).
- Bits: S = 1 is epb_conv16_fprop; two runs at S > 1 agree; a deconv phase view is written and
  nothing around it (the NaN-sentinel method of test_gpu_conv16_store).
- PosePredictor: C1 logits against the reference golden; coordinates against the eager path
  (plain, flip test, boxes); graph reuse, a second N, snapshot / refresh(), train() mode.

Bars of the predictor against the eager forward: the two run the same kernels on the same
weights except that the split-K convs sum K in another fp32 order, so the logits differ by
accumulation rounding amplified through the network: bar 1e-4 of the largest |logit| (measured
on the H100: 3.6e-5 to 9.7e-5 at N = 1..32).  The coordinates follow from the logits: the graph's
decode must equal the eager decode of the graph's own logits bit for bit, and against the eager
coordinates each joint may move no more than the soft-argmax can for the measured logit change
of its volume, dl: the weights of its bins change by factors within exp(+-2 dl), so the expected
coordinate (a range of 256 patch px) moves by at most 256 (exp(2 dl) - 1) px.  A fixed pixel bar
does not hold: the C1 volumes of a random-init network are nearly one-hot, and a 1e-4 logit change
flips the winning bin of near-tied joints (measured: identical coordinates at N = 1 and 2, jumps
of 0.5-2 px at N = 3, 5, 32)."""
import numpy as np
import pytest
import torch

from tests import emul_splitk as es
from tests.step_cases import C4_LAYERS_SPLIT16, _bench_conv, _coord_bound, _splitk_layer
from tests.step_cases import _splitk_run as _run

pytestmark = pytest.mark.gpu

LOGIT_BAR = 1e-4


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _layer(dev, layer, N):
    """conv, geoms, split operands, bias and the float64 reference [N, Ho, Wo, Cout] with bias"""
    conv, hw = _bench_conv(layer)
    geoms, opnds, bias, ref, _ = _splitk_layer(dev, conv, hw, N)
    return conv, geoms, opnds, bias, ref


CASES = [(l, N) for l in C4_LAYERS_SPLIT16 for N in (1, 32)]


@pytest.mark.parametrize("case", CASES, ids=["%s-N%d" % (c[0][0], c[1]) for c in CASES])
def test_splitk_vs_torch_float64(dev, case):
    layer, N = case
    conv, geoms, opnds, bias, ref = _layer(dev, layer, N)
    cout = layer[3]
    kb = es.kblocks(geoms[0])
    for splits in (None, 2, 3, kb):
        out = torch.zeros(ref.shape, device=dev)
        stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
        _run(geoms, opnds, bias, out, stats, splits)
        torch.cuda.synchronize()
        e = float((out.double() - ref).abs().max() / ref.abs().max())
        assert e <= 5e-5, "S=%s output %.3e" % (splits, e)
        r = ref.reshape(-1, cout)
        e1 = float((stats[:cout] - r.sum(0)).abs().max() / r.abs().sum(0).max())
        e2 = float((stats[cout:] - (r * r).sum(0)).abs().max() / (r * r).sum(0).max())
        assert e1 <= 5e-5 and e2 <= 5e-5, "S=%s statistics %.3e / %.3e" % (splits, e1, e2)


BITS = [c for c in C4_LAYERS_SPLIT16 if c[0] in ("l4_3x3_512", "deconv0", "l3_1x1_1024_256", "final")]


@pytest.mark.parametrize("layer", BITS, ids=[c[0] for c in BITS])
def test_splitk_bits(dev, layer):
    from epipolarpose_b200 import ops
    conv, geoms, opnds, bias, ref = _layer(dev, layer, 1)
    cout = layer[3]
    runs = {}
    for key in ("fused", 1, 5, 5):
        out = torch.zeros(ref.shape, device=dev)
        stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
        if key == "fused":
            for gm in geoms:
                ops.conv16_fprop(gm, *opnds, out, bias, stats)
        else:
            _run(geoms, opnds, bias, out, stats, key)
        runs.setdefault(key, []).append((out, stats))
    torch.cuda.synchronize()
    (fo, fs), (o1, s1) = runs["fused"][0], runs[1][0]
    assert torch.equal(fo.view(torch.int32), o1.view(torch.int32)), "S = 1 differs from epb_conv16_fprop"
    assert torch.equal(fs.view(torch.int64), s1.view(torch.int64))
    (a, _), (b, _) = runs[5]
    assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "S = 5 is not run-to-run identical"


def test_splitk_writes_exactly_the_phase_view(dev):
    """deconv0 at N = 1 (2 tiles per phase, split 32 ways): every phase call writes its view and
    leaves the rest of the tensor and a guard band past its end at their sentinels."""
    sentinels, guard = (0x7FC0DEAD, 0x7FC0BEEF), 4096
    layer = [c for c in C4_LAYERS_SPLIT16 if c[0] == "deconv0"][0]
    conv, geoms, opnds, bias, ref = _layer(dev, layer, 1)
    shape = tuple(ref.shape)
    n = int(np.prod(shape))
    for gm in geoms:
        bufs = [torch.full((n + guard,), s, dtype=torch.int32, device=dev).view(torch.float32)
                for s in sentinels]
        for b in bufs:
            _run([gm], opnds, bias, b[:n].view(shape), None, None)
        torch.cuda.synchronize()
        a, b = (t.view(torch.int32).cpu() for t in bufs)
        inside = torch.zeros(n + guard, dtype=torch.bool)
        m = torch.zeros(shape, dtype=torch.bool)
        m[:, gm.ph::gm.os, gm.pw::gm.os] = True
        inside[:n] = m.view(-1)
        assert torch.equal(a[inside], b[inside])
        assert bool((a[~inside] == sentinels[0]).all()) and bool((b[~inside] == sentinels[1]).all())
        got = bufs[0][:n].view(shape)[:, gm.ph::gm.os, gm.pw::gm.os].double()
        want = ref[:, gm.ph::gm.os, gm.pw::gm.os]
        assert float((got - want).abs().max() / want.abs().max()) <= 5e-5


# ------------------------------------------------------------------ PosePredictor
@pytest.fixture(scope="module")
def c1(dev):
    from tests import golden_inputs as gi
    from tests.golden_inputs import _model
    c = gi.SIZE_CASES["c1"]
    return c, _model(dev, c, "f16x3", train=False)


def _images(N, seed, HW=256):
    return np.random.default_rng(seed).standard_normal((N, 3, HW, HW)).astype(np.float32)


def _eager(model, x):
    import lib.core.integral_loss as il
    with torch.no_grad():
        out = model.eval()(torch.from_numpy(x).cuda())
        return out, il.get_joint_location_result(x.shape[3], x.shape[2], out)


def _close(pred, model, x):
    """predictor coordinates and logits against the eager forward (see the module docstring)"""
    import lib.core.integral_loss as il
    got = pred(x)
    assert np.array_equal(got, il.get_joint_location_result(x.shape[3], x.shape[2], pred.logits))
    logits, want = _eager(model, x)
    N = x.shape[0]
    e = float((pred.logits - logits).abs().max() / logits.abs().max())
    dl = (pred.logits - logits).abs().reshape(N, 16, -1).amax(-1).cpu().numpy()      # [N, J]
    d = np.abs(got - want)[:, :, :3].max(-1)
    print("N=%d logits %.2e coords %.2e px (largest bound %.2e px)" % (N, e, d.max(), _coord_bound(dl).max()))
    assert e <= LOGIT_BAR, e
    assert np.all(d <= _coord_bound(dl)), (d.max(), _coord_bound(dl).min())
    return got


def test_predictor_c1_vs_reference(golden, c1):
    from tests import golden_inputs as gi
    from tests.golden_inputs import _check_output
    from lib.core.inference import PosePredictor
    c, model = c1
    pred = PosePredictor(model, flip_test=False)
    pred(gi.images(c["N"], c["HW"], c["seed"]))
    _check_output(pred.logits, golden("net_c1"))


@pytest.mark.parametrize("N", [1, 3, 32])
def test_predictor_vs_eager(c1, N):
    from lib.core.inference import PosePredictor
    _, model = c1
    pred = PosePredictor(model, flip_test=False)
    got = _close(pred, model, _images(N, 100 + N))
    assert got.shape == (N, 16, 4) and got.dtype == np.float64 and np.all(got[:, :, 3] == 1)


def test_predictor_flip_vs_validate(c1):
    from lib.core.function import validate_integral
    from lib.core.inference import PosePredictor
    from lib.dataset.synthetic import MPII_FLIP_PAIRS
    _, model = c1
    x = _images(4, 5)

    class _DS:
        flip_pairs = MPII_FLIP_PAIRS

        def __len__(self):
            return 4

    class _Loader(list):
        dataset = _DS()

    import lib.core.integral_loss as il
    want = validate_integral(_Loader([(torch.from_numpy(x),)]), model, flip_test=True, shift_heatmap=True)
    pred = PosePredictor(model, flip_test=True, shift_heatmap=True, flip_pairs=MPII_FLIP_PAIRS)
    got = pred(x)
    assert pred.logits.shape[0] == 8
    assert np.array_equal(got, il.get_joint_location_result_flip(256, 256, pred.logits, MPII_FLIP_PAIRS, True))
    buf = torch.from_numpy(x).cuda()
    with torch.no_grad():
        logits = model.eval()(torch.cat([buf, torch.flip(buf, [3])]))
    assert float((pred.logits - logits).abs().max() / logits.abs().max()) <= LOGIT_BAR
    # a merged volume moves by at most the largest move of the two it averages
    dl = float((pred.logits - logits).abs().max())
    assert float(np.abs(got - want)[:, :, :3].max()) <= _coord_bound(dl)


def test_predictor_boxes(c1):
    from lib.core.inference import PosePredictor
    from lib.utils.img_utils import trans_coords_from_patch_to_org_3d_batch
    _, model = c1
    N = 3
    x = _images(N, 9)
    rng = np.random.default_rng(3)
    meta = {"center_x": rng.uniform(200, 800, N), "center_y": rng.uniform(200, 600, N),
            "width": rng.uniform(150, 400, N), "height": rng.uniform(150, 400, N),
            "scale": rng.uniform(0.8, 1.2, N), "rot": rng.uniform(-30, 30, N)}
    pred = PosePredictor(model, flip_test=False)
    patch = pred(x)
    img = pred(x, boxes=meta)
    want = trans_coords_from_patch_to_org_3d_batch(patch, meta["center_x"], meta["center_y"], meta["width"],
                                                   meta["height"], 256, 256, 2000, meta["scale"], meta["rot"])
    assert float(np.abs(img - want).max()) <= 1e-6 * float(np.abs(want).max())


def test_predictor_graphs_snapshot_and_modes(dev):
    from lib.core.inference import PosePredictor
    from tests import golden_inputs as gi
    from tests.golden_inputs import _model
    model = _model(dev, gi.SIZE_CASES["c1"], "f16x3", train=False)     # its own: the test edits it
    pred = PosePredictor(model, flip_test=False)
    a, b = _images(2, 1), _images(2, 2)
    _close(pred, model, a)
    _close(pred, model, b)                     # the same graph, another batch
    assert len(pred.graphs) == 1
    _close(pred, model, _images(5, 3))
    assert len(pred.graphs) == 2               # a second N, a second graph
    before = pred(a)
    with torch.no_grad():
        sd = model.state_dict()
        sd["final_layer.bias"].add_(0.5 * torch.randn_like(sd["final_layer.bias"]))
        sd["layer4.2.conv2.weight"].mul_(1.5)
        sd["deconv_layers.1.running_var"].mul_(2.0)
    old_logits = pred.logits.clone()
    new_logits, _ = _eager(model, a)
    assert float((new_logits - old_logits).abs().max() / old_logits.abs().max()) > 100 * LOGIT_BAR
    assert np.array_equal(pred(a), before)     # the snapshot: unchanged until refresh()
    assert torch.equal(pred.logits, old_logits)
    pred.refresh()
    _close(pred, model, a)
    model.train()
    got = pred(a)
    assert model.training
    model.eval()
    assert np.array_equal(got, pred(a))        # eval semantics whatever model.training says


def test_predictor_refuses_unsupported_models(dev):
    import lib.models as models
    from lib.core.inference import PosePredictor
    from tools.bench_cfg import make_cfg
    cfg = make_cfg(num_layers=18, num_joints=4, volume=False, depth_res=16, image_size=(64, 64))
    with pytest.raises(ValueError, match="VOLUME"):
        PosePredictor(models.pose3d_resnet.get_pose_net(cfg, False).to(dev))
    cfg = make_cfg(num_layers=18, num_joints=4, volume=True, depth_res=16, image_size=(64, 64))
    with pytest.raises(ValueError, match="precision"):
        PosePredictor(models.pose3d_resnet.get_pose_net(cfg, False, precision="tf32x3").to(dev))
    with pytest.raises(ValueError, match="flip_pairs"):
        PosePredictor(models.pose3d_resnet.get_pose_net(cfg, False).to(dev), flip_test=True)
