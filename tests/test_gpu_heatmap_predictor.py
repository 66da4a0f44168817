"""GPU (-m gpu): joints from the MODEL.VOLUME = false head.

1. epb_heatmap_decode: bit-identical to its CPU build (tests/harness/host_heatmap_decode.cu); x, y and
   maxval bit-identical to epb_argmax2d / epb_final_preds; both layouts give the same output, with
   NaN in the padding channels of the channels-last buffer; N = 1, 3, 32; flip against the numpy
   merge; the image affine against epb_patch_to_image.
2. The flat head's inference forward (Engine16.prepare_inference with depth_fc) against a float64
   torch forward of the same weights with eval BatchNorm on calibrated running statistics: heat-maps
   and depth logits within 1e-3 of the largest |value| (test_gpu_infer_step's end-to-end bar), at
   R50 / J16 / 64² (N = 2) and R50 / J16 / 256² (N = 1 and 32).
3. HeatmapPredictor: the graph's output is the eager decode of the graph's own buffers bit for bit;
   against model.eval()(x) + decode, heat-maps within 3e-4 of the largest |value| (the split-K
   summation order, see HM_BAR), coordinates equal wherever the top-two margin of the map
   exceeds twice the measured heat-map change, depth within the soft-argmax bound
   depth_range (exp(2 dl) - 1); boxes, flip, a second N, refresh(), train() mode, the refusals
   (including a ResNet-18 trunk, which cannot feed depth_fc).
4. validate_integral + eval_integral on the MPII and H36M fixture trees against eager forward ->
   numpy reference decode -> the same evaluate.
5. The entries a HeatmapPredictor capture launches each have a test here or in a named module."""
import numpy as np
import pytest
import torch

from tests import heatmap_cases as hc

pytestmark = pytest.mark.gpu

# predictor vs eager forward, of the largest |value|: the two differ only in the split-K summation
# order.  test_gpu_predictor's 1e-4 was measured on a random-init C1 network; this R50 flat model with
# calibrated running statistics measured 1.13e-4 (N = 1) and 1.20e-4 (N = 4) on the H100, so the bar is
# 3e-4 (still a third of the prepared forward's float64 bar)
HM_BAR = 3e-4
FWD_BAR = 1e-3          # prepared forward vs float64


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def host():
    run = hc.harness()
    if run is None:
        pytest.skip("nvcc not available")
    return run


def _dec(dev, hm, depth, D, box=None, pairs=None, shift=False, layout=0, C=None, post_process=True):
    """epb_heatmap_decode on numpy inputs, the heat-maps laid out as `layout` (NaN padding)."""
    from lib.core.inference import heatmap_decode_device
    B, J, H, W = hm.shape
    if layout == 1:
        buf = torch.full((B, H, W, C), float("nan"), device=dev)
        buf[..., :J] = torch.from_numpy(hm).to(dev).permute(0, 2, 3, 1)
        t = buf.permute(0, 3, 1, 2)[:, :J]
    else:
        t = torch.from_numpy(np.ascontiguousarray(hm)).to(dev)
    b = None if box is None else torch.from_numpy(np.ascontiguousarray(box)).to(dev)
    out = heatmap_decode_device(t, torch.from_numpy(depth).to(dev), D, b, post_process=post_process,
                                flip_pairs=pairs, shift_heatmap=shift)
    return out.cpu().numpy()


# ------------------------------------------------------------------------------- 1. the kernel
@pytest.mark.parametrize("N", [1, 3, 32])
@pytest.mark.parametrize("J,D", [(16, 64), (17, 16)])
def test_decode_bits(dev, host, N, J, D):
    H, W = 64, 32            # non-square; power-of-two patch / map ratios keep the x, y checks exact
    hm, depth = hc.seeded(N, J, H, W, D, 7 * N + J)
    box = hc.boxes(N, N)
    C = (J + 3) // 4 * 4 + 4
    for post_process in (True, False):
        a = _dec(dev, hm, depth, D, post_process=post_process)
        assert np.array_equal(a, host(hm, depth, D, post_process=post_process))
        assert np.array_equal(a, _dec(dev, hm, depth, D, layout=1, C=C, post_process=post_process))
        hc.check_against_ref(a, hm, depth, D, 256.0, 256.0, 2000.0, post_process)
    kb = _dec(dev, hm, depth, D, box=box, layout=1, C=C)
    assert np.array_equal(kb, host(hm, depth, D, box=box))
    # x, y and maxval against epb_argmax2d (no refinement) and epb_final_preds' refined coordinates
    from lib.core.inference import get_max_preds_device, get_final_preds_device
    t = torch.from_numpy(hm).to(dev)
    preds, maxvals, _ = get_max_preds_device(t)
    plain = _dec(dev, hm, depth, D, post_process=False)
    assert np.array_equal(plain[..., 0], preds[..., 0].double().cpu().numpy() * (256.0 / W))
    assert np.array_equal(plain[..., 1], preds[..., 1].double().cpu().numpy() * (256.0 / H))
    assert np.array_equal(plain[..., 3], maxvals[..., 0].double().cpu().numpy())
    # transform_preds with center (W/2, H/2) and scale W/200 maps heat-map px to themselves up to the
    # affine's rounding; the refined coordinates are quarter pixels
    ctr = np.tile([W / 2.0, H / 2.0], (N, 1))
    scl = np.tile([W / 200.0, H / 200.0], (N, 1))
    fp, fm = get_final_preds_device(t, ctr, scl, True)
    fp = fp.double().cpu().numpy()
    assert np.max(np.abs(fp - np.round(fp * 4) / 4)) <= 1e-3
    refined = _dec(dev, hm, depth, D)
    assert np.array_equal(refined[..., 0] / (256.0 / W), np.round(fp[..., 0] * 4) / 4)
    assert np.array_equal(refined[..., 1] / (256.0 / H), np.round(fp[..., 1] * 4) / 4)
    assert np.array_equal(refined[..., 3], fm[..., 0].double().cpu().numpy())


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("J", [16, 17])
def test_decode_flip(dev, host, J, shift):
    N, D, H, W = 5, 64, 64, 64
    pairs = hc.pairs_of(J)
    hm2, d2 = hc.seeded(N, J, H, W, D, 60 + J, B=2 * N)
    mh, md = hc.flip_merge(hm2, d2, pairs, shift)
    want = _dec(dev, mh, md, D)
    C = (J + 3) // 4 * 4
    for layout in (0, 1):
        got = _dec(dev, hm2, d2, D, pairs=pairs, shift=shift, layout=layout, C=C + 4)
        assert np.array_equal(got, want)
    assert np.array_equal(want, host(hm2, d2, D, pairs=pairs, shift=shift))
    hc.check_against_ref(want, mh, md, D, 256.0, 256.0, 2000.0)


def test_decode_affine_is_patch_to_image(dev):
    from epipolarpose_b200 import ops
    N, J, D = 6, 17, 64
    hm, depth = hc.seeded(N, J, 64, 64, D, 3)
    box = hc.boxes(N, 4)
    patch = _dec(dev, hm, depth, D)
    img = _dec(dev, hm, depth, D, box=box)
    c = torch.from_numpy(hc.exact_patch_coords(patch[..., 0], patch[..., 1], 256.0, 256.0)).to(dev)
    kps = torch.empty((N, J, 4), device=dev, dtype=torch.float64)
    ops.patch_to_image(c.reshape(N, J * 3).contiguous(), torch.from_numpy(box).to(dev), N, J, 256.0, 256.0,
                       2000.0, kps)
    assert np.array_equal(img[..., :2], kps[..., :2].cpu().numpy())
    assert np.array_equal(img[..., 2:], patch[..., 2:])


def test_decode_refusals(dev):
    from epipolarpose_b200 import ops
    from epipolarpose_b200._lib import EpbError
    hm = torch.zeros((2, 4, 8, 8), device=dev)
    d = torch.zeros((2, 4 * 16), device=dev)
    k = torch.empty((2, 4, 4), device=dev, dtype=torch.float64)
    with pytest.raises(EpbError):         # J*D larger than the depth row
        ops.heatmap_decode(hm, 0, 4, d, 60, None, 2, 4, 8, 8, 16, 256, 256, 2000, 1, None, 0, k)
    with pytest.raises(EpbError):         # channels-last C < J
        ops.heatmap_decode(hm, 1, 3, d, 64, None, 2, 4, 8, 8, 16, 256, 256, 2000, 1, None, 0, k)
    with pytest.raises(EpbError):         # not an involution
        ops.heatmap_decode(hm, 0, 4, d, 64, None, 1, 4, 8, 8, 16, 256, 256, 2000, 1, [1, 2, 3, 0], 0,
                           k[:1])


# ------------------------------------------------------------------------------- 2. the forward
def _flat_model(dev, J, D, HW, seed):
    """An R50 VOLUME = false model with init_state weights and calibrated running statistics: one
    float64 training forward sets each BatchNorm's running statistics to its batch statistics, then a
    per-channel perturbation makes eval and batch statistics differ (as step_cases.calibrated_state)."""
    import lib.models as models
    from oracle import restate_net as rn
    from tools.bench_cfg import make_cfg
    sd = rn.init_state(rn.param_shapes(num_layers=50, num_joints=J, volume=False, depth_res=D), seed)
    sd64 = {k: v.to(dev, torch.float64) if v.is_floating_point() else v.to(dev) for k, v in sd.items()}
    x = torch.from_numpy(np.random.default_rng(seed + 1).standard_normal((4, 3, HW, HW))).to(dev)
    ns = {}
    with torch.no_grad():
        rn.forward(sd64, x, num_layers=50, volume=False, image_size=(HW, HW), training=True, new_stats=ns)
    rng = np.random.default_rng(seed + 2)
    m = rn.BN_MOMENTUM
    for k in sorted(ns):
        if not k.endswith(".running_mean"):
            continue
        p = k[:-len("running_mean")]
        mean = ((ns[k].cpu() - (1 - m) * sd[k].double()) / m).numpy()
        var = ((ns[p + "running_var"].cpu() - (1 - m) * sd[p + "running_var"].double()) / m).numpy()
        C = mean.size
        sd[p + "running_var"] = torch.from_numpy((var * rng.uniform(0.5, 2.0, C)).astype(np.float32))
        sd[p + "running_mean"] = torch.from_numpy((mean + rng.uniform(-0.5, 0.5, C) * np.sqrt(var)).astype(np.float32))
    model = models.pose3d_resnet.get_pose_net(make_cfg(num_layers=50, num_joints=J, volume=False, depth_res=D,
                                                       image_size=(HW, HW)), False)
    model.load_state_dict(sd)
    return model.to(dev), sd


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize("HW,Ns", [(64, (2,)), (256, (1, 32))])
def test_flat_inference_forward_vs_float64(dev, HW, Ns):
    from epipolarpose_b200 import net16
    from oracle import restate_net as rn
    J, D = 16, 64
    model, sd = _flat_model(dev, J, D, HW, 31)
    eng = net16.Engine16(model._plan)
    params = {k: v.detach() for k, v in model.named_parameters()}
    params.update(dict(model.named_buffers()))
    state = eng.prepare_inference(params, dev)
    sd64 = {k: v.to(dev, torch.float64) if v.is_floating_point() else v.to(dev) for k, v in sd.items()}
    for N in Ns:
        x = torch.from_numpy(np.random.default_rng(N).standard_normal((N, 3, HW, HW)).astype(np.float32)).to(dev)
        with torch.no_grad():
            logits, depth, _ = eng.forward(x, None, training=False, save=False, prepared=state)
            hm64, d64 = rn.forward(sd64, x.double(), num_layers=50, volume=False, image_size=(HW, HW),
                                   training=False)
        hm = logits.permute(0, 3, 1, 2)[:, :J]
        eh, ed = _rel(hm, hm64), _rel(depth.reshape(N, -1)[:, :J * D], d64)
        print("R50 J%d %d² N %d: heat-maps %.2e, depth %.2e of the largest |value| (bar %.0e)"
              % (J, HW, N, eh, ed, FWD_BAR))
        assert eh <= FWD_BAR and ed <= FWD_BAR
    # refresh refills the prepared depth_fc bias in place
    params["depth_fc.bias"].add_(1.0)
    st2 = eng.prepare_inference(params, dev, state)
    assert st2["dbias"] is state["dbias"]
    assert torch.equal(st2["dbias"][:J * D], params["depth_fc.bias"])
    params["depth_fc.bias"].sub_(1.0)


# ------------------------------------------------------------------------------- 3. the predictor
def _eager(model, x):
    model.eval()
    with torch.no_grad():
        return model(x)


def _top2_margin(hm):
    f = hm.reshape(hm.shape[0], hm.shape[1], -1).double()
    t = f.topk(2, dim=2).values
    return (t[..., 0] - t[..., 1]).cpu().numpy()


def _compare_to_eager(pred, model, x, D, flip_pairs=None, shift=False):
    """rows of the predictor against the eager forward + decode (see the module docstring)"""
    from lib.core.inference import get_heatmap_location_result
    x = x.cuda()
    got = pred(x)
    xin = torch.cat([x, torch.flip(x, [3])]) if flip_pairs is not None else x
    hm_e, d_e = _eager(model, xin)
    hm_g, d_g = pred.heatmaps, pred.depth
    assert hm_g.shape == hm_e.shape
    eh = _rel(hm_g, hm_e)
    assert eh <= HM_BAR, eh
    want = get_heatmap_location_result(x.shape[3], x.shape[2], (hm_e, d_e), depth_res=D, depth_range=2000.0,
                                       post_process=True, flip_pairs=flip_pairs, shift_heatmap=shift)
    # the margin test runs on the maps the decode reads (merged with flip test)
    if flip_pairs is not None:
        mh, _ = hc.flip_merge(hm_e.cpu().numpy(), d_e.cpu().numpy(), flip_pairs, shift)
        mh = torch.from_numpy(mh)
    else:
        mh = hm_e
    dh = float((hm_g.double() - hm_e.double()).abs().max())
    safe = _top2_margin(mh) > 2 * dh
    assert safe.mean() > 0.5, safe.mean()
    assert np.array_equal(got[..., :2][safe], want[..., :2][safe])
    dl = float((d_g.double() - d_e.double()).abs().max())
    dz = np.abs(got[..., 2] - want[..., 2]) / 256.0 * 2000.0             # mm
    assert np.all(dz <= 2000.0 * np.expm1(2 * dl) + 1e-6), (dz.max(), dl)
    return got, eh


@pytest.fixture(scope="module")
def flat64(dev):
    return _flat_model(dev, 16, 64, 64, 5)


def test_predictor_graph_equals_eager_decode_of_its_buffers(dev, flat64):
    from lib.core.inference import HeatmapPredictor, heatmap_decode_device, heatmap_rows
    model, _ = flat64
    pred = HeatmapPredictor(model, flip_test=False)
    x = torch.from_numpy(np.random.default_rng(1).standard_normal((3, 3, 64, 64)).astype(np.float32))
    got = pred(x)
    assert pred.heatmaps.shape == (3, 16, 16, 16) and pred.depth.shape == (3, 16 * 64)
    ref = heatmap_decode_device(pred.heatmaps, pred.depth, 64, None, 64, 64, 2000.0, True).cpu().numpy()
    assert np.array_equal(got, heatmap_rows(ref, 64))
    box = {"center_x": np.array([300.0, 500.0, 120.0]), "center_y": np.array([200.0, 410.0, 90.0]),
           "width": np.array([180.0, 250.0, 60.0]), "height": np.array([200.0, 240.0, 64.0]),
           "scale": np.array([1.0, 1.1, 0.9]), "rot": np.array([0.0, 12.0, -20.0])}
    gb = pred(x, boxes=box)
    from lib.utils.img_utils import _boxes
    bt = _boxes(dict(box), 3, dev)
    refb = heatmap_decode_device(pred.heatmaps, pred.depth, 64, bt, 64, 64, 2000.0, True).cpu().numpy()
    assert np.array_equal(gb, refb)
    assert np.array_equal(gb[..., 2:], ref[..., 2:])
    assert np.array_equal(pred(x), got)                  # the box of a boxed call does not stick


def test_predictor_against_eager(dev, flat64):
    from lib.core.inference import HeatmapPredictor
    model, _ = flat64
    pred = HeatmapPredictor(model, flip_test=False)
    for N in (1, 4):
        x = torch.from_numpy(np.random.default_rng(10 + N).standard_normal((N, 3, 64, 64)).astype(np.float32))
        _, eh = _compare_to_eager(pred, model, x, 64)
        print("HeatmapPredictor N %d: heat-maps %.2e of the largest |value| (bar %.0e)" % (N, eh, HM_BAR))
    assert set(pred.graphs) == {(1, 64, 64), (4, 64, 64)}


@pytest.mark.parametrize("shift", [False, True])
def test_predictor_flip(dev, flat64, shift):
    from lib.core.inference import HeatmapPredictor, heatmap_decode_device, heatmap_rows
    model, _ = flat64
    pairs = hc.MPII_PAIRS
    pred = HeatmapPredictor(model, flip_test=True, shift_heatmap=shift, flip_pairs=pairs)
    x = torch.from_numpy(np.random.default_rng(2).standard_normal((3, 3, 64, 64)).astype(np.float32))
    got, _ = _compare_to_eager(pred, model, x, 64, pairs, shift)
    assert pred.heatmaps.shape[0] == 6
    ref = heatmap_decode_device(pred.heatmaps, pred.depth, 64, None, 64, 64, 2000.0, True, pairs, shift)
    assert np.array_equal(got, heatmap_rows(ref.cpu().numpy(), 64))
    mh, md = hc.flip_merge(pred.heatmaps.cpu().numpy(), pred.depth.cpu().numpy(), pairs, shift)
    hc.check_against_ref(ref.cpu().numpy(), mh, md, 64, 64.0, 64.0, 2000.0)


def test_predictor_refresh_and_train_mode(dev):
    from lib.core.inference import HeatmapPredictor
    model, _ = _flat_model(dev, 16, 64, 64, 9)
    pred = HeatmapPredictor(model, flip_test=False)
    x = torch.from_numpy(np.random.default_rng(3).standard_normal((2, 3, 64, 64)).astype(np.float32))
    a = pred(x)
    with torch.no_grad():
        model.depth_fc.bias.add_(torch.linspace(-3, 3, model.depth_fc.bias.numel(), device=dev))
        model.final_layer.bias.add_(torch.linspace(-1, 1, model.final_layer.bias.numel(), device=dev))
    assert np.array_equal(pred(x), a)                    # a snapshot until refresh()
    pred.refresh()
    b, _ = _compare_to_eager(pred, model, x, 64)
    assert not np.array_equal(a, b)
    model.train()
    got = pred(x)
    assert model.training
    assert np.array_equal(got, b)                        # eval semantics whatever model.training says


def test_predictor_refusals(dev):
    import lib.models as models
    from lib.core.inference import HeatmapPredictor
    from tools.bench_cfg import make_cfg
    cfg = make_cfg(num_layers=18, num_joints=4, volume=True, depth_res=16, image_size=(64, 64))
    with pytest.raises(ValueError, match="VOLUME.*PosePredictor"):
        HeatmapPredictor(models.pose3d_resnet.get_pose_net(cfg, False).to(dev))
    cfg = make_cfg(num_layers=50, num_joints=4, volume=False, depth_res=16, image_size=(64, 64))
    with pytest.raises(ValueError, match="precision"):
        HeatmapPredictor(models.pose3d_resnet.get_pose_net(cfg, False, precision="tf32x3").to(dev))
    with pytest.raises(ValueError, match="flip_pairs"):
        HeatmapPredictor(models.pose3d_resnet.get_pose_net(cfg, False).to(dev), flip_test=True)
    cfg = make_cfg(num_layers=18, num_joints=4, volume=False, depth_res=16, image_size=(64, 64))
    with pytest.raises(ValueError, match="2048-channel trunk"):     # depth_fc reads 2048 channels, R18 has 512
        HeatmapPredictor(models.pose3d_resnet.get_pose_net(cfg, False).to(dev))


# ------------------------------------------------------------------------------- 4. validation
@pytest.mark.parametrize("name,J", [("mpii_valid", 16), ("h36m_valid", 17)])
@pytest.mark.parametrize("flip", [False, True])
def test_validate_and_evaluate_flat_model(dev, tmp_path, name, J, flip):
    from tests import dataset_cases as dc
    from lib.core.config import config, reset_config
    from lib.core.function import _flip_pairs, eval_integral, loader_batch, validate_integral
    D = 16
    reset_config()
    config.MODEL.DEPTH_RES = D
    config.MODEL.NUM_JOINTS = J
    model, _ = _flat_model(dev, J, D, 64, 40 + J)
    ds = dc.build(name)
    loader = torch.utils.data.DataLoader(ds, batch_size=3, shuffle=False, num_workers=0)
    try:
        rows = validate_integral(loader, model, flip_test=flip, shift_heatmap=True)
        assert rows.shape == (len(ds), J, 4)
        perf, names = eval_integral(0, rows, loader, str(tmp_path), with_names=True)
        ref = []
        model.eval()
        with torch.no_grad():
            for data in loader:
                x = loader_batch(data)[0].cuda()
                if flip:
                    x = torch.cat([x, torch.flip(x, [3])])
                hm, d = model(x)
                hm, d = hm.cpu().numpy(), d.cpu().numpy()
                if flip:
                    hm, d = hc.flip_merge(hm, d, _flip_pairs(ds), True)
                _, maxvals, dmm, px = hc.decode_ref(hm, d, D, 256.0, 256.0, float(config.DATASET.DEPTH_RANGE))
                ref.append(np.concatenate([px, (dmm / 2000.0 * 256.0)[..., None], maxvals[..., None]], axis=2))
        ref = np.concatenate(ref)
        assert np.array_equal(rows[..., [0, 1, 3]], ref[..., [0, 1, 3]])
        assert np.max(np.abs(rows[..., 2] - ref[..., 2])) <= 1e-9
        perf_r, names_r = eval_integral(0, ref, loader, str(tmp_path), with_names=True)
        assert [n for n, _ in names] == [n for n, _ in names_r]
        for (n, v), (_, vr) in zip(names, names_r):
            assert abs(v - vr) <= 1e-6 * max(1.0, abs(vr)), (n, v, vr)
        print("%s flip %d: %s" % (name, flip, ", ".join("%s %.4f" % nv for nv in names)))
    finally:
        reset_config()


# ------------------------------------------------------------------------------- 5. the gate
# every C-ABI entry a HeatmapPredictor capture launches, and the tests that check it against float64
# or bit for bit
COVERED = {
    "epb_heatmap_decode": ["test_decode_bits", "test_decode_flip", "test_decode_affine_is_patch_to_image"],
    "epb_avgpool_split": ["test_gpu_c2_flat_step.py", "test_flat_inference_forward_vs_float64"],
    "epb_conv_fprop": ["test_gpu_c2_flat_step.py (depth_fc)", "test_flat_inference_forward_vs_float64"],
    "epb_conv16_fprop_splitk": ["test_gpu_infer_step.py", "test_flat_inference_forward_vs_float64"],
    "epb_conv16_splits": ["test_gpu_infer_step.py"],
    "epb_act_scale": ["test_gpu_infer_step.py"],
    "epb_bn_act_split": ["test_gpu_infer_step.py"],
    "epb_bn_relu_maxpool_split": ["test_gpu_infer_step.py"],
    "epb_im2col_split": ["test_gpu_infer_step.py"],
}
PREPARE = {"epb_pack_weight_batch", "epb_split16_batch", "epb_bn_eval_affine"}   # refresh(), not the graph


def test_capture_launches_only_covered_entries(dev, flat64):
    from lib.core.inference import HeatmapPredictor
    from tests.step_cases import _record_calls
    model, _ = flat64
    pred = HeatmapPredictor(model, flip_test=True, flip_pairs=hc.MPII_PAIRS)
    x = torch.zeros((2, 3, 64, 64))
    with _record_calls() as names:
        pred(x)
    torch.cuda.synchronize()
    names = {n for n in names if n.startswith("epb_")} - PREPARE
    missing = sorted(n for n in names if n not in COVERED)
    assert not missing, "entries without a test: %s" % missing
    assert "epb_heatmap_decode" in names and "epb_conv16_fprop_splitk" in names
