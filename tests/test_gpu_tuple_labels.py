"""GPU: online labels of whole camera tuples (epb_tuple_labels) and the robust training step.

  * the entry against the float64 restatement (tests/tuple_label_cases.py) for V in {2, 3, 4, 8},
    J in {16, 17}, T in {1, 32, 4096} (at T = 4096 on 40 of the tuples, the first and last among
    them), with planted outliers, with and without the soft-argmax confidences: X within 1e-4 mm,
    labels within 1e-6, status, inliers and weights equal;
  * a tuple whose root failed has all-zero weights; run to run, and split into sub-batches of
    tuples, every output is bit-identical;
  * V = 2 without failures or confidences is the two-ray DLT of epb_triangulate method 0;
  * the robust online loss captured in a CUDA graph and replayed on three batches: loss, labels and
    logit gradient bit-identical to eager; the graphed robust training step against eager steps;
  * the script flow on the fixture tree with DATASET.TRI_VIEWS: 4 and the robust method."""
import math

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from tests import dataset_cases as dc
from tests import tuple_label_cases as tc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _meta_dev(meta, dev):
    return {k: torch.as_tensor(np.asarray(v, dtype=np.float64)).to(dev) for k, v in meta.items()}


def _run(dev, coords, lse, meta, V, thr=15.0):
    import lib.utils.img_utils as iu
    c = torch.from_numpy(coords).to(dev)
    ls = None if lse is None else torch.from_numpy(lse).to(dev)
    out = iu.tuple_labels_device(c, ls, _meta_dev(meta, dev), V, thr, full=True)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def _check(got, want, rows, tuples):
    label, weight, X, st, inl, res = got
    lo, wo, Xo, so, io, ro = want
    assert np.isfinite(label).all() and np.isfinite(X).all() and np.isfinite(res).all()
    assert np.array_equal(st[tuples], so[tuples]) and np.array_equal(inl[tuples], io[tuples])
    assert np.array_equal(weight[rows], wo[rows])
    assert np.max(np.abs(X[tuples] - Xo[tuples])) <= 1e-4, np.max(np.abs(X[tuples] - Xo[tuples]))
    assert np.max(np.abs(res[tuples] - ro[tuples])) <= 1e-6
    assert np.max(np.abs(label[rows] - lo[rows])) <= 1e-6, np.max(np.abs(label[rows] - lo[rows]))


@pytest.mark.parametrize("T", [1, 32, 4096])
@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("V", [2, 3, 4, 8])
def test_kernel_vs_restatement(dev, V, J, T):
    coords, lse, meta, _, _ = tc.case(1000 * V + 10 * J + T % 997, T, V, J, outliers=0.25, lse=True)
    tuples = np.arange(T) if T <= 32 else np.unique(np.r_[0, T - 1, np.random.default_rng(T).integers(0, T, 38)])
    rows = np.array([v * T + t for v in range(V) for t in tuples])
    for ls in (lse, None):
        got = _run(dev, coords, ls, meta, V)
        want = tc.tuple_labels(coords, ls, meta, V, tuples=tuples)
        _check(got, want, rows, tuples)
        if T <= 32 and V > 2:                             # V = 2: a planted outlier fails its joint
            assert got[3].sum() >= 0.9 * T * J


def test_failed_root_zero_weights_and_bit_identical_splits(dev):
    V, J, T = 4, 17, 64
    coords, lse, meta, _, _ = tc.case(9, T, V, J, outliers=0.25, lse=True)
    c = coords.reshape(V * T, J, 3)
    c[[v * T + 5 for v in range(V - 1)], 0, :2] = np.nan
    coords = c.reshape(V * T, J * 3)
    a = _run(dev, coords, lse, meta, V)
    assert a[3][5, 0] == 0
    rows5 = [v * T + 5 for v in range(V)]
    assert not a[1][rows5].any() and not a[0][rows5].any()
    _check(a, tc.tuple_labels(coords, lse, meta, V, tuples=[5, 6]), np.array(rows5 + [v * T + 6 for v in range(V)]),
           np.array([5, 6]))
    b = _run(dev, coords, lse, meta, V)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    for part in (np.arange(0, 24), np.arange(24, T)):
        rows = np.array([v * T + t for v in range(V) for t in part])
        sub = {k: np.asarray(v)[rows] for k, v in meta.items()}
        s = _run(dev, coords[rows], lse[rows], sub, V)
        assert np.array_equal(s[0], a[0][rows]) and np.array_equal(s[1], a[1][rows])
        for k in range(2, 6):
            assert np.array_equal(s[k], a[k][part])


def test_v2_is_the_two_ray_dlt(dev):
    """Two views, no failures, weights 1, a threshold nothing exceeds: X is epb_triangulate's
    method 0 (both the homogeneous two-ray DLT) to 1e-6 mm."""
    import lib.utils.img_utils as iu
    from lib.utils import triangulation as tri
    V, J, T = 2, 17, 256
    coords, _, meta, _, _ = tc.case(21, T, V, J)
    label, weight, X, st, inl, _ = _run(dev, coords, None, meta, V, thr=1e12)
    assert st.all() and (inl == 3).all() and weight.all()
    md = _meta_dev(meta, dev)
    kps = iu.patch_to_image_device(torch.from_numpy(coords).to(dev), md)
    P = iu.pack_meta(md, V * T, dev)["P"]
    Xp, sp = tri.triangulate_pairs(kps[:T], kps[T:], P[:T], P[T:], method="linear_eigen", stride_u=4)
    assert sp.all()
    err = np.max(np.abs(Xp.cpu().numpy() - X))
    print("V = 2: max |X - epb_triangulate(method 0)| = %.3e mm" % err)
    assert err <= 1e-6
    ref, _ = iu.labels_from_global_coords_device(torch.cat([Xp, Xp]), md)
    assert np.max(np.abs(ref.cpu().numpy() - label)) <= 1e-6


def test_captured_robust_loss_matches_eager(dev):
    """online_epipolar_loss(method='robust', V = 4) and its backward captured in a CUDA graph on one
    resident batch of logits, replayed with three others: loss, labels, weights and logit gradient
    bit-identical to eager."""
    import lib.core.function as fn
    import lib.core.integral_loss as il
    import lib.utils.img_utils as iu
    J, D, T, V = 16, 16, 4, 4
    B = V * T
    crit = il.SmoothL1JointLocationLoss(J)
    _, _, meta, _, _ = tc.case(31, T, V, J)
    g = iu.pack_meta(_meta_dev(meta, dev), B, dev)
    gen = torch.Generator(device=dev).manual_seed(5)
    xs = [torch.randn(B, J * D, D, D, device=dev, generator=gen) * 4 for _ in range(4)]

    def run(x):
        x.grad = None
        loss = fn.online_epipolar_loss(crit, x, {"_packed": g}, "robust", views=V, threshold_px=15.0)
        coords, lse = il.softmax_integral_tensor_lse(x.detach(), J, D, D, D)
        lab, w = iu.tuple_labels_device(coords, lse, {"_packed": g}, V, 15.0)
        loss.backward()
        return loss, lab, w

    eager = []
    for x in xs[1:]:
        xe = x.clone().requires_grad_(True)
        loss, lab, w = run(xe)
        eager.append((loss.item(), lab.cpu().numpy(), w.cpu().numpy(), xe.grad.cpu().numpy()))
    sx = xs[0].clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(sx)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    sx.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        sloss, slab, sw = run(sx)
    for x, ref in zip(xs[1:], eager):
        with torch.no_grad():
            sx.copy_(x)
        graph.replay()
        torch.cuda.synchronize()
        assert math.isfinite(ref[0]) and sloss.item() == ref[0]
        assert np.array_equal(slab.cpu().numpy(), ref[1]) and np.array_equal(sw.cpu().numpy(), ref[2])
        assert np.array_equal(sx.grad.cpu().numpy(), ref[3])


def test_graphed_robust_step_matches_eager(dev):
    """Three steps on a resident synthetic batch (R18, J = 16, D = 16, 4 tuples x 4 views of 64 x
    64): GraphedTrainStep (eager warm-up, capture, replays) against eager_step on a second copy of
    the model, and two graph runs against each other."""
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    J, D, HW = 16, 16, 64
    x, _, _, meta = tc.synthetic_batch(J, HW, 4)
    x = x.to(dev)
    out = {}
    for mode in ("eager", "graph", "graph2"):
        m, opt = tc.r18(dev, J, D, HW)
        step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J).to(dev), opt, online=True, method="robust",
                                   views=4)
        losses = []
        for _ in range(3):
            if mode == "eager":
                losses.append(float(step.eager_step(x, None, None, iu.pack_meta(meta, x.shape[0], dev))))
            else:
                losses.append(float(step(x, meta=meta)))
        if mode != "eager":
            assert step.graph is not None and step.key[2:5] == ("robust", 4, 15.0)
        out[mode] = losses
    print("losses: %s" % out)
    assert all(math.isfinite(v) for l in out.values() for v in l)
    assert out["graph"] == out["graph2"]
    for a, b in zip(out["graph"], out["eager"]):
        assert abs(a - b) <= 2e-2 * abs(b) + 1e-6


def test_script_flow_h36m_tri_views_robust(dev, tmp_path, monkeypatch):
    """train-ss with DATASET.TRI, DATASET.TRI_VIEWS: 4, TRAIN.ONLINE_TRIANGULATION and
    TRAIN.TRIANGULATION_METHOD: robust, loader workers, the graphed step: the first batch is 4B rows
    of four distinct images per tuple, the labels the step used are tuple_labels_device of the
    network's output on that batch, and the losses are finite."""
    import lib.core.integral_loss as loss_m
    import lib.core.function as fn
    import lib.dataset as dataset_m
    import lib.models as models
    import lib.utils.img_utils as iu
    from lib.core.config import config, reset_config
    from lib.utils.utils import get_optimizer
    seen = {}
    orig_batch, orig_labels = fn.loader_batch, iu.tuple_labels_device

    def rec_batch(data):
        out = orig_batch(data)
        seen.setdefault("batch", (out[0].clone(), out[3]))
        return out

    def rec_labels(*a, **k):
        out = orig_labels(*a, **k)
        seen.setdefault("labels", (out[0].clone(), out[1].clone()))
        return out
    monkeypatch.setattr(fn, "loader_batch", rec_batch)
    monkeypatch.setattr(iu, "tuple_labels_device", rec_labels)
    reset_config()
    try:
        config.WORKERS = 2
        config.MODEL.NUM_JOINTS, config.MODEL.DEPTH_RES, config.MODEL.IMAGE_SIZE = 17, 16, np.array([64, 64])
        config.MODEL.EXTRA.NUM_LAYERS, config.MODEL.INIT_WEIGHTS = 18, False
        config.LOSS.FN = "SmoothL1JointLocationLoss"
        config.DATASET.DATASET, config.DATASET.ROOT, config.DATASET.TRAIN_SET = "h36m", dc.H36M_ROOT, "train-ss"
        config.DATASET.TRI, config.DATASET.TRI_VIEWS = True, 4
        config.TRAIN.ONLINE_TRIANGULATION, config.TRAIN.TRIANGULATION_METHOD = True, "robust"
        config.TRAIN.BATCH_SIZE, config.PRINT_FREQ = 1, 1
        model = models.pose3d_resnet.get_pose_net(config, is_train=True)
        model = torch.nn.DataParallel(model, device_ids=[0]).cuda()
        before = {k: v.detach().clone() for k, v in model.module.state_dict().items()}
        crit = loss_m.SmoothL1JointLocationLoss(num_joints=17, norm=False).cuda()
        opt = get_optimizer(config, model)
        ds = dataset_m.h36m(cfg=config, root=config.DATASET.ROOT, image_set="train-ss", is_train=True)
        loader = DataLoader(ds, batch_size=1, shuffle=True, num_workers=config.WORKERS, pin_memory=True)
        for epoch in range(2):
            assert np.isfinite(fn.train_integral(config, loader, model, crit, opt, epoch))
        stepper = model._epb_graphed_step
        assert stepper.graph is not None and stepper.views == 4 and stepper.method == "robust"
        x, meta = seen["batch"]
        assert x.shape[0] == 4 and len(meta["image"]) == 4
        frames = {p.rsplit("_c", 1)[0] for p in meta["image"]}
        assert len(frames) == 1 and len(set(meta["image"])) == 4
        net = models.pose3d_resnet.get_pose_net(config, is_train=True)
        net.load_state_dict(before)
        net = net.to(dev).train()
        with torch.no_grad():
            coords, lse = loss_m.softmax_integral_tensor_lse(net(x.to(dev)), 17, 16, 16, 16)
            label, weight = orig_labels(coords, lse, meta, 4, 15.0)
        used_label, used_weight = seen["labels"]
        assert torch.isfinite(used_label).all()
        assert torch.equal(weight, used_weight)
        assert torch.max(torch.abs(label - used_label)).item() <= 1e-5
    finally:
        reset_config()
