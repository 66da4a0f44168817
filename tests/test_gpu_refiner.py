"""GPU: the eval-mode refiner kernel (epb_refiner_forward through refiner.model.Refiner) against the
float64 oracle (oracle/restate_refiner.py) and the training engine, its batch invariance, graph
capture, and the camera-frame pose kernels epb_pose_errors / epb_pose_to_camera against the
restatement (tests/refiner_cases.py), the reference's goldens and epb_h36m_eval."""
import os
import shutil

import numpy as np
import pytest
import torch

from tests import refiner_cases as rc

pytestmark = pytest.mark.gpu

L, K_ACC, LAYERS = 1024, 1024, 12
EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def net(dev):
    """A LinearModelPG(1024, 45 -> 45) with seeded weights and non-trivial running statistics."""
    from oracle import restate_refiner as rr
    from refiner import model as rmodel
    sd = rr.init_state(rr.param_shapes(L, 45, 45), 23)
    m = rmodel.LinearModelPG(linear_size=L, p_dropout=0.5, input_size=45, output_size=45)
    m.load_state_dict(sd)
    return m.to(dev), sd


def _inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn((N, 45), generator=g)


def _oracle(sd, x, dev):
    from oracle import restate_refiner as rr
    sd64 = {k: (v.to(dev, torch.float64) if v.is_floating_point() else v) for k, v in sd.items()}
    with torch.no_grad():
        return rr.forward(sd64, x.to(dev, torch.float64), training=False)[1]


@pytest.mark.parametrize("N", [1, 3, 64, 1000, 65537])
def test_forward_vs_float64_oracle(net, dev, N):
    """Bar: each layer is an fp32 FMA chain over K <= 1024 terms (relative error <= K eps32 of the
    sum of |terms|), compounded over 12 layers: 12 * 1024 * eps32 of max |p2|.  Ratio asserted < 1."""
    from refiner.model import Refiner
    m, sd = net
    r = Refiner(m, None)
    x = _inputs(N, N)
    y = r.forward(x.to(dev), normalize=False, denormalize=False)
    ref = _oracle(sd, x, dev)
    err = (y.double() - ref).abs().max().item()
    bar = LAYERS * K_ACC * EPS32 * ref.abs().max().item()
    print("N=%d max err %.3e bar %.3e ratio %.3g" % (N, err, bar, err / bar))
    assert err / bar < 1


def test_batch_invariance(net, dev):
    """Every row's bits are the same whatever N, the row's position and the form (GEMV / tiled)."""
    from refiner.model import Refiner
    r = Refiner(net[0], None)
    x = _inputs(1000, 5).to(dev)
    full = r.forward(x, normalize=False, denormalize=False)                    # tiled
    gemv = r.forward(x, normalize=False, denormalize=False, force_form=1)
    tiled = r.forward(x, normalize=False, denormalize=False, force_form=2)
    assert torch.equal(full, gemv) and torch.equal(full, tiled)
    perm = torch.randperm(1000, generator=torch.Generator().manual_seed(1)).to(dev)
    assert torch.equal(r.forward(x[perm], normalize=False, denormalize=False), full[perm])
    for i in (0, 1, 63, 64, 500, 999):
        assert torch.equal(r.forward(x[i:i + 1], normalize=False, denormalize=False)[0], full[i])
        assert torch.equal(r.forward(x[i:i + 3], normalize=False, denormalize=False)[0], full[i])
    big = torch.cat([x] * 66)                                                   # 66000 rows
    assert torch.equal(r.forward(big, normalize=False, denormalize=False)[-1000:], full)


def test_repeatable_and_graph_replay(net, dev):
    from refiner.model import Refiner
    r = Refiner(net[0], ([0.5] * 45, [2.0] * 45, [10.0] * 45, [3.0] * 45))
    xs = torch.zeros((32, 45), device=dev)
    out = torch.empty((32, 45), device=dev)
    xs.copy_(_inputs(32, 1).to(dev))
    a, b = r.forward(xs).clone(), r.forward(xs).clone()
    assert torch.equal(a, b)
    r.forward(xs, out=out)                           # sizes the workspace before capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        r.forward(xs, out=out)
    for seed in (2, 3):
        xs.copy_(_inputs(32, seed).to(dev))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, r.forward(xs.clone()))


def test_normalisation_and_refine(net, dev):
    """forward(normalize, denormalize) is the reference's float32 (x - mean) / std and p * std + mean
    around the network; refine() drops the hip and puts it back at 0."""
    from refiner.model import Refiner
    rng = np.random.default_rng(8)
    norm = tuple(rng.uniform(lo, hi, 45).astype(np.float32) for lo, hi in ((-50, 50), (20, 90), (-50, 50), (20, 90)))
    r = Refiner(net[0], norm)
    x = _inputs(50, 9).numpy() * 60
    xn = (x - norm[0]) / norm[1]
    plain = r.forward(torch.from_numpy(xn).to(dev), normalize=False, denormalize=False).cpu().numpy()
    y = r.forward(torch.from_numpy(x).to(dev)).cpu().numpy()
    assert np.array_equal(y, plain * norm[3] + norm[2])
    poses = np.insert(x.reshape(50, 15, 3), 6, 0.0, axis=1)
    out = r.refine(poses)
    assert out.shape == (50, 16, 3) and np.all(out[:, 6] == 0)
    assert np.array_equal(np.delete(out, 6, axis=1).reshape(50, 45), y)
    assert torch.equal(r.refine(torch.from_numpy(poses).to(dev)).cpu(), torch.from_numpy(out))


def test_snapshot_and_refresh(net, dev):
    from refiner.model import Refiner
    m, sd = net
    r = Refiner(m, None)
    x = _inputs(8, 4).to(dev)
    before = r.forward(x, normalize=False, denormalize=False).clone()
    with torch.no_grad():
        m.w4.bias.add_(1.0)
    try:
        assert torch.equal(r.forward(x, normalize=False, denormalize=False), before)
        after = r.refresh().forward(x, normalize=False, denormalize=False)
        assert torch.allclose(after, before + 1.0, atol=1e-4)
    finally:
        with torch.no_grad():
            m.w4.bias.sub_(1.0)


def test_agrees_with_the_training_engine_in_eval_mode(net, dev):
    from refiner.model import Refiner
    m, _ = net
    x = _inputs(256, 11).to(dev)
    m.eval()
    with torch.no_grad():
        p2 = m(x)[1]
    y = Refiner(m, None).forward(x, normalize=False, denormalize=False)
    rel = ((y - p2).abs().max() / p2.abs().max()).item()
    print("vs LinearModelPG.eval(): rel %.3e" % rel)
    assert rel <= 1e-3


def test_refuses_bad_shapes(net, dev):
    from epipolarpose_b200._lib import EpbError
    from refiner.model import Refiner
    r = Refiner(net[0], None)
    with pytest.raises(ValueError):
        r.forward(torch.zeros((4, 48), device=dev))
    with pytest.raises(ValueError):
        r.refine(np.zeros((4, 17, 3)))
    with pytest.raises(ValueError):
        Refiner(net[0], (np.zeros(45), np.ones(44), np.zeros(45), np.ones(45)))
    with pytest.raises(EpbError):
        r.ops.refiner_forward(45, 1022, 45, r.params, torch.zeros((1, 45), device=dev), 1, 0, 0,
                              torch.zeros((1, 45), device=dev), torch.zeros(1 << 16, device=dev))


def test_pose_errors_vs_restatement_and_goldens(dev, golden, tmp_path):
    from refiner import data
    rng = np.random.default_rng(12)
    gt = rc.poses(rng, 4099, 15)
    pred = gt + rng.normal(0, 30, gt.shape)
    m, pj = data.pose_errors(pred, gt)
    rm, rpj = rc.pose_errors(pred, gt)
    assert np.max(np.abs(m - rm)) <= 1e-9 and np.max(np.abs(pj - rpj)) <= 1e-9
    g = golden("refiner_data")
    for name in ("train.pkl", "valid.pkl"):
        shutil.copy(os.path.join(rc.FIXTURE, name), tmp_path / name)
    np.random.seed(int(g["seed"]))
    data.Human36M(is_train=True, root=str(tmp_path))
    va = data.Human36M(is_train=False, root=str(tmp_path))
    ret = va.evaluate(g["eval_preds"])
    bar = 64 * EPS32 * g["eval_return"]           # the reference evaluates in float32
    got = np.array([va.last_results[k] for k in data.RESULT_NAMES])
    ratio = max(np.max(np.abs(got - g["eval_results"])),
                np.max(np.abs(np.array(va.last_per_joint) - g["eval_per_joint"]))) / bar
    print("evaluate vs the reference's float32 goldens: worst ratio to the bar %.3g" % ratio)
    assert ratio < 1 and abs(ret - g["eval_return"]) < bar
    preds = g["eval_preds"] * va.labels_std + va.labels_mean
    rm, _ = rc.pose_errors(preds.reshape(-1, 15, 3), va.labels.reshape(-1, 15, 3))
    assert abs(ret - rm[:, 0].mean()) <= 1e-9


def test_pose_to_camera_is_the_h36m_eval_pred_column(dev):
    from epipolarpose_b200 import ops
    rng = np.random.default_rng(13)
    S, J, root = 777, 16, 6
    pred = np.stack([rng.uniform(200, 800, (S, J)), rng.uniform(100, 900, (S, J)), rng.normal(0, 200, (S, J))], 2)
    gt = pred + rng.normal(0, 5, pred.shape)
    cam = np.stack([rng.uniform(1100, 1200, S), rng.uniform(1100, 1200, S), rng.uniform(500, 520, S),
                    rng.uniform(500, 520, S), rng.uniform(3000, 6000, S)], 1)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)
    P, G, C = t(pred), t(gt), t(cam)
    metrics = torch.empty((S, 9), dtype=torch.float64, device=dev)
    poses = torch.empty((S, J, 9), dtype=torch.float64, device=dev)
    ops.h36m_eval(P, G, C, S, J, root, 0, 150.0, metrics, None, None, poses)
    out = torch.empty((S, J, 3), dtype=torch.float64, device=dev)
    ops.pose_to_camera(P, C, S, J, root, out)
    assert torch.equal(out, poses[:, :, 0:3])
    assert np.max(np.abs(out.cpu().numpy() - rc.pose_to_camera(pred, cam, root))) <= 1e-9


def test_refiner_main_test_mode_on_the_fixture(net, dev, tmp_path):
    """refiner/main.py --mode test --load <checkpoint> on the fixture files: the reference's
    Human36M and evaluate, the network through LinearModelPG.forward."""
    from refiner import data, main as rmain
    from refiner.model import Refiner
    import lib.utils.utils as U
    m, _ = net
    for name in ("train.pkl", "valid.pkl"):
        shutil.copy(os.path.join(rc.FIXTURE, name), tmp_path / name)
    ckpt = str(tmp_path / "ckpt.pth.tar")
    opt = U.FusedAdam(list(m.parameters()), lr=1e-3)
    torch.save({"epoch": 1, "lr": 1e-3, "step": 0, "err": 100.0, "state_dict": m.state_dict(),
                "optimizer": opt.state_dict()}, ckpt)
    np.random.seed(0)
    err = rmain.main(["--mode", "test", "--load", ckpt], log_root=str(tmp_path / "exp"), data_root=str(tmp_path))
    va = data.Human36M(is_train=False, root=str(tmp_path))
    y = Refiner(m, None).forward(torch.from_numpy(va.data).to(dev), normalize=False, denormalize=False)
    mine = va.evaluate(y.cpu().numpy())
    assert np.isfinite(err) and abs(err - mine) <= 1e-3 * abs(mine)


@pytest.mark.parametrize("N", [1, 3, 200])
def test_small_width_tails_vs_float64_oracle(dev, N):
    """linear_size 100 (not a multiple of 32 or 64): partial column tiles in both forms."""
    from oracle import restate_refiner as rr
    from refiner import model as rmodel
    from refiner.model import Refiner
    sd = rr.init_state(rr.param_shapes(100, 45, 45), 31)
    m = rmodel.LinearModelPG(linear_size=100, input_size=45, output_size=45)
    m.load_state_dict(sd)
    r = Refiner(m.to(dev), None)
    x = _inputs(N, 40 + N)
    ref = _oracle(sd, x, dev)
    a = r.forward(x.to(dev), normalize=False, denormalize=False, force_form=1)
    b = r.forward(x.to(dev), normalize=False, denormalize=False, force_form=2)
    assert torch.equal(a, b)
    bar = LAYERS * 100 * EPS32 * ref.abs().max().item()
    err = (a.double() - ref).abs().max().item()
    print("L=100 N=%d ratio %.3g" % (N, err / bar))
    assert err / bar < 1


def _checkpoint(tmp_path, seed):
    """A seeded LinearModelPG(1024) checkpoint in the reference's layout and a norm.pkl."""
    import pickle
    from oracle import restate_refiner as rr
    sd = rr.init_state(rr.param_shapes(L, 45, 45), seed)
    ck, nm = str(tmp_path / "refiner.pth.tar"), str(tmp_path / "norm.pkl")
    torch.save({"epoch": 1, "state_dict": sd}, ck)
    rng = np.random.default_rng(seed)
    norm = (rng.normal(0, 50, 45).astype(np.float32), rng.uniform(50, 150, 45).astype(np.float32),
            rng.normal(0, 50, 45).astype(np.float32), rng.uniform(50, 150, 45).astype(np.float32))
    with open(nm, "wb") as f:
        pickle.dump(norm, f)
    return ck, nm


def test_h36m_evaluate_with_refiner(dev, golden, tmp_path):
    """TEST.REFINER on the fixture tree (MPII order): the nine protocol entries and perf bit-identical
    to the evaluation without it, then the four Refined-* entries equal to the restatement (the
    Refiner on the evaluation's pred column, errors against gt with the hip dropped)."""
    import types
    import lib.dataset as dataset
    from lib.core import refine
    from lib.dataset.h36m_eval import evaluate_h36m
    from tests import dataset_cases as dc
    ck, nm = _checkpoint(tmp_path, 41)
    g = golden("datasets")
    preds = g["h36m_eval_mpii/preds"].copy()
    preds[:, :, :3] += np.random.default_rng(2).normal(0, 10, preds[:, :, :3].shape)

    def run(refiner, norm):
        cfg = dc.cfg(MPII_ORDER=True)
        cfg.TEST = types.SimpleNamespace(PSS_K=[], PSS_CENTROIDS='', REFINER=refiner, REFINER_NORM=norm)
        dc.seeded(dc.SEED % 1000)
        ds = dataset.h36m(cfg, dc.H36M_ROOT, "valid", False)
        return ds, ds.evaluate(preds.copy(), None)
    _, (nv0, perf0) = run('', '')
    ds, (nv, perf) = run(ck, nm)
    assert nv[:9] == nv0 and perf == perf0
    assert [n for n, _ in nv[9:]] == list(refine.REFINED_NAMES)
    S = len(preds)
    get = lambda k: np.stack([np.asarray(r[k], dtype=np.float64).reshape(-1) for r in ds.db[:S]])
    _, _, det = evaluate_h36m(preds, np.stack([r['joints_3d'] for r in ds.db[:S]]), get('pelvis'), get('fl'),
                              get('c_p'), mpii_order=True, return_poses=True)
    pred, gt = refine.pairs_of(det['poses'])
    refined = refine.load_refiner(ck, nm).refine(pred)
    keep = [j for j in range(16) if j != 6]
    rm, _ = rc.pose_errors(refined[:, keep], gt[:, keep])
    assert np.max(np.abs(np.array([v for _, v in nv[9:]]) - rm.mean(axis=0)[:4])) <= 1e-9


def _boxes_cams(N, seed, HW):
    rng = np.random.default_rng(seed)
    boxes = {"center_x": rng.uniform(400, 600, N), "center_y": rng.uniform(400, 600, N),
             "width": rng.uniform(300, 500, N), "height": rng.uniform(300, 500, N)}
    boxes["height"] = boxes["width"].copy()
    cams = {"fl": rng.uniform(1100, 1200, (N, 2)), "c_p": rng.uniform(500, 520, (N, 2)),
            "depth": rng.uniform(3000, 6000, N)}
    return boxes, cams


def test_refined_pose_predictor(dev, tmp_path):
    """RefinedPosePredictor against PosePredictor(boxes) -> epb_h36m_eval's pred column -> Refiner.refine:
    bit-identical (pose_to_camera is that column's arithmetic, the refiner is batch-invariant); the
    graph reused with new images, boxes and cameras; refresh() re-reads the refiner."""
    from epipolarpose_b200 import ops
    from oracle import restate_refiner as rr
    from refiner import model as rmodel
    from refiner.model import Refiner
    from lib.core.inference import PosePredictor, RefinedPosePredictor
    from tests import golden_inputs as gi
    from tests.test_gpu_sizes import _model
    c = gi.SIZE_CASES["c1"]
    model = _model(dev, c, "f16x3", train=False)
    HW = c["HW"]
    sd = rr.init_state(rr.param_shapes(L, 45, 45), 43)
    rnet = rmodel.LinearModelPG(linear_size=L, input_size=45, output_size=45)
    rnet.load_state_dict(sd)
    rnet = rnet.to(dev)
    norm = (np.full(45, 3.0, np.float32), np.full(45, 120.0, np.float32), np.full(45, -2.0, np.float32),
            np.full(45, 90.0, np.float32))
    rp = RefinedPosePredictor(model, rnet, norm, flip_test=False)
    pp = PosePredictor(model, flip_test=False)

    def check(N, seed):
        x = np.random.default_rng(seed).standard_normal((N, 3, HW, HW)).astype(np.float32)
        boxes, cams = _boxes_cams(N, seed, HW)
        got = rp(x, boxes, cams)
        kps = pp(x, boxes=boxes)
        assert np.array_equal(got["kps"], kps)
        cam = np.concatenate([cams["fl"], cams["c_p"], cams["depth"][:, None]], 1)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).to(dev)
        poses = torch.empty((N, 16, 9), dtype=torch.float64, device=dev)
        metrics = torch.empty((N, 9), dtype=torch.float64, device=dev)
        ops.h36m_eval(t(kps[:, :, :3]), t(kps[:, :, :3]), t(cam), N, 16, 6, 0, 150.0, metrics, None, None, poses)
        assert np.array_equal(got["pose"], poses[:, :, 0:3].cpu().numpy())
        want = Refiner(rnet, norm).refine(poses[:, :, 0:3].cpu().numpy())
        assert np.array_equal(got["refined"], want)
        return got
    check(1, 1)
    check(1, 2)                                   # the N = 1 graph again, new images, boxes, cameras
    check(3, 3)
    assert len(rp.graphs) == 2
    with torch.no_grad():
        rnet.w4.bias.add_(0.5)
    rp.refresh()
    check(3, 4)
    with pytest.raises(ValueError):
        rp(np.zeros((1, 3, HW, HW), np.float32), None, None)
