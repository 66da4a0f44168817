"""GPU (-m gpu): pseudo-label records for self-supervised Human3.6M training.
  * epb_pseudo_records against the numpy restatement (tests/pseudo_cases.py) at T in {1, 64, 4096},
    one pose per frame and one per camera, V 4 and 8; two launches give the same bits; refusals;
  * save_triangulations on the fixture tree with the network bypassed: a predictor with
    MultiViewPredictor's (PosePredictor's) interface whose 2-D joints are exact projections of the
    records' ground truth, triangulated by the library -> the source's joints_3d and pelvis back;
    with 3 px noise, the restatement's triangulation and projection;
  * with a seeded random-init network, the builder equals "predictor, then epb_pseudo_records";
  * the written pickle trains as train-ss (TRI false and true); two runs write the same bytes."""
import os

import numpy as np
import pytest
import torch

from tests import dataset_cases as dc
from tests import multiview_cases as mc
from tests import pseudo_cases as pc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _gpu(X, st, cam, root, dev):
    from lib.utils.prep_h36m import pseudo_records
    return [a.cpu().numpy() for a in pseudo_records(_t(X, dev), _t(st.astype(np.int32), dev), _t(cam, dev), root)]


@pytest.mark.parametrize("V", [4, 8])
@pytest.mark.parametrize("per_camera", [False, True])
def test_kernel_vs_restatement(dev, V, per_camera):
    S = V if per_camera else 1
    for T, J, step in ((1, 17, 1), (64, 16, 4), (4096, 17, 256)):
        root = 6 if J == 16 else 0
        X, st, cam = pc.case(T + V + S, T, S, V, J, root)
        got = _gpu(X, st, cam, root, dev)
        rows = list(range(0, T, step)) + [min(T - 1, i) for i in (1, 2, 3, 4)]
        rows = sorted(set(rows))
        want = pc.restated(X[rows], st[rows], cam[rows], root)
        pc.assert_same([a[rows] for a in got], want)
        again = _gpu(X, st, cam, root, dev)
        for a, b in zip(got, again):
            assert np.array_equal(a, b)


def test_argument_checks(dev):
    from epipolarpose_b200 import ops
    from epipolarpose_b200._lib import EpbError
    X, st, cam = pc.case(3, 2, 1, 4, 17)
    Xd, sd, cd = _t(X, dev), _t(st, dev), _t(cam, dev)
    out = lambda: (torch.zeros((2, 4, 17, 3), device=dev, dtype=torch.float64),
                   torch.zeros((2, 4, 17, 3), device=dev, dtype=torch.float64),
                   torch.zeros((2, 4, 3), device=dev, dtype=torch.float64),
                   torch.zeros((2, 4), device=dev, dtype=torch.int32))
    for T, S, V, J, root in ((2, 2, 4, 17, 0), (2, 1, 9, 17, 0), (2, 1, 1, 17, 0), (2, 1, 4, 17, 17),
                             (-1, 1, 4, 17, 0), (2, 1, 4, 17, -1)):
        with pytest.raises(EpbError):
            ops.pseudo_records(Xd, sd, cd, T, S, V, J, root, *out())
    o = out()
    ops.pseudo_records(Xd, sd, cd, 0, 1, 4, 17, 0, *o)            # T = 0: nothing written
    torch.cuda.synchronize()
    assert not any(a.any() for a in o)


# ------------------------------------------------------------------ save_triangulations, network bypassed
def _world(anno, k):
    from lib.core.function import world_joints_of_record
    V = len(anno)
    return np.mean([world_joints_of_record(anno[c + 1][k]) for c in range(V)], axis=0)


def _exact_multiview(anno, dev, noise=0.0, log=None):
    """MultiViewPredictor's interface: exact (or noisy) projections of the records' ground truth,
    triangulated by epb_triangulate_robust."""
    import lib.utils.triangulation as tri
    from oracle import restate
    seen = []
    rng = np.random.default_rng(5)

    def predictor(images, boxes, P):
        T, V = images.shape[:2]
        ks = range(len(seen), len(seen) + T)
        seen.extend(ks)
        W = np.stack([_world(anno, k) for k in ks])
        u = np.stack([np.stack([restate.project(P[i, v], W[i]) for v in range(V)]) for i in range(T)])
        u = u + rng.normal(0, noise, u.shape) if noise else u
        X, st, inl, res = tri.triangulate_views_robust(_t(u, dev), _t(P, dev))
        if log is not None:
            log.append((u, P))
        return {"world": X.cpu().numpy(), "status": st.cpu().numpy(), "inliers": inl.cpu().numpy(),
                "resid": res.cpu().numpy()}
    return predictor


def _exact_single(anno):
    """PosePredictor's interface: exact projections of the records' ground truth, [N, J, 4]."""
    from oracle import restate
    seen = []

    def predictor(images, boxes):
        V = len(anno)
        T = images.shape[0] // V
        ks = range(len(seen), len(seen) + T)
        seen.extend(ks)
        out = []
        for k in ks:
            W = _world(anno, k)
            for c in range(V):
                u = restate.project(np.asarray(anno[c + 1][k]["cam"].projection_matrix, np.float64)[:3], W)
                out.append(np.concatenate([u, np.zeros((len(W), 1)), np.ones((len(W), 1))], axis=1))
        return np.stack(out)
    return predictor


def _source():
    from lib.dataset.JointIntegralDataset import load_pickle
    return load_pickle(os.path.join(dc.H36M_ROOT, "annot", "valid.pkl"))


@pytest.mark.parametrize("method", ["robust", "iterative", "polynomial"])
def test_exact_projections_give_the_source_back(dev, tmp_path, method):
    from lib.utils.prep_h36m import save_triangulations
    from lib.dataset.JointIntegralDataset import load_pickle
    anno = _source()
    ds = dc.build("h36m_valid")
    pred = _exact_multiview(anno, dev) if method == "robust" else _exact_single(anno)
    dst = str(tmp_path / "ss.pkl")
    rep = save_triangulations(None, ds, anno, dst, method=method, tuples_per_batch=2, workers=2, predictor=pred)
    assert rep["frames"] == 3 and rep["dropped"] == 0 and rep["failed"] == 0.0
    assert rep["agreement_mm"] < 1e-6
    assert (rep["inlier_views"] == 4.0) if method == "robust" else rep["inlier_views"] is None
    out = load_pickle(dst)
    for c in anno:
        assert len(out[c]) == 3
        for r, s in zip(out[c], anno[c]):
            assert r["image"] == s["image"]
            assert np.max(np.abs(r["joints_3d"] - s["joints_3d"])) <= 1e-6
            assert np.max(np.abs(r["pelvis"] - s["pelvis"])) <= 1e-6
            assert np.all(r["joints_3d_vis"] == 1)


def test_noisy_projections_match_the_restatement(dev, tmp_path):
    from lib.utils.prep_h36m import save_triangulations, _cam16
    from lib.dataset.JointIntegralDataset import load_pickle
    anno = _source()
    log = []
    dst = str(tmp_path / "ss.pkl")
    rep = save_triangulations(None, dc.build("h36m_valid"), anno, dst, tuples_per_batch=2, workers=1,
                              predictor=_exact_multiview(anno, dev, noise=3.0, log=log))
    out = load_pickle(dst)
    u = np.concatenate([a for a, _ in log])
    P = np.concatenate([b for _, b in log])
    Xr = np.stack([mc.robust_nview_triangulation(u[t], P[t], None, 15.0)[0] for t in range(len(u))])
    str_ = np.stack([mc.robust_nview_triangulation(u[t], P[t], None, 15.0)[1] for t in range(len(u))])
    cam = np.stack([np.stack([_cam16(anno[c + 1][k]) for c in range(4)]) for k in range(3)])
    jt, vis, pel, ok = pc.restated(Xr[:, None], str_[:, None].astype(np.int32), cam, 0)
    keep = np.flatnonzero(ok.all(axis=1))
    assert rep["frames"] == len(keep) == 3
    for i, k in enumerate(keep):
        for c in range(4):
            r = out[c + 1][i]
            assert np.array_equal(r["joints_3d_vis"], vis[k, c])
            assert np.max(np.abs(r["joints_3d"] - jt[k, c])) <= 1e-4
            assert np.max(np.abs(r["pelvis"] - pel[k, c])) <= 1e-4
    # agreement_mm: root-relative camera-frame MPJPE against the source (CamBackProj restated), over
    # the joints visible in both (the fixture's source hides two)
    def cam_frame(j, f, c, depth):
        d = j[:, 2] + depth
        y = np.stack([(j[:, 0] - c[0]) / f[0] * d, (j[:, 1] - c[1]) / f[1] * d, d], axis=1)
        return y - y[0]
    e = [np.linalg.norm(cam_frame(jt[k, c], cam[k, c, 12:14], cam[k, c, 14:16], pel[k, c, 2])
                        - cam_frame(anno[c + 1][k]["joints_3d"], anno[c + 1][k]["fl"], anno[c + 1][k]["c_p"],
                                    anno[c + 1][k]["pelvis"][2]), axis=1)
         [(vis[k, c, :, 0] == 1) & (anno[c + 1][k]["joints_3d_vis"][:, 0] > 0)]
         for k in keep for c in range(4)]
    assert abs(rep["agreement_mm"] - np.concatenate(e).mean()) <= 1e-3        # the 1e-4 mm of the joints


def test_two_runs_write_the_same_bytes(dev, tmp_path):
    from lib.utils.prep_h36m import save_triangulations
    anno = _source()
    blobs = []
    for i in range(2):
        dst = str(tmp_path / ("ss%d.pkl" % i))
        save_triangulations(None, dc.build("h36m_valid"), os.path.join(dc.H36M_ROOT, "annot", "valid.pkl"), dst,
                            tuples_per_batch=2, workers=2, predictor=_exact_multiview(anno, dev, noise=3.0))
        with open(dst, "rb") as f:
            blobs.append(f.read())
    assert blobs[0] == blobs[1]


# ------------------------------------------------------------------ a seeded random-init network
@pytest.fixture(scope="module")
def c1(dev):
    from tests import golden_inputs as gi
    from tests.golden_inputs import _model
    return _model(dev, gi.SIZE_CASES["c1"], "f16x3", train=False)         # R50, J 16, 256x256


class _Recording:
    """Wraps a predictor and keeps every call's inputs and outputs."""

    def __init__(self, inner):
        self.inner, self.calls = inner, []

    def __call__(self, images, *a):
        x = images.clone() if torch.is_tensor(images) else np.array(images)
        out = self.inner(images, *a)
        self.calls.append((x, a, out))
        return out


@pytest.mark.parametrize("method", ["robust", "iterative", "polynomial"])
def test_random_network_equals_the_composition(c1, dev, tmp_path, method):
    from lib.core.inference import MultiViewPredictor, PosePredictor
    from lib.dataset.JointIntegralDataset import load_pickle
    from lib.utils.prep_h36m import save_triangulations, pseudo_records, _cam16
    from lib.utils.triangulation import triangulate_pairs
    import lib.dataset as dataset
    dc.seeded(dc.SEED % 1000)
    cfg = dc.cfg()
    cfg.MODEL.IMAGE_SIZE = [256, 256]
    ds = dataset.h36m(cfg, dc.H36M_ROOT, "valid", False)
    anno = _source()
    inner = MultiViewPredictor(c1, flip_test=False, threshold_px=1e4) if method == "robust" \
        else PosePredictor(c1, flip_test=False)
    rec = _Recording(inner)
    dst = str(tmp_path / "ss.pkl")
    rep = save_triangulations(c1, ds, anno, dst, method=method, tuples_per_batch=2, workers=2, predictor=rec)
    out = load_pickle(dst)
    assert [len(c[1][0]["center_x"]) for c in rec.calls] == [8, 4]
    assert all(x.shape[-2:] == (256, 256) for x, _, _ in rec.calls)
    # the composition, on the images the builder assembled
    want = {c: [] for c in anno}
    k0, nfail = 0, 0
    for x, args, _ in rec.calls:
        boxes = args[0]
        T = len(boxes["center_x"]) // 4
        cam = np.stack([np.stack([_cam16(anno[c + 1][k]) for c in range(4)]) for k in range(k0, k0 + T)])
        P = np.stack([np.stack([np.asarray(anno[c + 1][k]["cam"].projection_matrix)[:3] for c in range(4)])
                      for k in range(k0, k0 + T)])
        if method == "robust":
            r = inner(x, boxes, P)
            X, st = _t(r["world"], dev)[:, None], _t(r["status"], dev)[:, None]
        else:
            kps = _t(inner(x, boxes).reshape(T, 4, -1, 4), dev)
            nb = torch.tensor([1, 0, 0, 1], device=dev)
            Pd = _t(P, dev)
            X, st = triangulate_pairs(kps.reshape(4 * T, -1, 4), kps[:, nb].reshape(4 * T, -1, 4),
                                      Pd.reshape(4 * T, 3, 4), Pd[:, nb].reshape(4 * T, 3, 4),
                                      "iterative_LS" if method == "iterative" else "polynomial")
            X, st = X.view(T, 4, -1, 3), st.view(T, 4, -1)
        nfail += int((st != 1).sum())
        jt, vis, pel, ok = (a.cpu().numpy() for a in pseudo_records(X, st, _t(cam, dev), 6))
        for i in range(T):
            if ok[i].all():
                for c in range(4):
                    want[c + 1].append((k0 + i, jt[i, c], vis[i, c], pel[i, c]))
        k0 += T
    assert rep["frames"] == len(want[1]) and rep["failed"] == nfail / (3 * 16 * (1 if method == "robust" else 4))
    for c in anno:
        assert len(out[c]) == len(want[c])
        for r, (k, jt, vis, pel) in zip(out[c], want[c]):
            assert r["image"] == anno[c][k]["image"]
            assert np.array_equal(r["joints_3d"], jt) and np.array_equal(r["joints_3d_vis"], vis)
            assert np.array_equal(r["pelvis"], pel) and len(r["parent_ids"]) == 16
    print(method, rep)


# ------------------------------------------------------------------ the written file trains
def _train_epoch(root, tri):
    """One train_integral epoch (three steps at batch 1) of scripts/train.py's set-up on the written
    file, R18, 64x64; the loader's batches are not pinned, so nothing allocates pinned memory
    beside the graph capture of the training step."""
    from torch.utils.data import DataLoader
    import lib.core.integral_loss as loss
    import lib.dataset as dataset
    import lib.models as models
    from lib.core.config import config, reset_config
    from lib.core.function import train_integral
    from lib.utils.utils import get_optimizer
    reset_config()
    try:
        config.WORKERS, config.PRINT_FREQ = 2, 1
        config.MODEL.NUM_JOINTS, config.MODEL.DEPTH_RES = 17, 16
        config.MODEL.IMAGE_SIZE = np.array([64, 64])
        config.MODEL.EXTRA.NUM_LAYERS, config.MODEL.INIT_WEIGHTS = 18, False
        config.LOSS.FN = "SmoothL1JointLocationLoss"
        config.DATASET.DATASET, config.DATASET.ROOT, config.DATASET.TRAIN_SET = "h36m", root, "train-ss"
        config.DATASET.TRI = tri
        config.TRAIN.ONLINE_TRIANGULATION = tri
        config.TRAIN.BATCH_SIZE = 1
        model = torch.nn.DataParallel(models.pose3d_resnet.get_pose_net(config, is_train=True), device_ids=[0]).cuda()
        criterion = loss.SmoothL1JointLocationLoss(num_joints=17, norm=config.LOSS.NORM).cuda()
        optimizer = get_optimizer(config, model)
        ds = dataset.h36m(cfg=config, root=root, image_set="train-ss", is_train=True)
        dl = DataLoader(ds, batch_size=1, shuffle=True, num_workers=config.WORKERS)
        avg = train_integral(config, dl, model, criterion, optimizer, 0)
    finally:
        reset_config()
    return avg, len(ds)


@pytest.mark.parametrize("tri", [False, True])
def test_written_pickle_trains_as_train_ss(dev, tmp_path, tri):
    from lib.utils.prep_h36m import save_triangulations
    import lib.dataset as dataset
    root = tmp_path / "h36m"
    (root / "annot").mkdir(parents=True)
    os.symlink(os.path.join(dc.H36M_ROOT, "images"), str(root / "images"))
    anno = _source()
    save_triangulations(None, dc.build("h36m_valid"), anno, str(root / "annot" / "train-ss.pkl"), workers=1,
                        predictor=_exact_multiview(anno, dev, noise=3.0))
    dc.seeded(1)
    ds = dataset.h36m(dc.cfg(TRI=tri), str(root), "train-ss", True)
    assert len(ds) == (3 if tri else 12)
    item = ds[0]
    views = [item["cam_1"], item["cam_2"]] if tri else [item]
    for v in views:
        assert v[0].shape == (3, 64, 64) and np.isfinite(v[1]).all() and v[2].size == 51
    avg, n = _train_epoch(str(root), tri)
    assert n == len(ds) and np.isfinite(avg)
