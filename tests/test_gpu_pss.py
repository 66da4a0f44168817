"""GPU (-m gpu): the Pose Structure Score kernels of csrc/pss.cu against the numpy restatement
(tests/pss_cases.py), bit for bit: pose normalisation, every k-means++ index, every Lloyd pass's
labels, the final centroids and the inertia; run-to-run identity; an emptied cluster; the
properties of a 1.5 M-pose fit; H36M_Integral.evaluate and the training-script flow with
TEST.PSS_K on the fixture tree."""
import logging

import numpy as np
import pytest
import torch

from tests import dataset_cases as dc
from tests import pss_cases as pc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture
def clean_cache():
    import lib.core.pss as pss
    pss._CLUSTERS.clear()
    yield pss
    pss._CLUSTERS.clear()


def _fit(dev, x, k, seed, restart, max_iter):
    from epipolarpose_b200 import ops
    N, d = x.shape
    xt = torch.from_numpy(x).to(dev)
    ws = torch.empty(ops.kmeans_workspace(N, d, k), dtype=torch.uint8, device=dev)
    cen = torch.empty(k, d, dtype=torch.float64, device=dev)
    lab = torch.empty(N, dtype=torch.int32, device=dev)
    idx = torch.empty(k, dtype=torch.int32, device=dev)
    trace = torch.full((max_iter + 1, N), -1, dtype=torch.int32, device=dev)
    inertia, n_iter = ops.kmeans_fit(xt, N, d, k, seed, restart, max_iter, cen, lab, idx, trace, ws)
    return dict(init_idx=idx.cpu().numpy(), trace=trace[:n_iter + 1].cpu().numpy(), centroids=cen.cpu().numpy(),
                labels=lab.cpu().numpy(), inertia=inertia, n_iter=n_iter)


def _same(a, b):
    assert np.array_equal(a["init_idx"], b["init_idx"])
    assert a["n_iter"] == b["n_iter"]
    assert np.array_equal(a["trace"], b["trace"])
    assert np.array_equal(a["centroids"], b["centroids"])
    assert np.array_equal(a["labels"], b["labels"])
    assert a["inertia"] == b["inertia"]


@pytest.mark.parametrize("J,root", [(17, 0), (16, 6)])
def test_pose_normalize_bit_identical(dev, J, root):
    from epipolarpose_b200 import ops
    rng = np.random.default_rng(J)
    S = 4099
    pose = np.concatenate([rng.uniform(100, 900, (S, J, 2)), rng.normal(0, 300, (S, J, 1))], axis=2)
    cam = np.concatenate([rng.uniform(1100, 1200, (S, 2)), rng.uniform(480, 540, (S, 2)),
                          rng.uniform(3000, 6000, (S, 1))], axis=1)
    pose[5] = pose[5, root]                                              # a zero pose
    out = torch.empty(S, 3 * J, dtype=torch.float64, device=dev)
    ops.pose_normalize(torch.from_numpy(pose).to(dev), torch.from_numpy(cam).to(dev), S, J, root, out)
    ref = pc.normalize(pose, cam, root)
    assert np.array_equal(out.cpu().numpy(), ref)
    assert not ref[5].any()


# the restatement's Lloyd costs ~N*k*d numpy work per pass: the 65 537-point fits stop after 6 updates
@pytest.mark.parametrize("N", [1000, 65537])
@pytest.mark.parametrize("k", [3, 50, 100])
@pytest.mark.parametrize("d", [48, 51])
def test_kmeans_restart_bit_identical(dev, N, k, d):
    x = pc.skeleton_poses(np.random.default_rng(N + k + d), N, d // 3, k_true=max(8, k // 2))
    max_iter = 300 if N <= 1000 else 6
    got = _fit(dev, x, k, 11, 2, max_iter)
    _same(got, pc.fit_restart(x, k, 11, 2, max_iter))
    if N == 65537 and k == 100 and d == 51:
        _same(got, _fit(dev, x, k, 11, 2, max_iter))                      # run to run
    from epipolarpose_b200 import ops
    lab = torch.empty(N, dtype=torch.int32, device=dev)
    d2 = torch.empty(N, dtype=torch.float64, device=dev)
    ops.kmeans_assign(torch.from_numpy(x).to(dev), N, d, torch.from_numpy(got["centroids"]).to(dev), k, lab, d2)
    rl, rd = pc.assign(x, got["centroids"])
    assert np.array_equal(lab.cpu().numpy(), rl) and np.array_equal(d2.cpu().numpy(), rd)


def test_kmeans_relocation_bit_identical(dev):
    x, k, seed = pc.relocation_case()
    ref = pc.fit_restart(x, k, seed, 0, 50)
    assert ref["relocated"] == 1
    _same(_fit(dev, x, k, seed, 0, 50), ref)


def test_kmeans_errors(dev):
    from epipolarpose_b200 import ops
    from epipolarpose_b200._lib import EpbError
    x = pc.skeleton_poses(np.random.default_rng(6), 20, 16)
    with pytest.raises(EpbError):
        ops.kmeans_workspace(20, 48, 21)
    with pytest.raises(EpbError):
        ops.kmeans_workspace(200, 300, 100)                               # shared memory
    with pytest.raises(EpbError, match="distinct"):
        _fit(dev, np.repeat(x[:2], 10, axis=0), 3, 0, 0, 10)
    bad = x.copy()
    bad[7, 5] = np.inf
    with pytest.raises(EpbError, match="non-finite"):
        _fit(dev, bad, 3, 0, 0, 10)
    lab = torch.empty(20, dtype=torch.int32, device=dev)
    with pytest.raises(EpbError, match="non-finite"):
        ops.kmeans_assign(torch.from_numpy(bad).to(dev), 20, 48, torch.from_numpy(x[:3]).to(dev), 3, lab, None)


def test_kmeans_large_fit_properties(dev):
    """N = 1.5e6, k = 100, d = 51: the final labels are the argmin of the returned centroids (torch
    float64, sequential over coordinates, first minimum); each centroid is the mean of the members
    of the last update's labels within 1e-12 relative."""
    N, k, d = 1_500_000, 100, 51
    x = pc.skeleton_poses(np.random.default_rng(15), N, 17, k_true=100)
    f = _fit(dev, x, k, 0, 0, 300)
    assert f["n_iter"] >= 1
    xt = torch.from_numpy(x).to(dev)
    c = torch.from_numpy(f["centroids"]).to(dev)
    lab = torch.empty(N, dtype=torch.int64, device=dev)
    for i0 in range(0, N, 100_000):
        xb = xt[i0:i0 + 100_000]
        s = torch.zeros(len(xb), k, dtype=torch.float64, device=dev)
        for t in range(d):
            e = xb[:, t, None] - c[None, :, t]
            s = s + e * e
        lab[i0:i0 + 100_000] = torch.argmin(s, dim=1)
    assert np.array_equal(lab.cpu().numpy(), f["labels"])
    prev = torch.from_numpy(f["trace"][f["n_iter"] - 1].astype(np.int64)).to(dev)
    cnt = torch.bincount(prev, minlength=k)
    sums = torch.zeros(k, d, dtype=torch.float64, device=dev).index_add_(0, prev, xt)
    full = cnt > 0
    mean = sums[full] / cnt[full, None]
    rel = ((c[full] - mean).abs().amax(1) / mean.abs().amax(1)).max().item()
    assert rel <= 1e-12, rel


def _evaluate(g, order, pss_k):
    import types
    import lib.dataset as dataset
    cfg = dc.cfg(MPII_ORDER=order == "mpii")
    cfg.TEST = types.SimpleNamespace(PSS_K=pss_k, PSS_CENTROIDS='')
    dc.seeded(dc.SEED % 1000)
    ds = dataset.h36m(cfg, dc.H36M_ROOT, "valid", False)
    preds = g["h36m_eval_" + order + "/preds"].copy()
    preds[:, :, :3] += np.random.default_rng(9).normal(0, 25, preds[:, :, :3].shape)
    return ds, preds, ds.evaluate(preds.copy(), None)


@pytest.mark.parametrize("order", ["h36m", "mpii"])
def test_h36m_evaluate_pss_on_device(dev, golden, clean_cache, order):
    g = golden("datasets")
    _, _, (nv0, perf0) = _evaluate(g, order, [])
    ds, preds, (nv, perf) = _evaluate(g, order, [2, 3])
    assert nv[:9] == nv0 and perf == perf0
    assert nv[9:] == pc.fixture_pss(ds.db, preds, order == "mpii", [2, 3])


def test_script_flow_logs_pss(dev, clean_cache, tmp_path, caplog):
    """scripts/valid.py's call sequence (validate_integral, eval_integral) with TEST.PSS_K set and
    WORKERS: 2 logs one Validation-PSS@k line per k."""
    from torch.utils.data import DataLoader
    import lib.dataset as dataset_m
    import lib.models as models
    from lib.core.config import config, reset_config
    from lib.core.function import validate_integral, eval_integral
    reset_config()
    try:
        config.WORKERS = 2
        config.MODEL.NUM_JOINTS, config.MODEL.DEPTH_RES = 17, 16
        config.MODEL.IMAGE_SIZE = np.array([64, 64])
        config.MODEL.EXTRA.NUM_LAYERS, config.MODEL.INIT_WEIGHTS = 18, False
        config.DATASET.DATASET, config.DATASET.ROOT = "h36m", dc.H36M_ROOT
        config.TEST.PSS_K = [2, 3]
        model = torch.nn.DataParallel(models.pose3d_resnet.get_pose_net(config, is_train=False), device_ids=[0]).cuda()
        valid_ds = dataset_m.h36m(cfg=config, root=config.DATASET.ROOT, image_set=config.DATASET.TEST_SET,
                                  is_train=False)
        loader = DataLoader(valid_ds, batch_size=config.TEST.BATCH_SIZE, shuffle=False, num_workers=config.WORKERS)
        preds = validate_integral(loader, model)
        with caplog.at_level(logging.INFO):
            perf = eval_integral(0, preds, loader, str(tmp_path))
    finally:
        reset_config()
    assert np.isfinite(perf)
    lines = [r.getMessage() for r in caplog.records if "Validation-PSS@" in r.getMessage()]
    assert len(lines) == 2 and "Validation-PSS@2" in lines[0] and "Validation-PSS@3" in lines[1]
