"""CPU: the Pose Structure Score definition (lib/core/pss.py) through its numpy restatement
(tests/pss_cases.py): the restatement's fixed orders and draws, its agreement with scikit-learn's
Lloyd, the empty-cluster rule, the config keys, the errors, and H36M_Integral.evaluate on the
fixture tree through the emulated C ABI."""
import types

import numpy as np
import pytest

from tests import dataset_cases as dc
from tests import emul_ops
from tests import emul_pss
from tests import pss_cases as pc


@pytest.fixture
def emulated():
    import lib.core.pss as pss
    import lib.dataset.h36m_eval as he
    pss._CLUSTERS.clear()
    pss._backend[0], he._backend[0] = emul_pss, emul_ops
    yield pss
    ops = __import__("epipolarpose_b200.ops", fromlist=["ops"])
    pss._backend[0] = he._backend[0] = ops
    pss._CLUSTERS.clear()


def test_splitmix64_and_fixed_orders():
    """splitmix64's first output from state 0, and the restatement's sums really are sequential:
    np.cumsum per chunk and np.add.at against explicit loops, on values whose sums depend on order."""
    assert pc.uniform(0, 0, 0) == (0xE220A8397B1DCDAF >> 11) * 2.0 ** -53
    assert pc.uniform(7, 3, 5) != pc.uniform(7, 4, 5)
    rng = np.random.default_rng(1)
    v = np.exp(rng.uniform(-30, 30, 2500))
    pre = pc.chunk_prefix(v)
    for c in range(3):
        s = 0.0
        for i in range(c * pc.CHUNK, min((c + 1) * pc.CHUNK, len(v))):
            s += v[i]
            assert pre[c, i - c * pc.CHUNK] == s
    x = np.exp(rng.uniform(-30, 30, (300, 4)))
    lab = rng.integers(0, 3, 300)
    part = np.zeros((3, 4))
    np.add.at(part, lab, x)
    ref = np.zeros((3, 4))
    for i in range(300):
        ref[lab[i]] = ref[lab[i]] + x[i]
    assert np.array_equal(part, ref)


@pytest.mark.parametrize("N,J,k,k_true", [(3000, 17, 5, 5), (2500, 16, 12, 12)])
def test_restatement_matches_sklearn_lloyd(N, J, k, k_true):
    """From the same k-means++ seeds, scikit-learn's Lloyd (tol=0) on well-separated poses ends with
    the same labels and centroids within 1e-10."""
    sk = pytest.importorskip("sklearn.cluster")
    x = pc.skeleton_poses(np.random.default_rng(N), N, J, k_true=k_true, spread=0.01)
    f = pc.fit_restart(x, k, 0, 0, 300)
    assert f["relocated"] == 0 and f["n_iter"] < 300
    km = sk.KMeans(n_clusters=k, init=x[f["init_idx"]], n_init=1, algorithm="lloyd", tol=0, max_iter=300).fit(x)
    assert np.array_equal(km.labels_, f["labels"])
    assert np.max(np.abs(km.cluster_centers_ - f["centroids"])) <= 1e-10


def test_relocation_rule():
    """Empty clusters, in cluster order, take the points farthest from their centres; equal
    distances go to the lower index; no point twice."""
    x = np.arange(12, dtype=np.float64).reshape(6, 2)
    labels = np.array([0, 0, 2, 2, 2, 0], dtype=np.int32)
    dist2 = np.array([1.0, 5.0, 2.0, 5.0, 0.5, 3.0])
    cen = np.full((4, 2), -1.0)
    new = pc.update(x, labels, dist2, cen)
    assert np.array_equal(new[0], (x[0] + x[1] + x[5]) / 3) and np.array_equal(new[2], (x[2] + x[3] + x[4]) / 3)
    assert np.array_equal(new[1], x[1]) and np.array_equal(new[3], x[3])
    # a fit in which a cluster empties (pss_cases.relocation_case)
    xr, k, seed = pc.relocation_case()
    f = pc.fit_restart(xr, k, seed, 0, 50)
    assert list(f["init_idx"]) == [2, 12, 0] and f["relocated"] == 1
    c0 = xr[f["init_idx"]]
    c1 = pc.update(xr, f["trace"][0], pc.assign(xr, c0)[1], c0)
    lab1, d1 = pc.assign(xr, c1)
    assert np.array_equal(lab1, f["trace"][1]) and np.bincount(lab1, minlength=k)[0] == 0
    far = int(np.lexsort((np.arange(len(xr)), -d1))[0])
    assert far == 12                                                    # y = -4, farthest from -1.87
    assert np.array_equal(pc.update(xr, lab1, d1, c1)[0], xr[far])


def test_normalize_is_scale_free_root_relative():
    rng = np.random.default_rng(2)
    S, J = 40, 17
    pose = np.concatenate([rng.uniform(100, 900, (S, J, 2)), rng.normal(0, 300, (S, J, 1))], axis=2)
    cam = np.concatenate([rng.uniform(1100, 1200, (S, 2)), rng.uniform(480, 540, (S, 2)),
                          rng.uniform(3000, 6000, (S, 1))], axis=1)
    pose[3] = pose[3, 0]                                                 # every joint on the root
    out = pc.normalize(pose, cam, 0)
    b = pc.back_project(pose, cam)
    v = (b - b[:, :1]).reshape(S, -1)
    n = np.linalg.norm(v, axis=1)
    ok = n > 0
    assert np.max(np.abs(out[ok] - v[ok] / n[ok, None])) <= 1e-15
    assert not ok[3] and np.array_equal(out[3], np.zeros(J * 3))
    assert np.allclose(np.linalg.norm(out[ok], axis=1), 1.0, rtol=0, atol=1e-15)


def test_public_interface_emulated(emulated):
    pss = emulated
    x = pc.skeleton_poses(np.random.default_rng(4), 1500, 17)
    c = pss.fit_pose_clusters(x, 6, seed=3, n_init=3, max_iter=40)
    assert np.array_equal(c, pc.fit(x, 6, seed=3, n_init=3, max_iter=40))
    assert np.array_equal(pss.assign_clusters(x, c), pc.assign(x, c)[0])
    y = x + 0.05 * np.random.default_rng(5).normal(size=x.shape)
    assert pss.pose_structure_score(y, x, c) == pc.pss(y, x, c)


def test_errors_emulated(emulated):
    """k > N, fewer than k distinct poses and non-finite input raise."""
    from epipolarpose_b200._lib import EpbError
    pss = emulated
    x = pc.skeleton_poses(np.random.default_rng(6), 20, 16)
    with pytest.raises(EpbError):
        pss.fit_pose_clusters(x, 21)
    with pytest.raises(EpbError):
        pss.fit_pose_clusters(np.repeat(x[:2], 10, axis=0), 3)
    bad = x.copy()
    bad[7, 5] = np.nan
    with pytest.raises(EpbError):
        pss.fit_pose_clusters(bad, 3)
    with pytest.raises(EpbError):
        pss.assign_clusters(bad, x[:3])


def test_config_keys(tmp_path):
    from lib.core.config import config, reset_config, update_config
    reset_config()
    assert config.TEST.PSS_K == [] and config.TEST.PSS_CENTROIDS == ''
    p = tmp_path / "e.yaml"
    p.write_text("TEST:\n  PSS_K: [50, 100]\n  PSS_CENTROIDS: 'c.npz'\n")
    try:
        update_config(str(p))
        assert config.TEST.PSS_K == [50, 100] and config.TEST.PSS_CENTROIDS == 'c.npz'
    finally:
        reset_config()


def _evaluate(order, g, pss_k=None, centroids_file=''):
    import lib.dataset as dataset
    cfg = dc.cfg(MPII_ORDER=order == "mpii")
    if pss_k is not None:
        cfg.TEST = types.SimpleNamespace(PSS_K=pss_k, PSS_CENTROIDS=centroids_file)
    dc.seeded(dc.SEED % 1000)
    ds = dataset.h36m(cfg, dc.H36M_ROOT, "valid", False)
    preds = g["h36m_eval_" + order + "/preds"].copy()
    preds[:, :, :3] += np.random.default_rng(9).normal(0, 25, preds[:, :, :3].shape)   # so that PSS < 1
    return ds, preds, ds.evaluate(preds.copy(), None)


@pytest.mark.parametrize("order", ["h36m", "mpii"])
def test_h36m_evaluate_pss_emulated(golden, emulated, order, monkeypatch):
    """TEST.PSS_K = [2, 3]: the nine protocol entries bit-identical to PSS off, then PSS@2, PSS@3
    equal to the restatement (clusters of the 12 train-fs poses); perf unchanged.  PSS_K empty
    makes no PSS call."""
    g = golden("datasets")
    _, _, (nv0, perf0) = _evaluate(order, g)
    import importlib
    h36m = importlib.import_module("lib.dataset.h36m")        # the package exports the class as `h36m`
    ds, preds, (nv, perf) = _evaluate(order, g, [2, 3])
    assert nv[:9] == nv0 and perf == perf0
    assert [n for n, _ in nv[9:]] == ["PSS@2", "PSS@3"]
    assert nv[9:] == pc.fixture_pss(ds.db, preds, order == "mpii", [2, 3])
    assert len(emulated._CLUSTERS) == 2
    monkeypatch.setattr(h36m, "h36m_pss", lambda *a, **k: pytest.fail("PSS computed with PSS_K empty"))
    assert _evaluate(order, g, [])[2] == (nv0, perf0)


def test_h36m_evaluate_pss_centroids_file(golden, emulated, tmp_path, monkeypatch):
    """TEST.PSS_CENTROIDS: the given centroids are used, nothing is fitted."""
    g = golden("datasets")
    rng = np.random.default_rng(8)
    cents = {k: rng.normal(size=(k, 51)) / 7.0 for k in (2, 3)}
    f = tmp_path / "c.npz"
    np.savez(str(f), k2=cents[2], k3=cents[3])
    monkeypatch.setattr(emulated, "fit_pose_clusters", lambda *a, **k: pytest.fail("fitted"))
    ds, preds, (nv, _) = _evaluate("h36m", g, [2, 3], str(f))
    assert nv[9:] == pc.fixture_pss(ds.db, preds, False, [2, 3], centroids=cents)
    np.savez(str(f), k2=cents[2], k3=cents[3][:, :48])
    with pytest.raises(ValueError):
        _evaluate("h36m", g, [2, 3], str(f))
