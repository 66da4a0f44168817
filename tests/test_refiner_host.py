"""CPU: the refiner's Human3.6M dataset (refiner/data.py) against the goldens the unmodified
reference class wrote from the same files (tests/golden/refiner_data*), its evaluate through the
emulated C ABI, main.py's choice of dataset, and the per-sample bodies of epb_pose_errors /
epb_pose_to_camera (csrc/geometry.cu) built for the CPU by tests/harness/host_pose_eval.cu against
the float64 restatement (tests/refiner_cases.py), once more under AddressSanitizer / UBSan."""
import logging
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest

from tests import emul_refiner
from tests import refiner_cases as rc
from tests.conftest import ROOT


@pytest.fixture
def data_dir(tmp_path):
    for name in ("train.pkl", "valid.pkl"):
        shutil.copy(os.path.join(rc.FIXTURE, name), tmp_path / name)
    return str(tmp_path)


@pytest.fixture
def emulated():
    from refiner import data
    data._backend[0] = emul_refiner
    yield data
    data._backend[0] = None


def test_dataset_matches_the_reference(data_dir, golden):
    from refiner import data
    g = golden("refiner_data")
    np.random.seed(int(g["seed"]))
    tr = data.Human36M(is_train=True, root=data_dir)
    assert os.path.exists(os.path.join(data_dir, "norm.pkl"))
    for k in ("data_mean", "data_std", "labels_mean", "labels_std"):
        assert getattr(tr, k).dtype == np.float32
        assert np.array_equal(getattr(tr, k), g[k]), k
    assert np.array_equal(tr.data, g["train_data"]) and np.array_equal(tr.labels, g["train_labels"])
    assert tr.data.shape == (96, 45) and tr.data.dtype == np.float32
    np.random.seed(int(g["seed"]))
    assert np.array_equal(np.random.permutation(len(tr)), g["perm"])
    va = data.Human36M(is_train=False, root=data_dir)
    assert np.array_equal(va.data, g["valid_data"]) and np.array_equal(va.labels, g["valid_labels"])
    x, y = va[3]
    assert np.array_equal(x, g["valid_data"][3]) and np.array_equal(y, g["valid_labels"][3])


def test_norm_pkl_is_loaded_not_recomputed(data_dir):
    from refiner import data
    stats = tuple(np.full(45, v, np.float32) for v in (1.0, 2.0, 3.0, 4.0))
    with open(os.path.join(data_dir, "norm.pkl"), "wb") as f:
        pickle.dump(stats, f)
    tr = data.Human36M(is_train=True, root=data_dir)
    assert all(np.array_equal(a, b) for a, b in zip(tr.norm(), stats))
    with open(os.path.join(rc.FIXTURE, "train.pkl"), "rb") as f:
        raw = pickle.load(f)
    inp = np.delete(np.asarray(raw["inp"], np.float32).reshape(-1, 48), np.s_[18:21], axis=1)
    assert sorted(map(tuple, tr.data)) == sorted(map(tuple, (inp - 1.0) / 2.0))


def test_valid_split_without_norm_raises(data_dir):
    from refiner import data
    with pytest.raises(FileNotFoundError, match="norm.pkl"):
        data.Human36M(is_train=False, root=data_dir)


def test_evaluate_through_the_emulated_abi(data_dir, golden, emulated, caplog):
    """The restatement in float64 against the reference's float32 evaluate.  Bar: the reference
    rounds every step to float32 (SVD included), so its means carry relative errors of a few
    float32 epsilons; 64 eps32 of the mean error is the bar, and the worst ratio is asserted < 1."""
    g = golden("refiner_data")
    np.random.seed(int(g["seed"]))
    emulated.Human36M(is_train=True, root=data_dir)
    va = emulated.Human36M(is_train=False, root=data_dir)
    with caplog.at_level(logging.INFO, logger=emulated.logger.name):
        ret = va.evaluate(g["eval_preds"])
    bar = 64 * np.finfo(np.float32).eps * g["eval_return"]
    got = np.array([va.last_results[k] for k in emulated.RESULT_NAMES])
    ratio = max(np.max(np.abs(got - g["eval_results"])), np.max(np.abs(np.array(va.last_per_joint) -
                                                                        g["eval_per_joint"]))) / bar
    assert ratio < 1, ratio
    assert abs(ret - g["eval_return"]) < bar
    assert "hm36_17j_14_al" in caplog.text and "LWrist" in caplog.text


def test_main_uses_the_files_when_present(data_dir, emulated, tmp_path, monkeypatch):
    """main() builds its loaders from Human36M when train.pkl and valid.pkl exist, and falls back
    to the synthetic poses otherwise (checked without running the network: the loaders are what
    test() would get)."""
    from refiner import main as rmain
    seen = []

    def fake_test(model, test_dl):
        seen.append(type(test_dl.dataset).__name__)
        return 0.0
    monkeypatch.setattr(rmain, "test", fake_test)
    monkeypatch.setattr(rmain, "get_model", lambda weights: _Stub())
    np.random.seed(0)
    rmain.main(["--mode", "test"], log_root=str(tmp_path / "exp"), data_root=data_dir)
    rmain.main(["--mode", "test"], log_root=str(tmp_path / "exp"), data_root=str(tmp_path / "absent"))
    assert seen == ["Human36M", "SyntheticPoses"]


class _Stub:
    def cuda(self):
        return self

    def apply(self, fn):
        return self

    def parameters(self):
        import torch
        return [torch.zeros(1, requires_grad=True)]


def _harness(tmp_path_factory, sanitize):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / ("host_pose_eval" + ("_san" if sanitize else "")))
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1", "-std=c++17"]
    if sanitize:
        cmd += ["-Xcompiler", "-fsanitize=address", "-Xcompiler", "-fsanitize=undefined",
                "-Xcompiler", "-fno-sanitize-recover=all", "-lasan", "-lubsan"]
    r = subprocess.run(cmd + ["-o", exe, os.path.join(ROOT, "tests", "harness", "host_pose_eval.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0")

    def errors(pred, gt, mask):
        S, J = pred.shape[:2]
        out = subprocess.run([exe, "errors", str(S), str(J), str(mask)], env=env, capture_output=True,
                             input=np.concatenate([pred.ravel(), gt.ravel()]).astype(np.float64).tobytes())
        assert out.returncode == 0, out.stderr
        a = np.frombuffer(out.stdout, np.float64)
        return a[:S * 7].reshape(S, 7), a[S * 7:].reshape(S, J)

    def camera(joints, cam, root):
        N, J = joints.shape[:2]
        out = subprocess.run([exe, "camera", str(N), str(J), str(root)], env=env, capture_output=True,
                             input=np.concatenate([joints.ravel(), cam.ravel()]).astype(np.float64).tobytes())
        assert out.returncode == 0, out.stderr
        return np.frombuffer(out.stdout, np.float64).reshape(N, J, 3)
    return errors, camera


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    return _harness(tmp_path_factory, False)


MASK = sum(1 << j for j in rc.J14)


def _cases():
    rng = np.random.default_rng(3)
    gt = rc.poses(rng, 64, 15)
    pred = gt + rng.normal(0, 30, gt.shape)
    pred[1] = gt[1]                                          # exact
    pred[2] = 1.7 * gt[2] @ np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1.]]) + 5.0   # similar
    pred[3] = gt[3] @ np.diag([1, 1, -1.])                   # a reflection
    return pred, gt


def test_pose_errors_body_vs_restatement(host):
    pred, gt = _cases()
    m, pj = host[0](pred, gt, MASK)
    rm, rpj = rc.pose_errors(pred, gt)
    assert np.max(np.abs(m - rm)) <= 1e-9 and np.max(np.abs(pj - rpj)) <= 1e-9
    assert m[1, [0, 2, 4, 5, 6]].max() == 0.0 and m[1, [1, 3]].max() <= 1e-9 and m[2, 1] <= 1e-9


def test_pose_errors_degenerate_poses(host):
    """All joints equal (zero spread: alignment divides 0 by 0) and collinear joints (rank-1
    covariance): the plain errors stay exact and finite."""
    rng = np.random.default_rng(4)
    gt = rc.poses(rng, 2, 15)
    pred = np.zeros_like(gt)
    pred[0] = 12.5                                           # all joints equal
    t = np.linspace(-1, 1, 15)[:, None]
    pred[1] = t * np.array([[100.0, 50.0, -20.0]])           # collinear
    m, pj = host[0](pred, gt, MASK)
    rm, rpj = rc.pose_errors(pred[1:], gt[1:])
    assert np.array_equal(pj, np.linalg.norm(gt - pred, axis=2))
    assert np.all(np.isfinite(m[1])) and np.max(np.abs(m[1] - rm[0])) <= 1e-9
    assert np.all(np.isfinite(m[0, [0, 2, 4, 5, 6]]))


def test_pose_to_camera_body_vs_restatement(host):
    rng = np.random.default_rng(5)
    N, J = 32, 16
    joints = np.stack([rng.uniform(200, 800, (N, J)), rng.uniform(100, 900, (N, J)),
                       rng.normal(0, 200, (N, J))], axis=2)
    cam = np.stack([rng.uniform(1100, 1200, N), rng.uniform(1100, 1200, N), rng.uniform(500, 520, N),
                    rng.uniform(500, 520, N), rng.uniform(3000, 6000, N)], axis=1)
    out = host[1](joints, cam, 6)
    assert np.max(np.abs(out - rc.pose_to_camera(joints, cam, 6))) <= 1e-9
    assert np.all(out[:, 6] == 0.0)


def test_bodies_under_address_and_ub_sanitizers(tmp_path_factory):
    errors, camera = _harness(tmp_path_factory, True)
    pred, gt = _cases()
    pred[5] = 0.0
    m, _ = errors(pred, gt, MASK)
    rm, _ = rc.pose_errors(np.delete(pred, 5, 0), np.delete(gt, 5, 0))
    assert np.max(np.abs(np.delete(m, 5, 0) - rm)) <= 1e-9
    rng = np.random.default_rng(6)
    joints = rng.uniform(0, 500, (4, 32, 3))
    cam = np.tile([1150.0, 1150.0, 512.0, 512.0, 4500.0], (4, 1))
    assert np.max(np.abs(camera(joints, cam, 31) - rc.pose_to_camera(joints, cam, 31))) <= 1e-9


# ------------------------------------------------------------------ H36M evaluation and export
def test_refiner_config_keys_and_refusals():
    import types
    from lib.core.config import config
    from lib.core.refine import check_refiner_config
    assert config.TEST.REFINER == '' and config.TEST.REFINER_NORM == ''
    T = types.SimpleNamespace
    assert check_refiner_config(T(REFINER='', REFINER_NORM=''), False, 17) is None
    assert check_refiner_config(T(REFINER='r.pth', REFINER_NORM='n.pkl'), True, 16) == ('r.pth', 'n.pkl')
    with pytest.raises(ValueError, match="REFINER_NORM"):
        check_refiner_config(T(REFINER='r.pth', REFINER_NORM=''), True, 16)
    with pytest.raises(ValueError, match="MPII"):
        check_refiner_config(T(REFINER='r.pth', REFINER_NORM='n.pkl'), False, 16)
    with pytest.raises(ValueError, match="17 joints"):
        check_refiner_config(T(REFINER='r.pth', REFINER_NORM='n.pkl'), True, 17)


@pytest.fixture
def emulated_eval():
    import lib.dataset.h36m_eval as he
    from tests import emul_ops
    from epipolarpose_b200 import ops
    he._backend[0] = emul_ops
    yield he
    he._backend[0] = ops


def _fixture_h36m(mpii, refiner='', norm=''):
    import types
    import lib.dataset as dataset
    from tests import dataset_cases as dc
    cfg = dc.cfg(MPII_ORDER=mpii)
    cfg.TEST = types.SimpleNamespace(PSS_K=[], PSS_CENTROIDS='', REFINER=refiner, REFINER_NORM=norm)
    dc.seeded(dc.SEED % 1000)
    return dataset.h36m(cfg, dc.H36M_ROOT, "valid", False)


def test_evaluate_refuses_and_skips(golden, emulated_eval, monkeypatch):
    """TEST.REFINER with H36M order is refused before any work; with REFINER empty the nine
    protocol entries come back and no refinement call is made."""
    import importlib
    h36m = importlib.import_module("lib.dataset.h36m")        # the package exports the class as `h36m`
    g = golden("datasets")
    ds = _fixture_h36m(False, 'r.pth', 'n.pkl')
    with pytest.raises(ValueError, match="MPII"):
        ds.evaluate(g["h36m_eval_h36m/preds"].copy(), None)
    monkeypatch.setattr(h36m, "h36m_refined", lambda *a, **k: pytest.fail("refined with TEST.REFINER empty"))
    nv, _ = _fixture_h36m(True).evaluate(g["h36m_eval_mpii/preds"].copy(), None)
    assert len(nv) == 9


def test_export_refiner_pairs_round_trips_through_human36m(golden, emulated_eval, tmp_path):
    from lib.core.function import export_refiner_pairs
    from refiner import data
    g = golden("datasets")
    preds = g["h36m_eval_mpii/preds"].copy()
    ds = _fixture_h36m(True)
    for name in ("train.pkl", "valid.pkl"):
        assert export_refiner_pairs(preds, ds, str(tmp_path / name)) == len(preds)
    with open(tmp_path / "valid.pkl", "rb") as f:
        pairs = pickle.load(f)
    S = len(preds)
    gts = ds.db[:S]
    get = lambda k: np.stack([np.asarray(r[k], dtype=np.float64).reshape(-1) for r in gts])
    _, _, det = emulated_eval.evaluate_h36m(preds[:, :, :3], np.stack([r['joints_3d'] for r in gts]), get('pelvis'),
                                            get('fl'), get('c_p'), mpii_order=True, return_poses=True)
    assert pairs['inp'].dtype == np.float32 and pairs['inp'].shape == (S, 16, 3)
    assert np.array_equal(pairs['inp'], det['poses'][:, :, 0:3].astype(np.float32))
    assert np.array_equal(pairs['out'], det['poses'][:, :, 6:9].astype(np.float32))
    assert np.all(pairs['inp'][:, 6] == 0) and np.all(pairs['out'][:, 6] == 0)
    data.Human36M(is_train=True, root=str(tmp_path))
    va = data.Human36M(is_train=False, root=str(tmp_path))
    keep = [j for j in range(16) if j != 6]
    assert np.array_equal(va.labels, pairs['out'][:, keep].reshape(S, 45))
    with pytest.raises(ValueError):
        export_refiner_pairs(preds, _fixture_h36m(False), str(tmp_path / "x.pkl"))
