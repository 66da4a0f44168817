"""CPU: pseudo-label records for self-supervised Human3.6M training.  The per-(frame, camera) body
of pseudo_records_kernel (csrc/camera.cuh cam_pseudo_record) run on the CPU by
tests/harness/host_pseudo_records.cu against the numpy restatement (tests/pseudo_cases.py), the
argument checks of epb_pseudo_records, and the host logic of lib/utils/prep_h36m.save_triangulations
on the fixture tree with the network bypassed and the C ABI emulated."""
import os
import pickle
import shutil
import subprocess

import numpy as np
import pytest
import torch

from tests import pseudo_cases as pc
from tests.conftest import ROOT


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    """tests/harness/host_pseudo_records.cu: cam_pseudo_record and the entry's checks, built for the CPU."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / "host_pseudo_records")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1", "-std=c++17",
                        "-o", exe, os.path.join(ROOT, "tests", "harness", "host_pseudo_records.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def records(X, status, cam, root):
        T, S, J = X.shape[:3]
        V = cam.shape[1]
        inp = (np.ascontiguousarray(X, np.float64).tobytes() + np.ascontiguousarray(status, np.int32).tobytes()
               + np.ascontiguousarray(cam, np.float64).tobytes())
        out = subprocess.run([exe, "records", str(T), str(S), str(V), str(J), str(root)], input=inp,
                             capture_output=True)
        assert out.returncode == 0, out.stderr
        a = np.frombuffer(out.stdout, dtype=np.float64)
        n = T * V * J * 3
        assert a.size == 2 * n + T * V * 4
        return (a[:n].reshape(T, V, J, 3), a[n:2 * n].reshape(T, V, J, 3), a[2 * n:2 * n + T * V * 3].reshape(T, V, 3),
                a[2 * n + T * V * 3:].reshape(T, V).astype(np.int32))

    def args(T, S, V, J, root):
        out = subprocess.run([exe, "args", str(T), str(S), str(V), str(J), str(root)], capture_output=True, text=True)
        assert out.returncode == 0, (out.returncode, out.stderr)
        return int(out.stdout)
    return records, args


@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("V", [2, 4, 8])
@pytest.mark.parametrize("per_camera", [False, True])
def test_kernel_body_on_host_vs_restatement(harness, V, J, per_camera):
    records, _ = harness
    S = V if per_camera else 1
    root = 6 if J == 16 else 0
    X, st, cam = pc.case(100 * V + J + S, 9, S, V, J, root)
    got, want = records(X, st, cam, root), pc.restated(X, st, cam, root)
    pc.assert_same(got, want)
    jt, vis, pel, ok = got
    # what the planted cases must show
    assert ok[0].all() and not ok[1].any()
    assert not vis[1].any() and not jt[1].any() and not pel[1].any()         # root failed: all rows 0
    assert vis[2, 0, (root + 1) % J].sum() == 0                               # behind camera 0
    assert vis[3, 0, (root + 2) % J].sum() == 0                               # on camera 0's centre
    assert not vis[4, :, (root + 3) % J].any()                                # status -1
    s_of = lambda v: 0 if S == 1 else v
    for t in (0, 5, 6):
        for v in range(V):
            assert np.array_equal(vis[t, v, :, 0] == 1, st[t, s_of(v)] == 1)
    assert np.array_equal(vis[..., 0], vis[..., 1]) and np.array_equal(vis[..., 0], vis[..., 2])
    assert np.all(jt[ok == 1][:, root, 2] == 0)                               # the root's relative depth


def test_one_pose_per_frame_equals_it_repeated_per_camera(harness):
    records, _ = harness
    X, st, cam = pc.case(7, 5, 1, 4, 17)
    a = records(X, st, cam, 0)
    b = records(np.repeat(X, 4, axis=1), np.repeat(st, 4, axis=1), cam, 0)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_world_ground_truth_round_trips_through_the_records(harness):
    """world_joints_of_record of the fixture's validation records, projected again: the records."""
    from tests import dataset_cases as dc
    from lib.core.function import world_joints_of_record
    from lib.utils.prep_h36m import _cam16
    records, _ = harness
    ds = dc.build("h36m_valid")
    tups = [ds.tuple_records(r) for r in ds.view_tuples()]
    X = np.stack([np.mean([world_joints_of_record(r) for r in tup], axis=0) for tup in tups])[:, None]
    cam = np.stack([np.stack([_cam16(r) for r in tup]) for tup in tups])
    jt, vis, pel, ok = records(X, np.ones(X.shape[:3], np.int32), cam, 0)
    assert ok.all() and vis.all()
    for t, tup in enumerate(tups):
        for v, r in enumerate(tup):
            assert np.max(np.abs(jt[t, v] - r["joints_3d"])) <= 1e-6
            assert np.max(np.abs(pel[t, v] - r["pelvis"])) <= 1e-6


def test_argument_checks(harness):
    _, args = harness
    assert args(0, 1, 4, 17, 0) == 0                     # T = 0: returns before any launch
    assert args(0, 4, 4, 17, 16) == 0
    assert args(5, 1, 4, 17, 0) == 0 and args(5, 8, 8, 16, 6) == 0
    for bad in ((-1, 1, 4, 17, 0), (5, -1, 4, 17, 0), (5, 1, 4, -1, 0), (5, 1, -4, 17, 0),
                (5, 2, 4, 17, 0), (5, 0, 4, 17, 0), (5, 3, 4, 17, 0),       # S not in {1, V}
                (5, 1, 1, 17, 0), (5, 1, 9, 17, 0), (5, 9, 9, 17, 0),       # V outside 2..8
                (5, 1, 4, 17, 17), (5, 1, 4, 17, -1), (5, 1, 4, 0, 0),      # root outside [0, J)
                (16000000, 1, 8, 17, 0), (0, 1, 4, 17, 17)):                # T*V*J > 2^31-1; T = 0 checked too
        assert args(*bad) == -1, bad


# ------------------------------------------------------------------ save_triangulations, emulated
@pytest.fixture
def emulated(monkeypatch):
    """The builder with the C ABI emulated and the image batch replaced by zeros (no device)."""
    import lib.utils.prep_h36m as prep
    monkeypatch.setattr(prep, "_backend", [pc.Emulated])
    monkeypatch.setattr(prep, "_assemble", lambda batch, dev: torch.zeros((len(batch["jpeg"]), 3, 64, 64)))
    return prep


def _gt_predictor(anno, fail=(), J_out=None, perm=None):
    """MultiViewPredictor's interface; the world pose of frame k is the ground truth of the source
    records (world_joints_of_record averaged over the views); frames in `fail` have a failed root."""
    from lib.core.function import world_joints_of_record
    V = len(anno)
    seen = []

    def predictor(images, boxes, P):
        T = images.shape[0]
        assert tuple(images.shape[1:3]) == (V, 3) and P.shape == (T, V, 3, 4)
        assert boxes["center_x"].shape == (T * V,) and np.all(boxes["scale"] == 1)
        ks = range(len(seen), len(seen) + T)
        for i, k in enumerate(ks):
            assert boxes["center_x"][i * V] == anno[1][k]["center_x"]            # tuple-major views
            assert np.array_equal(P[i, V - 1], np.asarray(anno[V][k]["cam"].projection_matrix)[:3])
        seen.extend(ks)
        W = np.stack([np.mean([world_joints_of_record(anno[c + 1][k]) for c in range(V)], axis=0) for k in ks])
        if perm is not None:
            W = W[:, perm]
        st = np.ones(W.shape[:2], np.int32)
        root = 6 if perm is not None else 0
        for i, k in enumerate(ks):
            if k in fail:
                st[i, root] = 0
        return {"world": W * st[..., None], "status": st, "inliers": st * ((1 << V) - 1),
                "resid": np.zeros(st.shape), "kps": None}
    predictor.seen = seen
    return predictor


def _source(tmp_path, n_frames=7):
    """The fixture's validation pickle with its frames repeated to n_frames (distinct centres)."""
    from tests import dataset_cases as dc
    from lib.dataset.JointIntegralDataset import load_pickle
    anno = load_pickle(os.path.join(dc.H36M_ROOT, "annot", "valid.pkl"))
    out = {c: [] for c in anno}
    for k in range(n_frames):
        for c in anno:
            r = dict(anno[c][k % len(anno[c])])
            r["center_x"] = float(r["center_x"]) + k * 1e-3
            out[c].append(r)
    p = str(tmp_path / "src.pkl")
    with open(p, "wb") as f:
        pickle.dump(out, f, protocol=4)
    return p, out


def test_builder_keeps_order_and_drops_aligned(emulated, tmp_path):
    from tests import dataset_cases as dc
    from lib.dataset.JointIntegralDataset import load_pickle
    src, anno = _source(tmp_path)
    ds = dc.build("h36m_valid")
    pred = _gt_predictor(anno, fail={2, 5})
    rep = emulated.save_triangulations(None, ds, src, str(tmp_path / "out" / "dst.pkl"), tuples_per_batch=3,
                                       workers=2, predictor=pred)
    assert pred.seen == list(range(7))
    assert rep["frames"] == 5 and rep["dropped"] == 2
    assert rep["failed"] == pytest.approx(2 / (7 * 17)) and rep["agreement_mm"] < 1e-6
    assert rep["inlier_views"] == pytest.approx(4 * (1 - 2 / (7 * 17)))
    out = load_pickle(str(tmp_path / "out" / "dst.pkl"))
    assert sorted(out) == [1, 2, 3, 4]
    kept = [0, 1, 3, 4, 6]
    for c in out:
        assert len(out[c]) == 5
        for r, k in zip(out[c], kept):
            s = anno[c][k]
            assert r["center_x"] == s["center_x"] and r["image"] == s["image"]
            assert set(r) == set(s) and r["flip_pairs"] == s["flip_pairs"]
            assert np.array_equal(r["parent_ids"], s["parent_ids"])
            assert np.max(np.abs(r["joints_3d"] - s["joints_3d"])) <= 1e-6
            assert np.max(np.abs(r["pelvis"] - s["pelvis"])) <= 1e-6
            assert np.all(r["joints_3d_vis"] == 1)
    assert ds.is_train is False and len(ds.db) == 12          # the dataset is left as it was


def test_builder_writes_mpii_order_from_17_joints(emulated, tmp_path):
    from tests import dataset_cases as dc
    from lib.dataset.h36m_eval import H36M_TO_MPII_PERM, H36M_NAMES, MPII_NAMES
    from lib.dataset.JointIntegralDataset import load_pickle
    src, anno = _source(tmp_path, 3)
    ds = dc.build("h36m_valid")
    pred = _gt_predictor(anno, perm=H36M_TO_MPII_PERM)
    emulated.save_triangulations(None, ds, src, str(tmp_path / "dst.pkl"), workers=1, predictor=pred)
    out = load_pickle(str(tmp_path / "dst.pkl"))
    r, s = out[2][1], anno[2][1]
    assert r["joints_3d"].shape == (16, 3)
    assert np.max(np.abs(r["joints_3d"] - s["joints_3d"][H36M_TO_MPII_PERM])) <= 1e-6
    assert np.max(np.abs(r["pelvis"] - s["pelvis"])) <= 1e-6
    name = lambda i: MPII_NAMES[i]
    pairs = {frozenset((name(a), name(b))) for a, b in r["flip_pairs"]}
    assert pairs == {frozenset((H36M_NAMES[a], H36M_NAMES[b])) for a, b in s["flip_pairs"]}
    assert len(r["parent_ids"]) == 16
    for i in range(16):
        assert name(int(r["parent_ids"][i])) == H36M_NAMES[int(s["parent_ids"][H36M_TO_MPII_PERM[i]])]
    assert "Spine" not in {name(i) for p in r["flip_pairs"] for i in p}


def test_joint_layout_refusals():
    from lib.utils.prep_h36m import joint_layout
    pairs, parents = [[1, 4]], np.zeros(17, np.int64)
    assert joint_layout(17, 17, pairs, parents)[:2] == (None, 0)
    assert joint_layout(16, 16, pairs, parents)[:2] == (None, 6)
    for J, Js in ((15, 17), (17, 16), (16, 18)):
        with pytest.raises(ValueError, match="joints"):
            joint_layout(J, Js, pairs, parents)


def test_builder_refuses_list_form_and_unknown_methods(emulated, tmp_path):
    from tests import dataset_cases as dc
    ds = dc.build("h36m_valid")
    with pytest.raises(ValueError, match="dict-form"):
        emulated.save_triangulations(None, ds, os.path.join(dc.H36M_ROOT, "annot", "train-fs.pkl"),
                                     str(tmp_path / "x.pkl"), predictor=lambda *a: None)
    with pytest.raises(ValueError, match="method"):
        emulated.save_triangulations(None, ds, {1: [], 2: []}, str(tmp_path / "x.pkl"), method="dlt",
                                     predictor=lambda *a: None)
    bad = dc.build("h36m_valid")
    bad.cam_config = [[1], [0]]
    _, anno = _source(tmp_path, 2)
    with pytest.raises(ValueError, match="cam_config"):
        emulated.save_triangulations(None, bad, anno, str(tmp_path / "x.pkl"), method="iterative",
                                     predictor=lambda *a: None)
    assert not os.path.exists(str(tmp_path / "x.pkl"))
