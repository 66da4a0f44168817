"""CPU: online labels of whole camera tuples (epb_tuple_labels).  The label body shared by
project_labels_kernel and tuple_label_kernel, and the entry's per-(tuple, joint) and per-(row,
joint) bodies, built for the CPU by tests/harness/host_tuple_labels.cu, against the numpy
restatement (tests/tuple_label_cases.py); robust V = 4 labels against the pair path on tuples with
planted outliers; the TRI_VIEWS dataset items and their camera draws; the configuration refusals;
the view-major loader batch and synthetic sampler."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import restate
from tests import dataset_cases as dc
from tests import tuple_label_cases as tc
from tests.conftest import ROOT


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    """tests/harness/host_tuple_labels.cu: the epb_tuple_labels bodies of csrc/geometry.cu on the CPU."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / "host_tuple_labels")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1", "-std=c++17",
                        "-o", exe, os.path.join(ROOT, "tests", "harness", "host_tuple_labels.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(args, arrays):
        inp = b"".join(np.ascontiguousarray(a, dtype=np.float64).tobytes() for a in arrays)
        out = subprocess.run([exe] + [str(a) for a in args], input=inp, capture_output=True)
        assert out.returncode == 0, out.stderr
        a = np.frombuffer(out.stdout, dtype=np.float64)
        assert np.isfinite(a).all(), "a non-finite value left the kernel body"
        return a

    def tuple_labels(coords, lse, meta, V, thr=15.0):
        B, J = coords.shape[0], coords.shape[1] // 3
        T = B // V
        box, P, cam = tc.packed(meta)
        a = run(["tuple", T, V, J, repr(float(thr)), int(lse is not None)],
                [coords, box, P, cam] + ([lse] if lse is not None else []))
        n = B * J * 3
        label, weight, rest = a[:n].reshape(B, J * 3), a[n:2 * n].reshape(B, J * 3), a[2 * n:]
        X = rest[:T * J * 3].reshape(T, J, 3)
        inl, res, st = (rest[T * J * (3 + k):T * J * (4 + k)].reshape(T, J) for k in range(3))
        return label, weight, X, st.astype(np.int32), inl.astype(np.int32), res

    def project(X, meta):
        B, J = X.shape[0], X.shape[1]
        box, _, cam = tc.packed(meta)
        a = run(["project", B, J], [X, cam, box])
        return a[:B * J * 3].reshape(B, J * 3), a[B * J * 3:B * J * 4].reshape(B, J), a[B * J * 4:].reshape(B, J)

    run.tuple_labels, run.project = tuple_labels, project
    return run


def _same(got, want, xtol=1e-4):
    label, weight, X, st, inl, res = got
    lo, wo, Xo, so, io, ro = want
    assert np.array_equal(st, so) and np.array_equal(inl, io)
    assert np.array_equal(weight, wo)
    assert np.max(np.abs(X - Xo)) <= xtol, np.max(np.abs(X - Xo))
    assert np.max(np.abs(res - ro)) <= 1e-6
    assert np.max(np.abs(label - lo)) <= 1e-6, np.max(np.abs(label - lo))


def test_shared_label_body_is_the_reference_projection(host):
    """project_label_point (the body project_labels_kernel now calls) against the oracle's
    labels_from_global_coords, which the reference goldens pin; the depths it returns are the
    camera-frame depths of the joint and the root."""
    coords, _, meta, Xw, _ = tc.case(3, 6, 4, 17)
    B = len(coords)
    X = Xw[np.arange(B) % 6]
    label, cz, pz = host.project(X, meta)
    ref, _ = restate.labels_from_global_coords(X, meta)
    assert np.max(np.abs(label - ref)) <= 1e-6
    Xc = np.einsum("bij,bkj->bki", meta["R"], X - meta["T"].reshape(B, 1, 3))
    assert np.max(np.abs(cz - Xc[:, :, 2])) <= 1e-9 and np.max(np.abs(pz - Xc[:, :1, 2])) <= 1e-9


@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("V", [2, 3, 4, 8])
def test_entry_bodies_on_host_vs_restatement(host, V, J):
    """3 px noise; with and without confidences; a quarter of the joints with one 80 px outlier view"""
    for k, (outl, lse) in enumerate([(0.0, False), (0.0, True), (0.25, False), (0.25, True)]):
        coords, ls, meta, _, _ = tc.case(10 * V + J + k, 5, V, J, outliers=outl, lse=lse)
        _same(host.tuple_labels(coords, ls, meta, V), tc.tuple_labels(coords, ls, meta, V))


def test_weight_rule_failed_root_and_behind_camera(host):
    """a tuple whose root fails contributes nothing; a joint behind one camera has weight 0 in that
    view only; the other rows are untouched"""
    V, J, T = 4, 17, 3
    coords, _, meta, _, _ = tc.case(5, T, V, J)
    coords = coords.reshape(V * T, J, 3)
    coords[[v * T + 1 for v in range(V - 1)], 0, :2] = np.nan           # root of tuple 1 in 3 of 4 views
    coords = coords.reshape(V * T, J * 3)
    meta = dict(meta)
    meta["T"] = meta["T"].copy()
    got = host.tuple_labels(coords, None, meta, V)
    _same(got, tc.tuple_labels(coords, None, meta, V))
    label, weight, X, st = got[:4]
    assert st[1, 0] == 0 and st[1, 1:].all()
    rows1 = [v * T + 1 for v in range(V)]
    assert not weight[rows1].any() and not label[rows1].any()
    others = [r for r in range(V * T) if r not in rows1]
    assert weight[others].all()
    # move camera 2 of tuple 0 to the far side of the subject: everything is behind it
    r = 2 * T + 0
    meta["R"] = meta["R"].copy()
    meta["R"][r] = -meta["R"][r]
    got = host.tuple_labels(coords, None, meta, V)
    assert not got[1][r].any() and not got[0][r].any()
    _same(got, tc.tuple_labels(coords, None, meta, V))


def test_robust_v4_labels_beat_the_pair_path_on_outliers(host):
    """Ring-camera tuples, 3 px noise, one 80 px outlier view in a quarter of the joints: the median
    3-D error of the robust V = 4 result on the affected joints is below that of the pair path
    (iterative, views (0,3) and (1,2) triangulated on their own), in every view's labels."""
    V, J, T = 4, 17, 48
    coords, _, meta, Xw, hit = tc.case(77, T, V, J, outliers=0.25)
    X = host.tuple_labels(coords, None, meta, V)[2]
    e_rob = np.linalg.norm(X - Xw, axis=2)[hit]
    u = tc.image_points(coords, meta)
    P = np.asarray(meta["projection_matrix"])[:, :3, :4]
    e_pair = []
    for a, b in ((0, 3), (1, 2)):
        Xp = np.stack([restate.iterative_LS_triangulation(u[a * T + t], P[a * T + t], u[b * T + t], P[b * T + t])[0]
                       for t in range(T)])
        e_pair.append(np.linalg.norm(Xp - Xw, axis=2)[hit])
    e_pair = np.concatenate(e_pair)
    print("outlier joints: robust median %.1f mm, pair median %.1f mm" % (np.median(e_rob), np.median(e_pair)))
    assert np.median(e_rob) < np.median(e_pair)


# ------------------------------------------------------------------ dataset and configuration
def _tri_ds(views):
    import lib.dataset as dataset
    dc.seeded(dc.SEED % 1000)
    _, _, _, zw = dc.H36M_CASES["h36m_ss_tri"]
    return dataset.h36m(dc.cfg(TRI=True, TRI_VIEWS=views, Z_WEIGHT=zw), dc.H36M_ROOT, "train-ss", True)


def _frame_cam(path):
    frame, cam = os.path.basename(path).rsplit("_c", 1)
    return frame, int(cam.split(".")[0])


def test_tri_views_items_are_distinct_cameras_of_one_frame(monkeypatch):
    """TRI_VIEWS = 4 (= NUM_CAMS): every camera in camera order, of the same frame index, with no
    camera draw; in a worker the views are deferred samples of those records."""
    ds = _tri_ds(4)
    calls = []
    monkeypatch.setattr(ds, "get_data", lambda rec: calls.append(rec["image"]) or rec["image"])
    for idx in range(len(ds)):
        np.random.seed(idx)
        before = np.random.get_state()
        item = ds[idx]
        after = np.random.get_state()
        assert np.array_equal(after[1], before[1]) and after[2] == before[2]
        assert list(item) == ["cam_%d" % (k + 1) for k in range(4)]
        fc = [_frame_cam(item[k]) for k in item]
        assert len({f for f, _ in fc}) == 1 and [c for _, c in fc] == [1, 2, 3, 4]
        assert [item["cam_%d" % (c + 1)] for c in range(4)] == [r["image"] for r in ds.tuple_records(
            ds.view_tuples()[idx])]


def test_tri_views_deferred_items_in_a_worker(monkeypatch):
    import lib.dataset.JointIntegralDataset as jid
    from lib.dataset import deferred
    from torch.utils.data import default_collate
    monkeypatch.setattr(jid, "get_worker_info", lambda: object())
    ds = _tri_ds(4)
    items = [ds[i] for i in range(min(3, len(ds)))]
    for it in items:
        fc = [_frame_cam(it["cam_%d" % (k + 1)]["meta"]["image"]) for k in range(4)]
        assert len({f for f, _ in fc}) == 1 and sorted(c for _, c in fc) == [1, 2, 3, 4]
    batch = default_collate(items)
    assert deferred.is_deferred(batch) and deferred.view_keys(batch) == ["cam_1", "cam_2", "cam_3", "cam_4"]


def test_tri_views_3_draw_order_is_pinned(monkeypatch):
    """2 < V < NUM_CAMS: np.random.choice(NUM_CAMS, V, replace=False), sorted, and nothing else"""
    ds = _tri_ds(3)
    monkeypatch.setattr(ds, "get_data", lambda rec: rec["image"])
    for idx in range(len(ds)):
        np.random.seed(100 + idx)
        item = ds[idx]
        after = np.random.get_state()[1].copy()
        np.random.seed(100 + idx)
        want = sorted(np.random.choice(4, 3, replace=False))
        assert np.array_equal(np.random.get_state()[1], after)
        assert list(item) == ["cam_1", "cam_2", "cam_3"]
        fc = [_frame_cam(item[k]) for k in item]
        assert len({f for f, _ in fc}) == 1 and [c - 1 for _, c in fc] == want


def test_tri_views_2_keeps_the_reference_pair_draw(monkeypatch):
    ds = _tri_ds(2)
    monkeypatch.setattr(ds, "get_data", lambda rec: rec["image"])
    import random
    for idx in range(len(ds)):
        dc.seeded(idx)
        item = ds[idx]
        dc.seeded(idx)
        c1 = np.random.randint(4)
        c2 = ds.cam_config[c1][0] if random.random() <= 0.5 else ds.cam_config[c1][1]
        assert list(item) == ["cam_1", "cam_2"]
        assert [_frame_cam(item[k])[1] - 1 for k in item] == [c1, c2]


def test_tri_views_refuses_list_form_pickles():
    import lib.dataset as dataset
    dc.seeded(1)
    with pytest.raises(ValueError, match="dict-form"):
        dataset.h36m(dc.cfg(TRI=True, TRI_VIEWS=4), dc.H36M_ROOT, "train-fs", True)


def _cfg(**kw):
    from lib.core.config import AttrDict, _DEFAULTS
    c = AttrDict(_DEFAULTS)
    for k, v in kw.items():
        sec, key = k.split("__")
        c[sec][key] = v
    return c


def test_config_refusals():
    from lib.core.config import check_config, tuple_settings
    assert tuple_settings(_cfg()) == (2, None, 15.0)
    assert tuple_settings(_cfg(DATASET__TRI_VIEWS=4, TRAIN__ONLINE_TRIANGULATION=True,
                               TRAIN__TRIANGULATION_METHOD="robust")) == (4, "robust", 15.0)
    bad = [dict(TRAIN__ONLINE_TRIANGULATION=True, TRAIN__TRIANGULATION_METHOD="robust", TRAIN__ESTIMATE_EXTRINSICS=True),
           dict(DATASET__TRI_VIEWS=4, TRAIN__ONLINE_TRIANGULATION=True),
           dict(DATASET__TRI_VIEWS=3, TRAIN__ONLINE_TRIANGULATION=True, TRAIN__TRIANGULATION_METHOD="polynomial"),
           dict(DATASET__TRI_VIEWS=5),
           dict(DATASET__TRI_VIEWS=1),
           dict(DATASET__TRI_VIEWS=9, DATASET__NUM_CAMS=12),
           dict(TRAIN__ONLINE_TRIANGULATION=True, TRAIN__TRIANGULATION_METHOD="robust", TRAIN__ROBUST_THRESHOLD_PX=0.0)]
    for kw in bad:
        with pytest.raises(ValueError):
            check_config(_cfg(**kw))
    check_config(_cfg(DATASET__TRI_VIEWS=8, DATASET__NUM_CAMS=8, TRAIN__ONLINE_TRIANGULATION=True,
                      TRAIN__TRIANGULATION_METHOD="robust"))


def test_config_yaml_and_training_entry_refuse(tmp_path):
    import lib.core.config as C
    import lib.core.function as fn
    y = tmp_path / "x.yaml"
    y.write_text("DATASET:\n  TRI_VIEWS: 4\nTRAIN:\n  ONLINE_TRIANGULATION: true\n")
    try:
        with pytest.raises(ValueError, match="robust"):
            C.update_config(str(y))
    finally:
        C.reset_config()
    with pytest.raises(ValueError):
        fn.train_integral(_cfg(DATASET__TRI_VIEWS=3, TRAIN__ONLINE_TRIANGULATION=True), [], torch.nn.Linear(1, 1),
                          None, None, 0)
    with pytest.raises(ValueError):
        fn.GraphedTrainStep(None, None, None, online=True, method="robust", estimate_extrinsics=True)
    with pytest.raises(ValueError):
        fn.GraphedTrainStep(None, None, None, online=True, method="iterative", views=4)


# ------------------------------------------------------------------ batch layout
def test_loader_batch_is_view_major_and_pairs_unchanged():
    from lib.core.function import loader_batch
    g = torch.Generator().manual_seed(0)

    def view(n, tag):
        return (torch.randn(n, 3, 4, 4, generator=g), torch.randn(n, 6, generator=g), torch.ones(n, 6),
                {"center_x": torch.full((n,), float(tag), dtype=torch.float64), "image": ["%d" % tag] * n})
    views = {"cam_%d" % (k + 1): view(3, k) for k in range(4)}
    x, lab, w, meta = loader_batch(views)
    assert torch.equal(x, torch.cat([views["cam_%d" % (k + 1)][0] for k in range(4)]))
    assert meta["center_x"].tolist() == [float(k) for k in range(4) for _ in range(3)]
    assert meta["image"] == [str(k) for k in range(4) for _ in range(3)]
    two = {k: views[k] for k in ("cam_1", "cam_2")}
    a, b = two["cam_1"], two["cam_2"]
    x2, l2, _, m2 = loader_batch(two)
    assert torch.equal(x2, torch.cat([a[0], b[0]])) and torch.equal(l2, torch.cat([a[1], b[1]]))
    assert torch.equal(m2["center_x"], torch.cat([a[3]["center_x"], b[3]["center_x"]]))


def test_synthetic_tuple_batch_sampler_is_view_major():
    from lib.dataset.synthetic import SyntheticH36M
    from lib.core.config import AttrDict, _DEFAULTS
    c = AttrDict(_DEFAULTS)
    c.MODEL.NUM_JOINTS, c.DATASET.SYNTHETIC_LEN = 16, 48
    ds = SyntheticH36M(c)
    batches = list(ds.tuple_batch_sampler(3))
    assert len(batches) == 4
    for b, idx in enumerate(batches):
        for v in range(4):
            for t in range(3):
                rec = ds.db[idx[v * 3 + t]]
                assert rec["tuple"] == 3 * b + t and rec["view"] == v
    assert list(ds.tuple_batch_sampler(2, views=3))[0] == [0, 4, 1, 5, 2, 6]
