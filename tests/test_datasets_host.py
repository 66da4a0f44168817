"""CPU: the h36m / mpii_integral dataset classes against what the unmodified reference classes
made of the fixture tree (tests/golden/make_golden_datasets.py): db order and records, the
evaluation protocols, deferred samples (what a DataLoader worker returns) and the annotation
pickles under both import names of the package."""
import os

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader, default_collate

from tests import dataset_cases as dc
from tests import emul_ops

CASES = list(dc.H36M_CASES) + list(dc.MPII_CASES)


@pytest.fixture(scope="module")
def g(golden):
    return golden("datasets")


@pytest.fixture
def in_worker(monkeypatch):
    """Index datasets as a DataLoader worker does."""
    import lib.dataset.JointIntegralDataset as jid
    monkeypatch.setattr(jid, "get_worker_info", lambda: object())


def _flat(db):
    return [r for d in db for r in d] if db and isinstance(db[0], list) else db


@pytest.mark.parametrize("case", CASES)
def test_db_parity(g, case):
    """Same length, order and records as the reference for the same seeds: both annotation
    forms, TRI's per-camera lists, train / valid, and the MPII json rules (0-based joints, the
    1-visible-joint record skipped, the 1.25 aspect-ratio box)."""
    ds = dc.build(case)
    root = dc.root_of(case)
    assert len(ds) == int(g[case + "/db_length"])
    flat = _flat(ds.db)
    assert [os.path.relpath(os.path.join(root, r["image"]), root) for r in flat] == list(g[case + "/db_image"])
    box = np.array([[r[k] for k in ("center_x", "center_y", "width", "height")] for r in flat], dtype=np.float64)
    assert np.array_equal(box, g[case + "/db_box"])
    assert np.array_equal(np.stack([r["joints_3d"] for r in flat]), g[case + "/db_joints"])
    assert np.array_equal(np.stack([r["joints_3d_vis"] for r in flat]), g[case + "/db_vis"])
    if dc.H36M_CASES.get(case, (0, 0, False))[2]:
        assert len(ds.db) == 4 and all(len(d) == len(ds) for d in ds.db)


def test_calc_kpt_bound_and_actions():
    from lib.utils.utils import calc_kpt_bound
    from lib.utils.data_utils import define_actions
    k = np.array([[3.0, 4.0, 0], [10.0, -2.0, 0], [7.0, 9.0, 0]])
    v = np.array([[1.0] * 3, [0.0] * 3, [1.0] * 3])
    assert calc_kpt_bound(k, v) == (4.0, 9.0, 3.0, 7.0)
    assert calc_kpt_bound(k, 0 * v) == (10000, -1, 10000, -1)
    assert len(define_actions("All")) == 15 and define_actions("Eating") == ["Eating"]
    with pytest.raises(ValueError):
        define_actions("Juggling")


def test_mpii_evaluate_bit_identical(g, tmp_path):
    """PCKh@0.5: name_value bit-identical to the reference, pred.mat written (1-based), and the
    early {'Null': 0.0} return for a test set."""
    from scipy.io import loadmat
    ds = dc.build("mpii_valid")
    nv, perf = ds.evaluate(g["mpii_eval/preds"].copy(), str(tmp_path))
    assert [n for n, _ in nv] == list(g["mpii_eval/names"])
    assert np.array_equal(np.array([float(v) for _, v in nv]), g["mpii_eval/values"])
    assert float(perf) == float(g["mpii_eval/perf"])
    assert np.array_equal(loadmat(str(tmp_path / "pred.mat"))["preds"], g["mpii_eval/pred_mat"])
    ds.cfg.DATASET.TEST_SET = "test"
    os.remove(str(tmp_path / "pred.mat"))
    assert ds.evaluate(g["mpii_eval/preds"].copy(), str(tmp_path)) == ({'Null': 0.0}, 0.0)
    assert os.path.exists(str(tmp_path / "pred.mat"))


@pytest.mark.parametrize("order", ["h36m", "mpii"])
def test_h36m_evaluate_emulated(g, order):
    """H36M_Integral.evaluate through the CPU emulation of epb_h36m_eval: the nine protocol means,
    perf and the actionwise (MPJPE, aligned MPJPE) means against the reference."""
    import lib.dataset.h36m_eval as he
    he._backend[0] = emul_ops
    try:
        dc.seeded(dc.SEED % 1000)
        import lib.dataset as dataset
        ds = dataset.h36m(dc.cfg(MPII_ORDER=order == "mpii"), dc.H36M_ROOT, "valid", False)
        tag = "h36m_eval_" + order
        nv, perf = ds.evaluate(g[tag + "/preds"].copy(), None, actionwise=True)
    finally:
        he._backend[0] = __import__("epipolarpose_b200.ops", fromlist=["ops"])
    assert [n for n, _ in nv] == list(g[tag + "/names"])
    assert np.max(np.abs(np.array([v for _, v in nv]) - g[tag + "/values"])) <= 1e-8
    assert abs(perf - float(g[tag + "/perf"])) <= 1e-8
    from lib.utils.data_utils import define_actions
    got = np.array([ds.action_errors[a] for a in define_actions("All")], dtype=np.float64)
    ref = g[tag + "/actions"]
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    assert np.nanmax(np.abs(got - ref)) <= 1e-8


def _views(item):
    return [item["cam_1"], item["cam_2"]] if "cam_1" in item else [item]


@pytest.mark.parametrize("case", CASES)
def test_deferred_samples_carry_reference_draws(g, case, in_worker):
    """In a worker an item is a deferred sample: the reference's augmentation draws (scale, rot)
    and box for the same seeds, the joints / weights it labels with, and default_collate batches
    it unchanged (bytes as a list)."""
    from lib.dataset import deferred
    ds = dc.build(case)
    items = []
    for idx in range(len(ds)):
        dc.seeded(1000 + idx)
        items.append(ds[idx])
    keys = [case + "/cam_1", case + "/cam_2"] if dc.H36M_CASES.get(case, (0, 0, False))[2] else [case]
    for v, key in enumerate(keys):
        views = [_views(it)[v] for it in items]
        assert all(deferred.KEY in s for s in views)
        w = np.stack([s["joints_vis"].reshape(-1) for s in views]).astype(np.float32)
        assert np.array_equal(w, g[key + "/weight"])
        if key + "/scale_rot" in g:
            sr = np.stack([s["aug"][0:2] for s in views])
            assert np.array_equal(sr, g[key + "/scale_rot"])
            assert np.array_equal(np.stack([s["box"] for s in views]), g[key + "/meta_box"])
            assert np.array_equal(np.stack([[s["meta"]["scale"], s["meta"]["rot"]] for s in views]),
                                  g[key + "/scale_rot"])
            assert np.array_equal(np.stack([dc.meta_cam(s["meta"]) for s in views]), g[key + "/meta_cam"])
        root = dc.root_of(case)
        assert [os.path.relpath(s["meta"]["image"], root) for s in views] == list(g[key + "/image"])
        for s in views:
            with open(s["meta"]["image"], "rb") as f:
                assert s["jpeg"] == f.read()
    batch = default_collate(items[:3])
    assert deferred.is_deferred(batch)
    one = batch["cam_1"] if "cam_1" in batch else batch
    assert isinstance(one["jpeg"], list) and len(one["jpeg"]) == 3
    assert one["aug"].shape == (3, 6) and one["joints"].shape[0] == 3


def test_deferred_flip_and_occluder_packing():
    """A flipped draw mirrors the joints by the width in the JPEG header, as fliplr_joints does
    with the decoded frame; occluder lists survive the bytes packing."""
    from lib.dataset import deferred
    from lib.utils.img_utils import fliplr_joints
    with open(os.path.join(dc.MPII_ROOT, "images", "000.jpg"), "rb") as f:
        blob = f.read()
    assert deferred.jpeg_width(blob) == 160
    with open(os.path.join(dc.H36M_ROOT, "images", "s02_t1_c2.jpg"), "rb") as f:
        assert deferred.jpeg_width(f.read()) == 128            # the progressive frame
    rng = np.random.default_rng(3)
    occ = [(rng.integers(0, 255, (h, w, 4), dtype=np.uint8), (int(cx), int(cy)))
           for h, w, cx, cy in ((5, 7, 3, -2), (1, 1, 60, 61), (12, 3, 0, 9))]
    back = deferred.unpack_occluders(deferred.pack_occluders(occ))
    assert len(back) == 3 and all(np.array_equal(a[0], b[0]) and a[1] == b[1] for a, b in zip(occ, back))
    assert deferred.unpack_occluders(deferred.pack_occluders([])) == []
    import lib.utils.img_utils as iu
    j = rng.uniform(0, 100, (16, 3))
    v = np.ones((16, 3))
    orig = iu.do_augmentation
    iu.do_augmentation = lambda: (1.0, 0, True, [1.0, 1.0, 1.0])
    try:
        s = deferred.make_deferred(blob, (80, 60, 90, 90), j, v, [[0, 5], [1, 4]], True, None, (64, 64, 2000.),
                                   np.zeros(3), np.ones(3), {'image': 'x'})
    finally:
        iu.do_augmentation = orig
    ref_j, _ = fliplr_joints(j, v, 160, [[0, 5], [1, 4]])
    assert np.array_equal(s["joints"], ref_j) and s["aug"][2] == 1.0


class _NoDevice:
    """An ops backend that fails on any call."""

    def __getattr__(self, name):
        raise AssertionError("ops.%s called in a DataLoader worker" % name)


def _worker_without_cuda(_):
    import lib.utils.img_utils as iu
    import lib.dataset.h36m_eval as he

    def no_cuda(*a, **k):
        raise AssertionError("CUDA initialised in a DataLoader worker")
    torch.cuda._lazy_init = no_cuda
    iu._backend[0] = _NoDevice()
    he._backend[0] = _NoDevice()


@pytest.mark.parametrize("case", ["h36m_ss_tri", "h36m_valid", "mpii_train"])
def test_workers_make_no_device_call(case):
    """DataLoader(num_workers=2) whose workers fail on any ops call or CUDA initialisation
    completes: the workers only read files and draw."""
    from lib.dataset import deferred
    ds = dc.build(case)
    dl = DataLoader(ds, batch_size=2, shuffle=False, num_workers=2, worker_init_fn=_worker_without_cuda)
    n = 0
    for batch in dl:
        assert deferred.is_deferred(batch)
        one = batch["cam_1"] if "cam_1" in batch else batch
        n += len(one["jpeg"])
    assert n == len(ds)


@pytest.mark.parametrize("pkg", ["lib", "epipolarpose_b200.lib"])
@pytest.mark.parametrize("name", ["train-fs", "train-ss", "valid"])
def test_annotation_pickles_load_under_both_names(pkg, name):
    """The fixture pickles name the reference's lib.utils.cameras.Camera; they load as the
    package's own Camera whichever name the package was imported under."""
    import importlib
    jid = importlib.import_module(pkg + ".dataset.JointIntegralDataset")
    cams = importlib.import_module(pkg + ".utils.cameras")
    anno = jid.load_pickle(os.path.join(dc.H36M_ROOT, "annot", name + ".pkl"))
    recs = anno if isinstance(anno, list) else [r for k in sorted(anno) for r in anno[k]]
    assert len(recs) == 12
    for r in recs:
        cam = r["cam"]
        assert type(cam) is cams.Camera
        K = cam.get_intrinsic_matrix()
        P = K @ np.concatenate([cam.R, cam.R @ -cam.T], axis=1)
        assert np.allclose(cam.projection_matrix, P, rtol=0, atol=1e-9)
