"""GPU: transcode_jpeg_batch_device (epb_jpeg_transcode, csrc/jpeg.cu).
  * output bytes equal to the CPU build of the same bodies (tests/harness/host_jpeg_transcode.cu)
    for every fixture blob at every interval, in one mixed batch and one at a time; runs repeat;
  * device decodes of the outputs equal those of the sources and cv2's frames (tests/golden/jpeg.npz);
  * transcoded 1000x1002 frames need no sequential walk and at most the phase-A rounds their
    longest interval allows;
  * a write pass given an output smaller than the first call read back fails the call;
  * the dataset classes read a transcoded copy of tests/golden/datasets exactly as the original,
    and H36M_Integral / MPIIDataset evaluate a network's predictions on it to the same results."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from tests import dataset_cases as dc
from tests.conftest import ROOT
from tests.transcode_cases import INTERVALS, _build, _runner

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases(golden):
    g = golden("jpeg")
    out = []
    for i, name in enumerate(g["names"]):
        H, W = (int(v) for v in g["hw"][i])
        pix = g["pix_data"][g["pix_off"][i]:g["pix_off"][i + 1]]
        out.append(dict(name=str(name), kind=str(g["kind"][i]), hw=(H, W), sha=str(g["sha256"][i]),
                        pix=pix.reshape(H, W, 3) if pix.size else None,
                        blob=g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes()))
    return out


@pytest.fixture(scope="module")
def host_tc(tmp_path_factory):
    return _runner(_build(tmp_path_factory, "host_jpeg_transcode", ["-O1"]))


STATUS = {"ok": 0, "unsupported": 1, "truncated": 2}


@pytest.mark.parametrize("R", INTERVALS)
def test_device_bytes_equal_host_build(cases, host_tc, R):
    import lib.utils.img_utils as iu
    interval = "auto" if R == 0 else R
    want = host_tc([c["blob"] for c in cases], R)
    out, st = iu.transcode_jpeg_batch_device([c["blob"] for c in cases], interval=interval, verify=False)
    again, st2 = iu.transcode_jpeg_batch_device([c["blob"] for c in cases], interval=interval, verify=False)
    assert out == again and list(st) == list(st2)
    for c, w, o, s in zip(cases, want, out, st):
        assert s == STATUS[c["kind"]], (c["name"], s)
        assert o == (w["out"] if c["kind"] == "ok" else c["blob"]), c["name"]
    for c, w in zip(cases, want):
        if c["kind"] == "ok":
            one, s1 = iu.transcode_jpeg_batch_device([c["blob"]], interval=interval, verify=False)
            assert s1[0] == 0 and one[0] == w["out"], c["name"]


@pytest.mark.parametrize("R", [1, 0])
def test_decodes_equal_sources_and_cv2(cases, R):
    import lib.utils.img_utils as iu
    ok = [c for c in cases if c["kind"] == "ok"]
    out, st = iu.transcode_jpeg_batch_device([c["blob"] for c in ok], interval="auto" if R == 0 else R, verify=True)
    assert list(st) == [0] * len(ok)                 # verify flags nothing on the fixture
    a = iu.decode_jpeg_batch_device([c["blob"] for c in ok])
    b = iu.decode_jpeg_batch_device(out)
    assert list(b.status) == [0] * len(ok)
    for i, c in enumerate(ok):
        assert torch.equal(a.frame(i), b.frame(i)), c["name"]
        f = b.frame(i).cpu().numpy()
        if c["pix"] is not None:
            assert np.array_equal(f, c["pix"]), c["name"]
        else:
            assert hashlib.sha256(f.tobytes()).hexdigest() == c["sha"], c["name"]


def test_unsupported_and_truncated_come_back_unchanged(cases):
    import lib.utils.img_utils as iu
    other = [c for c in cases if c["kind"] != "ok"]
    out, st = iu.transcode_jpeg_batch_device([c["blob"] for c in other])
    for c, o, s in zip(other, out, st):
        assert o == c["blob"] and s == STATUS[c["kind"]], c["name"]


def test_transcoded_frames_synchronise_within_their_intervals(cases):
    """At R = auto 10.6 % (frame a) and 6.0 % (frame b) of the intervals exceed kJpegSubBits
    (tests/test_jpeg_transcode_host.py), the longest 3379 bits: at most 4 subsequences per segment,
    so at most 3 phase-A rounds change a state and the sequential walk never runs."""
    import lib.utils.img_utils as iu
    frames = [c["blob"] for c in cases if c["name"].startswith("frame1000_")]
    out, st = iu.transcode_jpeg_batch_device(frames)
    assert list(st) == [0, 0]
    batch = [out[i % 2] for i in range(128)]
    stats = torch.zeros(7, dtype=torch.int32, device="cuda")
    d = iu.decode_jpeg_batch_device(batch, stats=stats)
    s = stats.cpu().numpy()
    assert list(d.status) == [0] * 128
    assert s[3:].tolist() == [0, 0, 0, 0], s


# ------------------------------------------------------------------ the dataset classes on a prepared tree
@pytest.fixture(scope="module")
def prepared(tmp_path_factory):
    dst = tmp_path_factory.mktemp("prepared")
    summary = {}
    for name, root in (("h36m", dc.H36M_ROOT), ("mpii", dc.MPII_ROOT)):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "prep_frames.py"), root, str(dst / name)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
        summary[name] = r.stdout
    return dst, summary


def _build_at(name, root):
    import lib.dataset as dataset
    dc.seeded(dc.SEED % 1000)
    if name in dc.H36M_CASES:
        image_set, is_train, tri, zw = dc.H36M_CASES[name]
        return dataset.h36m(dc.cfg(TRI=tri, Z_WEIGHT=zw), root, image_set, is_train)
    image_set, is_train = dc.MPII_CASES[name]
    return dataset.mpii_integral(dc.cfg(ROOT=root), root, image_set, is_train)


def _np(v):
    return v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)


def test_prepared_tree_was_transcoded(prepared):
    import json
    for name, out in prepared[1].items():
        s = json.loads(out.strip().splitlines()[-1])
        assert s["transcoded"] >= 1 and s["transcoded"] + sum(s["passed_through"].values()) == s["frames"], (name, s)


@pytest.mark.parametrize("case", list(dc.H36M_CASES) + list(dc.MPII_CASES))
def test_main_process_items_equal_on_prepared_tree(prepared, case):
    root = str(prepared[0] / ("h36m" if case in dc.H36M_CASES else "mpii"))
    a, b = _build_at(case, dc.root_of(case)), _build_at(case, root)
    assert len(a) == len(b)
    for idx in range(len(a)):
        dc.seeded(1000 + idx)
        x = a[idx]
        dc.seeded(1000 + idx)
        y = b[idx]
        views = [("cam_1", "cam_2")] if isinstance(x, dict) and "cam_1" in x else [None]
        pairs = [(x[k], y[k]) for k in views[0]] if views[0] else [(x, y)]
        for u, v in pairs:
            for k in range(3):
                assert np.array_equal(_np(u[k]), _np(v[k])), (case, idx, k)


@pytest.mark.parametrize("case", ["h36m_ss_tri", "h36m_fs_train", "h36m_valid", "mpii_train"])
def test_worker_batches_equal_on_prepared_tree(prepared, case):
    from lib.dataset import assemble_batch
    root = str(prepared[0] / ("h36m" if case in dc.H36M_CASES else "mpii"))
    got = []
    for r in (dc.root_of(case), root):
        ds = _build_at(case, r)
        torch.manual_seed(5)
        got.append([assemble_batch(b)[:3] for b in DataLoader(ds, batch_size=4, shuffle=True, num_workers=2)])
    assert len(got[0]) == len(got[1])
    for p, q in zip(*got):
        for u, v in zip(p, q):
            assert torch.equal(u, v), case


def test_write_pass_fails_loudly_on_an_output_smaller_than_read_back(cases, monkeypatch):
    """The second call checks every interval against the sizes of the first call on the device and
    fails the call, so a short output never comes back as status 0 with unwritten bytes."""
    import lib.utils.img_utils as iu
    from epipolarpose_b200 import _lib, ops
    first = ops.jpeg_transcode

    def shrunk(*a, **k):
        info = first(*a, **k)
        info["bytes"][0] //= 2
        return info
    monkeypatch.setattr(ops, "jpeg_transcode", shrunk)
    blob = next(c["blob"] for c in cases if c["name"] == "frame1000_a")
    with pytest.raises(_lib.EpbError, match="disagree"):
        iu.transcode_jpeg_batch_device([blob], verify=False)


@pytest.mark.parametrize("dataset,name,J", [("h36m", "h36m", 17), ("mpii_integral", "mpii", 16)])
def test_evaluation_equal_on_prepared_tree(prepared, tmp_path, dataset, name, J):
    """H36M_Integral / MPIIDataset evaluation as scripts/valid.py runs it (validate_integral, then
    eval_integral / dataset.evaluate) on the original and the prepared tree, with the same seeds:
    the batches the network reads, its predictions and the evaluation results are identical."""
    import lib.dataset as dataset_m
    import lib.models as models
    from lib.core.config import config, reset_config
    from lib.core.function import validate_integral, eval_integral, loader_batch
    reset_config()
    config.WORKERS = 2
    config.MODEL.NUM_JOINTS = J
    config.MODEL.DEPTH_RES = 16
    config.MODEL.IMAGE_SIZE = np.array([64, 64])
    config.MODEL.EXTRA.NUM_LAYERS = 18
    config.MODEL.INIT_WEIGHTS = False
    config.DATASET.DATASET = dataset
    torch.manual_seed(0)
    model = torch.nn.DataParallel(models.pose3d_resnet.get_pose_net(config, is_train=False), device_ids=[0]).cuda()
    got = []
    for k, root in enumerate((dc.H36M_ROOT if name == "h36m" else dc.MPII_ROOT, str(prepared[0] / name))):
        config.DATASET.ROOT = root
        dc.seeded(dc.SEED % 1000)            # construction draws from the global generators
        ds = getattr(dataset_m, dataset)(cfg=config, root=root, image_set=config.DATASET.TEST_SET, is_train=False)
        loader = DataLoader(ds, batch_size=config.TEST.BATCH_SIZE, shuffle=False, num_workers=config.WORKERS)
        torch.manual_seed(7)                 # the workers' draws come from the loader's base seed
        x = [loader_batch(b)[0].cpu() for b in loader]
        torch.manual_seed(7)
        preds = validate_integral(loader, model)
        out = tmp_path / str(k)
        out.mkdir()
        got.append(dict(x=x, preds=preds, perf=eval_integral(0, preds, loader, str(out)),
                        named=ds.evaluate(preds.copy(), str(out))[0]))
    reset_config()
    a, b = got
    assert len(a["x"]) == len(b["x"]) >= 1 and all(torch.equal(u, v) for u, v in zip(a["x"], b["x"]))
    assert a["preds"].shape[0] == len(ds) and np.isfinite(a["preds"]).all()
    assert np.array_equal(a["preds"], b["preds"])
    assert np.array_equal(np.array([a["perf"]], np.float64), np.array([b["perf"]], np.float64), equal_nan=True)
    assert [n for n, _ in a["named"]] == [n for n, _ in b["named"]]
    assert np.array_equal(np.array([v for _, v in a["named"]], np.float64),
                          np.array([v for _, v in b["named"]], np.float64), equal_nan=True)
