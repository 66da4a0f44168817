"""GPU (-m gpu): the h36m / mpii_integral datasets on the device, over the committed fixture tree.
  * main-process items against what the unmodified reference classes produced
    (tests/golden/datasets.npz): patches bit-exact by digest (the progressive frame included,
    decoded by cv2), labels to 1e-12, weights, scale, rot and meta exact;
  * DataLoader worker batches through assemble_batch against each sample materialised alone
    with the draws it recorded;
  * the call sequence of the reference's scripts/train.py / valid.py with WORKERS: 2."""
import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from tests import dataset_cases as dc

pytestmark = pytest.mark.gpu

CASES = list(dc.H36M_CASES) + list(dc.MPII_CASES)


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def g(golden):
    return golden("datasets")


def _check_views(g, key, views):
    assert [dc.digest(v[0]) for v in views] == list(g[key + "/sha256"]), key
    assert np.max(np.abs(np.stack([v[1] for v in views]).astype(np.float64) - g[key + "/label"])) <= 1e-12, key
    assert np.array_equal(np.stack([v[2] for v in views]), g[key + "/weight"]), key
    if key + "/scale_rot" in g:
        metas = [v[3] for v in views]
        assert np.array_equal(np.array([[m["scale"], m["rot"]] for m in metas]), g[key + "/scale_rot"]), key
        assert np.array_equal(np.array([[m[k] for k in ("center_x", "center_y", "width", "height")] for m in metas],
                                       dtype=np.float64), g[key + "/meta_box"]), key
        assert np.array_equal(np.stack([dc.meta_cam(m) for m in metas]), g[key + "/meta_cam"]), key


@pytest.mark.parametrize("case", CASES)
def test_main_process_items_match_reference(g, dev, case):
    ds = dc.build(case)
    items = []
    for idx in range(len(ds)):
        dc.seeded(1000 + idx)
        items.append(ds[idx])
    if dc.H36M_CASES.get(case, (0, 0, False))[2]:
        _check_views(g, case + "/cam_1", [it["cam_1"] for it in items])
        _check_views(g, case + "/cam_2", [it["cam_2"] for it in items])
    else:
        _check_views(g, case, items)


def _materialise(s):
    """One deferred sample alone, in the main process: cv2 decode, then the crop and the labels
    with the draws the worker recorded (get_single_patch_sample's device steps)."""
    import cv2
    import lib.utils.img_utils as iu
    img = cv2.imdecode(np.frombuffer(s["jpeg"], np.uint8), cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    a, b = s["aug"].numpy(), s["box"].numpy()
    pw, ph, rect = s["geometry"].numpy()
    ms = s["mean_std"].numpy()
    patch, trans, box = iu.generate_patch_batch_device([img], [b[0]], [b[1]], [b[2]], [b[3]], int(pw), int(ph),
                                                       [a[0]], [a[1]], [a[2] != 0], [a[3:6]], ms[:3], ms[3:])
    label = iu.patch_labels_device(s["joints"].numpy()[None], box, trans, pw, ph, rect)
    return patch[0], label[0].float(), torch.from_numpy(s["joints_vis"].numpy().reshape(-1)).float()


@pytest.mark.parametrize("case", ["h36m_ss_tri", "h36m_fs_train", "h36m_valid", "mpii_train"])
def test_worker_batches_assemble_bit_exact(dev, case):
    from lib.dataset import assemble_batch, is_deferred
    from lib.dataset.deferred import KEY
    ds = dc.build(case)
    dl = DataLoader(ds, batch_size=4, shuffle=False, num_workers=2)
    n = 0
    for batch in dl:
        assert is_deferred(batch)
        x, label, weight, meta = assemble_batch(batch)
        halves = [batch["cam_1"], batch["cam_2"]] if "cam_1" in batch else [batch]
        B = len(halves[0]["jpeg"])
        assert x.shape == (B * len(halves), 3, 64, 64) and x.is_cuda and label.is_cuda and weight.is_cuda
        for h, half in enumerate(halves):
            for i in range(B):
                s = {k: (v[i] if k not in ("meta", KEY) else None) for k, v in half.items()}
                p, lab, w = _materialise(s)
                r = h * B + i
                assert torch.equal(x[r], p), (case, r)
                assert torch.equal(label[r], lab), (case, r)
                assert torch.equal(weight[r].cpu(), w), (case, r)
                if "scale" in meta:
                    assert float(meta["scale"][r]) == float(s["aug"][0]) and float(meta["rot"][r]) == float(s["aug"][1])
        n += B
    assert n == len(ds)


def _script_flow(tmp_path, dataset, root, image_set, J, tri=False, online=False, batch=2):
    """scripts/train.py (:83-182) / scripts/valid.py call sequence with the loaders the unchanged
    scripts build (num_workers=config.WORKERS, no collate_fn)."""
    import lib.core.integral_loss as loss            # noqa: F401  (eval by name below)
    import lib.dataset as dataset_m                  # noqa: F401
    import lib.models as models
    from lib.core.config import config, reset_config
    from lib.core.function import train_integral, validate_integral, eval_integral
    from lib.utils.utils import get_optimizer, save_checkpoint
    reset_config()
    config.WORKERS = 2
    config.MODEL.NUM_JOINTS = J
    config.MODEL.DEPTH_RES = 16
    config.MODEL.IMAGE_SIZE = np.array([64, 64])
    config.MODEL.EXTRA.NUM_LAYERS = 18
    config.MODEL.INIT_WEIGHTS = False
    config.LOSS.FN = "SmoothL1JointLocationLoss"
    config.DATASET.DATASET = dataset
    config.DATASET.ROOT = root
    config.DATASET.TRAIN_SET = image_set
    config.DATASET.TRI = tri
    config.TRAIN.ONLINE_TRIANGULATION = online
    config.TRAIN.BATCH_SIZE = batch
    config.PRINT_FREQ = 1
    model = models.pose3d_resnet.get_pose_net(config, is_train=True)
    model = torch.nn.DataParallel(model, device_ids=[0]).cuda()
    criterion = eval("loss." + config.LOSS.FN)(num_joints=config.MODEL.NUM_JOINTS, norm=config.LOSS.NORM).cuda()
    optimizer = get_optimizer(config, model)
    sched = torch.optim.lr_scheduler.MultiStepLR(optimizer, [1], 0.1)
    ds = eval("dataset_m." + config.DATASET.DATASET)
    train_ds = ds(cfg=config, root=config.DATASET.ROOT, image_set=config.DATASET.TRAIN_SET, is_train=True)
    valid_ds = ds(cfg=config, root=config.DATASET.ROOT, image_set=config.DATASET.TEST_SET, is_train=False)
    mk = lambda d, bs, sh: DataLoader(d, batch_size=bs, shuffle=sh, num_workers=config.WORKERS, pin_memory=True)
    train_loader = mk(train_ds, config.TRAIN.BATCH_SIZE, config.TRAIN.SHUFFLE)
    valid_loader = mk(valid_ds, config.TEST.BATCH_SIZE, False)
    before = {k: v.detach().clone() for k, v in model.module.state_dict().items()}
    for epoch in range(2):
        avg = train_integral(config, train_loader, model, criterion, optimizer, epoch)
        sched.step()
        assert np.isfinite(avg)
        preds = validate_integral(valid_loader, model)
        assert preds.shape == (len(valid_ds), J, 4) and np.isfinite(preds).all()
        perf = eval_integral(epoch, preds, valid_loader, str(tmp_path), debug=False)
        assert np.isfinite(perf)
        save_checkpoint({"epoch": epoch + 1, "model": "pose3d_resnet", "state_dict": model.state_dict(),
                         "perf": perf, "optimizer": optimizer.state_dict()}, True, str(tmp_path))
    stepper = getattr(model, "_epb_graphed_step", None)
    assert stepper is not None and stepper.graph is not None          # the graphed step replayed
    after = model.module.state_dict()
    assert any(not torch.equal(before[k], after[k]) for k in before if before[k].is_floating_point())
    ck = torch.load(str(tmp_path / "checkpoint.pth.tar"), map_location="cpu", weights_only=False)
    fresh = models.pose3d_resnet.get_pose_net(config, is_train=False)
    fresh.load_state_dict({k[len("module."):]: v for k, v in ck["state_dict"].items()})
    for k, v in fresh.state_dict().items():
        assert torch.equal(v.cpu(), after[k].cpu()), k
    reset_config()
    return before


def test_script_flow_h36m_supervised(dev, tmp_path):
    _script_flow(tmp_path, "h36m", dc.H36M_ROOT, "train-fs", 17, batch=4)


def test_script_flow_mpii(dev, tmp_path):
    _script_flow(tmp_path, "mpii_integral", dc.MPII_ROOT, "train", 16, batch=1)


def test_script_flow_h36m_tri_online(dev, tmp_path, monkeypatch):
    """TRI + TRAIN.ONLINE_TRIANGULATION on the graphed step: the [cam_1 ; cam_2] batches are
    assembled on a side stream while the previous step replays, and the labels of the first
    step are self_supervision_device of the network's output on that assembled batch."""
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    import lib.models as models
    seen = {}
    orig_batch, orig_labels = fn.loader_batch, iu.labels_from_global_coords_device

    def rec_batch(data):
        out = orig_batch(data)
        seen.setdefault("batch", (out[0].clone(), out[3]))
        return out

    def rec_labels(X, meta, *a, **k):
        out = orig_labels(X, meta, *a, **k)
        seen.setdefault("labels", (out[0].clone(), out[1].clone()))
        return out
    monkeypatch.setattr(fn, "loader_batch", rec_batch)
    monkeypatch.setattr(iu, "labels_from_global_coords_device", rec_labels)
    before = _script_flow(tmp_path, "h36m", dc.H36M_ROOT, "train-ss", 17, tri=True, online=True, batch=1)
    x, meta = seen["batch"]
    assert x.shape[0] == 2 and len(meta["image"]) == 2
    assert meta["image"][0] != meta["image"][1]
    from lib.core.config import config
    config.MODEL.NUM_JOINTS, config.MODEL.DEPTH_RES, config.MODEL.IMAGE_SIZE = 17, 16, np.array([64, 64])
    config.MODEL.EXTRA.NUM_LAYERS, config.MODEL.INIT_WEIGHTS = 18, False
    net = models.pose3d_resnet.get_pose_net(config, is_train=True)
    net.load_state_dict(before)
    net = net.to(dev).train()
    with torch.no_grad():
        label, weight = iu.self_supervision_device(net(x), meta)
    used_label, used_weight = seen["labels"]
    assert torch.equal(weight, used_weight)
    assert torch.max(torch.abs(label - used_label)).item() <= 1e-5
