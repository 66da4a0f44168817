"""GPU (-m gpu): the training launcher (epipolarpose_b200/train.py) under torch.distributed.run on the
H36M fixture tree (tests/golden/datasets/h36m), R18 at 64x64, graphed step, two epochs, with and without
DATASET.TRI (+ online triangulation).  The batch sizes give every rank at least two full batches per
epoch, so the step is captured and replayed (each rank reports it); at world 1 the plain case's epoch
ends on a ragged batch, which runs eagerly after the replays.
  * one GPU: the run exits 0 and writes its checkpoints; the logged validation metrics and predictions
    equal validate_integral + eval_integral of final_state.pth.tar in this process; a checkpoint of
    epoch 1 loads bit for bit (parameters, BatchNorm buffers, Adam state), and the run resumed from it
    uses the uninterrupted run's learning rate and sample indices in epoch 2;
  * two GPUs (skipped with fewer): parameters, Adam state and BatchNorm buffers identical on both ranks
    after every epoch, disjoint shards covering the training set, and the gathered validation equal to
    one process's validate_integral of the same checkpoint to 1e-4 px;
  * the launcher's sharded step (tools/ddp_launcher_check.py): the all-reduced gradient of one step on
    each rank's first shard batch equals the mean of the ranks' single-GPU gradients on those batches,
    to 1e-5, and is identical on every rank.  On two GPUs (skipped with fewer) that is the
    DataParallel equivalence; on one GPU the same tool checks its plumbing (the step's gradient against
    a recomputation of the same batch).
Bit-exact final parameters across runs are checked on the CPU only (tests/test_train_dist_host.py):
the BatchNorm statistics' float64 atomics make two GPU runs differ in the last bits."""
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import dataset_cases as dc
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu

# TRAIN_SET, TRI, per-GPU BATCH_SIZE at world 1 and 2.  train-fs has 12 items: 5 + 5 + 2 on one GPU,
# 2 + 2 + 2 per rank on two; train-ss has 3 tuples: 1 + 1 + 1 on one GPU, 1 + 1 per rank on two.
CASES = {"plain": ("train-fs", False, {1: 5, 2: 2}), "tri": ("train-ss", True, {1: 1, 2: 1})}


def _yaml(path, out, case, end_epoch, resume="", world=1):
    train_set, tri, batches = CASES[case]
    batch = batches[world]
    extra = dict(NUM_LAYERS=18, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[256, 256, 256],
                 NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1, TARGET_TYPE="gaussian",
                 HEATMAP_SIZE=[16, 16], SIGMA=2)
    cfg = dict(OUTPUT_DIR=out, WORKERS=2, PRINT_FREQ=1,
               MODEL=dict(INIT_WEIGHTS=False, NUM_JOINTS=17, DEPTH_RES=16, IMAGE_SIZE=[64, 64], RESUME=resume,
                          PRECISION="f16x3", EXTRA=extra),
               LOSS=dict(FN="SmoothL1JointLocationLoss"),
               DATASET=dict(DATASET="h36m", ROOT=dc.H36M_ROOT, TRAIN_SET=train_set, TEST_SET="valid", TRI=tri),
               TRAIN=dict(BATCH_SIZE=batch, END_EPOCH=end_epoch, LR=1e-3, LR_STEP=[2], LR_FACTOR=0.1,
                          ONLINE_TRIANGULATION=tri, CUDA_GRAPH=True),
               TEST=dict(BATCH_SIZE=4))
    with open(path, "w") as f:
        json.dump(cfg, f)                 # JSON is YAML
    return path


def _launch(tmp, name, case, end_epoch, nproc=1, resume="", seed=5, port=29710):
    cfg = _yaml(os.path.join(tmp, name + ".yaml"), os.path.join(tmp, name), case, end_epoch, resume, nproc)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                          str(nproc), "--master-addr", "127.0.0.1", "--master-port", str(port),
                          "-m", "epipolarpose_b200.train", "--cfg", cfg, "--seed", str(seed)],
                         cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    d = os.path.join(tmp, name, "h36m", "pose3d_resnet_18", "default")
    with open(os.path.join(d, "history.json")) as f:
        return d, cfg, json.load(f)


def _in_process(cfg_path, seed=5):
    """The launcher's model and validation set, built in this process from the same yaml: the
    training set, then the validation set, after seed_all(seed), so the dict-form db has the same order."""
    import lib.dataset as dataset
    import lib.models as models
    from lib.core.config import config, reset_config, update_config
    from lib.core.distributed import seed_all
    reset_config()
    update_config(cfg_path)
    model = models.pose3d_resnet.get_pose_net(config, is_train=False).cuda()
    seed_all(seed)
    dataset.h36m(cfg=config, root=config.DATASET.ROOT, image_set=config.DATASET.TRAIN_SET, is_train=True)
    valid = dataset.h36m(cfg=config, root=config.DATASET.ROOT, image_set="valid", is_train=False)
    loader = torch.utils.data.DataLoader(valid, batch_size=config.TEST.BATCH_SIZE, shuffle=False, num_workers=2)
    return config, model, loader


@pytest.mark.parametrize("case", list(CASES))
def test_one_gpu_launcher_run_validation_and_resume(case, tmp_path):
    from lib.core.function import eval_integral, validate_integral
    from lib.utils.utils import get_optimizer
    from epipolarpose_b200.train import load_checkpoint
    tmp = str(tmp_path)
    full_dir, full_cfg, full = _launch(tmp, "full", case, 2)
    for f in ("checkpoint.pth.tar", "model_best.pth.tar", "final_state.pth.tar", "valid_preds.npy"):
        assert os.path.exists(os.path.join(full_dir, f)), f
    assert full["world"] == 1 and full["seed"] == 5 and [e["epoch"] for e in full["epochs"]] == [0, 1]
    assert all(e["ranks"][0]["graph_captured"] for e in full["epochs"])
    # the logged metrics are those of the saved final state, evaluated here
    config, model, loader = _in_process(full_cfg)
    model.load_state_dict(torch.load(os.path.join(full_dir, "final_state.pth.tar"), map_location="cuda"))
    preds = validate_integral(loader, model, flip_test=False)
    assert np.max(np.abs(preds - np.load(os.path.join(full_dir, "valid_preds.npy")))) <= 1e-4
    perf, names = eval_integral(1, preds, loader, tmp, with_names=True)
    logged = full["epochs"][1]["metrics"]
    assert set(logged) == {n for n, _ in names}
    for n, v in names:
        assert abs(logged[n] - v) <= 1e-6 * max(abs(v), 1e-12), (n, logged[n], v)
    # stop after epoch 1: the checkpoint loads bit for bit, and the resumed run repeats epoch 2
    half_dir, _, half = _launch(tmp, "half", case, 1)
    ck_path = os.path.join(half_dir, "checkpoint.pth.tar")
    ck = torch.load(ck_path, map_location="cuda", weights_only=False)
    assert ck["epoch"] == 1 and ck["seed"] == 5 and ck["world"] == 1
    opt = get_optimizer(config, model)
    epoch, _, seed = load_checkpoint(ck_path, model, opt, torch.device("cuda"))
    assert (epoch, seed) == (1, 5)
    for k, v in model.state_dict().items():
        assert torch.equal(v, ck["state_dict"]["module." + k]), k
    got, want = opt.state_dict(), ck["optimizer"]
    assert got["state"].keys() == want["state"].keys()
    for i, st in want["state"].items():
        for k, v in st.items():
            assert torch.equal(torch.as_tensor(got["state"][i][k]).cpu(), torch.as_tensor(v).cpu()), (i, k)
    res_dir, _, res = _launch(tmp, "resumed", case, 2, resume=ck_path, seed=99)     # the checkpoint's seed wins
    assert res["seed"] == 5 and [e["epoch"] for e in res["epochs"]] == [1]
    a, b = full["epochs"][1], res["epochs"][0]
    assert a["lr"] == b["lr"] == 1e-3 * 0.1
    assert a["ranks"][0]["indices_sha256"] == b["ranks"][0]["indices_sha256"]
    assert a["ranks"][0]["samples"] == b["ranks"][0]["samples"]


@pytest.mark.parametrize("case", list(CASES))
def test_two_gpu_launcher_ranks_agree_and_shards_partition(case, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    from lib.core.distributed import shard_indices
    from lib.core.function import validate_integral
    import lib.dataset as dataset
    d, cfg, hist = _launch(str(tmp_path), "two", case, 2, nproc=2, port=29720)
    assert hist["world"] == 2
    config, model, loader = _in_process(cfg, hist["seed"])
    n = len(dataset.h36m(cfg=config, root=config.DATASET.ROOT, image_set=config.DATASET.TRAIN_SET, is_train=True))
    for e in hist["epochs"]:
        r0, r1 = e["ranks"]
        for k in ("params", "bn_buffers", "optimizer"):
            assert r0[k] == r1[k], (e["epoch"], k)
        assert r0["graph_captured"] and r1["graph_captured"]
        shards = [shard_indices(n, r, 2, True, hist["seed"], e["epoch"]) for r in range(2)]
        for r, rec in enumerate(e["ranks"]):
            assert rec["indices_sha256"] == hashlib.sha256(np.asarray(shards[r], dtype=np.int64).tobytes()).hexdigest()
        assert sorted(set(shards[0]) | set(shards[1])) == list(range(n))
        assert len(set(shards[0]) & set(shards[1])) == 2 * len(shards[0]) - n
    ck = torch.load(os.path.join(d, "final_state.pth.tar"), map_location="cuda")
    model.load_state_dict(ck)
    want = validate_integral(loader, model, flip_test=False)
    assert np.max(np.abs(np.load(os.path.join(d, "valid_preds.npy")) - want)) <= 1e-4


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_sharded_step_gradient_is_mean_of_rank_gradients(case, world, tmp_path):
    if torch.cuda.device_count() < world:
        pytest.skip("needs >= %d GPUs" % world)
    cfg = _yaml(os.path.join(str(tmp_path), "grad.yaml"), os.path.join(str(tmp_path), "grad"), case, 1, world=world)
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                          str(world), "--master-addr", "127.0.0.1", "--master-port", str(29730 + world),
                          os.path.join(ROOT, "tools", "ddp_launcher_check.py"), "--cfg", cfg, "--seed", "5"],
                         cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    line = json.loads([ln for ln in out.stdout.splitlines() if ln.startswith("{")][-1])
    assert line["world"] == world and line["identical_on_all_ranks"] and line["online"] == CASES[case][1]
    assert line["batch"][0] == CASES[case][2][world] * (2 if CASES[case][1] else 1)
    if world > 1:
        assert line["rank_batches_differ"]
    # the same kernels on the same inputs: only the order of the float64 atomics differs
    assert line["worst_rel_err_vs_replica_mean"] <= 1e-5, line
