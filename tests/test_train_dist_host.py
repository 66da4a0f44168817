"""CPU: multi-process training (lib/core/distributed.py, epipolarpose_b200/train.py) on gloo ranks with
the CPU emulation of the C ABI (tests/emul_ops.py): the sharded sampler and validation blocks, the
common seed and the startup fingerprint check on the H36M fixture tree, the lockstep guard, the
BatchNorm buffer broadcast, sharded validation against one process's validate_integral, and the
launcher's epoch loop over two ranks, stopped and resumed.

gloo has no ReduceOp.AVG: the workers emulate it with SUM / world, as test_host_logic does."""
import json
import os
import random

import numpy as np
import pytest
import torch

from oracle import refshim, restate_net
from tests import dataset_cases as dc, emul_ops

TIMEOUT = 300


# ------------------------------------------------------------------------------- sampler, blocks
@pytest.mark.parametrize("world", range(1, 9))
def test_shards_equal_disjoint_and_covering(world):
    from lib.core.distributed import ShardSampler, shard_indices
    for n in range(1, 38):
        for shuffle in (True, False):
            shards = []
            for r in range(world):
                s = ShardSampler(n, r, world, shuffle, seed=11)
                s.set_epoch(3)
                shards.append(list(s))
                assert len(s) == len(shards[-1])
            per = -(-n // world)
            assert all(len(sh) == per for sh in shards)
            flat = [i for sh in shards for i in sh]
            assert sorted(set(flat)) == list(range(n))                       # covers everything
            # every rank derives the same permutation: rank r's shard is its every-world-th slice
            order = [shards[k % world][k // world] for k in range(per * world)]
            assert order[:n] == shard_indices(n, 0, 1, shuffle, 11, 3)      # one process's permutation
            if not shuffle:
                assert order[:n] == list(range(n))                           # SHUFFLE: false keeps order
            assert shards[0] == shard_indices(n, 0, world, shuffle, 11, 3)


def test_permutation_changes_with_epoch_and_seed():
    from lib.core.distributed import shard_indices
    a = shard_indices(37, 0, 1, True, 5, 0)
    assert a != shard_indices(37, 0, 1, True, 5, 1) and a != shard_indices(37, 0, 1, True, 6, 0)
    assert a == shard_indices(37, 0, 1, True, 5, 0) and sorted(a) == list(range(37))


@pytest.mark.parametrize("world", range(1, 9))
def test_validation_blocks_reassemble_in_dataset_order(world):
    from lib.core.distributed import val_block
    for n in range(1, 38):
        blocks = [val_block(n, r, world) for r in range(world)]
        assert len({len(b) for b in blocks}) == 1
        assert [i for b in blocks for i in b][:n] == list(range(n))


def test_worker_seeds_depend_on_seed_epoch_rank_worker():
    from lib.core.distributed import WorkerSeeder, derive_seed
    draws = set()
    for key in [(1, 0, 0, 0), (1, 1, 0, 0), (1, 0, 1, 0), (1, 0, 0, 1), (2, 0, 0, 0)]:
        w = WorkerSeeder(key[0], key[2])
        w.epoch = key[1]
        w(key[3])
        draws.add((np.random.random(), random.random(), float(torch.rand(1))))
    assert len(draws) == 5
    assert derive_seed(1, 2, 3) == derive_seed(1, 2, 3) != derive_seed(1, 2, 4)


# ------------------------------------------------------------------------------ process harness
def _spawn(target, world=2, args=()):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29000 + (os.getpid() * 7 + hash(target.__name__)) % 900
    ps = [ctx.Process(target=_entry, args=(target, r, world, port, q) + tuple(args)) for r in range(world)]
    for p in ps:
        p.start()
    try:
        res = dict(q.get(timeout=TIMEOUT) for _ in ps)
    finally:
        for p in ps:
            p.join(60)
            if p.is_alive():
                p.kill()
                p.join(10)
    for r in range(world):
        if isinstance(res[r], BaseException):
            raise res[r]
    return res


def _entry(target, rank, world, port, q, *args):
    """A gloo rank with the emulated ABI: torchrun's variables, ReduceOp.AVG as SUM / world, and
    Tensor.cuda() a no-op (train_integral / validate_integral move host batches with it)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    import torch.distributed as dist
    import lib.core.integral_loss as il
    import lib.utils.img_utils as iu
    import lib.utils.utils as U
    il._backend[0] = iu._backend[0] = U._backend[0] = EMUL
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.set_num_threads(1)                  # two ranks share the host's cores
    orig = dist.all_reduce

    class _Done:
        def wait(self):
            return True

    def all_reduce(t, op=dist.ReduceOp.SUM, group=None, async_op=False):
        if op == dist.ReduceOp.AVG:
            orig(t, group=group)
            t /= dist.get_world_size()
            return _Done()
        return orig(t, op=op, group=group, async_op=async_op)
    dist.all_reduce = all_reduce
    try:
        from lib.core.distributed import init_from_env
        init_from_env("gloo")
        out = target(rank, world, *args)
    except BaseException:             # reported to the parent with its traceback; every rank answers
        import traceback
        out = RuntimeError("rank %d: %s" % (rank, traceback.format_exc()))
    q.put((rank, _host(out)))
    if dist.is_initialized():
        dist.destroy_process_group()


def _host(v):
    """Tensors as numpy arrays: a tensor sent through the queue would live in this process's shared
    memory, gone when the rank exits."""
    if torch.is_tensor(v):
        return v.detach().numpy().copy()
    if isinstance(v, dict):
        return {k: _host(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return type(v)(_host(x) for x in v)
    return v


class _EmulFlip:
    """emul_ops plus epb_softargmax_flip_fwd (its contract in include/epb.h: merge each volume with
    its flipped-back mirror, then the soft-argmax)."""

    def __getattr__(self, name):
        return getattr(emul_ops, name)

    @staticmethod
    def softargmax_flip_fwd(logits2N, N, J, D, H, W, perm, shift, coords):
        v = logits2N.reshape(2 * N, H, W, J, D).permute(0, 3, 4, 1, 2).double()
        w = torch.arange(W)
        src = torch.where(w == 0, W - 1, W - w) if shift else W - 1 - w
        merged = 0.5 * (v[:N] + v[N:][:, [int(q) for q in perm]][..., src])
        c = torch.empty(N * J * 3)
        emul_ops.softargmax_fwd(merged.reshape(N, J * D, H, W), 0, N, J, D, H, W, c,
                                torch.empty(N * J * 2, dtype=torch.float64))
        coords.view(-1).copy_(c)


EMUL = _EmulFlip()


# --------------------------------------------------------------------------- seeding, fingerprint
def _seed_worker(rank, world):
    import lib.core.distributed as D
    import lib.dataset as dataset
    seed = D.common_seed(None)                 # drawn by rank 0
    out = {"seed": seed}
    for other in (False, True):
        D.seed_all(seed + (1 if other and rank == 1 else 0))
        tr = dataset.h36m(dc.cfg(), dc.H36M_ROOT, "train-fs", True)
        va = dataset.h36m(dc.cfg(), dc.H36M_ROOT, "valid", False)
        if not other:
            out["train"] = [r["image"] for r in tr.db]
            out["valid"] = [r["image"] for r in va.db]
        try:
            D.check_consistency([("training set", D.dataset_fingerprint(tr)),
                                 ("validation set", D.dataset_fingerprint(va)),
                                 ("config", D.config_fingerprint({"a": [1, 2]}))])
            out["raised_%d" % other] = None
        except RuntimeError as e:
            out["raised_%d" % other] = str(e)
    return out


def test_common_seed_builds_identical_h36m_db_and_fingerprint_mismatch_raises_on_both_ranks():
    res = _spawn(_seed_worker)
    assert res[0]["seed"] == res[1]["seed"]
    assert res[0]["train"] == res[1]["train"] and res[0]["valid"] == res[1]["valid"]
    assert len(res[0]["train"]) > 1
    assert res[0]["raised_0"] is None and res[1]["raised_0"] is None
    for r in (0, 1):
        msg = res[r]["raised_1"]
        assert msg is not None and "rank 1: training set" in msg and "rank 1: config" not in msg, msg


# ------------------------------------------------------------------------------ lockstep, buffers
def _lockstep_worker(rank, world):
    from lib.core.distributed import check_lockstep
    check_lockstep(5, "same")
    try:
        check_lockstep(3 + rank, "epoch 0 training")
    except RuntimeError as e:
        return str(e)
    return None


def test_lockstep_raises_on_both_ranks():
    res = _spawn(_lockstep_worker)
    for r in (0, 1):
        assert res[r] is not None and "between 3 and 4 batches" in res[r] and "epoch 0 training" in res[r]


def _model(J=2, D=8, HW=32, seed=1):
    import lib.models as models
    cfg = refshim.make_cfg(num_layers=18, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    m = models.pose3d_resnet.get_pose_net(cfg, False, ops=emul_ops)
    m.load_state_dict(restate_net.init_state(restate_net.param_shapes(18, J, True, D), seed))
    return m


def _bn_worker(rank, world):
    from lib.core.distributed import BN_BUFFERS, broadcast_bn_buffers
    m = _model()
    g = torch.Generator().manual_seed(50 + rank)
    before = {}
    for n, b in m.named_buffers():
        if n.rsplit(".", 1)[-1] in BN_BUFFERS:
            b.copy_((torch.rand(b.shape, generator=g) * 100).to(b.dtype))
            before[n] = b.clone()
    broadcast_bn_buffers(m)
    return before, {n: b.clone() for n, b in m.named_buffers() if n in before}


def test_broadcast_bn_buffers_gives_rank0s_bit_for_bit():
    res = _spawn(_bn_worker)
    before0 = res[0][0]
    assert len(before0) == 3 * 23                    # R18's 20 BatchNorms + the three deconvs'
    for r in (0, 1):
        for n, v in res[r][1].items():
            assert np.array_equal(v, before0[n]), (r, n)
    assert any(not np.array_equal(res[1][0][n], before0[n]) for n in before0)


# ------------------------------------------------------------------------------ fixture dataset
class TinyPoses(torch.utils.data.Dataset):
    """In-file dataset: n seeded 32x32 images of J joints, no image files.  The db order comes from
    random.shuffle at construction (as H36M_Integral's), and a training item adds one np.random
    augmentation draw, so both the common seed and the per-rank draws matter."""
    flip_pairs = [[0, 1]]

    def __init__(self, n, is_train, J=2):
        self.is_train, self.J = is_train, J
        self.db = [{"image": "frame_%03d" % i, "idx": i, "center_x": 100.0 + i, "center_y": 90.0,
                    "width": 150.0, "height": 150.0} for i in range(n)]
        random.shuffle(self.db)

    def __len__(self):
        return len(self.db)

    def __getitem__(self, k):
        i = self.db[k]["idx"]
        g = np.random.default_rng(i)
        img = g.standard_normal((3, 32, 32)).astype(np.float32)
        if self.is_train:
            img = img * np.float32(1.0 + 0.1 * np.random.randn())
        label = (g.random(self.J * 3) - 0.5).astype(np.float32)
        return torch.from_numpy(img), torch.from_numpy(label), torch.ones(self.J * 3), {"image": self.db[k]["image"]}

    def evaluate(self, preds, save_path=None, debug=False):
        err = float(np.mean(np.abs(np.asarray(preds)[:, :, 0:2])))
        return [("err", err)], err


def _make_datasets(cfg):
    return TinyPoses(11, True), TinyPoses(7, False)


def _sharded_worker(rank, world, n, flip):
    from lib.core.distributed import val_block, validate_sharded
    from lib.core.function import validate_integral
    from lib.core.config import config
    config.MODEL.NUM_JOINTS, config.MODEL.DEPTH_RES, config.MODEL.IMAGE_SIZE = 2, 8, [32, 32]
    m = _model().eval()
    random.seed(3)                            # the same db order on both ranks
    ds = TinyPoses(n, False)
    from epipolarpose_b200.train import _Block
    blk = torch.utils.data.DataLoader(_Block(ds, val_block(n, rank, world)), batch_size=2)
    got = validate_sharded(blk, m, n, flip_test=flip, shift_heatmap=True)
    want = validate_integral(torch.utils.data.DataLoader(ds, batch_size=3), m, flip_test=flip,
                             shift_heatmap=True) if rank == 0 else None
    return got, want


@pytest.mark.parametrize("flip", [False, True])
def test_validate_sharded_equals_single_process(flip):
    res = _spawn(_sharded_worker, world=2, args=(7, flip))
    got, want = res[0]
    assert res[1][0] is None
    assert got.shape == want.shape == (7, 2, 4)
    assert np.array_equal(got, want)


# -------------------------------------------------------------------------------- launcher loop
def _yaml(path, out, end_epoch, resume=""):
    extra = dict(NUM_LAYERS=18, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[256, 256, 256],
                 NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1, TARGET_TYPE="gaussian",
                 HEATMAP_SIZE=[8, 8], SIGMA=2)
    cfg = dict(OUTPUT_DIR=out, WORKERS=0, PRINT_FREQ=1,
               MODEL=dict(INIT_WEIGHTS=False, NUM_JOINTS=2, DEPTH_RES=8, IMAGE_SIZE=[32, 32], RESUME=resume,
                          EXTRA=extra),
               DATASET=dict(DATASET="h36m"),
               TRAIN=dict(BATCH_SIZE=4, END_EPOCH=end_epoch, LR=1e-3, LR_STEP=[2], LR_FACTOR=0.1, SHUFFLE=True),
               TEST=dict(BATCH_SIZE=3))
    with open(path, "w") as f:
        json.dump(cfg, f)                 # JSON is YAML
    return path


def _launcher_worker(rank, world, tmp):
    from epipolarpose_b200 import train as T

    def go(name, end, resume="", seed=None):
        cfg = _yaml(os.path.join(tmp, "%s.rank%d.yaml" % (name, rank)), os.path.join(tmp, name), end, resume)
        r = T.run(cfg, seed=seed,
                  backend="gloo", ops=emul_ops, make_datasets=_make_datasets)
        state = {k: v.clone() for k, v in r["model"].state_dict().items()}
        return {k: r[k] for k in ("seed", "output_dir", "history", "saved", "world")}, state

    full = go("full", 2, seed=7)
    half = go("half", 1, seed=7)
    ck = half[0]["saved"][0] if rank == 0 else None
    import torch.distributed as dist
    box = [ck]
    dist.broadcast_object_list(box, 0)
    resumed = go("resumed", 2, resume=box[0])
    return full, half, resumed


def test_launcher_two_ranks_identical_one_checkpoint_and_exact_resume(tmp_path):
    res = _spawn(_launcher_worker, world=2, args=(str(tmp_path),))
    (f0, fs0), (h0, hs0), (r0, rs0) = res[0]
    (f1, fs1), (h1, hs1), (r1, rs1) = res[1]
    assert f0["world"] == 2 and f0["seed"] == f1["seed"] == 7 and r0["seed"] == 7
    for hist in (f0["history"], h0["history"], r0["history"]):
        for e in hist:
            a, b = e["ranks"]
            for k in ("params", "bn_buffers", "optimizer"):
                assert a[k] == b[k], (e["epoch"], k)           # identical on both ranks after each epoch
            assert a["indices_sha256"] != b["indices_sha256"] and a["samples"] == b["samples"] == 6
    assert [e["epoch"] for e in f0["history"]] == [0, 1] and [e["epoch"] for e in r0["history"]] == [1]
    assert [e["lr"] for e in f0["history"]] == [1e-3, 1e-3 * 0.1]
    for k in fs0:
        assert np.array_equal(fs0[k], fs1[k]), k
        assert np.array_equal(hs0[k], hs1[k]), k
        assert np.array_equal(rs0[k], fs0[k]), k             # resumed == never stopped, bit for bit
    assert any(not np.array_equal(hs0[k], fs0[k]) for k in fs0 if fs0[k].dtype == np.float32)
    e_full, e_res = f0["history"][1], r0["history"][0]
    assert e_res["lr"] == e_full["lr"] and e_res["metrics"] == e_full["metrics"]
    for a, b in zip(e_full["ranks"], e_res["ranks"]):
        a.pop("train_seconds"), b.pop("train_seconds")
        assert a == b                        # loss, indices drawn, parameters, buffers, optimiser state
    # rank 0 alone writes, in the reference's layout plus seed and world
    assert f1["saved"] == [] and h1["saved"] == [] and r1["saved"] == []
    names = sorted(os.path.basename(p) for p in f0["saved"])
    assert "checkpoint.pth.tar" in names and "final_state.pth.tar" in names
    ck = torch.load(os.path.join(f0["output_dir"], "checkpoint.pth.tar"), weights_only=False)
    assert {"epoch", "model", "state_dict", "perf", "optimizer", "seed", "world"} <= set(ck)
    assert ck["epoch"] == 2 and ck["seed"] == 7 and ck["world"] == 2
    assert all(k.startswith("module.") for k in ck["state_dict"])
    with open(os.path.join(f0["output_dir"], "history.json")) as f:
        assert [e["epoch"] for e in json.load(f)["epochs"]] == [0, 1]
