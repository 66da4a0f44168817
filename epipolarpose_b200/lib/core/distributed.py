"""One training run over N processes, one per GPU (torchrun): what makes the ranks' loaders, seeds,
BatchNorm buffers and validation agree.  The per-step exchange itself is the model's gradient
all-reduce (lib/models/pose3d_resnet.py); everything here runs between steps.

  * init_from_env: torchrun's RANK / WORLD_SIZE / LOCAL_RANK -> (rank, world, device);
  * ShardSampler: one permutation of the training items per epoch, the same on every rank, cut into
    equal per-rank shards (a DATASET.TRI item -- a whole camera pair or tuple -- stays on one rank);
    val_block: the contiguous validation block of a rank;
  * common_seed / seed_all / derive_seed / WorkerSeeder: identical construction-time draws on every
    rank, then augmentation draws that depend only on (seed, epoch, rank, worker);
  * check_consistency / check_lockstep: raise on every rank, instead of training on different data or
    waiting forever in an all-reduce that one rank never reaches;
  * broadcast_bn_buffers: rank 0's BatchNorm running statistics everywhere (nn.DataParallel keeps
    replica 0's);
  * validate_sharded: validate_integral on each rank's block, gathered on rank 0 in dataset order.

With one process (no process group) every collective here is a no-op."""
import hashlib
import json
import math
import os
import random
import secrets

import numpy as np
import torch
import torch.distributed as dist

from .function import validate_integral

BN_BUFFERS = ('running_mean', 'running_var', 'num_batches_tracked')


def world_size():
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def rank_of():
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def _coll_device():
    """Where collective tensors live: the current GPU under NCCL, the host otherwise (gloo)."""
    if dist.get_backend() == 'nccl':
        return torch.device('cuda', torch.cuda.current_device())
    return torch.device('cpu')


def init_from_env(backend='nccl'):
    """(rank, world, device) from torchrun's RANK / WORLD_SIZE / LOCAL_RANK.  Under NCCL the process
    binds LOCAL_RANK's GPU before the group is made (as bench.py does); gloo ranks run on the host.
    A process group is initialised only for world > 1.  Without the variables: (0, 1, cuda:0)."""
    if 'RANK' not in os.environ or 'WORLD_SIZE' not in os.environ:
        return 0, 1, torch.device('cuda', 0)
    rank, world = int(os.environ['RANK']), int(os.environ['WORLD_SIZE'])
    local = int(os.environ.get('LOCAL_RANK', rank))
    if backend == 'nccl':
        torch.cuda.set_device(local)
        dev = torch.device('cuda', local)
    else:
        dev = torch.device('cpu')
    if world > 1 and not dist.is_initialized():
        if backend == 'nccl':
            dist.init_process_group(backend, device_id=dev)
        else:
            dist.init_process_group(backend, rank=rank, world_size=world)
    return rank, world, dev


# ---------------------------------------------------------------------------------------- sharding
def shard_indices(n, rank, world, shuffle, seed, epoch):
    """This rank's training items of one epoch: the permutation of range(n) drawn from (seed, epoch)
    (the identity without shuffle), padded by wrap-around to a multiple of `world`; rank r takes
    every world-th index from r.  Every shard has ceil(n / world) items."""
    order = np.random.default_rng([int(seed), int(epoch)]).permutation(n) if shuffle else np.arange(n)
    total = int(math.ceil(n / world)) * world
    return np.resize(order, total)[rank::world].tolist()


class ShardSampler(torch.utils.data.Sampler):
    """DataLoader sampler of shard_indices(n, rank, world, shuffle, seed, epoch); set_epoch(e) before
    each epoch's iterator.  `drawn` holds the indices of the last iteration."""

    def __init__(self, n, rank, world, shuffle, seed):
        self.n, self.rank, self.world = int(n), int(rank), int(world)
        self.shuffle, self.seed, self.epoch = bool(shuffle), int(seed), 0
        self.drawn = []

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def indices(self):
        return shard_indices(self.n, self.rank, self.world, self.shuffle, self.seed, self.epoch)

    def __iter__(self):
        self.drawn = self.indices()
        return iter(self.drawn)

    def __len__(self):
        return int(math.ceil(self.n / self.world))


def val_block(n, rank, world):
    """Rank r's validation items: the contiguous block [r*b, (r+1)*b) with b = ceil(n / world),
    indices past n wrapped to the start.  The blocks of ranks 0..world-1, concatenated and cut to n,
    are range(n)."""
    b = int(math.ceil(n / world))
    return [(rank * b + k) % n for k in range(b)]


# ----------------------------------------------------------------------------------------- seeding
def derive_seed(*keys):
    """A 32-bit seed from a tuple of non-negative integers (numpy SeedSequence)."""
    return int(np.random.SeedSequence([int(k) for k in keys]).generate_state(1)[0])


def seed_all(s):
    random.seed(s)
    np.random.seed(s % 2 ** 32)
    torch.manual_seed(s)


def common_seed(seed=None):
    """The run's seed: `seed`, or one rank 0 draws, broadcast so that every rank has it."""
    s = int(seed) if seed is not None else (secrets.randbits(31) if rank_of() == 0 else 0)
    if s < 0:
        raise ValueError("the seed must be a non-negative integer, got %d" % s)
    if world_size() > 1:
        t = torch.tensor([s], dtype=torch.int64, device=_coll_device())
        dist.broadcast(t, 0)
        s = int(t.item())
    return s


class WorkerSeeder:
    """DataLoader worker_init_fn: each worker seeds random, np.random and torch from
    (seed, epoch, rank, worker_id).  Set `epoch` before the epoch's iterator starts its workers."""

    def __init__(self, seed, rank):
        self.seed, self.rank, self.epoch = int(seed), int(rank), 0

    def __call__(self, worker_id):
        seed_all(derive_seed(self.seed, self.epoch, self.rank, worker_id))


# ------------------------------------------------------------------------------------- consistency
def _records(db):
    for rec in db:
        if isinstance(rec, (list, tuple)):          # a DATASET.TRI training db: one list per camera
            yield from _records(rec)
        else:
            yield rec


def dataset_fingerprint(ds):
    """(len(ds), sha256 of the image names in db order)."""
    h = hashlib.sha256()
    for rec in _records(getattr(ds, 'db', [])):
        h.update(str(rec.get('image', '') if isinstance(rec, dict) else rec).encode())
        h.update(b'\0')
    return len(ds), h.digest()


def _plain(v):
    if isinstance(v, dict):
        return {str(k): _plain(x) for k, x in v.items()}
    if isinstance(v, (np.ndarray, list, tuple)):
        return [_plain(x) for x in (v.tolist() if isinstance(v, np.ndarray) else v)]
    if isinstance(v, np.generic):
        return v.item()
    return v


def config_fingerprint(cfg):
    """(0, sha256 of the resolved config as sorted JSON)."""
    return 0, hashlib.sha256(json.dumps(_plain(cfg), sort_keys=True, default=repr).encode()).digest()


def check_consistency(named):
    """named: [(what, (length, 32-byte digest)), ...].  One all_gather compares every rank's entries
    with rank 0's; on a mismatch every rank raises RuntimeError naming the ranks and entries."""
    if world_size() == 1:
        return
    row = []
    for _, (n, digest) in named:
        row.append(int(n))
        row.extend(int(v) for v in np.frombuffer(digest, dtype='<i8'))
    t = torch.tensor(row, dtype=torch.int64, device=_coll_device())
    parts = [torch.empty_like(t) for _ in range(world_size())]
    dist.all_gather(parts, t)
    rows = [p.cpu().tolist() for p in parts]
    bad = []
    for r in range(1, len(rows)):
        for k, (what, _) in enumerate(named):
            a, b = rows[0][5 * k:5 * k + 5], rows[r][5 * k:5 * k + 5]
            if a != b:
                detail = ' (length %d on rank 0, %d on rank %d)' % (a[0], b[0], r) if a[0] != b[0] else ''
                bad.append('rank %d: %s%s' % (r, what, detail))
    if bad:
        raise RuntimeError("the ranks do not agree with rank 0: " + '; '.join(bad) +
                           ". Every rank must read the same files with the same config and seed.")


def check_lockstep(n_batches, tag):
    """Raise on every rank, before any step, when the ranks would run different numbers of batches:
    a rank that stops early would leave the others waiting in the gradient all-reduce.  The MIN and
    the MAX of the counts come from one all_reduce(MAX) of (n, -n)."""
    if world_size() == 1:
        return
    t = torch.tensor([int(n_batches), -int(n_batches)], dtype=torch.int64, device=_coll_device())
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    hi, lo = int(t[0]), -int(t[1])
    if hi != lo:
        raise RuntimeError("%s: the ranks have between %d and %d batches (this rank: %d); every rank must "
                           "run the same number of steps" % (tag, lo, hi, int(n_batches)))


def broadcast_bn_buffers(model):
    """Rank 0's BatchNorm running_mean, running_var and num_batches_tracked on every rank, in place."""
    if world_size() == 1:
        return
    for name, b in model.named_buffers():
        if name.rsplit('.', 1)[-1] in BN_BUFFERS:
            dist.broadcast(b, 0)


def validate_sharded(val_loader, model, n_total, flip_test=None, shift_heatmap=None):
    """validate_integral on this rank's block (val_loader iterates val_block(n_total, rank, world)),
    gathered with one all_gather and cut to n_total: rank 0 gets the [n_total, J, 4] array a single
    process's validate_integral over the whole set returns, the other ranks None."""
    out = validate_integral(val_loader, model, flip_test, shift_heatmap)
    if world_size() == 1:
        return out[:n_total]
    t = torch.from_numpy(np.ascontiguousarray(out)).to(_coll_device())
    parts = [torch.empty_like(t) for _ in range(world_size())]
    dist.all_gather(parts, t)
    if rank_of() != 0:
        return None
    return torch.cat(parts).cpu().numpy()[:n_total]
