"""Training on one or more GPUs, one process per GPU:

    python -m torch.distributed.run --nproc-per-node N -m epipolarpose_b200.train --cfg <yaml> [--seed S]

With one process (or plain `python -m epipolarpose_b200.train`) it is a single-GPU trainer.  The flow is
the reference's scripts/train.py, written on this package's API: config, model, get_optimizer,
MultiStepLR (stepped at the start of each epoch, as the reference does), MODEL.RESUME, the
DATASET.DATASET train / validation sets, then per epoch train_integral, validation and eval_integral.

What makes N processes one run (lib/core/distributed.py): the datasets are built under one common
seed and compared across ranks; each epoch's training items are one permutation cut into equal
per-rank shards (TRAIN.BATCH_SIZE is per GPU, as the reference's BATCH_SIZE x len(gpus)); the batch
counts are checked before the training and validation loops; the gradient is averaged inside the
model's backward; after training, rank 0's BatchNorm running statistics are broadcast (nn.DataParallel
keeps replica 0's); validation runs on contiguous per-rank blocks gathered on rank 0, which evaluates,
logs and writes checkpoint.pth.tar / model_best.pth.tar / final_state.pth.tar in the reference's layout
plus `seed`, `world` and `best_perf`, valid_preds.npy (the last validation's [n, J, 4] patch
coordinates) and `history.json` (per epoch: lr, metrics, and for every rank its loss, training time,
the digest of the sample indices it drew and of its parameters, BatchNorm buffers and optimiser state).
Data order and augmentation depend only on (seed, epoch, rank, loader worker), so a resumed run
repeats the run that never stopped.

Best model: lower is better except for mpii_integral (PCKh).  The reference compares 500 - acc for
every dataset (its `== 'h36m' or 'mpii_3dhp' or 'jta'` test is always true) and so keeps MPII's worst
epoch."""
import argparse
import hashlib
import json
import logging
import os
import shutil
import sys
import time
import types
import warnings

import numpy as np
import torch
import torch.distributed as dist

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (_ROOT, os.path.join(_ROOT, 'epipolarpose_b200')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import lib.core.distributed as D  # noqa: E402
import lib.core.integral_loss as loss  # noqa: E402,F401  (criterion by name, as the reference)
import lib.dataset as dataset  # noqa: E402,F401  (dataset by name, as the reference)
import lib.models as models  # noqa: E402
from lib.core.config import config, get_model_name, reset_config, update_config  # noqa: E402
from lib.core.function import eval_integral, train_integral  # noqa: E402
from lib.utils.utils import create_logger, get_optimizer, save_checkpoint  # noqa: E402

logger = logging.getLogger(__name__)

HIGHER_IS_BETTER = ('mpii_integral',)


class _Block(torch.utils.data.Subset):
    """A rank's validation block that still answers for its dataset (db, flip_pairs, ...)."""

    def __getattr__(self, name):
        if name in ('dataset', 'indices') or name.startswith('__'):
            raise AttributeError(name)
        return getattr(self.dataset, name)


def _strip_module(sd):
    if sd and all(k.startswith('module.') for k in sd):
        return {k[len('module.'):]: v for k, v in sd.items()}
    return sd


def load_checkpoint(ck, model, optimizer, device=None):
    """Load a checkpoint (a path, read with map_location `device`, or the loaded dict) into model /
    optimizer.  A training checkpoint gives (epoch to continue at, best_perf, seed); a bare state_dict
    gives (None, None, None)."""
    if not isinstance(ck, dict):
        ck = torch.load(ck, map_location=device, weights_only=False)
    if 'epoch' not in ck:
        model.load_state_dict(_strip_module(ck))
        return None, None, None
    model.load_state_dict(_strip_module(ck['state_dict']))
    optimizer.load_state_dict(ck['optimizer'])
    return int(ck['epoch']), ck.get('best_perf'), ck.get('seed')


def set_schedule(scheduler, epoch):
    """Put the MultiStepLR where the uninterrupted run is after `epoch` epochs (one step() per epoch
    from the initial LR, so the learning rate is the same float)."""
    for g in scheduler.optimizer.param_groups:
        g['lr'] = g.get('initial_lr', g['lr'])
    scheduler.last_epoch = 0
    with warnings.catch_warnings():
        warnings.simplefilter('ignore')          # step() before optimizer.step(): the reference's order
        for _ in range(epoch):
            scheduler.step()


def _digest(tensors):
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().cpu().contiguous().numpy().tobytes())
    return h.hexdigest()


def state_digests(model, optimizer):
    """sha256 of the parameters, the BatchNorm buffers and the optimiser state of this rank."""
    params = [p for _, p in model.named_parameters()]
    bufs = [b for n, b in model.named_buffers() if n.rsplit('.', 1)[-1] in D.BN_BUFFERS]
    st = optimizer.state_dict()['state']
    opt = [v if torch.is_tensor(v) else torch.tensor(float(v))
           for k in sorted(st) for _, v in sorted(st[k].items())]
    return {'params': _digest(params), 'bn_buffers': _digest(bufs), 'optimizer': _digest(opt)}


def _captured(model):
    """Whether the training step ran as a CUDA-graph replay (lib/core/function.py GraphedTrainStep)."""
    stepper = getattr(model, '_epb_graphed_step', None)
    return stepper is not None and stepper.graph is not None


def _make_datasets(cfg):
    ds = getattr(dataset, cfg.DATASET.DATASET)
    return (ds(cfg=cfg, root=cfg.DATASET.ROOT, image_set=cfg.DATASET.TRAIN_SET, is_train=True),
            ds(cfg=cfg, root=cfg.DATASET.ROOT, image_set=cfg.DATASET.TEST_SET, is_train=False))


def run(cfg_file, seed=None, backend='nccl', ops=None, make_datasets=None):
    """The training run of one rank.  backend: the process group's ('nccl'; 'gloo' runs the ranks on
    the host); ops: the model's implementation of the C ABI (default: libepb.so); make_datasets:
    cfg -> (train, valid), default DATASET.DATASET from the registry.  A process group is made from
    torchrun's variables unless one exists, and destroyed at the end if it was made here.

    Returns {'rank', 'world', 'seed', 'output_dir' (rank 0), 'history' (one entry per epoch run),
    'saved' (files this rank wrote), 'model', 'optimizer'}."""
    made = not (dist.is_available() and dist.is_initialized())
    rank, world, dev = D.init_from_env(backend)
    try:
        return _run(cfg_file, seed, ops, make_datasets, rank, world, dev)
    finally:
        if made and dist.is_available() and dist.is_initialized():
            dist.destroy_process_group()


def setup(cfg_file, seed, ops, make_datasets, rank, world, dev):
    """Everything a rank builds before its first epoch, as a namespace: config read, the seed made common,
    logging (rank 0 creates the output directory), model, criterion, optimizer, scheduler (resumed when
    MODEL.RESUME is set), the datasets built under the common seed and checked across ranks, and the
    sharded loaders."""
    reset_config()
    update_config(cfg_file)
    ck = None
    if config.MODEL.RESUME:                        # read once; its seed keeps the run's data order and draws
        ck = torch.load(config.MODEL.RESUME, map_location=dev, weights_only=False)
        if isinstance(ck, dict) and ck.get('seed') is not None:
            seed = int(ck['seed'])
    seed = D.common_seed(seed)

    out_dir = None
    if rank == 0:
        _, out_dir = create_logger(config, cfg_file, 'train')
        shutil.copy2(cfg_file, out_dir)
        logger.info('world %d, seed %d, per-GPU batch %d', world, seed, config.TRAIN.BATCH_SIZE)
    else:
        logging.basicConfig(format='%(asctime)-15s rank ' + str(rank) + ' %(message)s')
        logging.getLogger().setLevel(logging.WARNING)

    D.seed_all(seed)
    model = models.pose3d_resnet.get_pose_net(config, is_train=True,
                                              **({'ops': ops} if ops is not None else {})).to(dev)
    criterion = eval('loss.' + config.LOSS.FN)(num_joints=config.MODEL.NUM_JOINTS,
                                               norm=config.LOSS.NORM).to(dev)
    optimizer = get_optimizer(config, model)
    scheduler = torch.optim.lr_scheduler.MultiStepLR(optimizer, config.TRAIN.LR_STEP, config.TRAIN.LR_FACTOR)
    begin, best = int(config.TRAIN.BEGIN_EPOCH), None
    if ck is not None:
        epoch, best, _ = load_checkpoint(ck, model, optimizer)
        del ck
        begin = begin if epoch is None else epoch
        logger.info('=> resume from %s at epoch %d', config.MODEL.RESUME, begin)
    set_schedule(scheduler, begin)

    D.seed_all(seed)                               # identical construction-time draws on every rank
    train_ds, valid_ds = (make_datasets or _make_datasets)(config)
    D.check_consistency([('training set', D.dataset_fingerprint(train_ds)),
                         ('validation set', D.dataset_fingerprint(valid_ds)),
                         ('config', D.config_fingerprint(config))])
    D.seed_all(D.derive_seed(seed, rank))

    # no pin-memory thread: its cudaHostAlloc calls would invalidate the graphed step's capture, which
    # runs while the loader's next batches are pinned (deferred batches are host bytes anyway)
    seeder = D.WorkerSeeder(seed, rank)
    sampler = D.ShardSampler(len(train_ds), rank, world, config.TRAIN.SHUFFLE, seed)
    train_loader = torch.utils.data.DataLoader(train_ds, batch_size=config.TRAIN.BATCH_SIZE, sampler=sampler,
                                               num_workers=config.WORKERS, worker_init_fn=seeder)
    block = _Block(valid_ds, D.val_block(len(valid_ds), rank, world))
    valid_loader = torch.utils.data.DataLoader(block, batch_size=config.TEST.BATCH_SIZE, shuffle=False,
                                               num_workers=config.WORKERS, worker_init_fn=seeder)
    eval_loader = torch.utils.data.DataLoader(valid_ds, batch_size=config.TEST.BATCH_SIZE)   # its .dataset only
    return types.SimpleNamespace(seed=seed, out_dir=out_dir, model=model, criterion=criterion, optimizer=optimizer,
                                 scheduler=scheduler, begin=begin, best=best, train_ds=train_ds, valid_ds=valid_ds,
                                 seeder=seeder, sampler=sampler, train_loader=train_loader,
                                 valid_loader=valid_loader, eval_loader=eval_loader)


def start_epoch(s, epoch, rank):
    """Point the sampler, the loader workers' seeds and this process's RNGs at `epoch`."""
    s.sampler.set_epoch(epoch)
    s.seeder.epoch = epoch
    D.seed_all(D.derive_seed(s.seed, epoch, rank))


def _run(cfg_file, seed, ops, make_datasets, rank, world, dev):
    s = setup(cfg_file, seed, ops, make_datasets, rank, world, dev)
    seed, out_dir, model, criterion, optimizer, scheduler = \
        s.seed, s.out_dir, s.model, s.criterion, s.optimizer, s.scheduler
    begin, best, valid_ds, sampler = s.begin, s.best, s.valid_ds, s.sampler
    train_loader, valid_loader, eval_loader = s.train_loader, s.valid_loader, s.eval_loader

    hist_path = os.path.join(out_dir, 'history.json') if out_dir else None
    history = []
    if hist_path and os.path.exists(hist_path):
        with open(hist_path) as f:
            history = [e for e in json.load(f)['epochs'] if e['epoch'] < begin]
    run_history, saved = [], []
    higher = config.DATASET.DATASET in HIGHER_IS_BETTER
    for epoch in range(begin, int(config.TRAIN.END_EPOCH)):
        with warnings.catch_warnings():
            warnings.simplefilter('ignore')
            scheduler.step()
        lr = float(optimizer.param_groups[0]['lr'])
        start_epoch(s, epoch, rank)
        D.check_lockstep(len(train_loader), 'epoch %d training' % epoch)
        t0 = time.perf_counter()
        avg = train_integral(config, train_loader, model, criterion, optimizer, epoch)   # ends on a loss read-back
        seconds = time.perf_counter() - t0
        D.broadcast_bn_buffers(model)
        D.check_lockstep(len(valid_loader), 'epoch %d validation' % epoch)
        preds = D.validate_sharded(valid_loader, model, len(valid_ds))
        mine = {'rank': rank, 'loss': float(avg), 'batches': len(train_loader), 'samples': len(sampler.drawn),
                'train_seconds': seconds, 'graph_captured': _captured(model),
                'indices_sha256': hashlib.sha256(np.asarray(sampler.drawn, dtype=np.int64).tobytes()).hexdigest()}
        mine.update(state_digests(model, optimizer))
        ranks = [None] * world
        if world > 1:
            dist.all_gather_object(ranks, mine)
        else:
            ranks = [mine]
        decision = [None, None, None]
        if rank == 0:
            perf, names = eval_integral(epoch, preds, eval_loader, out_dir, debug=config.DEBUG.DEBUG, with_names=True)
            perf = float(perf)
            np.save(os.path.join(out_dir, 'valid_preds.npy'), preds)
            is_best = best is None or (perf > best if higher else perf < best)
            decision = [is_best, perf, dict(names)]
        if world > 1:
            dist.broadcast_object_list(decision, 0)
        is_best, perf, metrics = decision
        if is_best:
            best = perf
        entry = {'epoch': epoch, 'lr': lr, 'perf': perf, 'best': bool(is_best), 'metrics': metrics, 'ranks': ranks}
        run_history.append(entry)
        if rank == 0:
            logger.info('=> saving checkpoint to %s', out_dir)
            save_checkpoint({'epoch': epoch + 1, 'model': get_model_name(config),
                             'state_dict': {'module.' + k: v for k, v in model.state_dict().items()},
                             'perf': perf, 'best_perf': best, 'optimizer': optimizer.state_dict(),
                             'seed': seed, 'world': world}, is_best, out_dir)
            saved.append(os.path.join(out_dir, 'checkpoint.pth.tar'))
            if is_best:
                saved.append(os.path.join(out_dir, 'model_best.pth.tar'))
            history.append(entry)
            with open(hist_path, 'w') as f:
                json.dump({'seed': seed, 'world': world, 'epochs': history}, f, indent=1)
        if world > 1:
            dist.barrier()
    if rank == 0:
        final = os.path.join(out_dir, 'final_state.pth.tar')
        logger.info('saving final model state to %s', final)
        torch.save(model.state_dict(), final)
        saved.append(final)
    if world > 1:
        dist.barrier()
    return {'rank': rank, 'world': world, 'seed': seed, 'output_dir': out_dir, 'history': run_history,
            'saved': saved, 'model': model, 'optimizer': optimizer}


def main(argv=None):
    ap = argparse.ArgumentParser(description='Train PoseResNet on one or more GPUs (one process per GPU)')
    ap.add_argument('--cfg', required=True, help='experiment configure file name')
    ap.add_argument('--seed', type=int, default=None,
                    help='the run seed (default: drawn by rank 0; a resumed run keeps its own)')
    a = ap.parse_args(argv)
    run(a.cfg, seed=a.seed)


if __name__ == '__main__':
    main()
