"""Refiner training / evaluation loop -- host-side mirror of the reference refiner/main.py:
`parse_args` (:17-29), `train(model, train_dl, optimizer, glob_step, lr_now, criterion, args,
logger)` (:31-62), `test(model, test_dl)` (:64-84) and the `__main__` driver (:86-175), same
checkpoint dictionary (epoch / lr / step / err / state_dict / optimizer; optimizer state in the
torch.optim layout, so checkpoints interchange with the reference).

The model is refiner.model.LinearModelPG on the libepb.so kernels, the optimiser the fused Adam
(one kernel over the flat parameter buffer), gradient clipping refiner.utils.clip_grad_norm_ on
the device.  The loss value stays on the device and is folded into the meter at the end of the
epoch (the reference's per-step loss.item() sync, :54, is gone)."""
import argparse
import logging
import os
import time

import numpy as np
import torch
import torch.nn as nn

from .model import get_model, weight_init
from .utils import AverageMeter, clip_grad_norm_, lr_decay, save_ckpt


# command line of the reference script (refiner/main.py:17-29): (flag, type, default, help)
_OPTIONS = (
    ("--exp", str, "test", "ID of experiment"),
    ("--load", str, None, "path to load a pretrained checkpoint"),
    ("--mode", str, "train", "mode: [train, test]"),
    ("--num_epochs", int, 200, "num epochs"),
    ("--lr", float, 1e-3, "learning rate"),
    ("--lr_decay", int, 100000, "# steps of lr decay"),
    ("--lr_gamma", float, 0.96, None),
)


def parse_args(argv=None):
    ap = argparse.ArgumentParser()
    for flag, kind, default, text in _OPTIONS:
        ap.add_argument(flag, type=kind, default=default, help=text)
    return ap.parse_args(argv)


def _to_device(t):
    return t.cuda(non_blocking=True) if torch.cuda.is_available() else t


def train(model, train_dl, optimizer, glob_step, lr_now, criterion, args, logger):
    """One epoch.  Both heads of the refiner are regressed on the same target (reference :50);
    the gradient is clipped to unit norm (:57).  Returns (glob_step, lr_now)."""
    meter = AverageMeter()
    model.train()
    on_device = []                            # (loss, batch size): read back once, after the epoch
    for batch, target in train_dl:
        glob_step += 1
        if glob_step == 1 or glob_step % args.lr_decay == 0:
            lr_now = lr_decay(optimizer, glob_step, args.lr, args.lr_decay, args.lr_gamma)
        batch, target = _to_device(batch), _to_device(target)
        first, second = model(batch)[:2]
        optimizer.zero_grad()
        loss = criterion(first, target) + criterion(second, target)
        on_device.append((loss.detach(), target.size(0)))
        loss.backward()
        clip_grad_norm_(model.parameters(), max_norm=1.)
        optimizer.step()
    for value, count in on_device:
        meter.update(value.item(), count)
    logger.info("Avg Loss: %.5f", meter.avg)
    return glob_step, lr_now


def test(model, test_dl):
    """Refined poses of the whole loader (second head) -> dataset.evaluate (reference :64-84)."""
    model.eval()
    refined = []
    with torch.no_grad():
        for batch, _ in test_dl:
            refined.append(model(_to_device(batch))[-1])
    refined = torch.cat(refined, 0).cpu().numpy() if refined else np.zeros((0, 45), np.float32)
    return test_dl.dataset.evaluate(refined)


def _restore(path, model, optimizer, logger):
    """Checkpoint dictionary of the reference (:118-127): epoch, err, step, lr, state_dict, optimizer."""
    logger.info("loading checkpoint %s", path)
    ckpt = torch.load(path, map_location="cpu", weights_only=False)
    model.load_state_dict(ckpt["state_dict"])
    optimizer.load_state_dict(ckpt["optimizer"])
    logger.info("checkpoint of epoch %s, error %s", ckpt["epoch"], ckpt["err"])
    return ckpt["epoch"], ckpt["err"], ckpt["step"], ckpt["lr"]


def main(argv=None, train_dl=None, test_dl=None, log_root='refiner/experiments', data_root='refiner/data'):
    args = parse_args(argv)
    out_dir = os.path.join(log_root, args.exp)
    os.makedirs(out_dir, exist_ok=True)
    logger = logging.getLogger("refiner")
    logger.setLevel(logging.INFO)
    model = get_model(weights=None)
    if torch.cuda.is_available():
        model = model.cuda()
    model.apply(weight_init)
    criterion = nn.MSELoss(reduction='mean')
    from lib.utils.utils import FusedAdam
    optimizer = FusedAdam(list(model.parameters()), lr=args.lr)
    best, glob_step, lr_now = 1000, 0, args.lr
    if args.load:
        _, best, glob_step, lr_now = _restore(args.load, model, optimizer, logger)
    if train_dl is None or test_dl is None:
        from .data import Human36M, SyntheticPoses
        if all(os.path.exists(os.path.join(data_root, f)) for f in ("train.pkl", "valid.pkl")):
            make = lambda is_train: Human36M(is_train=is_train, root=data_root)
        else:
            logger.info("no train.pkl / valid.pkl under %s: using synthetic poses", data_root)
            make = lambda is_train: SyntheticPoses(is_train=is_train)
        train_dl = torch.utils.data.DataLoader(make(True), batch_size=64, shuffle=True)
        test_dl = torch.utils.data.DataLoader(make(False), batch_size=64, shuffle=False)
    if args.mode == 'test':
        return test(model, test_dl)
    if args.mode != 'train':
        print('mode input error!')
        return None
    logger.info("training for %d epoch(s)", args.num_epochs)
    for epoch in range(args.num_epochs):
        logger.info("epoch %d of %d, lr %.6f", epoch, args.num_epochs, lr_now)
        glob_step, lr_now = train(model, train_dl, optimizer, glob_step, lr_now, criterion, args, logger)
        error = test(model, test_dl)
        improved = error < best
        best = min(best, error)
        save_ckpt({'epoch': epoch + 1, 'lr': lr_now, 'step': glob_step, 'err': error,
                   'state_dict': model.state_dict(), 'optimizer': optimizer.state_dict()},
                  ckpt_path=out_dir, is_best=improved)
        if improved:
            logger.info("new best error %s", error)
    return best


if __name__ == '__main__':
    main()
