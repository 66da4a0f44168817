"""Gradient semantics of the training launcher's sharded step (launched by tests/test_gpu_train_dist.py
under torch.distributed.run, one rank per GPU, NCCL):

    python -m torch.distributed.run --nproc-per-node N tools/ddp_launcher_check.py --cfg <yaml> --seed S

Each rank builds what epipolarpose_b200/train.py builds (train.setup: common seed, datasets, ShardSampler
loaders) and takes the first batch of its own shard in the first epoch, assembled as train_integral
assembles it.  One training step's backward all-reduces the gradient (the model's five stage slices,
ReduceOp.AVG).  Rank 0 then gathers every rank's batch and recomputes each rank's single-GPU gradient
with a copy of the same weights and allreduce_grads=False, without any collective.  The all-reduced
gradient must equal the MEAN of those (per-replica BatchNorm statistics: nn.DataParallel's step on the
global batch) and be bit-identical on every rank.  Prints one JSON line on rank 0:
world, identical_on_all_ranks, worst_rel_err_vs_replica_mean (largest over the parameter tensors of
max |got - mean| / max |mean|), the per-rank batch shape, and whether the rank batches differed."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from epipolarpose_b200 import train as T  # noqa: E402
import lib.core.distributed as D  # noqa: E402
import lib.core.function as fn  # noqa: E402
import lib.models as models  # noqa: E402
from lib.core.config import config, tuple_settings  # noqa: E402
from lib.utils.img_utils import pack_meta  # noqa: E402


def _gather(t, world):
    if world == 1:
        return [t]
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous())
    return parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cfg", required=True)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    rank, world, dev = D.init_from_env("nccl")
    s = T.setup(a.cfg, a.seed, None, None, rank, world, dev)
    T.start_epoch(s, s.begin, rank)
    online = fn._online_tri(config)
    views, method, thr = tuple_settings(config)
    x, label, weight, meta = fn.loader_batch(next(iter(s.train_loader)))
    x = x.to(dev)
    geom = pack_meta(meta, x.shape[0], dev, False) if online else None
    label = None if online else label.to(dev)
    weight = None if online else weight.to(dev)

    def grads(model, x, label, weight, geom):
        model.zero_grad(set_to_none=True)
        with fn._fused_head(model):
            preds = model(x)
        if online:
            loss = fn.online_epipolar_loss(s.criterion, preds, {"_packed": geom}, method, False, views, thr)
        else:
            loss = s.criterion(preds, label, weight)
        loss.backward()
        return {k: p.grad.detach().clone() for k, p in model.named_parameters()}

    model = s.model.train()
    weights = {k: v.detach().clone() for k, v in model.state_dict().items()}
    got = grads(model, x, label, weight, geom)
    torch.cuda.synchronize()
    same = True
    for g_ in got.values():
        ref0 = g_.clone()
        if world > 1:
            dist.broadcast(ref0, 0)
        same = same and bool(torch.equal(ref0, g_))
    xs = _gather(x, world)
    if online:
        gs = {k: _gather(v, world) for k, v in geom.items()}
        batches = [(xs[r], None, None, {k: gs[k][r] for k in gs}) for r in range(world)]
    else:
        ls, ws = _gather(label, world), _gather(weight, world)
        batches = [(xs[r], ls[r], ws[r], None) for r in range(world)]
    worst = 0.0
    if rank == 0:
        m1 = models.pose3d_resnet.get_pose_net(config, False, allreduce_grads=False).to(dev)
        m1.load_state_dict(weights)
        m1.train()
        ref = None
        for b in batches:
            cur = {k: v.double() / world for k, v in grads(m1, *b).items()}
            ref = cur if ref is None else {k: ref[k] + cur[k] for k in ref}
        for k in got:
            e = float((got[k].double() - ref[k]).abs().max() / ref[k].abs().max().clamp_min(1e-300))
            worst = max(worst, e)
    flag = torch.tensor([1.0 if same else 0.0], device=dev)
    if world > 1:
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(json.dumps({"world": world, "identical_on_all_ranks": bool(flag.item() == 1.0),
                          "worst_rel_err_vs_replica_mean": worst, "batch": list(x.shape), "online": online,
                          "rank_batches_differ": world > 1 and not torch.equal(xs[0], xs[1])}))
    sys.stdout.flush()
    torch.cuda.synchronize()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
