"""Cost of flip test at validation (TEST.FLIP_TEST) on one GPU.  Prints one JSON line: GPU name and
power limit; validate_integral throughput (images/s) at TEST.BATCH_SIZE 32 with flip test off and
on (R50, J = 16, D = 64, 256x256 inputs already in pinned host memory, so the loader costs nothing),
alternated over several rounds; the fused epb_softargmax_flip_fwd time (CUDA events) at N = 32,
J16 D64 64x64 and its rate against the 2*4*J*D*H*W*N bytes it has to read; the torch-op composition
(integral_loss.flip_merge_torch: flip-back copy, shift, average, then epb_softargmax_fwd) on the
same logits.
    python tools/bench_valid.py [--rounds 3] [--batches 8]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.bench_relpose import power_limit_w  # noqa: E402

J, D, HW, BATCH = 16, 64, 256, 32


class _Loader:
    """The part of a DataLoader validate_integral reads: iteration over batches and .dataset."""

    def __init__(self, batches, dataset):
        self.batches, self.dataset = batches, dataset

    def __iter__(self):
        return iter(self.batches)


class _Dataset:
    def __init__(self, n):
        self.n = n
        self.flip_pairs = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]

    def __len__(self):
        return self.n


def validate_ips(model, loader, flip):
    from lib.core.function import validate_integral
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = validate_integral(loader, model, flip_test=flip, shift_heatmap=True)
    e1.record()
    torch.cuda.synchronize()
    assert np.isfinite(out).all()
    return len(loader.dataset) / (e0.elapsed_time(e1) / 1e3)


def merge_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    from epipolarpose_b200 import ops
    import lib.core.integral_loss as il
    import lib.models as models
    from tools.bench_cfg import make_cfg
    dev = torch.device("cuda")
    ops.device_check()
    out = {"gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit_w()}

    # ---- the fused merge vs the torch-op composition, N = 32, J16 D64 64x64
    N, H, W = 32, 64, 64
    g = torch.Generator(device=dev).manual_seed(3)
    logits = (3.0 * torch.randn((2 * N, H, W, J * D), device=dev, generator=g)).permute(0, 3, 1, 2)
    perm = il.flip_permutation(_Dataset(0).flip_pairs, J)
    coords = torch.empty((N, J * 3), device=dev)
    fused = merge_ms(lambda: ops.softargmax_flip_fwd(logits.permute(0, 2, 3, 1), N, J, D, H, W, perm, 1, coords),
                     args.reps)
    composed = merge_ms(lambda: il.flip_merge_torch(logits, J, D, H, W, perm, True), max(3, args.reps // 4))
    c_torch = il.flip_merge_torch(logits, J, D, H, W, perm, True)
    nbytes = 2 * 4 * J * D * H * W * N
    out["merge"] = {"N": N, "J": J, "D": D, "HW": H, "bytes": nbytes,
                    "fused_ms": round(fused, 4), "fused_GBps": round(nbytes / fused / 1e6, 1),
                    "torch_ms": round(composed, 3), "torch_over_fused": round(composed / fused, 2),
                    "max_abs_diff": float((coords - c_torch).abs().max())}
    del logits, c_torch
    torch.cuda.empty_cache()

    # ---- validate_integral, flip test off / on
    cfg = make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    torch.manual_seed(0)
    model = models.pose3d_resnet.get_pose_net(cfg, False).to(dev).eval()
    gen = torch.Generator().manual_seed(1)
    batches = [(torch.randn(BATCH, 3, HW, HW, generator=gen).pin_memory(),) for _ in range(args.batches)]
    loader = _Loader(batches, _Dataset(BATCH * args.batches))
    validate_ips(model, loader, False)               # warm-up: workspaces, both batch sizes
    validate_ips(model, loader, True)
    off, on = [], []
    for _ in range(args.rounds):
        off.append(validate_ips(model, loader, False))
        on.append(validate_ips(model, loader, True))
    out["validate_batch_size"] = BATCH
    out["validate_images_per_s_flip_off"] = [round(v, 1) for v in off]
    out["validate_images_per_s_flip_on"] = [round(v, 1) for v in on]
    out["flip_on_over_off_median"] = round(float(np.median(np.array(on) / np.array(off))), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
