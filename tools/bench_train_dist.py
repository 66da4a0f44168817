"""Throughput of the training launcher (epipolarpose_b200/train.py) on a real-data loader: end to end
from JPEG files to the graphed step, on `--gpus` ranks.

Writes a seeded synthetic H36M-shaped tree under --out as tools/bench_prep_ss.py does (dict-form
annotation of 4-view tuples, 17 joints, ring cameras; `--files` distinct 1000x1000 q90 JPEG frames
transcoded to short restart intervals, so file reads come from the page cache), with
`--steps` x `--batch` x `--gpus` training tuples and 8 validation tuples.  Then runs the launcher under
torch.distributed.run for two epochs: R50, J17, D64, 256², f16x3, DATASET.TRI with TRI_VIEWS 4 and the
robust online labels, `--batch` tuples (x 4 views) per GPU, `--workers` loader workers per rank.  The
first epoch warms up (graph capture); the second is timed by each rank (train_integral, which ends on a
loss read-back) and the slowest rank counts: tuples/s is the training set's size over that time (the
shards' wrap-around padding is not counted).  Prints ONE JSON line: GPU name, power limit and max SM
clock (read in the same run), world, tuples/s, fed ms/step, and the host's CPU count.  Needs a GPU.

    python tools/bench_train_dist.py --out DIR [--gpus 1] [--steps 20] [--batch 32] [--workers 8]"""
import argparse
import json
import os
import pickle
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.bench_jpeg import card  # noqa: E402
from tools.bench_prep_ss import make_tree  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--files", type=int, default=32)
    ap.add_argument("--port", type=int, default=29780)
    a = ap.parse_args()
    from lib.dataset.JointIntegralDataset import load_pickle
    tuples = a.steps * a.batch * a.gpus
    src = make_tree(a.out, tuples, a.files)
    anno = load_pickle(src)
    with open(os.path.join(a.out, "annot", "valid8.pkl"), "wb") as f:
        pickle.dump({c: anno[c][:8] for c in anno}, f, protocol=4)
    extra = dict(NUM_LAYERS=50, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3, NUM_DECONV_FILTERS=[256, 256, 256],
                 NUM_DECONV_KERNELS=[4, 4, 4], FINAL_CONV_KERNEL=1, TARGET_TYPE="gaussian",
                 HEATMAP_SIZE=[64, 64], SIGMA=2)
    cfg = dict(OUTPUT_DIR=os.path.join(a.out, "run"), WORKERS=a.workers, PRINT_FREQ=1000,
               MODEL=dict(INIT_WEIGHTS=False, NUM_JOINTS=17, DEPTH_RES=64, IMAGE_SIZE=[256, 256],
                          PRECISION="f16x3", EXTRA=extra),
               LOSS=dict(FN="SmoothL1JointLocationLoss"),
               DATASET=dict(DATASET="h36m", ROOT=a.out, TRAIN_SET="src", TEST_SET="valid8", TRI=True, TRI_VIEWS=4),
               TRAIN=dict(BATCH_SIZE=a.batch, END_EPOCH=2, LR=1e-3, LR_STEP=[100], ONLINE_TRIANGULATION=True,
                          TRIANGULATION_METHOD="robust", CUDA_GRAPH=True),
               TEST=dict(BATCH_SIZE=32))
    path = os.path.join(a.out, "train.yaml")
    with open(path, "w") as f:
        json.dump(cfg, f)
    before = card()
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node",
                          str(a.gpus), "--master-addr", "127.0.0.1", "--master-port", str(a.port),
                          "-m", "epipolarpose_b200.train", "--cfg", path, "--seed", "0"],
                         cwd=ROOT, capture_output=True, text=True)
    if out.returncode != 0:
        sys.stderr.write(out.stdout[-3000:] + out.stderr[-12000:])
        sys.exit(out.returncode)
    with open(os.path.join(a.out, "run", "h36m", "pose3d_resnet_50", "default", "history.json")) as f:
        hist = json.load(f)
    timed = hist["epochs"][1]["ranks"]
    sec = max(r["train_seconds"] for r in timed)
    steps = timed[0]["batches"]
    print(json.dumps({"card_before": before, "card_after": card(), "world": a.gpus,
                      "tuples_per_s": tuples / sec,             # the training set, not the padded shards
                      "fed_ms_per_step": 1e3 * sec / steps, "steps": steps, "tuples_per_gpu_step": a.batch,
                      "views": 4, "workers_per_rank": a.workers, "host_cpus": os.cpu_count(),
                      "network": "R50 J17 D64 256x256 f16x3 random init", "frame": "1000x1000 q90 JPEG"}))


if __name__ == "__main__":
    main()
