"""Lossless transcode to short restart intervals (transcode_jpeg_batch_device) and what it buys
the device decoder and the h36m loader.  Builds tools/bench_data.py's tree of the two 1000x1002
q90 4:2:0 fixture frames, a transcoded copy of it (R = auto), and prints JSON lines, each with the
card name, power limit and max SM clock:
  transcode  (a) frames/s of transcode_jpeg_batch_device at 128 frames per call, verify off / on;
  decode     (b) decode_jpeg_batch_device of 128 original / transcoded frames, alternating in one
             loop: frames/s, median per-stage times from the EPB_JPEG_EVENTS marks, and the
             phase-A round flags (stats) of the last call;
  loader     (c) bench_data's DataLoader(8 workers) + assemble_batch frames/s and its fed R50
             step in ms/step, original / transcoded tree, alternating twice (both passes listed);
  size       (d) bytes of the transcoded frames over the originals.
    python tools/bench_transcode.py [--frames 2048] [--batches 8] [--iters 20]"""
import argparse
import gc
import json
import os
import random
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tools.bench_jpeg import card  # noqa: E402
from tools import bench_data as bd  # noqa: E402

STAGES = ("unstuff", "phase_a", "phase_bc", "idct", "colour")


def event():
    e = torch.cuda.Event(enable_timing=True)
    e.record()                                      # created on first record; the C ABI records it again
    return e


def timed(fn, iters):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2048)
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--layers", type=int, default=50)
    ap.add_argument("--precision", default=os.environ.get("EPB_PRECISION", "f16x3"))
    args = ap.parse_args()
    from epipolarpose_b200 import _lib, ops
    import lib.dataset as dataset
    import lib.utils.img_utils as iu
    ops.device_check()
    info = card()
    with tempfile.TemporaryDirectory() as tmp:
        orig, prep = os.path.join(tmp, "orig"), os.path.join(tmp, "prep")
        os.makedirs(orig)
        bd.make_tree(orig, args.frames)
        os.makedirs(os.path.join(prep, "images"))
        shutil.copytree(os.path.join(orig, "annot"), os.path.join(prep, "annot"))
        src = {}
        for tag in ("a", "b"):
            with open(os.path.join(orig, "images", tag + ".jpg"), "rb") as f:
                src[tag] = f.read()
        out, st = iu.transcode_jpeg_batch_device([src["a"], src["b"]])
        assert list(st) == [0, 0], st
        new = dict(a=out[0], b=out[1])
        for tag in ("a", "b"):
            with open(os.path.join(prep, "images", tag + ".jpg"), "wb") as f:
                f.write(new[tag])
        batch = {k: [d["ab"[i % 2]] for i in range(128)] for k, d in (("orig", src), ("prep", new))}

        # (a)
        for v in (False, True):
            iu.transcode_jpeg_batch_device(batch["orig"], verify=v)
        ms = {v: timed(lambda: iu.transcode_jpeg_batch_device(batch["orig"], verify=v), 5) for v in (False, True)}
        print(json.dumps(dict(info, bench="transcode", frames_per_call=128,
                              frames_per_s=round(128 / ms[False], 1), frames_per_s_verify=round(128 / ms[True], 1))),
              flush=True)

        # (b)
        ev = [event() for _ in range(_lib.EPB_JPEG_EVENTS)]
        stats = torch.zeros(_lib.EPB_JPEG_STATS, dtype=torch.int32, device="cuda")
        res = {k: dict(t=[], st=[]) for k in batch}
        for it in range(args.iters + 2):
            for k in ("orig", "prep"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                iu.decode_jpeg_batch_device(batch[k], stats=stats, events=ev)
                torch.cuda.synchronize()
                if it >= 2:
                    res[k]["t"].append(time.perf_counter() - t0)
                    res[k]["st"].append([ev[i].elapsed_time(ev[i + 1]) for i in range(len(STAGES))])
        for k in ("orig", "prep"):                     # the round flags of one more call of each
            iu.decode_jpeg_batch_device(batch[k], stats=stats)
            res[k]["stats"] = stats.cpu().tolist()
        for k in ("orig", "prep"):
            med = np.median(np.array(res[k]["st"]), axis=0)
            print(json.dumps(dict(info, bench="decode", tree=k, frames=128,
                                  frames_per_s=round(128 / float(np.median(res[k]["t"])), 1),
                                  call_ms=round(1e3 * float(np.median(res[k]["t"])), 2),
                                  device_ms=round(float(med.sum()), 2),
                                  **{s + "_ms": round(float(m), 3) for s, m in zip(STAGES, med)},
                                  stats=res[k]["stats"])), flush=True)

        # (c)
        fps, step = {}, {}
        for k, root in (("orig", orig), ("prep", prep), ("orig", orig), ("prep", prep)):
            cfg = bd.config(root, args.layers, args.precision)
            np.random.seed(0)
            random.seed(0)
            ds = dataset.h36m(cfg, root, "train", True)
            fps.setdefault(k, []).append(bd.bench_loader(ds, args.batches, 8))
            step.setdefault(k, []).append(bd.bench_step(cfg, ds, args.precision, args.batches)[0])
            gc.collect()                               # the model and its captured step graph hold each other
            torch.cuda.empty_cache()
        for k in ("orig", "prep"):
            print(json.dumps(dict(info, bench="loader", tree=k, workers=8, frames_per_batch=2 * bd.PAIRS,
                                  frames_per_s=[round(v, 1) for v in fps[k]],
                                  resident_ms_per_step=[round(v["resident"], 2) for v in step[k]],
                                  loader_ms_per_step=[round(v["loader"], 2) for v in step[k]])), flush=True)

        # (d)
        print(json.dumps(dict(info, bench="size", bytes_orig=len(src["a"]) + len(src["b"]),
                              bytes_transcoded=len(new["a"]) + len(new["b"]),
                              ratio=round((len(new["a"]) + len(new["b"])) / (len(src["a"]) + len(src["b"])), 4))),
              flush=True)


if __name__ == "__main__":
    main()
