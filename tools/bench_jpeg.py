"""Device JPEG decode on one GPU.  Tiles the two 1000x1002 q90 4:2:0 fixture frames of
tests/golden/jpeg.npz to a batch of 128 (one training step's frames: 32 tuples x 4 views) and
prints JSON lines, each with the card name, power limit and max SM clock:
  decode        CUDA-event time per batch, frames/s, compressed MB/s, decoded GB/s, and the stage
                breakdown (unstuff, phase A + its rounds, phase B/C, IDCT, upsample/colour);
  files_to_patches  decode + 256x256 patch_sample per batch, and the host->device bytes of this
                path next to uploading decoded frames (counted, not timed);
  interference  the R50 self-supervised training step (GraphedTrainStep replay) alone and with
                the next batch's decode + crop on a side stream, alternated;
  host_cv2      cv2.imdecode frames/s on one and on all host cores (a CPU number), if cv2 imports.
    python tools/bench_jpeg.py [--reps 20] [--rounds 3] [--steps 10]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

B = 128


def card():
    r = {"gpu": torch.cuda.get_device_name(), "power_limit_w": None, "max_sm_clock_mhz": None}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        pl, clk = q.stdout.strip().splitlines()[0].split(",")
        r["power_limit_w"], r["max_sm_clock_mhz"] = float(pl), float(clk)
    except Exception:
        pass
    return r


def fixture_blobs():
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg.npz"))
    names = list(g["names"])
    two = [g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes()
           for i in (names.index("frame1000_a"), names.index("frame1000_b"))]
    return [two[i % 2] for i in range(B)]


def ev():
    e = torch.cuda.Event(enable_timing=True)
    e.record()
    return e


def bench_decode(blobs, reps, base):
    import lib.utils.img_utils as iu
    from epipolarpose_b200 import _lib
    stats = torch.zeros(_lib.EPB_JPEG_STATS, dtype=torch.int32, device="cuda")
    events = [ev() for _ in range(_lib.EPB_JPEG_EVENTS)]
    for _ in range(3):
        f = iu.decode_jpeg_batch_device(blobs)
    torch.cuda.synchronize()
    tot, stage = [], np.zeros(_lib.EPB_JPEG_EVENTS - 1)
    for _ in range(reps):
        f = iu.decode_jpeg_batch_device(blobs, stats=stats, events=events)
        torch.cuda.synchronize()
        t = [events[i].elapsed_time(events[i + 1]) for i in range(len(events) - 1)]
        stage += t
        tot.append(sum(t))
    assert list(f.status) == [0] * B
    st = stats.cpu().numpy()
    rounds = int(np.argmin(st[:6])) + 1 if (st[:6] == 0).any() else 6
    ms = float(np.median(tot))
    comp = sum(len(b) for b in blobs)
    dec = sum(h * w * 3 for h, w in f.sizes)
    names = ["unstuff", "phase_a", "phase_bc", "idct", "upsample_colour"]
    out = dict(base, line="decode", batch=B, ms_per_batch=round(ms, 3), frames_per_s=round(B / ms * 1e3, 1),
               compressed_MB_per_s=round(comp / ms / 1e3, 1), decoded_GB_per_s=round(dec / ms / 1e6, 2),
               stage_ms={k: round(v / reps, 3) for k, v in zip(names, stage)}, phase_a_rounds=rounds,
               sequential_walk=bool(st[6]), step_consumes_frames_per_s=1526)
    print(json.dumps(out), flush=True)
    return f


def bench_patches(blobs, reps, base):
    import lib.utils.img_utils as iu
    rng = np.random.default_rng(0)
    cx, cy = 500 + rng.uniform(-50, 50, B), 500 + rng.uniform(-50, 50, B)
    w = 800 + rng.uniform(-100, 100, B)

    def run():
        f = iu.decode_jpeg_batch_device(blobs)
        return iu.generate_patch_batch_device(f, cx, cy, w, w, 256, 256)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0 = ev()
    for _ in range(reps):
        run()
    e1 = ev()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    comp = sum((len(b) + 16 + 15) // 16 * 16 for b in blobs) + B * (8192 + 8 + 8 + 12 + 4)
    frames = B * (1000 * 1002 * 3)
    print(json.dumps(dict(base, line="files_to_patches", batch=B, ms_per_batch=round(ms, 3),
                          frames_per_s=round(B / ms * 1e3, 1), h2d_bytes_jpeg_path=comp,
                          h2d_bytes_decoded_frame_path=frames)), flush=True)
    return cx, cy, w


def bench_interference(blobs, rounds, steps, base, crop):
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    from tools.bench_relpose import step_ms
    state = {}
    step_ms(False, 1, torch.device("cuda"), state)          # builds the R50 model, data and meta
    stepper = fn.GraphedTrainStep(state["model"], state["crit"], state["opt"], online=True, method="iterative")
    for i in range(3):                                      # eager, capture, replay
        stepper(state["x"][i % 2], meta=state["meta"])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    cx, cy, w = crop

    def run(with_decode):
        e0 = ev()
        for i in range(steps):
            stepper(state["x"][i % 2], meta=state["meta"])
            if with_decode:                                 # the next batch, on a side stream
                with torch.cuda.stream(side):
                    f = iu.decode_jpeg_batch_device(blobs)
                    iu.generate_patch_batch_device(f, cx, cy, w, w, 256, 256)
        torch.cuda.current_stream().wait_stream(side)
        e1 = ev()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps
    alone, busy = [], []
    for _ in range(rounds):
        alone.append(run(False))
        busy.append(run(True))
    print(json.dumps(dict(base, line="interference", step_ms_alone=[round(v, 2) for v in alone],
                          step_ms_with_decode=[round(v, 2) for v in busy],
                          median_difference_ms=round(float(np.median(np.array(busy) - np.array(alone))), 3))),
          flush=True)


def bench_host(blobs, base):
    try:
        import cv2
    except ImportError:
        print(json.dumps(dict(base, line="host_cv2", cpu="not measured (cv2 not importable)")), flush=True)
        return
    import concurrent.futures
    bufs = [np.frombuffer(b, np.uint8) for b in blobs[:32]]
    flags = cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for b in bufs:
        cv2.imdecode(b, flags)
    one = len(bufs) / (time.perf_counter() - t0)
    n = os.cpu_count() or 1
    work = bufs * max(1, n // 4)
    with concurrent.futures.ThreadPoolExecutor(n) as ex:
        t0 = time.perf_counter()
        list(ex.map(lambda b: cv2.imdecode(b, flags), work))
        allc = len(work) / (time.perf_counter() - t0)
    print(json.dumps(dict(base, line="host_cv2", cpu_number=True, cores=n, frames_per_s_one_core=round(one, 1),
                          frames_per_s_all_cores=round(allc, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    from epipolarpose_b200 import ops
    ops.device_check()
    base = card()
    blobs = fixture_blobs()
    bench_decode(blobs, args.reps, base)
    crop = bench_patches(blobs, args.reps, base)
    bench_interference(blobs, args.rounds, args.steps, base, crop)
    bench_host(blobs, base)


if __name__ == "__main__":
    main()
