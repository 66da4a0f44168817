"""Prepare a Human3.6M or MPII frame tree for the device JPEG decoder: every JPEG under
SRC/images is transcoded losslessly on the GPU (transcode_jpeg_batch_device: the quantised
coefficients are kept, restart intervals short enough that the decoder's Huffman stage starts
from exact states, Huffman tables regenerated) and written to the same relative path under
DST/images.  Every decoder gives the same pixels as from SRC, so training and evaluation inputs
do not change; point DATASET.ROOT at DST.  Files the device cannot transcode (progressive,
4:1:1, CMYK, malformed, ...) and files that are not JPEG are copied unchanged.  Bytes after a
JPEG's EOI are dropped.  DST/annot links to SRC/annot (a copy where links are not possible).
SRC is only read; DST may not lie inside SRC, nor SRC inside DST.  Prints one JSON summary.
    python tools/prep_frames.py SRC DST [--interval auto|N] [--batch 128]"""
import argparse
import json
import os
import shutil
import sys
import time

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
REASONS = {1: "unsupported", 2: "malformed", 3: "verify_mismatch"}


def _inside(a, b):
    """a is b or lies under b."""
    return a == b or a.startswith(b.rstrip(os.sep) + os.sep)


def check_trees(src, dst):
    src, dst = os.path.realpath(src), os.path.realpath(dst)
    if _inside(dst, src) or _inside(src, dst):
        raise SystemExit("prep_frames: SRC %s and DST %s overlap; DST must lie outside SRC and SRC outside DST"
                         % (src, dst))
    if not os.path.isdir(os.path.join(src, "images")):
        raise SystemExit("prep_frames: %s has no images/ directory" % src)
    return src, dst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("src")
    ap.add_argument("dst")
    ap.add_argument("--interval", default="auto", help="restart interval in MCUs, or auto")
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    src, dst = check_trees(args.src, args.dst)
    interval = args.interval if args.interval == "auto" else int(args.interval)
    for p in (ROOT, os.path.join(ROOT, "epipolarpose_b200")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import lib.utils.img_utils as iu

    files = []
    for d, _, names in os.walk(os.path.join(src, "images")):
        for n in sorted(names):
            files.append(os.path.relpath(os.path.join(d, n), src))
    files.sort()
    jpegs = [f for f in files if f.lower().endswith((".jpg", ".jpeg"))]
    summary = dict(frames=len(jpegs), transcoded=0, passed_through={}, other_files=len(files) - len(jpegs),
                   bytes_in=0, bytes_out=0)

    def write(rel, data):
        p = os.path.join(dst, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, "wb") as f:
            f.write(data)

    t0 = time.perf_counter()
    for k in range(0, len(jpegs), args.batch):
        part = jpegs[k:k + args.batch]
        blobs = []
        for rel in part:
            with open(os.path.join(src, rel), "rb") as f:
                blobs.append(f.read())
        out, status = iu.transcode_jpeg_batch_device(blobs, interval=interval, verify=True)
        for rel, b, o, s in zip(part, blobs, out, status):
            write(rel, o)
            summary["bytes_in"] += len(b)
            summary["bytes_out"] += len(o)
            if s == 0:
                summary["transcoded"] += 1
            else:
                why = REASONS.get(int(s), str(int(s)))
                summary["passed_through"][why] = summary["passed_through"].get(why, 0) + 1
    dt = time.perf_counter() - t0
    jset = set(jpegs)
    for rel in files:
        if rel not in jset:
            os.makedirs(os.path.dirname(os.path.join(dst, rel)), exist_ok=True)
            shutil.copy2(os.path.join(src, rel), os.path.join(dst, rel))
    annot = os.path.join(src, "annot")
    if os.path.isdir(annot) and not os.path.exists(os.path.join(dst, "annot")):
        try:
            os.symlink(annot, os.path.join(dst, "annot"), target_is_directory=True)
            summary["annot"] = "linked"
        except OSError:
            shutil.copytree(annot, os.path.join(dst, "annot"))
            summary["annot"] = "copied"
    summary["frames_per_s"] = round(len(jpegs) / dt, 1) if dt > 0 else None
    summary["size_ratio"] = round(summary["bytes_out"] / summary["bytes_in"], 4) if summary["bytes_in"] else None
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
