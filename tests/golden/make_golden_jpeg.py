"""Writes tests/golden/jpeg.npz: JPEG blobs encoded with cv2.imencode from seeded, natural-looking
frames (smooth gradients, edges, mild noise), and what cv2.imdecode(blob, IMREAD_COLOR |
IMREAD_IGNORE_ORIENTATION) makes of them -- the frames get_single_patch_sample reads.

Arrays: names, kind ('ok' | 'unsupported' | 'truncated'), blob_data + blob_off (blob i is
blob_data[blob_off[i]:blob_off[i+1]]), hw [n,2], sha256 (of cv2's decoded BGR frame, C order), and
pix_data + pix_off: the frame itself for frames of at most SMALL pixels (empty otherwise).  A frame
is checked bit for bit by its hash; storing every frame would make the file megabytes.  The two
1000x1002 frames are what tools/bench_jpeg.py tiles.
    python tests/golden/make_golden_jpeg.py"""
import hashlib
import os
import struct

import cv2
import numpy as np

FLAGS = cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION
SAMPLING = {"444": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, "422": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            "440": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, "420": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420,
            "411": cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411}
SMALL = 40 * 40
MID = (120, 136)             # H, W of the quality / optimise / restart / EXIF / fallback cases


def frame(rng, H, W, gray=False):
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    ch = []
    for _ in range(1 if gray else 3):
        f = rng.uniform(0.002, 0.03, 2)
        v = 128 + 60 * np.sin(x * f[0] + rng.uniform(0, 6)) * np.cos(y * f[1] + rng.uniform(0, 6))
        v += rng.uniform(-0.1, 0.1) * x + rng.uniform(-0.1, 0.1) * y
        ch.append(v)
    img = np.stack(ch, axis=2)
    for _ in range(6):                                   # hard edges: boxes and discs
        c = rng.uniform(0, 255, img.shape[2])
        cx, cy, r = rng.uniform(0, W), rng.uniform(0, H), rng.uniform(2, max(3, min(H, W) / 3))
        m = ((x - cx) ** 2 + (y - cy) ** 2 < r * r) if rng.uniform() < 0.5 else \
            ((np.abs(x - cx) < r) & (np.abs(y - cy) < r * 0.6))
        img[m] = c
    img += rng.normal(0, 1.5, img.shape)
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    return img[:, :, 0] if gray else img


def encode(img, q=75, sampling="420", optimize=False, rst=0, progressive=False):
    p = [cv2.IMWRITE_JPEG_QUALITY, q]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    if optimize:
        p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if progressive:
        p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode(".jpg", img, p)
    assert ok
    return buf.tobytes()


def with_exif_orientation(blob, orientation=6):
    """An APP1 EXIF segment (one IFD0 entry: Orientation) spliced in right after SOI."""
    tiff = b"II*\x00" + struct.pack("<I", 8) + struct.pack("<H", 1) + \
        struct.pack("<HHII", 0x0112, 3, 1, orientation) + struct.pack("<I", 0)
    payload = b"Exif\x00\x00" + tiff
    return blob[:2] + b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload + blob[2:]


def cases():
    rng = np.random.default_rng(20261016)
    out = []
    for (H, W) in [(1, 1), (7, 9), (8, 8), (16, 16), (17, 33), (255, 257)]:
        for s in ("444", "422", "440", "420", "gray"):
            img = frame(rng, H, W, gray=s == "gray")
            out.append(("s%dx%d_%s" % (H, W, s), "ok", encode(img, 75, s)))
    base = frame(rng, *MID)
    for q in (50, 90, 95, 100):
        for s in ("420", "444"):
            out.append(("q%d_%s" % (q, s), "ok", encode(base, q, s)))
    for s in ("420", "444", "gray"):
        img = frame(rng, *MID, gray=s == "gray")
        out.append(("opt_%s" % s, "ok", encode(img, 90, s, optimize=True)))
    for r, s in ((1, "420"), (4, "420"), (17, "420"), (17, "422"), (5, "gray")):
        img = frame(rng, *MID, gray=s == "gray")
        if r == 17:                            # the last restart interval is a partial one
            mh, mw = {"420": (16, 16), "422": (8, 16)}[s]
            assert (-(-MID[0] // mh) * -(-MID[1] // mw)) % r != 0
        out.append(("rst%d_%s" % (r, s), "ok", encode(img, 90, s, optimize=(r == 4), rst=r)))
    exif = encode(base, 90, "420")
    out.append(("exif_orientation6", "ok", with_exif_orientation(exif)))
    out.append(("progressive", "unsupported", encode(base, 90, "420", progressive=True)))
    out.append(("s411", "unsupported", encode(base, 90, "411")))
    trunc = encode(frame(rng, *MID), 90, "420")
    out.append(("truncated", "truncated", trunc[:len(trunc) * 3 // 5]))
    for tag in ("a", "b"):
        out.append(("frame1000_" + tag, "ok", encode(frame(rng, 1000, 1002), 90, "420")))
    return out


def main():
    names, kinds, blobs, pix, hw, sha = [], [], [], [], [], []
    for name, kind, blob in cases():
        img = cv2.imdecode(np.frombuffer(blob, np.uint8), FLAGS)
        if kind == "truncated":
            assert img is None, "cv2 decodes the truncated blob"
            img = np.zeros((0, 0, 3), np.uint8)
        names.append(name)
        kinds.append(kind)
        blobs.append(np.frombuffer(blob, np.uint8))
        hw.append(img.shape[:2])
        sha.append(hashlib.sha256(img.tobytes()).hexdigest())
        pix.append(img.reshape(-1) if img.shape[0] * img.shape[1] <= SMALL else np.zeros(0, np.uint8))
    off = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.int64)
    poff = np.concatenate([[0], np.cumsum([len(p) for p in pix])]).astype(np.int64)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "jpeg.npz")
    np.savez_compressed(path, names=np.array(names), kind=np.array(kinds), blob_data=np.concatenate(blobs),
                        blob_off=off, hw=np.array(hw, np.int32), pix_data=np.concatenate(pix), pix_off=poff,
                        sha256=np.array(sha))
    print(path, os.path.getsize(path), "bytes,", len(names), "cases")


if __name__ == "__main__":
    main()
