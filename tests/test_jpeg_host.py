"""CPU: the JPEG decoder of csrc/jpeg.cu -- parser, self-synchronising Huffman decode (phase A / B /
C bodies), ISLOW IDCT, fancy upsampling and colour -- built for the CPU by
tests/harness/host_jpeg.cu and checked against cv2.imdecode (tests/golden/jpeg.npz, and live cv2
when it is importable).  The subsequence length is swept so that synchronisation happens many
times even in small images; the coefficients must equal a plain sequential decode."""
import hashlib
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from tests.conftest import ROOT

OK, UNSUPPORTED, MALFORMED = 0, 1, 2


@pytest.fixture(scope="module")
def host_jpeg(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / "host_jpeg")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O1", "-std=c++17", "-o", exe,
                        os.path.join(ROOT, "tests", "harness", "host_jpeg.cu")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(blobs, sub_bits=1024, order="fwd"):
        inp = struct.pack("<i", len(blobs)) + b"".join(struct.pack("<q", len(b)) + bytes(b) for b in blobs)
        out = subprocess.run([exe, str(sub_bits), order], input=inp, capture_output=True)
        assert out.returncode == 0, out.stderr
        res, pos = [], 0
        for _ in blobs:
            st, H, W, eq, rounds = struct.unpack_from("<5i", out.stdout, pos)
            pos += 20
            pix = None
            if st == OK:
                pix = np.frombuffer(out.stdout, np.uint8, H * W * 3, pos).reshape(H, W, 3)
                pos += H * W * 3
            res.append(dict(status=st, H=H, W=W, coef_equal=eq, rounds=rounds, pix=pix))
        return res
    return run


@pytest.fixture(scope="module")
def jpeg_cases(golden):
    g = golden("jpeg")
    out = []
    for i, name in enumerate(g["names"]):
        blob = g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes()
        H, W = g["hw"][i]
        pix = g["pix_data"][g["pix_off"][i]:g["pix_off"][i + 1]]
        out.append(dict(name=str(name), kind=str(g["kind"][i]), blob=blob, hw=(int(H), int(W)),
                        pix=pix.reshape(H, W, 3) if pix.size else None, sha=str(g["sha256"][i])))
    return out


def _expect(case, r):
    assert (r["H"], r["W"]) == case["hw"], case["name"]
    if case["pix"] is not None:
        assert np.array_equal(r["pix"], case["pix"]), case["name"]
    else:
        assert hashlib.sha256(np.ascontiguousarray(r["pix"]).tobytes()).hexdigest() == case["sha"], case["name"]


def test_parser_status_every_case(host_jpeg, jpeg_cases):
    res = host_jpeg([c["blob"] for c in jpeg_cases])
    for c, r in zip(jpeg_cases, res):
        want = {"ok": OK, "unsupported": UNSUPPORTED, "truncated": MALFORMED}[c["kind"]]
        assert r["status"] == want, (c["name"], r["status"])


@pytest.mark.parametrize("sub_bits,order", [(1024, "fwd"), (64, "fwd"), (32, "rev")])
def test_goldens_bit_exact_and_sync_equals_sequential(host_jpeg, jpeg_cases, sub_bits, order):
    ok = [c for c in jpeg_cases if c["kind"] == "ok"]
    res = host_jpeg([c["blob"] for c in ok], sub_bits, order)
    for c, r in zip(ok, res):
        assert r["status"] == OK, c["name"]
        assert r["coef_equal"] == 1, c["name"]
        _expect(c, r)
    if sub_bits == 32:                      # many subsequences: synchronisation was exercised
        assert max(r["rounds"] for r in res) >= 2


def _segments(blob):
    """(marker, payload start, length) of every marker segment before the entropy data."""
    out, i = [], 2
    while i + 4 <= len(blob):
        m, ln = blob[i + 1], (blob[i + 2] << 8) | blob[i + 3]
        out.append((m, i, ln))
        if m == 0xDA:
            break
        i += 2 + ln
    return out


def test_malformed_inputs_are_statuses(host_jpeg, jpeg_cases):
    base = next(c for c in jpeg_cases if c["name"] == "q90_420")["blob"]
    segs = _segments(base)
    bad = []
    bad.append(base[:len(base) // 2])                                   # entropy data ends early
    dht = next(s for s in segs if s[0] == 0xC4)
    b = bytearray(base)
    b[dht[1] + 5] = 3                       # three 1-bit codes in the first table: over-full
    bad.append(bytes(b))
    dqt = next(s for s in segs if s[0] == 0xDB)
    b = bytearray(base)
    b[dqt[1] + 4] = (b[dqt[1] + 4] & 0xF0) | 5                           # table index 5
    bad.append(bytes(b))
    sof = next(s for s in segs if s[0] == 0xC0)
    b = bytearray(base)
    b[sof[1] + 7] = 0
    b[sof[1] + 8] = 0                                                   # width 0
    bad.append(bytes(b))
    bad.append(base[:40])                                               # header cut short
    bad.append(b"\xff\xd8\xff\xd9")
    for r in host_jpeg(bad, 64):
        assert r["status"] == MALFORMED, r


def test_live_cv2_sweep(host_jpeg):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    samp = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, None]
    blobs, want = [], []
    for _ in range(300):
        H, W = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        s = samp[int(rng.integers(0, 5))]
        y, x = np.mgrid[0:H, 0:W]
        img = (128 + 80 * np.sin(x * rng.uniform(0.02, 0.4) + y * rng.uniform(0.02, 0.4))[..., None] +
               rng.normal(0, 8, (H, W, 3))).clip(0, 255).astype(np.uint8)
        if s is None:
            img = img[:, :, 0]
        p = [cv2.IMWRITE_JPEG_QUALITY, int(rng.integers(30, 101))]
        if s is not None:
            p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, s]
        if rng.uniform() < 0.3:
            p += [cv2.IMWRITE_JPEG_RST_INTERVAL, int(rng.integers(1, 20))]
        if rng.uniform() < 0.3:
            p += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
        ok, buf = cv2.imencode(".jpg", img, p)
        assert ok
        blobs.append(buf.tobytes())
        want.append(cv2.imdecode(buf, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION))
    for i, r in enumerate(host_jpeg(blobs, 64)):
        assert r["status"] == OK and r["coef_equal"] == 1, i
        assert np.array_equal(r["pix"], want[i]), i
