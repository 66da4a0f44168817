"""CPU: the lossless JPEG transcode of csrc/jpeg.cu (symbol, Annex K.2 table, length and write
bodies, and the header) built for the CPU by tests/harness/host_jpeg_transcode.cu, which also
decodes each output again with the decoder's bodies.  Outputs are checked against cv2.imdecode of
the source, the parser's view of the output (DRI, number of intervals) and the source's
coefficients; the table builder against a restatement of Annex K.2."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from tests.conftest import ROOT
from tests.transcode_cases import INTERVALS, MALFORMED, OK, UNSUPPORTED, _build, _runner


@pytest.fixture(scope="module")
def host_exe(tmp_path_factory):
    return _build(tmp_path_factory, "host_jpeg_transcode", ["-O1"])


@pytest.fixture(scope="module")
def host_tc(host_exe):
    return _runner(host_exe)


@pytest.fixture(scope="module")
def cases(golden):
    g = golden("jpeg")
    return [dict(name=str(n), kind=str(g["kind"][i]), blob=g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes())
            for i, n in enumerate(g["names"])]


def _mcus(blob):
    """MCU count from SOF0/1 (8-bit baseline, the only kind the device decodes)."""
    i = 2
    while True:
        m, ln = blob[i + 1], (blob[i + 2] << 8) | blob[i + 3]
        if m in (0xC0, 0xC1):
            s = blob[i + 4:i + 2 + ln]
            H, W, nc = (s[1] << 8) | s[2], (s[3] << 8) | s[4], s[5]
            h = max(s[7 + 3 * c] >> 4 for c in range(nc)) if nc > 1 else 1
            v = max(s[7 + 3 * c] & 15 for c in range(nc)) if nc > 1 else 1
            return -(-W // (8 * h)) * -(-H // (8 * v))
        i += 2 + ln


def _check_structure(blob, r, R):
    assert r["status"] == OK
    if R:
        assert r["ri"] == R
    assert r["coef_equal"] == 1
    assert r["out_ri"] == r["ri"]
    assert r["nint"] == -(-_mcus(blob) // r["ri"]) == r["out_nseg"]
    assert r["out"][:2] == b"\xff\xd8" and r["out"][-2:] == b"\xff\xd9"


def _imdecode(cv2, b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)


@pytest.mark.parametrize("R", INTERVALS)
def test_goldens_every_interval(host_tc, cases, R):
    ok = [c for c in cases if c["kind"] == "ok"]
    res = host_tc([c["blob"] for c in ok], R)
    for c, r in zip(ok, res):
        _check_structure(c["blob"], r, R)
    cv2 = pytest.importorskip("cv2")
    for c, r in zip(ok, res):
        assert np.array_equal(_imdecode(cv2, r["out"]), _imdecode(cv2, c["blob"])), (c["name"], R)


def test_auto_interval_of_the_fixture_frame(host_tc, cases):
    """The 82 KB 1000x1002 4:2:0 frame: about 166 bits per MCU, so R = 4."""
    c = next(c for c in cases if c["name"] == "frame1000_a")
    assert len(c["blob"]) // 1000 == 82
    assert host_tc([c["blob"]], 0)[0]["ri"] == 4


def test_frame_intervals_against_subsequence_length(host_tc, cases):
    """At R = auto the mean interval is at most 768 bits but single intervals are not bounded:
    the largest interval and the share above kJpegSubBits = 1024 bits (stated in DESIGN.md 5)."""
    got = {}
    for tag in ("a", "b"):
        c = next(c for c in cases if c["name"] == "frame1000_" + tag)
        r = host_tc([c["blob"]], 0)[0]
        got[tag] = (r["ri"], r["nint"], int(r["bits"].max()), int((r["bits"] > 1024).sum()))
        mean = r["bits"].sum() / r["nint"]
        assert mean <= 768, (tag, mean)
        sys.stdout.write("frame1000_%s: R %d, %d intervals, mean %.0f bits, largest %d bits, %d over 1024 (%.1f %%)\n"
                         % (tag, got[tag][0], got[tag][1], mean, got[tag][2], got[tag][3],
                            100.0 * got[tag][3] / got[tag][1]))
    assert got == {"a": (4, 993, 3379, 105), "b": (5, 794, 3107, 48)}


def test_unsupported_and_truncated_statuses(host_tc, cases):
    other = [c for c in cases if c["kind"] != "ok"]
    for c, r in zip(other, host_tc([c["blob"] for c in other], 0)):
        assert r["status"] == {"unsupported": UNSUPPORTED, "truncated": MALFORMED}[c["kind"]], c["name"]
        assert r["out"] == b""


def test_live_cv2_sweep(host_tc):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(17)
    samp = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
            cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, None]
    blobs = {R: [] for R in INTERVALS}
    for n in range(300):
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
        blobs[INTERVALS[n % len(INTERVALS)]].append(buf.tobytes())
    for R, bl in blobs.items():
        for i, (b, r) in enumerate(zip(bl, host_tc(bl, R))):
            _check_structure(b, r, R)
            assert np.array_equal(_imdecode(cv2, r["out"]), _imdecode(cv2, b)), (R, i)


# ------------------------------------------------------------------ Annex K.2
def k2_restated(counts):
    """Annex K.2 (K.1 code sizes with the reserved symbol 256 of count 1, K.2 counts per length,
    K.3 limit to 16 bits and drop of the reserved code, K.4 order); of equal counts the larger
    symbol is taken first.  -> (bits[17], val list)."""
    freq = {s: int(c) for s, c in enumerate(counts) if c > 0}
    if not freq:
        return [0] * 17, []
    freq[256] = 1
    size = dict.fromkeys(freq, 0)
    nxt = dict.fromkeys(freq, None)
    while True:
        live = sorted((s for s in freq if freq[s] > 0), key=lambda s: (freq[s], -s))
        if len(live) < 2:
            break
        v1, v2 = live[0], live[1]
        freq[v1] += freq[v2]
        freq[v2] = 0
        size[v1] += 1
        while nxt[v1] is not None:
            v1 = nxt[v1]
            size[v1] += 1
        nxt[v1] = v2
        size[v2] += 1
        while nxt[v2] is not None:
            v2 = nxt[v2]
            size[v2] += 1
    bits = np.zeros(max(size.values()) + 1, np.int64)
    for s in size:
        bits[size[s]] += 1
    i = len(bits) - 1
    while i > 16:
        if bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
        else:
            i -= 1
    i = min(16, len(bits) - 1)
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    val = [s for s in sorted(size, key=lambda s: (size[s], s)) if s != 256]
    out = [0] * 17
    for l in range(1, min(17, len(bits))):
        out[l] = int(bits[l])
    return out, val


def _histograms():
    rng = np.random.default_rng(3)
    out = [np.zeros(256, np.int64) for _ in range(3)]
    out[0][7] = 5                                        # one symbol
    out[1][:] = 1                                        # all 256, counts of 1
    out[2][:] = rng.integers(1, 4, 256)                  # all 256, many ties
    fib = np.zeros(256, np.int64)                        # Fibonacci counts: unlimited codes far past 16 bits
    a, b = 1, 1
    for s in range(40):
        fib[s] = a
        a, b = b, a + b
    out.append(fib)
    dc = np.zeros(16, np.int64)
    dc[[0, 3, 11]] = [1, 1, 1]
    out.append(dc)
    for _ in range(40):
        n = 16 if rng.uniform() < 0.3 else 256
        h = np.where(rng.uniform(size=n) < rng.uniform(0.05, 1), rng.geometric(rng.uniform(1e-4, 0.5), n), 0)
        out.append(h.astype(np.int64))
    return out


def test_table_builder_against_annex_k2(host_exe):
    hs = _histograms()
    inp = struct.pack("<i", len(hs)) + b"".join(struct.pack("<i", len(h)) + h.astype("<i8").tobytes() for h in hs)
    r = subprocess.run([host_exe, "table"], input=inp, capture_output=True)
    assert r.returncode == 0, r.stderr
    for k, h in enumerate(hs):
        rec = r.stdout[k * 273:(k + 1) * 273]
        bits = list(rec[:17])
        n = sum(bits)
        val = list(rec[17:17 + n])
        want_bits, want_val = k2_restated(h)
        assert bits == want_bits and val == want_val, k
        assert n == int((h > 0).sum())
        assert sorted(val) == list(np.nonzero(h)[0])
        assert max(l for l in range(17) if bits[l] or l == 0) <= 16
        assert sum(bits[l] * 2.0 ** -l for l in range(1, 17)) < 1.0, k


def test_harness_under_sanitizers(tmp_path_factory, cases):
    exe = _build(tmp_path_factory, "host_jpeg_transcode_san",
                 ["-O1", "-Xcompiler", "-fsanitize=address", "-Xcompiler", "-fsanitize=undefined",
                  "-Xcompiler", "-fno-sanitize-recover=all", "-lasan", "-lubsan"])
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1", UBSAN_OPTIONS="halt_on_error=1")
    run = _runner(exe)
    blobs = [c["blob"] for c in cases if "frame1000" not in c["name"]]
    for R in (1, 0):
        for c, r in zip([c for c in cases if "frame1000" not in c["name"]], run(blobs, R, env)):
            assert r["status"] == {"ok": OK, "unsupported": UNSUPPORTED, "truncated": MALFORMED}[c["kind"]]


def test_prep_frames_refuses_overlapping_trees(tmp_path):
    src = tmp_path / "src"
    (src / "images").mkdir(parents=True)
    (src / "annot").mkdir()
    for dst in (src, src / "prepared", tmp_path):
        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "prep_frames.py"), str(src), str(dst)],
                           capture_output=True, text=True)
        assert r.returncode != 0 and "overlap" in r.stderr, (dst, r.stderr)
    assert sorted(os.listdir(src)) == ["annot", "images"]
