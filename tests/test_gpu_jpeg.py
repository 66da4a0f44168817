"""GPU: decode_jpeg_batch_device (csrc/jpeg.cu) against cv2.imdecode's frames
(tests/golden/jpeg.npz), in one mixed batch and one image at a time; the host fallback for
unsupported and malformed blobs; device frames straight into the patch sampler; the batched,
device-decoded get_patch_batch_device against B get_single_patch_sample calls."""
import hashlib
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cases(golden):
    g = golden("jpeg")
    out = []
    for i, name in enumerate(g["names"]):
        H, W = (int(v) for v in g["hw"][i])
        pix = g["pix_data"][g["pix_off"][i]:g["pix_off"][i + 1]]
        out.append(dict(name=str(name), kind=str(g["kind"][i]),
                        blob=g["blob_data"][g["blob_off"][i]:g["blob_off"][i + 1]].tobytes(), hw=(H, W),
                        pix=pix.reshape(H, W, 3) if pix.size else None, sha=str(g["sha256"][i])))
    return out


@pytest.fixture(scope="module")
def cv2_frames(cases):
    """cv2's decode of every supported case as a host array: the stored frame, or else the frame
    decoded alone on the device once its SHA-256 equals that of cv2's frame."""
    import lib.utils.img_utils as iu
    out = {}
    for c in cases:
        if c["kind"] != "ok":
            continue
        if c["pix"] is not None:
            out[c["name"]] = c["pix"]
            continue
        f = iu.decode_jpeg_batch_device([c["blob"]]).frame(0).cpu().numpy()
        assert hashlib.sha256(f.tobytes()).hexdigest() == c["sha"], c["name"]
        out[c["name"]] = f
    return out


def _parity_cases(cases):
    return [c for c in cases if c["kind"] == "ok" and min(c["hw"]) >= 16]


def _have_cv2():
    try:
        import cv2  # noqa: F401
        return True
    except ImportError:
        return False


def _check(frames, i, c):
    assert frames.sizes[i] == c["hw"], c["name"]
    got = frames.frame(i).cpu().numpy()
    if c["pix"] is not None:
        assert np.array_equal(got, c["pix"]), c["name"]
    else:
        assert hashlib.sha256(got.tobytes()).hexdigest() == c["sha"], c["name"]


def test_goldens_mixed_batch_and_singly(cases):
    import lib.utils.img_utils as iu
    dec = [c for c in cases if c["kind"] == "ok"]
    frames = iu.decode_jpeg_batch_device([c["blob"] for c in dec])
    assert list(frames.status) == [0] * len(dec)
    for i, c in enumerate(dec):
        _check(frames, i, c)
    for c in dec:
        one = iu.decode_jpeg_batch_device([np.frombuffer(c["blob"], np.uint8)])
        assert np.array_equal(one.frame(0).cpu().numpy(), frames.frame(dec.index(c)).cpu().numpy()), c["name"]


def test_truncated_blob_raises(cases):
    import lib.utils.img_utils as iu
    trunc = next(c for c in cases if c["kind"] == "truncated")
    good = next(c for c in cases if c["name"] == "q90_420")
    with pytest.raises(IOError, match="blob 1"):
        iu.decode_jpeg_batch_device([good["blob"], trunc["blob"]])


def test_unsupported_blobs_fall_back(cases):
    import lib.utils.img_utils as iu
    from epipolarpose_b200 import ops
    uns = [c for c in cases if c["kind"] == "unsupported"]
    bufs = [np.frombuffer(c["blob"], np.uint8) for c in uns]
    assert list(ops.jpeg_parse(bufs)[1]) == [1] * len(uns)
    if not _have_cv2():
        pytest.skip("cv2 not importable: the host fallback cannot run")
    frames = iu.decode_jpeg_batch_device([c["blob"] for c in uns] + [cases[0]["blob"]])
    for i, c in enumerate(uns):
        _check(frames, i, c)
    _check(frames, len(uns), cases[0])


def _occluders(rng, B, n_max=3):
    out = []
    for _ in range(B):
        occ = []
        for _ in range(int(rng.integers(1, n_max + 1))):
            h, w = int(rng.integers(8, 60)), int(rng.integers(8, 60))
            occ.append((rng.integers(0, 256, (h, w, 4), dtype=np.uint8), (int(rng.integers(0, 256)),
                                                                          int(rng.integers(0, 256)))))
        out.append(occ)
    return out


def test_patch_parity_device_frames_vs_host_frames(cases, cv2_frames):
    import lib.utils.img_utils as iu
    dec = _parity_cases(cases)
    B = len(dec)
    rng = np.random.default_rng(5)
    frames = iu.decode_jpeg_batch_device([c["blob"] for c in dec])
    hw = np.array([c["hw"] for c in dec], dtype=np.float64)
    args = (hw[:, 1] * rng.uniform(0.3, 0.7, B), hw[:, 0] * rng.uniform(0.3, 0.7, B), hw[:, 1] * 0.6, hw[:, 0] * 0.6,
            256, 256, rng.uniform(0.75, 1.25, B), rng.uniform(-60, 60, B), rng.uniform(size=B) < 0.5,
            rng.uniform(0.8, 1.2, (B, 3)), [123.675, 116.28, 103.53], [58.395, 57.12, 57.375])
    occ = _occluders(rng, B)
    a = iu.generate_patch_batch_device(frames, *args, occluders=occ)
    b = iu.generate_patch_batch_device([cv2_frames[c["name"]] for c in dec], *args, occluders=occ)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_batch_parity_with_single_patch_sample(cases, cv2_frames, tmp_path):
    import lib.utils.img_utils as iu
    dec = _parity_cases(cases)[::2]
    B, J = len(dec), 5
    paths = []
    for i, c in enumerate(dec):
        p = tmp_path / ("%02d.jpg" % i)
        p.write_bytes(c["blob"])
        paths.append(str(p))
    rng = np.random.default_rng(9)
    hw = np.array([c["hw"] for c in dec], dtype=np.float64)
    cx, cy = hw[:, 1] * rng.uniform(0.3, 0.7, B), hw[:, 0] * rng.uniform(0.3, 0.7, B)
    bw, bh = hw[:, 1] * 0.7, hw[:, 0] * 0.7
    joints = np.concatenate([rng.uniform(0, 1, (B, J, 2)) * hw[:, None, ::-1], rng.uniform(-500, 500, (B, J, 1))], 2)
    vis = np.ones((B, J, 3))
    occluder = None
    if _have_cv2():
        occluder = [np.random.default_rng(3).integers(0, 256, (40, 30, 4), dtype=np.uint8)]
    common = ([[0, 1]], None, 256, 256, 2000.0, 2000.0, [123.675, 116.28, 103.53], [58.395, 57.12, 57.375], True, None)
    np.random.seed(11)
    random.seed(11)
    got = iu.get_patch_batch_device(paths, cx, cy, bw, bh, joints, vis, *common, occluder=occluder)
    np.random.seed(11)
    random.seed(11)
    ref = [iu.get_single_patch_sample(cv2_frames[c["name"]], cx[i], cy[i], bw[i], bh[i], joints[i], vis[i], *common,
                                      occluder=occluder) for i, c in enumerate(dec)]
    assert np.array_equal(got[0].cpu().numpy(), np.stack([r[0] for r in ref]))
    assert np.array_equal(got[1], np.stack([r[1] for r in ref]))
    assert np.array_equal(got[2], np.stack([r[2] for r in ref]))
    assert np.array_equal(got[3], np.array([r[3] for r in ref], dtype=np.float64))
    assert np.array_equal(got[4], np.array([r[4] for r in ref], dtype=np.float64))


def test_decode_is_deterministic(cases):
    import lib.utils.img_utils as iu
    blobs = [c["blob"] for c in cases if c["kind"] == "ok"]
    a = iu.decode_jpeg_batch_device(blobs)
    b = iu.decode_jpeg_batch_device(blobs)
    for i in range(len(blobs)):
        assert torch.equal(a.frame(i), b.frame(i)), i
