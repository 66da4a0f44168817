"""Seeded synthetic inputs shared by the golden-vector generator
(tests/golden/make_golden.py, runs the reference in the build container) and
by the tests (which run anywhere).  numpy Generator streams are stable across
platforms, so only reference OUTPUTS need to be stored."""
import numpy as np

from oracle import restate

# tag -> (N, J, D, H, W, seed, logit scale)
SOFTARGMAX_CASES = {
    "small": (2, 3, 8, 8, 8, 11, 3.0),
    "cube16": (3, 5, 16, 16, 16, 12, 2.0),
    "ragged": (1, 2, 4, 12, 20, 13, 4.0),     # D != H != W
    "peaky": (2, 17, 16, 16, 16, 14, 12.0),
}


def logits(N, J, D, H, W, seed, scale):
    rng = np.random.default_rng(seed)
    return (scale * rng.standard_normal((N, J * D, H, W))).astype(np.float32)


def labels(N, J, seed):
    rng = np.random.default_rng(seed + 100)
    gt = (rng.uniform(-0.5, 0.5, (N, J * 3))).astype(np.float32)
    wt = (rng.uniform(0, 1, (N, J * 3)) > 0.2).astype(np.float32)
    return gt, wt


def argmax_heatmaps():
    rng = np.random.default_rng(21)
    hm = rng.standard_normal((3, 6, 16, 12)).astype(np.float32)
    hm[0, 0] = -np.abs(hm[0, 0])            # all negative -> masked to (0,0)
    hm[0, 1] = 0.0                           # all equal (ties) -> first index, masked (max == 0)
    hm[0, 2, 5, 7] = 9.0
    hm[0, 2, 9, 3] = 9.0                     # planted tie -> first occurrence (5,7)
    hm[1, 0, 15, 11] = 50.0                  # last element
    hm[1, 1, 0, 0] = 50.0                    # first element
    hm[2, 3] = np.float32(0.25)              # positive constant
    return hm


def triangulation_case(n_pairs=16, J=17, seed=31, noise_px=3.0):
    rng = np.random.default_rng(seed)
    R, T, f, c, P = restate.synthetic_cameras(rng, n_pairs, 4)
    X = rng.normal(0.0, 400.0, size=(n_pairs, J, 3))
    P1, P2 = P[:, 0], P[:, 1]
    u1 = np.stack([restate.project(P1[i], X[i]) for i in range(n_pairs)])
    u2 = np.stack([restate.project(P2[i], X[i]) for i in range(n_pairs)])
    u1 = u1 + rng.normal(0, noise_px, u1.shape)
    u2 = u2 + rng.normal(0, noise_px, u2.shape)
    return u1, u2, P1.copy(), P2.copy(), X


def exact_projections(P1, P2, X):
    u1 = np.stack([restate.project(P1[i], X[i]) for i in range(len(X))])
    u2 = np.stack([restate.project(P2[i], X[i]) for i in range(len(X))])
    return u1, u2


def patch_case(B=6, J=5, seed=41):
    rng = np.random.default_rng(seed)
    coords = np.concatenate([rng.uniform(0, 256, (B, J, 2)), rng.uniform(-128, 128, (B, J, 1)),
                             np.ones((B, J, 1))], axis=2)
    boxes = np.stack([500 + rng.uniform(-50, 50, B), 500 + rng.uniform(-50, 50, B),
                      800 + rng.uniform(-100, 100, B), 800 + rng.uniform(-100, 100, B),
                      np.array([1.0, 1.0, 1.1, 0.85, 1.25, 0.9]),
                      np.array([0.0, 0.0, 15.0, -30.0, 7.5, 0.0])], axis=1)
    return coords, boxes


def selfsup_case(n_tuples=2, J=4, D=16, seed=51):
    """Batch of 2*n_tuples*... laid out [view0 | view1] of each tuple, logits whose
    soft-argmax lands near the projection of a true 3-D pose."""
    rng = np.random.default_rng(seed)
    R, T, f, c, P = restate.synthetic_cameras(rng, n_tuples, 4)
    B = 2 * n_tuples
    views = [(t, 0) for t in range(n_tuples)] + [(t, 1) for t in range(n_tuples)]
    meta = {"center_x": np.zeros(B), "center_y": np.zeros(B), "width": np.zeros(B),
            "height": np.zeros(B), "scale": np.ones(B), "rot": np.zeros(B),
            "R": np.zeros((B, 3, 3)), "T": np.zeros((B, 3, 1)), "f": np.zeros((B, 2)),
            "c": np.zeros((B, 2)), "projection_matrix": np.zeros((B, 3, 4))}
    logits = (0.5 * rng.standard_normal((B, J * D, D, D))).astype(np.float32)
    X = rng.normal(0.0, 300.0, size=(n_tuples, J, 3))
    for b, (t, v) in enumerate(views):
        meta["R"][b], meta["T"][b, :, 0], meta["f"][b], meta["c"][b] = R[t, v], T[t, v], f[t, v], c[t, v]
        meta["projection_matrix"][b] = P[t, v]
        uv = restate.project(P[t, v], X[t])
        meta["center_x"][b], meta["center_y"][b] = uv[:, 0].mean(), uv[:, 1].mean()
        meta["width"][b] = meta["height"][b] = 700.0 + 20.0 * b
        for j in range(J):   # plant a peak near the projected joint inside the patch
            px = (uv[j, 0] - meta["center_x"][b]) / meta["width"][b] * D + D / 2
            py = (uv[j, 1] - meta["center_y"][b]) / meta["height"][b] * D + D / 2
            xi, yi = int(np.clip(px, 0, D - 1)), int(np.clip(py, 0, D - 1))
            logits[b, j * D + D // 2, yi, xi] += 6.0
    return logits, meta


NET_CASES = {
    "r18": dict(layers=18, J=3, D=8, HW=64, N=2, volume=True, seed=61,
                grad_keys=["conv1.weight", "layer2.0.downsample.0.weight", "layer4.1.bn2.weight",
                           "deconv_layers.7.weight", "final_layer.weight", "final_layer.bias"]),
    "r50": dict(layers=50, J=2, D=8, HW=128, N=3, volume=True, seed=62,
                grad_keys=["final_layer.weight", "final_layer.bias", "deconv_layers.7.weight"]),
    "r50flat": dict(layers=50, J=3, D=4, HW=64, N=2, volume=False, seed=63,
                    grad_keys=["depth_fc.weight", "final_layer.bias"]),
}


def images(N, HW, seed):
    return np.random.default_rng(seed).standard_normal((N, 3, HW, HW)).astype(np.float32)


def grad_like(shape, seed):
    return np.random.default_rng(seed).standard_normal(tuple(shape)).astype(np.float32)


def heatmap_case(N, J, H, W, seed, sigma=2.0):
    """VOLUME=False objective inputs (SURVEY 8(d) C2(ii)): predicted heat-maps ~ N(0, 0.5),
    Gaussian targets exp(-((x-mx)^2+(y-my)^2)/(2 sigma^2)) (sigma = 2, config.py:34) with
    centres U{8..W-9} (margin W/4 on small maps), per-joint visibility weights in {0, 1}, joint vector + labels + weights."""
    rng = np.random.default_rng(seed)
    hm = (0.5 * rng.standard_normal((N, J, H, W))).astype(np.float32)
    bx, by = min(8, W // 4), min(8, H // 4)          # keep the blob inside the map
    mx = rng.integers(bx, max(bx + 1, W - bx), size=(N, J, 1, 1))
    my = rng.integers(by, max(by + 1, H - by), size=(N, J, 1, 1))
    yy, xx = np.mgrid[0:H, 0:W]
    tgt = np.exp(-((xx - mx) ** 2 + (yy - my) ** 2) / (2.0 * sigma * sigma)).astype(np.float32)
    wh = (rng.random((N, J, 1)) > 0.2).astype(np.float32)
    x = (rng.random((N, J * 3)) - 0.5).astype(np.float32)
    t = (rng.random((N, J * 3)) - 0.5).astype(np.float32)
    w = (rng.random((N, J * 3)) > 0.1).astype(np.float32)
    return hm, tgt, wh, x, t, w


def eval_case(S=24, J=17, seed=81):
    """H36M-protocol evaluation inputs: gt joints in camera space ~ N(0, 300 mm) around a
    pelvis at depth 4.5 m +- 0.5, projected with f ~ (1145, 1144), c ~ (512, 515) to
    `joints_3d` (x px, y px, root-relative depth mm); predictions = gt + N(0, 8 px / 40 mm)
    and a random global scale error."""
    rng = np.random.default_rng(seed)
    fl = np.stack([1145.0 + rng.uniform(-5, 5, S), 1144.0 + rng.uniform(-5, 5, S)], axis=1)
    c_p = np.stack([512.0 + rng.uniform(-5, 5, S), 515.0 + rng.uniform(-5, 5, S)], axis=1)
    pelvis = np.stack([rng.normal(0, 200, S), rng.normal(0, 200, S), 4500 + rng.uniform(-500, 500, S)], axis=1)
    X = pelvis[:, None, :] + rng.normal(0, 300, (S, J, 3))
    X[:, 0, :] = pelvis
    gt = np.zeros((S, J, 3))
    gt[:, :, 0] = X[:, :, 0] / X[:, :, 2] * fl[:, None, 0] + c_p[:, None, 0]
    gt[:, :, 1] = X[:, :, 1] / X[:, :, 2] * fl[:, None, 1] + c_p[:, None, 1]
    gt[:, :, 2] = X[:, :, 2] - pelvis[:, None, 2]
    pred = gt.copy()
    pred[:, :, :2] += rng.normal(0, 8, (S, J, 2))
    pred[:, :, 2] = pred[:, :, 2] * rng.uniform(0.8, 1.2, (S, 1)) + rng.normal(0, 40, (S, J))
    pred = np.concatenate([pred, np.ones((S, J, 1))], axis=2)      # score column as in the loop
    return pred, gt, pelvis, fl, c_p


PATCH_CASES = {
    # tag: (img H, img W, patch_w, patch_h, seed, smooth image?)
    "noise64": (1000, 1002, 64, 64, 91, False),
    "smooth96x128": (1002, 1000, 96, 128, 92, True),
    "edge48": (480, 640, 48, 48, 93, False),      # box partly outside the image: border zeros
}


def frame_case(tag):
    """Decoded BGR frame (uint8) + box + joints for the input-pipeline tests; the augmentation
    parameters are NOT here: the reference draws them (np.random / random seeded with `seed`)."""
    H, W, pw, ph, seed, smooth = PATCH_CASES[tag]
    rng = np.random.default_rng(seed)
    if smooth:
        yy, xx = np.mgrid[0:H, 0:W]
        img = np.stack([127 + 120 * np.sin(xx / 37.0 + c) * np.cos(yy / 23.0 - c) for c in range(3)], axis=2)
        img = np.clip(img + rng.normal(0, 3, img.shape), 0, 255).astype(np.uint8)
    else:
        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    if tag == "edge48":
        box = (600.5, 30.25, 300.0, 280.0)
    else:
        box = (W / 2 + rng.uniform(-50, 50), H / 2 + rng.uniform(-50, 50), 800 + rng.uniform(-100, 100),
               800 + rng.uniform(-100, 100))
    J = 17
    joints = np.stack([box[0] + rng.uniform(-300, 300, J), box[1] + rng.uniform(-300, 300, J),
                       rng.uniform(-800, 800, J)], axis=1)
    joints_vis = (rng.random((J, 3)) > 0.1).astype(np.float64)
    return img, box, joints, joints_vis, pw, ph, seed


# ---- BASELINE.json configuration sizes (tests/golden/make_golden_sizes.py)
SIZE_CASES = {
    "c1": dict(layers=50, J=16, D=64, HW=256, N=1, train=False, seed=71),
    "c2": dict(layers=50, J=17, D=64, HW=256, N=8, train=True, seed=72),
    "c5": dict(layers=101, J=17, D=96, HW=384, N=16, train=True, seed=75),
}


def grad_like_big(shape, seed):
    """Output gradient for the large cases: N(0,1) float32, generated per image so that the
    generator state never holds more than one image's worth."""
    rng = np.random.default_rng(seed)
    out = np.empty(tuple(shape), dtype=np.float32)
    for n in range(shape[0]):
        out[n] = rng.standard_normal(tuple(shape[1:]), dtype=np.float32)
    return out


def sample_output(out):
    """Strided sample (<= ~600k values) + per-(image, channel) sums of an [N,C,H,W] heat-map tensor."""
    o = np.asarray(out)
    st = 8
    while o[:, :, 1::st, 2::st].size > 600000:
        st *= 2
    return {"out_sample": o[:, :, 1::st, 2::st].astype(np.float32),
            "out_chan_sum": o.sum((2, 3), dtype=np.float64),
            "out_chan_abs": np.abs(o).sum((2, 3), dtype=np.float64),
            "out_max": np.float64(np.abs(o).max())}


def sample_grad(g):
    """<= 4096 strided elements of a gradient tensor and [sum, sum |g|, max |g|] (float64)."""
    f = np.asarray(g).reshape(-1)
    stride = max(1, f.size // 4096)
    return f[::stride].astype(np.float32), np.array([f.sum(dtype=np.float64), np.abs(f).sum(dtype=np.float64),
                                         np.abs(f).max()], dtype=np.float64)



def final_preds_case(seed=23):
    """Heat-maps for get_final_preds (lib/core/inference.py:43-68): the argmax cases plus smooth
    blobs with interior / border / corner peaks and exact-tie neighbours (sign(0) = 0);
    per-image centres and (box / 200) scales as the MPII loaders pass them."""
    rng = np.random.default_rng(seed)
    hm = argmax_heatmaps()                                   # [3, 6, 16, 12]
    n, j, h, w = hm.shape
    yy, xx = np.mgrid[0:h, 0:w]
    for (a, b, cy, cx) in ((1, 2, 7.3, 5.6), (1, 3, 1.2, 1.4), (1, 4, 14.0, 10.2), (2, 0, 8.0, 6.0),
                           (2, 1, 0.0, 0.0), (2, 2, 15.0, 11.0)):
        hm[a, b] = np.exp(-((xx - cx) ** 2 + (yy - cy) ** 2) / 6.0).astype(np.float32)
    hm[2, 4] = 0.0
    hm[2, 4, 6, 5] = 1.0
    hm[2, 4, 6, 6] = 0.5
    hm[2, 4, 6, 4] = 0.5                                       # x neighbours tie -> no x shift
    hm[2, 4, 7, 5] = 0.25
    center = np.stack([500 + rng.uniform(-60, 60, n), 480 + rng.uniform(-60, 60, n)], axis=1)
    scale = np.stack([2.0 + rng.uniform(0, 2, n)] * 2, axis=1) * np.array([1.0, 1.25])
    return hm, center, scale


def occluder_set(seed=97, n=5):
    """Synthetic stand-ins for the Pascal-VOC occluders of lib/utils/augmentation.py:8-58 (no
    dataset offline): RGBA uint8 blobs of various sizes whose alpha plane has the three levels
    the loader produces (0 outside, 192 on the eroded border, 255 inside)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        h, w = int(rng.integers(40, 140)), int(rng.integers(40, 140))
        yy, xx = np.mgrid[0:h, 0:w]
        r = np.sqrt(((xx - w / 2) / (w / 2)) ** 2 + ((yy - h / 2) / (h / 2)) ** 2)
        alpha = np.where(r < 0.8, 255, np.where(r < 0.95, 192, 0)).astype(np.uint8)
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        out.append(np.concatenate([rgb, alpha[..., None]], axis=-1))
    return out


# ---- device models and checks of the configuration sizes (tests/test_gpu_sizes.py and the tests
# and tools that reuse its C1 network)
def _model(dev, c, precision, train):
    """The network of size case c with the unmodified reference's seeded initial weights."""
    import lib.models as models
    from oracle import restate_net
    from tools.bench_cfg import make_cfg
    cfg = make_cfg(num_layers=c["layers"], num_joints=c["J"], volume=True, depth_res=c["D"],
                   image_size=(c["HW"], c["HW"]))
    model = models.pose3d_resnet.get_pose_net(cfg, False, precision=precision)
    shapes = restate_net.param_shapes(num_layers=c["layers"], num_joints=c["J"], volume=True,
                                      depth_res=c["D"])
    model.load_state_dict(restate_net.init_state(shapes, c["seed"]))
    model = model.to(dev)
    return model.train() if train else model.eval()


def _check_output(out, g, tol=1e-3):
    """Heat-maps against the unmodified reference (north_star: <= 1e-3 rel)."""
    o = out.detach().cpu().numpy()
    s = sample_output(o)
    mx = float(g["ref/out_max"])
    e = float(np.max(np.abs(s["out_sample"] - g["ref/out_sample"])) / mx)
    e64 = float(np.max(np.abs(s["out_sample"] - g["f64/out_sample"])) / mx)
    r64 = float(np.max(np.abs(g["ref/out_sample"] - g["f64/out_sample"])) / mx)
    # per-(image, channel) sums over the map: error relative to the summed magnitudes
    es = float(np.max(np.abs(s["out_chan_sum"] - g["ref/out_chan_sum"]) / (g["ref/out_chan_abs"] + 1e-30)))
    print("heat-maps: vs reference %.2e (channel sums %.2e); vs float64 %.2e (the reference's own "
          "float32 run: %.2e)" % (e, es, e64, r64))
    assert e <= tol and es <= tol
    assert abs(float(s["out_max"]) - mx) <= tol * mx


def _ring_meta(tuples, seed):
    """Cameras / boxes of the bench workload (SURVEY 8(d) C3): batch laid out
    [view0 | view3 | view1 | view2] of every tuple so the half-split pairs (0,1) and (3,2)."""
    from lib.dataset.synthetic import ring_camera
    rng = np.random.default_rng(seed)
    n_img = tuples * 4
    order = [(t, 0) for t in range(tuples)] + [(t, 3) for t in range(tuples)] + \
            [(t, 1) for t in range(tuples)] + [(t, 2) for t in range(tuples)]
    cams = {(t, v): ring_camera(rng, v) for t in range(tuples) for v in range(4)}
    return {"center_x": 500 + rng.uniform(-50, 50, n_img), "center_y": 500 + rng.uniform(-50, 50, n_img),
            "width": 800 + rng.uniform(-100, 100, n_img), "height": 800 + rng.uniform(-100, 100, n_img),
            "scale": np.ones(n_img), "rot": np.zeros(n_img),
            "R": np.stack([cams[o][0] for o in order]), "T": np.stack([cams[o][1] for o in order]),
            "f": np.stack([cams[o][2] for o in order]), "c": np.stack([cams[o][3] for o in order]),
            "projection_matrix": np.stack([cams[o][4] for o in order])}
