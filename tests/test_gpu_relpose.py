"""GPU: relative_pose_kernel (self-supervision without camera extrinsics) against the numpy
oracle, the label chain through self_supervision_device against the known-camera path, outlier
rejection, independence from R / T / projection_matrix, and the captured training step."""
import numpy as np
import pytest
import torch

from oracle import restate, restate_net, restate_relpose as rr
from tests import relpose_cases as rc
from tests.conftest import relerr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda")


def _pack(d, dev):
    """rig_pairs -> kps [B,J,2], intr [B,4], box [B,6] with sample i paired with i + NP."""
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    kps = t(np.concatenate([d["ua"], d["ub"]]))
    intr = t(np.concatenate([d["intr_a"], d["intr_b"]]))
    box = t(np.concatenate([d["box_a"], d["box_b"]]))
    return kps, intr, box


def test_relative_pose_kernel_matches_oracle(dev):
    """4096 pairs (0-3 px noise, 0-3 outliers): discrete choices identical to the oracle (a
    different hypothesis is accepted only as a tie: both scores equal to 1e-12 relative); P and
    cam to 1e-9 relative; no NaN anywhere."""
    from lib.utils import triangulation as tri
    NP = 4096
    d = rc.rig_pairs(NP, 101)
    kps, intr, box = _pack(d, dev)
    Pa, Pb, cam, inl, st, dg = [x.cpu().numpy() for x in tri.relative_pose_pairs(kps, intr, box, diag=True)]
    for a in (Pa, Pb, cam):
        assert np.isfinite(a).all()
    ties, n_ok = [], 0
    for i in range(NP):
        o = rr.relative_pose(d["ua"][i], d["ub"][i], d["intr_a"][i], d["intr_b"][i], d["box_a"][i], d["box_b"][i])
        if dg[i, 0] != o["best_h"]:
            s = o["scores"]
            assert dg[i, 0] >= 0 and o["best_h"] >= 0, i
            assert abs(s[dg[i, 0]] - s[o["best_h"]]) <= 1e-12 * abs(s[o["best_h"]]), (i, dg[i], o["best_h"])
            ties.append(i)
            continue
        assert (dg[i, 1], dg[i, 2], st[i]) == (o["cand"], o["n_inl"], o["status"]), (i, dg[i], st[i])
        assert np.array_equal(inl[i] != 0, o["inliers"]), i
        assert relerr(Pa[i], o["P_a"]) <= 1e-9 and relerr(Pb[i], o["P_b"]) <= 1e-9, i
        assert relerr(cam[i], o["cam_a"]) <= 1e-9 and relerr(cam[NP + i], o["cam_b"]) <= 1e-9, i
        n_ok += o["status"]
    if ties:
        print("relative_pose: %d tied hypothesis choices: %s" % (len(ties), ties[:20]))
    assert len(ties) <= NP // 100
    assert n_ok >= 0.85 * NP


def _plant(uv, box, J, D, patch=256.0):
    """Logits [B, J*D, D, D] whose soft-argmax lands on the image points uv [B,J,2] (box rot 0):
    a bilinear split of the mass over the 4 voxels around the target, all other logits 0."""
    B = uv.shape[0]
    logits = np.zeros((B, J * D, D, D), np.float32)
    for b in range(B):
        cx, cy, w, h, s, _ = box[b]
        for j in range(J):
            ix = ((uv[b, j, 0] - cx) / (w * s) + 0.5) * D          # soft-argmax index units
            iy = ((uv[b, j, 1] - cy) / (h * s) + 0.5) * D
            x0, y0 = int(np.floor(ix)), int(np.floor(iy))
            assert 0 <= x0 < D - 1 and 0 <= y0 < D - 1
            fx, fy = ix - x0, iy - y0
            for dy, wy in ((0, 1 - fy), (1, fy)):
                for dx, wx in ((0, 1 - fx), (1, fx)):
                    logits[b, j * D + D // 2, y0 + dy, x0 + dx] = np.log(max(wx * wy, 1e-30)) + 120.0
    return logits


def _known_case(n, seed, consistent, J=17, D=32):
    d = rc.rig_pairs(n, seed, J=J, noise_px=(0.0, 0.0), n_out=(0, 0), box_consistent=consistent,
                     spread=150.0)
    if not consistent:
        d["box_a"][:, 5] = 0.0
        d["box_b"][:, 5] = 0.0
    box = np.concatenate([d["box_a"], d["box_b"]])
    box[:, 3] = box[:, 2]
    uv = np.concatenate([d["ua"], d["ub"]])
    meta = {"center_x": box[:, 0], "center_y": box[:, 1], "width": box[:, 2], "height": box[:, 3],
            "scale": box[:, 4], "rot": box[:, 5],
            "R": np.concatenate([d["R"][:, 0], d["R"][:, 1]]),
            "T": np.concatenate([d["T"][:, 0], d["T"][:, 1]])[:, :, None],
            "f": np.concatenate([d["f"][:, 0], d["f"][:, 1]]),
            "c": np.concatenate([d["c"][:, 0], d["c"][:, 1]]),
            "projection_matrix": np.concatenate([d["P"][:, 0], d["P"][:, 1]])}
    # k_v = f_x rect3d_w / (bb_w scale Z_root_true)
    k = meta["f"][:, 0] * 2000.0 / (box[:, 2] * box[:, 4] * np.concatenate([d["zroot"][:, 0], d["zroot"][:, 1]]))
    return d, _plant(uv, box, J, D), meta, k


@pytest.mark.parametrize("consistent", [True, False])
def test_known_answer_through_self_supervision(dev, consistent):
    """Exact projections from a ring rig, planted as soft-argmax peaks: the labels from estimated
    extrinsics equal the known-camera labels (x, y always; z times sqrt(k_a k_b), which is 1
    when the boxes satisfy bb_w scale Z_root / f_x = rect3d_w), to the float32 rounding of the
    8-point inputs."""
    import lib.utils.img_utils as iu
    n = 8
    d, logits, meta, k = _known_case(n, 131, consistent)
    x = torch.from_numpy(logits).to(dev)
    mt = {kk: torch.from_numpy(np.asarray(v)) for kk, v in meta.items()}
    lab_k, w_k = iu.self_supervision_device(x, mt)
    lab_e, w_e = iu.self_supervision_device(x, mt, estimate_extrinsics=True)
    lab_k, lab_e, w_e = [a.cpu().numpy().reshape(2 * n, -1, 3) for a in (lab_k, lab_e, w_e)]
    assert np.all(w_e == 1.0)                          # every pair estimated
    err_xy = np.max(np.abs(lab_e[..., :2] - lab_k[..., :2]))
    kk = np.sqrt(k[:n] * k[n:])
    zk = lab_k[..., 2] * np.concatenate([kk, kk])[:, None]
    err_z = np.max(np.abs(lab_e[..., 2] - zk))
    print("known answer (consistent=%s): max |dxy| %.2e, max |dz| %.2e" % (consistent, err_xy, err_z))
    # fundamental_8point rounds its points to float32 as cv2.findFundamentalMat does: R is then good
    # to a few 1e-6 rad, i.e. ~3e-3 px of reprojection (1.4e-5 in label units measured on an H100)
    assert err_xy <= 5e-5 and err_z <= 5e-5
    if consistent:
        assert np.max(np.abs(k - 1.0)) <= 1e-12


def test_outliers_are_rejected(dev):
    """Up to 3 of 17 joints replaced by random points: those joints are not inliers, and R, t
    match the outlier-free estimate (exact projections: to the float32 rounding of the 8-point
    inputs)."""
    from lib.utils import triangulation as tri
    clean = rc.rig_pairs(64, 141, noise_px=(0.0, 0.0), n_out=(0, 0))
    dirty = rc.rig_pairs(64, 141, noise_px=(0.0, 0.0), n_out=(0, 0))
    rng = np.random.default_rng(142)
    bad = np.zeros((64, 17), bool)
    for i in range(64):
        m = int(rng.integers(1, 4))
        j = rng.choice(np.arange(1, 17), size=m, replace=False)
        bad[i, j] = True
        dirty["ua"][i, j] = rng.uniform(0, 1024, (m, 2))
        dirty["ub"][i, j] = rng.uniform(0, 1024, (m, 2))
    out = {}
    for name, d in (("clean", clean), ("dirty", dirty)):
        _, _, cam, inl, st = [x.cpu().numpy() for x in tri.relative_pose_pairs(*_pack(d, dev))]
        assert np.all(st == 1), name
        out[name] = (cam, inl != 0)
    assert not np.any(out["dirty"][1] & bad)
    R = lambda cam: cam[64:, :9].reshape(-1, 3, 3)
    tdir = lambda cam: -np.einsum("nij,nj->ni", R(cam), cam[64:, 9:12])
    tc, td = tdir(out["clean"][0]), tdir(out["dirty"][0])
    tc /= np.linalg.norm(tc, axis=1, keepdims=True)
    td /= np.linalg.norm(td, axis=1, keepdims=True)
    assert np.max(np.abs(R(out["dirty"][0]) - R(out["clean"][0]))) <= 1e-4
    assert np.max(np.abs(td - tc)) <= 1e-4
    assert np.max(np.abs(R(out["clean"][0]) - clean["R_ab"])) <= 1e-4


def test_extrinsics_are_unused(dev):
    """R, T and projection_matrix set to NaN, or removed: bit-identical loss and labels."""
    import lib.core.function as fn
    import lib.core.integral_loss as il
    import lib.utils.img_utils as iu
    d, logits, meta, _ = _known_case(4, 151, False)
    crit = il.SmoothL1JointLocationLoss(17)
    res = []
    for variant in ("full", "nan", "removed"):
        mt = {k: torch.from_numpy(np.array(v, dtype=np.float64)) for k, v in meta.items()}
        for k in ("R", "T", "projection_matrix"):
            if variant == "nan":
                mt[k][:] = float("nan")
            elif variant == "removed":
                del mt[k]
        x = torch.from_numpy(logits).to(dev).requires_grad_(True)
        loss = fn.online_epipolar_loss(crit, x, mt, "iterative", estimate_extrinsics=True)
        lab, w = iu.self_supervision_device(x.detach(), mt, estimate_extrinsics=True)
        res.append((loss.item(), lab.cpu().numpy(), w.cpu().numpy()))
    for r in res[1:]:
        assert r[0] == res[0][0]
        assert np.array_equal(r[1], res[0][1]) and np.array_equal(r[2], res[0][2])
    assert np.isfinite(res[0][0]) and np.all(res[0][2] == 1.0)


def test_graphed_train_step_estimated_extrinsics(dev):
    """test_graphed_train_step_matches_eager's bars with J = 16 in the estimated-extrinsics mode:
    graph vs eager, two graph runs bit-identical, everything finite (random-init nets give
    near-degenerate 2-D joints, so pairs may fail and carry weight 0)."""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    import lib.utils.utils as U
    from oracle import refshim
    from tests import golden_inputs as gi
    J, D, HW = 16, 16, 64
    _, meta_np = gi.selfsup_case(n_tuples=2, J=J, D=D)
    B = 4
    meta = {k: torch.from_numpy(v) for k, v in meta_np.items()}
    cfg = refshim.make_cfg(num_layers=18, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    sd = restate_net.init_state(restate_net.param_shapes(18, J, True, D), 3)
    xs = [torch.from_numpy(gi.images(B, HW, 40 + i)).to(dev) for i in range(5)]
    out = {}
    for mode in ("eager", "graph", "graph2"):
        model = models.pose3d_resnet.get_pose_net(cfg, False)
        model.load_state_dict(sd)
        model = model.to(dev).train()
        crit = il.SmoothL1JointLocationLoss(J)
        opt = U.FusedAdam(list(model.parameters()), lr=1e-4)
        stepper = fn.GraphedTrainStep(model, crit, opt, online=True, estimate_extrinsics=True)
        losses = []
        for i in range(5):
            if mode == "eager":
                geom = iu.pack_meta(meta, B, dev, estimate_extrinsics=True)
                losses.append(float(stepper.eager_step(xs[i], None, None, geom)))
            else:
                losses.append(float(stepper(xs[i], meta=meta)))
        if mode != "eager":
            assert stepper.graph is not None and stepper.key[-1] is True
        out[mode] = (losses, {k: v.detach().cpu().numpy() for k, v in model.named_parameters()})
    for losses, params in out.values():
        assert np.all(np.isfinite(losses))
        assert all(np.isfinite(v).all() for v in params.values())
    assert out["graph"][0] == out["graph2"][0]
    for k, v in out["graph"][1].items():
        assert np.array_equal(v, out["graph2"][1][k]), k
    for a, b in zip(out["graph"][0], out["eager"][0]):
        assert abs(a - b) <= 2e-2 * abs(b) + 1e-6, (out["graph"][0], out["eager"][0])
    assert abs(out["graph"][0][0] - out["eager"][0][0]) <= 1e-5 * abs(out["eager"][0][0]) + 1e-7
    for k, v in out["eager"][1].items():
        assert relerr(out["graph"][1][k], v) <= 5e-2, k


def test_captured_online_loss_matches_eager(dev):
    """online_epipolar_loss (and the labels) in the estimated-extrinsics mode captured in a CUDA
    graph on planted-peak logits, replayed with new logits and meta: loss, labels and the logit
    gradient bit-identical to eager, with estimated (non-zero status) pairs."""
    import lib.core.function as fn
    import lib.core.integral_loss as il
    import lib.utils.img_utils as iu
    crit = il.SmoothL1JointLocationLoss(17)
    cases = [_known_case(4, s, False) for s in (161, 162)]
    B = 8

    def geom(meta):
        mt = {k: torch.from_numpy(np.asarray(v, dtype=np.float64)) for k, v in meta.items()}
        return iu.pack_meta(mt, B, dev, estimate_extrinsics=True)

    def run(x, g):
        x.grad = None
        loss = fn.online_epipolar_loss(crit, x, {"_packed": g}, "iterative", estimate_extrinsics=True)
        lab, w = iu.self_supervision_device(x.detach(), {"_packed": g}, estimate_extrinsics=True)
        loss.backward()
        return loss, lab, w

    eager = []
    for _, logits, meta, _ in cases:
        x = torch.from_numpy(logits).to(dev).requires_grad_(True)
        loss, lab, w = run(x, geom(meta))
        eager.append((loss.item(), lab.cpu().numpy(), w.cpu().numpy(), x.grad.cpu().numpy()))
        assert np.all(eager[-1][2] == 1.0)
    sx = torch.from_numpy(cases[0][1]).to(dev).requires_grad_(True)
    sg = geom(cases[0][2])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(sx, sg)                                     # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    sx.grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        sloss, slab, sw = run(sx, sg)
    for (_, logits, meta, _), ref in zip(cases[::-1], eager[::-1]):
        with torch.no_grad():
            sx.copy_(torch.from_numpy(logits).to(dev))
        for k, v in geom(meta).items():
            sg[k].copy_(v)
        g.replay()
        torch.cuda.synchronize()
        assert sloss.item() == ref[0]
        assert np.array_equal(slab.cpu().numpy(), ref[1]) and np.array_equal(sw.cpu().numpy(), ref[2])
        assert np.array_equal(sx.grad.cpu().numpy(), ref[3])
