"""GPU (-m gpu): multi-view inference.  epb_triangulate_robust against the numpy restatement
(tests/multiview_cases.py) at V in {2,3,4,6,8}, J in {16,17}, NT in {1,64,4096}, its determinism
and argument checks; the soft-argmax confidence against a float64 softmax peak, with and without
flip test; MultiViewPredictor against "PosePredictor per view, then the restatement on its 2-D
output"; graph replays; validate_multiview on the fixture tree with the network bypassed.

Bars: the kernel's one-sided Jacobi against numpy's SVD agree to 1e-4 mm at 3 px noise (as
test_gpu_parity.test_nview_dlt_vs_oracle).  MultiViewPredictor and PosePredictor run the same
kernels at the same batch size; their 2-D joints are held to the bound test_gpu_predictor derives
from the measured logit difference."""
import ctypes

import numpy as np
import pytest
import torch

from tests import multiview_cases as mc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _gpu(u, P, w, thr, dev):
    import lib.utils.triangulation as tri
    out = tri.triangulate_views_robust(_t(u, dev), _t(P, dev), None if w is None else _t(w, dev), thr)
    return [o.cpu().numpy() for o in out]


def _case(V, J, NT):
    P, X, ue, un = mc.rig(1000 * V + 10 * J + NT % 7, NT, V, J)
    uo, _ = mc.plant_outliers(un, V + J)
    rng = np.random.default_rng(NT + V)
    w = rng.uniform(0.05, 1.0, un.shape[:3]) * (rng.uniform(size=un.shape[:3]) > 0.1)
    return P, uo, w


@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("V", [2, 3, 4, 6, 8])
def test_kernel_vs_restatement(dev, V, J):
    for NT, step in ((1, 1), (64, 8), (4096, 512)):
        P, u, w = _case(V, J, NT)
        X, st, inl, res = _gpu(u, P, w, 12.0, dev)
        assert np.isfinite(X).all() and np.isfinite(res).all()
        assert np.all((st == 0) | (st == 1)) and np.all(inl[st == 0] == 0) and np.all(X[st == 0] == 0)
        for t in range(0, NT, step):
            xo, so, io, ro = mc.robust_nview_triangulation(u[t], P[t], w[t], 12.0)
            assert np.array_equal(st[t], so) and np.array_equal(inl[t], io), (NT, t)
            assert np.max(np.abs(X[t] - xo)) <= 1e-4 and np.max(np.abs(res[t] - ro)) <= 1e-6, (NT, t)
        # a second launch, and the tuples launched on their own, give the same bits
        again = _gpu(u, P, w, 12.0, dev)
        part = _gpu(u[NT // 2:], P[NT // 2:], w[NT // 2:], 12.0, dev)
        for a, b, c in zip((X, st, inl, res), again, part):
            assert np.array_equal(a, b) and np.array_equal(a[NT // 2:], c)
    # no weights = weights of one
    P, u, w = _case(V, J, 5)
    for a, b in zip(_gpu(u, P, None, 15.0, dev), _gpu(u, P, np.ones_like(w), 15.0, dev)):
        assert np.array_equal(a, b)


def test_degenerate_inputs_on_the_device(dev):
    V, J = 4, 17
    P, X, ue, _ = mc.rig(5, 3, V, J)
    w = np.zeros((3, V, J))
    w[1, 2] = 1.0
    w[2] = 1.0
    u = ue.copy()
    u[2, :3, 5] = np.nan
    u[2, 1, 3, 0] = np.inf
    Xg, st, inl, res = _gpu(u, P, w, 15.0, dev)
    assert not st[:2].any() and not Xg[:2].any() and not inl[:2].any() and not res[:2].any()
    assert st[2, 5] == 0 and st[2, 3] == 1 and inl[2, 3] == 0b1101
    assert np.isfinite(Xg).all() and np.isfinite(res).all()
    ok = st[2] == 1
    assert np.max(np.abs(Xg[2][ok] - X[2][ok])) <= 1e-6
    for a in _gpu(ue, -P, None, 15.0, dev):                   # behind every camera
        assert not a.any()
    import lib.utils.triangulation as tri
    e = tri.triangulate_views_robust(_t(ue[:0], dev), _t(P[:0], dev))
    assert e[0].shape == (0, J, 3) and e[1].shape == (0, J)


def test_argument_checks(dev):
    from epipolarpose_b200 import _lib
    L = _lib.lib()
    V, J, NT = 4, 17, 2
    u = torch.zeros((NT, V, J, 2), device=dev, dtype=torch.float64)
    P = torch.zeros((NT, V, 12), device=dev, dtype=torch.float64)
    X = torch.zeros((NT, J, 3), device=dev, dtype=torch.float64)
    res = torch.zeros((NT, J), device=dev, dtype=torch.float64)
    inl = torch.zeros((NT, J), device=dev, dtype=torch.int32)
    st = torch.zeros((NT, J), device=dev, dtype=torch.int32)
    p = lambda t: ctypes.c_void_p(t.data_ptr())

    def call(V=V, stride=2, NT=NT, J=J, thr=15.0, u_=u):
        return L.epb_triangulate_robust(p(u_) if u_ is not None else None, stride, p(P), None, NT, V, J, thr,
                                        p(X), p(inl), p(res), p(st), None)
    assert call() == 0
    assert call(NT=0) == 0 and call(J=0) == 0
    for kw in (dict(V=1), dict(V=9), dict(stride=1), dict(NT=-1), dict(J=-1), dict(thr=0.0), dict(thr=-1.0),
               dict(thr=float("nan")), dict(thr=float("inf")), dict(u_=None), dict(NT=1 << 20, J=1 << 12)):
        assert call(**kw) != 0, kw
        assert b"invalid argument" in L.epb_last_error()
    torch.cuda.synchronize()
    import lib.utils.triangulation as tri
    with pytest.raises(ValueError, match="2..8"):
        tri.triangulate_views_robust(torch.zeros((1, 9, J, 2), device=dev, dtype=torch.float64),
                                     torch.zeros((1, 9, 3, 4), device=dev, dtype=torch.float64))


# ------------------------------------------------------------------ confidence
def _logits(dev, N, J, D, seed):
    g = torch.Generator().manual_seed(seed)
    x = (2.0 * torch.randn(N, J * D, D, D, generator=g)).to(dev)
    return x.contiguous(memory_format=torch.channels_last)


def test_confidence_is_the_softmax_peak(dev):
    import lib.core.integral_loss as il
    N, J, D = 3, 17, 16
    x = _logits(dev, N, J, D, 1)
    coords, peak = il.get_joint_location_coords_peak(x)
    want = torch.softmax(x.double().reshape(N, J, -1), dim=2).amax(dim=2)
    assert float(((peak.double() - want).abs() / want).max()) <= 1e-5
    assert torch.equal(coords, il.get_joint_location_coords(x))
    # NCHW storage takes the other kernel and the same reading of its workspace
    _, peak2 = il.get_joint_location_coords_peak(x.contiguous())
    assert float(((peak2.double() - want).abs() / want).max()) <= 1e-5


@pytest.mark.parametrize("shift", [False, True])
def test_confidence_with_flip_test(dev, shift):
    import lib.core.integral_loss as il
    from lib.dataset.synthetic import MPII_FLIP_PAIRS
    N, J, D = 2, 16, 16
    x = _logits(dev, 2 * N, J, D, 2 + shift)
    coords, peak = il.get_joint_location_coords_flip_peak(x, MPII_FLIP_PAIRS, shift)
    assert torch.equal(coords, il.get_joint_location_coords_flip(x, MPII_FLIP_PAIRS, shift))   # same bits
    perm = il.flip_permutation(MPII_FLIP_PAIRS, J)
    v = x.double().reshape(2 * N, J, D, D, D)
    fb = v[N:].flip(-1)[:, perm]
    if shift:
        fb = torch.cat([fb[..., :1], fb[..., :-1]], dim=-1)
    want = torch.softmax((0.5 * (v[:N] + fb)).reshape(N, J, -1), dim=2).amax(dim=2)
    assert float(((peak.double() - want).abs() / want).max()) <= 1e-5
    # contiguous NCHW logits take the torch-op merge; the same confidence
    _, peak2 = il.get_joint_location_coords_flip_peak(x.contiguous(), MPII_FLIP_PAIRS, shift)
    assert float(((peak2.double() - want).abs() / want).max()) <= 1e-5


# ------------------------------------------------------------------ MultiViewPredictor
PATCH = 256.0


@pytest.fixture(scope="module")
def c1(dev):
    from tests import golden_inputs as gi
    from tests.golden_inputs import _model
    return _model(dev, gi.SIZE_CASES["c1"], "f16x3", train=False)


_rig_inputs = mc.rig_inputs


def _check_against_composition(mv, pp, x, boxes, P, thr, use_conf):
    T, V = x.shape[:2]
    out = mv(x, boxes, P)
    J = out["world"].shape[1]
    assert out["world"].shape == (T, J, 3) and out["kps"].shape == (T, V, J, 4)
    assert out["inliers"].shape == out["resid"].shape == out["status"].shape == (T, J)
    mv_logits = mv.logits.clone()
    single = pp(x.reshape((T * V,) + x.shape[2:]), boxes=boxes).reshape(T, V, J, 4)
    # 2-D: the bound of test_gpu_predictor for the measured logit difference, scaled to image px
    dl = (pp.logits - mv_logits).abs().reshape(pp.logits.shape[0], J, -1).amax(-1).cpu().numpy()
    if len(dl) == T * V:
        dl = dl.reshape(T, V, J)
    else:                       # flip test: a merged volume moves by at most the larger of its two halves
        dl = np.full((T, V, J), dl.max())
    scale = (np.maximum(boxes["width"], boxes["height"]) / PATCH).reshape(T, V, 1)
    bound = (PATCH * np.expm1(2.0 * dl) + 1e-3) * np.maximum(scale, 2000.0 / PATCH)
    d = np.abs(out["kps"][..., :3] - single[..., :3]).max(-1)
    assert np.all(d <= bound), (d.max(), bound.min())
    conf = out["kps"][..., 3]
    assert np.all(conf > 0) and np.all(conf <= 1.0 + 1e-6)
    # 3-D: the restatement on the predictor's own 2-D output
    n_ok = 0
    for t in range(T):
        xo, so, io, ro = mc.robust_nview_triangulation(out["kps"][t], P[t], conf[t] if use_conf else None, thr)
        assert np.array_equal(out["status"][t], so) and np.array_equal(out["inliers"][t], io)
        assert np.max(np.abs(out["world"][t] - xo)) <= 1e-4 and np.max(np.abs(out["resid"][t] - ro)) <= 1e-6
        n_ok += int(so.sum())
    return out, n_ok


def test_multiview_predictor_vs_composition(c1):
    from lib.core.inference import MultiViewPredictor, PosePredictor
    x, boxes, P = _rig_inputs(2, 4, 21)
    pp = PosePredictor(c1, flip_test=False)
    # a threshold no reprojection error exceeds: the confidence-weighted DLT of the views the point is in front of
    mv = MultiViewPredictor(c1, flip_test=False, threshold_px=1e4)
    out, n_ok = _check_against_composition(mv, pp, x, boxes, P, 1e4, True)
    assert n_ok >= out["status"].size // 2
    # the default threshold, unweighted: views of an untrained network rarely agree
    mv15 = MultiViewPredictor(c1, flip_test=False, use_confidence=False)
    out15, _ = _check_against_composition(mv15, pp, x, boxes, P, 15.0, False)
    # replays of one graph give the same bits
    again = mv(x, boxes, P)
    assert len(mv.graphs) == 1
    for k in out:
        assert np.array_equal(out[k], again[k]), k
    # other boxes and cameras through the same graph: the static buffers are read again
    x2, boxes2, P2 = _rig_inputs(2, 4, 22)
    out2, _ = _check_against_composition(mv, pp, x, boxes2, P2, 1e4, True)
    assert len(mv.graphs) == 1
    assert not np.array_equal(out2["kps"][..., :2], out["kps"][..., :2])
    assert not np.array_equal(out2["world"], out["world"])
    assert np.array_equal(out2["kps"][..., 3], out["kps"][..., 3])         # the same images
    # another (T, V): a second graph
    x3, boxes3, P3 = _rig_inputs(1, 3, 23)
    _check_against_composition(mv, pp, x3, boxes3, P3, 1e4, True)
    assert len(mv.graphs) == 2
    with pytest.raises(ValueError, match="boxes"):
        mv(x)
    with pytest.raises(ValueError, match="boxes"):
        mv(x, boxes)
    with pytest.raises(ValueError, match="T, V, 3, H, W"):
        mv(x[0], boxes, P)
    with pytest.raises(ValueError, match="threshold_px"):
        MultiViewPredictor(c1, threshold_px=0.0)


def test_multiview_predictor_flip_test(c1):
    from lib.core.inference import MultiViewPredictor, PosePredictor
    from lib.dataset.synthetic import MPII_FLIP_PAIRS
    x, boxes, P = _rig_inputs(1, 4, 31)
    pp = PosePredictor(c1, flip_test=True, shift_heatmap=True, flip_pairs=MPII_FLIP_PAIRS)
    mv = MultiViewPredictor(c1, flip_test=True, shift_heatmap=True, flip_pairs=MPII_FLIP_PAIRS, threshold_px=1e4)
    _check_against_composition(mv, pp, x, boxes, P, 1e4, True)
    assert mv.logits.shape[0] == 8
    with pytest.raises(ValueError, match="flip_pairs"):
        MultiViewPredictor(c1, flip_test=True)


def test_validate_multiview_with_exact_projections(dev):
    """The fixture tree's validation db, the network bypassed: the 'predictor' answers with the
    records' own 2-D joints (exact projections) through the triangulation kernel."""
    from tests import dataset_cases as dc
    from lib.core.function import validate_multiview
    import lib.utils.triangulation as tri
    ds = dc.build("h36m_valid")
    recs = [ds.tuple_records(r) for r in ds.view_tuples()]
    seen = []

    def predictor(images, boxes, P):
        T, V = images.shape[:2]
        assert images.shape[2:] == (3, 64, 64) and images.dtype == np.float32 and P.shape == (T, V, 3, 4)
        assert boxes["center_x"].shape == (T * V,) and np.all(boxes["scale"] == 1) and np.all(boxes["rot"] == 0)
        chunk = recs[len(seen):len(seen) + T]
        seen.extend(chunk)
        u = np.stack([np.stack([r["joints_3d"][:, :2] for r in tup]) for tup in chunk])
        X, st, inl, res = tri.triangulate_views_robust(_t(u, dev), _t(P, dev))
        return {"world": X.cpu().numpy(), "status": st.cpu().numpy(), "inliers": inl.cpu().numpy(),
                "resid": res.cpu().numpy()}

    r = validate_multiview(ds, predictor, tuples_per_batch=2)
    assert len(seen) == len(recs) == r["tuples"]
    assert r["mpjpe"] < 1e-3 and r["failed"] == 0.0 and r["inlier_views"] == 4.0
    acts = {tup[0]["action"] for tup in recs}
    assert set(r["per_action"]) == acts and all(v["mpjpe"] < 1e-3 for v in r["per_action"].values())
    assert ds.is_train is False
