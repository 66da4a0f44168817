"""CPU: robust V-view triangulation for multi-view inference.  The numpy restatement
(tests/multiview_cases.py) against the reference's pair triangulation (tests/golden), the
per-(tuple, joint) body of triangulate_robust_kernel (csrc/geometry.cu) run on the CPU by
tests/harness/host_multiview.cu against the restatement, planted outliers, degenerate inputs,
absent views, and H36M_Integral.view_tuples() on the fixture trees."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import restate
from tests import golden_inputs as gi
from tests import multiview_cases as mc
from tests.conftest import ROOT

HUGE = 1e12


def test_restatement_reduces_to_the_reference_pair_case(golden):
    """V = 2, weights 1 and a threshold nothing exceeds: the reference's linear_eigen_triangulation."""
    g = golden("triangulation")
    u1, u2, P1, P2, _ = gi.triangulation_case()
    for i in range(len(u1)):
        x, st, inl, res = mc.robust_nview_triangulation(np.stack([u1[i], u2[i]]), np.stack([P1[i], P2[i]]),
                                                        threshold_px=HUGE)
        assert np.max(np.abs(x - g["linear_eigen_triangulation_x"][i])) <= 1e-9
        assert st.all() and np.all(inl == 3) and np.all(np.isfinite(res))


@pytest.fixture(scope="module")
def host_robust(tmp_path_factory):
    """tests/harness/host_multiview.cu: robust_point of csrc/geometry.cu built for the CPU."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / "host_multiview")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1", "-std=c++17",
                        "-o", exe, os.path.join(ROOT, "tests", "harness", "host_multiview.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(u, P, w=None, thr=15.0):
        """u [N,V,J,2], P [N,V,3,4], w [N,V,J] or None -> (X [N,J,3], status, inliers, resid)"""
        N, V, J = u.shape[:3]
        inp = b"".join(np.concatenate([u[t].ravel(), P[t].ravel()] + ([w[t].ravel()] if w is not None else []))
                       .astype(np.float64).tobytes() for t in range(N))
        out = subprocess.run([exe, "robust", str(N), str(V), str(J), repr(float(thr)), str(int(w is not None))],
                             input=inp, capture_output=True)
        assert out.returncode == 0, out.stderr
        a = np.frombuffer(out.stdout, dtype=np.float64).reshape(N, 6 * J)
        assert np.isfinite(a).all(), "a non-finite value left the kernel body"
        return (a[:, :3 * J].reshape(N, J, 3), a[:, 5 * J:].astype(np.int32), a[:, 3 * J:4 * J].astype(np.int32),
                a[:, 4 * J:5 * J])
    return run


def _restated(u, P, w=None, thr=15.0):
    r = [mc.robust_nview_triangulation(u[t], P[t], None if w is None else w[t], thr) for t in range(len(u))]
    return tuple(np.stack([x[k] for x in r]) for k in range(4))


def _same(got, want, tol=1e-4):
    X, st, inl, res = got
    Xo, so, io, ro = want
    assert np.array_equal(st, so) and np.array_equal(inl, io)
    assert np.max(np.abs(X - Xo)) <= tol, np.max(np.abs(X - Xo))
    assert np.max(np.abs(res - ro)) <= 1e-6


@pytest.mark.parametrize("J", [16, 17])
@pytest.mark.parametrize("V", [2, 3, 4, 6, 8])
def test_kernel_body_on_host_vs_restatement(host_robust, V, J):
    """3 px noise, one 80 px outlier per joint, random weights with absent views"""
    P, X, ue, un = mc.rig(100 * V + J, 6, V, J)
    uo, _ = mc.plant_outliers(un, V + J)
    rng = np.random.default_rng(V * J)
    w = rng.uniform(0.05, 1.0, un.shape[:3]) * (rng.uniform(size=un.shape[:3]) > 0.15)
    _same(host_robust(un, P), _restated(un, P))
    _same(host_robust(uo, P), _restated(uo, P))
    _same(host_robust(uo, P, w, 10.0), _restated(uo, P, w, 10.0))


def test_v2_unit_weights_is_the_pair_dlt_bit_for_bit(host_robust, golden):
    """the masked refit with zero rows for the absent views is dlt_nview<2>: the golden pair case"""
    g = golden("triangulation")
    u1, u2, P1, P2, _ = gi.triangulation_case()
    X, st, inl, _ = host_robust(np.stack([u1, u2], axis=1), np.stack([P1, P2], axis=1), thr=HUGE)
    assert np.max(np.abs(X - g["linear_eigen_triangulation_x"])) <= 1e-6 and st.all() and np.all(inl == 3)


@pytest.mark.parametrize("V", [3, 4, 5, 6, 8])
def test_planted_outlier_is_excluded(host_robust, V):
    """exact projections and one view per joint moved by 80 px.  On cameras spread evenly over the
    ring: with three views of which two face each other, a point moved along the ray those two
    share stays consistent with all three, and no method can tell."""
    P, X, ue = mc.even_rig(7 + V, 8, V, 17)
    uo, which = mc.plant_outliers(ue, V)
    for fn in (host_robust, _restated):
        Xr, st, inl, res = fn(uo, P)
        assert st.all()
        assert np.array_equal(inl, ((1 << V) - 1) & ~(1 << which))
        assert np.max(np.abs(Xr - X)) <= 1e-6 and res.max() <= 1e-6


@pytest.mark.parametrize("V", [3, 4, 8])
def test_noise_and_outliers_against_the_plain_dlt(host_robust, V):
    """3 px noise: never worse than the plain V-view DLT by more than the noise level (3 px at
    about 4.5 m and f = 1145 px is 12 mm); with an outlier planted, less than half its mean error."""
    P, X, ue = mc.even_rig(31 + V, 16, V, 17)
    un = ue + np.random.default_rng(V).normal(0, 3.0, ue.shape)
    plain = lambda u: np.stack([restate.linear_eigen_triangulation_nview(u[t], P[t])[0] for t in range(len(u))])
    level = 3.0 * 5000.0 / 1145.0
    e_r = np.linalg.norm(host_robust(un, P)[0] - X, axis=2)
    e_p = np.linalg.norm(plain(un) - X, axis=2)
    assert np.all(e_r <= e_p + level)
    uo, _ = mc.plant_outliers(un, V)
    Xr, st, _, _ = host_robust(uo, P)
    e_r, e_p = np.linalg.norm(Xr - X, axis=2), np.linalg.norm(plain(uo) - X, axis=2)
    assert st.all() and e_r.mean() < 0.5 * e_p.mean()


def test_degenerate_inputs(host_robust):
    V, J = 4, 17
    P, X, ue, _ = mc.rig(5, 1, V, J)
    zero = lambda r: all(np.all(a == 0) for a in r)
    # all weights zero / a single weighted view
    w = np.zeros((1, V, J))
    assert zero(host_robust(ue, P, w)) and zero(_restated(ue, P, w))
    w[:, 2] = 1.0
    assert zero(host_robust(ue, P, w)) and zero(_restated(ue, P, w))
    # a point behind every camera: the rays meet, but in no camera's front half-space
    assert zero(host_robust(ue, -P)) and zero(_restated(ue, -P))
    # NaN in u: that view is absent for that joint; NaN in three of four views fails the joint
    un = ue.copy()
    un[0, 1, 3, 0] = np.nan
    un[0, :3, 5, 1] = np.nan
    un[0, :, 6] = np.inf
    got, want = host_robust(un, P), _restated(un, P)
    _same(got, want)
    assert got[2][0, 3] == 0b1101 and got[1][0, 3] == 1
    assert got[1][0, 5] == 0 and got[1][0, 6] == 0 and np.all(got[0][0, 5] == 0)
    # NaN / Inf in P or the weights
    Pn = P.copy()
    Pn[0, 0, 1, 2] = np.nan
    _same(host_robust(ue, Pn), _restated(ue, Pn))
    wn = np.ones((1, V, J))
    wn[0, 0, :5], wn[0, 1, 5:9] = np.nan, np.inf
    _same(host_robust(ue, P, wn), _restated(ue, P, wn))
    # identical cameras: depth is undetermined
    Pi = np.repeat(P[:, :1], V, axis=1)
    ui = np.repeat(ue[:, :1], V, axis=1)
    got, want = host_robust(ui, Pi), _restated(ui, Pi)
    assert np.array_equal(got[1], want[1]) and not got[1].any()      # rank 2: reported, not guessed
    ui = ui + np.random.default_rng(2).normal(0, 1.0, ui.shape)
    host_robust(ui, Pi)                              # finite outputs (checked by the fixture)


@pytest.mark.parametrize("V", [3, 4, 8])
def test_zero_weight_equals_deleting_the_view(host_robust, V):
    P, X, ue, un = mc.rig(60 + V, 4, V, 17)
    uo, _ = mc.plant_outliers(un, 3)
    rng = np.random.default_rng(V)
    for drop in (0, V // 2, V - 1):
        w = rng.uniform(0.1, 1.0, uo.shape[:3])
        w[:, drop] = 0.0
        keep = [v for v in range(V) if v != drop]
        Xa, sa, ia, ra = host_robust(uo, P, w)
        Xb, sb, ib, rb = host_robust(uo[:, keep], P[:, keep], w[:, keep])
        low = (1 << drop) - 1
        assert np.array_equal(Xa, Xb) and np.array_equal(sa, sb) and np.array_equal(ra, rb)
        assert np.array_equal(ia, (ib & low) | ((ib & ~low) << 1))


def test_pair_order_is_generated_from_v():
    for V in range(2, mc.MAX_V + 1):
        p = mc.pairs(V)
        assert len(p) == V * (V - 1) // 2 <= 28 and p == sorted(p) and p[0] == (0, 1) and p[-1] == (V - 2, V - 1)


# ------------------------------------------------------------------ view tuples of the H36M db
@pytest.mark.parametrize("name", ["h36m_valid", "h36m_ss_tri"])
def test_view_tuples_on_dict_form_trees(name):
    from tests import dataset_cases as dc
    ds = dc.build(name)
    rows = ds.view_tuples()
    assert rows.shape == (len(ds.db[0]) if name == "h36m_ss_tri" else len(ds.db) // 4, 4)
    seen = set()
    for row in rows:
        recs = ds.tuple_records(row)
        frames = {os.path.basename(r["image"]).rsplit("_c", 1)[0] for r in recs}
        assert len(frames) == 1, frames                   # the same frame ...
        assert [os.path.basename(r["image"]).rsplit("_c", 1)[1] for r in recs] == \
            ["%d.jpg" % (c + 1) for c in range(4)]        # ... once per camera, in camera order
        seen |= frames
    assert len(seen) == len(rows)


@pytest.mark.parametrize("name", ["h36m_fs_train", "h36m_fs_valid", "h36m_ss_train"])
def test_view_tuples_refuses_unaligned_dbs(name):
    """a list-form pickle, and a dict-form one flattened and shuffled for non-TRI training"""
    from tests import dataset_cases as dc
    with pytest.raises(ValueError, match="frame-aligned"):
        dc.build(name).view_tuples()


def test_world_ground_truth_of_the_records_agrees_across_views():
    from tests import dataset_cases as dc
    from lib.core.function import world_joints_of_record
    ds = dc.build("h36m_valid")
    for row in ds.view_tuples():
        recs = ds.tuple_records(row)
        W = np.stack([world_joints_of_record(r) for r in recs])
        assert np.max(np.abs(W - W.mean(0))) <= 1e-9
        for r in recs:
            uv = restate.project(np.asarray(r["cam"].projection_matrix, dtype=np.float64)[:3], W.mean(0))
            assert np.max(np.abs(uv - r["joints_3d"][:, :2])) <= 1e-9
