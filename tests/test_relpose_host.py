"""CPU: the relative-pose estimator for self-supervision without camera extrinsics.  The numpy
oracle (oracle/restate_relpose.py) against OpenCV (tests/golden/relpose.npz), the per-pair body
of relative_pose_kernel (csrc/geometry.cu) run on the CPU by tests/harness/host_relpose.cu
against the oracle, degenerate inputs, and the configuration rule."""
import os
import subprocess

import numpy as np
import pytest

from oracle import restate_relpose as rr
from tests import relpose_cases as rc
from tests.conftest import ROOT, relerr

N_HYP = rr.N_HYP


def _unit(x):
    return x / np.linalg.norm(x)


def test_oracle_against_opencv(golden):
    g = golden("relpose")
    d = rc.rig_pairs(len(g["f8"]), 11)
    for i in range(len(g["f8"])):
        o = rr.relative_pose(d["ua"][i], d["ub"][i], d["intr_a"][i], d["intr_b"][i], d["box_a"][i],
                             d["box_b"][i])
        # F up to sign and scale
        F, Fc = o["F"] / np.linalg.norm(o["F"]), g["f8"][i] / np.linalg.norm(g["f8"][i])
        Fc = Fc if np.sum(F * Fc) > 0 else -Fc
        assert np.max(np.abs(F - Fc)) <= 1e-9, i
        # the two rotations of E (as a set) and t up to sign
        c = rr.candidates(o["E"])
        mine = [c[0][0], c[2][0]]
        for Rc in (g["R1"][i], g["R2"][i]):
            assert min(np.max(np.abs(Rc - R)) for R in mine) <= 1e-9, i
        assert min(np.max(np.abs(c[0][1] - s * g["t"][i])) for s in (1, -1)) <= 1e-9, i
    e = rc.rig_pairs(len(g["rp_R"]), 12, noise_px=(0.0, 0.0), n_out=(0, 0))
    for i in range(len(g["rp_R"])):
        o = rr.relative_pose(e["ua"][i], e["ub"][i], e["intr_a"][i], e["intr_b"][i], e["box_a"][i],
                             e["box_b"][i])
        assert o["status"] == 1
        assert np.max(np.abs(o["R"] - g["rp_R"][i])) <= 1e-9, i
        assert np.max(np.abs(_unit(o["t"]) - _unit(g["rp_t"][i]))) <= 1e-9, i
        # and both against the rig's true relative pose
        assert np.max(np.abs(o["R"] - e["R_ab"][i])) <= 1e-4     # float32 points (FM_8POINT)
        assert np.max(np.abs(_unit(o["t"]) - e["t_dir"][i])) <= 1e-4


@pytest.fixture(scope="module")
def host_relpose(tmp_path_factory):
    """tests/harness/host_relpose.cu: relpose_pair of csrc/geometry.cu built for the CPU."""
    import shutil
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("harness") / "host_relpose")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "--fmad=false", "-O1",
                        "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "harness", "host_relpose.cu")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(ua, ub, ia, ib, ba, bb, rect3d_w=2000.0):
        n, J = ua.shape[0], ua.shape[1]
        inp = b"".join(np.concatenate([ua[i].ravel(), ub[i].ravel(), ia[i], ib[i], ba[i], bb[i],
                                       [rect3d_w]]).astype(np.float64).tobytes() for i in range(n))
        out = subprocess.run([exe, "pairs", str(n), str(J)], input=inp, capture_output=True)
        assert out.returncode == 0, out.stderr
        a = np.frombuffer(out.stdout, dtype=np.float64).reshape(n, -1)
        return [dict(P_a=r[0:12], P_b=r[12:24], cam_a=r[24:40], cam_b=r[40:56], inliers=r[56:56 + J] != 0,
                     status=int(r[56 + J]), best_h=int(r[57 + J]), cand=int(r[58 + J]), n_inl=int(r[59 + J]),
                     scores=r[60 + J:60 + J + N_HYP]) for r in a]
    return run


def _run_both(host_relpose, d):
    keys = ("ua", "ub", "intr_a", "intr_b", "box_a", "box_b")
    res = host_relpose(*[d[k] for k in keys])
    orc = [rr.relative_pose(*[d[k][i] for k in keys]) for i in range(len(d["ua"]))]
    return res, orc


def test_relative_pose_kernel_body_on_host(host_relpose):
    """relpose_pair, the per-pair body of relative_pose_kernel, on the CPU against the oracle:
    identical hypothesis, inliers and candidate; P and cam to 1e-9 relative."""
    d = rc.rig_pairs(64, 7)
    res, orc = _run_both(host_relpose, d)
    n_ok = 0
    for i, (a, o) in enumerate(zip(res, orc)):
        assert np.array_equal(np.isnan(a["scores"]), np.isnan(o["scores"])), i
        assert (a["best_h"], a["cand"], a["n_inl"], a["status"]) == \
            (o["best_h"], o["cand"], o["n_inl"], o["status"]), i
        assert np.array_equal(a["inliers"], o["inliers"]), i
        for k in ("P_a", "P_b", "cam_a", "cam_b"):
            assert relerr(a[k], np.ravel(o[k])) <= 1e-9, (i, k)
        n_ok += o["status"]
    assert n_ok >= 56                        # the estimate fails only for a few noisy pairs


def test_outlier_joints_are_rejected_on_host(host_relpose):
    """Exact projections with up to 3 joints replaced by random points: the replaced joints are
    not inliers and the pose is the rig's own."""
    d = rc.rig_pairs(16, 21, noise_px=(0.0, 0.0), n_out=(1, 3))
    res, _ = _run_both(host_relpose, d)
    for i, a in enumerate(res):
        assert a["status"] == 1, i
        assert not np.any(a["inliers"] & d["outliers"][i]), i
        R = a["cam_b"][:9].reshape(3, 3)
        t = -R @ a["cam_b"][9:12]
        assert np.max(np.abs(R - d["R_ab"][i])) <= 1e-4, i      # float32 points (FM_8POINT)
        assert np.max(np.abs(_unit(t) - d["t_dir"][i])) <= 1e-4, i


def test_degenerate_inputs_give_status_zero_on_host(host_relpose):
    d = rc.rig_pairs(3, 23, noise_px=(1.0, 1.0), n_out=(0, 0))
    cases = []
    same = {k: d[k][0:1].copy() for k in ("ua", "ub", "intr_a", "intr_b", "box_a", "box_b")}
    same["ua"][:] = 500.0
    same["ub"][:] = 480.0
    cases.append(same)                                   # all points equal
    ident = {k: d[k][1:2].copy() for k in ("ua", "ub", "intr_a", "intr_b", "box_a", "box_b")}
    ident["ub"] = ident["ua"].copy()
    ident["intr_b"] = ident["intr_a"].copy()
    cases.append(ident)                                  # identical views
    j8 = {k: d[k][2:3].copy() for k in ("ua", "ub", "intr_a", "intr_b", "box_a", "box_b")}
    j8["ua"], j8["ub"] = j8["ua"][:, :8].copy(), j8["ub"][:, :8].copy()
    j8["ua"][0, 5, 0] = np.nan
    cases.append(j8)                                     # J = 8 with one NaN joint
    for c in cases:
        (a,), (o,) = _run_both(host_relpose, c)
        assert a["status"] == 0 and o["status"] == 0
        for k in ("P_a", "P_b", "cam_a", "cam_b"):
            assert np.isfinite(a[k]).all(), k
        assert np.array_equal(a["cam_b"][:12], np.concatenate([np.eye(3).ravel(), np.zeros(3)]))


def test_estimate_extrinsics_needs_online_triangulation(tmp_path):
    from lib.core.config import update_config, reset_config, config
    import lib.core.function as fn
    y = tmp_path / "est.yaml"
    y.write_text("TRAIN:\n  ESTIMATE_EXTRINSICS: true\n")
    reset_config()
    try:
        with pytest.raises(ValueError):
            update_config(str(y))
        reset_config()
        config.TRAIN.ESTIMATE_EXTRINSICS = True
        with pytest.raises(ValueError):
            fn._estimate_extrinsics(config)
        y.write_text("TRAIN:\n  ONLINE_TRIANGULATION: true\n  ESTIMATE_EXTRINSICS: true\n")
        reset_config()
        update_config(str(y))
        assert fn._estimate_extrinsics(config) is True
        with pytest.raises(ValueError):
            fn.GraphedTrainStep(None, None, None, online=False, estimate_extrinsics=True)
    finally:
        reset_config()
