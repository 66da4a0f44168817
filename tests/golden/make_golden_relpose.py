"""Golden vectors for the relative-pose estimator (oracle/restate_relpose.py), produced with the
installed OpenCV -- not with reference code, which has no caller for this step.  Build
container only:
    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_relpose.py

Inputs: tests/relpose_cases.py::rig_pairs (ring rigs, 0-3 px noise, 0-3 outlier joints), plus
noise- and outlier-free pairs for recoverPose.
  f8      : cv2.findFundamentalMat(FM_8POINT) on the oracle's inlier set of each pair;
  R1, R2, t : cv2.decomposeEssentialMat of the oracle's E;
  rp_R, rp_t : cv2.recoverPose(E, K_a^-1 u_a, K_b^-1 u_b) on the well-conditioned (exact) pairs."""
import os
import sys

import cv2
import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
sys.path.insert(0, ROOT)
from oracle import restate_relpose as rr  # noqa: E402
from tests import relpose_cases as rc  # noqa: E402

N, N_EXACT = 24, 8


def normalised(u, intr):
    return np.stack([(u[:, 0] - intr[2]) / intr[0], (u[:, 1] - intr[3]) / intr[1]], axis=1)


d = rc.rig_pairs(N, 11)
e = rc.rig_pairs(N_EXACT, 12, noise_px=(0.0, 0.0), n_out=(0, 0))
out = {k: [] for k in ("f8", "R1", "R2", "t", "rp_R", "rp_t")}
for i in range(N):
    o = rr.relative_pose(d["ua"][i], d["ub"][i], d["intr_a"][i], d["intr_b"][i], d["box_a"][i], d["box_b"][i])
    assert o["F"] is not None and o["status"] == 1, i
    inl = o["inliers"]
    out["f8"].append(cv2.findFundamentalMat(d["ua"][i][inl], d["ub"][i][inl], cv2.FM_8POINT)[0])
    R1, R2, t = cv2.decomposeEssentialMat(o["E"])
    out["R1"].append(R1); out["R2"].append(R2); out["t"].append(t.reshape(3))
for i in range(N_EXACT):
    o = rr.relative_pose(e["ua"][i], e["ub"][i], e["intr_a"][i], e["intr_b"][i], e["box_a"][i], e["box_b"][i])
    na, nb = normalised(e["ua"][i], e["intr_a"][i]), normalised(e["ub"][i], e["intr_b"][i])
    _, R, t, _ = cv2.recoverPose(o["E"], na, nb)
    out["rp_R"].append(R); out["rp_t"].append(t.reshape(3))
np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "relpose.npz"),
                    **{k: np.asarray(v) for k, v in out.items()})
print("wrote relpose", {k: np.asarray(v).shape for k, v in out.items()})
