"""TEST INFRASTRUCTURE: CPU emulation of epb_pose_errors / epb_pose_to_camera with the SAME
signatures as epipolarpose_b200.ops, on torch CPU tensors, running the float64 restatement of
tests/refiner_cases.py, so that host tests can swap it in as refiner/data.py's backend
(`data._backend[0]`).  Never imported by the product path."""
import torch

from tests import refiner_cases as rc


def pose_errors(pred, gt, S, J, submask, metrics, per_joint):
    subset = [j for j in range(J) if (submask >> j) & 1]
    m, pj = rc.pose_errors(pred.reshape(S, J, 3).numpy(), gt.reshape(S, J, 3).numpy(), subset)
    metrics.copy_(torch.from_numpy(m).view_as(metrics))
    if per_joint is not None:
        per_joint.copy_(torch.from_numpy(pj).view_as(per_joint))


def pose_to_camera(joints, cam, N, J, root, out):
    out.copy_(torch.from_numpy(rc.pose_to_camera(joints.reshape(N, J, 3).numpy(), cam.reshape(N, 5).numpy(),
                                                 root)).view_as(out))
