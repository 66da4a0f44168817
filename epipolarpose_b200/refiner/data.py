"""Refiner datasets -- host-side mirror of the reference refiner/data.py.

`Human36M(is_train, root='refiner/data')` is the reference class (refiner/data.py:29-160): it reads
`train.pkl` / `valid.pkl` ({'inp', 'out'}, [S,16,3] or [S,48], MPII joint order), drops the hip
(columns 18:21, joint 6), normalises with `norm.pkl` (written by the train split when absent),
shuffles the train split with the global numpy generator, and `evaluate(preds)` scores
denormalised second-head outputs.  One difference: the valid split without `norm.pkl` raises
FileNotFoundError (the reference fails there with UnboundLocalError).  The reference never
released the script that wrote its files: reading the inputs as `pred_to_save['pred']` of the H36M
evaluation (root-relative camera-frame mm, MPII order) and the targets as its `gt` is an inference
from the reference.

`SyntheticPoses` is a stand-in with the same interface over seeded root-relative 15-joint poses
(inputs = targets + noise), for runs without the data files."""
import logging
import os
import pickle

import numpy as np
import torch

logger = logging.getLogger(__name__)

MPII_NAMES = ['RFoot', 'RKnee', 'RHip', 'LHip', 'LKnee', 'LFoot', 'Thorax', 'Neck/Nose', 'Head',
              'RWrist', 'RElbow', 'RShoulder', 'LShoulder', 'LElbow', 'LWrist']   # hip removed
J14 = [0, 1, 2, 3, 4, 5, 6, 9, 10, 11, 12, 13, 14]
RESULT_NAMES = ('hm36_17j', 'hm36_17j_align', 'hm36_17j_14', 'hm36_17j_14_al',
                'hm36_17j_x', 'hm36_17j_y', 'hm36_17j_z')

_backend = [None]      # test hook: an ops module emulating the C ABI on the CPU


def pose_errors(pred, gt, subset=J14):
    """Per-sample errors of camera-frame poses pred, gt [S, J, 3] (epb_pose_errors, float64):
    -> (metrics [S, 7] in the order of RESULT_NAMES, per-joint errors [S, J])."""
    from epipolarpose_b200 import ops as _ops
    ops = _backend[0] or _ops
    dev = torch.device("cuda") if ops is _ops else torch.device("cpu")
    p = torch.as_tensor(np.ascontiguousarray(pred, dtype=np.float64)).to(dev)
    g = torch.as_tensor(np.ascontiguousarray(gt, dtype=np.float64)).to(dev)
    S, J = p.shape[0], p.shape[1]
    if g.shape != p.shape or p.dim() != 3 or p.shape[2] != 3:
        raise ValueError("pred and gt must both be [S, J, 3]")
    metrics = torch.empty((S, 7), dtype=torch.float64, device=dev)
    per_joint = torch.empty((S, J), dtype=torch.float64, device=dev)
    ops.pose_errors(p, g, S, J, sum(1 << j for j in subset), metrics, per_joint)
    return metrics.cpu().numpy(), per_joint.cpu().numpy()


class Human36M(torch.utils.data.Dataset):
    def __init__(self, is_train, root='refiner/data'):
        fname = os.path.join(root, 'train.pkl' if is_train else 'valid.pkl')
        self.is_train = is_train
        self.root = root
        (self.data, self.labels, self.data_mean, self.data_std, self.labels_mean,
         self.labels_std) = self.get_db(fname)
        logger.info('loaded %s samples from %s', len(self.data), fname)

    def get_db(self, fname):
        with open(fname, 'rb') as f:
            anno = pickle.load(f)
        data = np.asarray(anno['inp'], dtype=np.float32).reshape(len(anno['inp']), -1)
        labels = np.asarray(anno['out'], dtype=np.float32).reshape(len(anno['out']), -1)
        data = np.delete(data, np.s_[18:21], axis=1)          # the hip joint
        labels = np.delete(labels, np.s_[18:21], axis=1)
        norm = os.path.join(self.root, 'norm.pkl')
        if os.path.exists(norm):
            with open(norm, 'rb') as f:
                data_mean, data_std, labels_mean, labels_std = pickle.load(f)
        elif self.is_train:
            data_mean, data_std = data.mean(axis=0), data.std(axis=0)
            labels_mean, labels_std = labels.mean(axis=0), labels.std(axis=0)
            with open(norm, 'wb') as f:
                pickle.dump((data_mean, data_std, labels_mean, labels_std), f)
        else:
            raise FileNotFoundError("%s does not exist: the valid split is normalised with the statistics "
                                    "the train split writes there" % norm)
        data = (data - data_mean) / data_std
        if self.is_train:
            labels = (labels - labels_mean) / labels_std
            rnd = np.random.permutation(labels.shape[0])
            data, labels = data[rnd], labels[rnd]
        return data, labels, data_mean, data_std, labels_mean, labels_std

    def __getitem__(self, index):
        return self.data[index], self.labels[index]

    def __len__(self):
        return len(self.labels)

    def norm(self):
        """(data_mean, data_std, labels_mean, labels_std), the contents of norm.pkl."""
        return self.data_mean, self.data_std, self.labels_mean, self.labels_std

    def evaluate(self, preds):
        """preds [S, 45] normalised second-head outputs -> mean per-joint error (mm); logs the
        per-joint errors and the seven means under the reference's names."""
        preds = np.asarray(preds) * self.labels_std + self.labels_mean        # float32, as the reference
        preds = preds.reshape((preds.shape[0], -1, 3))
        gt = self.labels[:len(preds)].reshape((len(preds), -1, 3))
        metrics, per_joint = pose_errors(preds, gt)
        per_joint_error = per_joint.mean(axis=0).tolist()
        logger.info('=== JOINTS ===')
        for name, e in zip(MPII_NAMES, per_joint_error):
            logger.info('%s : %s', name, e)
        results = dict(zip(RESULT_NAMES, metrics.mean(axis=0)))
        logger.info('=== RESULTS ===')
        for k, v in results.items():
            logger.info('%s : %s', k, v)
        logger.info('===============')
        self.last_results, self.last_per_joint = results, per_joint_error
        return results['hm36_17j']


class SyntheticPoses(torch.utils.data.Dataset):
    def __init__(self, is_train=True, n=None, seed=0, noise=0.05):
        n = n if n is not None else (4096 if is_train else 1024)
        rng = np.random.default_rng(seed + (0 if is_train else 1))
        tar = rng.normal(0.0, 0.3, (n, 15, 3)).astype(np.float32)
        tar[:, 0] = 0.0                                            # root-relative
        self.tar = tar.reshape(n, 45)
        self.inp = (self.tar + rng.normal(0.0, noise, (n, 45))).astype(np.float32)

    def __len__(self):
        return len(self.tar)

    def __getitem__(self, i):
        return torch.from_numpy(self.inp[i]), torch.from_numpy(self.tar[i])

    def evaluate(self, preds):
        """mean per-joint position error of [n, 45] predictions (reference data.py evaluate)."""
        p = np.asarray(preds, dtype=np.float64).reshape(-1, 15, 3)
        t = self.tar[:len(p)].astype(np.float64).reshape(-1, 15, 3)
        return float(np.sqrt(((p - t) ** 2).sum(2)).mean())
