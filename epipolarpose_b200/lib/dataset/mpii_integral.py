"""MPII -- mirror of the reference lib/dataset/mpii_integral.py, `DATASET: mpii_integral`.

The db comes from `<root>/annot/<image_set>.json` (:48-108): 1-based joints made 0-based, records
with fewer than 2 visible joints skipped, the box of the visible joints grown to the patch's
aspect ratio and then by 1.25.  Items are the reference's 4-tuple (meta = {'image'}) in the main
process and deferred samples in a DataLoader worker (JointIntegralDataset.sample).

`evaluate` is PCKh@0.5 (SC_BIAS 0.6) against `annot/gt_<TEST_SET>.mat` (:110-195), restated as
the same few vectorised numpy operations on the host: `preds + 1`, `pred.mat` when save_path is
given, {'Null': 0.0} for a test set, joints 6-7 left out of the means, Mean@0.1 from row 11 of
the threshold sweep np.arange(0, 0.51, 0.01)."""
import copy
import json
import logging
import os

import numpy as np

from .JointIntegralDataset import JointsIntegralDataset
from ..utils.utils import calc_kpt_bound

logger = logging.getLogger(__name__)


class MPIIDataset(JointsIntegralDataset):
    def __init__(self, cfg, root, image_set, is_train):
        super().__init__(cfg, root, image_set, is_train)
        self.num_joints = 16
        self.flip_pairs = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
        self.parent_ids = [1, 2, 6, 6, 3, 4, 6, 6, 7, 8, 11, 12, 7, 7, 13, 14]
        self.db = self._get_db()
        self.db_length = len(self.db)
        logger.info('=> load {} samples'.format(len(self.db)))

    def __getitem__(self, idx):
        the_db = copy.deepcopy(self.db[idx])
        return self.sample(the_db['image'], the_db, the_db['joints_3d_vis'].copy(), self.flip_pairs,
                           self.parent_ids, {'image': the_db['image']})

    def _get_db(self):
        with open(os.path.join(self.root, 'annot', self.image_set + '.json')) as f:
            anno = json.load(f)
        aspect_ratio = self.patch_width * 1.0 / self.patch_height
        gt_db = []
        for a in anno:
            jts_3d = np.zeros((self.num_joints, 3), dtype=np.float64)
            jts_3d_vis = np.zeros((self.num_joints, 3), dtype=np.float64)
            if self.image_set != 'test':
                jts = np.array(a['joints'])
                jts[:, 0:2] = jts[:, 0:2] - 1
                jts_vis = np.array(a['joints_vis'])
                assert len(jts) == self.num_joints, 'joint num diff: {} vs {}'.format(len(jts), self.num_joints)
                jts_3d[:, 0:2] = jts[:, 0:2]
                jts_3d_vis[:, 0] = jts_vis[:]
                jts_3d_vis[:, 1] = jts_vis[:]
            if np.sum(jts_3d_vis[:, 0]) < 2:
                continue
            u, d, l, r = calc_kpt_bound(jts_3d, jts_3d_vis)
            center = np.array([(l + r) * 0.5, (u + d) * 0.5], dtype=np.float32)
            assert center[0] >= 1
            w, h = r - l, d - u
            assert w > 0 and h > 0
            if w > aspect_ratio * h:
                h = w * 1.0 / aspect_ratio
            elif w < aspect_ratio * h:
                w = h * aspect_ratio
            gt_db.append({'image': os.path.join(self.root, 'images', a['image']),
                          'center_x': center[0], 'center_y': center[1],
                          'width': w * 1.25, 'height': h * 1.25,
                          'flip_pairs': self.flip_pairs, 'parent_ids': self.parent_ids,
                          'joints_3d': jts_3d, 'joints_3d_vis': jts_3d_vis})
        return gt_db

    def evaluate(self, preds, save_path=None, debug=False):
        preds = preds[:, :, 0:2] + 1.0                      # 0-based -> 1-based
        if save_path:
            from scipy.io import savemat
            savemat(os.path.join(save_path, 'pred.mat'), mdict={'preds': preds})
        if 'test' in self.cfg.DATASET.TEST_SET:
            return {'Null': 0.0}, 0.0
        from scipy.io import loadmat
        gt = loadmat(os.path.join(self.cfg.DATASET.ROOT, 'annot', 'gt_{}.mat'.format(self.cfg.DATASET.TEST_SET)))
        names = gt['dataset_joints']
        jid = lambda n: np.where(names == n)[1][0]
        visible = 1 - gt['jnt_missing']                                          # [16, S]
        err = np.linalg.norm(np.transpose(preds, [1, 2, 0]) - gt['pos_gt_src'], axis=1)
        head = np.linalg.norm(gt['headboxes_src'][1, :, :] - gt['headboxes_src'][0, :, :], axis=0)
        head *= 0.6                                                              # SC_BIAS
        scaled = np.multiply(np.divide(err, np.multiply(head, np.ones((len(err), 1)))), visible)
        count = np.sum(visible, axis=1)

        def pck(threshold):
            return np.divide(100. * np.sum(np.multiply(scaled <= threshold, visible), axis=1), count)

        PCKh = pck(0.5)
        sweep = np.arange(0, 0.5 + 0.01, 0.01)
        pck_all = np.zeros((len(sweep), 16))
        for r in range(len(sweep)):
            pck_all[r, :] = pck(sweep[r])
        PCKh = np.ma.array(PCKh, mask=False)
        PCKh.mask[6:8] = True                                # pelvis and thorax
        count = np.ma.array(count, mask=False)
        count.mask[6:8] = True
        ratio = count / np.sum(count).astype(np.float64)
        pair = lambda a, b: 0.5 * (PCKh[jid(a)] + PCKh[jid(b)])
        name_value = [('Head', PCKh[jid('head')]), ('Shoulder', pair('lsho', 'rsho')),
                      ('Elbow', pair('lelb', 'relb')), ('Wrist', pair('lwri', 'rwri')),
                      ('Hip', pair('lhip', 'rhip')), ('Knee', pair('lkne', 'rkne')),
                      ('Ankle', pair('lank', 'rank')), ('Mean', np.sum(PCKh * ratio)),
                      ('Mean@0.1', np.sum(pck_all[11, :] * ratio))]
        return name_value, np.sum(PCKh * ratio)
