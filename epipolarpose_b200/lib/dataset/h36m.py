"""Human3.6M -- mirror of the reference lib/dataset/h36m.py (:18-378), `DATASET: h36m`.

The db comes from `<root>/annot/<image_set>.pkl`: a list of records, or a dict of per-camera
lists keyed 1..NUM_CAMS.  The construction-time draws are the reference's, in its order
(np.random.permutation of the dict form, then random.shuffle), so a seeded run builds the same
db.  With DATASET.TRI a training item draws a camera (np.random) and one of its neighbours in
cam_config (random) and returns {'cam_1': view, 'cam_2': view} of the same frame index.

A view is the reference's (img_patch, label, label_weight, meta) in the main process and a
deferred sample in a DataLoader worker (JointIntegralDataset.sample).  `evaluate` runs the H36M
protocol through evaluate_h36m (epb_h36m_eval) and, for each k of TEST.PSS_K, appends PSS@k
(lib/core/pss.py), and with TEST.REFINER the four Refined-* entries of the refined poses
(lib/core/refine.py); the DEBUG.DEBUG plots are not built."""
import copy
import logging
import os
import random

import numpy as np

from .JointIntegralDataset import JointsIntegralDataset, H36M_NAMES, MPII_NAMES, load_pickle
from .h36m_eval import evaluate_h36m
from ..core.pss import h36m_pss
from ..core.refine import check_refiner_config, h36m_refined
from ..utils.data_utils import define_actions

logger = logging.getLogger(__name__)

_META_CAM = ('R', 'T', 'f', 'c', 'projection_matrix')


class H36M_Integral(JointsIntegralDataset):
    def __init__(self, cfg, root, image_set, is_train):
        super().__init__(cfg, root, image_set, is_train)
        self.parent_ids = np.array([0, 0, 1, 2, 0, 4, 5, 0, 8, 8, 9, 8, 11, 12, 8, 14, 15], dtype=np.int64)
        self.cam_config = [[1, 2], [0, 3], [0, 3], [1, 2]]          # camera neighbourhoods (:25)
        self.db = self._get_train_db() if is_train else self._get_val_db()
        logger.info('=> load {} samples'.format(self.db_length))

    def __getitem__(self, idx):
        if self.is_train and self.cfg.DATASET.TRI:
            cam_1 = np.random.randint(self.num_cams)
            cam_2 = self.cam_config[cam_1][0] if random.random() <= 0.5 else self.cam_config[cam_1][1]
            bundle_1 = self.get_data(copy.deepcopy(self.db[cam_1][idx]))
            bundle_2 = self.get_data(copy.deepcopy(self.db[cam_2][idx]))
            return {'cam_1': bundle_1, 'cam_2': bundle_2}
        return self.get_data(copy.deepcopy(self.db[idx]))

    def get_data(self, the_db):
        image_file = os.path.join(self.root, the_db['image'])
        cam = the_db['cam']
        joints_vis = the_db['joints_3d_vis'].copy()
        joints_vis[:, 2] *= self.cfg.DATASET.Z_WEIGHT
        meta = {'image': image_file, 'center_x': the_db['center_x'], 'center_y': the_db['center_y'],
                'width': the_db['width'], 'height': the_db['height'], 'scale': 1.0, 'rot': 0.0}
        for k in _META_CAM:
            meta[k] = getattr(cam, k)
        return self.sample(image_file, the_db, joints_vis, the_db['flip_pairs'], the_db['parent_ids'], meta)

    def _load(self):
        anno = load_pickle(os.path.join(self.root, 'annot', self.image_set + '.pkl'))
        self._dict_form = isinstance(anno, dict)
        return anno

    def view_tuples(self):
        """int array [T, V]: row k holds, camera by camera, the db indices that show frame k.
        The dict-form annotation keeps one frame-aligned list per camera and _per_camera applies
        one permutation to all of them, so in the validation db (flattened camera by camera) row
        k is [cid * T + k for cid in range(NUM_CAMS)]; in the DATASET.TRI training db, which stays
        per camera, entry [k, cid] indexes self.db[cid] (it is k).  tuple_records(row) returns the
        records either way.  A list-form pickle, and the shuffled non-TRI training db, carry no
        such alignment: ValueError."""
        tri = self.is_train and self.cfg.DATASET.TRI
        if not self._dict_form or (self.is_train and not tri):
            raise ValueError("view_tuples needs frame-aligned cameras: a dict-form annotation pickle (one list "
                             "per camera), read as the validation db or as the DATASET.TRI training db; a "
                             "list-form pickle or a shuffled training db does not say which records show the "
                             "same frame")
        V = self.num_cams
        if tri:
            T = len(self.db[0])
            return np.repeat(np.arange(T, dtype=np.int64)[:, None], V, axis=1)
        T = len(self.db) // V
        return np.arange(T, dtype=np.int64)[:, None] + T * np.arange(V, dtype=np.int64)[None, :]

    def tuple_records(self, row):
        """The V records of one row of view_tuples()."""
        if self.is_train and self.cfg.DATASET.TRI:
            return [self.db[cid][int(i)] for cid, i in enumerate(row)]
        return [self.db[int(i)] for i in row]

    @staticmethod
    def _per_camera(anno, num_cams):
        """dict form: one list per camera, frames in one np.random.permutation order."""
        gt_db = [[] for _ in range(num_cams)]
        for idx in np.random.permutation(len(anno[1])):
            for cid in range(num_cams):
                gt_db[cid].append(anno[cid + 1][idx])
        return gt_db

    def _get_train_db(self):
        anno = self._load()
        if isinstance(anno, dict):
            gt_db = self._per_camera(anno, self.num_cams)
            self.db_length = len(gt_db[0])
            if not self.cfg.DATASET.TRI:
                gt_db = [rec for db in gt_db for rec in db]
                random.shuffle(gt_db)
                self.db_length = len(gt_db)
        else:
            gt_db = list(anno)
            random.shuffle(gt_db)
            self.db_length = len(gt_db)
        return gt_db

    def _get_val_db(self):
        anno = self._load()
        if isinstance(anno, dict):
            gt_db = [rec for db in self._per_camera(anno, self.num_cams) for rec in db]
        else:
            gt_db = list(anno)
        self.db_length = len(gt_db)
        return gt_db

    def evaluate(self, preds, save_path=None, debug=False, actionwise=False):
        """H36M protocol #1 / aligned / scale-normalised errors (reference :168-378) ->
        (name_value, perf).  With `actionwise`, `self.action_errors` maps each action of
        define_actions('All') to the mean (MPJPE, aligned MPJPE) of its samples, as printed."""
        preds = np.asarray(preds)[:, :, 0:3]
        S = preds.shape[0]
        gts = self.db[:S]
        get = lambda k: np.stack([np.asarray(g[k], dtype=np.float64).reshape(-1) for g in gts]) \
            if S else np.zeros((0, 3))
        mpii = bool(self.cfg.DATASET.MPII_ORDER)
        gt = np.stack([np.asarray(g['joints_3d'], dtype=np.float64) for g in gts]) if S else np.zeros((0, 17, 3))
        test = getattr(self.cfg, 'TEST', None)
        refiner = check_refiner_config(test, mpii, preds.shape[1])
        name_value, perf, details = evaluate_h36m(preds, gt, get('pelvis'), get('fl'), get('c_p'), mpii_order=mpii,
                                                  return_poses=refiner is not None)
        pss_k = list(getattr(test, 'PSS_K', None) or [])
        if pss_k:
            name_value = name_value + h36m_pss(preds, gt, get('pelvis'), get('fl'), get('c_p'), mpii, pss_k,
                                               os.path.join(self.root, 'annot', 'train-fs.pkl'),
                                               getattr(test, 'PSS_CENTROIDS', ''))
        if refiner is not None:
            name_value = name_value + h36m_refined(details['poses'], *refiner)
        per_joint_error = details['per_joint'].mean(axis=0).tolist()
        for name, err in zip(MPII_NAMES if mpii else H36M_NAMES, per_joint_error):
            print(name, err)
        if actionwise:
            m = details['metrics']
            acts = np.array([g['action'] for g in gts])
            self.action_errors = {}
            for col in (0, 1):
                print('========================')
                for act in define_actions('All'):
                    sel = m[acts == act, col]
                    v = sel.mean() if sel.size else float('nan')
                    self.action_errors.setdefault(act, [None, None])[col] = v
                    print(act, v)
                print('========================')
            self.action_errors = {k: tuple(v) for k, v in self.action_errors.items()}
        return name_value, perf
