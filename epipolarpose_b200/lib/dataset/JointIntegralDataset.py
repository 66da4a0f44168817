"""Base class of the image datasets -- mirror of the reference lib/dataset/JointIntegralDataset.py
(:9-91): the joint-name tables, H36M_TO_MPII_PERM (one copy, shared with h36m_eval.py), the
patch / depth geometry and normalisation constants, occluders from DATASET.VOC when
DATASET.OCCLUSION is set for training.

What the reference does in one `get_single_patch_sample` call (read, augment, crop, label) is
split here in two, so that DataLoader workers never touch CUDA:
  * in the main process (direct indexing, num_workers=0) `sample` returns the reference's
    4-tuple through get_single_patch_sample, as the reference does;
  * in a DataLoader worker it returns a deferred sample (deferred.make_deferred): the file's
    bytes and the augmentation / occluder draws, which `assemble_batch` turns into a device
    batch in the main process.
Annotation pickles name the reference's `lib.utils.cameras.Camera`; `load_pickle` resolves
`lib.*` to this package, however it was imported."""
import logging
import os
import pickle

import numpy as np
from torch.utils.data import Dataset, get_worker_info

from ..core.integral_loss import get_label_func
from ..utils.augmentation import load_occluders
from ..utils.img_utils import get_single_patch_sample
from . import deferred as _deferred
from .h36m_eval import H36M_NAMES, MPII_NAMES, H36M_TO_MPII_PERM  # noqa: F401  (reference :9-48)

logger = logging.getLogger(__name__)

_LIB = __name__.rsplit('.dataset.', 1)[0]          # 'lib' or 'epipolarpose_b200.lib'


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if module == 'lib' or module.startswith('lib.'):
            module = _LIB + module[3:]
        return super().find_class(module, name)


def load_pickle(path):
    """pickle.load of an annotation file whose records may hold reference `lib.*` objects."""
    with open(path, 'rb') as f:
        return _Unpickler(f).load()


class JointsIntegralDataset(Dataset):
    def __init__(self, cfg, root, image_set, is_train):
        self.cfg = cfg
        self.is_train = is_train
        self.root = root
        self.image_set = image_set
        self.patch_width = cfg.MODEL.IMAGE_SIZE[0]
        self.patch_height = cfg.MODEL.IMAGE_SIZE[1]
        self.rect_3d_width = 2000.
        self.rect_3d_height = 2000.
        self.mean = np.array([123.675, 116.280, 103.530])
        self.std = np.array([58.395, 57.120, 57.375])
        self.num_cams = cfg.DATASET.NUM_CAMS
        self.label_func = get_label_func()
        self.occluders = load_occluders(cfg.DATASET.VOC) if cfg.DATASET.OCCLUSION and is_train else None
        self.cam_config = []
        self.parent_ids = None
        self.db_length = 0
        self.db = []

    def __len__(self):
        return self.db_length

    def __getitem__(self, idx):
        raise NotImplementedError

    def evaluate(self, preds, save_path=None, debug=False):
        raise NotImplementedError

    def sample(self, image_file, rec, joints_vis, flip_pairs, parent_ids, meta):
        """One view: the reference's (img_patch, label, label_weight, meta) in the main process,
        a deferred sample in a DataLoader worker.  `meta` gets the drawn scale / rot."""
        box = (rec['center_x'], rec['center_y'], rec['width'], rec['height'])
        if get_worker_info() is not None:
            with open(image_file, 'rb') as f:
                blob = f.read()
            return _deferred.make_deferred(
                blob, box, rec['joints_3d'], joints_vis, flip_pairs, self.is_train, self.occluders,
                (self.patch_width, self.patch_height, self.rect_3d_width), self.mean, self.std, meta)
        img_patch, label, label_weight, scale, rot = get_single_patch_sample(
            image_file, box[0], box[1], box[2], box[3], rec['joints_3d'].copy(), joints_vis,
            list(flip_pairs).copy(), np.copy(parent_ids), self.patch_width, self.patch_height,
            self.rect_3d_width, self.rect_3d_height, self.mean, self.std, self.is_train, self.label_func,
            occluder=self.occluders)
        if 'scale' in meta:
            meta['scale'], meta['rot'] = float(scale), float(rot)
        return img_patch.astype(np.float32), label.astype(np.float32), label_weight.astype(np.float32), meta
