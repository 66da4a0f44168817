"""Shared by tests/test_datasets_host.py and tests/test_gpu_datasets.py: the fixture tree of
tests/golden/make_golden_datasets.py, its cases and the config the reference classes were run with."""
import hashlib
import os
import random
import types

import numpy as np

from tests.conftest import GOLDEN

TREE = os.path.join(GOLDEN, "datasets")
H36M_ROOT = os.path.join(TREE, "h36m")
MPII_ROOT = os.path.join(TREE, "mpii")
SEED = 20261016

H36M_CASES = {          # name: (image_set, is_train, TRI, Z_WEIGHT)
    "h36m_fs_train": ("train-fs", True, False, 1.0),
    "h36m_ss_train": ("train-ss", True, False, 0.5),
    "h36m_ss_tri": ("train-ss", True, True, 1.0),
    "h36m_valid": ("valid", False, False, 1.0),
    "h36m_fs_valid": ("train-fs", False, False, 1.0),
}
MPII_CASES = {"mpii_train": ("train", True), "mpii_valid": ("valid", False)}


def cfg(**ds):
    S = types.SimpleNamespace
    d = dict(NUM_CAMS=4, OCCLUSION=False, VOC="", TRI=False, Z_WEIGHT=1.0, MPII_ORDER=False, TEST_SET="valid",
             ROOT="")
    d.update(ds)
    return S(MODEL=S(IMAGE_SIZE=[64, 64]), DATASET=S(**d), DEBUG=S(DEBUG=False))


def seeded(s):
    np.random.seed(s)
    random.seed(s)


def build(name):
    """The mirror's dataset of case `name`, constructed after the generator's seeding."""
    import lib.dataset as dataset
    seeded(SEED % 1000)
    if name in H36M_CASES:
        image_set, is_train, tri, zw = H36M_CASES[name]
        return dataset.h36m(cfg(TRI=tri, Z_WEIGHT=zw), H36M_ROOT, image_set, is_train)
    image_set, is_train = MPII_CASES[name]
    return dataset.mpii_integral(cfg(ROOT=MPII_ROOT), MPII_ROOT, image_set, is_train)


def root_of(name):
    return H36M_ROOT if name in H36M_CASES else MPII_ROOT


def digest(patch):
    return hashlib.sha256(np.ascontiguousarray(patch, dtype=np.float32).tobytes()).hexdigest()


META_CAM = ("R", "T", "f", "c", "projection_matrix")


def meta_cam(m):
    return np.concatenate([np.ravel(np.asarray(m[k], dtype=np.float64)) for k in META_CAM])
