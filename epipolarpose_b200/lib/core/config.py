"""Global experiment configuration -- host-side mirror of the reference's
lib/core/config.py surface (module-global `config`, `update_config`,
`update_dir`, `gen_config`, `get_model_name`), re-implemented without easydict
(absent here) and with yaml.safe_load (reference :173 uses the removed
yaml.load(f) form).  Field names / defaults follow reference config.py:8-139 so
the six experiments/*.yaml files parse unchanged; unknown keys raise
ValueError exactly like reference :167,184.

Extra keys (superset, all default-off): TRAIN.ONLINE_TRIANGULATION,
TRAIN.TRIANGULATION_METHOD, TRAIN.ESTIMATE_EXTRINSICS (self-supervision without camera
extrinsics: each view pair's pose is estimated from its 2-D joints; needs
TRAIN.ONLINE_TRIANGULATION, ValueError otherwise), DATASET.TRI_VIEWS (views per DATASET.TRI training
item, default 2: the reference's pairs), TRAIN.TRIANGULATION_METHOD: robust (online labels from the
robust triangulation of every view of a tuple) with TRAIN.ROBUST_THRESHOLD_PX (default 15.0; see
tuple_settings for the combinations refused), TRAIN.CUDA_GRAPH (default on),
MODEL.PRECISION, DATASET.SYNTHETIC_LEN, TEST.PSS_K (list of k: the H36M evaluation appends
PSS@k, lib/core/pss.py; default []), TEST.PSS_CENTROIDS (.npz of `k<k>` centroids used instead
of fitting them on train-fs; default ''), TEST.REFINER (a refiner checkpoint: the H36M evaluation
also refines its poses and appends the Refined-* entries, lib/core/refine.py; default '') and
TEST.REFINER_NORM (the refiner's norm.pkl, required with TEST.REFINER).
"""
import os

import numpy as np
import yaml


class AttrDict(dict):
    """dict with attribute access; nested dicts are converted on assignment."""

    def __init__(self, d=None, **kw):
        super().__init__()
        for k, v in dict(d or {}, **kw).items():
            self[k] = v

    def __setitem__(self, k, v):
        if isinstance(v, dict) and not isinstance(v, AttrDict):
            v = AttrDict(v)
        super().__setitem__(k, v)

    def __setattr__(self, k, v):
        self[k] = v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)


_POSE_RESNET = dict(NUM_LAYERS=50, DECONV_WITH_BIAS=False, NUM_DECONV_LAYERS=3,
                    NUM_DECONV_FILTERS=[256, 256, 256], NUM_DECONV_KERNELS=[4, 4, 4],
                    FINAL_CONV_KERNEL=1, TARGET_TYPE='gaussian', HEATMAP_SIZE=[64, 64], SIGMA=2)

_DEFAULTS = dict(
    OUTPUT_DIR='', LOG_DIR='', DATA_DIR='', GPUS='0', WORKERS=8, PRINT_FREQ=20,
    EXP_NAME='default',
    CUDNN=dict(BENCHMARK=True, DETERMINISTIC=False, ENABLED=True),
    MODEL=dict(NAME='pose3d_resnet', INIT_WEIGHTS=True, PRETRAINED='', RESUME='', NUM_JOINTS=17,
               IMAGE_SIZE=[256, 256], DEPTH_RES=64, VOLUME=True, EXTRA=_POSE_RESNET,
               PRECISION='tf32x3'),
    LOSS=dict(USE_TARGET_WEIGHT=True, FN='L1JointLocationLoss', USE_SOFT=True, NORM=False,
              DEPTH_LAMBDA=1.),
    DATASET=dict(ROOT='', DATASET='mpii', TRAIN_SET='train', TEST_SET='valid', DATA_FORMAT='jpg',
                 HYBRID_JOINTS_TYPE='', SELECT_DATA=False, TRI=False, MPII_ORDER=False,
                 TRAIN_FRAME=32, VAL_FRAME=64, NUM_CAMS=4, DEPTH_RANGE=2000, FLIP=True,
                 SCALE_FACTOR=0.25, ROT_FACTOR=30, OCCLUSION=False, VOC='', BG_AUG=False,
                 Z_WEIGHT=1., SYNTHETIC_LEN=256, TRI_VIEWS=2),
    TRAIN=dict(LR_FACTOR=0.1, LR_STEP=[90, 110], LR=0.001, OPTIMIZER='adam', MOMENTUM=0.9,
               WD=0.0001, NESTEROV=False, GAMMA1=0.99, GAMMA2=0.0, BEGIN_EPOCH=0, END_EPOCH=140,
               RESUME=False, CHECKPOINT='', BATCH_SIZE=32, SHUFFLE=True,
               ONLINE_TRIANGULATION=False, TRIANGULATION_METHOD='iterative', ESTIMATE_EXTRINSICS=False,
               ROBUST_THRESHOLD_PX=15.0, CUDA_GRAPH=True),
    TEST=dict(BATCH_SIZE=32, FLIP_TEST=False, POST_PROCESS=True, SHIFT_HEATMAP=True,
              USE_GT_BBOX=False, OKS_THRE=0.5, IN_VIS_THRE=0.0, COCO_BBOX_FILE='', BBOX_THRE=1.0,
              MODEL_FILE='', IMAGE_THRE=0.0, NMS_THRE=1.0, PSS_K=[], PSS_CENTROIDS='',
              REFINER='', REFINER_NORM=''),
    DEBUG=dict(DEBUG=False, SAVE_BATCH_IMAGES_GT=False, SAVE_BATCH_IMAGES_PRED=False,
               SAVE_HEATMAPS_GT=False, SAVE_HEATMAPS_PRED=False, SAVE_3D=False),
)

config = AttrDict(_DEFAULTS)


def reset_config():
    """Restore defaults in place (the object identity of `config` is kept)."""
    config.clear()
    for k, v in AttrDict(_DEFAULTS).items():
        config[k] = v
    return config


def _as_pair(v):
    return np.array([v, v]) if isinstance(v, int) else np.array(v)


def _merge_section(name, values):
    section = config[name]
    if name == 'DATASET':
        for key in ('MEAN', 'STD'):
            if values.get(key):
                values[key] = np.array([eval(x) if isinstance(x, str) else x for x in values[key]])
    if name == 'MODEL':
        if 'EXTRA' in values and 'HEATMAP_SIZE' in values['EXTRA']:
            values['EXTRA']['HEATMAP_SIZE'] = _as_pair(values['EXTRA']['HEATMAP_SIZE'])
        if 'IMAGE_SIZE' in values:
            values['IMAGE_SIZE'] = _as_pair(values['IMAGE_SIZE'])
    for key, val in values.items():
        if key not in section:
            raise ValueError("{}.{} not exist in config.py".format(name, key))
        section[key] = val


def update_config(config_file):
    with open(config_file) as f:
        exp = yaml.safe_load(f) or {}
    for key, val in exp.items():
        if key not in config:
            raise ValueError("{} not exist in config.py".format(key))
        if isinstance(val, dict):
            _merge_section(key, val)
        else:
            config[key] = val
    check_config(config)


def check_config(cfg):
    """Combinations of keys that cannot be trained: ValueError."""
    train = cfg.get('TRAIN', {})
    if train.get('ESTIMATE_EXTRINSICS', False) and not train.get('ONLINE_TRIANGULATION', False):
        raise ValueError("TRAIN.ESTIMATE_EXTRINSICS needs TRAIN.ONLINE_TRIANGULATION: the estimated "
                         "camera geometry only feeds the online epipolar labels")
    tuple_settings(cfg)


def tuple_settings(cfg):
    """(views, method, threshold_px) of online self-supervised training: DATASET.TRI_VIEWS, and
    TRAIN.TRIANGULATION_METHOD / TRAIN.ROBUST_THRESHOLD_PX when TRAIN.ONLINE_TRIANGULATION is set
    (method None otherwise).  ValueError for TRI_VIEWS outside 2..min(NUM_CAMS, 8), more than two
    views with online labels from any method but 'robust' (the pair triangulators take two views),
    'robust' with TRAIN.ESTIMATE_EXTRINSICS (the relative pose is estimated per view pair), and a
    threshold that is not a positive number of pixels.  Missing keys take their defaults."""
    ds, train = getattr(cfg, 'DATASET', None), getattr(cfg, 'TRAIN', None)
    views = int(getattr(ds, 'TRI_VIEWS', 2))
    cams = int(getattr(ds, 'NUM_CAMS', 4))
    if not (views == 2 or 2 < views <= min(cams, 8)):       # 2: the reference's pairs, any NUM_CAMS
        raise ValueError("DATASET.TRI_VIEWS must be in 2..min(NUM_CAMS, 8) = 2..%d, got %d" % (min(cams, 8), views))
    online = bool(getattr(train, 'ONLINE_TRIANGULATION', False))
    method = getattr(train, 'TRIANGULATION_METHOD', 'iterative') if online else None
    thr = float(getattr(train, 'ROBUST_THRESHOLD_PX', 15.0))
    if online and views > 2 and method != 'robust':
        raise ValueError("DATASET.TRI_VIEWS = %d with TRAIN.ONLINE_TRIANGULATION needs TRAIN.TRIANGULATION_METHOD: "
                         "robust; the pair triangulators (%r) take two views" % (views, method))
    if method == 'robust' and bool(getattr(train, 'ESTIMATE_EXTRINSICS', False)):
        raise ValueError("TRAIN.TRIANGULATION_METHOD: robust needs calibrated cameras; TRAIN.ESTIMATE_EXTRINSICS "
                         "estimates the relative pose of view pairs only")
    if method == 'robust' and not (np.isfinite(thr) and thr > 0):
        raise ValueError("TRAIN.ROBUST_THRESHOLD_PX must be a positive number of pixels, got %r" % (thr,))
    return views, method, thr


def gen_config(config_file):
    def plain(v):
        if isinstance(v, dict):
            return {k: plain(x) for k, x in v.items()}
        if isinstance(v, np.ndarray):
            return v.tolist()
        return v
    with open(config_file, 'w') as f:
        yaml.dump(plain(config), f, default_flow_style=False)


def update_dir(model_dir, log_dir, data_dir):
    if model_dir:
        config.OUTPUT_DIR = model_dir
    if log_dir:
        config.LOG_DIR = log_dir
    if data_dir:
        config.DATA_DIR = data_dir
    config.DATASET.ROOT = os.path.join(config.DATA_DIR, config.DATASET.ROOT)
    config.TEST.COCO_BBOX_FILE = os.path.join(config.DATA_DIR, config.TEST.COCO_BBOX_FILE)
    config.MODEL.PRETRAINED = os.path.join(config.DATA_DIR, config.MODEL.PRETRAINED)


def get_model_name(cfg):
    """(name, full_name) as reference config.py:211-249."""
    extra = cfg.MODEL.EXTRA
    base = cfg.MODEL.NAME
    h, w = cfg.MODEL.IMAGE_SIZE[1], cfg.MODEL.IMAGE_SIZE[0]
    name = '{}_{}'.format(base, extra.NUM_LAYERS)
    if base == 'pose_resnet':
        suffix = ''.join('d{}'.format(n) for n in extra.NUM_DECONV_FILTERS)
    elif base == 'pose3d_resnet':
        suffix = 'DR%s_S%s_DL%s' % (cfg.MODEL.DEPTH_RES, int(cfg.LOSS.USE_SOFT),
                                    int(cfg.LOSS.DEPTH_LAMBDA))
    else:
        raise ValueError('Unkown model: {}'.format(cfg.MODEL))
    full_name = '{}x{}_{}_{}'.format(h, w, name, suffix)
    print(name, full_name)
    return name, full_name


if __name__ == '__main__':
    import sys
    gen_config(sys.argv[1])
