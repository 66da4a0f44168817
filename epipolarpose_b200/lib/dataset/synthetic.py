"""Synthetic multi-view dataset with the reference Dataset contract
(lib/dataset/h36m.py:73-88): __getitem__ -> (img f32 [3,256,256], label f32
[J*3], weight f32 [J*3], meta) with meta keys image, center_x, center_y, width,
height, scale, rot, R, T, f, c, projection_matrix; `.db`, `.evaluate`, `len`.
Selected by yaml `DATASET.DATASET: synthetic_h36m` through the name-based
registry scripts/train.py:125 uses.  H36M / MPII image data is not available
offline; frames are seeded noise, cameras follow SURVEY.md section 8(d): four
cameras per view-tuple on a ring r = 4.5 m +- 0.5 at azimuths
{45,135,225,315} +- 10 deg, height 1.5 m +- 0.2, f = (1145,1144), c = (512,515),
P = K.[R | -R.T].

Sample order: index = tuple*NUM_CAMS + view.  `pair_batch_sampler` lays a
batch out as [views 0 and 3 of each tuple | views 1 and 2] so that the
first-half/second-half pairing of reference img_utils.py:194-199 triangulates
(0,1) and (3,2), both legal neighbours in reference h36m.py:25.  `tuple_batch_sampler` lays
out whole tuples view-major (row v*T + t is view v of tuple t), the layout of the robust online
labels.

`flip_pairs` (read by the flip test of validate_integral): the MPII pairs for 16 joints, the
H36M-17 pairs for 17 (reference prep_h36m.py:71,68), none for any other joint count."""
import numpy as np
import torch
from torch.utils.data import Dataset


MPII_FLIP_PAIRS = [[0, 5], [1, 4], [2, 3], [10, 15], [11, 14], [12, 13]]
H36M_FLIP_PAIRS = [[1, 4], [2, 5], [3, 6], [14, 11], [15, 12], [16, 13]]


def ring_camera(rng, view):
    az = np.deg2rad(45.0 + 90.0 * view + rng.uniform(-10, 10))
    r = 4500.0 + rng.uniform(-500, 500)
    h = 1500.0 + rng.uniform(-200, 200)
    C = np.array([r * np.cos(az), r * np.sin(az), h])
    zc = -C / np.linalg.norm(C)
    xc = np.cross(zc, np.array([0.0, 0.0, 1.0]))
    xc /= np.linalg.norm(xc)
    yc = np.cross(zc, xc)
    R = np.stack([xc, yc, zc], axis=0)
    f = np.array([1145.0, 1144.0])
    c = np.array([512.0, 515.0])
    K = np.array([[f[0], 0., c[0]], [0., f[1], c[1]], [0., 0., 1.]])
    P = K @ np.concatenate([R, R @ (-C.reshape(3, 1))], axis=1)
    return R, C.reshape(3, 1), f, c, P


class SyntheticH36M(Dataset):
    def __init__(self, cfg, root=None, image_set='train', is_train=True, rank=0):
        self.cfg = cfg
        self.is_train = is_train
        self.num_joints = cfg.MODEL.NUM_JOINTS
        self.num_cams = int(getattr(cfg.DATASET, 'NUM_CAMS', 4))
        self.flip_pairs = {16: MPII_FLIP_PAIRS, 17: H36M_FLIP_PAIRS}.get(self.num_joints, [])
        self.patch_width, self.patch_height = int(cfg.MODEL.IMAGE_SIZE[0]), int(cfg.MODEL.IMAGE_SIZE[1])
        n_tuples = max(1, int(getattr(cfg.DATASET, 'SYNTHETIC_LEN', 256)) // self.num_cams)
        self.seed = 1000 * rank + (0 if is_train else 7)
        rng = np.random.default_rng(self.seed)
        self.db = []
        for t in range(n_tuples):
            X = rng.normal(0.0, 400.0, size=(self.num_joints, 3))     # world mm
            for v in range(self.num_cams):
                R, T, f, c, P = ring_camera(rng, v)
                # ground truth in the db layout of reference h36m.py (:204-216): image-space
                # joints with root-relative depth, pelvis in camera space, focal / centre
                Xc = (R @ (X.T - T)).T
                j3d = np.stack([Xc[:, 0] / Xc[:, 2] * f[0] + c[0], Xc[:, 1] / Xc[:, 2] * f[1] + c[1],
                                Xc[:, 2] - Xc[0, 2]], axis=1)
                self.db.append(dict(
                    joints_3d=j3d, joints_3d_vis=np.ones_like(j3d), pelvis=Xc[0].copy(), fl=f, c_p=c,
                    image='synthetic_%06d_%d' % (t, v), tuple=t, view=v,
                    center_x=float(500 + rng.uniform(-50, 50)),
                    center_y=float(500 + rng.uniform(-50, 50)),
                    width=float(800 + rng.uniform(-100, 100)),
                    height=float(800 + rng.uniform(-100, 100)),
                    R=R, T=T, f=f, c=c, projection_matrix=P, joints_world=X))

    def __len__(self):
        return len(self.db)

    def __getitem__(self, idx):
        d = self.db[idx]
        g = torch.Generator().manual_seed(self.seed * 100003 + idx)
        img = torch.randn(3, self.patch_height, self.patch_width, generator=g)
        label = torch.rand(self.num_joints * 3, generator=g) - 0.5
        weight = torch.ones(self.num_joints * 3)
        meta = {k: d[k] for k in ('image', 'center_x', 'center_y', 'width', 'height', 'R', 'T',
                                  'f', 'c', 'projection_matrix')}
        meta['scale'] = 1.0
        meta['rot'] = 0.0
        return img, label, weight, meta

    def pair_batch_sampler(self, tuples_per_batch):
        """Index batches whose halves pair views (0,1) and (3,2) of each tuple."""
        assert self.num_cams == 4
        n_tuples = len(self.db) // 4
        for b in range(0, n_tuples - tuples_per_batch + 1, tuples_per_batch):
            ts = range(b, b + tuples_per_batch)
            yield [t * 4 + 0 for t in ts] + [t * 4 + 3 for t in ts] + \
                  [t * 4 + 1 for t in ts] + [t * 4 + 2 for t in ts]

    def tuple_batch_sampler(self, tuples_per_batch, views=None):
        """Index batches of whole view tuples in the view-major layout of online triangulation
        with TRAIN.TRIANGULATION_METHOD robust: row v*T + t is view v of tuple t (T =
        tuples_per_batch, views 0..views-1 of each tuple, default all NUM_CAMS)."""
        V = self.num_cams if views is None else int(views)
        if not 2 <= V <= self.num_cams:
            raise ValueError("views must be in 2..%d, got %d" % (self.num_cams, V))
        n_tuples = len(self.db) // self.num_cams
        for b in range(0, n_tuples - tuples_per_batch + 1, tuples_per_batch):
            yield [t * self.num_cams + v for v in range(V) for t in range(b, b + tuples_per_batch)]

    def evaluate(self, preds, save_path=None, debug=False):
        """H36M protocol (reference lib/dataset/h36m.py:168-378) of the predictions against the
        synthetic ground truth, on the device (lib/dataset/h36m_eval.py).  The images are noise,
        so the numbers only exercise the metric code; joints keep the db order (root = joint 0)."""
        from .h36m_eval import evaluate_h36m
        n = min(len(preds), len(self.db))
        get = lambda k: np.stack([np.asarray(self.db[i][k], dtype=np.float64) for i in range(n)]) \
            if n else np.zeros((0, 3))
        name_value, perf, _ = evaluate_h36m(np.asarray(preds)[:n], get('joints_3d'), get('pelvis'),
                                            get('fl'), get('c_p'), mpii_order=False)
        return name_value, perf
