"""Writes the dataset fixture tree tests/golden/datasets/ and tests/golden/datasets.npz: what the
UNMODIFIED reference dataset classes (lib/dataset/h36m.py, lib/dataset/mpii_integral.py) make
of that tree for fixed np.random / random seeds.  Build container only:
    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_datasets.py

Tree (in the reference's file formats):
  h36m/images/*.jpg              12 frames: 3 poses x 4 cameras on a ring (the geometry of
                                 lib/dataset/synthetic.py, intrinsics scaled to 128x128 frames)
  h36m/annot/train-fs.pkl        list form, records hold reference lib.utils.cameras.Camera
  h36m/annot/{train-ss,valid}.pkl  dict form {1..4: per-camera lists}
  mpii/images/*.jpg, mpii/annot/{train,valid}.json, mpii/annot/gt_valid.mat
Frames are cv2 JPEGs: 4:2:0 q90, one 4:4:4 and one progressive (decoded by cv2 on the host).

npz keys, per case <c>: <c>/db_length, <c>/db_image, <c>/db_box [N,4], <c>/db_joints, <c>/db_vis
(db order); per item (item idx drawn after seeding both generators with 1000 + idx):
<c>/sha256 (of the float32 patch, C order), <c>/label, <c>/weight, <c>/image, and for h36m
<c>/scale_rot, <c>/meta_box [N,4], <c>/meta_cam [N,28] (R T f c P); TRI cases key the two views
<c>/cam_1/..., <c>/cam_2/....  Evaluation: h36m_eval_<order>/preds, /names, /values, /perf,
/actions [15,2] (MPJPE, aligned); mpii_eval/preds, /names, /values, /perf, /pred_mat.
Patches are 64x64: their digests pin them bit for bit."""
import contextlib
import copy
import hashlib
import importlib
import io
import json
import os
import pickle
import random
import sys
import tempfile
import types

import cv2
import numpy as np
from scipy.io import loadmat, savemat

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
from oracle import refshim  # noqa: E402

TREE = os.path.join(HERE, "datasets")
H36M_FLIP = [[1, 4], [2, 5], [3, 6], [14, 11], [15, 12], [16, 13]]
PARENTS = np.array([0, 0, 1, 2, 0, 4, 5, 0, 8, 8, 9, 8, 11, 12, 8, 14, 15])
ACTIONS = ["Directions", "Eating", "Walking"]
MPII_JOINTS = ['rank', 'rkne', 'rhip', 'lhip', 'lkne', 'lank', 'pelv', 'thrx', 'neck', 'head',
               'rwri', 'relb', 'rsho', 'lsho', 'lelb', 'lwri']
SEED = 20261016


def frame(rng, H, W):
    """A smooth, natural-looking BGR frame (gradients, edges, mild noise)."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    ch = []
    for _ in range(3):
        f = rng.uniform(0.01, 0.06, 2)
        ch.append(128 + 60 * np.sin(x * f[0] + rng.uniform(0, 6)) * np.cos(y * f[1] + rng.uniform(0, 6)))
    img = np.stack(ch, axis=2)
    for _ in range(4):
        cx, cy, r = rng.uniform(0, W), rng.uniform(0, H), rng.uniform(4, min(H, W) / 4)
        img[(x - cx) ** 2 + (y - cy) ** 2 < r * r] = rng.uniform(0, 255, 3)
    img += rng.normal(0, 1.0, img.shape)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def write_jpeg(path, img, kind):
    p = [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
         cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444 if kind == "444" else cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
    if kind == "progressive":
        p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, buf = cv2.imencode(".jpg", img, p)
    assert ok
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "wb") as f:
        f.write(buf.tobytes())


def ring_camera(rng, view, f, c):
    az = np.deg2rad(45.0 + 90.0 * view + rng.uniform(-10, 10))
    r = 4500.0 + rng.uniform(-500, 500)
    h = 1500.0 + rng.uniform(-200, 200)
    C = np.array([r * np.cos(az), r * np.sin(az), h])
    zc = -C / np.linalg.norm(C)
    xc = np.cross(zc, np.array([0.0, 0.0, 1.0]))
    xc /= np.linalg.norm(xc)
    yc = np.cross(zc, xc)
    return np.stack([xc, yc, zc], axis=0), C.reshape(3, 1)


def make_h36m(ref_cameras, rng):
    """3 poses x 4 cameras; records in the db layout reference h36m.py reads."""
    f, c = np.array([146.5, 146.4]), np.array([64.0, 64.5])
    recs = {v: [] for v in range(4)}
    n = 0
    for t in range(3):
        X = rng.normal(0.0, 300.0, size=(17, 3)) + np.array([0.0, 0.0, 900.0])
        for v in range(4):
            R, T = ring_camera(rng, v, f, c)
            cam = ref_cameras.Camera((R, T, f.copy(), c.copy(), np.zeros((3, 1)), np.zeros((2, 1)), "cam%d" % v))
            Xc = (R @ (X.T - T)).T
            j3d = np.stack([Xc[:, 0] / Xc[:, 2] * f[0] + c[0], Xc[:, 1] / Xc[:, 2] * f[1] + c[1],
                            Xc[:, 2] - Xc[0, 2]], axis=1)
            vis = np.ones((17, 3))
            if (t + v) % 5 == 0:
                vis[(t + 2 * v) % 17] = 0.0
            lo, hi = j3d[:, :2].min(0), j3d[:, :2].max(0)
            size = float(max(hi - lo) * 1.3 + 8)
            kind = "progressive" if n == 5 else ("444" if n == 9 else "420")
            name = "images/s%02d_t%d_c%d.jpg" % (1 + t % 2, t, v + 1)
            write_jpeg(os.path.join(TREE, "h36m", name), frame(rng, 128, 128), kind)
            recs[v].append(dict(image=name, joints_3d=j3d, joints_3d_vis=vis, pelvis=Xc[0].copy(),
                                fl=f.copy(), c_p=c.copy(), cam=cam, center_x=float((lo[0] + hi[0]) / 2),
                                center_y=float((lo[1] + hi[1]) / 2), width=size, height=size,
                                flip_pairs=H36M_FLIP, parent_ids=PARENTS.copy(), subject=1 + t % 2,
                                action=ACTIONS[t], tuple=t, view=v))
            n += 1
    annot = os.path.join(TREE, "h36m", "annot")
    os.makedirs(annot, exist_ok=True)
    flat = [r for t in range(3) for r in (recs[0][t], recs[1][t], recs[2][t], recs[3][t])]
    with open(os.path.join(annot, "train-fs.pkl"), "wb") as fh:
        pickle.dump(flat, fh)
    with open(os.path.join(annot, "train-ss.pkl"), "wb") as fh:
        pickle.dump({v + 1: recs[v] for v in range(4)}, fh)
    with open(os.path.join(annot, "valid.pkl"), "wb") as fh:
        pickle.dump({v + 1: copy.deepcopy(recs[v]) for v in range(4)}, fh)


def make_mpii(rng):
    """6 frames; one annotation with a single visible joint (skipped by the db)."""
    out = {"train": [], "valid": []}
    pos, miss, heads = [], [], []
    for i in range(7):
        H, W = 120, 160
        name = "%03d.jpg" % i
        if i < 6:
            write_jpeg(os.path.join(TREE, "mpii", "images", name), frame(rng, H, W), "420" if i != 2 else "444")
        jts = np.stack([rng.uniform(30, 130, 16), rng.uniform(20, 100, 16)], axis=1)
        vis = (rng.uniform(size=16) > 0.15).astype(np.float64)
        vis[9] = 1.0
        if i == 6:
            vis[:] = 0.0
            vis[3] = 1.0
            name = "005.jpg"
        a = dict(image=name, joints=(jts + 1).tolist(), joints_vis=vis.tolist(),
                 center=[80.0, 60.0], scale=1.0)
        out["train" if i % 2 == 0 or i == 6 else "valid"].append(a)
        if i % 2 == 1:
            pos.append(jts + 1)
            miss.append(1 - vis)
            hx, hy = jts[9]
            heads.append([[hx - 9, hy - 11], [hx + 9, hy + 11]])
    annot = os.path.join(TREE, "mpii", "annot")
    os.makedirs(annot, exist_ok=True)
    for k, v in out.items():
        with open(os.path.join(annot, k + ".json"), "w") as fh:
            json.dump(v, fh)
    names = np.empty((1, 16), dtype=object)
    for j, n in enumerate(MPII_JOINTS):
        names[0, j] = n
    savemat(os.path.join(annot, "gt_valid.mat"), mdict={
        "dataset_joints": names, "jnt_missing": np.stack(miss, axis=1).astype(np.uint8),
        "pos_gt_src": np.stack(pos, axis=2), "headboxes_src": np.transpose(np.array(heads), [1, 2, 0])})


def cfg(**ds):
    S = types.SimpleNamespace
    d = dict(NUM_CAMS=4, OCCLUSION=False, VOC="", TRI=False, Z_WEIGHT=1.0, MPII_ORDER=False, TEST_SET="valid",
             ROOT="")
    d.update(ds)
    return S(MODEL=S(IMAGE_SIZE=[64, 64]), DATASET=S(**d), DEBUG=S(DEBUG=False))


def seeded(s):
    np.random.seed(s)
    random.seed(s)


def record_items(rec, key, items, root):
    imgs = [it[0] for it in items]
    rec[key + "/sha256"] = np.array([hashlib.sha256(np.ascontiguousarray(p).tobytes()).hexdigest() for p in imgs])
    rec[key + "/label"] = np.stack([it[1] for it in items])
    rec[key + "/weight"] = np.stack([it[2] for it in items])
    metas = [it[3] for it in items]
    rec[key + "/image"] = np.array([os.path.relpath(m["image"], root) for m in metas])
    if "center_x" in metas[0]:
        rec[key + "/meta_box"] = np.array([[m[k] for k in ("center_x", "center_y", "width", "height")]
                                           for m in metas], dtype=np.float64)
        rec[key + "/scale_rot"] = np.array([[m["scale"], m["rot"]] for m in metas], dtype=np.float64)
        rec[key + "/meta_cam"] = np.array([np.concatenate([np.ravel(m[k]) for k in ("R", "T", "f", "c",
                                                                                     "projection_matrix")])
                                           for m in metas])


def db_arrays(rec, key, db, root):
    flat = [r for d in db for r in d] if isinstance(db[0], list) else db
    rec[key + "/db_image"] = np.array([os.path.relpath(os.path.join(root, r["image"]), root) for r in flat])
    rec[key + "/db_box"] = np.array([[r[k] for k in ("center_x", "center_y", "width", "height")] for r in flat],
                                    dtype=np.float64)
    rec[key + "/db_joints"] = np.stack([r["joints_3d"] for r in flat])
    rec[key + "/db_vis"] = np.stack([r["joints_3d_vis"] for r in flat])


H36M_CASES = {          # name: (image_set, is_train, TRI, Z_WEIGHT)
    "h36m_fs_train": ("train-fs", True, False, 1.0),
    "h36m_ss_train": ("train-ss", True, False, 0.5),
    "h36m_ss_tri": ("train-ss", True, True, 1.0),
    "h36m_valid": ("valid", False, False, 1.0),
    "h36m_fs_valid": ("train-fs", False, False, 1.0),
}
MPII_CASES = {"mpii_train": ("train", True), "mpii_valid": ("valid", False)}


def main():
    ref = refshim.ref()
    h36m = importlib.import_module("lib.dataset.h36m")
    mpii = importlib.import_module("lib.dataset.mpii_integral")
    if os.path.isdir(TREE):
        import shutil
        shutil.rmtree(TREE)
    rng = np.random.default_rng(SEED)
    make_h36m(ref.cameras, rng)
    make_mpii(rng)
    rec = {}
    hroot = os.path.join(TREE, "h36m")
    for k, (image_set, is_train, tri, zw) in H36M_CASES.items():
        seeded(SEED % 1000)
        ds = h36m.H36M_Integral(cfg(TRI=tri, Z_WEIGHT=zw), hroot, image_set, is_train)
        rec[k + "/db_length"] = np.array(len(ds))
        db_arrays(rec, k, ds.db, hroot)
        items = []
        for idx in range(len(ds)):
            seeded(1000 + idx)
            items.append(ds[idx])
        if tri:
            record_items(rec, k + "/cam_1", [it["cam_1"] for it in items], hroot)
            record_items(rec, k + "/cam_2", [it["cam_2"] for it in items], hroot)
        else:
            record_items(rec, k, items, hroot)
    mroot = os.path.join(TREE, "mpii")
    for k, (image_set, is_train) in MPII_CASES.items():
        seeded(SEED % 1000)
        ds = mpii.MPIIDataset(cfg(ROOT=mroot), mroot, image_set, is_train)
        rec[k + "/db_length"] = np.array(len(ds))
        db_arrays(rec, k, ds.db, mroot)
        items = []
        for idx in range(len(ds)):
            seeded(1000 + idx)
            items.append(ds[idx])
        record_items(rec, k, items, mroot)
    # evaluation on fabricated predictions
    prng = np.random.default_rng(SEED + 1)
    for order in (False, True):
        seeded(SEED % 1000)
        ds = h36m.H36M_Integral(cfg(MPII_ORDER=order), hroot, "valid", False)
        gt = np.stack([r["joints_3d"] for r in ds.db])
        if order:
            gt = gt[:, h36m.H36M_TO_MPII_PERM]
        preds = gt + prng.normal(0, [3.0, 3.0, 40.0], gt.shape)
        preds = np.concatenate([preds, np.ones(preds.shape[:2] + (1,))], axis=2)
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            nv, perf = ds.evaluate(preds.copy(), None, actionwise=True)
        lines = buf.getvalue().splitlines()
        acts = ref_actions(lines)
        tag = "h36m_eval_" + ("mpii" if order else "h36m")
        rec[tag + "/preds"] = preds
        rec[tag + "/names"] = np.array([n for n, _ in nv])
        rec[tag + "/values"] = np.array([v for _, v in nv], dtype=np.float64)
        rec[tag + "/perf"] = np.array(perf)
        rec[tag + "/actions"] = acts
    ds = mpii.MPIIDataset(cfg(ROOT=mroot), mroot, "valid", False)
    gt = np.stack([r["joints_3d"][:, :2] for r in ds.db])
    preds = gt + prng.normal(0, 4.0, gt.shape)
    preds = np.concatenate([preds, np.zeros(preds.shape[:2] + (1,))], axis=2)
    with tempfile.TemporaryDirectory() as tmp:
        nv, perf = ds.evaluate(preds.copy(), tmp)
        rec["mpii_eval/pred_mat"] = loadmat(os.path.join(tmp, "pred.mat"))["preds"]
    rec["mpii_eval/preds"] = preds
    rec["mpii_eval/names"] = np.array([n for n, _ in nv])
    rec["mpii_eval/values"] = np.array([float(v) for _, v in nv], dtype=np.float64)
    rec["mpii_eval/perf"] = np.array(float(perf))
    np.savez_compressed(os.path.join(HERE, "datasets.npz"), cv2_version=np.array(cv2.__version__), **rec)
    size = sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(TREE) for f in fs)
    print("tree %d bytes, datasets.npz %d bytes" % (size, os.path.getsize(os.path.join(HERE, "datasets.npz"))))


def ref_actions(lines):
    """The two per-action blocks the reference prints with actionwise=True -> [15, 2]."""
    from collections import OrderedDict
    blocks, cur = [], None
    for ln in lines:
        if ln.startswith("====="):
            if cur is None:
                cur = OrderedDict()
            else:
                blocks.append(cur)
                cur = None
        elif cur is not None:
            k, v = ln.rsplit(" ", 1)
            cur[k] = float(v)
    assert len(blocks) == 2 and len(blocks[0]) == 15
    return np.array([[blocks[0][k], blocks[1][k]] for k in blocks[0]], dtype=np.float64)


if __name__ == "__main__":
    main()
