"""float64 numpy restatement of the Pose Structure Score definition (lib/core/pss.py docstring,
DESIGN.md section 3): pose normalisation, the splitmix64 draws, k-means++ with the two-level
prefix, Lloyd with the two-level update order and the empty-cluster rule, the inertia.  Every
floating-point operation is the one the kernels of csrc/pss.cu perform, in the same order, so
results compare bit for bit.  Shared by tests/test_pss_host.py and tests/test_gpu_pss.py;
tests/emul_pss.py runs it as the CPU emulation of the C ABI."""
import numpy as np

CHUNK = 1024
_M64 = (1 << 64) - 1


def uniform(seed, restart, j):
    """Draw j (0-based) of splitmix64 seeded by (seed, restart): the top 53 bits in [0, 1)."""
    z = ((seed ^ ((restart * 0xD1B54A32D192ED03) & _M64)) + (j + 1) * 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    z ^= z >> 31
    return float(z >> 11) * 2.0 ** -53


def back_project(pose, cam):
    """CamBackProj of every joint: pose [S,J,3] (x px, y px, root-relative depth mm), cam [S,5]."""
    d = pose[:, :, 2] + cam[:, 4:5]
    return np.stack([(pose[:, :, 0] - cam[:, 2:3]) / cam[:, 0:1] * d,
                     (pose[:, :, 1] - cam[:, 3:4]) / cam[:, 1:2] * d, d], axis=2)


def normalize(pose, cam, root):
    """[S, 3J]: back-projected, root-relative, divided by the Frobenius norm (zero stays zero)."""
    b = back_project(np.asarray(pose, np.float64), np.asarray(cam, np.float64))
    v = (b - b[:, root:root + 1, :]).reshape(len(b), -1)
    ss = np.zeros(len(v))
    for t in range(v.shape[1]):
        ss = ss + v[:, t] * v[:, t]
    n = np.sqrt(ss)
    out = v.copy()
    nz = n > 0
    out[nz] = v[nz] / n[nz, None]
    return out


def sqdist(x, c, block=4096):
    """[N, k]: sum_t (x_t - c_t)^2 in coordinate order, no fused multiply-add."""
    out = np.empty((len(x), len(c)))
    for i0 in range(0, len(x), block):
        xb = x[i0:i0 + block]
        s = np.zeros((len(xb), len(c)))
        for t in range(x.shape[1]):
            e = xb[:, t, None] - c[None, :, t]
            s = s + e * e
        out[i0:i0 + block] = s
    return out


def assign(x, c):
    """labels (lowest centre on ties) and squared distances."""
    s = sqdist(x, c)
    lab = np.argmin(s, axis=1)
    return lab.astype(np.int32), s[np.arange(len(x)), lab]


def chunk_prefix(v):
    """[nchunks, CHUNK] inclusive prefix of v within each chunk of CHUNK points (index order)."""
    nch = (len(v) + CHUNK - 1) // CHUNK
    pad = np.zeros(nch * CHUNK)
    pad[:len(v)] = v
    return np.cumsum(pad.reshape(nch, CHUNK), axis=1)


def two_level_sum(v):
    s = 0.0
    for t in chunk_prefix(v)[:, -1]:
        s += t
    return s


def kmeanspp(x, k, seed, restart):
    N = len(x)
    idx = [min(int(uniform(seed, restart, 0) * N), N - 1)]
    D2 = None
    for j in range(1, k):
        s = sqdist(x, x[idx[-1]][None])[:, 0]
        D2 = s if D2 is None else np.where(s < D2, s, D2)
        pre = chunk_prefix(D2)
        total = 0.0
        for t in pre[:, -1]:
            total += t
        if total == 0.0:
            raise ValueError("fewer than k = %d distinct points" % k)
        target = uniform(seed, restart, j) * total
        base, pick = 0.0, N - 1
        for c in range(len(pre)):
            nxt = base + pre[c, -1]
            if nxt > target:
                pick = c * CHUNK + int(np.argmax(base + pre[c] > target))
                break
            base = nxt
        idx.append(pick)
    return np.array(idx, dtype=np.int32)


def update(x, labels, dist2, cen):
    """Member means (chunk partials in point order, combined in chunk order); empty clusters, in
    cluster order, take the points farthest from their centres (lowest index on ties)."""
    N, d = x.shape
    k = len(cen)
    S = np.zeros((k, d))
    for c0 in range(0, N, CHUNK):
        part = np.zeros((k, d))
        np.add.at(part, labels[c0:c0 + CHUNK], x[c0:c0 + CHUNK])
        S = S + part
    cnt = np.bincount(labels, minlength=k)
    new = cen.copy()
    nz = cnt > 0
    new[nz] = S[nz] / cnt[nz, None].astype(np.float64)
    empty = np.flatnonzero(cnt == 0)
    if len(empty):
        order = np.lexsort((np.arange(N), -dist2))
        for e, j in enumerate(empty):
            new[j] = x[order[e]]
    return new


def check(x, k):
    x = np.asarray(x, np.float64)
    if k < 1 or k > len(x):
        raise ValueError("k = %d outside [1, N = %d]" % (k, len(x)))
    if not np.isfinite(x).all():
        raise ValueError("non-finite input")
    return x


def fit_restart(x, k, seed, restart, max_iter):
    """One restart: dict(init_idx, trace (labels of every pass), centroids, labels, inertia, n_iter,
    relocated = empty clusters refilled over all updates)."""
    x = check(x, k)
    idx = kmeanspp(x, k, seed, restart)
    cen = x[idx].copy()
    labels, dist2 = assign(x, cen)
    trace = [labels]
    it = relocated = 0
    while it < max_iter:
        relocated += int(np.count_nonzero(np.bincount(labels, minlength=k) == 0))
        cen = update(x, labels, dist2, cen)
        new, dist2 = assign(x, cen)
        it += 1
        trace.append(new)
        changed = bool(np.any(new != labels))
        labels = new
        if not changed:
            break
    return dict(init_idx=idx, trace=np.stack(trace), centroids=cen, labels=labels,
                inertia=two_level_sum(dist2), n_iter=it, relocated=relocated)


def fit(x, k, seed=0, n_init=10, max_iter=300):
    best = None
    for r in range(n_init):
        f = fit_restart(x, k, seed, r, max_iter)
        if best is None or f["inertia"] < best["inertia"]:
            best = f
    return best["centroids"]


def pss(pred, gt, cen):
    return np.count_nonzero(assign(pred, cen)[0] == assign(gt, cen)[0]) / len(pred)


def relocation_case():
    """A fit that empties a cluster: with seed 453, k-means++ picks y = 1.0, -4.0, 2.2 (indices
    2, 12, 0); after the first update the cluster of y = 1.0 (members 1.0, -1.0, mean 0) loses
    y = 1.0 to the centre 1.925 and y = -1.0 to the centre -1.87, so the second update refills it.
    Returns (x [13, 2], k, seed)."""
    y = np.array([2.2, 1.65, 1.0, -1.0] + list(np.linspace(-1.52, -1.7, 8)) + [-4.0])
    return np.stack([y, np.zeros_like(y)], 1), 3, 453


def fixture_pss(valid, preds, mpii_order, ks, centroids=None):
    """PSS@k of H36M_Integral.evaluate on the fixture tree (tests/golden/datasets/h36m), restated:
    `valid` = the dataset's db records, clusters fitted on train-fs (list form) unless given."""
    import os
    from lib.dataset.JointIntegralDataset import load_pickle
    from oracle import restate
    from tests.dataset_cases import H36M_ROOT
    perm = restate.H36M_TO_MPII_PERM if mpii_order else np.arange(17)
    root = 6 if mpii_order else 0

    def poses(recs, joints=None):
        j = np.stack([r["joints_3d"] for r in recs])[:, perm] if joints is None else joints
        cam = np.stack([np.concatenate([r["fl"][:2], r["c_p"][:2], r["pelvis"][2:3]]) for r in recs])
        return normalize(np.asarray(j, np.float64)[:, :, :3], cam, root)
    valid = valid[:len(preds)]
    P, G = poses(valid, np.asarray(preds)[:, :, :3]), poses(valid)
    train = list(load_pickle(os.path.join(H36M_ROOT, "annot", "train-fs.pkl")))
    out = []
    for k in ks:
        c = centroids[k] if centroids is not None else fit(poses(train), k)
        out.append(("PSS@%d" % k, pss(P, G, c)))
    return out


def skeleton_poses(rng, N, J, k_true=8, spread=0.02):
    """Normalised skeleton-like poses: k_true random base skeletons (bones of 100-450 mm on a
    kinematic chain) plus per-sample jitter, root-relative, unit Frobenius norm; [N, 3J]."""
    parents = [0, 0, 1, 2, 0, 4, 5, 0, 7, 8, 9, 8, 11, 12, 8, 14, 15] + list(range(16, 32))
    base = np.zeros((k_true, J, 3))
    for j in range(1, J):
        dirs = rng.normal(size=(k_true, 3))
        dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
        base[:, j] = base[:, parents[j]] + dirs * rng.uniform(100, 450, (k_true, 1))
    p = base[rng.integers(0, k_true, N)] + rng.normal(0, spread * 1000, (N, J, 3))
    p = (p - p[:, :1]).reshape(N, -1)
    return p / np.linalg.norm(p, axis=1, keepdims=True)
