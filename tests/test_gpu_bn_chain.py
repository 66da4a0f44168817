"""The split-fp16 BatchNorm chain against float64 at the bench's sizes: the statistics the conv16
epilogue sums (tc::stats_add / stats_flush), bn_finalize_scale, the post-activation producers
bn_act_split / bn_relu_maxpool_split, bn_bwd_split and softargmax_bwd_split.  Every reference is
torch float64 on the device, computed from the exact fp32 values the kernels read or wrote (the
kernel's own z, the joined planes), so each bar is the kernel's rounding and nothing else.

Bars (u = 2^-24, one fp32 rounding):

  * Statistics.  A value passes through at most d = 13 + T fp32 roundings before its CTA's partial
    becomes a double: 4 (5 with the square) in the 16-row shuffle tree, one per tile the CTA ran
    for its N tile (T, from the tile schedule, `_stats_depth`), 8 in the warp-order flush.  So per
    channel |dS1| <= d u sum|z| and |dS2| <= d u sum z^2.  A warp slice lost from one flush moves
    a sum by ~1 / (8 x CTAs per N tile), at least 100x that.
    The variance var = S2/M - mean^2 is then off by (eps2 + 2 eps1)(1 + r^2) relative, r = |mean| /
    std, eps the two relative errors.  Those errors are a random walk of roundings, ~u sqrt(T / 3)
    per CTA, averaged over the CTAs: 1e-8 .. 3e-8.  VAR_BAR = 1e-7 (1 + r^2) keeps a 3x margin:
    1e-5 at r = 10, 1e-3 at r = 100.  The same sums bound the error the act scale assumes
    (split16.cu channel_bound, kappa = 16 + ceil(M / (16 * 132))), which is checked too.
  * Finalize: float64 arithmetic rounded once to fp32, so 1 fp32 ulp.
  * Apply: the folded affine y = fma(z, sc, sh) (+ q) with sc, sh rounded to fp32 is off by at most
    4u (|z sc| + |sh| + |residual terms|), the planes hold y to 2^-22 max|y|, and the statistics'
    own (measured) error adds |g invstd dmean| + |g xhat| dvar / (2 (var + eps)).
  * Backward: each bn_bwd_partial thread sums R rows in fp32 (R from bn_bwd_workers, `_bwd_rows`),
    then the rpi row slots of its CTA: depth d = R + rpi + 2, so |d dbeta| <= d u sum|g| and
    |d dgamma| <= (d + 1) u sum|g xhat| + sum|g| e_xhat, e_xhat = 4u (|xhat| + |mean| invstd) the
    fp32 xhat from the fp32 mean / invstd.  Not from max|dgamma|: dgamma cancels.
  * Scale contract: s is the power of two its rule gives from the bound computed here in float64
    from its definition (a factor of 2 only within 1e-3 of a power of two), and no element of a
    hi plane is +-65504, the clamp in split2 (a silent clip).

CPU tests below run the same bars against emulations of the kernels' arithmetic and show that
each has teeth."""
import math

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

U = 2.0 ** -24
HALF_MAX = 65504.0
NUM_SMS = 132          # common.cuh kNumSMs
EPS, MOM = 1e-5, 0.1
VAR_COEF = 1e-7        # VAR_BAR = VAR_COEF * (1 + r^2)


# ------------------------------------------------------------------ arithmetic shared with the bars
def _kappa(M):
    """split16.cu channel_bound: fp32 roundings a value meets in the conv16 statistics"""
    return 16 + math.ceil(M / (16.0 * NUM_SMS))


def _bound_def(s1, s2, sc, sh, M):
    """per-channel bound of |sc z + sh| from float64 statistics (split16.cu channel_bound)"""
    mean, q = s1 / M, s2 / M
    var = (q - mean * mean).clamp_min(0)
    ku = _kappa(M) * U
    return (sc * mean + sh).abs() + sc.abs() * (torch.sqrt(M * (var + 4 * ku * q)) + ku * torch.sqrt(q))


def _act_rule(bound):
    """publish_act_scale: the largest power of two s with s * bound < 2^15"""
    if not bound > 0:
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 15 - math.frexp(bound)[1])))


def _grad_rule(bound):
    """pow2_scale: 2^(13 - floor(log2 bound))"""
    if not bound > 0 or not math.isfinite(bound):
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 13 - (math.frexp(bound)[1] - 1))))


def _scale_ok(s, bound, rule):
    want = rule(bound)
    edge = bound > 0 and abs(math.log2(bound) - round(math.log2(bound))) < 1e-3
    return s == want or (edge and s in (want / 2, want * 2))


def _tile_runs(M, bm=128):
    """conv16 with statistics (m-fastest order) on a dense [M] grid: the tiles each CTA runs per
    N tile -- the length of the longest run and the number of CTAs per N tile"""
    tiles = -(-M // bm)
    grid = min(tiles, NUM_SMS)
    return -(-tiles // grid), grid


def _stats_depth(M):
    return 13 + _tile_runs(M)[0]


def _bwd_rows(M, C):
    """split16.cu make_rowmap + bn_bwd_workers: rows each partial thread sums, row slots per CTA"""
    C4 = C // 4
    tpr = min(C4, 256)
    rpi = max(256 // tpr, 1)
    chunks = -(-C4 // tpr)
    nblk = -(-M // rpi)
    cap = max(NUM_SMS * 3 // chunks, 1)
    workers = max(min(-(-nblk // 4), cap), 1)
    return -(-nblk // workers), rpi


# ------------------------------------------------------------------ CPU: emulations and teeth
def _emul_stats(z, ctas=NUM_SMS, drop_slice=False, drop_row=False):
    """conv16 epilogue order for the columns of z [M, C] (M a multiple of 128): per CTA, tiles
    cta, cta + ctas, ...; per warp 16 rows, two per lane, a shuffle tree over 8 lanes; fp32 slice
    adds over the tiles; the 8 slices added in warp order; one double add per CTA.
    drop_slice: the flush skips warp 7 of CTA 0.  drop_row: row 0 missing from the squares."""
    f = np.float32
    z = z.astype(f)
    M, C = z.shape
    X = z.reshape(M // 128, 8, 8, 2, C)             # tile, warp, lane group (8 lanes), row pair
    sq = X * X
    if drop_row:
        sq = sq.copy()
        sq[0, 0, 0, 0] = 0
    s1 = (X[:, :, :, 0] + X[:, :, :, 1]).astype(f)
    s2 = (sq[:, :, :, 0] + sq[:, :, :, 1]).astype(f)
    for _ in range(3):                              # xor 4, 8, 16
        s1 = (s1[:, :, 0::2] + s1[:, :, 1::2]).astype(f)
        s2 = (s2[:, :, 0::2] + s2[:, :, 1::2]).astype(f)
    s1, s2 = s1[:, :, 0], s2[:, :, 0]               # [tile, warp, C]
    S1, S2 = np.zeros(C), np.zeros(C)
    for c in range(ctas):
        w1 = np.add.accumulate(s1[c::ctas], axis=0, dtype=f)[-1]
        w2 = np.add.accumulate(s2[c::ctas], axis=0, dtype=f)[-1]
        v1, v2 = np.zeros(C, f), np.zeros(C, f)
        for w in range(8):
            if drop_slice and c == 0 and w == 7:
                continue
            v1, v2 = (v1 + w1[w]).astype(f), (v2 + w2[w]).astype(f)
        S1 += v1
        S2 += v2
    return S1, S2


def _stats_errors(S1, S2, z):
    """per channel: relative errors of S1 (to sum|z|), S2 (to sum z^2), var, and r = |mean| / std"""
    z = np.asarray(z, np.float64)
    M = z.shape[0]
    t1, t2, a1 = z.sum(0), (z * z).sum(0), np.abs(z).sum(0)
    mu, var = t1 / M, z.var(0)
    vk = np.maximum(S2 / M - (S1 / M) ** 2, 0)
    return (np.abs(S1 - t1) / a1, np.abs(S2 - t2) / t2, np.abs(vk - var) / var, np.abs(mu) / np.sqrt(var))


def test_stats_bars_hold_for_the_epilogue_order_and_have_teeth():
    """l1's M = 524288 rows over 132 CTAs, channels at r = 0, 1, 10, 100: the emulated epilogue
    meets the sum bar and VAR_BAR; a dropped warp slice misses the sum bar by > 100x, and a square
    dropped from S2 misses VAR_BAR."""
    M = 524288
    rng = np.random.default_rng(3)
    R = np.array([0.0, 1.0, 10.0, 100.0])
    z = (R + rng.standard_normal((M, 4))).astype(np.float32)
    z[0] = R + 2                                            # the row drop_row loses
    bar = _stats_depth(M) * U
    e1, e2, ev, r = _stats_errors(*_emul_stats(z), z)
    vbar = VAR_COEF * (1 + r * r)
    print("emulated eps1 %s eps2 %s var %s (bar %.1e, var bar %s)" % (e1, e2, ev, bar, vbar))
    assert (e1 <= bar).all() and (e2 <= bar).all() and (ev <= vbar).all()
    d1, d2, _, _ = _stats_errors(*_emul_stats(z, drop_slice=True), z)
    assert (d1[1:] >= 100 * bar).all() and (d2 >= 100 * bar).all()
    _, _, dv, _ = _stats_errors(*_emul_stats(z, drop_row=True), z)
    assert (dv[:2] >= 3 * vbar[:2]).all()


def _finalize64(s1, s2, M, gamma, beta, rm, rv):
    """bn_finalize_scale in float64 on float64 statistics and the fp32 parameters it reads"""
    eps, mom = float(np.float32(EPS)), float(np.float32(MOM))
    mean = s1 / M
    var = np.maximum(s2 / M - mean * mean, 0)
    inv = 1 / np.sqrt(var + eps)
    g, b = gamma.astype(np.float64), beta.astype(np.float64)
    unb = var * (M / (M - 1.0 if M > 1 else 1.0))
    return dict(mean=mean, invstd=inv, scale=g * inv, shift=b - mean * g * inv,
                rm=(1 - mom) * rm.astype(np.float64) + mom * mean,
                rv=(1 - mom) * rv.astype(np.float64) + mom * unb)


def _ulps(got, ref):
    """|got - ref| in units of the fp32 spacing at ref"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    sp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    sp = np.where(sp > 0, sp, np.spacing(np.float32(0)))
    return np.abs(got - ref) / sp


def test_finalize_ulp_bar_has_teeth():
    """A finalize that forms mean and var in fp32 misses the 1-ulp bar on invstd and scale by
    several ulps at the bench's M (var = E[x^2] - mean^2 cancels)."""
    rng = np.random.default_rng(5)
    C, M = 256, 524288
    mean = rng.standard_normal(C) * 3
    var = rng.uniform(0.1, 4, C)
    s1, s2 = mean * M, (var + mean * mean) * M
    g, b = rng.uniform(0.5, 1.5, C).astype(np.float32), (rng.standard_normal(C) * 0.1).astype(np.float32)
    ref = _finalize64(s1, s2, M, g, b, np.zeros(C, np.float32), np.ones(C, np.float32))
    assert _ulps(ref["mean"].astype(np.float32), ref["mean"]).max() <= 0.5
    f = np.float32
    m32 = s1.astype(f) / f(M)
    v32 = np.maximum(s2.astype(f) / f(M) - m32 * m32, f(0))
    inv32 = f(1) / np.sqrt(v32 + f(EPS))
    assert _ulps(inv32, ref["invstd"]).max() > 4 and _ulps(g * inv32, ref["scale"]).max() > 4


def test_act_scale_bound_covers_all_constant_channels():
    """Channels whose rows are all equal (gamma = 1, beta = 0), statistics in the epilogue order at
    M = 524288: with the bound |sc mean + sh| + |sc| sqrt(M var) alone, s * |y| passes 65504 in some
    trials (split2 would clip); with channel_bound's rounding terms it never does."""
    f = np.float32
    rng = np.random.default_rng(1)
    M = 524288
    old_over, new_over = 0, 0
    c = rng.uniform(0.1, 3.0, 24).astype(f)
    z = np.broadcast_to(c, (M, c.size))
    S1, S2 = _emul_stats(np.ascontiguousarray(z))
    mean, q = S1 / M, S2 / M
    var = np.maximum(q - mean * mean, 0)
    inv = 1 / np.sqrt(var + float(f(EPS)))
    sc, sh = inv.astype(f), (0.0 - mean * inv).astype(f)
    scd, shd = sc.astype(np.float64), sh.astype(np.float64)
    y = (c.astype(np.float64) * scd + shd).astype(f).astype(np.float64)      # fma: one rounding
    old = np.abs(scd * mean + shd) + np.abs(scd) * np.sqrt(M * var)
    new = _bound_def(*(torch.from_numpy(a) for a in (S1, S2, scd, shd)), M).numpy()
    for k in range(c.size):                       # one channel per tensor: s from that channel alone
        old_over += abs(y[k]) * _act_rule(float(f(old[k] * 1.001))) > HALF_MAX
        new_over += abs(y[k]) * _act_rule(float(f(new[k] * 1.001))) > HALF_MAX
    print("all-constant channels over 65504: old bound %d of %d, new bound %d" % (old_over, c.size, new_over))
    assert old_over > 0 and new_over == 0


def test_bwd_bars_have_teeth():
    """dbeta with the last of bn_bwd_combine's 32 groups of partials dropped misses the dbeta bar
    at 524288 x 256 by far (the partials of W workers, group g = w mod 32)."""
    M, C = 524288, 256
    R, rpi = _bwd_rows(M, C)
    W = -(-(-(-M // rpi)) // R)
    rng = np.random.default_rng(9)
    g = rng.standard_normal((W, C)) * np.sqrt(R * rpi)     # per-worker partial sums of unit-normal g
    err = np.abs(g[np.arange(W) % 32 == 31].sum(0))
    bar = (R + rpi + 2) * U * M * math.sqrt(2 / math.pi)    # d u sum|g|, E|g| = sqrt(2/pi)
    print("dropped group: median err / bar %.1f" % np.median(err / bar))
    assert (err > bar).mean() > 0.8 and err.max() >= 10 * bar


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _split_dev(v):
    """fp32 -> split planes through the engine's split16_batch: (planes, sc, joined float64)"""
    from epipolarpose_b200 import ops
    h = torch.empty(2 * v.numel(), device=v.device, dtype=torch.float16)
    sc = torch.ones(2, device=v.device)
    ops.split16_batch(ops.SplitBatch([(v.reshape(-1), h, sc)]))
    return h.view((2,) + tuple(v.shape)), sc, _join(h.view((2,) + tuple(v.shape)), sc)


def _join(planes, sc):
    return (planes[0].double() + planes[1].double()) * float(sc[1])


def _no_clamp(planes):
    """no element of the hi plane sits at split2's clamp"""
    return not bool((planes[0].float().abs() >= HALF_MAX).any())


def _contract_act(what, planes, sc, bound, ymax):
    s = float(sc[0])
    print("  %-34s s 2^%d bound %.4e s*max|y| %.1f" % (what, int(math.log2(s)), bound, s * ymax))
    assert _no_clamp(planes), "%s: hi plane at the fp16 clamp" % what
    assert s * ymax < HALF_MAX
    assert _scale_ok(s, bound, _act_rule), "%s: s %g, rule gives %g from %g" % (what, s, _act_rule(bound), bound)
    assert float(sc[1]) == 1 / s


def _stats64(z2d):
    z = z2d.double()
    return torch.cat([z.sum(0), (z * z).sum(0)])


# ------------------------------------------------------------------ 1. statistics from conv16
# (name, kind, cin, cout, k, stride, pad, N, hw, offset taps): the offset taps are the weight taps
# that read the constant input channel 0 at every output pixel exactly once (never padding)
STATS_CASES = [
    ("stem_col_192_64", "conv", 192, 64, 1, 1, 0, 128, 128, [(0, 0)]),
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 128, 64, [(0, 0)]),
    ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 128, 16, [(1, 1)]),
    ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 128, 8, [(0, 0)]),
    ("deconv2", "deconv", 256, 256, 4, 2, 1, 128, 32, [(a, b) for a in (1, 2) for b in (1, 2)]),
]
R_TARGETS = (0.0, 1.0, 10.0, 100.0)
_PRODUCED = {}


def _produce(dev, case):
    """conv16_fprop with statistics at a bench shape.  Input: relu(randn) with channel 0 == 1,
    so adding o_c to the weights of channel 0 at the offset taps shifts output channel c by o_c
    exactly; o_c targets mean / std = R_TARGETS[c % 4].  Returns (z [M, C], stats, stats of a
    second run)."""
    key = case[:9]
    if key in _PRODUCED:
        return _PRODUCED[key]
    from epipolarpose_b200 import net, ops
    name, kind, cin, cout, k, s, p, N, hw, taps = case
    conv = net.Conv("t", kind, cin, cout, k, s, p, 0)
    Ho, Wo = conv.out_hw(hw, hw)
    g = torch.Generator(device=dev).manual_seed(17)
    xf = torch.relu(torch.randn(N, hw, hw, cin, device=dev, generator=g))
    xf[..., 0] = 1.0
    x, x_sc, _ = _split_dev(xf)
    del xf
    K = k * k * cin
    w = torch.randn((cout, cin, k, k) if kind == "conv" else (cin, cout, k, k), device=dev, generator=g)
    w *= (2.0 / K) ** 0.5
    wc = w if kind == "conv" else w.transpose(0, 1)             # [cout][cin][k][k] view
    wc[:, 0] = 0
    # z_c ~ sum w x over the taps one pixel meets (all of a conv's, 1/4 of this deconv's);
    # relu(randn) has mean 1/sqrt(2 pi) and variance 1/2 - 1/(2 pi)
    frac = 1.0 if kind == "conv" else 0.25
    sd = torch.sqrt((wc[:, 1:] ** 2).sum((1, 2, 3)) * frac * (0.5 - 0.5 / math.pi))
    mu = wc[:, 1:].sum((1, 2, 3)) * frac / math.sqrt(2 * math.pi)
    rt = torch.tensor([R_TARGETS[c % 4] for c in range(cout)], device=dev)
    off = rt * sd - mu
    for a, b in taps:
        wc[:, 0, a, b] = off
    wf32, _ = conv.pack(ops, w)
    wf, wf_sc, _ = _split_dev(wf32)
    out = torch.empty(N, Ho, Wo, cout, device=dev)
    runs = []
    for _ in range(2):
        st = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
        for gm in conv.fprop_geoms(ops, N, hw, hw, 3):
            if gm is not None:
                gm.in_relu, gm.accumulate = 0, 0
                ops.conv16_fprop(gm, x, x_sc, wf, wf_sc, out, None, st)
        runs.append(st)
    torch.cuda.synchronize()
    M = N * Ho * Wo
    res = (out.view(M, cout), runs[0], runs[1], conv)
    if name.endswith(("stem_col_192_64", "l1_1x1_64_256")):   # reused by the apply / pool tests
        _PRODUCED[key] = res
    return res


@gpu
@pytest.mark.parametrize("case", STATS_CASES, ids=[c[0] for c in STATS_CASES])
def test_conv16_stats_vs_float64(dev, case):
    """S1 and S2 per channel against float64 sums of the returned z, mean and var within their
    bars and within what channel_bound assumes, two runs bit-identical."""
    z, st, st2, conv = _produce(dev, case)
    M, C = z.shape
    assert torch.equal(st, st2), "statistics not run-to-run identical"
    zd = z.double()
    t1, t2, a1 = zd.sum(0), (zd * zd).sum(0), zd.abs().sum(0)
    mu64, var64 = t1 / M, (zd - t1 / M).pow(2).sum(0) / M
    del zd
    s1, s2 = st[:C], st[C:]
    e1, e2 = (s1 - t1).abs() / a1, (s2 - t2).abs() / t2
    # deconv: four phase launches, each with its own (shorter) tile runs; the dense M is the worst
    d = _stats_depth(M)
    bar = d * U
    mk = s1 / M
    vk = (s2 / M - mk * mk).clamp_min(0)
    r = mu64.abs() / var64.sqrt()
    ev = (vk - var64).abs() / var64
    vbar = VAR_COEF * (1 + r * r)
    ku, q = _kappa(M) * U, t2 / M
    for lo, hi in ((0, 0.5), (0.5, 3), (3, 30), (30, 1e9)):
        sel = (r >= lo) & (r < hi)
        if sel.any():
            print("  %-18s r in [%g, %g): eps1 %.2e eps2 %.2e var %.2e (var bar %.2e) bar %.2e"
                  % (case[0], lo, hi, float(e1[sel].max()), float(e2[sel].max()), float(ev[sel].max()),
                     float(vbar[sel].max()), bar))
    assert float(e1.max()) <= bar and float(e2.max()) <= bar, "sum %.3e / squares %.3e (bar %.2e)" % (
        float(e1.max()), float(e2.max()), bar)
    assert bool((ev <= vbar).all()), "var %.3e at r %.1f" % (float((ev / vbar).max()), float(r[(ev / vbar).argmax()]))
    assert bool(((mk - mu64).abs() <= ku * q.sqrt()).all())                     # channel_bound's dmean
    assert bool((var64 - vk <= 4 * ku * q).all())                               # and its var deficit


# ------------------------------------------------------------------ 2. finalize
def _finalize_dev(dev, st, M, C, gamma, beta, rm, rv, group2=(None, None, None), res_sc=None):
    from epipolarpose_b200 import ops
    out = {k: torch.empty(C, device=dev) for k in ("scale", "shift", "mean", "invstd")}
    sc = torch.empty(4, device=dev)
    ops.bn_finalize_scale(st, M, C, gamma, beta, EPS, MOM, rm, rv, out["scale"], out["shift"],
                          out["mean"], out["invstd"], *group2, res_sc, sc)
    out["sc"] = sc
    return out


@gpu
@pytest.mark.parametrize("M", [1, 2, 524288, 2097152])
def test_bn_finalize_scale_vs_float64(dev, M):
    """Every output within 1 fp32 ulp of float64 arithmetic on the same statistics and fp32
    parameters: gamma < 0 and = 0 channels, running statistics (unbiased, momentum), a second
    group and res_sc; the published scale is the rule's power of two of the float64 bound."""
    C = 256
    rng = np.random.default_rng(M)
    mean = rng.standard_normal(C) * 3
    var = rng.uniform(0.01, 4, C) if M > 1 else np.zeros(C)
    var[:4] = 0 if M > 1 else var[:4]                        # constant channels
    s1, s2 = mean * M, (var + mean * mean) * M
    g = rng.uniform(0.5, 1.5, C).astype(np.float32)
    g[4:12] *= -1
    g[12:16] = 0
    b = (rng.standard_normal(C) * 0.3).astype(np.float32)
    rm0, rv0 = rng.standard_normal(C).astype(np.float32), rng.uniform(0.5, 2, C).astype(np.float32)
    st2 = torch.tensor(np.concatenate([mean[::-1] * M, (var[::-1] + mean[::-1] ** 2) * M]), device=dev)
    sc2 = torch.tensor(rng.uniform(0.5, 1.5, C).astype(np.float32), device=dev)
    sh2 = torch.tensor((rng.standard_normal(C) * 0.1).astype(np.float32), device=dev)
    res_sc = torch.tensor([4.0, 0.25, 37.5, 0.0], device=dev)
    T = lambda a: torch.tensor(a, device=dev)
    st = torch.tensor(np.concatenate([s1, s2]), device=dev)
    for second in (False, True):
        rm, rv = T(rm0.copy()), T(rv0.copy())
        out = _finalize_dev(dev, st, M, C, T(g), T(b), rm, rv, (st2, sc2, sh2) if second else (None,) * 3,
                            res_sc if second else None)
        torch.cuda.synchronize()
        ref = _finalize64(st[:C].cpu().numpy(), st[C:].cpu().numpy(), M, g, b, rm0, rv0)
        got = dict(mean=out["mean"], invstd=out["invstd"], scale=out["scale"], shift=out["shift"], rm=rm, rv=rv)
        for k in got:
            u = _ulps(got[k].cpu().numpy(), ref[k])
            assert u.max() <= 1, "%s: %.2f ulp at channel %d" % (k, u.max(), u.argmax())
        scd, shd = out["scale"].double(), out["shift"].double()
        bound = float(_bound_def(st[:C], st[C:], scd, shd, M).max())
        if second:
            bound += float(_bound_def(st2[:C], st2[C:], sc2.double(), sh2.double(), M).max())
        bound = bound * 1.001 + (37.5 if second else 0.0)
        s = float(out["sc"][0])
        assert _scale_ok(s, bound, _act_rule) and abs(float(out["sc"][2]) - bound) <= 1e-6 * bound


# ------------------------------------------------------------------ 3. apply at bench M
def _apply_bar(zd, scd, shd, res_terms, ymax):
    return 4 * U * ((zd * scd).abs() + shd.abs() + res_terms) + 2.0 ** -22 * ymax


@gpu
@pytest.mark.parametrize("res", ["none", "split", "affine"])
def test_bn_act_split_vs_float64_at_bench_M(dev, res):
    """l1's conv16 output (524288 x 256, r up to 100) -> bn_finalize_scale -> bn_act_split against
    float64 relu(gamma (z - mean64) / sqrt(var64 + eps) + beta (+ residual)); the ReLU bit mask
    against the float64 sign (flips only within the bar); the scale contract."""
    _check_bn_act_split(dev, res, STATS_CASES[1])


def _check_bn_act_split(dev, res, case):
    from epipolarpose_b200 import ops
    z, st, _, _ = _produce(dev, case)
    M, C = z.shape
    g = torch.Generator(device=dev).manual_seed(23)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    gamma[::7] *= -1
    beta = torch.randn(C, device=dev, generator=g) * 0.2
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    r = rs = r_sc = rscale = rshift = None
    group2, res_terms, res64 = (None,) * 3, 0.0, 0.0
    if res == "split":
        rs, rsc2, res64 = _split_dev(torch.relu(torch.randn(M, C, device=dev, generator=g)) * 2)
        r_sc = torch.tensor([float(rsc2[0]), float(rsc2[1]), float(res64.abs().max()), 0.0], device=dev)
        res_terms = res64.abs()
    elif res == "affine":
        r = torch.randn(M, C, device=dev, generator=g) * 1.5 + 0.3
        rscale = torch.rand(C, device=dev, generator=g) + 0.5
        rshift = torch.randn(C, device=dev, generator=g) * 0.1
        rst = _stats64(r)
        group2 = (rst, rscale, rshift)
        rd = r.double()
        res64 = rd * rscale.double() + rshift.double()
        res_terms = (rd * rscale.double()).abs() + rshift.double().abs() + res64.abs()
        del rd
    out = _finalize_dev(dev, st, M, C, gamma, beta, rm, rv, group2, r_sc)
    y = torch.empty(2, M, C, device=dev, dtype=torch.float16)
    bits = torch.empty(M * C // 8, device=dev, dtype=torch.uint8)
    ops.bn_act_split(z, out["scale"], out["shift"], r, rscale, rshift, rs, r_sc, 1, M, C, y, out["sc"], bits)
    torch.cuda.synchronize()
    zd = z.double()
    mu64 = zd.mean(0)
    var64 = (zd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    xh = (zd - mu64) * inv64
    pre = gamma.double() * xh + beta.double() + res64
    y64 = pre.clamp_min(0)
    # the statistics' own error, first order (test_conv16_stats_vs_float64 bounds it)
    mk = st[:C] / M
    vk = (st[C:] / M - mk * mk).clamp_min(0)
    stat_term = (gamma.double() * inv64 * (mk - mu64)).abs() + \
        (gamma.double() * xh).abs() * (vk - var64).abs() / (2 * (var64 + EPS))
    ymax = float(y64.max())
    bar = _apply_bar(zd, out["scale"].double(), out["shift"].double(), res_terms, ymax) + stat_term
    del xh
    got = _join(y, out["sc"]).view(M, C)
    err = (got - y64).abs()
    print("  apply %-6s max err %.3e, worst err / bar %.3f" % (res, float(err.max()), float((err / bar).max())))
    assert bool((err <= bar).all()), "apply error %.3e over its bar" % float((err - bar).max())
    flips = torch.from_numpy(np.unpackbits(bits.cpu().numpy(), bitorder="little").astype(bool)).to(dev) \
        ^ (pre > 0).view(-1)
    if bool(flips.any()):
        assert bool((pre.view(-1)[flips].abs() <= bar.view(-1)[flips]).all()), "ReLU mask flip outside the bar"
    scd, shd = out["scale"].double(), out["shift"].double()
    zs = _stats64(z)
    bound = float(_bound_def(zs[:C], zs[C:], scd, shd, M).max())
    if res == "affine":
        bound += float(_bound_def(rst[:C], rst[C:], rscale.double(), rshift.double(), M).max())
    bound = bound * 1.001 + (float(r_sc[2]) if r_sc is not None else 0.0)
    _contract_act("apply %s" % res, y, out["sc"], bound, ymax)


@gpu
def test_bn_relu_maxpool_split_vs_float64_at_stem_size(dev):
    """The stem's conv16 output (N = 128, 128 x 128 x 64) -> bn_finalize_scale ->
    bn_relu_maxpool_split against float64 BatchNorm + ReLU + 3x3/2 max pool; argidx may pick
    another window entry only if its value is within the bar of the maximum (ties)."""
    _check_bn_relu_maxpool_split(dev, STATS_CASES[0])


def _check_bn_relu_maxpool_split(dev, case):
    """the pool over the stem_col case's conv16 output (N images of hw x hw)"""
    from epipolarpose_b200 import ops
    z, st, _, _ = _produce(dev, case)
    M, C = z.shape
    N, H = case[7], case[8]
    W = H
    Ho, Wo = H // 2, W // 2
    g = torch.Generator(device=dev).manual_seed(29)
    gamma, beta = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g) * 0.2
    out = _finalize_dev(dev, st, M, C, gamma, beta, torch.zeros(C, device=dev), torch.ones(C, device=dev))
    y = torch.empty(2, N, Ho, Wo, C, device=dev, dtype=torch.float16)
    arg = torch.empty(N, Ho, Wo, C, device=dev, dtype=torch.uint8)
    ops.bn_relu_maxpool_split(z, out["scale"], out["shift"], y, out["sc"], arg, N, H, W, C)
    torch.cuda.synchronize()
    zd = z.double()
    mu64 = zd.mean(0)
    var64 = (zd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    mk = st[:C] / M
    vk = (st[C:] / M - mk * mk).clamp_min(0)
    xh = (zd - mu64) * inv64
    a64 = (gamma.double() * xh + beta.double()).clamp_min(0)
    e = 4 * U * ((zd * out["scale"].double()).abs() + out["shift"].double().abs()) + \
        (gamma.double() * inv64 * (mk - mu64)).abs() + (gamma.double() * xh).abs() * (vk - var64).abs() / (2 * (var64 + EPS))
    del zd, xh
    pa = torch.full((N, H + 2, W + 2, C), float("-inf"), device=dev, dtype=torch.float64)
    pa[:, 1:-1, 1:-1] = a64.view(N, H, W, C)
    pe = torch.zeros((N, H + 2, W + 2, C), device=dev, dtype=torch.float64)
    pe[:, 1:-1, 1:-1] = e.view(N, H, W, C)
    del a64, e
    cand = torch.stack([pa[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)])
    ce = torch.stack([pe[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)])
    del pa, pe
    ref = cand.max(0).values
    ymax = float(ref.max())
    bar = ce.max(0).values + 2.0 ** -22 * ymax
    got = _join(y, out["sc"])
    err = (got - ref).abs()
    print("  maxpool max err %.3e, worst err / bar %.3f" % (float(err.max()), float((err / bar).max())))
    assert bool((err <= bar).all())
    picked = cand.gather(0, arg.long().unsqueeze(0)).squeeze(0)
    assert bool((picked >= ref - 2 * bar).all()), "argidx picks an entry below the window maximum"
    zs = _stats64(z)
    bound = float(_bound_def(zs[:C], zs[C:], out["scale"].double(), out["shift"].double(), M).max()) * 1.001
    _contract_act("stem maxpool", y, out["sc"], bound, ymax)


# ------------------------------------------------------------------ 4. the scale contract, adversarial
ADV = ["one_hot", "zeros", "const_beside", "all_const_b0", "all_const_b1e-6", "big_beta", "res_at_bound",
       "eval_far", "eval_const"]


def _adv_inputs(dev, case, M, C):
    """input x [M, C] >= 0 and weights [C][C] of a 1x1 conv for an adversarial case"""
    g = torch.Generator(device=dev).manual_seed(31)
    x = torch.relu(torch.randn(M, C, device=dev, generator=g))
    w = torch.randn(C, C, device=dev, generator=g) * (2.0 / C) ** 0.5
    if case == "one_hot":
        x[:, 0] = 0
        x[M // 3, 0] = 1.0
        w[0] = 0
        w[0, 0] = 1
    elif case == "zeros":
        x.zero_()
    elif case in ("const_beside", "eval_const", "eval_far"):
        x[:, 1] = 1.7
        w[1] = 0
        w[1, 1] = 1
    elif case.startswith("all_const"):
        x[:] = (torch.rand(C, device=dev, generator=g) * 2.9 + 0.1)
        w = torch.eye(C, device=dev)
    return x, w


@gpu
@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("case", ADV)
def test_scale_contract_adversarial(dev, case, relu):
    """conv16 (1x1, 64 -> 64, M = 524288) -> bn_finalize_scale (or, eval, bn_eval_affine +
    act_scale) -> bn_act_split: s is the rule's power of two of the bound computed here, the hi
    plane never reaches the fp16 clamp, and the joined planes are the float64 affine of z."""
    from epipolarpose_b200 import net, ops
    M, C = 524288, 64
    x, w = _adv_inputs(dev, case, M, C)
    conv = net.Conv("t", "conv", C, C, 1, 1, 0, 0)
    xs, xsc, _ = _split_dev(x)
    ws, wsc, _ = _split_dev(w.contiguous())
    z = torch.empty(M, C, device=dev)
    st = torch.zeros(2 * C, device=dev, dtype=torch.float64)
    for gm in conv.fprop_geoms(ops, 128, 64, 64, 3):
        gm.in_relu, gm.accumulate = 0, 0
        ops.conv16_fprop(gm, xs, xsc, ws, wsc, z, None, st)
    g = torch.Generator(device=dev).manual_seed(37)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    beta = torch.randn(C, device=dev, generator=g) * 0.1
    if case.startswith("all_const"):
        gamma.fill_(1)
        beta.fill_(0 if case.endswith("b0") else 1e-6)
    if case == "big_beta":
        beta[5], beta[7] = 3e4, -1e5
    rs = r_sc = None
    res64 = 0.0
    if case == "res_at_bound":
        rv = torch.relu(torch.randn(M, C, device=dev, generator=g))
        rs, rsc2, res64 = _split_dev(rv)
        r_sc = torch.tensor([float(rsc2[0]), float(rsc2[1]), float(res64.abs().max()), 0.0], device=dev)
    zd = z.double()
    if case.startswith("eval"):
        mu, var = zd.mean(0), zd.var(0, unbiased=False)
        rmean = (mu + 50 * var.sqrt() + 1).float()
        rvar = (var * 1e-4).float()
        if case == "eval_const":
            rmean[1], rvar[1] = z[0, 1], 0.0                    # running mean == the constant
        scale, shift = torch.empty(C, device=dev), torch.empty(C, device=dev)
        ops.bn_eval_affine(C, gamma, beta, rmean, rvar, EPS, scale, shift)
        sc = torch.empty(4, device=dev)
        ops.act_scale(st, scale, shift, M, C, None, None, None, r_sc, sc)
    else:
        out = _finalize_dev(dev, st, M, C, gamma, beta, torch.zeros(C, device=dev), torch.ones(C, device=dev),
                            res_sc=r_sc)
        scale, shift, sc = out["scale"], out["shift"], out["sc"]
    y = torch.empty(2, M, C, device=dev, dtype=torch.float16)
    ops.bn_act_split(z, scale, shift, None, None, None, rs, r_sc, relu, M, C, y, sc)
    torch.cuda.synchronize()
    scd, shd = scale.double(), shift.double()
    y64 = zd * scd + shd + res64
    if relu:
        y64 = y64.clamp_min(0)
    ymax = float(y64.abs().max())
    zs = _stats64(z)
    bound = float(_bound_def(zs[:C], zs[C:], scd, shd, M).max()) * 1.001 + (float(r_sc[2]) if r_sc is not None else 0.0)
    _contract_act("%s relu=%d" % (case, relu), y, sc, bound, ymax)
    res_terms = res64.abs() if r_sc is not None else 0.0
    err = (_join(y, sc).view(M, C) - y64).abs()
    assert bool((err <= _apply_bar(zd, scd, shd, res_terms, ymax)).all())


# ------------------------------------------------------------------ 5. backward at bench M
BWD_SHAPES = [(2097152, 64), (524288, 256), (8192, 2048)]


@gpu
@pytest.mark.parametrize("mode", ["relu", "mask", "bits_inplace"])
@pytest.mark.parametrize("M,C", BWD_SHAPES, ids=["%dx%d" % s for s in BWD_SHAPES])
def test_bn_bwd_split_vs_float64_at_bench_M(dev, M, C, mode):
    """bn_bwd_split against float64 autograd of the forward BatchNorm: dgamma, dbeta per channel
    and the joined dz elementwise, with a constant channel (invstd = 316), one huge gradient
    element and a fully masked channel beside ordinary ones; two runs bit-identical; the scale of
    dz from its bound."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(M + C)
    mu_c = torch.randn(C, device=dev, generator=g) * 2
    x = torch.randn(M, C, device=dev, generator=g) * (torch.rand(C, device=dev, generator=g) * 2 + 0.2) + mu_c
    x[:, 0] = 0.37                                           # var 0: invstd = 1 / sqrt(eps)
    dy = torch.randn(M, C, device=dev, generator=g) * 1e-4
    dy[M // 2, 1] = 3.0                                      # one huge element
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    beta = torch.randn(C, device=dev, generator=g) * 0.1
    xd = x.double()
    mu64 = xd.mean(0)
    var64 = (xd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    mean, invstd = mu64.float(), inv64.float()
    scale, shift = (gamma.double() * inv64).float(), (beta.double() - mu64 * gamma.double() * inv64).float()
    mask = bits = None
    if mode == "relu":
        scale[2], shift[2] = 0.0, -1.0                         # fully masked channel
    elif mode == "mask":
        mask = torch.relu(torch.randn(M, C, device=dev, generator=g)).half()
        mask[:, 2] = 0
    else:
        keep = torch.rand(M, C, device=dev, generator=g) > 0.4
        keep[:, 2] = False
        bits = torch.from_numpy(np.packbits(keep.cpu().numpy().reshape(-1), bitorder="little")).to(dev)
    runs = []
    for _ in range(2):
        dyk = dy.clone()
        dm = dyk if mode == "bits_inplace" else torch.empty_like(dy)
        dz = torch.empty(2, M, C, device=dev, dtype=torch.float16)
        sc = torch.empty(2, device=dev)
        dg, db = torch.empty(C, device=dev), torch.empty(C, device=dev)
        ops.bn_bwd_split(dyk, x, mask, scale, shift, mean, invstd, gamma, int(mode == "relu"), M, C, dz, sc, dm,
                         dg, db, mask_bits=bits)
        torch.cuda.synchronize()
        runs.append((dz, sc, dg, db, dm))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a,
                           b.view(torch.int16) if b.dtype == torch.float16 else b), "not run-to-run identical"
    dz, sc, dg, db, dm = runs[0]
    del runs
    # the gradient the kernel masked: its own mask in relu mode (a fp32 fma at the threshold),
    # which must agree with the float64 sign except within one rounding of zero
    if mode == "relu":
        pre = xd * scale.double() + shift.double()
        keep64 = pre > 0
        flip = (dm != 0) != keep64
        flip &= dy != 0
        if bool(flip.any()):
            assert bool((pre[flip].abs() <= 2 * U * ((xd * scale.double()).abs() + shift.double().abs())[flip]).all())
        g64 = dm.double()
        del pre, keep64, flip
    elif mode == "mask":
        g64 = dy.double() * (mask != 0)
    else:
        g64 = dy.double() * keep
        assert torch.equal(dm, g64.float())
    z64 = xd.clone().requires_grad_(True)
    m = z64.mean(0)
    v = (z64 - m).pow(2).mean(0)
    yref = gamma.double() * (z64 - m) / torch.sqrt(v + float(np.float32(EPS))) + beta.double()
    yref.backward(g64)
    dz64 = z64.grad
    del z64, m, v, yref
    xh = (xd - mu64) * inv64
    dgam64, dbet64 = (g64 * xh).sum(0), g64.sum(0)
    R, rpi = _bwd_rows(M, C)
    d = R + rpi + 2
    ag = g64.abs()
    e_xh = 4 * U * (xh.abs() + mu64.abs() * inv64)
    bar_b = d * U * ag.sum(0)
    bar_g = (d + 1) * U * (ag * xh.abs()).sum(0) + (ag * e_xh).sum(0)
    eb = (db.double() - dbet64).abs() - U * dbet64.abs()
    eg = (dg.double() - dgam64).abs() - U * dgam64.abs()
    print("  bwd %dx%d %-12s R %d dbeta %.2e (bar %.2e) dgamma %.2e (bar %.2e)" % (
        M, C, mode, R, float((eb + U * dbet64.abs()).max()), float(bar_b.max()),
        float((eg + U * dgam64.abs()).max()), float(bar_g.max())))
    assert bool((eb <= bar_b).all()), "dbeta"
    assert bool((eg <= bar_g).all()), "dgamma"
    k1, k2 = dbet64 / M, dgam64 / M
    a = (gamma.double() * inv64).abs()
    dzmax = float(dz64.abs().max())
    bar = a * (4 * U * (ag + k1.abs() + (xh * k2).abs()) + bar_b / M + xh.abs() * (bar_g / M) + k2.abs() * e_xh) \
        + 2 * U * dz64.abs() + 2.0 ** -22 * dzmax
    err = (_join(dz, sc).view(M, C) - dz64).abs()
    print("  bwd %dx%d %-12s dz max err %.3e, worst err / bar %.3f" % (M, C, mode, float(err.max()),
                                                                     float((err / bar).max())))
    assert bool((err <= bar).all()), "dz"
    # the scale of dz: pow2_scale of max_c |gamma invstd| (max|g| + |k1| + max|xhat| |k2|)
    bound = float((a * (ag.max(0).values + k1.abs() + xh.abs().max(0).values * k2.abs())).max())
    s = float(sc[0])
    assert _scale_ok(s, bound, _grad_rule) and float(sc[1]) == 1 / s
    assert _no_clamp(dz) and s * dzmax < HALF_MAX


# ------------------------------------------------------------------ 6. logit gradient at the bench shape
@gpu
def test_softargmax_bwd_split_vs_float64_at_bench_shape(dev):
    """N = 128, J = 16, D = 64, 64 x 64 (2.1 GB of logits): the joined planes against float64
    p (s - E_p[s]), the bias column sums over 524288 rows against float64, the scale contract,
    and the bias sums bit-identical over two runs."""
    from epipolarpose_b200 import ops
    N, J, D, H, W = 128, 16, 64, 64, 64
    C = J * D
    g = torch.Generator(device=dev).manual_seed(43)
    logits = torch.randn(N, H, W, C, device=dev, generator=g) * 3
    dco = torch.randn(N, J * 3, device=dev, generator=g)
    coords, lse = torch.empty(N, J * 3, device=dev), torch.empty(N * J * 2, device=dev)
    ops.softargmax_fwd(logits, 1, N, J, D, H, W, coords, lse)
    pl = torch.empty(2, N, H, W, C, device=dev, dtype=torch.float16)
    sc, db = torch.empty(2, device=dev), torch.empty(C, device=dev)
    ops.softargmax_bwd_split(logits, N, J, D, H, W, coords, lse, dco, pl, sc, db)
    db2 = torch.empty(C, device=dev)
    ops.softargmax_bwd_split(logits, N, J, D, H, W, coords, lse, dco, pl, torch.empty(2, device=dev), db2)
    torch.cuda.synchronize()
    assert torch.equal(db, db2), "bias sums not run-to-run identical"
    s = float(sc[0])
    inv_k = lse.view(N, J, 2)[..., 1].double()
    bound = float((inv_k * dco.view(N, J, 3).abs().double().sum(-1)).max())
    assert _scale_ok(s, bound, _grad_rule) and float(sc[1]) == 1 / s
    assert _no_clamp(pl)
    # S = split count and rows per thread of epb_softargmax_bwd_split
    C4, ppi = C // 4, max(512 // (C // 4), 1)
    S = 1
    while N * S < 8 * NUM_SMS and (H * W) // (S * 2) >= 16 * ppi:
        S *= 2
    depth = -(-(-(-(H * W) // S)) // ppi) + ppi + 1
    xs = torch.arange(W, device=dev, dtype=torch.float64).view(1, 1, W, 1, 1)
    ys = torch.arange(H, device=dev, dtype=torch.float64).view(1, H, 1, 1, 1)
    zs = torch.arange(D, device=dev, dtype=torch.float64).view(1, 1, 1, 1, D)
    colsum, colbar, colabs = (torch.zeros(C, device=dev, dtype=torch.float64) for _ in range(3))
    worst, dlmax = 0.0, 0.0
    ratio = 0.0
    B = 8
    for n0 in range(0, N, B):
        v = logits[n0:n0 + B].double().view(B, H, W, J, D)
        m = v.amax((1, 2, 4), keepdim=True)
        ex = torch.exp(v - m)
        tot = ex.sum((1, 2, 4), keepdim=True)
        p = ex / tot
        del ex
        dc = dco[n0:n0 + B].double().view(B, 1, 1, J, 3)
        gx, gy, gz = dc[..., 0:1] / W, dc[..., 1:2] / H, dc[..., 2:3] / D
        s_ = gx * xs + gy * ys + gz * zs
        sbar = (p * s_).sum((1, 2, 4), keepdim=True)
        dl = p * (s_ - sbar)
        # the kernel's sbar from its forward coords, and its 1 / sum(exp) from lse
        cr = coords[n0:n0 + B].double().view(B, 1, 1, J, 3)
        sbar_k = gx * (cr[..., 0:1] + 0.5) * W + gy * (cr[..., 1:2] + 0.5) * H + gz * (cr[..., 2:3] + 0.5) * D
        ik = lse.view(N, J, 2)[n0:n0 + B, :, 1].double().view(B, 1, 1, J, 1)
        e_inv = (ik * tot - 1).abs()
        e = p * ((6 + 3.5 * (v - m).abs()) * U * (s_ - sbar).abs()
                 + 6 * U * ((gx * xs).abs() + (gy * ys).abs() + (gz * (zs + 3)).abs() + sbar.abs())
                 + (sbar_k - sbar).abs() + e_inv * (s_ - sbar).abs())
        del v, p, s_
        got = _join(pl[:, n0:n0 + B], sc).view(B, H, W, J, D)
        err = (got - dl).abs()
        dlmax = max(dlmax, float(dl.abs().max()))
        ratio = max(ratio, float((err / (e + 2.0 ** -22 * float(dl.abs().max()) + 1e-300)).max()))
        worst = max(worst, float(err.max()))
        colsum += dl.sum((0, 1, 2)).reshape(C)
        colabs += dl.abs().sum((0, 1, 2)).reshape(C)
        colbar += e.sum((0, 1, 2)).reshape(C)
        del got, err, dl, e
    print("  softargmax bwd: max err %.3e, worst err / bar %.3f, s*max|dl| %.0f" % (worst, ratio, s * dlmax))
    assert ratio <= 1.0, "logit gradient over its bar"
    assert s * dlmax < HALF_MAX
    eb = (db.double() - colsum).abs()
    bbar = colbar + depth * U * colabs + U * colsum.abs()
    print("  softargmax dbias: max err %.3e, worst err / bar %.3f" % (float(eb.max()), float((eb / bbar).max())))
    assert bool((eb <= bbar).all()), "bias column sums"

