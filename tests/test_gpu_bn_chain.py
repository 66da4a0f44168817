"""The split-fp16 BatchNorm chain against float64 at the bench's sizes: the statistics the conv16
epilogue sums (tc::stats_add / stats_flush), bn_finalize_scale, the post-activation producers
bn_act_split / bn_relu_maxpool_split, bn_bwd_split and softargmax_bwd_split.  Every reference is
torch float64 on the device, computed from the exact fp32 values the kernels read or wrote (the
kernel's own z, the joined planes), so each bar is the kernel's rounding and nothing else.

Bars (u = 2^-24, one fp32 rounding), each derived in the docstring of the tests/step_cases.py
function that computes it:

  * Statistics: check_conv16_stats (VAR_BAR = VAR_COEF (1 + r^2)).
  * Finalize: check_bn_finalize_scale, 1 fp32 ulp.
  * Apply: _apply_bar.
  * Backward: check_bn_bwd_split.
  * Scale contract: _contract_act.

CPU tests below run the same bars against emulations of the kernels' arithmetic and show that
each has teeth."""
import math

import numpy as np
import pytest
import torch

from tests.step_cases import (EPS, HALF_MAX, NUM_SMS, U, VAR_COEF, _act_rule, _apply_bar, _bound_def, _bwd_rows,
                              _check_bn_act_split, _check_bn_relu_maxpool_split, _contract_act, _finalize64,
                              _finalize_dev, _grad_rule, _join, _no_clamp, _scale_ok, _split_dev, _stats64,
                              _stats_depth, _ulps, check_bn_bwd_split, check_bn_finalize_scale, check_conv16_stats)

gpu = pytest.mark.gpu


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


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


# ------------------------------------------------------------------ 1. statistics from conv16
# (name, kind, cin, cout, k, stride, pad, N, hw, offset taps): step_cases._produce
STATS_CASES = [
    ("stem_col_192_64", "conv", 192, 64, 1, 1, 0, 128, 128, [(0, 0)]),
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 128, 64, [(0, 0)]),
    ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 128, 16, [(1, 1)]),
    ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 128, 8, [(0, 0)]),
    ("deconv2", "deconv", 256, 256, 4, 2, 1, 128, 32, [(a, b) for a in (1, 2) for b in (1, 2)]),
]


@gpu
@pytest.mark.parametrize("case", STATS_CASES, ids=[c[0] for c in STATS_CASES])
def test_conv16_stats_vs_float64(dev, case):
    check_conv16_stats(dev, case)


# ------------------------------------------------------------------ 2. finalize
@gpu
@pytest.mark.parametrize("M", [1, 2, 524288, 2097152])
def test_bn_finalize_scale_vs_float64(dev, M):
    check_bn_finalize_scale(dev, M)


# ------------------------------------------------------------------ 3. apply at bench M
@gpu
@pytest.mark.parametrize("res", ["none", "split", "affine"])
def test_bn_act_split_vs_float64_at_bench_M(dev, res):
    """l1's conv16 output (524288 x 256, r up to 100) -> bn_finalize_scale -> bn_act_split"""
    _check_bn_act_split(dev, res, STATS_CASES[1])


@gpu
def test_bn_relu_maxpool_split_vs_float64_at_stem_size(dev):
    """The stem's conv16 output (N = 128, 128 x 128 x 64) -> bn_finalize_scale ->
    bn_relu_maxpool_split"""
    _check_bn_relu_maxpool_split(dev, STATS_CASES[0])


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
    check_bn_bwd_split(dev, M, C, mode)


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

