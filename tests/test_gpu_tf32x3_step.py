"""The tf32x3 training step (net.Engine at precision 3: the 3xTF32 wgmma convolutions and the fp32
bn.cu BatchNorm chain; MODEL.PRECISION's default, bench.py --precision tf32x3, and the engine
get_pose_net falls back to for plans net16 refuses) against float64 kernel by kernel at the bench's
sizes (R50, J = 16, D = 64, 256 x 256, N = 128: 32 tuples x 4 views).  tests/test_step_coverage.py
gates the tf32x3 step on these tests.

Every reference is torch float64 on the device, computed from the exact fp32 values the kernel
read, in image or row chunks where memory needs it.  Bars (u = 2^-24):

  * Convolutions (fprop, dgrad, wgrad at every distinct R50 conv of the step, with the step's
    operand modes: step_cases.C4_LAYERS_TF32X3): the bars of test_gpu_tf32.  fprop / dgrad:
    _tc_bar(FPROP_BAR, K, 3), K the longest taps x Cin of the call's geometries; wgrad: _tc_bar(WGRAD_BAR, R, 3), R the pixel
    run of one CTA from the TF32 wgrad planner (`_tf32_wgrad_plan` over each geometry's
    N Hp Wp pixels), since wgmma accumulates toward zero.  Statistics: STATS_SELF_BAR against
    the float64 sums of the kernel's own output, the fprop bar against the reference's sums.
    Every conv kernel that runs must be a three-pass instantiation `<*, 3>`.
  * bn_bwd_reduce + bn_bwd_apply (step_cases.check_bn_bwd).  Each thread adds kRowsPerThread =
    64 rows in fp32, the CTA's row slots and all CTAs add in double, so with d = 64 + 2,
    |d dbeta| <= d u sum|g| and |d dgamma| <= (d + 1) u sum|g xhat| + sum|g| e_xhat, where e_xhat = 4u (|xhat| + |mean|
    invstd) is the error of the fp32 xhat formed from the fp32 mean and invstd (the same terms
    as test_gpu_bn_chain's backward).  dgamma and dbeta then round once to fp32.  Not from
    max|dgamma|: dgamma cancels.  k0 = gamma invstd, k1 = sum g / M, k2 = sum g xhat / M round
    to fp32, and dx = k0 (g - k1 - xhat k2) takes four more roundings: |d dx| <= |gamma invstd|
    (4u (|g| + |k1| + |xhat k2|) + bar_b / M + |xhat| bar_g / M + |k2| e_xhat) + 2u |dx|.
    g is dy masked by y_out > 0 (the last BatchNorm of a block and every downsample BatchNorm)
    or by the BatchNorm's own ReLU, fma(z, scale, shift) > 0 (every other BatchNorm): the
    float64 sign of z scale + shift is that fma's sign, so the reference masks exactly alike.
  * bn_act (step_cases.check_bn_act): y = relu(fma(x, s, b) + q), q = fma(r, rs, rb), r or 0:
    three roundings on the terms, so |d y| <= 4u (|x s| + |b| + |r rs| + |rb|) (|r| for an
    identity residual); where the float64 value is below minus that bar, y must be exactly 0.
  * bn_relu_maxpool: the fp32 activations relu(fma(z, s, b)) are recomputed exactly (`_fma32`),
    the pool restated with the kernel's rule (the first strictly greater value in (kh, kw)
    order) must give y and argidx bit for bit, and y is within one rounding, u y64, of the
    float64 pool (the maximum is 1-Lipschitz).
  * add_masked, im2col, nchw_to_nhwc: data movement and one fp32 add, bit-exact with torch.
  * Soft-argmax backward (fp32 NHWC) and colsum at C4's shape: step_cases._sabwd_ref_bar and
    _check_colsum.

CPU tests below show against numpy emulations of the kernels' arithmetic that each new bar holds for the kernel's order and rejects a plausible
mistake: M - 1 in k1 / k2, a reduce that ignores y_out, a reduce that drops the last partial CTA,
bn_act without the residual's affine, a pool that keeps the last maximum or skips the ReLU, and a
3xTF32 wgrad that loses a correction pass at the longest C4 run."""
import numpy as np
import pytest
import torch

from tests import step_cases as sc
from tests.step_cases import (C4_LAYERS_TF32X3, KPIX, ROWS_PER_THREAD, RUN_BLOCKS3, U, WGRAD_BAR, _bn_act_check,
                              _bn_act_ref_bar, _bn_bwd_ratios, _bn_bwd_ref_bar, _bn_stats64, _emul_mma, _guarded,
                              _tc_bar, _tf32_np, _tf32_wgrad_plan, _trunc_np)

gpu = pytest.mark.gpu

NB, HWB, JB, DB, HMB = 128, 256, 16, 64, 64      # one GPU's bench batch: 32 tuples x 4 views


def _wgrad_runs(layer, N=NB):
    return sc.tf32_wgrad_runs(layer, N)


def _wgrad_run(layer):
    return sc.tf32_wgrad_run(layer, NB)


def test_c4_layer_table_wgrad_runs():
    """The restated planner over C4_LAYERS_TF32X3 at N = 128: every run within the three-pass cap, and
    the bar of the longest run under 1e-4."""
    runs = [(c[0], _wgrad_run(c)) for c in C4_LAYERS_TF32X3]
    for name, r in runs:
        assert 0 < r <= RUN_BLOCKS3 * KPIX and r % KPIX == 0, (name, r)
    R = max(r for _, r in runs)
    print("longest C4 wgrad run: %d pixels (%s), bar %.2e" % (R, [n for n, r in runs if r == R], _tc_bar(WGRAD_BAR, R, 3)))
    assert _tc_bar(WGRAD_BAR, R, 3) <= 1e-4


# ------------------------------------------------------------------ emulations against the bars of step_cases
def _fma_np(x, s, b):
    return (x.astype(np.float64) * s + b).astype(np.float32)


def _emul_bn_bwd(dy, x, y_out, scale, shift, mean, invstd, gamma, relu, mistake=None):
    """bn_bwd_reduce_kernel, bn_bwd_coef_kernel and bn_bwd_apply_kernel in numpy fp32 for
    C4 <= 256 (one channel chunk, rpi = 256 / C4 row slots).  mistake: "m_minus_1" (M - 1 in k1
    and k2), "ignore_y_out" (the ReLU mask of z in place of y_out > 0), "drop_last_cta" (the
    reduce loses its last, partial CTA)"""
    f = np.float32
    M, C = x.shape
    rpi = max(256 // (C // 4), 1)
    per = rpi * ROWS_PER_THREAD
    ctas = -(-M // per)
    if y_out is not None and mistake != "ignore_y_out":
        keep = y_out > 0
    elif relu or mistake == "ignore_y_out":
        keep = _fma_np(x, scale, shift) > 0
    else:
        keep = np.ones_like(x, dtype=bool)
    g = np.where(keep, dy, f(0)).astype(f)
    xm = (x - mean).astype(f)
    t = ((g * xm).astype(f) * invstd).astype(f)
    pad = lambda a: np.concatenate([a, np.zeros((ctas * per - M, C), f)]).reshape(ctas, ROWS_PER_THREAD, rpi, C)
    gp, tp = pad(g), pad(t)
    a0 = np.zeros((ctas, rpi, C), f)
    a1 = np.zeros((ctas, rpi, C), f)
    for k in range(ROWS_PER_THREAD):                   # row r0 + k rpi + slot, in fp32
        a0 = (a0 + gp[:, k]).astype(f)
        a1 = (a1 + tp[:, k]).astype(f)
    if mistake == "drop_last_cta":
        a0, a1 = a0[:-1], a1[:-1]
    sg = a0.astype(np.float64).sum((0, 1))
    sgx = a1.astype(np.float64).sum((0, 1))
    Md = M - 1 if mistake == "m_minus_1" else M
    k0 = (gamma.astype(np.float64) * invstd).astype(f)
    k1, k2 = (sg / Md).astype(f), (sgx / Md).astype(f)
    inner = ((g - k1).astype(f) - ((xm * invstd).astype(f) * k2).astype(f)).astype(f)
    return (k0 * inner).astype(f), sgx.astype(f), sg.astype(f)


def _bn_bwd_case_np(M, C, seed, relu):
    """z with per-channel means, dy with per-channel means (gradients rarely centre), y_out"""
    rng = np.random.default_rng(seed)
    f = np.float32
    x = (rng.standard_normal((M, C)) * rng.uniform(0.2, 2.2, C) + rng.standard_normal(C) * 2).astype(f)
    dy = ((rng.standard_normal((M, C)) + rng.standard_normal(C) * 0.5) * 1e-4).astype(f)
    gamma = rng.uniform(0.5, 1.5, C).astype(f)
    beta = (rng.standard_normal(C) * 0.1).astype(f)
    mu, inv = _bn_stats64(torch.from_numpy(x))
    scale = (gamma * inv.numpy()).astype(f)
    shift = (beta - mu.numpy() * gamma * inv.numpy()).astype(f)
    y_out = None if relu else np.maximum(rng.standard_normal((M, C)), 0).astype(f)
    return x, dy, y_out, scale, shift, mu, inv, gamma


@pytest.mark.parametrize("mistake", ["m_minus_1", "ignore_y_out", "drop_last_cta"])
def test_bn_bwd_bars_hold_for_the_kernel_order_and_reject(mistake):
    """The fp32 emulation of the reduce / coef / apply kernels meets the dbeta, dgamma and dx bars
    in both mask forms; the named mistake misses one of them.  M - 1 and y_out at M = 8192 (the
    smallest M of the step, where k1 and k2 move most), the dropped CTA at a ragged M = 8169."""
    M, C = (8192 - 23, 64) if mistake == "drop_last_cta" else (8192, 64)
    worst_ok, worst_bad = 0.0, 0.0
    for relu in ((0,) if mistake == "ignore_y_out" else (0, 1)):
        x, dy, y_out, scale, shift, mu, inv, gamma = _bn_bwd_case_np(M, C, 5 + relu, relu)
        mean, invstd = mu.float().numpy(), inv.float().numpy()
        keep = torch.from_numpy(y_out > 0 if y_out is not None else _fma_np(x, scale, shift) > 0)
        ref = _bn_bwd_ref_bar(torch.from_numpy(x), torch.from_numpy(dy), keep, torch.from_numpy(gamma), mu, inv)
        T = torch.from_numpy
        dx, dg, db = _emul_bn_bwd(dy, x, y_out, scale, shift, mean, invstd, gamma, relu)
        worst_ok = max(worst_ok, *_bn_bwd_ratios(T(db), T(dg), T(dx), ref))
        dx, dg, db = _emul_bn_bwd(dy, x, y_out, scale, shift, mean, invstd, gamma, relu, mistake)
        worst_bad = max(worst_bad, *_bn_bwd_ratios(T(db), T(dg), T(dx), ref))
    print("emulated BatchNorm backward: worst err / bar %.3f; %s: %.3g" % (worst_ok, mistake, worst_bad))
    assert worst_ok <= 1.0
    assert worst_bad > 2.0


def test_bn_act_bar_rejects_a_residual_without_its_affine():
    """The fp32 emulation of bn_act (residual with the downsample BatchNorm's affine) meets the
    bar with its exact zeros; adding the raw residual misses it."""
    rng = np.random.default_rng(9)
    f = np.float32
    M, C = 4096, 64
    x = (rng.standard_normal((M, C)) * 2 + 0.3).astype(f)
    r = (rng.standard_normal((M, C)) * 1.5 - 0.2).astype(f)
    s, b = rng.uniform(0.2, 1.5, C).astype(f), (rng.standard_normal(C) * 0.5).astype(f)
    rs, rb = rng.uniform(0.2, 1.5, C).astype(f), (rng.standard_normal(C) * 0.5).astype(f)
    ok = np.maximum((_fma_np(x, s, b) + _fma_np(r, rs, rb)).astype(f), 0)
    bad = np.maximum((_fma_np(x, s, b) + r).astype(f), 0)
    T = torch.from_numpy
    t, bar = _bn_act_ref_bar(T(x), T(s), T(b), T(r), T(rs), T(rb))
    r_ok, r_bad = _bn_act_check(T(ok), t, bar), _bn_act_check(T(bad), t, bar)
    print("emulated bn_act: %s; residual without its affine: %s" % (r_ok, r_bad))
    assert r_ok[0] <= 1.0 and r_ok[1:] == (0, 0)
    assert r_bad[0] > 10.0 and r_bad[1] > 0


def _fma32(x, s, b):
    """fp32 fma(x, s, b) as the kernel rounds it, broadcast over the last axis: x s is exact in
    double, and the TwoSum error of the double sum settles the one case in which rounding that
    sum to fp32 differs from rounding the exact value (a double on an fp32 midpoint)"""
    p = x.double() * s.double()
    bd = b.double().expand_as(p)
    s64 = p + bd
    a = s64 - bd
    e = (p - a) + (bd - (s64 - a))
    del p, bd, a
    f = s64.float()
    f64 = f.double()
    up = torch.nextafter(f, torch.tensor(float("inf"), device=f.device))
    dn = torch.nextafter(f, torch.tensor(float("-inf"), device=f.device))
    f = torch.where((s64 == (f64 + up.double()) / 2) & (e > 0), up, f)
    f = torch.where((s64 == (f64 + dn.double()) / 2) & (e < 0), dn, f)
    return f


def _pool_restated(z, s, b, last=False, relu=True):
    """bn_relu_maxpool_kernel in torch on the exact fp32 activations: (y, argidx) from the first
    strictly greater value in (kh, kw) order (last: the last of equal maxima), and the float64
    pool y64 of relu(z s + b)"""
    n, H, W, C = z.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    a32 = _fma32(z, s, b)
    a64 = z.double() * s.double() + b.double()
    if relu:
        a32, a64 = a32.clamp_min(0), a64.clamp_min(0)
    p32 = torch.full((n, H + 2, W + 2, C), float("-inf"), device=z.device)
    p64 = torch.full((n, H + 2, W + 2, C), float("-inf"), device=z.device, dtype=torch.float64)
    p32[:, 1:-1, 1:-1], p64[:, 1:-1, 1:-1] = a32, a64
    del a32, a64
    best = torch.full((n, Ho, Wo, C), float("-inf"), device=z.device)
    y64 = torch.full((n, Ho, Wo, C), float("-inf"), device=z.device, dtype=torch.float64)
    arg = torch.zeros((n, Ho, Wo, C), device=z.device, dtype=torch.uint8)
    for kh in range(3):
        for kw in range(3):
            v = p32[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2]
            take = (v >= best) & (v > float("-inf")) if last else v > best
            best = torch.where(take, v, best)
            arg = torch.where(take, torch.full_like(arg, kh * 3 + kw), arg)
            y64 = torch.maximum(y64, p64[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2])
    return best, arg, y64


def _pool_errors(y, arg, z, s, b):
    """(y bit-equal to the restated pool, argidx equal, worst |y - y64| / (u y64), windows whose
    maximum is a ReLU zero)"""
    yk, ak, y64 = _pool_restated(z, s, b)
    err = (y.double() - y64).abs()
    ratio = float((err / (U * y64)).nan_to_num(0.0, posinf=float("inf")).max()) if bool((err > 0).any()) else 0.0
    return (torch.equal(y.view(torch.int32), yk.view(torch.int32)), torch.equal(arg, ak), ratio,
            int((y64 == 0).sum()))


def test_pool_restatement_rejects_the_last_maximum_and_a_missing_relu():
    """A numpy emulation of bn_relu_maxpool on dyadic inputs (many equal maxima) and on random
    fp32 inputs matches the restatement bit for bit within u y64; keeping the last of equal
    maxima fails the argidx check, skipping the ReLU fails the value check."""
    rng = np.random.default_rng(13)
    f = np.float32
    n, H, W, C = 2, 17, 16, 8
    for dyadic in (True, False):
        z = rng.standard_normal((n, H, W, C))
        z = (np.round(z * 8) / 8 if dyadic else z).astype(f)
        s = (np.round(rng.uniform(0.5, 1.5, C) * 16) / 16 if dyadic else rng.uniform(0.5, 1.5, C)).astype(f)
        b = (np.round(rng.standard_normal(C) * 0.3 * 16) / 16 if dyadic else rng.standard_normal(C) * 0.3).astype(f)
        T = torch.from_numpy
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        act = _fma_np(z, s, b)

        def emul(last, relu):
            a = np.maximum(act, 0) if relu else act
            y = np.full((n, Ho, Wo, C), -np.inf, f)
            ai = np.zeros((n, Ho, Wo, C), np.uint8)
            for oh in range(Ho):
                for ow in range(Wo):
                    for kh in range(3):
                        for kw in range(3):
                            ih, iw = 2 * oh - 1 + kh, 2 * ow - 1 + kw
                            if 0 <= ih < H and 0 <= iw < W:
                                v = a[:, ih, iw]
                                t = v >= y[:, oh, ow] if last else v > y[:, oh, ow]
                                y[:, oh, ow] = np.where(t, v, y[:, oh, ow])
                                ai[:, oh, ow] = np.where(t, kh * 3 + kw, ai[:, oh, ow])
            return T(y), T(ai)
        same, arg_ok, ratio, zeros = _pool_errors(*emul(False, True), T(z), T(s), T(b))
        assert same and arg_ok and ratio <= 1.0, (dyadic, same, arg_ok, ratio)
        if dyadic:
            assert zeros > 0
            assert not _pool_errors(*emul(True, True), T(z), T(s), T(b))[1]
        y_nr, a_nr = emul(False, False)
        r = _pool_errors(y_nr, a_nr, T(z), T(s), T(b))
        assert not r[0] and r[2] > 1.0
        print("pool emulation (%s): bit-equal, %d ReLU-zero maxima; without ReLU: err / bar %.3g"
              % ("dyadic" if dyadic else "random", zeros, r[2]))


def test_tf32_wgrad_bar_rejects_a_lost_correction_pass_at_the_longest_c4_run():
    """The wgrad product at the longest pixel run of C4_LAYERS_TF32X3 (R from the planner), with the
    toward-zero accumulation of test_gpu_tf32: 3xTF32 meets _tc_bar(WGRAD_BAR, R, 3); dropping
    the dout lo pass or the activation lo pass misses it."""
    R = max(_wgrad_run(c) for c in C4_LAYERS_TF32X3)
    rng = np.random.default_rng(17)
    co, ci = 128, 64
    a = (rng.standard_normal((co, R)) * 1e-3).astype(np.float32)         # dz^T
    b = np.maximum(rng.standard_normal((R, ci)), 0).astype(np.float32)    # relu(BN(z)) of the producer
    ah, bh = _tf32_np(a), _tf32_np(b)
    al, bl = _trunc_np(a - ah), _trunc_np(b - bh)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    e = lambda x: float(np.max(np.abs(x - ref)) / np.max(np.abs(ref)))
    full = e(_emul_mma([(al, bh), (ah, bl), (ah, bh)], R, True))
    no_alo = e(_emul_mma([(ah, bl), (ah, bh)], R, True))
    no_blo = e(_emul_mma([(al, bh), (ah, bh)], R, True))
    bar = _tc_bar(WGRAD_BAR, R, 3)
    print("R = %d: 3xTF32 %.2e, dout lo lost %.2e, activation lo lost %.2e, bar %.2e" % (R, full, no_alo, no_blo, bar))
    assert full <= bar
    assert min(no_alo, no_blo) > bar


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """After the module, drop its cached model and hand the allocator's reserve back to the
    device for the tests after it; report the module's peak allocation."""
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        torch.cuda.reset_peak_memory_stats()
    yield
    sc.release("c4_tf32x3")
    if torch.cuda.is_initialized():
        print("\n  tf32x3 step module: peak device allocation %.1f GB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


def _r50(dev):
    """the bench model (R50, J = 16, D = 64, 256 x 256) on net.Engine at precision 3, with
    FusedAdam over its parameters"""
    from epipolarpose_b200 import net
    m, opt = sc.bench_model(dev, "c4_tf32x3")
    assert type(m._engine()) is net.Engine and m._engine().precision == 3
    return m, opt


# ------------------------------------------------------------------ 1. convolutions at N = 128
@gpu
@pytest.mark.parametrize("layer", C4_LAYERS_TF32X3, ids=[c[0] for c in C4_LAYERS_TF32X3])
def test_tf32x3_conv_layers_vs_float64(dev, layer):
    """fprop (statistics into a zeroed buffer, or the bias for the final layer), dgrad (written,
    or added into the block's input gradient for a downsample) and wgrad (into a zeroed dW) at
    N = 128 with the step's operand mode, each against torch float64 within its bar; every
    output followed by a guard band, every kernel a three-pass instantiation."""
    sc.check_tf32x3_layer(dev, layer, NB)


@gpu
def test_tf32x3_stem_wgrad_through_flat_buffer(dev):
    """The stem's weight gradient as the engine forms it: images -> nchw_to_nhwc -> im2col (the
    patch matrix, K padded 147 -> 160), Engine._conv_wgrad(stem_col, col, dz, ..., None) into the
    step's flat buffer, then the stage's batched unpack.  Columns 147 .. 159 of the [64][160]
    gradient are exactly zero, and both it and the unpacked [64, 3, 7, 7] gradient match float64
    within _tc_bar(WGRAD_BAR, R, 3)."""
    from epipolarpose_b200 import net, ops
    m, _ = _r50(dev)
    eng = m._engine()
    eng.dev = dev
    N, H = NB, HWB
    H1 = H // 2
    kpad = eng.stem_kpad
    g = torch.Generator(device=dev).manual_seed(23)
    img = torch.randn(N, 3, H, H, device=dev, generator=g)
    x = torch.empty(N, H, H, 4, device=dev)
    ops.nchw_to_nhwc(img, x, N, 3, H, H, 4)
    del img
    col = torch.empty(N, H1, H1, kpad, device=dev)
    ops.im2col(x, col, N, H, H, 4, 3, 7, 7, 2, 3, H1, H1, kpad)
    del x
    dz = torch.randn(N, H1, H1, 64, device=dev, generator=g) * 1e-3
    grads = {k: torch.full_like(v, float("nan")) for k, v in m.named_parameters()}
    gs = eng._grad_state(grads)
    gs["flat"].zero_()
    eng._gs, eng._side = gs, None
    try:
        eng._conv_wgrad(eng.stem_col, col, dz, N, H1, H1, None)
        ops.pack_weight_batch(gs["batches"][net.stage_of("conv1")])
    finally:
        eng._gs = None
    torch.cuda.synchronize()
    flat = gs["dwp"]["conv1"].view(64, kpad)
    ref = torch.zeros(64, kpad, device=dev, dtype=torch.float64)
    step = 1 << 18
    cf, df = col.view(-1, kpad), dz.view(-1, 64)
    for r0 in range(0, cf.shape[0], step):
        ref += df[r0:r0 + step].double().t() @ cf[r0:r0 + step].double()
    R = _tf32_wgrad_plan(N * H1 * H1, kpad, 64, 1, 3)[0]
    bar = _tc_bar(WGRAD_BAR, R, 3)
    scale = float(ref.abs().max())
    e_flat = float((flat.double() - ref).abs().max()) / scale
    w = grads["conv1.weight"]
    ref_w = ref[:, :147].view(64, 7, 7, 3).permute(0, 3, 1, 2)        # [64][(r s c)] -> [64, 3, 7, 7]
    e_w = float((w.double() - ref_w).abs().max()) / scale               # NaN (not written) fails
    print("  stem wgrad through the flat buffer: run %d, [64][160] %.2e, unpacked %.2e, bar %.2e"
          % (R, e_flat, e_w, bar))
    assert bool((flat[:, 147:] == 0).all()), "K-pad columns of the stem gradient are not zero"
    assert e_flat <= bar and e_w <= bar


# ------------------------------------------------------------------ 2. the fp32 BatchNorm chain
# (M, C, mask) of every BatchNorm backward of the step: "y_out" for the last BatchNorm of a block
# and the downsample BatchNorms, "relu" for the stem, the inner BatchNorms and the deconvs'
BN_BWD = [(2097152, 64, "relu"), (524288, 64, "relu"), (524288, 128, "relu"), (524288, 256, "y_out"),
          (524288, 256, "relu"), (131072, 128, "relu"), (131072, 256, "relu"), (131072, 512, "y_out"),
          (32768, 256, "relu"), (32768, 512, "relu"), (32768, 1024, "y_out"), (8192, 512, "relu"),
          (8192, 2048, "y_out")]
# make_rowmap beyond the step: a ragged M (not a multiple of rpi x 64 rows), C4 not dividing 256,
# C4 above 256 with a partial second channel chunk
BN_EDGE = [(524288 - 23, 256, "y_out"), (131072 - 23, 96, "relu"), (131072 - 23, 160, "y_out"),
           (32768 - 23, 1152, "relu")]


@gpu
@pytest.mark.parametrize("M,C,mode", BN_BWD, ids=["%dx%d-%s" % c for c in BN_BWD])
def test_tf32x3_bn_bwd_vs_float64(dev, M, C, mode):
    """bn_bwd_reduce + bn_bwd_apply at every (M, C) and mask form of the step: dbeta, dgamma per
    channel and dx per element against float64, with a constant channel (invstd = 316), one
    huge gradient element and a fully masked channel beside ordinary ones."""
    sc.check_bn_bwd(dev, M, C, mode)


@gpu
@pytest.mark.parametrize("M,C,mode", BN_EDGE, ids=["%dx%d-%s" % c for c in BN_EDGE])
def test_tf32x3_bn_bwd_edge_shapes(dev, M, C, mode):
    sc.check_bn_bwd(dev, M, C, mode)


BN_ACT = [(524288, 256), (131072, 512), (32768, 1024), (8192, 2048)]


@gpu
@pytest.mark.parametrize("res", ["affine", "identity", "relu"])
@pytest.mark.parametrize("M,C", BN_ACT, ids=["%dx%d" % c for c in BN_ACT])
def test_tf32x3_bn_act_vs_float64(dev, M, C, res):
    """bn_act at every block output: the residual with the downsample BatchNorm's affine, the
    identity residual, and ReLU alone; within 4u of the terms, exact zeros below -bar."""
    sc.check_bn_act(dev, M, C, res)


@gpu
def test_tf32x3_bn_relu_maxpool_vs_float64(dev):
    """The stem's pool at 128 x 128 x 128 x 64 -> 64 x 64: y and argidx bit-equal with the
    restated kernel (first strictly greater value in (kh, kw) order over the exact fp32
    activations; ties at ReLU zeros are common), y within u y64 of the float64 pool."""
    from epipolarpose_b200 import ops
    N, H, C = NB, HWB // 2, 64
    Ho = H // 2
    g = torch.Generator(device=dev).manual_seed(29)
    z = torch.randn(N, H, H, C, device=dev, generator=g) * 2 + 0.1
    s = torch.rand(C, device=dev, generator=g) + 0.3
    b = torch.randn(C, device=dev, generator=g) * 0.5 - 0.6
    b[:4] = -20.0                                             # channels that are all ReLU zeros
    y = torch.full((N, Ho, Ho, C), float("nan"), device=dev)
    arg = torch.full((N, Ho, Ho, C), 255, device=dev, dtype=torch.uint8)
    ops.bn_relu_maxpool(z, s, b, y, arg, N, H, H, C)
    torch.cuda.synchronize()
    same = arg_ok = True
    worst, zeros = 0.0, 0
    for n0 in range(0, N, 16):
        sl = slice(n0, n0 + 16)
        e_same, e_arg, ratio, nz = _pool_errors(y[sl], arg[sl], z[sl], s, b)
        same, arg_ok = same and e_same, arg_ok and e_arg
        worst, zeros = max(worst, ratio), zeros + nz
    print("  bn_relu_maxpool: bit-equal %s, argidx %s, worst err / (u y64) %.3f, %d ReLU-zero maxima"
          % (same, arg_ok, worst, zeros))
    assert same and arg_ok and worst <= 1.0
    assert zeros > 0


ADD_MASKED = [(524288, 256), (131072, 512), (32768, 1024), (8192, 2048)]


@gpu
@pytest.mark.parametrize("M,C", ADD_MASKED, ids=["%dx%d" % c for c in ADD_MASKED])
def test_tf32x3_add_masked_bit_exact(dev, M, C):
    """add_masked (a block's input gradient: dgrad + where(block output > 0, incoming, 0)) at
    every identity block's output size, bit-exact with torch, a guard band untouched."""
    from epipolarpose_b200 import ops
    n = M * C
    g = torch.Generator(device=dev).manual_seed(C)
    a = torch.randn(n, device=dev, generator=g)
    b = torch.randn(n, device=dev, generator=g)
    mask = torch.relu(torch.randn(n, device=dev, generator=g))
    mask[::7] = -0.0
    a[::11] = -0.0
    out, guard = _guarded((n,), dev, float("nan"))
    guard.fill_(1234.5)
    ops.add_masked(a, b, mask, out, n)
    torch.cuda.synchronize()
    ref = a + torch.where(mask > 0, b, torch.zeros_like(b))
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))
    print("  add_masked %d elements bit-exact" % n)


@gpu
def test_tf32x3_im2col_bit_exact_at_stem(dev):
    """im2col of all 128 images of 256 x 256 (7 x 7 / 2, pad 3, NHWC pitch 4 with a poisoned pad
    channel) against F.unfold, bit for bit; the K-pad columns 147 .. 159 exactly zero."""
    import torch.nn.functional as F
    from epipolarpose_b200 import ops
    N, H, kpad = NB, HWB, 160
    H1 = H // 2
    g = torch.Generator(device=dev).manual_seed(31)
    x = torch.randn(N, H, H, 4, device=dev, generator=g)
    x[..., 3] = 1e30                                          # the pad channel is never read
    col = torch.full((N, H1, H1, kpad), float("nan"), device=dev)
    ops.im2col(x, col, N, H, H, 4, 3, 7, 7, 2, 3, H1, H1, kpad)
    torch.cuda.synchronize()
    for n0 in range(0, N, 16):
        u = F.unfold(x[n0:n0 + 16, ..., :3].permute(0, 3, 1, 2), 7, padding=3, stride=2)   # [n, (c r s), L]
        u = u.view(-1, 3, 49, H1 * H1).permute(0, 3, 2, 1).reshape(-1, H1, H1, 147)         # [n, L, (r s c)]
        c = col[n0:n0 + 16]
        assert torch.equal(c[..., :147].contiguous().view(torch.int32), u.contiguous().view(torch.int32)), n0
        assert bool((c[..., 147:].view(torch.int32) == 0).all()), "K-pad columns not zero"
    print("  im2col: %d images bit-exact, K pad %d" % (N, kpad))


@gpu
def test_tf32x3_nchw_to_nhwc_bit_exact(dev):
    """nchw_to_nhwc of the bench batch (128 x 3 x 256 x 256 -> pitch 4), bit-exact, the pad
    channel +0, a guard band untouched."""
    from epipolarpose_b200 import ops
    N, H = NB, HWB
    g = torch.Generator(device=dev).manual_seed(37)
    src = torch.randn(N, 3, H, H, device=dev, generator=g)
    dst, guard = _guarded((N, H, H, 4), dev, float("nan"))
    guard.fill_(1234.5)
    ops.nchw_to_nhwc(src, dst, N, 3, H, H, 4)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    assert torch.equal(dst[..., :3].contiguous().view(torch.int32), src.permute(0, 2, 3, 1).contiguous().view(torch.int32))
    assert bool((dst[..., 3].view(torch.int32) == 0).all())


@gpu
@pytest.mark.parametrize("M", [131072, 32768, 8192])
def test_tf32x3_bn_finalize_vs_float64(dev, M):
    """bn_finalize at the step's other M (the bench test covers 524288 and 2097152)"""
    sc.check_bn_finalize(dev, M)


# ------------------------------------------------------------------ 3. the fp32 head at C4's shape
@gpu
def test_tf32x3_softargmax_bwd_fp32_vs_float64(dev):
    """epb_softargmax_bwd (fp32 NHWC) at N = 128, J = 16, D = 64, 64 x 64"""
    sc._check_softargmax_bwd_fp32(dev, NB, JB, DB, HMB, HMB)


@gpu
@pytest.mark.parametrize("M", [NB * HMB * HMB, NB * HMB * HMB - 23], ids=["524288", "524265"])
def test_tf32x3_colsum_vs_float64(dev, M):
    """epb_colsum over M x 1024 (the final layer's bias gradient; 524265 leaves a partial last CTA)"""
    sc._check_colsum(dev, M, JB * DB)


# ------------------------------------------------------------------ 4. weights and optimiser on the fp32 engine
@gpu
def test_tf32x3_pack_weight_batch_bit_exact_on_model_jobs(dev):
    """pack_weight_batch on net.Engine's own jobs for R50 / J16 / D64 (every layer's fprop and
    dgrad operands, the stem's [64][160] patch-matrix operand, the per-stage unpacks of the
    packed weight gradients), bit-exact with the CPU emulation"""
    sc._check_pack_weight_batch(dev, _r50(dev)[0])


@gpu
def test_tf32x3_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over the tf32x3 model's flat parameter buffer: steps 1, 2 and 1000"""
    sc._check_fused_adam(dev, *_r50(dev))
