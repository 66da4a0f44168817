"""The C5 training step (R101, 384 x 384, J = 17, D = 96; bench.py --workload c5) against float64
kernel by kernel at its own sizes.  tests/test_step_coverage.py gates the C5 step on these tests.

C5 runs code C4 does not.  J D = 1632 is not a whole number of 64-channel blocks, so the head's
backward leaves the split path (Engine16.takes_logit_sink() is False): the fp32 NHWC soft-argmax
backward, epb_colsum for the bias gradient, and the 3xTF32 weight and data gradients of the final
layer (epb_conv_wgrad with the last deconv's BatchNorm + ReLU applied on load, epb_conv_fprop with
K = 1632).  The final conv16 forward ends its 128-wide tiles in a 96-column tail; the shared
kernels run at other geometry (soft-argmax forward with 408 threads, M = 2359296 at the stem,
n = 3264 in the joint loss, J = 17 in the geometry, R101's jobs and 53.4M parameters).

Every reference is torch float64 on the device (or oracle/restate for the geometry), computed
from the exact values the kernel read, in chunks of at most 8 images.  Bars (u = 2^-24):

  * Shared kernels: the bars of the C4 tests, with C5's planner values (tests/step_cases.py).
    conv16 weight gradients: wgrad16's pixel splits (`_wgrad16_plan`, wgrad16.cu) leave each CTA
    a run of R = tiles_per_split x 64 pixels, so the bar is _tc_bar(WGRAD16_BASE, R, 3) (wgmma
    accumulates toward zero); WGRAD16_BASE = 2e-4 is the C4 contract.
  * Soft-argmax backward, fp32 NHWC: step_cases._sabwd_ref_bar.
  * epb_colsum: step_cases._check_colsum.
  * 3xTF32 final-layer weight gradient: _tc_bar(WGRAD_BAR, R, 3) with R the pixel run of one CTA
    from the TF32 wgrad planner (`_tf32_wgrad_plan`, conv_tc_wgrad.cu launch_wgrad).  Before the
    planner capped R, C5's final layer ran 5 splits of R = 117984 pixels: a bar of 2.0e-3, which
    a lost 3xTF32 correction pass (~2e-4 .. 3e-4) meets; the measured error was 9.4e-4.  With
    the cap (R <= 184 x 32 = 5888 for three passes) it runs 101 splits of 5856 pixels, the bar is
    9.8e-5 and the measured error 4.9e-5.  The C5 step at 8 tuples took 73.1 .. 73.2 ms with the
    cap and 73.3 .. 74.0 ms without (three alternating runs each); the default workload, which
    does not call this kernel, 65.6 and 65.7 ms.  Measured on one H100 80GB HBM3 at a 700 W
    power limit.
  * 3xTF32 data gradient, K = 1632: _tc_bar(FPROP_BAR, 1632, 3) = 2.7e-5.
  * conv16 final forward (K = 256 + bias): 5e-5 of max|ref|, the split suite's bar.

CPU tests below check the restated planners (step_cases) and show against numpy emulations that
the soft-argmax-backward bar rejects s_bar without the +1/2 shift, the colsum bar a dropped last
partial CTA, and the plan-derived TF32 wgrad bar a lost correction pass at C5's run length."""
import numpy as np
import pytest
import torch

from tests import step_cases as sc
from tests.step_cases import (C5_LAYERS, FPROP_BAR, KPIX, RUN_BLOCKS3, U, WGRAD_BAR, _check_colsum,
                              _check_softargmax_bwd_fp32, _emul_mma, _sabwd_ref_bar, _split_dev, _tc_bar,
                              _tf32_np, _tf32_wgrad_plan, _trunc_np, _wgrad16_plan)

gpu = pytest.mark.gpu

N5, HW5, J5, D5, HM5 = 64, 384, 17, 96, 96        # one GPU's C5 batch: 16 tuples x 4 views
M5 = N5 * HM5 * HM5                                # pixels of the last deconv / final layer: 589824
WGRAD16_BASE = 2e-4


# ------------------------------------------------------------------ the restated planners
def test_tf32_wgrad_planner_caps_the_accumulation_run():
    """The restated planner: every CTA's pixel run R stays within 184 x 32 (three passes) or
    3 x that (one pass), so _tc_bar(WGRAD_BAR, R, passes) <= 1e-4, at C4 and C5 layer shapes and
    at sizes around the cap; below the cap the plan is the uncapped one.  C5's final layer
    without the cap runs 5 splits of 117984 pixels (bar 2.0e-3)."""
    rows_old, splits_old, tiles = _tf32_wgrad_plan(M5, 256, 1632, 1, 3, cap=False)
    rows, splits, _ = _tf32_wgrad_plan(M5, 256, 1632, 1, 3)
    print("C5 final layer: %d tiles; uncapped %d splits x %d pixels (bar %.2e), capped %d x %d (bar %.2e)"
          % (tiles, splits_old, rows_old, _tc_bar(WGRAD_BAR, rows_old, 3), splits, rows, _tc_bar(WGRAD_BAR, rows, 3)))
    assert (tiles, splits_old, rows_old) == (26, 5, 117984)
    assert rows <= RUN_BLOCKS3 * KPIX and splits * rows >= M5 > (splits - 1) * rows
    # (M, Cin, Cout, T): C4 (N = 128, 256^2) and C5 (N = 64, 384^2) layers under tf32x3, and odd sizes
    shapes = [(128 * 64 * 64, 256, 1024, 1), (128 * 128 * 128, 192, 64, 1), (128 * 64 * 64, 64, 64, 9),
              (128 * 8 * 8, 2048, 256, 4), (M5, 256, 1632, 1), (64 * 192 * 192, 192, 64, 1),
              (64 * 96 * 96, 64, 256, 1), (64 * 12 * 12, 512, 512, 9), (64 * 48 * 48, 256, 256, 4)]
    shapes += [(m, 64, 64, 1) for m in (1, 31, 5888, 5889, 17664, 17665, 1 << 20)]
    for M, cin, cout, T in shapes:
        for ns in (1, 3):
            r, sp, _ = _tf32_wgrad_plan(M, cin, cout, T, ns)
            assert r <= RUN_BLOCKS3 * 3 // ns * KPIX and r % KPIX == 0 and (sp - 1) * r < M <= sp * r
            assert _tc_bar(WGRAD_BAR, r, ns) <= 1e-4
            if M <= RUN_BLOCKS3 * 3 // ns * KPIX:
                assert (r, sp) == _tf32_wgrad_plan(M, cin, cout, T, ns, cap=False)[:2]


# ------------------------------------------------------------------ bars shared by the CPU and GPU tests
def _colsum_bar(x64, rpi, ctas):
    S_ = x64.sum(0)
    return S_, 64 * U * x64.abs().sum(0) + (rpi + ctas) * 2.0 ** -53 * x64.abs().sum(0) + U * S_.abs()


def _emul_colsum(x, drop_last=False):
    """colsum_kernel for C >= 1024 (one row slot per CTA): per CTA 64 rows added in fp32, the CTA
    partials added in double, rounded to fp32; drop_last: the last (partial) CTA lost"""
    M, C = x.shape
    ctas = -(-M // 64)
    pad = np.zeros((ctas * 64, C), np.float32)
    pad[:M] = x
    pad = pad.reshape(ctas, 64, C)
    acc = np.zeros((ctas, C), np.float32)
    for k in range(64):
        acc = (acc + pad[:, k]).astype(np.float32)
    if drop_last:
        acc = acc[:-1]
    return acc.astype(np.float64).sum(0).astype(np.float32), ctas


def test_colsum_bar_rejects_a_dropped_partial_cta():
    """M = 64 x 200 + 23 rows of 1632 columns: the emulated colsum meets the bar, and with the
    last, partial CTA (23 rows) dropped misses it in almost every column (a column whose 23
    dropped values happen to sum to nearly zero can stay inside)."""
    rng = np.random.default_rng(3)
    M, C = 64 * 200 + 23, 1632
    x = rng.standard_normal((M, C)).astype(np.float32)
    x64 = torch.from_numpy(x).double()
    ok, ctas = _emul_colsum(x)
    bad, _ = _emul_colsum(x, drop_last=True)
    ref, bar = _colsum_bar(x64, 1, ctas)
    r_ok = float(((torch.from_numpy(ok).double() - ref).abs() / bar).max())
    r_bad = ((torch.from_numpy(bad).double() - ref).abs() / bar)
    print("colsum emulation: worst err / bar %.3f; last CTA dropped: median err / bar %.1f, %.4f of the "
          "columns over the bar" % (r_ok, float(r_bad.median()), float((r_bad > 1).double().mean())))
    assert r_ok <= 1.0
    assert float((r_bad > 1.0).double().mean()) > 0.95 and float(r_bad.median()) > 10


def _emul_sabwd(v, coords, lse, dco, H, W, D, shift=0.5):
    """softargmax_bwd_nhwc in numpy fp32 for logits v [B, H, W, J, D]; shift: the 1/2 added to
    the forward coords in s_bar"""
    f = np.float32
    B, J = v.shape[0], v.shape[3]
    l = lse.reshape(B, J, 2).astype(f)
    m, inv = l[..., 0].reshape(B, 1, 1, J, 1), l[..., 1].reshape(B, 1, 1, J, 1)
    dc = dco.reshape(B, J, 3).astype(f)
    gx, gy, gz = (dc[..., 0] / f(W)).astype(f), (dc[..., 1] / f(H)).astype(f), (dc[..., 2] / f(D)).astype(f)
    cr = coords.reshape(B, J, 3).astype(f)
    sh = f(shift)
    sbar = ((gx * (cr[..., 0] + sh).astype(f)).astype(f) * f(W)).astype(f)
    sbar = (sbar + ((gy * (cr[..., 1] + sh).astype(f)).astype(f) * f(H)).astype(f)).astype(f)
    sbar = (sbar + ((gz * (cr[..., 2] + sh).astype(f)).astype(f) * f(D)).astype(f)).astype(f)
    x = np.arange(W, dtype=f).reshape(1, 1, W, 1, 1)
    y = np.arange(H, dtype=f).reshape(1, H, 1, 1, 1)
    z0 = (np.arange(D) // 4 * 4).astype(f).reshape(1, 1, 1, 1, D)
    k = (np.arange(D) % 4).astype(f).reshape(1, 1, 1, 1, D)
    G = lambda a: a.reshape(B, 1, 1, J, 1)
    s0 = ((G(gx) * x).astype(f) + (G(gy) * y).astype(f)).astype(f)
    s0 = (s0 + (G(gz) * z0).astype(f)).astype(f)
    s0 = (s0 - G(sbar)).astype(f)
    s = np.where(k == 0, s0, (s0 + (k * G(gz)).astype(f)).astype(f)).astype(f)
    e = np.exp((v - m).astype(f)).astype(f)
    return ((e * inv).astype(f) * s).astype(f)


def test_softargmax_bwd_bar_rejects_sbar_without_half_shift():
    """2 images, J = 17, D = 96, 12 x 12, logits x 3: the fp32 emulation of softargmax_bwd_nhwc
    meets the per-element bar; with s_bar taken from the coords without the +1/2 it misses it."""
    rng = np.random.default_rng(5)
    B, H, W, J, D = 2, 12, 12, J5, D5
    v = (rng.standard_normal((B, H, W, J, D)) * 3).astype(np.float32)
    dco = rng.standard_normal((B, J * 3)).astype(np.float32)
    v64 = torch.from_numpy(v).double()
    m = v64.amax((1, 2, 4), keepdim=True)
    ex = torch.exp(v64 - m)
    tot = ex.sum((1, 2, 4), keepdim=True)
    p = ex / tot
    c = [(p.sum((1, 4)) * torch.arange(W).double().view(1, W, 1)).sum(1) / W - 0.5,
         (p.sum((2, 4)) * torch.arange(H).double().view(1, H, 1)).sum(1) / H - 0.5,
         (p.sum((1, 2)) * torch.arange(D).double().view(1, 1, D)).sum(2) / D - 0.5]
    coords = torch.stack(c, -1).float().numpy()                       # [B, J, 3], one rounding
    lse = torch.stack([m.view(B, J), 1 / tot.view(B, J)], -1).float().numpy()
    dl, e = _sabwd_ref_bar(v64, torch.from_numpy(coords), torch.from_numpy(lse), torch.from_numpy(dco), H, W, D)
    ratio = lambda out: float(((torch.from_numpy(out).double() - dl).abs() / (e + 1e-300)).max())
    r_ok = ratio(_emul_sabwd(v, coords, lse, dco, H, W, D))
    r_bad = ratio(_emul_sabwd(v, coords, lse, dco, H, W, D, shift=0.0))
    print("softargmax bwd emulation: worst err / bar %.3f; s_bar without +1/2: %.3g" % (r_ok, r_bad))
    assert r_ok <= 1.0
    assert r_bad > 10.0


def test_tf32_wgrad_plan_bar_rejects_a_lost_correction_pass():
    """The final layer's wgrad product at C5's capped run length (R = _tf32_wgrad_plan), with the
    toward-zero accumulation of test_gpu_tf32: 3xTF32 meets _tc_bar(WGRAD_BAR, R, 3); dropping
    the dout lo pass misses it.  The uncapped run's bar (R = 117984) would not reject it."""
    R = _tf32_wgrad_plan(M5, 256, 1632, 1, 3)[0]
    R_old = _tf32_wgrad_plan(M5, 256, 1632, 1, 3, cap=False)[0]
    rng = np.random.default_rng(11)
    co, ci = 128, 64
    a = (rng.standard_normal((co, R)) * 1e-3).astype(np.float32)         # dout^T: logit gradients
    b = np.maximum(rng.standard_normal((R, ci)), 0).astype(np.float32)    # relu(BN(z)) of the last deconv
    ah, bh = _tf32_np(a), _tf32_np(b)
    al, bl = _trunc_np(a - ah), _trunc_np(b - bh)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    e = lambda x: float(np.max(np.abs(x - ref)) / np.max(np.abs(ref)))
    full = e(_emul_mma([(al, bh), (ah, bl), (ah, bh)], R, True))
    no_alo = e(_emul_mma([(ah, bl), (ah, bh)], R, True))
    bar, bar_old = _tc_bar(WGRAD_BAR, R, 3), _tc_bar(WGRAD_BAR, R_old, 3)
    print("R = %d: 3xTF32 %.2e, dout lo pass lost %.2e, bar %.2e (uncapped R = %d: bar %.2e)"
          % (R, full, no_alo, bar, R_old, bar_old))
    assert full <= bar
    assert no_alo > bar
    assert no_alo < bar_old


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """The C5 references hold tens of GB at their peak: after the module, drop its cached model
    and conv outputs and hand the allocator's reserve back to the device for the tests after it."""
    yield
    sc.release("c5_")


# ------------------------------------------------------------------ 1. the head at C5 sizes
def _final_conv():
    from epipolarpose_b200 import net
    return net.Conv("final_layer", "conv", 256, J5 * D5, 1, 1, 0, 0)


@gpu
def test_c5_final_conv16_fprop_vs_float64(dev):
    """conv16 forward of the final layer (256 -> 1632 with bias, N = 64, 96 x 96: 12 tiles of 128
    columns and a 96-column tail) against float64 on the values the planes hold, within 5e-5 of
    max|ref|.  Run into two buffers pre-filled with different NaN sentinels and followed by a guard
    band: every element written, identically, and nothing past the end."""
    from epipolarpose_b200 import ops
    conv = _final_conv()
    C = conv.cout
    g = torch.Generator(device=dev).manual_seed(91)
    x, x_sc, xv = _split_dev(torch.relu(torch.randn(N5, HM5, HM5, 256, device=dev, generator=g)))
    w = torch.randn(C, 256, 1, 1, device=dev, generator=g) * (2.0 / 256) ** 0.5
    wf32, _ = conv.pack(ops, w)
    wf, wf_sc, wfv = _split_dev(wf32)
    bias = torch.randn(C, device=dev, generator=g) * 0.5
    n, guard = M5 * C, 4096
    outs = []
    for bits in (0x7FC0DEAD, 0x7FC0BEEF):
        buf = torch.full((n + guard,), bits, device=dev, dtype=torch.int32).view(torch.float32)
        for gm in conv.fprop_geoms(ops, N5, HM5, HM5, 3):
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv16_fprop(gm, x, x_sc, wf, wf_sc, buf[:n].view(N5, HM5, HM5, C), bias, None)
        outs.append(buf)
    torch.cuda.synchronize()
    a, b = (o.view(torch.int32) for o in outs)
    assert bool((a[n:] == 0x7FC0DEAD).all()) and bool((b[n:] == 0x7FC0BEEF).all()), "guard band written"
    assert torch.equal(a[:n], b[:n]), "output depends on the prior contents (an element not written)"
    out = outs[0][:n].view(M5, C)
    wq = wfv.view(C, 256).t().contiguous()
    worst, rmax = 0.0, 0.0
    for r0 in range(0, M5, 8 * HM5 * HM5):
        ref = xv.view(M5, 256)[r0:r0 + 8 * HM5 * HM5] @ wq + bias.double()
        worst = max(worst, float((out[r0:r0 + ref.shape[0]].double() - ref).abs().max()))
        tail = max(0.0, float((out[r0:r0 + ref.shape[0], 1536:].double() - ref[:, 1536:]).abs().max()))
        rmax = max(rmax, float(ref.abs().max()))
    e = worst / rmax
    print("  C5 final conv16 fprop 256 -> 1632: err %.2e (tail columns %.2e of max|ref|), bar 5.0e-05" % (e, tail / rmax))
    assert e <= 5e-5


@gpu
@pytest.mark.parametrize("kind", ["randn3", "peaks60", "constant"])
def test_c5_softargmax_fwd_vs_float64(dev, kind):
    """N = 64, J = 17, D = 96, 96 x 96 NHWC (3.85 GB of logits): 408 threads per CTA, the bar of
    test_softargmax_fwd_vs_float64_at_bench_shape with _nhwc_geometry(64, 17, 96, 96, 96)."""
    sc._check_softargmax_fwd(dev, kind, N5, J5, D5, HM5, HM5)


@gpu
def test_c5_softargmax_bwd_fp32_vs_float64(dev):
    """epb_softargmax_bwd (fp32 NHWC, the path C5's head takes) at N = 64, J = 17, D = 96,
    96 x 96: every element of the logit gradient against float64 p (s - s_bar) within its bar."""
    _check_softargmax_bwd_fp32(dev, N5, J5, D5, HM5, HM5)


@gpu
@pytest.mark.parametrize("M", [M5, M5 - 23], ids=["589824", "589801"])
def test_c5_colsum_vs_float64(dev, M):
    """epb_colsum over M x 1632 (the bias gradient of C5's final layer; M5 - 23 leaves a partial
    last CTA of 41 rows) against float64 column sums within the module's bar; a second run
    within one fp32 ulp."""
    _check_colsum(dev, M, J5 * D5)


@gpu
def test_c5_final_tf32_wgrad_vs_float64(dev):
    """3xTF32 weight gradient of the final layer as the C5 step runs it: the raw last-deconv
    output z [589824, 256] with its BatchNorm scale / shift and ReLU applied on load, the fp32
    logit gradient [589824, 1632], dW from zero.  Against float64 of relu(fp32 fma(z, sc, sh))
    summed over image chunks, within _tc_bar(WGRAD_BAR, R, 3), R the planner's pixel run."""
    from epipolarpose_b200 import ops
    conv = _final_conv()
    C = conv.cout
    g = torch.Generator(device=dev).manual_seed(97)
    z = torch.randn(N5, HM5, HM5, 256, device=dev, generator=g) * 2 + 0.5
    sc = torch.rand(256, device=dev, generator=g) + 0.25
    sh = torch.randn(256, device=dev, generator=g) * 0.5
    dout = torch.randn(N5, HM5, HM5, C, device=dev, generator=g) * 1e-4
    dw = torch.zeros(C * 256, device=dev)
    for gm in conv.fprop_geoms(ops, N5, HM5, HM5, 3):
        gm.in_relu, gm.accumulate = 1, 0
        ops.conv_wgrad(gm, z, dout, dw, sc, sh)
    torch.cuda.synchronize()
    ref = torch.zeros(C, 256, device=dev, dtype=torch.float64)
    step = 8 * HM5 * HM5
    for r0 in range(0, M5, step):
        a = torch.relu((z.view(M5, 256)[r0:r0 + step].double() * sc.double() + sh.double()).float()).double()
        ref += dout.view(M5, C)[r0:r0 + step].double().t() @ a
    R, splits, tiles = _tf32_wgrad_plan(M5, 256, C, 1, 3)
    bar = _tc_bar(WGRAD_BAR, R, 3)
    e = float((dw.view(C, 256).double() - ref).abs().max() / ref.abs().max())
    print("  C5 final 3xTF32 wgrad: %d tiles x %d splits, run %d pixels: err %.3e, bar %.3e" % (tiles, splits, R, e, bar))
    assert e <= bar


@gpu
def test_c5_final_tf32_dgrad_vs_float64(dev):
    """3xTF32 data gradient of the final layer (conv_fprop on the dgrad geometry, K = 1632) from
    the fp32 logit gradient: dIn [589824, 256] against float64 within _tc_bar(FPROP_BAR, 1632, 3)."""
    from epipolarpose_b200 import ops
    conv = _final_conv()
    C = conv.cout
    g = torch.Generator(device=dev).manual_seed(99)
    w = torch.randn(C, 256, 1, 1, device=dev, generator=g) * (2.0 / 256) ** 0.5
    _, wd = conv.pack(ops, w)
    dout = torch.randn(N5, HM5, HM5, C, device=dev, generator=g) * 1e-4
    din = torch.full((N5, HM5, HM5, 256), float("nan"), device=dev)
    for gm in conv.dgrad_geoms(ops, N5, HM5, HM5, 3):
        gm.in_relu, gm.accumulate = 0, 0
        ops.conv_fprop(gm, dout, wd, din, None, None, None, None)
    torch.cuda.synchronize()
    w64 = w.double().view(C, 256)
    step = 8 * HM5 * HM5
    worst, rmax = 0.0, 0.0
    for r0 in range(0, M5, step):
        ref = dout.view(M5, C)[r0:r0 + step].double() @ w64
        worst = max(worst, float((din.view(M5, 256)[r0:r0 + step].double() - ref).abs().max()))
        rmax = max(rmax, float(ref.abs().max()))
    bar = _tc_bar(FPROP_BAR, C, 3)
    print("  C5 final 3xTF32 dgrad K = %d: err %.3e, bar %.3e" % (C, worst / rmax, bar))
    assert worst / rmax <= bar          # NaN anywhere fails too


@gpu
@pytest.mark.parametrize("kind,norm", [(2, 0), (1, 0), (1, 1), (2, 1)], ids=["smoothl1", "l1", "l1_norm", "smoothl1_norm"])
def test_c5_jointloss_vs_float64(dev, kind, norm):
    """epb_jointloss_fwd_bwd at N = 64, J = 17 (n = 3264, not a multiple of 1024)."""
    sc._check_jointloss(dev, kind, norm, N5, J5)


# ------------------------------------------------------------------ 2. shared kernels at C5 sizes
@gpu
@pytest.mark.parametrize("layer", C5_LAYERS, ids=[c[0] for c in C5_LAYERS])
def test_c5_conv16_layers_vs_torch_float64(dev, layer):
    """conv16 fprop (statistics), dgrad and wgrad at N = 64 against torch float64 (the bars of
    test_conv16_bench_layer_shapes_vs_torch_float64); the wgrad bar from wgrad16's planner."""
    from epipolarpose_b200 import net, ops
    name, kind, cin, cout, k, s, p, hw = layer
    conv = net.Conv("t", kind, cin, cout, k, s, p, 0)
    plans = [_wgrad16_plan(gm) for gm in conv.fprop_geoms(ops, N5, hw, hw, 3) if gm is not None]
    R = max(r for r, _ in plans)
    bar = _tc_bar(WGRAD16_BASE, R, 3)
    e = sc._check_conv16_layer(dev, layer, N5, bar)
    print("  C5 %-18s fprop %.2e dgrad %.2e wgrad %.2e (splits %s, run %d pixels, bar %.2e)"
          % (name, e[0], e[1], e[2], [sp for _, sp in plans], R, bar))


C5_STATS = [("c5_stem_col_192_64", "conv", 192, 64, 1, 1, 0, N5, 192, [(0, 0)]),
            ("c5_l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, N5, 96, [(0, 0)])]


@gpu
@pytest.mark.parametrize("case", C5_STATS, ids=[c[0] for c in C5_STATS])
def test_c5_conv16_stats_vs_float64(dev, case):
    """conv16 BatchNorm statistics at M = 2359296 (stem) and 589824 (layer1)."""
    sc.check_conv16_stats(dev, case)


@gpu
@pytest.mark.parametrize("M", [2359296, 589824, 9216])
def test_c5_bn_finalize_scale_vs_float64(dev, M):
    sc.check_bn_finalize_scale(dev, M)


@gpu
@pytest.mark.parametrize("M", [589824, 147456, 36864, 9216])
def test_c5_bn_finalize_vs_float64(dev, M):
    """the downsample layers' BatchNorm of R101 at 384"""
    sc.check_bn_finalize(dev, M)


@gpu
@pytest.mark.parametrize("res", ["none", "split", "affine"])
def test_c5_bn_act_split_vs_float64(dev, res):
    """layer1's conv16 output (589824 x 256) -> bn_finalize_scale -> bn_act_split"""
    sc._check_bn_act_split(dev, res, C5_STATS[1])


@gpu
def test_c5_bn_relu_maxpool_split_vs_float64(dev):
    """the stem's conv16 output (64 x 192 x 192 x 64) -> bn_relu_maxpool_split -> 96 x 96"""
    sc._check_bn_relu_maxpool_split(dev, C5_STATS[0])


@gpu
def test_c5_maxpool_bwd_vs_float64(dev):
    sc._check_maxpool_bwd(dev, N5, 192)


C5_BWD = [(2359296, 64), (589824, 256), (9216, 2048)]


@gpu
@pytest.mark.parametrize("mode", ["relu", "bits_inplace"])
@pytest.mark.parametrize("M,C", C5_BWD, ids=["%dx%d" % s for s in C5_BWD])
def test_c5_bn_bwd_split_vs_float64(dev, M, C, mode):
    sc.check_bn_bwd_split(dev, M, C, mode)


@gpu
def test_c5_im2col_split_bit_exact_at_stem(dev):
    """the stem's patch matrix of 64 images of 384 x 384"""
    sc._check_im2col_split(dev, sc.bench_model(dev, "c5")[0]._engine().stem_kpad, N5, HW5)


@gpu
def test_c5_split16_batch_bit_exact_on_model_jobs(dev):
    """split16_batch on the jobs the f16x3 engine builds for R101 / J17 / D96 (1632-channel head)"""
    sc._check_split16_batch(dev, *sc.bench_model(dev, "c5"))


@gpu
def test_c5_pack_weight_batch_bit_exact_on_model_jobs(dev):
    sc._check_pack_weight_batch(dev, sc.bench_model(dev, "c5")[0])


@gpu
def test_c5_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over R101 / J17 / D96's flat parameter buffer: steps 1, 2 and 1000"""
    sc._check_fused_adam(dev, *sc.bench_model(dev, "c5"))


@gpu
def test_c5_selfsup_geometry_j17(dev):
    """patch_to_image -> triangulate (iterative) -> project_labels at 16 tuples x 4 views with
    J = 17, against oracle/restate on each stage's own input (the bars of
    test_c3_selfsup_chain_64_images)."""
    import lib.utils.img_utils as iu
    from oracle import restate
    from tests.golden_inputs import _ring_meta
    tuples, J = 16, J5
    B = 4 * tuples
    meta_np = _ring_meta(tuples, 1075)
    meta = {k: torch.from_numpy(v) for k, v in meta_np.items()}
    rng = np.random.default_rng(77)
    cg = torch.from_numpy((rng.uniform(-0.3, 0.3, (B, J * 3))).astype(np.float32)).to(dev)
    kps = iu.patch_to_image_device(cg, meta)
    X = iu.triangulate_device(kps, meta, "iterative")
    label, weight = iu.labels_from_global_coords_device(X, meta)
    _, _, _, kps_ref = restate.self_supervision(cg.cpu().numpy(), meta_np, "iterative")
    e_k = float(np.max(np.abs(kps.cpu().numpy() - kps_ref)))
    X_ref = restate.triangulate_batch(kps.cpu().numpy(), meta_np["projection_matrix"], "iterative")
    e_x = float(np.max(np.abs(X.cpu().numpy() - X_ref)))
    lab_ref, w_ref = restate.labels_from_global_coords(X.cpu().numpy(), meta_np)
    e_l = float(np.max(np.abs(label.cpu().numpy() - lab_ref)))
    print("  C5 geometry J17: kps %.2e px (bar 5e-3), X %.2e mm (bar 1e-4), labels %.2e (bar 2e-5)" % (e_k, e_x, e_l))
    assert X.shape[1] == J
    assert e_k <= 5e-3 and e_x <= 1e-4 and e_l <= 2e-5
    assert np.array_equal(weight.cpu().numpy(), w_ref)
