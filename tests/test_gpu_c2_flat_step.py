"""The C2(ii) training step (MODEL.VOLUME: false; R50, 256 x 256, J = 17, D = 64, N = 32, split fp16)
against float64 kernel by kernel at its own sizes.  tests/test_step_coverage.py gates the step on
these tests.

The step: forward to the 2-D heat-maps [32, 17, 64, 64] and depth_fc's output [32, 17 x 64],
HeatmapJointLoss(17, kind="l1") (heat-map MSE against Gaussian sigma = 2 targets with visibility
weights, plus an L1 term on the depth_fc output), backward, FusedAdam.  It runs code the C4 step
does not:

  * epb_avgpool_split (the trunk's [32, 8, 8, 2048] planes -> the depth_fc input) and
    epb_avgpool_bwd (depth_fc's data gradient added into the trunk gradient, accumulate = 1).
  * depth_fc, a 1 x 1 conv 2048 -> 1088 over 32 rows on the 3xTF32 kernels: forward (one M tile
    with 32 valid rows, K = 2048, a 64-column N tail), data gradient (K = 1088), weight gradient
    (one 32-pixel KPIX block per CTA, 144 tiles), epb_colsum (32 x 1088) for its bias.
  * J = 17 gives the final layer cout_p = 20, not a whole 64-channel block, so Engine16 takes the
    fp32 head backward: epb_colsum (131072 x 20), the weight gradient with the last deconv's
    BatchNorm + ReLU applied on load and the data gradient with K = 20.  20 is not a multiple of
    32, so epb_conv_wgrad / epb_conv_fprop dispatch these two to the fp32 CUDA-core kernels, not
    to 3xTF32 (conv.cu, epb_conv_tc_supported); the test holds them to the 3xTF32 bars and
    shows which kernels run from the restated dispatch predicate and from bit identity with the
    CUDA-core kernels, without a profiler session.
  * epb_heatmap_joint_loss at (32, 17, 64, 64) with n = 34816 joint elements: 1056 CTAs (the
    grid cap), three tail trips per thread, the joint part in the last CTA alone.
  * epb_nhwc_to_nchw / epb_nchw_to_nhwc: the heat-maps out of, and their gradient into, the
    engine's 20-channel NHWC layout.
  * The shared split-path kernels at N = 32: fewer tiles per layer, other wgrad16 split plans and
    other BatchNorm M (stem 524288; 131072 / 32768 / 8192 / 2048 for the trunk and deconvs).

Every reference is torch float64 on the device (numpy for the bit-exact restatements).  Bars
(u = 2^-24):

  * Shared kernels: the bars of the C4 tests with C2's planner values (tests/step_cases.py);
    conv16 weight gradients _tc_bar(WGRAD16_BASE, R, 3), R the pixel run of one CTA from
    wgrad16's planner (`_wgrad16_plan`), as in test_gpu_c5_step.
  * avgpool_split: step_cases._check_avgpool_split, from the kernel's order (a sequential fp32
    sum of HW (hi + lo) pairs, x the power-of-two scale, / HW).
  * avgpool_bwd: bit-exact against fp32 dx + dy / HW (the same IEEE division and add, nothing
    to contract, no fast-math); the fp32 engine's avgpool forward within HW u mean|x|.
  * fp32-operand convs (step_cases.check_tf32x3_layer): fprop / dgrad _tc_bar(FPROP_BAR, K, 3):
    3.4e-5 at K = 2048, 2e-5 at K = 1088 and K = 20; wgrad _tc_bar(WGRAD_BAR, R, 3) with R from
    `_tf32_wgrad_plan`: 3e-5 at R = 32 (depth_fc); 3.4e-5 for the final layer, whose fp32
    CUDA-core kernels (fma chains, no TF32 operand rounding) stay far inside it: measured 4.6e-7
    (fprop), 1.9e-7 (dgrad) and 5.1e-7 .. 5.7e-7 (wgrad: atomics, so it varies) on one H100 80GB HBM3.
  * colsum: step_cases._check_colsum.
  * Heat-map loss: step_cases.hm_loss_ref_bar, from the kernel's partition (per-thread fp32
    partials over 7 + q roundings, q the trips, then double; dhm = gs wr d within 5u of itself;
    dx exact up to one rounding).

CPU tests below check the restated TF32 wgrad plan quoted above, and show against a numpy
emulation of the heat-map kernel's partition that its loss bar holds and rejects a dropped CTA
partial and a weight applied once instead of squared."""
import numpy as np
import pytest
import torch

from tests import step_cases as sc
from tests.step_cases import (C2_LAYERS, FPROP_BAR, HM_THREADS, WGRAD_BAR, _check_colsum, _split_dev, _tc_bar,
                              _tf32_wgrad_plan, _wgrad16_plan)

gpu = pytest.mark.gpu

N2, HW2, J2, D2, HM2 = 32, 256, 17, 64, 64        # one GPU's C2(ii) batch: 8 tuples x 4 views
M2 = N2 * HM2 * HM2                                # pixels of the last deconv / final layer: 131072
WGRAD16_BASE = 2e-4

# fp32-operand head layers (C4_LAYERS_TF32X3 rows): depth_fc over the pooled trunk (a materialised
# input), the final layer with the last deconv's BatchNorm + ReLU on load; both data gradients
# written (dpool is added into the trunk gradient by avgpool_bwd).  Whether the layer runs on the
# tensor cores: depth_fc 3xTF32; the final layer (20 channels) the fp32 CUDA-core kernels.
C2_TC = [("depth_fc_2048_1088", "conv", 2048, J2 * D2, 1, 1, 0, 1, "in", "write"),
         ("final_256_17", "conv", 256, J2, 1, 1, 0, HM2, "act", "write")]
C2_TC_TENSOR_CORES = {"depth_fc_2048_1088": True, "final_256_17": False}


# ------------------------------------------------------------------ the restated planners
def test_c2_tf32_wgrad_plans():
    """The TF32 wgrad planner at depth_fc's weight gradient (32 pixels, Cin 2048, Cout 1088): one
    32-pixel block per CTA over 144 tiles, with or without the run cap, so its bar is WGRAD_BAR
    itself.  The final layer's bar from the planner's run (2016 pixels) stays under 3.4e-5."""
    fc = _tf32_wgrad_plan(N2, 2048, J2 * D2, 1, 3)
    print("depth_fc: run %d, %d splits, %d tiles" % fc)
    assert fc == (32, 1, 144) == _tf32_wgrad_plan(N2, 2048, J2 * D2, 1, 3, cap=False)
    assert [sc.tf32_wgrad_run(c, N2) for c in C2_TC] == [32, 2016]
    assert _tc_bar(WGRAD_BAR, 32, 3) == WGRAD_BAR and _tc_bar(WGRAD_BAR, 2016, 3) < 3.4e-5
    assert _tc_bar(FPROP_BAR, J2 * D2, 3) == FPROP_BAR


# ------------------------------------------------------------------ heat-map loss: the bar against the kernel's partition
def _emul_hm_loss(hm, tg, wh, drop_cta=None, wr_once=False):
    """heatmap_joint_loss_kernel's heat-map value (HW % 4 == 0) in numpy: per quad d = wr (h - g)
    and ((d0^2 + d1^2) + (d2^2 + d3^2)) in fp32, each thread's quads i, i + stride, ... added in
    fp32 in that order, the per-thread partials in double, L = fp32(sum / (R HW)).  drop_cta: one
    CTA's partial lost; wr_once: wr (h - g)^2 instead of (wr (h - g))^2."""
    f = np.float32
    R, HW = hm.shape
    blocks, trips = sc.hm_grid(R, HW)
    stride, total4 = blocks * HM_THREADS, R * HW // 4
    wr = np.repeat(wh, HW // 4)[:, None]
    diff = hm.reshape(total4, 4) - tg.reshape(total4, 4)
    if wr_once:
        sq = wr * (diff * diff)
    else:
        d = wr * diff
        sq = d * d
    qs = (sq[:, 0] + sq[:, 1]) + (sq[:, 2] + sq[:, 3])
    assert qs.dtype == f
    pad = np.zeros(trips * stride, f)
    pad[:total4] = qs
    facc = np.zeros(stride, f)
    for k in range(trips):
        facc = facc + pad[k * stride:(k + 1) * stride]
    parts = facc.astype(np.float64).reshape(blocks, HM_THREADS).sum(1)
    if drop_cta is not None:
        parts[drop_cta] = 0.0
    return float(np.float32(parts.sum() / (R * HW))), blocks, trips


def test_hm_loss_bar_rejects_a_dropped_partial_and_a_single_weight():
    """(32, 17, 64, 64), the C2(ii) shape: the emulated partition (1056 CTAs, three trips) meets
    hm_loss_ref_bar's heat-map bar; with the first or the last CTA's partial dropped, or with the
    weight applied once, it misses it."""
    N, R, HW = N2, N2 * J2, HM2 * HM2
    hm, tg, wh, x, t, w = sc.hm_case("cpu", N, J2, HM2, HM2, D2, 333)
    L_hm, _, _, _, _, bars = sc.hm_loss_ref_bar(hm.view(R, HW), tg.view(R, HW), wh, x, t, w, R, HW, N)
    h, g, wr = hm.view(R, HW).numpy(), tg.view(R, HW).numpy(), wh.numpy()
    ok, blocks, trips = _emul_hm_loss(h, g, wr)
    r = lambda v: abs(v - L_hm) / bars["hm"]
    bad = {"first CTA dropped": r(_emul_hm_loss(h, g, wr, drop_cta=0)[0]),
           "last CTA dropped": r(_emul_hm_loss(h, g, wr, drop_cta=blocks - 1)[0]),
           "weight once": r(_emul_hm_loss(h, g, wr, wr_once=True)[0])}
    print("heat-map loss emulation, %d CTAs x %d trips: err / bar %.3f; %s" % (
        blocks, trips, r(ok), ", ".join("%s %.3g" % kv for kv in bad.items())))
    assert (blocks, trips) == (1056, 3)
    assert r(ok) <= 1.0
    assert all(v > 10.0 for v in bad.values())


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """After the module, drop its cached model and conv outputs and hand the allocator's reserve
    back to the device for the tests after it."""
    yield
    sc.release("c2_")


# ------------------------------------------------------------------ 1. the VOLUME=False head at C2 sizes
HM_SHAPES = [(N2, HM2, HM2), (128, HM2, HM2), (128, 63, 63)]


@gpu
@pytest.mark.parametrize("N,H,W", HM_SHAPES, ids=["%dx%dx%d" % s for s in HM_SHAPES])
def test_c2_heatmap_joint_loss_vs_float64(dev, N, H, W):
    """epb_heatmap_joint_loss (L1 joint part over N x 17 x 64 depth_fc outputs) against float64:
    the three loss values, dhm and dx within step_cases.hm_loss_ref_bar.  (32, 64, 64): the capped
    grid with three tail trips per thread and n = 34816 in the last CTA; (128, 64, 64): the
    four-quad main loop twice plus a tail trip; 63 x 63: the per-element path under the capped
    grid."""
    R, HW = N * J2, H * W
    case = sc.hm_case(dev, N, J2, H, W, D2, 300 + N + H)
    loss, dhm, dx = sc.run_hm_loss(case, N, J2, H, W)
    torch.cuda.synchronize()
    hm, tg, wh, x, t, w = case
    L_hm, L_jt, L_tot, dhm64, dx64, bars = sc.hm_loss_ref_bar(hm.view(R, HW), tg.view(R, HW), wh, x, t, w, R, HW, N)
    blocks, trips = sc.hm_grid(R, HW)
    main = HW % 4 == 0 and trips >= 4
    r = {"hm": abs(float(loss[0]) - L_hm) / bars["hm"], "jt": abs(float(loss[1]) - L_jt) / bars["jt"],
         "tot": abs(float(loss[2]) - L_tot) / bars["tot"],
         "dhm": float(((dhm.view(R, HW).double() - dhm64).abs() / bars["dhm"].clamp_min(1e-300)).max()),
         "dx": float(((dx.double() - dx64).abs() / bars["dx"].clamp_min(1e-300)).max())}
    print("  heat-map loss (%d, %d, %d, %d), n %d: %d CTAs, %d trips per thread (%s)" % (
        N, J2, H, W, x.numel(), blocks, trips, "four-quad main loop" if main else
        ("quad tail only" if HW % 4 == 0 else "per element")))
    sc._report("loss / dhm / dx", r)
    assert all(v <= 1.0 for v in r.values()), r                 # NaN fails
    assert bool((dhm.view(R, HW)[wh == 0] == 0).all()), "invisible joints carry gradient"
    assert blocks == sc.HM_MAX_BLOCKS


@gpu
def test_c2_heatmap_loss_repeatable_across_grid_sizes(dev):
    """Launches alternating between (2, 17, 64, 64) (136 CTAs) and (128, 17, 64, 64) (1056 CTAs)
    give, bit for bit, what the first launch of each gave: the ticket is reset after every launch
    and a smaller grid never reads a partial a larger one left.  Two launches at N = 128 in a row
    are bit-identical too."""
    small, big = sc.hm_case(dev, 2, J2, HM2, HM2, D2, 71), sc.hm_case(dev, 128, J2, HM2, HM2, D2, 72)
    grids = sc.hm_grid(2 * J2, HM2 * HM2)[0], sc.hm_grid(128 * J2, HM2 * HM2)[0]
    print("  grids: %d and %d CTAs" % grids)
    assert grids == (136, 1056)
    ref_s = sc.run_hm_loss(small, 2, J2, HM2, HM2)
    ref_b = sc.run_hm_loss(big, 128, J2, HM2, HM2)
    runs = [sc.run_hm_loss(big, 128, J2, HM2, HM2)]
    for _ in range(3):
        runs.append(sc.run_hm_loss(small, 2, J2, HM2, HM2))
        runs.append(sc.run_hm_loss(big, 128, J2, HM2, HM2))
    torch.cuda.synchronize()
    for i, got in enumerate(runs):
        ref = ref_b if i % 2 == 0 else ref_s
        for a, b in zip(got, ref):
            assert torch.equal(a, b), "launch %d differs from the first launch of its shape" % i
    assert bool(torch.isfinite(ref_b[1]).all()) and bool(torch.isfinite(ref_s[2]).all())


@gpu
def test_c2_avgpool_split_vs_float64(dev):
    """the trunk's [32, 8 x 8, 2048] planes -> depth_fc's input"""
    sc._check_avgpool_split(dev, N2, 64, 2048)


AVGPOOL_BWD = [(hw, c, acc) for acc in (0, 1) for hw in (64, 144, 49) for c in (2048, 2044)]


@gpu
@pytest.mark.parametrize("HW,C,acc", AVGPOOL_BWD, ids=["hw%d-c%d-acc%d" % s for s in AVGPOOL_BWD])
def test_c2_avgpool_bwd_bit_exact(dev, HW, C, acc):
    """epb_avgpool_bwd at N = 32 (HW 64: C2's 8 x 8 trunk; 144, 49: 384 / 224 inputs; C 2044: a
    partial last CTA), bit-exact; the fp32 avgpool forward of the same shape against float64."""
    sc._check_avgpool_bwd(dev, N2, HW, C, acc)


@gpu
@pytest.mark.parametrize("layer", C2_TC, ids=[c[0] for c in C2_TC])
def test_c2_head_tf32x3_vs_float64(dev, layer):
    """depth_fc (fprop with bias, dgrad K = 1088, wgrad over 32 pixels: 3xTF32) and the final
    layer (wgrad with BatchNorm + ReLU on load over 131072 pixels, dgrad K = 20: the fp32
    CUDA-core kernels) at N = 32 against float64 (step_cases.check_tf32x3_layer).

    Which kernels run, without a profiler session: every fprop, dgrad and wgrad geometry meets
    the restated tensor-core predicate (step_cases.tc_supported) or, for the final layer, fails
    it; and on the device, the forward and the data gradient at precision 3 are bit-identical to
    the CUDA-core kernel's (precision 0, no atomics on those outputs) exactly when the predicate
    sends them there."""
    from epipolarpose_b200 import net, ops
    name, kind, cin, cout, k, s, p, hw, operand, _ = layer
    tc = C2_TC_TENSOR_CORES[name]
    conv = net.Conv("t", kind, cin, cout, k, s, p)
    fg, dg = conv.fprop_geoms(ops, N2, hw, hw, 3), conv.dgrad_geoms(ops, N2, hw, hw, 3)
    assert [sc.tc_supported(gm, False) for gm in fg + dg] == [tc] * len(fg + dg)
    assert [sc.tc_supported(gm, True) for gm in fg] == [tc] * len(fg)
    R, splits, tiles = _tf32_wgrad_plan(N2 * hw * hw, cin, conv.cout_p, 1, 3)
    print("  %s %s; TF32 wgrad plan: %d tiles x %d splits, run %d pixels" % (
        name, "3xTF32" if tc else "fp32 CUDA cores", tiles, splits, R))
    # precision 3 against precision 0 on the same operands
    g = torch.Generator(device=dev).manual_seed(41)
    x = torch.randn(N2, hw, hw, conv.cin_p, device=dev, generator=g)
    dout = torch.randn(N2, hw, hw, conv.cout_p, device=dev, generator=g)
    aff = (torch.rand(conv.cin_p, device=dev, generator=g) + 0.5, torch.randn(conv.cin_p, device=dev, generator=g) * 0.1) \
        if operand == "act" else (None, None)
    wf, wd = conv.pack(ops, torch.randn(cout, cin, k, k, device=dev, generator=g) * (2.0 / cin) ** 0.5)
    outs = {}
    for prec in (0, 3):
        o = torch.empty(N2, hw, hw, conv.cout_p, device=dev)
        for gm in conv.fprop_geoms(ops, N2, hw, hw, prec):
            gm.in_relu, gm.accumulate = int(operand == "act"), 0
            ops.conv_fprop(gm, x, wf, o, aff[0], aff[1], None, None)
        d = torch.empty(N2, hw, hw, conv.cin_p, device=dev)
        for gm in conv.dgrad_geoms(ops, N2, hw, hw, prec):
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv_fprop(gm, dout, wd, d, None, None, None, None)
        outs[prec] = (o, d)
    torch.cuda.synchronize()
    same = [torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(outs[0], outs[3])]
    print("  precision 3 bit-identical to the CUDA-core kernel: fprop %s, dgrad %s" % tuple(same))
    assert same == [not tc, not tc]
    del outs, x, dout
    sc.check_tf32x3_layer(dev, layer, N2, kernels=None)


@gpu
@pytest.mark.parametrize("M,C", [(M2, 20), (N2, J2 * D2)], ids=["131072x20", "32x1088"])
def test_c2_colsum_vs_float64(dev, M, C):
    """the final layer's bias gradient (cout_p 20) and depth_fc's (32 rows of 1088)"""
    _check_colsum(dev, M, C)


@gpu
def test_c2_final_conv16_fprop_vs_float64(dev):
    """conv16 forward of the final layer (256 -> 17, cout_p 20, bias zero-padded as the engine pads
    it; N = 32, 64 x 64) against float64 on the values the planes hold, within 5e-5 of max|ref|;
    the three pad channels exactly zero.  Run into two buffers pre-filled with different NaN
    sentinels and followed by a guard band: every element written, identically, nothing past
    the end."""
    from epipolarpose_b200 import net, ops
    conv = net.Conv("final_layer", "conv", 256, J2, 1, 1, 0, 0)
    C = conv.cout_p
    g = torch.Generator(device=dev).manual_seed(91)
    x, x_sc, xv = _split_dev(torch.relu(torch.randn(N2, HM2, HM2, 256, device=dev, generator=g)))
    w = torch.randn(J2, 256, 1, 1, device=dev, generator=g) * (2.0 / 256) ** 0.5
    wf32, _ = conv.pack(ops, w)
    wf, wf_sc, wfv = _split_dev(wf32)
    bias = torch.zeros(C, device=dev)
    bias[:J2] = torch.randn(J2, device=dev, generator=g) * 0.5
    n, guard = M2 * C, 4096
    outs = []
    for bits in (0x7FC0DEAD, 0x7FC0BEEF):
        buf = torch.full((n + guard,), bits, device=dev, dtype=torch.int32).view(torch.float32)
        for gm in conv.fprop_geoms(ops, N2, HM2, HM2, 3):
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv16_fprop(gm, x, x_sc, wf, wf_sc, buf[:n].view(N2, HM2, HM2, C), bias, None)
        outs.append(buf)
    torch.cuda.synchronize()
    a, b = (o.view(torch.int32) for o in outs)
    assert bool((a[n:] == 0x7FC0DEAD).all()) and bool((b[n:] == 0x7FC0BEEF).all()), "guard band written"
    assert torch.equal(a[:n], b[:n]), "output depends on the prior contents (an element not written)"
    out = outs[0][:n].view(M2, C)
    ref = xv.view(M2, 256) @ wfv.view(C, 256).t() + bias.double()
    e = float((out.double() - ref).abs().max() / ref.abs().max())
    print("  C2 final conv16 fprop 256 -> 17 (cout_p %d): err %.2e, bar 5.0e-05" % (C, e))
    assert e <= 5e-5
    assert bool((out[:, J2:] == 0).all())


@gpu
def test_c2_heatmap_layout_bit_exact(dev):
    """nhwc_to_nchw of the final layer's [32, 64, 64, 20] output to the [32, 17, 64, 64]
    heat-maps, and nchw_to_nhwc of their gradient back to pitch 20: bit-exact, the pad channels
    +0, guard bands untouched."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(39)
    Cp = 20
    src = torch.randn(N2, HM2, HM2, Cp, device=dev, generator=g)
    hm, guard = sc._guarded((N2, J2, HM2, HM2), dev, float("nan"))
    guard.fill_(1234.5)
    ops.nhwc_to_nchw(src, hm, N2, J2, HM2, HM2, Cp)
    dhm = torch.randn(N2, J2, HM2, HM2, device=dev, generator=g)
    back, guard2 = sc._guarded((N2, HM2, HM2, Cp), dev, float("nan"))
    guard2.fill_(1234.5)
    ops.nchw_to_nhwc(dhm, back, N2, J2, HM2, HM2, Cp)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()) and bool((guard2 == 1234.5).all()), "guard band overwritten"
    assert torch.equal(hm.view(torch.int32), src[..., :J2].permute(0, 3, 1, 2).contiguous().view(torch.int32))
    assert torch.equal(back[..., :J2].contiguous().view(torch.int32), dhm.permute(0, 2, 3, 1).contiguous().view(torch.int32))
    assert bool((back[..., J2:].view(torch.int32) == 0).all())


# ------------------------------------------------------------------ 2. shared kernels at C2 sizes
@gpu
@pytest.mark.parametrize("layer", C2_LAYERS, ids=[c[0] for c in C2_LAYERS])
def test_c2_conv16_layers_vs_torch_float64(dev, layer):
    """conv16 fprop (statistics), dgrad and wgrad at N = 32 against torch float64 (the bars of
    test_conv16_bench_layer_shapes_vs_torch_float64); the wgrad bar from wgrad16's planner."""
    from epipolarpose_b200 import net, ops
    name, kind, cin, cout, k, s, p, hw = layer
    conv = net.Conv("t", kind, cin, cout, k, s, p, 0)
    plans = [_wgrad16_plan(gm) for gm in conv.fprop_geoms(ops, N2, hw, hw, 3) if gm is not None]
    R = max(r for r, _ in plans)
    bar = _tc_bar(WGRAD16_BASE, R, 3)
    e = sc._check_conv16_layer(dev, layer, N2, bar)
    print("  C2 %-18s fprop %.2e dgrad %.2e wgrad %.2e (splits %s, run %d pixels, bar %.2e)"
          % (name, e[0], e[1], e[2], [sp for _, sp in plans], R, bar))


C2_STATS = [("c2_stem_col_192_64", "conv", 192, 64, 1, 1, 0, N2, 128, [(0, 0)]),
            ("c2_l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, N2, 64, [(0, 0)])]


@gpu
@pytest.mark.parametrize("case", C2_STATS, ids=[c[0] for c in C2_STATS])
def test_c2_conv16_stats_vs_float64(dev, case):
    """conv16 BatchNorm statistics at M = 524288 (stem) and 131072 (layer1)."""
    sc.check_conv16_stats(dev, case)


@gpu
@pytest.mark.parametrize("M", [524288, 131072, 32768, 8192, 2048])
def test_c2_bn_finalize_scale_vs_float64(dev, M):
    sc.check_bn_finalize_scale(dev, M)


@gpu
@pytest.mark.parametrize("M", [131072, 32768, 8192, 2048])
def test_c2_bn_finalize_vs_float64(dev, M):
    """the downsample layers' BatchNorm of R50 at 256 over 32 images"""
    sc.check_bn_finalize(dev, M)


@gpu
@pytest.mark.parametrize("res", ["none", "split", "affine"])
def test_c2_bn_act_split_vs_float64(dev, res):
    """layer1's conv16 output (131072 x 256) -> bn_finalize_scale -> bn_act_split"""
    sc._check_bn_act_split(dev, res, C2_STATS[1])


@gpu
def test_c2_bn_relu_maxpool_split_vs_float64(dev):
    """the stem's conv16 output (32 x 128 x 128 x 64) -> bn_relu_maxpool_split -> 64 x 64"""
    sc._check_bn_relu_maxpool_split(dev, C2_STATS[0])


@gpu
def test_c2_maxpool_bwd_vs_float64(dev):
    sc._check_maxpool_bwd(dev, N2, 128)


C2_BWD = [(524288, 64), (131072, 256), (32768, 512), (8192, 1024), (2048, 2048)]


@gpu
@pytest.mark.parametrize("mode", ["relu", "bits_inplace"])
@pytest.mark.parametrize("M,C", C2_BWD, ids=["%dx%d" % s for s in C2_BWD])
def test_c2_bn_bwd_split_vs_float64(dev, M, C, mode):
    sc.check_bn_bwd_split(dev, M, C, mode)


@gpu
def test_c2_im2col_split_bit_exact_at_stem(dev):
    """the stem's patch matrix of 32 images of 256 x 256"""
    sc._check_im2col_split(dev, sc.bench_model(dev, "c2_flat")[0]._engine().stem_kpad, N2, HW2)


@gpu
def test_c2_split16_batch_bit_exact_on_model_jobs(dev):
    """split16_batch on the jobs the f16x3 engine builds for R50 / J17 / D64 with the VOLUME=False
    head (a 20-channel final layer, depth_fc 2048 -> 1088)"""
    sc._check_split16_batch(dev, *sc.bench_model(dev, "c2_flat"))


@gpu
def test_c2_pack_weight_batch_bit_exact_on_model_jobs(dev):
    sc._check_pack_weight_batch(dev, sc.bench_model(dev, "c2_flat")[0])


@gpu
def test_c2_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over the C2(ii) model's flat parameter buffer (depth_fc's 2.2M weights
    included): steps 1, 2 and 1000"""
    m, opt = sc.bench_model(dev, "c2_flat")
    assert m.depth_fc.weight.numel() == 2048 * J2 * D2
    sc._check_fused_adam(dev, m, opt)
