"""The fp32-operand conv kernels (conv_tc.cu `conv_fprop_tc_kernel<BN, NS>`, conv_tc_wgrad.cu
`conv_wgrad_tc_kernel<BNW, NS>`, and the CUDA-core conv_simt.cu kernels) through the C ABI
against torch float64 convolutions on the device, on the exact values each kernel multiplies:

  * precision 3 (3xTF32) and 0 (fp32 CUDA cores): the fp32 operand f(x) = max(fma(x, sc, sh), lb)
    and the fp32 weights;
  * precision 1 (single-pass TF32): both operands rounded to TF32 (round to nearest, ties away,
    as tc::to_tf32).

So the bars are the fp32 accumulation noise of each path, not the precision trade-off:
fprop / dgrad <= 2e-5, wgrad <= 3e-5 (max|d| / max|ref|).  A 3xTF32 product with one
correction pass lost, or a single pass that truncates instead of rounding, is ~1e-4 .. 1e-3
off (test_tf32_emulation_bars_have_teeth shows it on the CPU).

The H100's wgmma adds into its fp32 accumulator rounding toward zero, so the tensor-core output
bar grows with K: `step_cases._tc_bar` (its docstring has the measurement).

The shapes reach what the small shapes of test_gpu_parity.py cannot: more tiles than SMs (the
persistent tile loop, the producers' flat k-block stream across tiles, ring phase wrap over
tiles), N tails of both tile widths, odd channel-block counts, Cin > 256 on 3x3 layers, every
phase-grid tap count of the transposed convolutions, and the wgrad ci / co tile tails and
slot-group splits.  Each case names the kernel instantiation it is meant to reach and checks,
from the profiler's kernel names, that it ran."""
import numpy as np
import pytest
import torch

from tests.step_cases import (FPROP_BAR, STATS_SELF_BAR, WGRAD_BAR, _act64, _emul_mma, _fwd64, _geoms, _guarded,
                              _layer, _ran, _tc_bar, _tf32, _tf32_np, _trunc_np)

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ operand rounding
def _relerr(a, ref):
    a, ref = a.double(), ref.double()
    return float((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300))


# ------------------------------------------------------------------ CPU: the bars have teeth
def test_tf32_emulation_bars_have_teeth():
    """At a 3x3 x 64-channel layer's K = 576: the emulated 3xTF32 product (RN hi, truncated lo,
    the mma3_tf32 pass order) and the single-pass TF32 product meet the fprop bar; dropping the
    a_lo or the b_lo pass, or truncating the single-pass operands instead of rounding them,
    misses it by at least 5x."""
    rng = np.random.default_rng(0)
    M, K, N = 128, 576, 64
    a = np.maximum(rng.standard_normal((M, K)), 0).astype(np.float32)       # post-ReLU activations
    b = (rng.standard_normal((K, N)) * np.sqrt(2.0 / K)).astype(np.float32)  # He-initialised weights
    ah, bh = _tf32_np(a), _tf32_np(b)
    al, bl = _trunc_np(a - ah), _trunc_np(b - bh)                            # the lo planes as read
    ref = a.astype(np.float64) @ b.astype(np.float64)
    e = lambda x, r: float(np.max(np.abs(x - r)) / np.max(np.abs(r)))
    full = e(_emul_mma([(al, bh), (ah, bl), (ah, bh)], K), ref)
    no_alo = e(_emul_mma([(ah, bl), (ah, bh)], K), ref)
    no_blo = e(_emul_mma([(al, bh), (ah, bh)], K), ref)
    ref1 = ah.astype(np.float64) @ bh.astype(np.float64)
    one = e(_emul_mma([(ah, bh)], K), ref1)
    one_trunc = e(_emul_mma([(_trunc_np(a), _trunc_np(b))], K), ref1)
    print("3xTF32 %.2e (a_lo dropped %.2e, b_lo dropped %.2e); TF32 %.2e (truncated %.2e); bar %.0e"
          % (full, no_alo, no_blo, one, one_trunc, FPROP_BAR))
    assert full <= FPROP_BAR and one <= FPROP_BAR
    assert min(no_alo, no_blo, one_trunc) >= 5 * FPROP_BAR


def test_tf32_toward_zero_accumulation_floor_and_bar():
    """With the accumulator adds rounded toward zero, at the largest K of the GPU cases (4608):
    3xTF32 and TF32 meet _tc_bar, and the mutants still miss it by at least 2x."""
    rng = np.random.default_rng(1)
    M, K, N = 128, 4608, 64
    a = np.maximum(rng.standard_normal((M, K)), 0).astype(np.float32)
    b = (rng.standard_normal((K, N)) * np.sqrt(2.0 / K)).astype(np.float32)
    ah, bh = _tf32_np(a), _tf32_np(b)
    al, bl = _trunc_np(a - ah), _trunc_np(b - bh)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    ref1 = ah.astype(np.float64) @ bh.astype(np.float64)
    e = lambda x, r: float(np.max(np.abs(x - r)) / np.max(np.abs(r)))
    full = e(_emul_mma([(al, bh), (ah, bl), (ah, bh)], K, True), ref)
    no_alo = e(_emul_mma([(ah, bl), (ah, bh)], K, True), ref)
    one = e(_emul_mma([(ah, bh)], K, True), ref1)
    one_trunc = e(_emul_mma([(_trunc_np(a), _trunc_np(b))], K, True), ref1)
    bar3, bar1 = _tc_bar(FPROP_BAR, K, 3), _tc_bar(FPROP_BAR, K, 1)
    print("toward zero, K=%d: 3xTF32 %.2e (a_lo dropped %.2e) bar %.2e; TF32 %.2e (truncated %.2e) bar %.2e"
          % (K, full, no_alo, bar3, one, one_trunc, bar1))
    assert full <= bar3 and one <= bar1
    assert no_alo >= 2 * bar3 and one_trunc >= 5 * bar1


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _expect(kind, which, precision):
    """which: 'tc64' / 'tc128' / 'tc32' or 'simt' -> the kernel tag _ran reports"""
    if which == "simt" or precision == 0:
        return "%s_simt" % kind
    return "%s_tc<%s,%d>" % (kind, which[2:], 3 if precision == 3 else 1)


def _uses_tc(which, precision):
    return precision != 0 and which != "simt"


def _out_bar(geoms, which, precision):
    """fprop / dgrad output bar: FPROP_BAR, raised to the tensor cores' accumulation floor for
    the longest K = taps x Cin of the call's geometries"""
    if not _uses_tc(which, precision):
        return FPROP_BAR
    K = max(gm.T * gm.Cin for gm in geoms if gm is not None)
    return _tc_bar(FPROP_BAR, K, 3 if precision == 3 else 1)


def _report(what, tags, **errs):
    print("  %-40s %-18s %s" % (what, ",".join(sorted(tags)),
                                " ".join("%s %.2e" % kv for kv in errs.items())))


# ------------------------------------------------------------------ cases
# (id, kind, cin, cout, k, stride, pad, opad, N, H, W, fprop kernel, dgrad kernel, bias, precision 0)
FPROP = [
    # more tiles than SMs: persistent tile loop, flat producer stream, ring phase wrap over tiles
    ("mt_1x1_64_128", "conv", 64, 128, 1, 1, 0, 0, 8, 64, 64, "tc128", "tc64", False, True),   # roll, dmt, once
    ("mt_3x3_256", "conv", 256, 256, 3, 1, 1, 0, 5, 64, 64, "tc128", "tc128", False, False),   # 320 tiles, S=3
    ("mt_3x3_64", "conv", 64, 64, 3, 1, 1, 0, 8, 64, 64, "tc64", "tc64", False, False),
    ("mt_stem_col_160", "conv", 160, 64, 1, 1, 0, 0, 2, 128, 128, "tc64", "tc128", False, False),  # CB = 5
    ("mt_ragged_57", "conv", 128, 128, 3, 1, 1, 0, 7, 57, 57, "tc128", "tc128", False, False),
    # geometry and tails
    ("3x3_s2_ragged", "conv", 64, 128, 3, 2, 1, 0, 3, 29, 29, "tc128", "tc64", False, True),
    ("1x1_s2", "conv", 256, 512, 1, 2, 0, 0, 4, 32, 32, "tc128", "tc128", False, False),
    ("3x3_512_8x8", "conv", 512, 512, 3, 1, 1, 0, 6, 8, 8, "tc128", "tc128", False, False),     # Cin > 256
    ("deconv4", "deconv", 256, 128, 4, 2, 1, 0, 3, 16, 16, "tc128", "tc128", False, False),     # 4 taps / phase
    ("deconv3_op1", "deconv", 128, 64, 3, 2, 1, 1, 3, 15, 15, "tc64", "tc128", False, True),    # 1, 2, 2, 4 taps
    ("cout96", "conv", 64, 96, 3, 1, 1, 0, 2, 20, 20, "tc64", "tc64", False, False),            # BN=64 tail, CB=3
    ("cout160", "conv", 128, 160, 1, 1, 0, 0, 2, 24, 24, "tc128", "tc128", False, False),       # BN=128 tail
    ("final_1632", "conv", 256, 1632, 1, 1, 0, 0, 2, 16, 16, "tc128", "tc128", True, False),    # J=17 x D=96
    # refiner MLP (1x1 convolutions on 1x1 images)
    ("mlp_1024_n64", "conv", 1024, 1024, 1, 1, 0, 0, 64, 1, 1, "tc128", "tc128", True, False),  # M < one tile
    ("mlp_1024_n300", "conv", 1024, 1024, 1, 1, 0, 0, 300, 1, 1, "tc128", "tc128", True, False),
    ("mlp_in_45", "conv", 45, 1024, 1, 1, 0, 0, 300, 1, 1, "simt", "simt", True, True),         # 48-padded
    ("mlp_out_45", "conv", 1024, 45, 1, 1, 0, 0, 300, 1, 1, "simt", "simt", True, True),
]
MULTI_TILE = {c[0] for c in FPROP if c[0].startswith("mt_")}


def _fprop_params():
    out = []
    for c in FPROP:
        for prec in ((0, 1, 3) if c[14] else (1, 3)):
            out.append(pytest.param(c, prec, id="%s-p%d" % (c[0], prec)))
    return out


def _run_fprop(dev, conv, x, wf, out, sc, sh, bias, stats, relu, acc, precision, N, H, W):
    from epipolarpose_b200 import ops
    geoms = _geoms(conv.fprop_geoms(ops, N, H, W, precision), relu if sc is not None else 0, acc)

    def run(o, st):
        for gm in geoms:
            ops.conv_fprop(gm, x, wf, o, sc, sh, bias, st)
    tags = _ran(lambda: run(out.clone(), None if stats is None else stats.clone()))
    run(out, stats)
    return tags


def _check_fprop(dev, case, precision, mode):
    """mode: 'relu' (affine + ReLU, statistics), 'affine' (no ReLU), 'noaffine', 'acc'
    (accumulate onto a random output of similar magnitude, no statistics)"""
    from epipolarpose_b200 import ops
    name, kind, cin, cout, k, s, p, opad, N, H, W, fk, _, with_bias, _ = case
    conv, Ho, Wo, x, sc, sh, w, _ = _layer(dev, kind, cin, cout, k, s, p, opad, N, H, W, 11)
    co = conv.cout_p
    relu = mode == "relu"
    aff = (sc, sh) if mode != "noaffine" else (None, None)
    bias = None
    if with_bias:
        bias = torch.randn(co, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) * 0.5
        bias[cout:] = 0
    tc = _uses_tc(fk, precision)
    a64 = _act64(x, *aff, relu)
    w64 = w.double()
    if tc and precision == 1:
        a64, w64 = _tf32(a64.float()).double(), _tf32(w).double()
    ref = _fwd64(conv, a64, w64)
    if bias is not None:
        ref = ref + bias.double()[None, :, None, None]
    ref = ref.permute(0, 2, 3, 1)
    geoms = conv.fprop_geoms(ops, N, H, W, precision)
    init = None
    if mode == "acc":
        init = torch.randn(N, Ho, Wo, co, device=dev, generator=torch.Generator(device=dev).manual_seed(9))
        init *= float(ref.abs().max()) / 3
        init[..., cout:] = 0
        out, guard = _guarded((N, Ho, Wo, co), dev, 0.0)
        out.copy_(init)
    else:
        # every phase of the output is written by some geometry: start from NaN to catch a missed row
        out, guard = _guarded((N, Ho, Wo, co), dev, 0.0 if any(gm is None for gm in geoms) else float("nan"))
    guard.fill_(1234.5)
    stats = sguard = None
    if mode != "acc":
        sbuf = torch.zeros(2 * co + 64, device=dev, dtype=torch.float64)   # zeroed, with a guard band
        stats, sguard = sbuf[:2 * co], sbuf[2 * co:]
    wf, _ = conv.pack(ops, w)
    tags = _run_fprop(dev, conv, x, wf, out, aff[0], aff[1], bias, stats, relu, int(mode == "acc"),
                      precision, N, H, W)
    assert tags == {_expect("fprop", fk, precision)}, tags
    assert bool((guard == 1234.5).all()), "output guard band overwritten"
    bar = _out_bar(geoms, fk, precision)
    base = init.double() if init is not None else 0.0
    err_out = float((out.double() - (base + ref)).abs().max() / ref.abs().max())
    errs = {"out": err_out}
    if stats is not None:
        assert bool((sguard == 0).all()), "statistics guard band overwritten"
        o = out.double().reshape(-1, co)[:, :co]
        s1, s2 = stats[:co], stats[co:]
        errs["st_self"] = max(float(((s1 - o.sum(0)).abs() / o.abs().sum(0).clamp_min(1e-300)).max()),
                              float(((s2 - (o * o).sum(0)).abs() / (o * o).sum(0).clamp_min(1e-300)).max()))
        # the per-channel sum against the reference's, relative to the channel's sum of |ref|
        r = ref.reshape(-1, co)
        errs["st_ref"] = max(float(((s1 - r.sum(0)).abs() / r.abs().sum(0).clamp_min(1e-300)).max()),
                             _relerr(s2, (r * r).sum(0)))
    errs["bar"] = bar
    _report("%s p%d %s" % (name, precision, mode), tags, **errs)
    assert err_out <= bar, "output %.3e (bar %.2e)" % (err_out, bar)
    if stats is not None:
        assert errs["st_self"] <= STATS_SELF_BAR, "statistics vs own output %.3e" % errs["st_self"]
        assert errs["st_ref"] <= bar, "statistics vs reference %.3e (bar %.2e)" % (errs["st_ref"], bar)
    return conv, x, wf, aff, bias, out, stats, N, H, W


@gpu
@pytest.mark.parametrize("case,precision", _fprop_params())
def test_tf32_fprop_vs_float64(dev, case, precision):
    """fprop with the producing layer's BatchNorm + ReLU fused, statistics into a zeroed buffer
    (and the bias where the layer has one); multi-tile cases also run twice, bit-identically."""
    conv, x, wf, aff, bias, out, stats, N, H, W = _check_fprop(dev, case, precision, "relu")
    if case[0] in MULTI_TILE:
        out2, st2 = torch.empty_like(out), torch.zeros_like(stats)
        _run_fprop(dev, conv, x, wf, out2, aff[0], aff[1], bias, st2, 1, 0, precision, N, H, W)
        assert torch.equal(out, out2) and torch.equal(stats, st2), "not run-to-run deterministic"


EPILOGUE = [c for c in FPROP if c[0] in ("cout96", "cout160", "mt_3x3_64", "final_1632")]


@gpu
@pytest.mark.parametrize("mode", ["affine", "noaffine", "acc"])
@pytest.mark.parametrize("precision", [1, 3])
@pytest.mark.parametrize("case", EPILOGUE, ids=[c[0] for c in EPILOGUE])
def test_tf32_fprop_epilogues_vs_float64(dev, case, precision, mode):
    """The other epilogue / operand flags: affine without ReLU, no affine, accumulate = 1 onto
    an output of the result's magnitude."""
    _check_fprop(dev, case, precision, mode)


DGRAD = [c for c in FPROP if c[12] is not None]


def _dgrad_params():
    out = []
    for c in DGRAD:
        for prec in ((0, 1, 3) if c[14] else (1, 3)):
            out.append(pytest.param(c, prec, id="%s-p%d" % (c[0], prec)))
    return out


@gpu
@pytest.mark.parametrize("case,precision", _dgrad_params())
def test_tf32_dgrad_vs_float64(dev, case, precision):
    """dIn = the transposed convolution of dOut (conv_fprop on the dgrad geometries), written
    (accumulate = 0, onto NaN where every pixel is written) and added (accumulate = 1)."""
    from epipolarpose_b200 import ops
    name, kind, cin, cout, k, s, p, opad, N, H, W, _, dk, _, _ = case
    conv, Ho, Wo, _, _, _, w, gout = _layer(dev, kind, cin, cout, k, s, p, opad, N, H, W, 21)
    ci = conv.cin_p
    tc = _uses_tc(dk, precision)
    g64, w64 = gout.permute(0, 3, 1, 2).double(), w.double()
    if tc and precision == 1:
        g64, w64 = _tf32(gout).permute(0, 3, 1, 2).double(), _tf32(w).double()
    import torch.nn.functional as F
    if kind == "conv":
        ref = torch.nn.grad.conv2d_input((N, ci, H, W), w64, g64, s, p)
    else:
        ref = F.conv2d(g64, w64, None, s, p)
    ref = ref.permute(0, 2, 3, 1)
    _, wd = conv.pack(ops, w)
    geoms = conv.dgrad_geoms(ops, N, H, W, precision)
    gen = torch.Generator(device=dev).manual_seed(9)
    for acc in (0, 1):
        gms = _geoms(geoms, 0, acc)
        fill = 0.0 if (acc or any(gm is None for gm in geoms)) else float("nan")
        din, guard = _guarded((N, H, W, ci), dev, fill)
        guard.fill_(1234.5)
        init = torch.zeros_like(din)
        if acc:
            init = torch.randn(din.shape, device=dev, generator=gen) * (float(ref.abs().max()) / 3)
            init[..., cin:] = 0
            din.copy_(init)

        def run(o):
            for gm in gms:
                ops.conv_fprop(gm, gout, wd, o, None, None, None, None)
        tags = _ran(lambda: run(din.clone()))
        run(din)
        assert tags == {_expect("fprop", dk, precision)}, tags
        assert bool((guard == 1234.5).all()), "output guard band overwritten"
        e = float((din.double() - (init.double() + ref)).abs().max() / ref.abs().max())
        bar = _out_bar(geoms, dk, precision)
        _report("%s dgrad p%d acc%d" % (name, precision, acc), tags, out=e, bar=bar)
        assert e <= bar, "dgrad acc=%d %.3e (bar %.2e)" % (acc, e, bar)


# (id, kind, cin, cout, k, stride, pad, opad, N, H, W, wgrad kernel, precision 0)
WGRAD = [
    ("w_1x1_64_256", "conv", 64, 256, 1, 1, 0, 0, 8, 64, 64, "tc64", True),       # dense in / out, pixel splits
    ("w_3x3_64", "conv", 64, 64, 3, 1, 1, 0, 4, 32, 32, "tc64", False),           # 5 slot groups, last NB = 1
    ("w_3x3_512", "conv", 512, 512, 3, 1, 1, 0, 4, 8, 8, "tc128", False),         # 36 groups
    ("w_3x3_32_40", "conv", 32, 40, 3, 1, 1, 0, 3, 20, 20, "tc32", True),         # Cout % 32 != 0
    ("w_cin96", "conv", 96, 64, 3, 1, 1, 0, 2, 16, 16, "tc64", False),            # ci-tile tail
    ("w_cin160", "conv", 160, 64, 1, 1, 0, 0, 2, 32, 32, "tc128", False),         # ci-tile tail
    ("w_1x1_s2", "conv", 256, 512, 1, 2, 0, 0, 4, 16, 16, "tc128", False),
    ("w_deconv4", "deconv", 256, 128, 4, 2, 1, 0, 2, 8, 8, "tc128", False),
    ("w_deconv3_op1", "deconv", 64, 64, 3, 2, 1, 1, 2, 12, 12, "tc64", False),
    ("w_final_1632", "conv", 256, 1632, 1, 1, 0, 0, 2, 16, 16, "tc128", False),   # co-tile tail of 96
]


def _wgrad_params():
    out = []
    for c in WGRAD:
        for prec in ((0, 1, 3) if c[12] else (1, 3)):
            for mode in ("relu", "affine", "noaffine"):
                out.append(pytest.param(c, prec, mode, id="%s-p%d-%s" % (c[0], prec, mode)))
    return out


@gpu
@pytest.mark.parametrize("case,precision,mode", _wgrad_params())
def test_tf32_wgrad_vs_float64(dev, case, precision, mode):
    """dW += sum over pixels of dOut x f(In) into a non-zero dW (the += contract)."""
    from epipolarpose_b200 import ops
    name, kind, cin, cout, k, s, p, opad, N, H, W, wk, _ = case
    conv, Ho, Wo, x, sc, sh, w, gout = _layer(dev, kind, cin, cout, k, s, p, opad, N, H, W, 31)
    ci, co, T = conv.cin_p, conv.cout_p, k * k
    aff = (sc, sh) if mode != "noaffine" else (None, None)
    relu = mode == "relu"
    tc = _uses_tc(wk, precision)
    a64, g64 = _act64(x, *aff, relu), gout.permute(0, 3, 1, 2).double()
    if tc and precision == 1:
        a64 = _tf32(a64.float()).double()
        g64 = _tf32(gout).permute(0, 3, 1, 2).double()
    w64 = w.double().requires_grad_(True)
    _fwd64(conv, a64, w64).backward(g64)
    gw = w64.grad
    ref = (gw.permute(0, 2, 3, 1) if kind == "conv" else gw.permute(1, 2, 3, 0)).reshape(co, T, ci)
    gen = torch.Generator(device=dev).manual_seed(13)
    init = torch.randn(co, T, ci, device=dev, generator=gen) * (float(ref.abs().max()) / 3)
    dw, guard = _guarded((co * T * ci,), dev, 0.0)
    guard.fill_(1234.5)
    dw.copy_(init.reshape(-1))
    gms = _geoms(conv.fprop_geoms(ops, N, H, W, precision), int(relu) if aff[0] is not None else 0, 0)

    def run(o):
        for gm in gms:
            ops.conv_wgrad(gm, x, gout, o, aff[0], aff[1])
    tags = _ran(lambda: run(dw.clone()))
    run(dw)
    assert tags == {_expect("wgrad", wk, precision)}, tags
    assert bool((guard == 1234.5).all()), "dW guard band overwritten"
    e = float((dw.view(co, T, ci).double() - (init.double() + ref)).abs().max() / ref.abs().max())
    _report("%s wgrad p%d %s" % (name, precision, mode), tags, dw=e, bar=WGRAD_BAR)
    assert e <= WGRAD_BAR, "wgrad %.3e" % e


@gpu
def test_tf32_every_wgmma_instantiation_is_covered():
    """The case tables above reach every conv_fprop_tc_kernel<64|128, 1|3> with a multi-tile
    case and every conv_wgrad_tc_kernel<32|64|128, 1|3>."""
    fk = {c[11] for c in FPROP if c[0] in MULTI_TILE}
    assert fk == {"tc64", "tc128"}
    assert {c[11] for c in WGRAD} == {"tc32", "tc64", "tc128"}


@gpu
def test_tf32_abi_rejects_stats_with_accumulate_and_precision_2(dev):
    from epipolarpose_b200 import _lib, net, ops
    conv = net.Conv("t", "conv", 64, 64, 1, 1, 0)
    x = torch.randn(1, 4, 4, 64, device=dev)
    wf = torch.randn(64 * 64, device=dev)
    out = torch.zeros(1, 4, 4, 64, device=dev)
    stats = torch.zeros(128, device=dev, dtype=torch.float64)
    g = conv.fprop_geoms(ops, 1, 4, 4, 3)[0]
    g.in_relu, g.accumulate = 0, 1
    with pytest.raises(_lib.EpbError):
        ops.conv_fprop(g, x, wf, out, None, None, None, stats)
    g.accumulate, g.precision = 0, 2
    with pytest.raises(_lib.EpbError):
        ops.conv_fprop(g, x, wf, out, None, None, None, stats)
    with pytest.raises(_lib.EpbError):
        ops.conv_wgrad(g, x, out, torch.zeros(64 * 64, device=dev))
    g.precision = 3
    ops.conv_fprop(g, x, wf, out, None, None, None, stats)      # the same call with valid flags runs
    torch.cuda.synchronize()
