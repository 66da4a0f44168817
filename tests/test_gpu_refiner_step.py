"""The refiner's training step (refiner/main.py train(): LinearModelPG through mlp.MLPEngine at
linear_size 1024, batch 64, p_dropout 0.5, the fp32 engine at 3xTF32, FusedAdam and the on-device
clip_grad_norm_) against float64 kernel by kernel at its own sizes.  tests/test_step_coverage.py
gates the refiner step on these tests.

Every reference is torch float64 on the device, computed from the exact fp32 values the kernel
read, or a bit-exact torch restatement where the kernel does no arithmetic or one fp32 operation
per element.  Row-shaped items run at N = 64 and at N = 37, an odd ragged last batch (the
DataLoader keeps it).  Bars (u = 2^-24):

  * The twelve linears are three distinct 1 x 1 convolutions over [N][C] rows (REFINER_LINEARS),
    through step_cases.check_tf32x3_layer with the bias and the statistics in one epilogue call,
    as MLPEngine.linear makes it; the 3xTF32 bars of that check.  Their kernels split across both
    families (epb_conv_tc_supported / epb_conv_wgrad_tc_supported, restated in
    step_cases.tc_supported): REFINER_KERNELS pins each product's kernel family, shown without a
    profiler session by the products' rounding at precision 1.  M = 64 is half of the tensor-core
    fprop's 128-row tile: rows 64 .. 127 must be neither stored nor counted.
  * bn_finalize, bn_act (ReLU, no residual) and bn_bwd_reduce + bn_bwd_apply (the BatchNorm's
    own ReLU, no y_out) at M = 64 and 37, C = 1024: the checks and bars of step_cases.
  * bn_eval_affine (the eval forward main.test() runs): invstd = 1 / sqrtf(rv + eps) takes three
    roundings (2.5u relative, the sqrt halving the add's), scale = gamma invstd one more, so
    |d scale| <= 4u |scale|; shift = beta - rm gamma invstd: the product carries 4.5u, the
    difference one more rounding, |d shift| <= 6u (|beta| + |rm gamma invstd|).
  * colsum at [N][48] and [N][1024]: step_cases._check_colsum.
  * pack_weight, mask_scale, add3: bit-exact against torch.
  * sumsq: the squares of fp32 values are exact in double, so only the double additions round:
    per thread, the warp tree, the CTA's 8 warps, one atomic per CTA over every tensor, at most
    ~5000 deep here: within 1e-12 relative of the float64 sum.  clip_scale multiplies by
    float32(max_norm / (sqrt(total) + 1e-6)): bit-exact with that product.
  * FusedAdam per tensor (the refiner's gradients are separate tensors): step_cases._adam_errors.
  * The training forward end to end: p1, p2 and the running statistics of all ten BatchNorms
    against oracle/restate_refiner.py in float64 with the dropout masks replayed, within
    12 * 1024 * eps32 * max|.|, the bar of test_gpu_refiner.  Gradients stay kernel-level: a
    ReLU unit within rounding of zero flips between evaluations, so a whole-step gradient bar does
    not hold."""
import collections
import contextlib
import math

import numpy as np
import pytest
import torch

from tests import step_cases as sc

gpu = pytest.mark.gpu

L, NB, N_TAIL = 1024, 64, 37          # refiner/main.py: linear_size 1024, batch_size 64
EPS32 = float(np.finfo(np.float32).eps)
ROWS = [NB, N_TAIL]

# (name, kind, cin, cout, k, stride, pad, input hw, operand, dgrad): every distinct linear of
# LinearModelPG as a 1 x 1 convolution over [N][1][1][C]; w3 is w1's shape, w4 w2's
REFINER_LINEARS = [
    ("w1_45_1024", "conv", 45, L, 1, 1, 0, 1, "in", "write"),
    ("stage_1024_1024", "conv", L, L, 1, 1, 0, 1, "in", "write"),
    ("w2_1024_45", "conv", L, 45, 1, 1, 0, 1, "in", "write"),
]
TC_FPROP, TC_WGRAD = "fprop_tc<128,3>", "wgrad_tc<128,3>"
# the kernel of each product (dgrad runs the fprop kernel on the transposed operand); cin_p /
# cout_p 48 is not a multiple of 32, so those products run on the fp32 CUDA cores
REFINER_KERNELS = {
    "w1_45_1024": {"fprop": "fprop_simt", "dgrad": "fprop_simt", "wgrad": "wgrad_simt"},
    "stage_1024_1024": {"fprop": TC_FPROP, "dgrad": TC_FPROP, "wgrad": TC_WGRAD},
    "w2_1024_45": {"fprop": "fprop_simt", "dgrad": "fprop_simt", "wgrad": TC_WGRAD},
}


def test_refiner_kernel_table_matches_the_dispatch_predicate():
    """REFINER_KERNELS agrees with step_cases.tc_supported on the engine's own geometries at
    N = 64 and 37: CUDA-core exactly where 48 channels meet a product's Cin (or fprop's Cout)."""
    from epipolarpose_b200 import net
    from tests import emul_ops as em
    for name, kind, cin, cout, k, s, p, hw, _, _ in REFINER_LINEARS:
        conv = net.Conv(name, kind, cin, cout, k, s, p, bias=True)
        for N in ROWS:
            fg = conv.fprop_geoms(em, N, hw, hw, 3)
            dg = conv.dgrad_geoms(em, N, hw, hw, 3)
            assert len(fg) == len(dg) == 1
            got = {"fprop": TC_FPROP if sc.tc_supported(fg[0], False) else "fprop_simt",
                   "dgrad": TC_FPROP if sc.tc_supported(dg[0], False) else "fprop_simt",
                   "wgrad": TC_WGRAD if sc.tc_supported(fg[0], True) else "wgrad_simt"}
            assert got == REFINER_KERNELS[name], (name, N, got)


def _one_row_refused(dev, L_):
    """A one-row training batch raises torch.nn.BatchNorm1d's ValueError before any running
    statistic moves; eval mode and two rows still run."""
    from oracle import restate_refiner as rr
    from epipolarpose_b200.refiner import model as rmodel
    sd = rr.init_state(rr.param_shapes(L_, 45, 45), 5)
    m = rmodel.LinearModelPG(linear_size=L_, p_dropout=0.5, input_size=45, output_size=45)
    m.load_state_dict(sd)
    m = m.to(dev).train()
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        torch.nn.BatchNorm1d(L_).to(dev).train()(torch.randn(1, L_, device=dev))
    before = {k: v.clone() for k, v in m.state_dict().items()}
    x = torch.randn(1, 45, device=dev)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        m(x)
    for k, v in m.state_dict().items():
        assert torch.equal(v, before[k]), k
    m.eval()
    with torch.no_grad():
        e1, e2 = m(x)
    assert bool(torch.isfinite(e1).all() and torch.isfinite(e2).all())
    m.train()
    p1, p2 = m(torch.randn(2, 45, device=dev))
    assert bool(torch.isfinite(p1).all() and torch.isfinite(p2).all())
    return m


def test_refiner_one_row_batch_refused_emulated():
    """On the emulated ABI: a linear_size-128 refiner refuses a training batch of one row."""
    from epipolarpose_b200.refiner import model as rmodel
    from tests import emul_ops
    rmodel.LinearModelPG._backend[0] = emul_ops
    try:
        _one_row_refused(torch.device("cpu"), 128)
    finally:
        rmodel.LinearModelPG._backend[0] = None


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _refiner(dev, seed, p_dropout=0.5):
    """LinearModelPG(1024, 45 -> 45) on the device with the oracle's seeded state (non-trivial
    BatchNorm affines and running statistics), and that state"""
    from oracle import restate_refiner as rr
    from epipolarpose_b200.refiner import model as rmodel
    sd = rr.init_state(rr.param_shapes(L, 45, 45), seed)
    m = rmodel.LinearModelPG(linear_size=L, p_dropout=p_dropout, input_size=45, output_size=45)
    m.load_state_dict(sd)
    return m.to(dev).train(), sd


@contextlib.contextmanager
def _count_calls():
    """C-ABI entry -> number of calls through ops._call"""
    from epipolarpose_b200 import ops
    counts, orig = collections.Counter(), ops._call

    def call(name, *a):
        counts[name] += 1
        return orig(name, *a)
    ops._call = call
    try:
        yield counts
    finally:
        ops._call = orig


# ------------------------------------------------------------------ 1. the linears
def _families_at_precision_1(dev, layer, N):
    """{product: "tc" or "simt"}: which kernel family each product of the layer runs, without a
    profiler session.  At precision 1 the tensor-core kernels make one pass on TF32-rounded
    operands and the CUDA-core kernels ignore the precision, so each product matches one of two
    float64 references within the fp32 bar (FPROP_BAR, WGRAD_BAR) and misses the other: the
    product on the exact fp32 operands (CUDA cores) or on the TF32-rounded ones (tensor cores).
    TF32 rounding moves a product by ~2^-12 relative, 10x the bar."""
    from epipolarpose_b200 import ops
    name, kind, cin, cout, k, s, p, hw, _, _ = layer
    conv, _, _, x, _, _, w, gout = sc._layer(dev, kind, cin, cout, k, s, p, 0, N, hw, hw, 61)
    ci, co = conv.cin_p, conv.cout_p
    wf, wd = conv.pack(ops, w)
    f = torch.empty(N, 1, 1, co, device=dev)
    d = torch.empty(N, 1, 1, ci, device=dev)
    dw = torch.zeros(co * ci, device=dev)
    for gm in conv.fprop_geoms(ops, N, hw, hw, 1):
        gm.in_relu, gm.accumulate = 0, 0
        ops.conv_fprop(gm, x, wf, f, None, None, None, None)
        ops.conv_wgrad(gm, x, gout, dw, None, None)
    for gm in conv.dgrad_geoms(ops, N, hw, hw, 1):
        gm.in_relu, gm.accumulate = 0, 0
        ops.conv_fprop(gm, gout, wd, d, None, None, None, None)
    torch.cuda.synchronize()
    X, G, W = (t.reshape(n, -1).double() for t, n in ((x, N), (gout, N), (w, co)))
    Xt, Gt, Wt = (sc._tf32(t).reshape(n, -1).double() for t, n in ((x, N), (gout, N), (w, co)))
    got = {"fprop": (f.view(N, co), X @ W.t(), Xt @ Wt.t(), sc.FPROP_BAR),
           "dgrad": (d.view(N, ci), G @ W, Gt @ Wt, sc.FPROP_BAR),
           "wgrad": (dw.view(co, ci), G.t() @ X, Gt.t() @ Xt, sc.WGRAD_BAR)}
    fam = {}
    for what, (out, exact, rounded, bar) in got.items():
        scale = float(exact.abs().max())
        e_x = float((out.double() - exact).abs().max()) / scale
        e_t = float((out.double() - rounded).abs().max()) / scale
        fam[what] = "simt" if e_x <= bar < e_t else ("tc" if e_t <= bar < e_x else "neither")
        print("  %-18s N %d %s at precision 1: err vs fp32 operands %.2e, vs TF32 operands %.2e (bar %.0e): %s"
              % (name, N, what, e_x, e_t, bar, fam[what]))
    return fam


@gpu
@pytest.mark.parametrize("N", ROWS)
@pytest.mark.parametrize("layer", REFINER_LINEARS, ids=[c[0] for c in REFINER_LINEARS])
def test_refiner_linears_vs_float64(dev, layer, N):
    """fprop with the bias and the statistics in one call, dgrad (written) and wgrad of each
    distinct linear over N rows against torch float64 within the 3xTF32 bars; the statistics
    within STATS_SELF_BAR of the kernel's own output and within the fprop bar of x W^T + b, and
    more than 100x over it with the bias left out; padding columns 45 .. 47 of w2's output
    exactly 0; guard bands untouched.  Each product runs the kernel family of REFINER_KERNELS
    (_families_at_precision_1); at precision 3 a single-pass tensor-core product would miss the
    3xTF32 bars by the same TF32 rounding, so the tensor-core products are three-pass."""
    want = {k: ("tc" if "_tc<" in v else "simt") for k, v in REFINER_KERNELS[layer[0]].items()}
    assert _families_at_precision_1(dev, layer, N) == want
    sc.check_tf32x3_layer(dev, layer, N, kernels=None, bias_stats=True)


# ------------------------------------------------------------------ 2. the BatchNorm chain at M = 64 and 37
@gpu
@pytest.mark.parametrize("M", ROWS)
def test_refiner_bn_finalize_vs_float64(dev, M):
    """bn_finalize over 1024 channels at the refiner's batch: every output, running_mean and the
    unbiased running_var with momentum within 1 fp32 ulp of float64"""
    sc.check_bn_finalize(dev, M, L)


@gpu
@pytest.mark.parametrize("M", ROWS)
def test_refiner_bn_act_vs_float64(dev, M):
    """bn_act with ReLU and no residual (MLPEngine.bn_relu) at M x 1024"""
    sc.check_bn_act(dev, M, L, "relu")


@gpu
@pytest.mark.parametrize("M", ROWS)
def test_refiner_bn_bwd_vs_float64(dev, M):
    """bn_bwd_reduce + bn_bwd_apply with the BatchNorm's own ReLU and no y_out at M x 1024"""
    sc.check_bn_bwd(dev, M, L, "relu")


@gpu
def test_refiner_bn_eval_affine_vs_float64(dev):
    """bn_eval_affine over 1024 channels against float64 within the module's bars, with
    negative and zero gammas and zero running variances (invstd = 1 / sqrt(eps))"""
    from epipolarpose_b200 import ops
    C = L
    g = torch.Generator(device=dev).manual_seed(19)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    gamma[4:12] *= -1
    gamma[12:16] = 0
    beta = torch.randn(C, device=dev, generator=g) * 0.3
    rm = torch.randn(C, device=dev, generator=g) * 2
    rv = torch.rand(C, device=dev, generator=g) * 3 + 0.01
    rv[:4] = 0
    scale, sguard = sc._guarded((C,), dev, float("nan"))
    shift, hguard = sc._guarded((C,), dev, float("nan"))
    sguard.fill_(1234.5)
    hguard.fill_(1234.5)
    ops.bn_eval_affine(C, gamma, beta, rm, rv, sc.EPS, scale, shift)
    torch.cuda.synchronize()
    assert bool((sguard == 1234.5).all() and (hguard == 1234.5).all()), "guard band overwritten"
    inv = 1 / torch.sqrt(rv.double() + float(np.float32(sc.EPS)))
    s64 = gamma.double() * inv
    p64 = rm.double() * s64
    h64 = beta.double() - p64
    rs = float(((scale.double() - s64).abs() / (4 * sc.U * s64.abs()).clamp_min(1e-300)).max())
    rh = float(((shift.double() - h64).abs() / (6 * sc.U * (beta.double().abs() + p64.abs()))).max())
    print("  bn_eval_affine C %d worst err / bar: scale %.3f shift %.3f" % (C, rs, rh))
    assert rs <= 1.0 and rh <= 1.0


# ------------------------------------------------------------------ 3. bias gradients
COLSUM = [(M, C) for M in ROWS for C in (48, L)]


@gpu
@pytest.mark.parametrize("M,C", COLSUM, ids=["%dx%d" % c for c in COLSUM])
def test_refiner_colsum_vs_float64(dev, M, C):
    """epb_colsum over M x C (the bias gradients of w2 / w4 and of the 1024-wide linears):
    make_rowmap(48) gives 21 row slots of 12 threads, the M rows one CTA"""
    sc._check_colsum(dev, M, C)


# ------------------------------------------------------------------ 4. weights, dropout, residual sums
PACK = [(L, 45), (L, L), (45, L)]     # state_dict [cout][cin] of w1 / w3, the stage linears, w2 / w4


@gpu
@pytest.mark.parametrize("A,B", PACK, ids=["%dx%d" % s for s in PACK])
def test_refiner_pack_weight_bit_exact(dev, A, B):
    """pack_weight of a [cout][cin] weight into the fprop operand [cout][cin_p] and the dgrad
    operand [cin][cout_p] (a transpose), zero padding, and the unpack (unpack=1) of a packed
    gradient back to [cout][cin], which must not read the padding; bit-exact with torch, guard
    bands untouched; Conv.pack's two operands likewise."""
    from epipolarpose_b200 import net, ops
    conv = net.Conv("t", "conv", B, A, 1, 1, 0, bias=True)
    ci, co = conv.cin_p, conv.cout_p
    g = torch.Generator(device=dev).manual_seed(A + B)
    w = torch.randn(A, B, device=dev, generator=g) * (2.0 / B) ** 0.5
    w.view(-1)[::13] = -0.0
    w.view(-1)[7::101] = 1e-40                                # subnormals
    bits = lambda t: t.contiguous().view(torch.int32)
    for swap, ypad, ref in ((0, ci, w), (1, co, w.t())):
        X, Y = ref.shape
        dst, guard = sc._guarded((X * ypad,), dev, float("nan"))
        guard.fill_(1234.5)
        ops.pack_weight(w, dst, A, B, 1, 1, swap, ypad)
        torch.cuda.synchronize()
        want = torch.zeros(X, ypad, device=dev)
        want[:, :Y] = ref
        assert bool((guard == 1234.5).all()), "guard band overwritten"
        assert torch.equal(bits(dst), bits(want).view(-1)), ("pack", swap)
    wf, wd = conv.pack(ops, w.reshape(A, B, 1, 1))
    want_f = torch.zeros(co, ci, device=dev)
    want_f[:A, :B] = w
    want_d = torch.zeros(ci, co, device=dev)
    want_d[:B, :A] = w.t()
    assert torch.equal(bits(wf), bits(want_f).view(-1)) and torch.equal(bits(wd), bits(want_d).view(-1))
    packed = torch.randn(co, ci, device=dev, generator=g)
    packed[:, B:] = float("nan")                              # never read
    packed[A:] = float("nan")
    gw, guard = sc._guarded((A, B), dev, float("nan"))
    guard.fill_(1234.5)
    ops.pack_weight(packed, gw, A, B, 1, 1, 0, ci, 1)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "unpack guard band overwritten"
    assert torch.equal(bits(gw), bits(packed[:A, :B])), "unpack"
    print("  pack_weight %d x %d: fprop [%d][%d], dgrad [%d][%d] and the unpack bit-exact" % (A, B, A, ci, B, co))


MASK = [(NB * L, 0.5), (NB * L, 0.3), (4099, 0.5), (4099, 0.3)]


@gpu
@pytest.mark.parametrize("n,p", MASK, ids=["%d-p%g" % c for c in MASK])
def test_refiner_mask_scale_bit_exact(dev, n, p):
    """mask_scale (dropout and its backward) with keep masks drawn as MLPEngine.dropout draws
    them, scale 1 / (1 - p) (2, and 1 / 0.7, not a power of two), at the step's 64 x 1024 and at
    an n that is not a multiple of 4: bit-exact with torch.where(mask, x * fp32(scale), 0), -0.0
    and subnormal inputs among them, a guard band untouched."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(n + int(p * 10))
    x = torch.randn(n, device=dev, generator=g) * 3
    x[::17] = -0.0
    x[5::29] = 3e-40
    keep = (torch.rand(n, device=dev, generator=g) >= p).to(torch.uint8)
    scale = 1.0 / (1.0 - p)
    out, guard = sc._guarded((n,), dev, float("nan"))
    guard.fill_(1234.5)
    ops.mask_scale(x, keep, scale, out, n)
    torch.cuda.synchronize()
    ref = torch.where(keep.bool(), x * torch.tensor(np.float32(scale), device=dev), torch.zeros_like(x))
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))
    print("  mask_scale n %d scale %.7g: bit-exact, %d kept" % (n, np.float32(scale), int(keep.sum())))


ADD3 = [(n, k) for n in (NB * L, NB * 48, 4097) for k in (2, 3)]


@gpu
@pytest.mark.parametrize("n,k", ADD3, ids=["%d-%dinputs" % c for c in ADD3])
def test_refiner_add3_bit_exact(dev, n, k):
    """add3 (the residual sums and the gradient accumulation) with 2 and 3 inputs: bit-exact with
    fp32 (a + b) + c in that order, a guard band untouched"""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(n + k)
    a = torch.randn(n, device=dev, generator=g) * 1e3
    b = torch.randn(n, device=dev, generator=g)
    c = torch.randn(n, device=dev, generator=g) * 1e-3 if k == 3 else None
    a[::11] = -b[::11]                                        # exact cancellations
    out, guard = sc._guarded((n,), dev, float("nan"))
    guard.fill_(1234.5)
    ops.add3(a, b, c, out, n)
    torch.cuda.synchronize()
    ref = a + b if c is None else (a + b) + c
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    assert torch.equal(out.view(torch.int32), ref.view(torch.int32))


# ------------------------------------------------------------------ 5. clip_grad_norm_ and FusedAdam
def _backward_grads(dev, seed):
    """the 44 gradient tensors of one real refiner backward (N = 64, dropout 0.5, both heads'
    MSELoss), as the training step produces them; (model, gradients)"""
    m, _ = _refiner(dev, seed)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(NB, 45, generator=g).to(dev)
    t = (torch.randn(NB, 45, generator=g) * 0.3).to(dev)
    torch.manual_seed(seed)
    p1, p2 = m(x)
    mse = torch.nn.MSELoss()
    (mse(p1, t) + mse(p2, t)).backward()
    grads = [p.grad for p in m.parameters()]
    assert len(grads) == 44 and all(gr is not None and gr.is_contiguous() for gr in grads)
    return m, grads


@gpu
def test_refiner_clip_grad_norm_vs_float64(dev):
    """sumsq over the 44 gradients of a real backward (45 to 1 048 576 floats): the device total
    within 1e-12 relative of float64 sum x^2, which an fp32-accumulated total misses; clip_scale
    at max_norm 1 bit-exact with x * float32(max_norm / (sqrt(total) + 1e-6)) on the device's own
    total;
    refiner.utils.clip_grad_norm_ with the norm below max_norm leaves every gradient unchanged bit
    for bit and returns torch.nn.utils.clip_grad_norm_'s float64 norm."""
    from epipolarpose_b200 import ops
    from epipolarpose_b200.refiner import utils as rutils
    m, grads = _backward_grads(dev, 41)
    sizes = sorted(gr.numel() for gr in grads)
    assert sizes[0] == 45 and sizes[-1] == L * L
    G0 = [gr.clone() for gr in grads]
    ref = float(sum((gr.double() ** 2).sum() for gr in G0))
    acc32 = torch.zeros((), device=dev)
    for gr in G0:
        acc32 += (gr * gr).sum()
    total = torch.zeros(1, device=dev, dtype=torch.float64)
    with _count_calls() as counts:
        for gr in grads:
            ops.sumsq(gr, gr.numel(), total)
    torch.cuda.synchronize()
    assert counts["epb_sumsq"] == 44
    tot = float(total)
    e64, e32 = abs(tot - ref) / ref, abs(float(acc32) - ref) / ref
    print("  sumsq over %d floats: rel err %.2e (bar 1e-12), fp32-accumulated %.2e" % (sum(sizes), e64, e32))
    assert e64 <= 1e-12
    assert e32 > 1e-12
    # clipping at the step's max_norm = 1: a factor that is not a power of two, so every product rounds
    norm = math.sqrt(tot)
    max_norm = 1.0
    c = np.float32(max_norm / (norm + 1e-6))
    assert norm > max_norm and math.frexp(float(c))[0] != 0.5
    for gr in grads:
        ops.clip_scale(gr, gr.numel(), total, max_norm)
    torch.cuda.synchronize()
    cd = torch.tensor(c, device=dev)
    for gr, g0 in zip(grads, G0):
        assert torch.equal(gr.view(torch.int32), (g0 * cd).view(torch.int32))
    # no clipping: max_norm above the norm
    for p, g0 in zip(m.parameters(), G0):
        p.grad = g0.clone()
    got = rutils.clip_grad_norm_(m.parameters(), max_norm=2 * norm)
    for p, g0 in zip(m.parameters(), G0):
        assert torch.equal(p.grad.view(torch.int32), g0.view(torch.int32))
    q = [torch.nn.Parameter(g0.double()) for g0 in G0]
    for qq, g0 in zip(q, G0):
        qq.grad = g0.double()
    tn = float(torch.nn.utils.clip_grad_norm_(q, max_norm=2 * norm))
    print("  clip_grad_norm_: norm %.6g, rel err against torch float64 %.2e, clip factor %.8g bit-exact"
          % (float(got), abs(float(got) - tn) / tn, c))
    assert abs(float(got) - tn) <= 1e-12 * tn


@gpu
def test_refiner_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over the refiner's flat buffer with separate gradient tensors, as the refiner's
    backward produces them: 44 epb_adam_step calls and no epb_adam_step_dev per step, 42 slices on
    the float4 kernel and w2.bias / w4.bias (45 floats) on the scalar one.  Steps 1, 2 and 1000,
    every element within step_cases._adam_errors' float64 contract on the lr the kernel read from
    the host group; then refiner.utils.lr_decay halves the lr and the next step meets the
    contract on the decayed lr and misses it on the old one."""
    import lib.utils.utils as Ut
    from epipolarpose_b200.refiner import utils as rutils
    m, _ = _refiner(dev, 43)
    opt = Ut.FusedAdam(list(m.parameters()), lr=1e-3)
    names = [n for n, _ in m.named_parameters()]
    info = opt._flat[0]
    buf, params = info["buf"], opt.param_groups[0]["params"]
    f32 = lambda v: float(np.float32(v))

    def grads(seed):
        g = torch.Generator(device=dev).manual_seed(seed)
        G = torch.zeros_like(buf)
        for p, o, s in zip(params, info["offs"], info["sizes"]):
            gr = torch.randn(p.shape, device=dev, generator=g) * \
                torch.pow(10.0, torch.rand(p.shape, device=dev, generator=g) * 6 - 6)
            gr.view(-1)[::97] = 0
            p.grad = gr                                       # its own allocation
            G[o:o + s] = gr.reshape(-1)
        return G

    def step(t, seed, lr_read):
        G = grads(seed)
        st = opt.state.get("flat0")
        if t == 1000:
            st["step"] = 999
            st["step_dev"].fill_(999)
        P0 = buf.clone()
        m0 = st["exp_avg"].clone() if st and "exp_avg" in st else torch.zeros_like(buf)
        v0 = st["exp_avg_sq"].clone() if st and "exp_avg_sq" in st else torch.zeros_like(buf)
        with _count_calls() as counts:
            opt.step()
        torch.cuda.synchronize()
        assert counts["epb_adam_step"] == 44 and counts["epb_adam_step_dev"] == 0, counts
        st = opt.state["flat0"]
        b1, b2 = opt.param_groups[0]["betas"]
        out = {}
        for what, lr in lr_read.items():
            h = [f32(lr), f32(b1), f32(b2), f32(opt.param_groups[0]["eps"]), 0.0, 1.0]
            out[what], _ = sc._adam_errors(P0, G, m0, v0, h, t, buf, st["exp_avg"], st["exp_avg_sq"])
        return out

    G = grads(10)
    vec = [n for n, p, o, s in zip(names, params, info["offs"], info["sizes"])
           if s % 4 == 0 and all((a % 16) == 0 for a in (buf.data_ptr() + 4 * o, p.grad.data_ptr()))]
    del G
    assert len(vec) == 42 and set(names) - set(vec) == {"w2.bias", "w4.bias"}, sorted(set(names) - set(vec))
    print("  flat buffer %d floats, 44 slices: 42 float4, w2.bias / w4.bias scalar" % buf.numel())
    for t, seed in ((1, 11), (2, 12), (1000, 13)):
        sc._report("FusedAdam per tensor step %d" % t, step(t, seed, {"lr": 1e-3})["lr"])
    lr = rutils.lr_decay(opt, 100000, 1e-3, 100000, 0.5)
    assert lr == 5e-4 and opt.param_groups[0]["lr"] == lr
    r = step(1001, 14, {"decayed": lr, "old": 1e-3})
    print("  step 1001 after lr_decay: contract on the old lr: upd err / bar %.3g" % r["old"]["upd"])
    sc._report("FusedAdam step 1001, decayed lr", r["decayed"])
    assert r["old"]["upd"] > 100


# ------------------------------------------------------------------ 6. the training forward end to end
@gpu
def test_refiner_training_forward_vs_float64(dev):
    """One training forward at N = 64 with dropout 0.5 (the keep masks replayed through the
    oracle): p1, p2 and running_mean / running_var of all ten BatchNorms against
    oracle.restate_refiner.forward in float64; then the eval forward (bn_eval_affine on the
    updated running statistics) against the oracle's eval forward on those statistics.  Bar
    12 * 1024 * eps32 * max|.| per tensor."""
    from oracle import restate_refiner as rr
    m, sd = _refiner(dev, 47)
    x = torch.randn(NB, 45, generator=torch.Generator().manual_seed(47)).to(dev)
    torch.manual_seed(7)
    with torch.no_grad():
        p1, p2 = m(x)
    torch.manual_seed(7)
    masks = [(torch.rand(NB, L, device=dev) >= 0.5) for _ in range(10)]
    sd64 = {k: (v.to(dev, torch.float64) if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
    ns = {}
    with torch.no_grad():
        o1, o2 = rr.forward(sd64, x.double(), training=True, masks=masks, p_dropout=0.5, new_stats=ns)
    assert len(ns) == 20
    bar = lambda ref: 12 * L * EPS32 * float(ref.abs().max())
    ratio = lambda got, ref: float((got.double() - ref).abs().max()) / bar(ref)
    state = m.state_dict()
    r = {"p1": ratio(p1, o1), "p2": ratio(p2, o2),
         "running_mean": max(ratio(state[k], v) for k, v in ns.items() if k.endswith("running_mean")),
         "running_var": max(ratio(state[k], v) for k, v in ns.items() if k.endswith("running_var"))}
    for k in ns:                               # every running statistic moved
        assert not torch.equal(state[k].double(), sd64[k]), k
    m.eval()
    with torch.no_grad():
        e1, e2 = m(x)
        sd_e = dict(sd64, **{k: state[k].double() for k in ns})
        r1, r2 = rr.forward(sd_e, x.double(), training=False)
    r["eval p1"], r["eval p2"] = ratio(e1, r1), ratio(e2, r2)
    sc._report("refiner forward N %d" % NB, r)


@gpu
def test_refiner_one_row_batch_refused_on_device(dev):
    """On the device: a one-row training batch raises the ValueError of torch.nn.BatchNorm1d,
    and refiner/main.py train() stops on a loader whose last batch has one row."""
    import logging
    import types
    import lib.utils.utils as Ut
    from epipolarpose_b200.refiner import data as rdata, main as rmain
    m = _one_row_refused(dev, L)
    dl = torch.utils.data.DataLoader(rdata.SyntheticPoses(is_train=True, n=NB + 1, seed=3), batch_size=NB,
                                     shuffle=False)
    args = types.SimpleNamespace(lr=1e-3, lr_decay=100000, lr_gamma=0.96)
    opt = Ut.FusedAdam(list(m.parameters()), lr=args.lr)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        rmain.train(m, dl, opt, 0, args.lr, torch.nn.MSELoss(), args, logging.getLogger("refiner"))
