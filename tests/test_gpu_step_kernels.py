"""The training step's remaining kernels against float64 at the bench's sizes (R50, J = 16, D = 64,
256 x 256, N = 128): the optimisers (layout.cu adam_dev_kernel, adam_kernel / adam_kernel1, the
three SGD kernels), the batched weight split (split16.cu split_amax_kernel / split_apply_kernel /
find_job) and the weight pack, the stem's patch matrix (im2col_split) and max-pool backward, the
soft-argmax forward (coords and lse) and the joint loss.  Data is generated on the device; every
reference is torch float64 on the device, computed from the exact fp32 / fp16 values the kernel
read.  tests/test_step_coverage.py gates the f16x3 step on these tests.

Bars (u = 2^-24, one fp32 rounding); those shared with the other compositions are derived in the
docstring of the tests/step_cases.py function that computes them:

  * Adam, the contract and against torch.optim.Adam: _adam_bar.
  * SGD: g (2u), the momentum buffer b = mom buf + g (2u on its terms), nesterov g + mom b (2u on
    its terms), p - lr d (u on lr d, u |p1|).  Fused or separate roundings both stay inside.
  * Weight split, pack, im2col_split: bit-exact with the CPU emulation (tests/emul_ops.py):
    _check_split16_batch, _check_pack_weight_batch, _check_im2col_split.
  * maxpool_bwd: _check_maxpool_bwd.
  * Soft-argmax forward, NHWC: _check_softargmax_fwd.
  * Joint loss: _check_jointloss.

The CPU test below runs the Adam bar against a numpy fp32 emulation of the kernel's arithmetic and
shows that it fails for a bias correction one step off, eps inside the square root, a missing
weight decay, and 1 - beta taken from the other beta."""
import math

import numpy as np
import pytest
import torch

from tests.step_cases import (U, _adam_bar, _adam_errors, _check_fused_adam, _check_im2col_split, _check_jointloss,
                              _check_maxpool_bwd, _check_pack_weight_batch, _check_softargmax_fwd,
                              _check_split16_batch, _hyper64, _report, bench_model, check_bn_finalize)

gpu = pytest.mark.gpu


# ------------------------------------------------------------------ Adam: the bar has teeth
def _emul_adam(P, G, m, v, h, t, mistake=None):
    """adam_dev_kernel in numpy fp32, operation by operation; mistake names one plausible error"""
    f = np.float32
    lr, b1, b2, eps, wd, gs = (f(x) for x in h)
    tb = t + 1 if mistake == "bias_off_by_one" else t
    bc1 = f(1.0 - math.pow(float(b1), tb))
    rbc2 = f(1.0 / math.sqrt(1.0 - math.pow(float(b2), tb)))
    step = f(lr / bc1)
    g = (G * gs).astype(f)
    if wd != 0 and mistake != "no_weight_decay":
        g = (g + (wd * P).astype(f)).astype(f)
    c1 = f(1) - (b2 if mistake == "wrong_beta" else b1)
    m1 = ((b1 * m).astype(f) + (c1 * g).astype(f)).astype(f)
    v1 = ((b2 * v).astype(f) + ((f(1) - b2) * ((g * g).astype(f))).astype(f)).astype(f)
    if mistake == "eps_in_sqrt":
        den = np.sqrt(((v1 * rbc2).astype(f) * rbc2 + eps).astype(f)).astype(f)
    else:
        den = ((np.sqrt(v1).astype(f) * rbc2).astype(f) + eps).astype(f)
    P1 = (P - (step * (m1 / den).astype(f)).astype(f)).astype(f)
    return P1, m1, v1


def _adam_state(n, seed):
    """p, g with log-uniform magnitudes over 1e-6 .. 1 (zeros included), m / v one step in"""
    rng = np.random.default_rng(seed)
    f = np.float32
    P = (rng.standard_normal(n) * 0.05).astype(f)
    G = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 0, n)).astype(f)
    G[::97] = 0
    return P, G


@pytest.mark.parametrize("mistake", ["bias_off_by_one", "eps_in_sqrt", "no_weight_decay", "wrong_beta"])
def test_adam_bar_holds_for_the_kernel_order_and_rejects(mistake):
    """The fp32 emulation of adam_dev_kernel meets every bar at steps 1, 2 and 1000 with weight
    decay; the named mistake misses one of them."""
    h = [float(np.float32(x)) for x in (1e-3, 0.9, 0.999, 1e-8, 1e-2, 1.0)]
    P, G = _adam_state(1 << 16, 7)
    m0 = np.zeros_like(P)
    v0 = np.zeros_like(P)
    T = lambda a: torch.from_numpy(np.asarray(a))
    worst_ok, worst_bad = 0.0, 0.0
    P1, m1, v1 = _emul_adam(P, G, m0, v0, h, 1)
    for t in (2, 1000):
        Pa, Ga = P1, _adam_state(1 << 16, t)[1]
        Pb, mb, vb = _emul_adam(Pa, Ga, m1, v1, h, t)
        r, _ = _adam_errors(T(Pa), T(Ga), T(m1), T(v1), h, t, T(Pb), T(mb), T(vb))
        worst_ok = max(worst_ok, *r.values())
        Pc, mc, vc = _emul_adam(Pa, Ga, m1, v1, h, t, mistake)
        r, _ = _adam_errors(T(Pa), T(Ga), T(m1), T(v1), h, t, T(Pc), T(mc), T(vc))
        worst_bad = max(worst_bad, *r.values())
    print("emulated Adam: worst err / bar %.3f, with %s %.3g" % (worst_ok, mistake, worst_bad))
    assert worst_ok <= 1.0
    assert worst_bad > 1.0


# ------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


# ------------------------------------------------------------------ 1. optimiser
@gpu
def test_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over the bench model's parameters (R50/J16/D64, the real flat buffer), gradients
    in the flat layout: epb_adam_step_dev is the path taken.  Steps 1, 2 and 1000 (step_dev set
    to 999 first), update / m / v per element against the float64 contract, and the update
    against torch.optim.Adam on the same fp32 state."""
    _check_fused_adam(dev, *bench_model(dev, "c4_f16x3"))


ADAM_CASES = [("step1", 1, 0.0, 1.0), ("step2", 2, 0.0, 1.0), ("step1000", 1000, 0.0, 1.0),
              ("wd", 2, 1e-2, 1.0), ("gscale", 2, 0.0, 0.37), ("wd_gscale_1000", 1000, 5e-4, 3.0)]


@gpu
@pytest.mark.parametrize("case", ADAM_CASES, ids=[c[0] for c in ADAM_CASES])
def test_adam_dev_cases_vs_float64(dev, case):
    """epb_adam_step_dev on the bench model's buffer size with hyper-parameters FusedAdam does not
    set (weight decay, grad_scale != 1), zeros in the gradient, m / v from one earlier step."""
    from epipolarpose_b200 import ops
    _, opt = bench_model(dev, "c4_f16x3")
    n = opt._flat[0]["n"]
    name, t, wd, gs = case
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, wd, gs], device=dev)
    g = torch.Generator(device=dev).manual_seed(t + 7)
    P0 = torch.randn(n, device=dev, generator=g) * 0.05
    G = torch.randn(n, device=dev, generator=g) * torch.pow(10.0, torch.rand(n, device=dev, generator=g) * 6 - 6)
    G[::97] = 0
    m0 = torch.randn(n, device=dev, generator=g) * 1e-3 if t > 1 else torch.zeros(n, device=dev)
    v0 = (m0 * m0 * 3 + 1e-12) if t > 1 else torch.zeros(n, device=dev)
    P1, m1, v1 = P0.clone(), m0.clone(), v0.clone()
    step_dev = torch.tensor([t], device=dev, dtype=torch.int32)
    ops.adam_step_dev(P1, G, m1, v1, n, hyper, step_dev)
    torch.cuda.synchronize()
    r, _ = _adam_errors(P0, G, m0, v0, _hyper64(hyper), t, P1, m1, v1)
    _report("adam_step_dev %s" % name, r)


@gpu
def test_adam_per_tensor_paths_vs_float64(dev):
    """epb_adam_step (the per-tensor path FusedAdam takes when the gradients are not flat):
    the float4 kernel and the scalar kernel (misaligned slice, n % 4 != 0), same contract."""
    from epipolarpose_b200 import ops
    n = (1 << 20) + 3
    g = torch.Generator(device=dev).manual_seed(5)
    base = torch.randn(4, n + 1, device=dev, generator=g)
    h = [float(np.float32(x)) for x in (1e-3, 0.9, 0.999, 1e-8, 1e-2, 1.0)]
    for label, sl in (("float4", slice(0, n - 3)), ("scalar", slice(1, n + 1))):
        P0, G, m0, v0 = (base[i, sl].contiguous() for i in range(4))
        G = G * torch.pow(10.0, torch.rand(G.numel(), device=dev, generator=g) * 6 - 6)
        m0, v0 = m0 * 1e-3, m0 * m0 * 3e-6 + 1e-12
        P0 = P0 * 0.05
        k = P0.numel()
        off = 0 if label == "float4" else 1                  # separate allocations: 16-byte aligned or not
        P1, Gk, m1, v1 = (torch.empty(k + 1, device=dev)[off:off + k] for _ in range(4))
        for dst, src in ((P1, P0), (Gk, G), (m1, m0), (v1, v0)):
            dst.copy_(src)
        ops.adam_step(P1, Gk, m1, v1, k, h[0], h[1], h[2], h[3], h[4], 3)
        torch.cuda.synchronize()
        r, _ = _adam_errors(P0, G, m0, v0, h, 3, P1, m1, v1)
        _report("adam_step %s n=%d" % (label, k), r)


@gpu
def test_adam_dev_multi_step_drift(dev):
    """10 steps of epb_adam_step_dev from its own state against 10 float64 steps from the same
    start: m, v and p within the compounded bars."""
    from epipolarpose_b200 import ops
    _, opt = bench_model(dev, "c4_f16x3")
    n = opt._flat[0]["n"]
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0], device=dev)
    h = _hyper64(hyper)
    g = torch.Generator(device=dev).manual_seed(77)
    P = torch.randn(n, device=dev, generator=g) * 0.05
    mk, vk, Pk = torch.zeros(n, device=dev), torch.zeros(n, device=dev), P.clone()
    P64, m64, v64 = P.double(), torch.zeros(n, device=dev, dtype=torch.float64), torch.zeros(n, device=dev, dtype=torch.float64)
    Em = Ev = Ep = 0.0
    scale = torch.pow(10.0, torch.rand(n, device=dev, generator=g) * 6 - 6)
    step_dev = torch.zeros(1, device=dev, dtype=torch.int32)
    lr, b1, b2, eps = h[:4]
    for t in range(1, 11):
        G = torch.randn(n, device=dev, generator=g) * scale
        G[t::97] = 0
        step_dev += 1
        P0 = Pk.clone()
        ops.adam_step_dev(Pk, G, mk, vk, n, hyper, step_dev)
        # the bar's terms along the float64 trajectory, carried errors added
        em, ev, eupd, _ = _adam_bar(P64, G, m64, v64, h, t, Pk, Em, Ev)
        Ep = Ep + eupd
        Em, Ev = em, ev
        gd = G.double()
        m64 = b1 * m64 + (1 - b1) * gd
        v64 = b2 * v64 + (1 - b2) * gd * gd
        P64 = P64 - (lr / (1 - b1 ** t)) * m64 / (v64.sqrt() / math.sqrt(1 - b2 ** t) + eps)
        del P0
    torch.cuda.synchronize()
    r = {"m": float(((mk.double() - m64).abs() / (Em + 1e-300)).max()),
         "v": float(((vk.double() - v64).abs() / (Ev + 1e-300)).max()),
         # P64 holds p exactly, Pk rounds each step: u |p| per step is inside Ep
         "p": float(((Pk.double() - P64).abs() / (Ep + 1e-300)).max())}
    _report("adam_step_dev 10 steps", r)


SGD_CASES = [(mom, nest, first, wd) for mom in (0.0, 0.9) for nest in (False, True) for first in (True, False)
             for wd in (0.0, 1e-3) if not (mom == 0.0 and nest)]


def _sgd_bar(P, G, buf, lr, mom, wd, nest, first, gs, P1):
    g = G.double() * gs + wd * P.double()
    eg = 2 * U * ((G.double() * gs).abs() + (wd * P.double()).abs())
    if mom:
        b = g if first else mom * buf.double() + g
        eb = eg if first else eg + 2 * U * ((mom * buf.double()).abs() + g.abs())
        d = g + mom * b if nest else b
        ed = eg + mom * eb + 2 * U * (g.abs() + (mom * b).abs()) if nest else eb
    else:
        b, eb, d, ed = None, None, g, eg
    return b, eb, -lr * d, lr * (ed + U * d.abs()) + U * P1.double().abs()


@gpu
@pytest.mark.parametrize("path", ["vec", "scalar", "dev"])
def test_sgd_paths_vs_float64(dev, path):
    """epb_sgd_step (float4 kernel; scalar kernel on a misaligned slice with n % 4 != 0) and
    epb_sgd_step_dev: momentum 0 / 0.9, nesterov, first step or not, weight decay, grad_scale."""
    from epipolarpose_b200 import ops
    n = (1 << 20) + (0 if path == "vec" else 3)
    g = torch.Generator(device=dev).manual_seed(9)
    worst = 0.0
    for mom, nest, first, wd in SGD_CASES:
        gs = 0.37 if path != "vec" else 1.0
        off = 1 if path == "scalar" else 0                   # separate allocations: 16-byte aligned or not
        P1, G, B1 = (torch.randn(n + 1, device=dev, generator=g)[off:off + n] for _ in range(3))
        G *= torch.pow(10.0, torch.rand(n, device=dev, generator=g) * 6 - 6)
        G[::97] = 0
        P0, B0 = P1.clone(), B1.clone()
        lr = 1e-2
        if path == "dev":
            hyper = torch.tensor([lr, mom, wd, 1.0 if nest else 0.0, gs], device=dev)
            ops.sgd_step_dev(P1, G, B1, n, hyper, torch.tensor([1 if first else 5], device=dev, dtype=torch.int32))
            lr, mom, wd, gs = (float(v) for v in hyper[[0, 1, 2, 4]].double().cpu())
        else:
            ops.sgd_step(P1, G, B1, n, lr, mom, wd, nest, first, gs)
            lr, mom, wd, gs = (float(np.float32(v)) for v in (lr, mom, wd, gs))
        torch.cuda.synchronize()
        b, eb, upd, eupd = _sgd_bar(P0, G, B0, lr, mom, wd, nest, first, gs, P1)
        r = float((((P1.double() - P0.double()) - upd).abs() / (eupd + 1e-300)).max())
        if b is not None:
            r = max(r, float(((B1.double() - b).abs() / (eb + 1e-300)).max()))
        else:
            assert torch.equal(B1, B0)                     # momentum 0 leaves the buffer alone
        worst = max(worst, r)
        assert r <= 1.0, (path, mom, nest, first, wd, r)
    print("  sgd %-6s worst err / bar %.3f over %d cases" % (path, worst, len(SGD_CASES)))


@gpu
def test_graph_replay_follows_a_nonzero_lr_change(dev):
    """FusedAdam.step captured in a CUDA graph; after lr 1e-3 -> 3e-4 through sync_hyper the replay
    equals an eager epb_adam_step_dev with lr = 3e-4 on the same state, bit for bit, and differs
    from the lr = 1e-3 result."""
    import lib.utils.utils as U
    from epipolarpose_b200 import ops
    torch.manual_seed(3)
    ps = [torch.nn.Parameter(torch.randn(s, device=dev)) for s in ((64, 3, 7, 7), (256,), (1000, 17))]
    opt = U.FusedAdam(ps, lr=1e-3)
    info = opt._flat[0]
    G = torch.randn(info["n"], device=dev)
    for p, o, s in zip(ps, info["offs"], info["sizes"]):
        p.grad = G[o:o + s].view(p.shape)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        opt.step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        opt.step()
    st = opt.state["flat0"]
    for gr in opt.param_groups:
        gr["lr"] = 3e-4
    opt.sync_hyper()
    torch.cuda.synchronize()
    snap = [t.clone() for t in (info["buf"], st["exp_avg"], st["exp_avg_sq"])]
    t_before = int(st["step_dev"])
    graph.replay()
    torch.cuda.synchronize()
    assert int(st["step_dev"]) == t_before + 1
    want = {}
    for lr in (3e-4, 1e-3):
        p, m_, v_ = (t.clone() for t in snap)
        ops.adam_step_dev(p, G, m_, v_, info["n"], torch.tensor([lr, 0.9, 0.999, 1e-8, 0.0, 1.0], device=dev),
                          torch.tensor([t_before + 1], device=dev, dtype=torch.int32))
        want[lr] = p
    torch.cuda.synchronize()
    assert torch.equal(info["buf"], want[3e-4])
    assert not torch.equal(info["buf"], want[1e-3])
    assert not torch.equal(info["buf"], snap[0])


@gpu
@pytest.mark.parametrize("M", [524288, 2097152])
def test_bn_finalize_vs_float64_at_bench_M(dev, M):
    check_bn_finalize(dev, M)


# ------------------------------------------------------------------ 2. weight split and pack at model scale
@gpu
def test_split16_batch_bit_exact_on_model_jobs(dev):
    """split16_batch on the jobs the f16x3 engine builds for R50/J16/D64 (after one Adam step) plus
    synthetic jobs in the same batch (all zeros, amax in the last partial block, amax a power of
    two, 1 / 3 / 2049 elements, 2^24 + 5 elements): bit-exact with the CPU emulation, planes as
    int16 and both scale words; s = pow2_scale(amax), max|hi| <= 2^14, no +-65504."""
    _check_split16_batch(dev, *bench_model(dev, "c4_f16x3"))


@gpu
def test_pack_weight_batch_bit_exact_on_model_jobs(dev):
    """pack_weight_batch on the engine's model-scale jobs (R50/J16/D64): the fprop / dgrad operand
    pack of every layer and the per-stage unpack of the weight gradients, bit-exact with the CPU
    emulation (a permutation: no arithmetic)."""
    _check_pack_weight_batch(dev, bench_model(dev, "c4_f16x3")[0])


# ------------------------------------------------------------------ 3. stem at the bench size
@gpu
def test_im2col_split_bit_exact_at_stem_bench_size(dev):
    """im2col_split over all 128 images of 256 x 256 (7 x 7 / 2, pad 3): bit-exact with the CPU
    emulation on the first, last and three middle images."""
    _check_im2col_split(dev, bench_model(dev, "c4_f16x3")[0]._engine().stem_kpad, 128, 256)


@gpu
def test_maxpool_bwd_vs_float64_at_stem_bench_size(dev):
    """The stem's pool at the bench size (N = 128, 128 x 128 x 64): argidx from
    bn_relu_maxpool_split on dyadic inputs (exact fma, many ties), fp32 dy.  maxpool_bwd against a
    float64 scatter within 3u sum|g|, bit-equal with an fp32 restatement adding in (kh, kw)
    order; where argidx differs from torch.max_pool2d's index the window holds a tie."""
    _check_maxpool_bwd(dev, 128, 128)


# ------------------------------------------------------------------ 4. soft-argmax forward and joint loss
@gpu
@pytest.mark.parametrize("kind", ["randn3", "peaks60", "constant"])
def test_softargmax_fwd_vs_float64_at_bench_shape(dev, kind):
    """N = 128, J = 16, D = 64, 64 x 64, NHWC (2.1 GB of logits): coords against float64 within
    the merge-depth bar, lse[0] the exact maximum, lse[1] * sum exp(v - m) - 1 within its bar.
    randn3: logits x 3 as in the backward test; peaks60: one logit of 60 per (image, joint);
    constant: every logit 0.7 (the uniform distribution)."""
    _check_softargmax_fwd(dev, kind, 128, 16, 64, 64, 64)


@gpu
@pytest.mark.parametrize("kind,norm", [(2, 0), (1, 0), (1, 1), (2, 1)], ids=["smoothl1", "l1", "l1_norm", "smoothl1_norm"])
def test_jointloss_vs_float64_at_bench_shape(dev, kind, norm):
    """epb_jointloss_fwd_bwd at N = 128, J = 16 (6144 elements), weights with zeros, |d| on both
    sides of 1 and exactly 1 (dyadic x, t: d exact without norm): loss and dx against float64."""
    _check_jointloss(dev, kind, norm, 128, 16)
