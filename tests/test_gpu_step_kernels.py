"""The training step's remaining kernels against float64 at the bench's sizes, and a coverage gate:
every C-ABI entry one bench-composition step calls must name the tests that hold it to float64.

Kernels: the optimisers (layout.cu adam_dev_kernel, adam_kernel / adam_kernel1, the three SGD
kernels), the batched weight split (split16.cu split_amax_kernel / split_apply_kernel / find_job)
and the weight pack, the stem's patch matrix (im2col_split) and max-pool backward, the soft-argmax
forward (coords and lse) and the joint loss.  Data is generated on the device; every reference is
torch float64 on the device, computed from the exact fp32 / fp16 values the kernel read.

Bars (u = 2^-24, one fp32 rounding):

  * Adam, the contract: Adam with lr, beta1, beta2, eps, wd, grad_scale AS STORED in the fp32
    `hyper` tensor, the bias corrections from those fp32 betas in double.  The kernel rounds
    g = G gs (+ wd P) (e_g <= 2u (|G gs| + |wd P|)), then m = b1 m0 + (1-b1) g and v = b2 v0 +
    (1-b2) g^2 (1-b fp32 is exact for b in [0.5, 1]).  m and v cancel, so their bars are on the
    terms, not on the result: e_m = (1-b1) e_g + 3u (|b1 m0| + |(1-b1) g|), e_v = 2 (1-b2) |g| e_g +
    4u (b2 v0 + (1-b2) g^2).  sqrt moves e_v to e_v / max(sqrt v, sqrt e_v); the denominator
    sqrt(v) rsqrt_bc2 + eps adds three roundings (rsqrt_bc2 stored in fp32, the product, + eps),
    the quotient one, lr / bc1 two, the product one, and p - step q rounds once more, to
    u |p1|.  The update p1 - p0 is compared, not p1, so that last term is the only one that
    depends on |p|.  K steps from the kernel's own state: m and v errors carry over as
    E_m <- b1 E_m + e_m, E_v <- b2 E_v + e_v, the parameter error adds each step's update bar.
  * Adam against torch.optim.Adam (fp32, same state): torch keeps the betas in double, so
    (1-b1), (1-b2) and the bias corrections differ by their fp32 rounding (r_c1 ~ 2.4e-7,
    r_c2 ~ 1.3e-5, measured here from the stored values) on top of both implementations'
    roundings (2x the kernel's u terms) and both final roundings of p.
  * SGD: g (2u), the momentum buffer b = mom buf + g (2u on its terms), nesterov g + mom b (2u on
    its terms), p - lr d (u on lr d, u |p1|).  Fused or separate roundings both stay inside.
  * Weight split, pack, im2col_split: bit-exact with the CPU emulation (tests/emul_ops.py):
    planes compared as int16, both scale words; the scale is pow2_scale(amax), max|hi| <= 2^14.
  * maxpool_bwd: each input element sums at most 4 window gradients in (kh, kw) order from 0:
    <= 3u sum|g| against float64, and bit-equal with an fp32 restatement in that order.
  * Soft-argmax forward, NHWC: a logit's term exp(v - m) meets d = L + 2 + D4 ppi + S additions
    (L pixels per thread, the quad, the CTA merge of D4 ppi partials, the S-way finalize) and at
    most as many rescale factors exp(m_a - m_b).  With the backward test's __expf model
    ((6 + 3.5|x|) u) and rescale arguments that add up to at most |v - m|, the factor a term
    carries into s, sx, sy, sz alike is off by eps_i <= (6 + 7|v - m| + 6 d) u; on top, each of
    those positive sums is off by 2 d u relative from its own additions and rescale products.
    So a coordinate c' = c + 1/2 is off by sum_i p_i |pos_i - c'| eps_i + 4 d u c' + 4u, lse[1]
    = 1 / sum exp(v - m) by sum_i p_i eps_i + 2 d u + 2u, and lse[0] is the maximum: exact.
  * Joint loss (one CTA of 1024 threads): each thread adds n / 1024 terms, then a 10-level tree:
    depth dl = n / 1024 + 12, |d loss| <= dl u sum|w l| / div.  Without norm x and t are dyadic,
    d is exact and dx rounds at most twice.  With norm, 1 / sum|x| and 1 / sum|t| carry dl + 1
    roundings into every d (ed = (dl + 3) u (|x_n| + |t_n|)), and the norm term of dx sums
    g x over all elements (3 dl + 6 roundings on sum|g x| / sum|x|^2).

The CPU tests below run the Adam bar against a numpy fp32 emulation of the kernel's arithmetic and
show that it fails for a bias correction one step off, eps inside the square root, a missing
weight decay, and 1 - beta taken from the other beta; and run the CPU half of the coverage gate
through the emulated ABI."""
import importlib
import inspect
import math
import re

import numpy as np
import pytest
import torch

gpu = pytest.mark.gpu

U = 2.0 ** -24
HALF_MAX = 65504.0
NUM_SMS = 132          # common.cuh kNumSMs
LOSS_THREADS = 1024    # softargmax.cu kLossThreads

# ------------------------------------------------------------------ coverage table
# C-ABI entry of the bench step -> tests that check it against float64 (or bit-exact against an
# exact restatement) at the bench's sizes.  C3 (test_c3_selfsup_chain_64_images) runs the geometry
# on 16 tuples x 4 views: half the bench's batch of 32 tuples.
COVERAGE = {
    "epb_im2col_split": ["test_gpu_step_kernels.py::test_im2col_split_bit_exact_at_stem_bench_size"],
    "epb_conv16_fprop": ["test_gpu_split16.py::test_conv16_bench_layer_shapes_vs_torch_float64",
                         "test_gpu_bn_chain.py::test_conv16_stats_vs_float64"],
    "epb_conv16_wgrad": ["test_gpu_split16.py::test_conv16_bench_layer_shapes_vs_torch_float64"],
    "epb_bn_finalize_scale": ["test_gpu_bn_chain.py::test_bn_finalize_scale_vs_float64"],
    "epb_bn_finalize": ["test_gpu_step_kernels.py::test_bn_finalize_vs_float64_at_bench_M",
                        "test_gpu_split16.py::test_bn_finalize_scale_vs_two_calls"],
    "epb_act_scale": ["test_gpu_bn_chain.py::test_scale_contract_adversarial"],
    "epb_bn_act_split": ["test_gpu_bn_chain.py::test_bn_act_split_vs_float64_at_bench_M"],
    "epb_bn_relu_maxpool_split": ["test_gpu_bn_chain.py::test_bn_relu_maxpool_split_vs_float64_at_stem_size"],
    "epb_maxpool_bwd": ["test_gpu_step_kernels.py::test_maxpool_bwd_vs_float64_at_stem_bench_size"],
    "epb_bn_bwd_split": ["test_gpu_bn_chain.py::test_bn_bwd_split_vs_float64_at_bench_M"],
    "epb_softargmax_fwd": ["test_gpu_step_kernels.py::test_softargmax_fwd_vs_float64_at_bench_shape"],
    "epb_softargmax_bwd_split": ["test_gpu_bn_chain.py::test_softargmax_bwd_split_vs_float64_at_bench_shape"],
    "epb_jointloss_fwd_bwd": ["test_gpu_step_kernels.py::test_jointloss_vs_float64_at_bench_shape"],
    "epb_split16_batch": ["test_gpu_step_kernels.py::test_split16_batch_bit_exact_on_model_jobs"],
    "epb_split16": ["test_gpu_step_kernels.py::test_split16_batch_bit_exact_on_model_jobs"],
    "epb_pack_weight_batch": ["test_gpu_step_kernels.py::test_pack_weight_batch_bit_exact_on_model_jobs"],
    "epb_adam_step_dev": ["test_gpu_step_kernels.py::test_fused_adam_vs_float64_on_model_buffer",
                          "test_gpu_step_kernels.py::test_adam_dev_cases_vs_float64",
                          "test_gpu_step_kernels.py::test_adam_dev_multi_step_drift"],
    "epb_adam_step": ["test_gpu_step_kernels.py::test_adam_per_tensor_paths_vs_float64"],
    "epb_patch_to_image": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
    "epb_triangulate": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
    "epb_project_labels": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
}


def _missing_coverage(recorded, table=COVERAGE):
    """entries without a row, and rows that name a test function that does not exist"""
    missing = sorted(set(recorded) - set(table))
    dangling = []
    for entry in sorted(set(recorded) & set(table)):
        for tid in table[entry]:
            mod, _, fn = tid.partition("::")
            m = importlib.import_module("tests." + mod[:-3])
            if not callable(getattr(m, fn, None)):
                dangling.append((entry, tid))
    return missing, dangling


def _entry_names(mod_ops):
    """ops wrapper name -> the C-ABI entries it calls"""
    out = {}
    for k, f in vars(mod_ops).items():
        if inspect.isfunction(f) and f.__module__ == mod_ops.__name__:
            e = re.findall(r'_call\("(epb_[a-z0-9_]+)"', inspect.getsource(f))
            if e:
                out[k] = e
    return out


def _bench_meta(tuples, seed=1000):
    """the bench's synthetic cameras / boxes for `tuples` 4-view tuples (bench.py run_gpu)"""
    from lib.dataset.synthetic import ring_camera
    rng = np.random.default_rng(seed)
    n = 4 * tuples
    order = [(t, 0) for t in range(tuples)] + [(t, 3) for t in range(tuples)] + \
            [(t, 1) for t in range(tuples)] + [(t, 2) for t in range(tuples)]
    cams = {(t, v): ring_camera(rng, v) for t in range(tuples) for v in range(4)}
    meta = {"center_x": torch.tensor(500 + rng.uniform(-50, 50, n)),
            "center_y": torch.tensor(500 + rng.uniform(-50, 50, n)),
            "width": torch.tensor(800 + rng.uniform(-100, 100, n)),
            "height": torch.tensor(800 + rng.uniform(-100, 100, n)),
            "scale": torch.ones(n, dtype=torch.float64), "rot": torch.zeros(n, dtype=torch.float64)}
    for i, k in enumerate(("R", "T", "f", "c", "projection_matrix")):
        meta[k] = torch.tensor(np.stack([cams[o][i] for o in order]))
    return meta


def _cfg(layers, J, D, HW):
    from oracle import refshim
    return refshim.make_cfg(num_layers=layers, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))


def test_coverage_gate_has_teeth():
    """Deleting a row, or pointing one at a test that does not exist, fails the gate."""
    rec = ["epb_adam_step_dev", "epb_maxpool_bwd"]
    assert _missing_coverage(rec) == ([], [])
    t = dict(COVERAGE)
    del t["epb_maxpool_bwd"]
    assert _missing_coverage(rec, t)[0] == ["epb_maxpool_bwd"]
    t = dict(COVERAGE, epb_adam_step_dev=["test_gpu_step_kernels.py::test_no_such_test"])
    assert _missing_coverage(rec, t)[1]


def test_coverage_gate_cpu_emulated_step():
    """One f16x3 training step (R18, J = 16, D = 64, 2 tuples x 4 views of 64 x 64) through the
    emulated ABI: GraphedTrainStep.eager_step, SmoothL1JointLocationLoss, FusedAdam.  The epipolar
    labels (epb_triangulate, epb_project_labels) have no CPU emulation, so this half runs the
    step with given labels; the GPU half below runs it online.  Nested emulations (an emulated
    entry that calls another) count as their outer entry only."""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.utils as U
    from epipolarpose_b200 import ops
    from tests import emul_ops
    rec, depth, saved = set(), [0], {}
    for k, e in _entry_names(ops).items():
        if not hasattr(emul_ops, k):
            continue
        f = saved[k] = getattr(emul_ops, k)

        def wrap(*a, _f=f, _e=e, **kw):
            if depth[0] == 0:
                rec.update(_e)
            depth[0] += 1
            try:
                return _f(*a, **kw)
            finally:
                depth[0] -= 1
        setattr(emul_ops, k, wrap)
    il._backend[0], U._backend[0] = emul_ops, emul_ops
    try:
        J, D, HW, B = 16, 64, 64, 8
        torch.manual_seed(0)
        m = models.pose3d_resnet.get_pose_net(_cfg(18, J, D, HW), False, ops=emul_ops, precision="f16x3").train()
        opt = U.FusedAdam(list(m.parameters()), lr=1e-3)
        step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J), opt, online=False)
        g = torch.Generator().manual_seed(1)
        loss = step.eager_step(torch.randn(B, 3, HW, HW, generator=g), torch.rand(B, J * 3, generator=g) - 0.5,
                               torch.ones(B, J * 3), None)
        assert math.isfinite(float(loss))
    finally:
        for k, f in saved.items():
            setattr(emul_ops, k, f)
        il._backend[0] = U._backend[0] = ops
    print("emulated step calls: %s" % sorted(rec))
    assert "epb_adam_step_dev" in rec and "epb_split16_batch" in rec
    missing, dangling = _missing_coverage(rec)
    assert not missing, "entries without a float64 test at bench size: %s" % missing
    assert not dangling, dangling


# ------------------------------------------------------------------ Adam: bars shared by CPU and GPU
def _hyper64(hyper):
    return [float(v) for v in hyper.double().cpu()]


def _adam64(P, G, m0, v0, h, t):
    """float64 Adam on the fp32 state with the stored fp32 hyper-parameters h"""
    lr, b1, b2, eps, wd, gs = h
    g = G.double() * gs + wd * P.double()
    m = b1 * m0.double() + (1 - b1) * g
    v = b2 * v0.double() + (1 - b2) * g * g
    bc1, rbc2 = 1 - b1 ** t, 1 / math.sqrt(1 - b2 ** t)
    den = v.sqrt() * rbc2 + eps
    return g, m, v, den, -(lr / bc1) * m / den


def _adam_bar(P, G, m0, v0, h, t, P1, Em=0.0, Ev=0.0, k=1.0, torch_ref=None):
    """(e_m, e_v, e_upd) of the module docstring; Em / Ev carried errors of m0 / v0;
    k scales the rounding terms; torch_ref: (r_c1, r_c2, r_b1, r_b2, r_lr, r_bc1, r_bc2)"""
    lr, b1, b2, eps, wd, gs = h
    g, m, v, den, upd = _adam64(P, G, m0, v0, h, t)
    c1, c2 = 1 - b1, 1 - b2
    eg = k * 2 * U * ((G.double() * gs).abs() + (wd * P.double()).abs())
    em = b1 * Em + c1 * eg + k * 3 * U * ((b1 * m0.double()).abs() + c1 * g.abs())
    ev = b2 * Ev + 2 * c2 * g.abs() * eg + c2 * eg * eg + k * 4 * U * (b2 * v0.double() + c2 * g * g)
    step_rel = k * 3 * U
    rbc2 = 1 / math.sqrt(1 - b2 ** t)
    sq = v.sqrt()
    den_extra = 0.0
    if torch_ref is not None:
        r_c1, r_c2, r_b1, r_b2, r_lr, r_bc1, r_bc2 = torch_ref
        em = em + r_c1 * c1 * g.abs() + r_b1 * (b1 * m0.double()).abs()
        ev = ev + r_c2 * c2 * g * g + r_b2 * b2 * v0.double()
        step_rel += r_lr + r_bc1
        den_extra = 0.5 * r_bc2 * rbc2 * sq
    esq = ev / torch.maximum(sq, ev.sqrt()).clamp_min(1e-300) + k * U * sq
    eden = rbc2 * esq + k * 3 * U * rbc2 * sq + k * U * den + den_extra
    q = m / den
    eq = (em + q.abs() * eden) / (den - eden).clamp_min(1e-300) + k * U * q.abs()
    step = lr / (1 - b1 ** t)
    eupd = step * (eq + step_rel * q.abs()) + U * P1.double().abs()
    return em, ev, eupd, (g, m, v, upd)


def _adam_errors(P0, G, m0, v0, h, t, P1, m1, v1, Em=0.0, Ev=0.0):
    em, ev, eupd, (_, m, v, upd) = _adam_bar(P0, G, m0, v0, h, t, P1, Em, Ev)
    tiny = 1e-300
    r = {"m": float(((m1.double() - m).abs() / (em + tiny)).max()),
         "v": float(((v1.double() - v).abs() / (ev + tiny)).max()),
         "upd": float((((P1.double() - P0.double()) - upd).abs() / (eupd + tiny)).max())}
    return r, (em, ev, eupd, m, v, upd)


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


def _record_calls():
    """context: the set of C-ABI entries called through ops._call (as bench.py's timed_call)"""
    from epipolarpose_b200 import ops

    class Rec:
        def __enter__(self):
            self.names, self.orig = set(), ops._call

            def call(name, *a):
                self.names.add(name)
                return self.orig(name, *a)
            ops._call = call
            return self.names

        def __exit__(self, *exc):
            ops._call = self.orig
    return Rec()


_MODEL = {}


def _r50(dev):
    """the bench model (R50, J = 16, D = 64, 256 x 256, f16x3) with FusedAdam over its parameters"""
    if "m" not in _MODEL:
        import lib.models as models
        import lib.utils.utils as U
        torch.manual_seed(0)
        m = models.pose3d_resnet.get_pose_net(_cfg(50, 16, 64, 256), False, precision="f16x3").to(dev).train()
        _MODEL["m"] = m
        _MODEL["opt"] = U.FusedAdam(list(m.parameters()), lr=1e-3)
    return _MODEL["m"], _MODEL["opt"]


def _flat_grads(opt, dev, seed):
    """a gradient buffer in the optimiser's flat layout (as the model's backward emits it), with
    log-uniform magnitudes and zeros; every p.grad a view of it"""
    info = opt._flat[0]
    n = info["n"]
    g = torch.Generator(device=dev).manual_seed(seed)
    G = torch.randn(n, device=dev, generator=g) * torch.pow(10.0, torch.rand(n, device=dev, generator=g) * 6 - 6)
    G[::97] = 0
    for p, o, s in zip(opt.param_groups[0]["params"], info["offs"], info["sizes"]):
        p.grad = G[o:o + s].view(p.shape)
    return G


def _report(what, r):
    print("  %-34s worst err / bar: %s" % (what, "  ".join("%s %.3f" % kv for kv in r.items())))
    assert max(r.values()) <= 1.0, (what, r)


# ------------------------------------------------------------------ 2. optimiser
@gpu
def test_fused_adam_vs_float64_on_model_buffer(dev):
    """FusedAdam over the bench model's parameters (R50/J16/D64, the real flat buffer), gradients
    in the flat layout: epb_adam_step_dev is the path taken.  Steps 1, 2 and 1000 (step_dev set
    to 999 first), update / m / v per element against the float64 contract, and the update
    against torch.optim.Adam on the same fp32 state."""
    _check_fused_adam(dev, *_r50(dev))


def _check_fused_adam(dev, m, opt):
    st_key = "flat0"
    opt.state.pop(st_key, None)                             # from step 1, whatever ran before
    buf = opt._flat[0]["buf"]
    print("  flat buffer: %d floats" % buf.numel())
    for t, seed in ((1, 11), (2, 12), (1000, 13)):
        G = _flat_grads(opt, dev, seed)
        st = opt.state.get(st_key)
        if t == 1000:
            st["step_dev"].fill_(999)
            st["step"] = 999
        P0 = buf.clone()
        m0 = st["exp_avg"].clone() if st else torch.zeros_like(buf)
        v0 = st["exp_avg_sq"].clone() if st else torch.zeros_like(buf)
        with _record_calls() as names:
            opt.step()
        torch.cuda.synchronize()
        assert "epb_adam_step_dev" in names and "epb_adam_step" not in names, names
        st = opt.state[st_key]
        assert int(st["step_dev"]) == t
        h = _hyper64(st["hyper"])
        r, (em, ev, eupd, m64, v64, upd64) = _adam_errors(P0, G, m0, v0, h, t, buf, st["exp_avg"], st["exp_avg_sq"])
        _report("FusedAdam step %d" % t, r)
        # torch.optim.Adam, fp32 on the device, from the same state
        q = torch.nn.Parameter(P0.clone())
        ta = torch.optim.Adam([q], lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
        q.grad = G.clone()
        ta.state[q] = {"step": torch.tensor(float(t - 1)), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
        ta.step()
        b1f, b2f = h[1], h[2]
        ref = (abs((1 - b1f) / 0.1 - 1), abs((1 - b2f) / 0.001 - 1), abs(b1f / 0.9 - 1), abs(b2f / 0.999 - 1),
               abs(h[0] / 1e-3 - 1), abs((1 - b1f ** t) / (1 - 0.9 ** t) - 1), abs((1 - b2f ** t) / (1 - 0.999 ** t) - 1))
        _, _, eupd_t, _ = _adam_bar(P0, G, m0, v0, h, t, buf, k=2.0, torch_ref=ref)
        eupd_t = eupd_t + U * q.detach().double().abs()
        dt = ((buf.double() - P0.double()) - (q.detach().double() - P0.double())).abs()
        _report("vs torch.optim.Adam step %d" % t, {"upd": float((dt / (eupd_t + 1e-300)).max())})
        del q, ta, em, ev, eupd, m64, v64, upd64, dt, eupd_t
    for p in m.parameters():
        p.grad = None


ADAM_CASES = [("step1", 1, 0.0, 1.0), ("step2", 2, 0.0, 1.0), ("step1000", 1000, 0.0, 1.0),
              ("wd", 2, 1e-2, 1.0), ("gscale", 2, 0.0, 0.37), ("wd_gscale_1000", 1000, 5e-4, 3.0)]


@gpu
@pytest.mark.parametrize("case", ADAM_CASES, ids=[c[0] for c in ADAM_CASES])
def test_adam_dev_cases_vs_float64(dev, case):
    """epb_adam_step_dev on the bench model's buffer size with hyper-parameters FusedAdam does not
    set (weight decay, grad_scale != 1), zeros in the gradient, m / v from one earlier step."""
    from epipolarpose_b200 import ops
    _, opt = _r50(dev)
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
    _, opt = _r50(dev)
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
    """epb_bn_finalize (the layers whose post-activation scale comes from elsewhere): every output
    within 1 fp32 ulp of float64 on the same statistics, gamma < 0 and = 0 channels, constant
    channels, running statistics."""
    from epipolarpose_b200 import ops
    from tests.test_gpu_bn_chain import EPS, MOM, _finalize64, _ulps
    C = 256
    rng = np.random.default_rng(M + 1)
    mean = rng.standard_normal(C) * 3
    var = rng.uniform(0.01, 4, C)
    var[:4] = 0
    g = rng.uniform(0.5, 1.5, C).astype(np.float32)
    g[4:12] *= -1
    g[12:16] = 0
    b = (rng.standard_normal(C) * 0.3).astype(np.float32)
    rm0, rv0 = rng.standard_normal(C).astype(np.float32), rng.uniform(0.5, 2, C).astype(np.float32)
    st = torch.tensor(np.concatenate([mean * M, (var + mean * mean) * M]), device=dev)
    T = lambda a: torch.tensor(a, device=dev)
    rm, rv = T(rm0.copy()), T(rv0.copy())
    out = {k: torch.empty(C, device=dev) for k in ("scale", "shift", "mean", "invstd")}
    ops.bn_finalize(st, M, C, T(g), T(b), EPS, MOM, rm, rv, out["scale"], out["shift"], out["mean"], out["invstd"])
    torch.cuda.synchronize()
    ref = _finalize64(st[:C].cpu().numpy(), st[C:].cpu().numpy(), M, g, b, rm0, rv0)
    worst = 0.0
    for k, t in dict(out, rm=rm, rv=rv).items():
        u = _ulps(t.cpu().numpy(), ref[k])
        worst = max(worst, float(u.max()))
        assert u.max() <= 1, "%s: %.2f ulp at channel %d" % (k, u.max(), u.argmax())
    print("  bn_finalize M %d: worst %.2f ulp" % (M, worst))


# ------------------------------------------------------------------ 3. weight split and pack at model scale
def _synthetic_split_jobs(dev):
    g = torch.Generator(device=dev).manual_seed(41)
    out = {"zeros": torch.zeros(5000, device=dev)}
    v = torch.randn(3 * 2048 + 100, device=dev, generator=g) * 0.1
    v[-7] = -3.0                                             # amax in the last, partial block
    out["amax_last_block"] = v
    v = (torch.rand(4099, device=dev, generator=g) * 2 - 1) * 3.9
    v[1234] = -4.0                                           # amax an exact power of two
    out["amax_pow2"] = v
    for k in (1, 3, 2049):
        out["n%d" % k] = torch.randn(k, device=dev, generator=g) * 0.01 + 1e-3
    v = torch.randn((1 << 24) + 5, device=dev, generator=g) * 1e-2
    v[(1 << 23) + 77] = 0.75                                 # one amax deep inside a 2^24-element job
    out["n2^24+5"] = v
    return out


def _grad_rule(bound):
    if not bound > 0 or not math.isfinite(bound):
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 13 - (math.frexp(bound)[1] - 1))))


@gpu
def test_split16_batch_bit_exact_on_model_jobs(dev):
    """split16_batch on the jobs the f16x3 engine builds for R50/J16/D64 (after one Adam step) plus
    synthetic jobs in the same batch (all zeros, amax in the last partial block, amax a power of
    two, 1 / 3 / 2049 elements, 2^24 + 5 elements): bit-exact with the CPU emulation, planes as
    int16 and both scale words; s = pow2_scale(amax), max|hi| <= 2^14, no +-65504."""
    _check_split16_batch(dev, *_r50(dev))


def _check_split16_batch(dev, m, opt):
    from epipolarpose_b200 import ops
    from tests import emul_ops
    if "flat0" not in opt.state:
        _flat_grads(opt, dev, 31)
        opt.step()
        for p in m.parameters():
            p.grad = None
    eng = m._engine()
    eng.dev = dev
    params = dict(m.named_parameters())
    with torch.no_grad():
        packed = eng._pack_weights(params)
    srcs = [(name, t) for name, pair in packed.items() for t in pair if t is not None]
    srcs += list(_synthetic_split_jobs(dev).items())
    jobs = [(t.reshape(-1), torch.empty(2 * t.numel(), device=dev, dtype=torch.float16),
             torch.full((2,), -1.0, device=dev)) for _, t in srcs]
    batch = ops.SplitBatch(jobs)
    print("  %d jobs, %d elements, %d blocks" % (len(jobs), sum(j[0].numel() for j in jobs), batch.total_blocks))
    ops.split16_batch(batch)
    torch.cuda.synchronize()
    for (name, _), (src, dst, sc) in zip(srcs, jobs):
        n = src.numel()
        cs = src.cpu()
        ch = torch.empty(2 * n, dtype=torch.float16)
        csc = torch.empty(2)
        emul_ops.split16_batch(emul_ops.SplitBatch([(cs, ch, csc)]))
        assert torch.equal(dst.cpu().view(torch.int16), ch.view(torch.int16)), name
        assert torch.equal(sc.cpu(), csc), (name, sc, csc)
        amax = float(cs.abs().max())
        s = float(sc[0])
        assert s == _grad_rule(amax) and float(sc[1]) == 1 / s, (name, s, amax)
        hi = dst[:n].float().abs()
        assert float(hi.max()) <= 2.0 ** 14 and not bool((hi >= HALF_MAX).any()), name
        if amax > 0:
            assert 2.0 ** 13 <= amax * s < 2.0 ** 14, name
        else:
            assert s == 1.0


@gpu
def test_pack_weight_batch_bit_exact_on_model_jobs(dev):
    """pack_weight_batch on the engine's model-scale jobs (R50/J16/D64): the fprop / dgrad operand
    pack of every layer and the per-stage unpack of the weight gradients, bit-exact with the CPU
    emulation (a permutation: no arithmetic)."""
    _check_pack_weight_batch(dev, _r50(dev)[0])


def _check_pack_weight_batch(dev, m):
    from epipolarpose_b200 import ops
    from tests import emul_ops
    eng = m._engine()
    eng.dev = dev
    params = dict(m.named_parameters())
    with torch.no_grad():
        eng._pack_weights(params)
    grads = {k: torch.empty_like(v) for k, v in params.items()}
    gs = eng._grad_state(grads)
    batches = [("pack", eng._wstate["batch"])] + [("unpack stage %d" % i, b) for i, b in enumerate(gs["batches"])
                                                  if b is not None]
    gs["flat"].copy_(torch.randn(gs["flat"].numel(), device=dev))
    njobs = 0
    for what, b in batches:
        # the same jobs into fresh NaN-filled destinations (the engine's buffers stay untouched)
        jobs = [(j[0], torch.full_like(j[1], float("nan"))) + tuple(j[2:]) for j in b.jobs]
        ops.pack_weight_batch(ops.PackBatch(jobs))
        torch.cuda.synchronize()
        for j in jobs:
            src, dst = j[0], j[1]
            cdst = torch.full(dst.shape, float("nan"))
            emul_ops.pack_weight_batch(emul_ops.PackBatch([(src.detach().cpu(), cdst) + tuple(j[2:])]))
            got = dst.detach().cpu()
            # every element the emulation writes (operand, zero padding) bit for bit
            w_ = ~torch.isnan(cdst)
            assert bool(w_.any()) and not bool(torch.isnan(got[w_]).any()), what
            assert torch.equal(got[w_].view(torch.int32), cdst[w_].view(torch.int32)), what
            njobs += 1
    print("  pack / unpack: %d jobs bit-exact" % njobs)


# ------------------------------------------------------------------ 4. stem at the bench size
@gpu
def test_im2col_split_bit_exact_at_stem_bench_size(dev):
    """im2col_split over all 128 images of 256 x 256 (7 x 7 / 2, pad 3): bit-exact with the CPU
    emulation on the first, last and three middle images."""
    _check_im2col_split(dev, _r50(dev)[0]._engine().stem_kpad, 128, 256)


def _check_im2col_split(dev, kpad, N, H):
    """im2col_split of N images of H x H (7 x 7 / 2, pad 3), bit-exact on five images"""
    from epipolarpose_b200 import ops, net16
    from tests import emul_ops
    W = H
    Ho = Wo = H // 2
    g = torch.Generator(device=dev).manual_seed(51)
    img = torch.randn(N, 3, H, W, device=dev, generator=g)
    img[5, :, 0, :] = 4094.0 / net16.IMG_SCALE              # the static scale's largest magnitude
    col = torch.empty(2, N, Ho, Wo, kpad, device=dev, dtype=torch.float16)
    sc = torch.tensor([net16.IMG_SCALE, 1.0 / net16.IMG_SCALE, 65504.0 / net16.IMG_SCALE, 0.0], device=dev)
    ops.im2col_split(img, col, sc, N, 3, H, W, 7, 7, 2, 3, Ho, Wo, kpad)
    torch.cuda.synchronize()
    pick = [0, 5, N // 2 - 1, N // 2, N - 1]
    cimg = img[pick].cpu()
    ccol = torch.empty(2, len(pick), Ho, Wo, kpad, dtype=torch.float16)
    emul_ops.im2col_split(cimg, ccol, sc.cpu(), len(pick), 3, H, W, 7, 7, 2, 3, Ho, Wo, kpad)
    got = col[:, pick].cpu()
    assert torch.equal(got.view(torch.int16), ccol.view(torch.int16))
    print("  im2col_split: images %s bit-exact (K pad %d)" % (pick, kpad))


@gpu
def test_maxpool_bwd_vs_float64_at_stem_bench_size(dev):
    """The stem's pool at the bench size (N = 128, 128 x 128 x 64): argidx from
    bn_relu_maxpool_split on dyadic inputs (exact fma, many ties), fp32 dy.  maxpool_bwd against a
    float64 scatter within 3u sum|g|, bit-equal with an fp32 restatement adding in (kh, kw)
    order; where argidx differs from torch.max_pool2d's index the window holds a tie."""
    _check_maxpool_bwd(dev, 128, 128)


def _check_maxpool_bwd(dev, N, H):
    """maxpool_bwd of the stem's pool over N images of H x H x 64"""
    from epipolarpose_b200 import ops
    W, C = H, 64
    Ho = Wo = H // 2
    g = torch.Generator(device=dev).manual_seed(61)
    z = torch.round(torch.randn(N, H, W, C, device=dev, generator=g) * 64) / 64
    scale = torch.round((torch.rand(C, device=dev, generator=g) + 0.5) * 256) / 256
    shift = torch.round(torch.randn(C, device=dev, generator=g) * 0.2 * 256) / 256
    a = (z.double() * scale.double() + shift.double()).clamp_min(0)     # exact: few-bit dyadics
    s = math.ldexp(1.0, 15 - math.frexp(float(a.max()))[1])
    y = torch.empty(2, N, Ho, Wo, C, device=dev, dtype=torch.float16)
    arg = torch.empty(N, Ho, Wo, C, device=dev, dtype=torch.uint8)
    ops.bn_relu_maxpool_split(z, scale, shift, y, torch.tensor([s, 1 / s, 0.0, 0.0], device=dev), arg, N, H, W, C)
    dy = torch.randn(N, Ho, Wo, C, device=dev, generator=g)
    dx = torch.empty(N, H, W, C, device=dev)
    ops.maxpool_bwd(dy, arg, dx, N, H, W, C)
    torch.cuda.synchronize()
    del y
    pad64 = torch.zeros(N, H + 2, W + 2, C, device=dev, dtype=torch.float64)
    pad32 = torch.zeros(N, H + 2, W + 2, C, device=dev)
    abs64 = torch.zeros(N, H + 2, W + 2, C, device=dev, dtype=torch.float64)
    for kh in range(3):
        for kw in range(3):
            sel = arg == kh * 3 + kw
            d = torch.where(sel, dy, torch.zeros_like(dy))
            pad32[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] += d
            pad64[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] += d.double()
            abs64[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] += d.double().abs()
    ref64, ref32, sab = pad64[:, 1:-1, 1:-1], pad32[:, 1:-1, 1:-1], abs64[:, 1:-1, 1:-1]
    err = (dx.double() - ref64).abs()
    bar = 3 * U * sab
    ratio = float((err / (bar + 1e-300)).max()) if bool((err > 0).any()) else 0.0
    print("  maxpool_bwd: max err %.3e, worst err / bar %.3f, fp32 restatement equal %s"
          % (float(err.max()), ratio, bool(torch.equal(dx, ref32))))
    assert bool((err <= bar).all())
    assert torch.equal(dx, ref32)
    del pad64, pad32, abs64, ref64, ref32, sab, err, bar, dx
    # the picks against torch's first-maximum indices on the same activation
    an = a.permute(0, 3, 1, 2).contiguous()
    del a
    mv, idx = torch.nn.functional.max_pool2d(an, 3, 2, 1, return_indices=True)
    arg_n = arg.permute(0, 3, 1, 2).long()
    oh = torch.arange(Ho, device=dev).view(1, 1, Ho, 1)
    ow = torch.arange(Wo, device=dev).view(1, 1, 1, Wo)
    kidx = (2 * oh - 1 + arg_n // 3) * W + (2 * ow - 1 + arg_n % 3)
    flat = an.view(N, C, H * W)
    picked = flat.gather(2, kidx.clamp(0, H * W - 1).view(N, C, -1)).view_as(mv)
    assert bool((kidx >= 0).all()), "argidx points into the padding"
    assert torch.equal(picked, mv), "argidx picks an entry below the window maximum"
    differ = kidx != idx
    ties = int(differ.sum())
    print("  maxpool argidx: %d picks differ from torch's index, all at ties" % ties)


# ------------------------------------------------------------------ 5. soft-argmax forward and joint loss
def _nhwc_geometry(N, J, D, H, W):
    """epb_softargmax_fwd (NHWC): split count S, pixels per trip ppi, depth d of a term"""
    C4 = J * D // 4
    ppi = max(512 // C4, 1)
    S = 1
    while N * S < 8 * NUM_SMS and (H * W) // (S * 2) >= 16 * ppi:
        S *= 2
    L = -(-(-(-(H * W) // S)) // ppi)
    return S, ppi, L + 2 + (D // 4) * ppi + S


@gpu
@pytest.mark.parametrize("kind", ["randn3", "peaks60", "constant"])
def test_softargmax_fwd_vs_float64_at_bench_shape(dev, kind):
    """N = 128, J = 16, D = 64, 64 x 64, NHWC (2.1 GB of logits): coords against float64 within
    the merge-depth bar, lse[0] the exact maximum, lse[1] * sum exp(v - m) - 1 within its bar.
    randn3: logits x 3 as in the backward test; peaks60: one logit of 60 per (image, joint);
    constant: every logit 0.7 (the uniform distribution)."""
    _check_softargmax_fwd(dev, kind, 128, 16, 64, 64, 64)


def _check_softargmax_fwd(dev, kind, N, J, D, H, W):
    """epb_softargmax_fwd (NHWC) at one shape against float64 within the merge-depth bar"""
    from epipolarpose_b200 import ops
    C = J * D
    g = torch.Generator(device=dev).manual_seed(71)
    if kind == "constant":
        logits = torch.full((N, H, W, C), 0.7, device=dev)
    else:
        logits = torch.randn(N, H, W, C, device=dev, generator=g) * 3
        if kind == "peaks60":
            pix = torch.randint(0, H * W, (N, J), device=dev, generator=g)
            dd = torch.randint(0, D, (N, J), device=dev, generator=g)
            nn_ = torch.arange(N, device=dev).view(N, 1).expand(N, J)
            jj = torch.arange(J, device=dev).view(1, J).expand(N, J)
            logits.view(N, H * W, J, D)[nn_, pix, jj, dd] = 60.0
    coords, lse = torch.empty(N, J * 3, device=dev), torch.empty(N * J * 2, device=dev)
    ops.softargmax_fwd(logits, 1, N, J, D, H, W, coords, lse)
    torch.cuda.synchronize()
    S, ppi, d = _nhwc_geometry(N, J, D, H, W)
    xs = torch.arange(W, device=dev, dtype=torch.float64).view(1, 1, W, 1, 1) / W
    ys = torch.arange(H, device=dev, dtype=torch.float64).view(1, H, 1, 1, 1) / H
    zs = torch.arange(D, device=dev, dtype=torch.float64).view(1, 1, 1, 1, D) / D
    lk = lse.view(N, J, 2)
    worst_c, worst_l, maxerr = 0.0, 0.0, 0.0
    B = 8
    for n0 in range(0, N, B):
        v = logits[n0:n0 + B].double().view(B, H, W, J, D)
        m = v.amax((1, 2, 4), keepdim=True)
        assert torch.equal(lk[n0:n0 + B, :, 0].double(), m.view(B, J)), "lse[0] is not the maximum"
        ex = torch.exp(v - m)
        tot = ex.sum((1, 2, 4), keepdim=True)
        p = ex / tot
        eps_i = (6 + 7 * (v - m).abs() + 6 * d) * U
        del v, ex
        pe = p * eps_i
        del eps_i
        ck = coords[n0:n0 + B].double().view(B, J, 3)
        for ax, pos in enumerate((xs, ys, zs)):
            c64 = (p * pos).sum((1, 2, 4))                          # c' = c + 1/2
            bar = (pe * (pos - c64.view(B, 1, 1, J, 1)).abs()).sum((1, 2, 4)) + 4 * d * U * c64 + 4 * U
            err = (ck[..., ax] + 0.5 - c64).abs()
            maxerr = max(maxerr, float(err.max()))
            worst_c = max(worst_c, float((err / bar).max()))
        lbar = pe.sum((1, 2, 4)) + (2 * d + 2) * U
        el = (lk[n0:n0 + B, :, 1].double() * tot.view(B, J) - 1).abs()
        worst_l = max(worst_l, float((el / lbar.view(B, J)).max()))
        del p, pe
    print("  softargmax fwd %-8s S %d ppi %d depth %d: coords max err %.3e worst err / bar %.3f, "
          "lse[1] worst err / bar %.3f" % (kind, S, ppi, d, maxerr, worst_c, worst_l))
    assert worst_c <= 1.0 and worst_l <= 1.0


def _jointloss64(x, t, w, kind, norm, div):
    xv = x.double().clone().requires_grad_(True)
    a, b = xv, t.double()
    if norm:
        a, b = xv / xv.abs().sum(), b / b.abs().sum()
    d = a - b
    l = d * d if kind == 0 else (d.abs() if kind == 1 else torch.where(d.abs() < 1, 0.5 * d * d, d.abs() - 0.5))
    tot = (l * w.double()).sum() / div
    tot.backward()
    return tot.item(), xv.grad, d.detach(), (l * w.double()).abs().sum().item() / abs(div)


@gpu
@pytest.mark.parametrize("kind,norm", [(2, 0), (1, 0), (1, 1), (2, 1)], ids=["smoothl1", "l1", "l1_norm", "smoothl1_norm"])
def test_jointloss_vs_float64_at_bench_shape(dev, kind, norm):
    """epb_jointloss_fwd_bwd at N = 128, J = 16 (6144 elements), weights with zeros, |d| on both
    sides of 1 and exactly 1 (dyadic x, t: d exact without norm): loss and dx against float64."""
    _check_jointloss(dev, kind, norm, 128, 16)


def _check_jointloss(dev, kind, norm, N, J):
    """epb_jointloss_fwd_bwd over n = N J 3 elements against float64 within the module's bar"""
    from epipolarpose_b200 import ops
    n = N * J * 3
    g = torch.Generator(device=dev).manual_seed(81 + kind + 2 * norm)
    t = torch.round((torch.rand(n, device=dev, generator=g) - 0.5) * 1024) / 1024
    d = torch.round(torch.randn(n, device=dev, generator=g) * 1.2 * 1024) / 1024
    d[:64] = 1.0
    d[64:128] = -1.0
    d[128:192] = 1.0 - 2.0 ** -10
    d[192:256] = 1.0 + 2.0 ** -10
    x = t + d
    w = (torch.rand(n, device=dev, generator=g) > 0.25).float() * torch.round(torch.rand(n, device=dev, generator=g) * 8) / 4
    loss, dx = torch.empty(1, device=dev), torch.empty(n, device=dev)
    div = float(N)
    ops.jointloss(x, t, w, n, kind, norm, div, loss, dx)
    torch.cuda.synchronize()
    l64, dx64, d64, sabs = _jointloss64(x, t, w, kind, norm, div)
    dl = -(-n // LOSS_THREADS) + 12
    if not norm:
        lbar = dl * U * sabs + U * abs(l64)
        gbar = 2 * U * dx64.abs()
    else:
        xa = x.double().abs()
        xn, tn = x.double() / xa.sum(), t.double() / t.double().abs().sum()
        ed = (dl + 3) * U * (xn.abs() + tn.abs())
        wd_ = w.double() / div
        assert float(d64.abs().max()) < 1                       # SmoothL1 stays on its quadratic side
        lbar = float((wd_ * ed * (1.0 if kind == 1 else d64.abs())).sum()) + dl * U * sabs + U * abs(l64)
        isx = 1 / xa.sum()
        gmag = wd_ * (1.0 if kind == 1 else d64.abs())
        dg = (0.0 if kind == 1 else wd_ * ed) + U * gmag
        gbar = (dl + 4) * U * gmag * isx + dg * isx + \
            ((3 * dl + 6) * U * (gmag * xa).sum() + (dg * xa).sum()) * isx * isx + U * dx64.abs()
        # L1: a sign of d within ed of zero could resolve either way; the data has none
        assert not bool(((d64.abs() <= ed) & (w != 0) & (ed > 0)).any())
    le = abs(float(loss) - l64)
    ge = (dx.double() - dx64).abs()
    print("  jointloss kind %d norm %d: loss err %.3e (bar %.3e), dx worst err / bar %.3f"
          % (kind, norm, le, lbar, float((ge / (gbar + 1e-300)).max()) if bool((ge > 0).any()) else 0.0))
    assert le <= lbar
    assert bool((ge <= gbar).all())


# ------------------------------------------------------------------ 1. coverage gate, GPU half
@gpu
def test_coverage_gate_bench_step(dev):
    """One bench-composition step at a reduced size (R18, J = 16, D = 64, 2 tuples x 4 views of
    256 x 256): GraphedTrainStep(online=True, method="iterative").eager_step, SmoothL1, FusedAdam.
    Every C-ABI entry it calls has a row in COVERAGE naming existing tests."""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    import lib.utils.utils as U
    J, D, HW, tuples = 16, 64, 256, 2
    B = 4 * tuples
    torch.manual_seed(0)
    m = models.pose3d_resnet.get_pose_net(_cfg(18, J, D, HW), False, precision="f16x3").to(dev).train()
    opt = U.FusedAdam(list(m.parameters()), lr=1e-3)
    step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J).to(dev), opt, online=True, method="iterative")
    meta = {k: v.to(dev) for k, v in _bench_meta(tuples).items()}
    x = torch.randn(B, 3, HW, HW, device=dev)
    with _record_calls() as names:
        loss = step.eager_step(x, None, None, iu.pack_meta(meta, B, dev))
        torch.cuda.synchronize()
    assert math.isfinite(float(loss))
    print("  bench step calls %d entries:" % len(names))
    for e in sorted(names):
        print("    %-28s -> %s" % (e, ", ".join(COVERAGE.get(e, ["(none)"]))))
    assert "epb_adam_step_dev" in names and "epb_triangulate" in names
    missing, dangling = _missing_coverage(names)
    assert not missing, "entries without a float64 test at bench size: %s" % missing
    assert not dangling, dangling
