"""GPU (-m gpu): the inference forward (Engine16.forward(..., prepared=...): PosePredictor,
MultiViewPredictor, RefinedPosePredictor, save_triangulations) against float64 kernel by kernel at
the predictors' own sizes, on three models: C1 (R50, J16, D64, 256^2), the H36M model (R50, J17,
D64, 256^2) and C5 (R101, J17, D96, 384^2).  The models load init_state weights with calibrated
running statistics (step_cases.calibrated_state), so that eval BatchNorm sees a trained-like regime
instead of running_mean 0 / running_var 1.

- epb_conv16_fprop_splitk with statistics at the planner's split count, at every distinct layer the
  forward runs (step_cases.infer_layers) for N = 1, 2 (flip of 1), 3 (ragged M tiles), 8 (one
  4-view tuple with flip) and 24 (a ragged 3-tuple batch with flip) on R50 with both finals, and N
  = 1, 2, 8 on C5.  Bar 5e-5 of the largest |output| and of the largest column sum, the fp32
  accumulation noise of test_gpu_split16 (the reference reads the joined planes), as
  test_gpu_predictor.  The bias is in the reference once, the statistics count the valid rows
  only; each S > 1 conv case shows that the reference without one split's partial misses the bar,
  and each batch with padded rows that statistics over them do.  The finals have K = 256, four
  k-blocks, which the planner never splits; their ragged column tiles (1088 = 8.5 x 128, 1632 =
  12.75 x 128) run at forced S = 2 and 4 against float64, inside a NaN guard band, and with a
  workspace of exactly ws_floats and one 1M floats larger (bit-identical results, the tail
  untouched).  Which split regimes the cases reach is checked on the CPU
  (test_splitk_host.test_inference_cases_reach_every_split_regime).
- N = 256, save_triangulations' batch: the planner gives S = 1 for every call and the split entry
  is bit-identical to epb_conv16_fprop, which test_gpu_split16.test_conv16_bench_layer_shapes_vs_
  torch_float64 and test_gpu_bn_chain.test_conv16_stats_vs_float64 hold to float64 at N = 128.
- epb_bn_eval_affine at every CNN BatchNorm width, running_var from 1e-6 to 1e3, gamma of both
  signs: within 1 fp32 ulp of float64 on the same fp32 inputs.  fp32 arithmetic misses that bar
  (shift = beta - mean * scale cancels), which the kernel had until it computed in double.
- The eval BatchNorm chain inside the prepared forward of the calibrated C1 model at N = 1 and 8:
  every epb_act_scale / epb_bn_act_split / epb_bn_relu_maxpool_split call (plain, identity
  residual, downsample) against float64 on the exact values it read, with the scale contract of
  step_cases._contract_act and every element within the bound.
- epb_im2col_split bit-exact with the emulation at N = 1 and 2, 256^2 and 384^2.
- The decode heads on the predictor's channels-last logits: epb_softargmax_fwd through
  step_cases._check_softargmax_fwd, and epb_softargmax_flip_fwd / epb_softargmax_flip_lse_fwd
  (coordinates within 1e-5 of the float64 merge as test_gpu_flip, lse within the bars of
  _check_softargmax_fwd over the merged fp32 volume, which the merge without / with the shift
  misses; the two entries' coordinates bit-identical), N = 1, 4, 128.
- End to end on the calibrated models: PosePredictor (C1, N = 1) and MultiViewPredictor (H36M,
  one 4-view tuple, flip test) against oracle.restate_net in float64 on the same state dict:
  logits within 1e-3 of the largest |logit| (BASELINE's north star), every joint within
  step_cases._coord_bound of the measured logit change from the float64 decode of the float64
  logits."""
import math

import numpy as np
import pytest
import torch

from tests import emul_splitk as es
from tests import step_cases as sc

pytestmark = pytest.mark.gpu

SPLITK_BAR = 5e-5
FLIP_BAR = 1e-5
LOGIT_BAR = 1e-3
FINALS = {"c1": 1024, "h36m": 1088, "c5": 1632}


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    sc.release("infer_")


def _layers(model):
    """the distinct layers of the model's inference forward; R50 with both finals"""
    return sc.infer_layers(["c1", "h36m"] if model == "r50" else ["c5"])


# ------------------------------------------------------------------ 1. split-K conv16
SPLITK = [("r50", N) for N in (1, 2, 3, 8, 24)] + [("c5", N) for N in (1, 2, 8)]


def _ratios(out, stats, ref, cout):
    """(output, S1, S2) error / bar of one run"""
    r = ref.reshape(-1, cout)
    e = float((out.double() - ref).abs().max() / ref.abs().max())
    e1 = float((stats[:cout] - r.sum(0)).abs().max() / r.abs().sum(0).max())
    e2 = float((stats[cout:] - (r * r).sum(0)).abs().max() / (r * r).sum(0).max())
    return e / SPLITK_BAR, e1 / SPLITK_BAR, e2 / SPLITK_BAR


@pytest.mark.parametrize("model,N", SPLITK, ids=["%s-N%d" % c for c in SPLITK])
def test_infer_splitk_vs_float64(dev, model, N):
    from epipolarpose_b200 import ops
    worst, pad_fault, padded, splits = 0.0, 0.0, False, set()
    for conv, hw in _layers(model):
        geoms, opnds, bias, ref, xw = sc._splitk_layer(dev, conv, hw, N)
        cout = conv.cout
        S = [ops.conv16_splits(gm)[0] for gm in geoms]
        splits.update(S)
        out = torch.zeros(ref.shape, device=dev)
        stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
        sc._splitk_run(geoms, opnds, bias, out, stats, None)
        torch.cuda.synchronize()
        rs = _ratios(out, stats, ref, cout)
        print("  %-22s %-6s hw %3d cout %4d S %-12s output %.3f S1 %.3f S2 %.3f of the bar"
              % (conv.name, conv.kind, hw, cout, S, *rs))
        assert max(rs) <= 1.0, (conv.name, rs)
        worst = max(worst, *rs)
        # teeth: the bias twice, one split's partial dropped; and over the layers, statistics over
        # the padded rows (they hold the bias alone)
        assert float(bias.abs().max() / ref.abs().max()) > SPLITK_BAR
        r = ref.reshape(-1, cout)
        pad = sum(es.phase_tiles(gm) * 128 - gm.N * gm.Hp * gm.Wp for gm in geoms)
        padded = padded or pad > 0
        pad_fault = max(pad_fault, float(pad * bias.abs().max() / r.abs().sum(0).max()) / SPLITK_BAR)
        if conv.kind == "conv" and S[0] > 1:
            lo, hi = es.split_ranges(es.kblocks(geoms[0]), S[0])[0]
            part = sc._split_partial64(conv, geoms[0], xw, lo, hi)
            assert float(part.abs().max() / ref.abs().max()) > SPLITK_BAR, conv.name
        del geoms, opnds, ref, xw, out
    print("  %s N %d: split counts %s, worst err / bar %.3f; statistics over the padded rows %.3g of the bar"
          % (model, N, sorted(splits), worst, pad_fault))
    assert pad_fault > 1.0 or not padded


FINAL_CASES = [(m, N, S) for m in ("h36m", "c5") for N in (1, 3) for S in (2, 4)]


@pytest.mark.parametrize("model,N,S", FINAL_CASES, ids=["%s-N%d-S%d" % c for c in FINAL_CASES])
def test_infer_splitk_ragged_final_writes_exactly_its_view(dev, model, N, S):
    """The final 1x1 layer (K = 256: four k-blocks) at forced S > 1: against float64, nothing
    written past the output (NaN-sentinel guard band), and the same output bits whether the
    workspace holds exactly the planner's ws_floats at S or 1M floats more, whose tail stays
    untouched."""
    from epipolarpose_b200 import ops
    conv = sc.infer_plan(model).final
    assert conv.cout == FINALS[model] and conv.cout % 128
    hw = sc.INFER_MODELS[model][3] // 4
    geoms, opnds, bias, ref, _ = sc._splitk_layer(dev, conv, hw, N)
    (gm,) = geoms
    assert ops.conv16_splits(gm)[0] == 1
    sentinel, guard, extra = 0x7FC0DEAD, 4096, 1 << 20
    n = ref.numel()
    need = S * es.phase_tiles(gm) * 128 * gm.Cout
    outs, tails = [], []
    for more in (0, extra):
        buf = torch.full((n + guard,), sentinel, dtype=torch.int32, device=dev).view(torch.float32)
        ws = torch.full((need + more,), sentinel, dtype=torch.int32, device=dev).view(torch.float32)
        stats = torch.zeros(2 * conv.cout, device=dev, dtype=torch.float64)
        ops.conv16_fprop_splitk(gm, opnds[0], opnds[1], opnds[2], opnds[3], buf[:n].view(ref.shape), bias,
                                stats, S, ws)
        torch.cuda.synchronize()
        outs.append((buf, stats))
        tails.append(ws[need:].view(torch.int32))
    (a, sa), (b, sb) = outs
    assert bool((a.view(torch.int32)[n:] == sentinel).all()), "written past the output"
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert bool((tails[1] == sentinel).all()), "workspace written past ws_floats"
    # the statistics of S > 1 are summed in a run-dependent order: each run within the bar
    rs = max(_ratios(a[:n].view(ref.shape), st, ref, conv.cout) for st in (sa, sb))
    print("  final %d N %d S %d: output %.3f S1 %.3f S2 %.3f of the bar" % (conv.cout, N, S, *rs))
    assert max(rs) <= 1.0


def test_infer_splitk_n256_is_the_fused_kernel(dev):
    """save_triangulations' batch of 256 on the H36M model: S = 1 at every call, and the split
    entry's output and statistics are epb_conv16_fprop's bits."""
    from epipolarpose_b200 import ops
    for conv, hw in sc.infer_layers(["h36m"]):
        geoms, opnds, bias, _, _ = sc._splitk_layer(dev, conv, hw, 256, ref=False)
        Ho, Wo = conv.out_hw(hw, hw)
        assert all(ops.conv16_splits(gm) == (1, 0) for gm in geoms), conv.name
        runs = []
        for split in (False, True):
            out = torch.zeros(256, Ho, Wo, conv.cout, device=dev)
            stats = torch.zeros(2 * conv.cout, device=dev, dtype=torch.float64)
            if split:
                sc._splitk_run(geoms, opnds, bias, out, stats, None)
            else:
                for gm in geoms:
                    ops.conv16_fprop(gm, *opnds, out, bias, stats)
            runs.append((out, stats))
        torch.cuda.synchronize()
        (fo, fs), (so, ss) = runs
        assert torch.equal(fo.view(torch.int32), so.view(torch.int32)), conv.name
        assert torch.equal(fs.view(torch.int64), ss.view(torch.int64)), conv.name
        del runs, fo, so, opnds


# ------------------------------------------------------------------ 2. eval BatchNorm affine
@pytest.mark.parametrize("C", [64, 128, 256, 512, 1024, 2048])
def test_infer_bn_eval_affine_within_one_ulp(dev, C):
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(C)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    gamma[1::2] *= -1
    beta = torch.randn(C, device=dev, generator=g) * 0.3
    rv = torch.exp(torch.empty(C, device=dev).uniform_(math.log(1e-6), math.log(1e3), generator=g))
    rm = torch.randn(C, device=dev, generator=g) * rv.sqrt() * 2
    rv[:2], rv[-1] = 1e-6, 1e3
    scale, shift = torch.empty(C, device=dev), torch.empty(C, device=dev)
    ops.bn_eval_affine(C, gamma, beta, rm, rv, sc.EPS, scale, shift)
    torch.cuda.synchronize()
    eps = float(np.float32(sc.EPS))
    s64 = gamma.double() / torch.sqrt(rv.double() + eps)
    h64 = beta.double() - rm.double() * s64
    us = sc._ulps(scale.cpu().numpy(), s64.cpu().numpy()).max()
    uh = sc._ulps(shift.cpu().numpy(), h64.cpu().numpy()).max()
    # teeth: the same formulas in fp32 arithmetic
    inv32 = 1 / torch.sqrt(rv + eps)
    uh32 = sc._ulps((beta - rm * gamma * inv32).cpu().numpy(), h64.cpu().numpy()).max()
    print("  bn_eval_affine C %d: scale %.2f ulp, shift %.2f ulp (fp32 arithmetic: %.1f ulp)" % (C, us, uh, uh32))
    assert us <= 1 and uh <= 1
    assert uh32 > 1


# ------------------------------------------------------------------ 3./4. eval BatchNorm chain of the prepared forward
class _Intercept:
    """Wraps the ops module's act_scale / bn_act_split / bn_relu_maxpool_split and checks every call
    against float64 on the values it read, right after it ran."""

    def __init__(self, ops):
        self.ops, self.saved, self.worst, self.calls, self.pending = ops, {}, 0.0, 0, {}

    def __enter__(self):
        for k in ("act_scale", "bn_act_split", "bn_relu_maxpool_split"):
            self.saved[k] = getattr(self.ops, k)
            setattr(self.ops, k, getattr(self, k))
        return self

    def __exit__(self, *a):
        for k, f in self.saved.items():
            setattr(self.ops, k, f)

    def act_scale(self, stats, scale, shift, M, C, stats2, scale2, shift2, res_sc, sc_):
        self.saved["act_scale"](stats, scale, shift, M, C, stats2, scale2, shift2, res_sc, sc_)
        self.pending[sc_.data_ptr()] = (stats2 is not None, res_sc is not None)

    def _contract(self, what, z, scale, shift, M, C, y, y_sc, ymax, extra=0.0, group2=None):
        zs = sc._stats64(z.reshape(M, C))
        bound = float(sc._bound_def(zs[:C], zs[C:], scale.double(), shift.double(), M).max())
        if group2 is not None:
            r, rscale, rshift = group2
            rs = sc._stats64(r.reshape(M, C))
            bound += float(sc._bound_def(rs[:C], rs[C:], rscale.double(), rshift.double(), M).max())
        bound = bound * 1.001 + extra
        assert ymax <= bound, "%s: max|y| %.4e over the bound %.4e" % (what, ymax, bound)
        sc._contract_act(what, y, y_sc, bound, ymax)

    def bn_act_split(self, x, scale, shift, r, rscale, rshift, r_split, r_sc, relu, M, C, y, y_sc, mask_bits=None):
        self.saved["bn_act_split"](x, scale, shift, r, rscale, rshift, r_split, r_sc, relu, M, C, y, y_sc, mask_bits)
        torch.cuda.synchronize()
        grp2, res = self.pending.pop(y_sc.data_ptr())
        zd = x.reshape(M, C).double()
        res64, res_terms, extra, what = 0.0, 0.0, 0.0, "plain"
        if r is not None:
            assert grp2
            rd = r.reshape(M, C).double()
            res64 = rd * rscale.double() + rshift.double()
            res_terms = (rd * rscale.double()).abs() + rshift.double().abs() + res64.abs()
            what = "downsample"
            del rd
        elif r_split is not None:
            assert res
            res64 = sc._join(r_split, r_sc).reshape(M, C)
            res_terms, extra, what = res64.abs(), float(r_sc[2]), "identity"
        pre = zd * scale.double() + shift.double() + res64
        y64 = pre.clamp_min(0) if relu else pre
        ymax = float(y64.abs().max())
        bar = sc._apply_bar(zd, scale.double(), shift.double(), res_terms, ymax)
        err = (sc._join(y, y_sc).reshape(M, C) - y64).abs()
        ratio = float((err / bar).max())
        self.worst, self.calls = max(self.worst, ratio), self.calls + 1
        assert ratio <= 1.0, "%s M %d C %d: err / bar %.3f" % (what, M, C, ratio)
        self._contract("%s M %d C %d" % (what, M, C), x, scale, shift, M, C, y, y_sc, ymax, extra,
                       (r, rscale, rshift) if r is not None else None)

    def bn_relu_maxpool_split(self, x, scale, shift, y, y_sc, argidx, N, H, W, C):
        self.saved["bn_relu_maxpool_split"](x, scale, shift, y, y_sc, argidx, N, H, W, C)
        torch.cuda.synchronize()
        self.pending.pop(y_sc.data_ptr())
        Ho, Wo = (H + 1) // 2, (W + 1) // 2
        zd = x.reshape(N, H, W, C).double()
        a64 = (zd * scale.double() + shift.double()).clamp_min(0)
        e = 4 * sc.U * ((zd * scale.double()).abs() + shift.double().abs())
        pa = torch.full((N, H + 2, W + 2, C), float("-inf"), device=x.device, dtype=torch.float64)
        pe = torch.zeros((N, H + 2, W + 2, C), device=x.device, dtype=torch.float64)
        pa[:, 1:-1, 1:-1], pe[:, 1:-1, 1:-1] = a64, e
        del a64, e
        ref = torch.stack([pa[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)]).max(0).values
        ce = torch.stack([pe[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)]).max(0).values
        ymax = float(ref.max())
        err = (sc._join(y, y_sc) - ref).abs()
        ratio = float((err / (ce + 2.0 ** -22 * ymax)).max())
        self.worst, self.calls = max(self.worst, ratio), self.calls + 1
        assert ratio <= 1.0, "stem max-pool err / bar %.3f" % ratio
        self._contract("stem maxpool N %d" % N, x, scale, shift, N * H * W, C, y, y_sc, ymax)


@pytest.mark.parametrize("N", [1, 8])
def test_infer_eval_chain_vs_float64(dev, N):
    """The prepared forward of the calibrated C1 model, eagerly: every act_scale + bn_act_split /
    bn_relu_maxpool_split pair on its eval affine (M = 64 rows at l4 for N = 1)."""
    from epipolarpose_b200 import net16
    model = sc.calibrated_model(dev, "c1")
    eng = net16.Engine16(model._plan, ops=model._ops)
    with torch.no_grad():
        params = {k: v.detach() for k, v in model.named_parameters()}
        params.update(dict(model.named_buffers()))
        state = eng.prepare_inference(params, dev)
        x = torch.from_numpy(np.random.default_rng(N).standard_normal((N, 3, 256, 256)).astype(np.float32)).to(dev)
        with _Intercept(eng.ops) as ic:
            eng.forward(x, None, training=False, save=False, prepared=state)
        torch.cuda.synchronize()
    n_bn = len(model._plan.all_bns())
    n_down = sum(1 for b in model._plan.blocks if b["down"])
    print("  eval chain N %d: %d calls, worst apply err / bar %.3f" % (N, ic.calls, ic.worst))
    assert ic.calls == n_bn - n_down and not ic.pending


# ------------------------------------------------------------------ 5. stem patch matrix
@pytest.mark.parametrize("H", [256, 384])
@pytest.mark.parametrize("N", [1, 2])
def test_infer_im2col_split_bit_exact(dev, N, H):
    from epipolarpose_b200.net16 import STEM_KPAD16
    sc._check_im2col_split(dev, STEM_KPAD16, N, H)


# ------------------------------------------------------------------ 6. decode heads
HEADS = [(N, J, D) for N in (1, 4, 128) for J, D in ((16, 64), (17, 64), (17, 96))]


@pytest.mark.parametrize("kind", ["random", "peaks60"])
@pytest.mark.parametrize("N,J,D", HEADS, ids=["N%d-J%d-D%d" % c for c in HEADS])
def test_infer_softargmax_fwd_vs_float64(dev, N, J, D, kind):
    sc._check_softargmax_fwd(dev, kind, N, J, D, D, D)


def _flip_logits(dev, N, J, D, seed):
    """[2N, H, W, J*D] logits of scale 3 with one peak of +14 per (image, joint) on every third image"""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = 3.0 * torch.randn((2 * N, D, D, J * D), device=dev, generator=g)
    rng = np.random.default_rng(seed)
    for n in range(0, 2 * N, 3):
        for j in range(J):
            h, w, d = rng.integers(0, D, 3)
            x[n, h, w, j * D + d] += 14.0
    return x


@pytest.mark.parametrize("shift", [False, True])
@pytest.mark.parametrize("N,J,D", HEADS, ids=["N%d-J%d-D%d" % c for c in HEADS])
def test_infer_softargmax_flip_vs_float64(dev, N, J, D, shift):
    from epipolarpose_b200 import ops
    import lib.core.integral_loss as il
    from tests import flip_cases as fc
    pairs = fc.MPII_PAIRS if J == 16 else fc.H36M_PAIRS
    perm = il.flip_permutation(pairs, J)
    L2 = _flip_logits(dev, N, J, D, 7 * N + J + D + int(shift))
    c1 = torch.empty(N, J * 3, device=dev)
    c2 = torch.empty(N, J * 3, device=dev)
    lse = torch.empty(N * J * 2, device=dev)
    ops.softargmax_flip_fwd(L2, N, J, D, D, D, perm, int(shift), c1)
    ops.softargmax_flip_lse_fwd(L2, N, J, D, D, D, perm, int(shift), c2, lse)
    torch.cuda.synchronize()
    assert torch.equal(c1, c2), "the two flip entries' coordinates differ"
    err = 0.0
    for n0 in range(0, N, 8):
        n1 = min(N, n0 + 8)
        pair = torch.cat([L2[n0:n1], L2[N + n0:N + n1]]).permute(0, 3, 1, 2).double()
        ref = sc._decode64(pair, J, D, pairs, shift).reshape(n1 - n0, J * 3)
        err = max(err, float((c1[n0:n1].double() - ref).abs().max()))
        del pair
    merged = sc._flip_merged32(L2, N, J, D, perm, shift)
    wc, wl, _, max_ok = sc._softargmax_ratios(merged, c2, lse, N, J, D, D, D)
    del merged
    other = sc._flip_merged32(L2, N, J, D, perm, not shift)
    tc, _, _, _ = sc._softargmax_ratios(other, c2, lse, N, J, D, D, D)
    print("  flip N %d J %d D %d shift %d: coords %.3e (bar %.0e), merged-volume coords %.3f lse[1] %.3f of "
          "the bar; the other shift's merge %.3g" % (N, J, D, shift, err, FLIP_BAR, wc, wl, tc))
    assert err <= FLIP_BAR
    assert max_ok, "lse[0] is not the merged volume's maximum"
    assert wc <= 1.0 and wl <= 1.0
    assert tc > 1.0


# ------------------------------------------------------------------ 7. end to end against float64
def _sd64(dev, key):
    return {k: v.to(dev, torch.float64) if v.is_floating_point() else v.to(dev)
            for k, v in sc.calibrated_state(dev, key).items()}


def _end_to_end(dev, key, logits, coords, x, pairs=None, shift=False):
    """logits [B, J*D, H/4, W/4] and normalised coordinates [N, J*3] of a predictor against the
    float64 forward and decode of the same images x [B, 3, H, W]"""
    from oracle import restate_net as rn
    import lib.core.integral_loss as il
    layers, J, D, HW, _ = sc.INFER_MODELS[key]
    with torch.no_grad():
        ref = rn.forward(_sd64(dev, key), x.to(dev, torch.float64), num_layers=layers,
                         image_size=(HW, HW), training=False)
    e = float((logits.double() - ref).abs().max() / ref.abs().max())
    B = ref.shape[0]
    dl = (logits.double() - ref).abs().reshape(B, J, -1).amax(-1).cpu().numpy()      # [B, J]
    if pairs is not None:
        N = B // 2
        dl = np.maximum(dl[:N], dl[N:][:, il.flip_permutation(pairs, J)])
    want = sc._decode64(ref, J, D, pairs, shift).cpu().numpy() * sc.PATCH
    got = coords.double().cpu().numpy().reshape(want.shape) * sc.PATCH
    d = np.abs(got - want).max(-1)
    bound = sc._coord_bound(dl)
    print("  %s: logits %.3e of the largest |logit| (bar %.0e); joints %.3e px, worst / bound %.3f"
          % (key, e, LOGIT_BAR, d.max(), (d / bound).max()))
    assert e <= LOGIT_BAR
    assert np.all(d <= bound), (d.max(), bound.min())


def test_infer_predictor_c1_vs_float64(dev):
    from lib.core.inference import PosePredictor
    model = sc.calibrated_model(dev, "c1")
    pred = PosePredictor(model, flip_test=False)
    x = np.random.default_rng(11).standard_normal((1, 3, 256, 256)).astype(np.float32)
    pred(x)
    ent = pred.graphs[(1, 256, 256)]
    _end_to_end(dev, "c1", pred.logits, ent["coords"], torch.from_numpy(x))


def test_infer_multiview_h36m_vs_float64(dev):
    from lib.core.inference import MultiViewPredictor
    from lib.dataset.synthetic import H36M_FLIP_PAIRS
    from tests import multiview_cases as mc
    model = sc.calibrated_model(dev, "h36m")
    mv = MultiViewPredictor(model, flip_test=True, shift_heatmap=True, flip_pairs=H36M_FLIP_PAIRS)
    x, boxes, P = mc.rig_inputs(1, 4, 12)
    mv(x, boxes, P)
    ent = mv.graphs[(1, 4, 256, 256)]
    xs = torch.from_numpy(x.reshape(4, 3, 256, 256))
    assert mv.logits.shape[0] == 8
    _end_to_end(dev, "h36m", mv.logits, ent["coords"], torch.cat([xs, torch.flip(xs, [3])]),
                H36M_FLIP_PAIRS, True)
