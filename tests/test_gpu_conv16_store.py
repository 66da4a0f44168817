"""GPU (-m gpu): the output footprint of conv16_kernel (epb_conv16_fprop), whose epilogue writes
the output through TMA stores (TMA reduce-adds with `accumulate`) bounded by the extents of the
output view.

- Every call writes exactly the elements of its output view -- the phase (ph, pw) positions of
  a transposed conv or a stride-2 data gradient, the whole tensor otherwise -- and leaves the
  rest of the tensor and a guard band past its end untouched: the call runs into two buffers
  pre-filled with different NaN sentinels, and the view must come out identical in both while
  everything else keeps its sentinel.  The written values are checked against the CPU
  emulation (tests/emul_ops.py) on the same split operands.
- With `accumulate` the result is the fp32 sum of the prior contents and the non-accumulating
  result, bit for bit.
- Output and BatchNorm statistics are bit-identical across two runs at multi-tile shapes."""
import numpy as np
import pytest
import torch

from tests import emul_ops as em
from tests.conftest import relerr
from tests.step_cases import _rand_split, _weights_split

pytestmark = pytest.mark.gpu

GUARD = 4096                                   # floats past the end of the output
SENTINELS = (0x7FC0DEAD, 0x7FC0BEEF)           # quiet NaNs with distinct payloads


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _cases():
    """(name, Conv ctor args, N, H, W, which) -- which: f(prop) / d(grad)."""
    from epipolarpose_b200.net import Conv
    return [
        ("dense_1x1_M588", Conv("a", "conv", 64, 256, 1, 1, 0), 3, 14, 14, "f"),
        ("3x3_8x8", Conv("b", "conv", 256, 256, 3, 1, 1), 4, 8, 8, "f"),
        ("3x3_s2", Conv("c", "conv", 128, 128, 3, 2, 1), 3, 13, 13, "f"),
        ("deconv4_phases", Conv("d", "deconv", 256, 256, 4, 2, 1), 2, 8, 8, "f"),
        ("deconv3_ragged_phases", Conv("e", "deconv", 128, 192, 3, 2, 1), 2, 6, 6, "f"),
        ("dgrad_3x3_s2_phases", Conv("f", "conv", 128, 128, 3, 2, 1), 2, 13, 13, "d"),
        ("dgrad_1x1_s2_phases", Conv("g", "conv", 256, 512, 1, 2, 0), 2, 15, 15, "d"),
        ("cout_1088", Conv("h", "conv", 256, 1088, 1, 1, 0), 1, 16, 16, "f"),
        ("cout_192", Conv("i", "conv", 64, 192, 1, 1, 0), 3, 10, 10, "f"),
    ]


CASES = _cases()


def _operands(conv, N, H, W, which):
    """geoms, split input, split weights, output shape (N, Ho, Wo, C) of one call site."""
    T = conv.k * conv.k
    Ho, Wo = conv.out_hw(H, W)
    if which == "f":
        geoms = conv.fprop_geoms(em, N, H, W, 3)
        x, x_sc = _rand_split((N, H, W, conv.cin_p), 1)
        w, w_sc = _weights_split(conv.cout_p, T * conv.cin_p, 2)
        return geoms, x, x_sc, w, w_sc, (N, Ho, Wo, conv.cout_p)
    geoms = conv.dgrad_geoms(em, N, H, W, 3)
    x, x_sc = _rand_split((N, Ho, Wo, conv.cout_p), 7, scale=None, relu=False, mag=3e-5)
    w, w_sc = _weights_split(conv.cin_p, T * conv.cout_p, 8)
    return geoms, x, x_sc, w, w_sc, (N, H, W, conv.cin_p)


def _view_mask(g, shape):
    m = torch.zeros(shape, dtype=torch.bool)
    m[:, g.ph::g.os, g.pw::g.os] = True
    return m


def _filled(shape, bits, dev):
    n = int(np.prod(shape))
    return torch.full((n + GUARD,), bits, dtype=torch.int32, device=dev).view(torch.float32)


def _call(g, ops_args, buf, shape, acc):
    from epipolarpose_b200 import ops
    x, x_sc, w, w_sc = ops_args
    g.in_relu, g.accumulate = 0, int(acc)
    ops.conv16_fprop(g, x, x_sc, w, w_sc, buf[:int(np.prod(shape))].view(shape), None, None)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv16_writes_exactly_its_view(dev, case):
    name, conv, N, H, W, which = case
    geoms, x, x_sc, w, w_sc, shape = _operands(conv, N, H, W, which)
    args = (x.to(dev), x_sc.to(dev), w.to(dev), w_sc.to(dev))
    n = int(np.prod(shape))
    ran = 0
    for g in geoms:
        if g is None:
            continue
        ran += 1
        bufs = [_filled(shape, s, dev) for s in SENTINELS]
        for b in bufs:
            _call(g, args, b, shape, 0)
        torch.cuda.synchronize()
        a, b = (t.view(torch.int32).cpu() for t in bufs)
        inside = torch.zeros(n + GUARD, dtype=torch.bool)
        inside[:n] = _view_mask(g, shape).view(-1)
        assert torch.equal(a[inside], b[inside]), "view elements depend on the prior contents"
        assert bool((a[~inside] == SENTINELS[0]).all()) and bool((b[~inside] == SENTINELS[1]).all()), \
            "%d elements outside the view were written" % int((a[~inside] != SENTINELS[0]).sum())
        ref = torch.zeros(shape)
        em.conv16_fprop(g, x, x_sc, w, w_sc, ref, None, None)
        got = bufs[0][:n].cpu().view(shape)[:, g.ph::g.os, g.pw::g.os]
        e = relerr(got.numpy(), ref[:, g.ph::g.os, g.pw::g.os].numpy())
        assert e <= 5e-5, "output relerr %.3e" % e
    assert ran


ACC = [c for c in CASES if c[0] in ("dense_1x1_M588", "deconv3_ragged_phases", "dgrad_3x3_s2_phases",
                                     "dgrad_1x1_s2_phases", "cout_192")]


@pytest.mark.parametrize("case", ACC, ids=[c[0] for c in ACC])
def test_conv16_accumulate_is_one_fp32_add(dev, case):
    name, conv, N, H, W, which = case
    geoms, x, x_sc, w, w_sc, shape = _operands(conv, N, H, W, which)
    args = (x.to(dev), x_sc.to(dev), w.to(dev), w_sc.to(dev))
    n = int(np.prod(shape))
    gen = torch.Generator().manual_seed(17)
    prior = torch.cat([torch.randn(n, generator=gen), torch.full((GUARD,), 3.0)]).to(dev)
    for g in geoms:
        if g is None:
            continue
        fresh = _filled(shape, SENTINELS[0], dev)
        _call(g, args, fresh, shape, 0)
        summed = prior.clone()
        _call(g, args, summed, shape, 1)
        torch.cuda.synchronize()
        inside = torch.zeros(n + GUARD, dtype=torch.bool, device=dev)
        inside[:n] = _view_mask(g, shape).view(-1).to(dev)
        want = torch.where(inside, prior + fresh, prior)
        assert torch.equal(summed.view(torch.int32), want.view(torch.int32)), \
            "%d elements differ from prior + result" % int((summed != want).sum())


DET = [("3x3_64_stats", "conv", 64, 64, 3, 1, 1, 8, 64, 64),
       ("1x1_64_256_stats", "conv", 64, 256, 1, 1, 0, 16, 32, 32),
       ("deconv4_256_stats", "deconv", 256, 256, 4, 2, 1, 64, 16, 16)]


@pytest.mark.parametrize("case", DET, ids=[c[0] for c in DET])
def test_conv16_output_and_stats_are_run_to_run_identical(dev, case):
    from epipolarpose_b200 import ops
    from epipolarpose_b200.net import Conv
    name, kind, cin, cout, k, s, p, N, H, W = case
    conv = Conv("x", kind, cin, cout, k, s, p)
    geoms, x, x_sc, w, w_sc, shape = _operands(conv, N, H, W, "f")
    xg, xs, wg, ws = x.to(dev), x_sc.to(dev), w.to(dev), w_sc.to(dev)
    runs = []
    for _ in range(2):
        out = torch.zeros(shape, device=dev)
        stats = torch.zeros(2 * shape[-1], dtype=torch.float64, device=dev)
        for g in geoms:
            if g is not None:
                g.in_relu, g.accumulate = 0, 0
                ops.conv16_fprop(g, xg, xs, wg, ws, out, None, stats)
        runs.append((out, stats))
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0].view(torch.int32), runs[1][0].view(torch.int32))
    assert torch.equal(runs[0][1].view(torch.int64), runs[1][1].view(torch.int64))


def test_conv16_accumulate_keeps_subnormals(dev):
    """accumulate=1 with a zero product: the new value is the bias, so normal and subnormal old
    and new values, and sums that round into the subnormal range, all meet in the L2 add; the
    result must be numpy's fp32 sum, bit for bit."""
    from epipolarpose_b200 import ops
    from epipolarpose_b200.net import Conv
    conv = Conv("s", "conv", 64, 64, 1, 1, 0)
    N, H, W = 2, 8, 16
    g = conv.fprop_geoms(em, N, H, W, 3)[0]
    x, x_sc = _rand_split((N, H, W, 64), 1, mag=0.0)
    w, w_sc = _weights_split(64, 64, 2)
    vals = np.array([1e-40, -1e-40, 1e-39, -1.4e-38, 1.5e-38, 3.0, 0.0], np.float32)
    rng = np.random.default_rng(5)
    bias = vals[rng.integers(0, len(vals), 64)]
    prior = np.append(vals, np.float32(-0.0))[rng.integers(0, len(vals) + 1, (N, H, W, 64))]
    want = prior + bias
    out = torch.from_numpy(prior.copy()).to(dev)
    g.in_relu, g.accumulate = 0, 1
    ops.conv16_fprop(g, x.to(dev), x_sc.to(dev), w.to(dev), w_sc.to(dev), out,
                     torch.from_numpy(bias).to(dev), None)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), \
        "%d sums differ" % int((got.view(np.uint32) != want.view(np.uint32)).sum())
