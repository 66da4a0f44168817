"""GPU (-m gpu): the split-fp16 ("f16x3") kernel family through the C ABI against the CPU
emulation of the same contracts (tests/emul_ops.py: exact fp16 planes, three-term products
accumulated in float64) on IDENTICAL split operands, so the bar is the fp32 accumulation
noise of the tensor pipe (<= 5e-5 of the tensor's max), not a precision trade-off.
Geometries: every conv kind of the network (reference lib/models/pose3d_resnet.py:12-15,
55-60,99,116-122,171-178) incl. strided / transposed / phase-decomposed forms, ragged
sizes, N tails, accumulate / bias / statistics epilogues."""
import numpy as np
import pytest
import torch

from tests import emul_ops as em
from tests.conftest import relerr
from tests.step_cases import C4_LAYERS_SPLIT16, H16, _check_conv16_layer, _rand_split, _weights_split

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _conv_cases():
    """(name, Conv ctor args, N, H, W, which) -- which in f(prop) / d(grad)."""
    from epipolarpose_b200.net import Conv
    C = []
    C.append(("1x1_64_256", Conv("a", "conv", 64, 256, 1, 1, 0), 2, 16, 16))
    C.append(("1x1_256_64", Conv("b", "conv", 256, 64, 1, 1, 0), 2, 16, 16))
    C.append(("1x1_ragged_M", Conv("c", "conv", 128, 128, 1, 1, 0), 3, 14, 14))
    C.append(("3x3_64_64", Conv("d", "conv", 64, 64, 3, 1, 1), 2, 16, 16))
    C.append(("3x3_128_ragged", Conv("e", "conv", 128, 128, 3, 1, 1), 3, 14, 14))
    C.append(("3x3_s2", Conv("f", "conv", 128, 128, 3, 2, 1), 2, 16, 16))
    C.append(("3x3_s2_ragged", Conv("g", "conv", 64, 128, 3, 2, 1), 3, 12, 12))
    C.append(("1x1_s2", Conv("h", "conv", 256, 512, 1, 2, 0), 2, 16, 16))
    C.append(("3x3_512_8x8", Conv("i", "conv", 512, 512, 3, 1, 1), 4, 8, 8))
    C.append(("3x3_256_4x4", Conv("j", "conv", 256, 256, 3, 1, 1), 5, 4, 4))
    C.append(("deconv4", Conv("k", "deconv", 256, 256, 4, 2, 1), 2, 8, 8))
    C.append(("deconv4_ragged", Conv("l", "deconv", 128, 64, 4, 2, 1), 3, 6, 6))
    C.append(("deconv3", Conv("m", "deconv", 128, 128, 3, 2, 1, 1), 2, 8, 8))
    C.append(("deconv2", Conv("n", "deconv", 64, 128, 2, 2, 0), 2, 8, 8))
    C.append(("1x1_N_tail_320", Conv("o", "conv", 64, 320, 1, 1, 0), 2, 16, 16))
    C.append(("final_1088", Conv("p", "conv", 256, 1088, 1, 1, 0), 1, 16, 16))
    C.append(("final_24", Conv("q", "conv", 64, 24, 1, 1, 0), 2, 16, 16))
    C.append(("3x3_final", Conv("r", "conv", 64, 24, 3, 1, 1), 2, 16, 16))
    C.append(("big_M_pairs", Conv("s", "conv", 64, 64, 3, 1, 1), 8, 64, 64))
    return C


CASES = _conv_cases()


def _run_fprop(dev, conv, N, H, W, geoms, x, x_sc, w, w_sc, Hin, Win, cin, Hout, Wout, cout, bias, stats, acc):
    from epipolarpose_b200 import ops
    out_ref = torch.zeros((N, Hout, Wout, cout))
    if acc:
        out_ref = torch.randn((N, Hout, Wout, cout), generator=torch.Generator().manual_seed(3))
    out_gpu = out_ref.clone().to(dev)
    st_ref = torch.zeros(2 * cout, dtype=torch.float64) if stats else None
    st_gpu = torch.zeros(2 * cout, dtype=torch.float64, device=dev) if stats else None
    xg, xs, wg, ws = x.to(dev), x_sc.to(dev), w.to(dev), w_sc.to(dev)
    bg = bias.to(dev) if bias is not None else None
    for g in geoms:
        if g is None:
            continue
        g.in_relu, g.accumulate = 0, int(acc)
        em.conv16_fprop(g, x, x_sc, w, w_sc, out_ref, bias, st_ref)
        ops.conv16_fprop(g, xg, xs, wg, ws, out_gpu, bg, st_gpu)
    torch.cuda.synchronize()
    e = relerr(out_gpu.cpu().numpy(), out_ref.numpy())
    assert e <= 5e-5, "output relerr %.3e" % e      # fp32 accumulation over K up to 4608
    if stats:
        e = relerr(st_gpu.cpu().numpy(), st_ref.numpy())
        assert e <= 1e-4, "stats relerr %.3e" % e


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_conv16_fprop_vs_emulation(dev, case):
    name, conv, N, H, W = case
    geoms = conv.fprop_geoms(em, N, H, W, 3)
    Ho, Wo = conv.out_hw(H, W)
    T = conv.k * conv.k
    x, x_sc = _rand_split((N, H, W, conv.cin_p), 1)
    w, w_sc = _weights_split(conv.cout_p, T * conv.cin_p, 2)
    bias = torch.randn(conv.cout_p, generator=torch.Generator().manual_seed(5)) if "final" in name else None
    stats = bias is None
    _run_fprop(dev, conv, N, H, W, geoms, x, x_sc, w, w_sc, H, W, conv.cin_p, Ho, Wo, conv.cout_p,
               bias, stats, False)


DGRAD = [c for c in CASES if c[1].cout % 64 == 0]


@pytest.mark.parametrize("case", DGRAD, ids=[c[0] for c in DGRAD])
@pytest.mark.parametrize("acc", [0, 1])
def test_conv16_dgrad_vs_emulation(dev, case, acc):
    name, conv, N, H, W = case
    geoms = conv.dgrad_geoms(em, N, H, W, 3)
    Ho, Wo = conv.out_hw(H, W)
    T = conv.k * conv.k
    dz, dz_sc = _rand_split((N, Ho, Wo, conv.cout_p), 7, scale=None, relu=False, mag=3e-5)
    w, w_sc = _weights_split(conv.cin_p, T * conv.cout_p, 8)
    _run_fprop(dev, conv, N, H, W, geoms, dz, dz_sc, w, w_sc, Ho, Wo, conv.cout_p, H, W, conv.cin_p,
               None, False, bool(acc))


WGRAD = [c for c in CASES if c[1].cout % 64 == 0]


@pytest.mark.parametrize("case", WGRAD, ids=[c[0] for c in WGRAD])
def test_conv16_wgrad_vs_emulation(dev, case):
    from epipolarpose_b200 import ops
    name, conv, N, H, W = case
    geoms = conv.fprop_geoms(em, N, H, W, 3)
    Ho, Wo = conv.out_hw(H, W)
    T = conv.k * conv.k
    x, x_sc = _rand_split((N, H, W, conv.cin_p), 11)
    dz, dz_sc = _rand_split((N, Ho, Wo, conv.cout_p), 12, scale=None, relu=False, mag=3e-5)
    n = conv.cout_p * T * conv.cin_p
    dw_ref = torch.zeros(n)
    dw_gpu = torch.zeros(n, device=dev)
    ws = torch.empty(8 << 20, device=dev)
    xg, xs, dg, ds = x.to(dev), x_sc.to(dev), dz.to(dev), dz_sc.to(dev)
    for rep in range(2):                      # second pass checks the += contract
        for g in geoms:
            if g is None:
                continue
            g.in_relu, g.accumulate = 0, 0
            em.conv16_wgrad(g, x, x_sc, dz, dz_sc, dw_ref, None)
            ops.conv16_wgrad(g, xg, xs, dg, ds, dw_gpu, ws)
    torch.cuda.synchronize()
    e = relerr(dw_gpu.cpu().numpy(), dw_ref.numpy())
    assert e <= 5e-5, "dw relerr %.3e" % e
    # deterministic: a second run from zero gives the same bits
    a = torch.zeros(n, device=dev)
    b = torch.zeros(n, device=dev)
    for buf in (a, b):
        for g in geoms:
            if g is not None:
                ops.conv16_wgrad(g, xg, xs, dg, ds, buf, ws)
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_split_elementwise_vs_emulation(dev):
    from epipolarpose_b200 import ops
    gen = torch.Generator().manual_seed(21)
    M, C = 1500, 192
    x = torch.randn(M, C, generator=gen) * 3
    sc, sh = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen)
    r = torch.randn(M, C, generator=gen)
    rsc, rsh = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen)
    rs, rs_sc = _rand_split((M, C), 22)
    asc = torch.tensor([16.0, 1 / 16.0])
    for kind in ("plain", "res", "res_affine", "res_split", "noaffine"):
        args = dict(plain=(sc, sh, None, None, None, None, None),
                    res=(sc, sh, r, None, None, None, None),
                    res_affine=(sc, sh, r, rsc, rsh, None, None),
                    res_split=(sc, sh, None, None, None, rs, rs_sc),
                    noaffine=(None, None, None, None, None, None, None))[kind]
        y_ref = torch.empty(2, M, C, dtype=H16)
        bits_ref = torch.empty(M * C // 8, dtype=torch.uint8)
        em.bn_act_split(x, *args, 1, M, C, y_ref, asc, bits_ref)
        y = torch.empty(2, M, C, dtype=H16, device=dev)
        bits = torch.empty(M * C // 8, dtype=torch.uint8, device=dev)
        ops.bn_act_split(x.to(dev), *[a.to(dev) if a is not None else None for a in args], 1, M, C,
                         y, asc.to(dev), bits)
        # the ReLU bit mask: identical except where the pre-activation is within rounding of zero
        diff = np.unpackbits((bits.cpu() ^ bits_ref).numpy(), bitorder="little").astype(bool)
        pre = em._join(y_ref, asc).reshape(-1).numpy()
        assert diff.sum() <= 2 and (diff.sum() == 0 or float(np.abs(pre[diff[:pre.size]]).max()) <= 1e-5)
        a = em._join(y.cpu(), asc).numpy()
        b = em._join(y_ref, asc).numpy()
        assert np.max(np.abs(a - b)) <= 2e-6 * max(1.0, np.max(np.abs(b))), kind
    # stem pool
    N, H, W, Cc = 2, 14, 18, 64
    z = torch.randn(N, H, W, Cc, generator=gen)
    s2, h2 = torch.rand(Cc, generator=gen) + 0.5, torch.randn(Cc, generator=gen) * 0.1
    Ho, Wo = (H + 2 - 3) // 2 + 1, (W + 2 - 3) // 2 + 1
    y_ref, a_ref = torch.empty(2, N, Ho, Wo, Cc, dtype=H16), torch.empty(N, Ho, Wo, Cc, dtype=torch.uint8)
    em.bn_relu_maxpool_split(z, s2, h2, y_ref, asc, a_ref, N, H, W, Cc)
    y, a = torch.empty_like(y_ref, device=dev), torch.empty_like(a_ref, device=dev)
    ops.bn_relu_maxpool_split(z.to(dev), s2.to(dev), h2.to(dev), y, asc.to(dev), a, N, H, W, Cc)
    assert np.max(np.abs(em._join(y.cpu(), asc).numpy() - em._join(y_ref, asc).numpy())) <= 1e-6
    # argmax slots may differ only where two window entries tie (post-ReLU zeros)
    diff = (a.cpu() != a_ref)
    assert float(em._join(y_ref, asc)[diff].abs().max() if diff.any() else 0.0) == 0.0
    # im2col
    img = torch.randn(2, 3, 20, 24, generator=gen)
    Ho, Wo = 10, 12
    c_ref = torch.empty(2, 2, Ho, Wo, 192, dtype=H16)
    em.im2col_split(img, c_ref, asc, 2, 3, 20, 24, 7, 7, 2, 3, Ho, Wo, 192)
    c = torch.empty_like(c_ref, device=dev)
    ops.im2col_split(img.to(dev), c, asc.to(dev), 2, 3, 20, 24, 7, 7, 2, 3, Ho, Wo, 192)
    assert torch.equal(c.cpu().view(torch.int16), c_ref.view(torch.int16))
    # several 64-pixel segments per output row, ragged last one (the staged kernel's window logic)
    img = torch.randn(1, 3, 11, 300, generator=gen)
    Ho, Wo = 6, 150
    c_ref = torch.empty(2, 1, Ho, Wo, 192, dtype=H16)
    em.im2col_split(img, c_ref, asc, 1, 3, 11, 300, 7, 7, 2, 3, Ho, Wo, 192)
    c = torch.empty_like(c_ref, device=dev)
    ops.im2col_split(img.to(dev), c, asc.to(dev), 1, 3, 11, 300, 7, 7, 2, 3, Ho, Wo, 192)
    assert torch.equal(c.cpu().view(torch.int16), c_ref.view(torch.int16))
    # batched fp32 -> split with amax scale
    srcs = [torch.randn(n, generator=gen) * s for n, s in ((5000, 1e-3), (777, 40.0), (4096, 1.0))]
    jobs_ref = [(s, torch.empty(2 * s.numel(), dtype=H16), torch.ones(2)) for s in srcs]
    em.split16_batch(em.SplitBatch(jobs_ref))
    jobs = [(s.to(dev), torch.empty(2 * s.numel(), dtype=H16, device=dev), torch.ones(2, device=dev)) for s in srcs]
    ops.split16_batch(ops.SplitBatch(jobs))
    for (s, h, c2), (_, hr, cr) in zip(jobs, jobs_ref):
        assert torch.equal(c2.cpu(), cr)
        assert torch.equal(h.cpu().view(torch.int16), hr.view(torch.int16))
    # avgpool
    t, tsc = _rand_split((3, 16, 2048), 31)
    yr = torch.empty(3, 2048)
    em.avgpool_split(t, tsc, yr, 3, 16, 2048)
    yg = torch.empty(3, 2048, device=dev)
    ops.avgpool_split(t.to(dev), tsc.to(dev), yg, 3, 16, 2048)
    assert relerr(yg.cpu().numpy(), yr.numpy()) <= 1e-6


@pytest.mark.parametrize("mode", ["relu", "mask", "mask_inplace", "plain"])
def test_bn_bwd_split_vs_emulation(dev, mode):
    from epipolarpose_b200 import ops
    gen = torch.Generator().manual_seed(41)
    M, C = 3000, 256
    x = torch.randn(M, C, generator=gen) * 2 + 0.3
    dy = torch.randn(M, C, generator=gen) * 1e-4
    gamma, beta = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen) * 0.1
    mean = x.mean(0)
    invstd = 1.0 / torch.sqrt(x.var(0, unbiased=False) + 1e-5)
    scale, shift = gamma * invstd, beta - mean * gamma * invstd
    out, _ = _rand_split((M, C), 42)
    mask = out[0].contiguous() if mode.startswith("mask") else None
    relu = 1 if mode == "relu" else 0
    sums_r, mx_r = torch.zeros(2 * C, dtype=torch.float64), torch.zeros(2 * C)
    em.bn_bwd_reduce_mx(dy, x, mask, scale, shift, mean, invstd, relu, M, C, sums_r, mx_r)
    D = lambda t: t.to(dev) if t is not None else None
    sums, mx = torch.zeros(2 * C, dtype=torch.float64, device=dev), torch.zeros(2 * C, device=dev)
    dyg = dy.to(dev)
    ops.bn_bwd_reduce_mx(dyg, D(x), D(mask), D(scale), D(shift), D(mean), D(invstd), relu, M, C, sums, mx)
    assert relerr(sums.cpu().numpy(), sums_r.numpy()) <= 1e-5
    assert np.max(np.abs(mx.cpu().numpy() - mx_r.numpy())) <= 1e-6 * float(mx_r.max())
    dz_r, sc_r = torch.empty(2, M, C, dtype=H16), torch.empty(2)
    dm_r = dy.clone() if mode == "mask_inplace" else None
    dg_r, db_r = torch.empty(C), torch.empty(C)
    em.bn_bwd_apply_split(dy, x, mask, scale, shift, mean, invstd, gamma, relu, sums_r, mx_r, M, C,
                          dz_r, sc_r, dm_r, dg_r, db_r)
    dz, sc = torch.empty(2, M, C, dtype=H16, device=dev), torch.empty(2, device=dev)
    dg, db = torch.empty(C, device=dev), torch.empty(C, device=dev)
    ops.bn_bwd_apply_split(dyg, D(x), D(mask), D(scale), D(shift), D(mean), D(invstd), D(gamma), relu,
                           sums, mx, M, C, dz, sc, dyg if mode == "mask_inplace" else None, dg, db)
    torch.cuda.synchronize()
    s_g, s_r = float(sc.cpu()[0]), float(sc_r[0])
    assert s_g in (s_r, 2 * s_r, s_r / 2)      # the bound is summed in a different order
    a = em._join(dz.cpu(), sc.cpu()).numpy()
    b = em._join(dz_r, sc_r).numpy()
    assert relerr(a, b) <= 1e-5
    assert float(np.max(np.abs(b))) * s_r < 32768
    assert relerr(dg.cpu().numpy(), dg_r.numpy()) <= 1e-5 and relerr(db.cpu().numpy(), db_r.numpy()) <= 1e-5
    if mode == "mask_inplace":
        assert torch.equal(dyg.cpu(), dm_r)


@pytest.mark.parametrize("N,J,D,H,W", [(2, 4, 16, 8, 8), (3, 16, 64, 16, 16), (1, 17, 12, 5, 7), (5, 1, 4, 3, 9)])
def test_softargmax_bwd_split_vs_emulation(dev, N, J, D, H, W):
    """epb_softargmax_bwd_split: planes == split of the fp32 gradient (same scale, values <= 2e-6 of the
    maximum apart: __expf), bias column sums, scale from the hard bound."""
    from epipolarpose_b200 import ops
    gen = torch.Generator().manual_seed(N * 100 + J)
    C = J * D
    logits = (torch.randn(N, H, W, C, generator=gen) * 3).contiguous()
    dco = torch.randn(N, J * 3, generator=gen)
    coords_r, lse_r = torch.empty(N, J * 3), torch.empty(N * J * 2)
    em.softargmax_fwd(logits, 1, N, J, D, H, W, coords_r, lse_r)
    pl_r, sc_r, db_r = torch.empty(2, N, H, W, C, dtype=H16), torch.empty(2), torch.empty(C)
    em.softargmax_bwd_split(logits, N, J, D, H, W, coords_r, lse_r, dco, pl_r, sc_r, db_r)
    lg = logits.to(dev)
    coords, lse = torch.empty(N, J * 3, device=dev), torch.empty(N * J * 2, device=dev)
    ops.softargmax_fwd(lg, 1, N, J, D, H, W, coords, lse)
    pl, sc, db = torch.empty(2, N, H, W, C, dtype=H16, device=dev), torch.empty(2, device=dev), torch.empty(C, device=dev)
    ops.softargmax_bwd_split(lg, N, J, D, H, W, coords, lse, dco.to(dev), pl, sc, db)
    ref32 = torch.empty(N, H, W, C, device=dev)
    ops.softargmax_bwd(lg, 1, N, J, D, H, W, coords, lse, dco.to(dev), ref32)
    torch.cuda.synchronize()
    assert float(sc.cpu()[0]) in (float(sc_r[0]), 2 * float(sc_r[0]), float(sc_r[0]) / 2)
    got = em._join(pl.cpu(), sc.cpu()).numpy()
    assert relerr(got, em._join(pl_r, sc_r).numpy()) <= 5e-6
    assert relerr(got, ref32.cpu().numpy()) <= 2e-6                    # == the fp32 kernel's gradient
    assert float(np.abs(got).max()) * float(sc.cpu()[0]) <= 32768
    assert relerr(db.cpu().numpy(), db_r.numpy()) <= 1e-5


@pytest.mark.parametrize("C,second,res", [(64, False, False), (256, True, False), (2048, False, True)])
def test_bn_finalize_scale_vs_two_calls(dev, C, second, res):
    """epb_bn_finalize_scale == epb_bn_finalize followed by epb_act_scale (same device kernels' arithmetic):
    scale / shift / mean / invstd / running statistics bit-identical, published scale identical."""
    from epipolarpose_b200 import ops
    gen = torch.Generator().manual_seed(7 + C)
    M = 5000

    def stats():
        x = torch.randn(M, C, generator=gen, dtype=torch.float64) * 3 + 0.7
        return torch.cat([x.sum(0), (x * x).sum(0)]).to(dev)

    st1, st2 = stats(), (stats() if second else None)
    gamma, beta = (torch.rand(C, generator=gen) + 0.5).to(dev), (torch.randn(C, generator=gen) * 0.1).to(dev)
    s2 = (torch.rand(C, generator=gen) + 0.5).to(dev) if second else None
    h2 = (torch.randn(C, generator=gen) * 0.1).to(dev) if second else None
    res_sc = torch.tensor([4.0, 0.25, 37.5, 0.0], device=dev) if res else None
    outs = []
    for fused in (False, True):
        rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
        sc_, sh_, mu, iv = (torch.empty(C, device=dev) for _ in range(4))
        sc = torch.empty(4, device=dev)
        if fused:
            ops.bn_finalize_scale(st1, M, C, gamma, beta, 1e-5, 0.1, rm, rv, sc_, sh_, mu, iv, st2, s2, h2, res_sc, sc)
        else:
            ops.bn_finalize(st1, M, C, gamma, beta, 1e-5, 0.1, rm, rv, sc_, sh_, mu, iv)
            ops.act_scale(st1, sc_, sh_, M, C, st2, s2, h2, res_sc, sc)
        outs.append([t.cpu() for t in (sc_, sh_, mu, iv, rm, rv, sc)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("M,C,mode", [(3000, 256, "mask_inplace"), (70001, 64, "relu"), (517, 2048, "mask"),
                                       (9, 64, "plain"), (40000, 1024, "relu"), (2, 512, "mask"),
                                       (3001, 256, "bits_inplace"), (517, 2048, "bits"), (70001, 64, "bits"),
                                       (5, 8, "bits_inplace")])
def test_bn_bwd_fused_entry_vs_emulation_and_deterministic(dev, M, C, mode):
    """epb_bn_bwd_split (partials -> fixed-order combine -> apply, what the engine calls) against the
    emulation of the two-call form; two runs are bit-identical (no atomics in the reduction)."""
    from epipolarpose_b200 import ops
    gen = torch.Generator().manual_seed(43 + C)
    x = torch.randn(M, C, generator=gen) * 2 + 0.3
    dy = torch.randn(M, C, generator=gen) * 1e-4
    gamma, beta = torch.rand(C, generator=gen) + 0.5, torch.randn(C, generator=gen) * 0.1
    mean = x.mean(0)
    invstd = 1.0 / torch.sqrt(x.var(0, unbiased=False) + 1e-5)
    scale, shift = gamma * invstd, beta - mean * gamma * invstd
    out, _ = _rand_split((M, C), 44)
    mask = out[0].contiguous() if mode.startswith("mask") else None
    bits = None
    if mode.startswith("bits"):
        bits = torch.from_numpy(np.packbits((torch.rand(M * C, generator=gen) > 0.4).numpy(), bitorder="little"))
    relu = 1 if mode == "relu" else 0
    inplace = mode.endswith("_inplace")
    dz_r, sc_r = torch.empty(2, M, C, dtype=H16), torch.empty(2)
    dm_r = dy.clone() if inplace else None
    dg_r, db_r = torch.empty(C), torch.empty(C)
    em.bn_bwd_split(dy, x, mask, scale, shift, mean, invstd, gamma, relu, M, C, dz_r, sc_r, dm_r, dg_r, db_r,
                    mask_bits=bits)
    D = lambda t: t.to(dev) if t is not None else None
    runs = []
    for _ in range(2):
        dyg = dy.to(dev)
        dz, sc = torch.empty(2, M, C, dtype=H16, device=dev), torch.empty(2, device=dev)
        dg, db = torch.empty(C, device=dev), torch.empty(C, device=dev)
        ops.bn_bwd_split(dyg, D(x), D(mask), D(scale), D(shift), D(mean), D(invstd), D(gamma), relu, M, C,
                         dz, sc, dyg if inplace else None, dg, db, mask_bits=D(bits))
        torch.cuda.synchronize()
        runs.append((dz.cpu(), sc.cpu(), dg.cpu(), db.cpu(), dyg.cpu()))
    dz, sc, dg, db, dyg = runs[0]
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.int16) if a.dtype == H16 else a, b.view(torch.int16) if b.dtype == H16 else b)
    s_g, s_r = float(sc[0]), float(sc_r[0])
    assert s_g in (s_r, 2 * s_r, s_r / 2) and float(sc[1]) == 1.0 / s_g
    b = em._join(dz_r, sc_r).numpy()
    assert relerr(em._join(dz, sc).numpy(), b) <= 1e-5
    assert float(np.max(np.abs(b))) * s_g <= 65504
    assert relerr(dg.numpy(), dg_r.numpy()) <= 2e-5 and relerr(db.numpy(), db_r.numpy()) <= 2e-5
    if inplace:
        assert torch.equal(dyg, dm_r)


# ------------------------------------------------------------------ the bench's own layer shapes
# step_cases.C4_LAYERS_SPLIT16; reference: torch float64 convolutions (cuDNN / cuBLAS fp64 on the
# same device -- none of this repo's code) of the EXACT values the fp16 planes hold.
@pytest.mark.parametrize("layer", C4_LAYERS_SPLIT16, ids=[c[0] for c in C4_LAYERS_SPLIT16])
def test_conv16_bench_layer_shapes_vs_torch_float64(dev, layer):
    _check_conv16_layer(dev, layer, 128, 2e-4)
