"""CPU emulation of the split-K conv16 entry (include/epb.h epb_conv16_fprop_splitk) and of the
host rules behind it: the phase-grid tiling of split16_common.cuh (epb_choose_tile) and the
split planner (epb_conv16_splits).  Same conventions as tests/emul_ops.py: torch CPU tensors,
exact fp16 planes, products in float64."""
import torch

from tests import emul_ops as em

BM = 128
NUM_SMS = 132
SPLIT_MIN_KB = 4
SPLIT_LONG_KB = 16


def choose_tile(N, Hp, Wp, rows=BM):
    """epb_choose_tile: the power-of-two box (tw, th, tn), tw*th*tn == rows, covering the fewest
    grid pixels (first found wins ties)."""
    best, out = None, (rows, 1, 1)
    a = rows
    while a >= 1:
        b = rows // a
        while b >= 1:
            c = rows // (a * b)
            cov = -(-Wp // a) * -(-Hp // b) * -(-N // c)
            if best is None or cov < best:
                best, out = cov, (a, b, c)
            b >>= 1
        a >>= 1
    return out


def phase_tiles(g):
    """Number of 128-row M tiles of the phase grid (a dense 1x1 layer is one row of M pixels)."""
    dense = (g.T == 1 and g.is_ == 1 and g.os == 1 and g.dh[0] == 0 and g.dw[0] == 0 and
             g.Hp == g.Hi and g.Wp == g.Wi and g.Hp == g.Ho and g.Wp == g.Wo)
    N, Hp, Wp = (1, 1, g.N * g.Hp * g.Wp) if dense else (g.N, g.Hp, g.Wp)
    tw, th, tn = choose_tile(N, Hp, Wp)
    return -(-Wp // tw) * -(-Hp // th) * -(-N // tn)


def n_tiles(g):
    bn = 64 if g.Cout <= 64 else 128
    return -(-g.Cout // bn)


def kblocks(g):
    return g.T * (g.Cin // 64)


def splits(g):
    """epb_conv16_splits: (splits, workspace floats)."""
    tiles = phase_tiles(g) * n_tiles(g)
    s = min(NUM_SMS // tiles, kblocks(g) // SPLIT_MIN_KB)
    if s < 4 and kblocks(g) < SPLIT_LONG_KB * s:
        s = 1
    s = max(1, s)
    return s, (s * phase_tiles(g) * BM * g.Cout if s > 1 else 0)


def split_ranges(KB, S):
    """k-block range [lo, hi) of each split: split s starts at s * KB / S (integer division)."""
    return [(s * KB // S, (s + 1) * KB // S) for s in range(S)]


def conv16_fprop_splitk(g, x, x_sc, w, w_sc, out, bias, stats, S):
    """The split entry: per split the three-term product over its k-blocks (k-block = 64 channels
    of one tap, taps outer), scaled and rounded to fp32 as the partial store does; the partials
    summed in fp32 in the order 0..S-1, then the bias; statistics ADDED from the fp32 result."""
    assert g.Cin % 64 == 0 and g.Cout % 4 == 0 and not g.accumulate
    CB = g.Cin // 64
    xh = x[0].reshape(g.N, g.Hi, g.Wi, g.Cin).double()
    xl = x[1].reshape(g.N, g.Hi, g.Wi, g.Cin).double()
    n = g.Cout * g.Tw * g.Cin
    wh = w.view(-1)[:n].view(g.Cout, g.Tw, g.Cin).double()
    wl = w.view(-1)[n:2 * n].view(g.Cout, g.Tw, g.Cin).double()
    alpha = float(x_sc[1]) * float(w_sc[1])
    total = None
    for lo, hi in split_ranges(kblocks(g), S):
        part = torch.zeros(g.N, g.Hp, g.Wp, g.Cout, dtype=torch.float64)
        for kb in range(lo, hi):
            t, c0 = kb // CB, (kb % CB) * 64
            ah = em._gather(g, xh, t, None, None)[..., c0:c0 + 64]
            al = em._gather(g, xl, t, None, None)[..., c0:c0 + 64]
            bh, bl = wh[:, g.wt[t], c0:c0 + 64].T, wl[:, g.wt[t], c0:c0 + 64].T
            part += al @ bh + ah @ bl + ah @ bh
        part = (part * alpha).float()
        total = part if total is None else total + part
    if bias is not None:
        total = total + bias
    o = out.view(g.N, g.Ho, g.Wo, g.Cout)
    o[:, g.ph::g.os, g.pw::g.os][:, :g.Hp, :g.Wp] = total
    if stats is not None:
        flat = total.reshape(-1, g.Cout).double()
        stats[:g.Cout] += flat.sum(0)
        stats[g.Cout:] += (flat * flat).sum(0)


def conv16_calls(plan, N, H=256, W=256, ops=em):
    """(layer name, geometry) of every conv16 fprop call of Engine16.forward at batch N, from the
    plan's shapes alone (stem patch matrix, blocks with their downsample, deconv phases, final)."""
    return [(conv.name, g) for conv, h, w in conv16_layers(plan, H, W)
            for g in conv.fprop_geoms(ops, N, h, w, 3) if g is not None]


def conv16_layers(plan, H=256, W=256):
    """(conv, input height, input width) of every conv16 layer of Engine16.forward, in call order"""
    from epipolarpose_b200.net import Conv
    from epipolarpose_b200.net16 import STEM_KPAD16
    out = []

    def add(conv, h, w):
        out.append((conv, h, w))
        return conv.out_hw(h, w)

    H1, W1 = plan.stem.out_hw(H, W)
    add(Conv("conv1", "conv", STEM_KPAD16, 64, 1, 1, 0), H1, W1)
    h, w = (H1 - 1) // 2 + 1, (W1 - 1) // 2 + 1          # 3x3 / 2 max-pool, pad 1
    for blk in plan.blocks:
        hh, ww = h, w
        for conv in blk["convs"]:
            hh, ww = add(conv, hh, ww)
        if blk["down"]:
            add(blk["down"][0], h, w)
        h, w = hh, ww
    for conv, _ in plan.deconvs:
        h, w = add(conv, h, w)
    add(plan.final, h, w)
    return out
