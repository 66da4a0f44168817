"""Shared by the training-step tests (test_gpu_step_kernels, test_gpu_c5_step, test_gpu_tf32x3_step,
test_gpu_c2_flat_step, test_gpu_refiner_step, test_gpu_infer_step, test_gpu_bn_chain, test_gpu_split16, test_gpu_tf32,
test_gpu_predictor, test_gpu_conv16_store and test_step_coverage): the float64 check bodies each composition runs at its own sizes, the bars and
the emulations they rest on, the restated planners, the layer tables, the device data makers and
one cache of models and conv outputs keyed by composition.

Every reference is torch float64 on the device, computed from the exact values the kernel read, so
each bar is the kernel's rounding and nothing else (u = 2^-24, one fp32 rounding).  A bar's
derivation is the docstring of the function that computes it."""
import contextlib
import math
import re

import numpy as np
import torch

from tests import emul_ops as em

U = 2.0 ** -24
HALF_MAX = 65504.0
NUM_SMS = 132          # common.cuh kNumSMs
EPS, MOM = 1e-5, 0.1
VAR_COEF = 1e-7        # VAR_BAR = VAR_COEF * (1 + r^2)
LOSS_THREADS = 1024    # softargmax.cu kLossThreads
H16 = torch.float16

FPROP_BAR = 2e-5       # fprop / dgrad output (and BatchNorm sums) against float64
WGRAD_BAR = 3e-5       # weight gradient: pixel reductions split over CTAs (red.add)
STATS_SELF_BAR = 1e-6  # BatchNorm sums against float64 sums of the kernel's own output


# ------------------------------------------------------------------ models and conv outputs, by composition
_CACHE = {}
# composition -> (layers, J, D, image size, precision) of its bench model
MODELS = {"c4_f16x3": (50, 16, 64, 256, "f16x3"), "c5": (101, 17, 96, 384, "f16x3"),
          "c4_tf32x3": (50, 16, 64, 256, "tf32x3"), "c2_flat": (50, 17, 64, 256, "f16x3")}
# compositions whose model has the VOLUME=False head: 2-D heat-maps and depth_fc (2048 -> J D)
FLAT_HEAD = {"c2_flat"}


def release(prefix):
    """drop every cached entry whose key starts with `prefix` and hand the allocator's reserve
    back to the device"""
    for k in [k for k in _CACHE if k.startswith(prefix)]:
        del _CACHE[k]
    if torch.cuda.is_initialized():
        import gc
        gc.collect()
        torch.cuda.empty_cache()


def bench_model(dev, comp):
    """the composition's bench model (MODELS) with FusedAdam over its parameters, built once;
    cached under `comp + "_model"`"""
    key = comp + "_model"
    if key not in _CACHE:
        import lib.models as models
        import lib.utils.utils as Ut
        layers, J, D, HW, precision = MODELS[comp]
        torch.manual_seed(0)
        m = models.pose3d_resnet.get_pose_net(_cfg(layers, J, D, HW, volume=comp not in FLAT_HEAD), False,
                                              precision=precision).to(dev).train()
        _CACHE[key] = (m, Ut.FusedAdam(list(m.parameters()), lr=1e-3))
    return _CACHE[key]


def _cfg(layers, J, D, HW, volume=True):
    from oracle import refshim
    return refshim.make_cfg(num_layers=layers, num_joints=J, volume=volume, depth_res=D, image_size=(HW, HW))


def _bench_meta(tuples, seed=1000):
    """the bench's synthetic cameras / boxes for `tuples` 4-view tuples (bench.py run_gpu)"""
    from tests.golden_inputs import _ring_meta
    return {k: torch.from_numpy(v) for k, v in _ring_meta(tuples, seed).items()}


# ------------------------------------------------------------------ device data
def _join(planes, sc):
    return (planes[0].double() + planes[1].double()) * float(sc[1])


def _split_dev(v):
    """fp32 -> split planes through the engine's split16_batch: (planes, sc, joined float64)"""
    from epipolarpose_b200 import ops
    h = torch.empty(2 * v.numel(), device=v.device, dtype=H16)
    sc = torch.ones(2, device=v.device)
    ops.split16_batch(ops.SplitBatch([(v.reshape(-1), h, sc)]))
    return h.view((2,) + tuple(v.shape)), sc, _join(h.view((2,) + tuple(v.shape)), sc)


def _rand_split(shape, seed, scale=16.0, relu=True, mag=1.0):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(shape, generator=g) * mag
    if relu:
        v = torch.relu(v)
    if scale is None:
        scale = em._pow2_scale(float(v.abs().max()))
    t = torch.empty((2,) + tuple(shape), dtype=H16)
    em._store_split(t, v, scale)
    sc = torch.tensor([scale, 1.0 / scale])
    return t, sc


def _weights_split(cout, K, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout * K, generator=g) * (2.0 / K) ** 0.5
    h = torch.empty(2 * cout * K, dtype=H16)
    sc = torch.ones(2)
    em.split16_batch(em.SplitBatch([(w, h, sc)]))
    return h, sc


# ------------------------------------------------------------------ what ran
@contextlib.contextmanager
def _record_calls():
    """the set of C-ABI entries called through ops._call (as bench.py's timed_call)"""
    from epipolarpose_b200 import ops
    names, orig = set(), ops._call

    def call(name, *a):
        names.add(name)
        return orig(name, *a)
    ops._call = call
    try:
        yield names
    finally:
        ops._call = orig


_KNAME = re.compile(r"conv_(fprop|wgrad)_(?:tc_kernel(?:<(\d+), ?(\d+)>|ILi(\d+)ELi(\d+)E)|(simt))")


def _ran(fn):
    """Runs fn under torch.profiler; returns the conv kernels that ran, as 'fprop_tc<128,3>',
    'wgrad_simt', ...  fn writes scratch buffers only: a short profiling session now and then
    delivers no device activity at all, and is then repeated (up to eight sessions).  Each
    session starts on an idle device and stays open a few milliseconds after fn's kernels have
    finished, so that their activity records are inside its window when it stops."""
    import time
    from torch.profiler import ProfilerActivity, profile
    tags = set()
    for _ in range(8):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
            time.sleep(0.005)
        for ev in prof.events():
            m = _KNAME.search(ev.name)
            if m:
                kind, a, b, c, d, simt = m.groups()
                tags.add("%s_simt" % kind if simt else "%s_tc<%s,%s>" % (kind, a or c, b or d))
        if tags:
            break
    return tags


_THREE_PASS = re.compile(r"^(fprop|wgrad)_tc<\d+,3>$")


def _all_three_pass(tags):
    """every conv kernel tag _ran reported is a 3xTF32 tensor-core instantiation"""
    return bool(tags) and all(_THREE_PASS.match(t) for t in tags)


# ------------------------------------------------------------------ TF32 operands and the tensor-core bar
def _tf32_np(x):
    """round to nearest TF32, ties away from zero (tc::to_tf32), in an fp32 container"""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def _tf32(t):
    """_tf32_np for a float32 torch tensor (int32 wrap-around == the unsigned add)"""
    return ((t.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def _trunc_np(x):
    """TF32 by truncation: what the tensor core reads from an fp32 container"""
    return (np.asarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)


def _tc_bar(base, K, passes):
    """Output bar of a tensor-core product over K: `base`, or the round-toward-zero accumulation
    floor of passes * K / 8 wgmma k-steps where that is larger.

    The H100's wgmma adds into its fp32 accumulator rounding toward zero, so that noise floor
    grows linearly with the number of k-steps x passes instead of as its square root.  Measured on
    one H100 80GB HBM3 at a 700 W power limit: 3.6e-5 .. 4.0e-5 for 3xTF32 and 1.2e-5 for TF32 at
    K = 4608 (3x3, 512 channels), ~7e-9 per 3xTF32 k-element; a round-toward-zero emulation of the
    same product gives the same numbers.  The tensor-core output bar is therefore
    max(2e-5, 0.75 * 2^-24 * passes * K / 8): 7.7e-5 for 3xTF32 at K = 4608, where a lost
    correction pass is still ~2e-4 off."""
    return max(base, 0.75 * 2.0 ** -24 * passes * K / 8)


def _rz32(x):
    """float64 -> fp32 rounded toward zero"""
    f = x.astype(np.float32)
    over = np.abs(f.astype(np.float64)) > np.abs(x)
    f[over] = np.nextafter(f[over], np.float32(0))
    return f


def _emul_mma(passes, K, toward_zero=False):
    """The tensor-core product of the kernels: per k-step of 8, each pass (a, b) adds the exact
    8-term dot products to the fp32 accumulator, in the order given; the add rounds to nearest,
    or toward zero as the H100's wgmma does."""
    M, N = passes[0][0].shape[0], passes[0][1].shape[1]
    acc = np.zeros((M, N), np.float32)
    for k0 in range(0, K, 8):
        for a, b in passes:
            part = a[:, k0:k0 + 8].astype(np.float64) @ b[k0:k0 + 8].astype(np.float64)
            acc = _rz32(acc + part) if toward_zero else acc + part.astype(np.float32)
    return acc


def _layer(dev, kind, cin, cout, k, s, p, opad, N, H, W, seed):
    """Random layer at the padded channel counts the engine uses: NHWC input x, BatchNorm affine
    (sc, sh) of the producing layer, weights in the state_dict layout with the padding rows /
    columns zero, and the upstream gradient of the output."""
    from epipolarpose_b200 import net
    conv = net.Conv("t", kind, cin, cout, k, s, p, opad)
    Ho, Wo = conv.out_hw(H, W)
    g = torch.Generator(device=dev).manual_seed(seed)
    ci, co = conv.cin_p, conv.cout_p
    x = torch.randn(N, H, W, ci, device=dev, generator=g)
    sc = torch.rand(ci, device=dev, generator=g) + 0.5
    sh = torch.randn(ci, device=dev, generator=g) * 0.1
    w = torch.randn((co, ci, k, k) if kind == "conv" else (ci, co, k, k), device=dev, generator=g)
    w *= (2.0 / (k * k * cin)) ** 0.5
    if kind == "conv":
        w[cout:], w[:, cin:] = 0, 0
    else:
        w[cin:], w[:, cout:] = 0, 0
    gout = torch.randn(N, Ho, Wo, co, device=dev, generator=g)
    gout[..., cout:] = 0
    return conv, Ho, Wo, x, sc, sh, w.contiguous(), gout


def _act64(x, sc, sh, relu):
    """f(x) = max(fma(x, sc, sh), lb) exactly as the producers compute it (one fp32 rounding), as
    float64 NCHW; affine None -> x itself"""
    if sc is None:
        f = x
    else:
        f = (x.double() * sc.double() + sh.double()).float()
        if relu:
            f = torch.relu(f)
    return f.permute(0, 3, 1, 2).double()


def _fwd64(conv, a, w):
    import torch.nn.functional as F
    if conv.kind == "conv":
        return F.conv2d(a, w, None, conv.stride, conv.pad)
    return F.conv_transpose2d(a, w, None, conv.stride, conv.pad, conv.opad)


def _guarded(shape, dev, fill):
    """A tensor followed by a 64-float guard band that must stay untouched."""
    n = int(np.prod(shape))
    buf = torch.full((n + 64,), fill, device=dev)
    return buf[:n].view(shape), buf[n:]


def _geoms(geoms, relu=0, acc=0):
    out = []
    for gm in geoms:
        if gm is not None:
            gm.in_relu, gm.accumulate = relu, acc
            out.append(gm)
    return out


# ------------------------------------------------------------------ planners restated
KPIX, WM_TF32 = 32, 128          # conv_tc_wgrad.cu: pixels per tile, co rows per tile
RUN_BLOCKS3 = 184                # conv_tc_wgrad.cu kMaxRunBlocks3


def _tf32_wgrad_plan(M, Cin, Cout, T, NS, cap=True):
    """conv_tc_wgrad.cu launch_wgrad: (pixel run per CTA, splits, tiles); cap=False is the
    planner without the run cap"""
    bnw = 128 if Cin >= 128 else (64 if Cin >= 64 else 32)
    co_tiles, ci_tiles = -(-Cout // WM_TF32), -(-Cin // bnw)
    total = T * ci_tiles
    groups = -(-total // (128 // bnw))
    nb = -(-total // groups)
    tiles = co_tiles * -(-total // nb)
    max_splits = -(-M // (8 * KPIX))
    min_splits = -(-M // (RUN_BLOCKS3 * 3 // NS * KPIX)) if cap else 1
    splits, best, sp = min_splits, -1, min_splits
    while sp <= max_splits and (sp - min_splits) * tiles <= 3 * NUM_SMS:
        cost = -(-(sp * tiles) // NUM_SMS) * (-(-(-(-M // sp)) // KPIX) + 6)
        if best < 0 or cost < best:
            best, splits = cost, sp
        sp += 1
    rows = -(-(-(-M // splits)) // KPIX) * KPIX
    return rows, -(-M // rows), tiles


def _choose_tile(N, Hp, Wp, rows):
    """split16_common.cuh epb_choose_tile: (tw, th, tn)"""
    best, out = -1, (rows, 1, 1)
    a = rows
    while a >= 1:
        b = rows // a
        while b >= 1:
            c = rows // (a * b)
            cov = -(-Wp // a) * -(-Hp // b) * -(-N // c)
            if best < 0 or cov < best:
                best, out = cov, (a, b, c)
            b >>= 1
        a >>= 1
    return out


def _wgrad16_plan(gm, ws_floats=48 << 20):
    """wgrad16.cu epb_conv16_wgrad: (pixel run per CTA = tiles_per_split x 64, splits)"""
    KT = 64
    N, Hp, Wp = gm.N, gm.Hp, gm.Wp
    if gm.T == 1 and gm.is_ == 1 and gm.os == 1 and gm.dh[0] == 0 and gm.dw[0] == 0 and \
            Hp == gm.Hi and Wp == gm.Wi and Hp == gm.Ho and Wp == gm.Wo:
        N, Hp, Wp = 1, 1, gm.N * gm.Hp * gm.Wp
    tw, th, tn = _choose_tile(N, Hp, Wp, KT)
    tiles = -(-Wp // tw) * -(-Hp // th) * -(-N // tn)
    CH = gm.T * (gm.Cin // 64)
    swap = gm.T == 1 and CH < 2 and gm.Cout // 64 > CH
    if swap:
        CH, Nn = gm.Cout // 64, gm.Cin
    else:
        Nn = gm.Cout
    bn = 64 if Nn <= 64 else 128
    basec = ((CH + 1) // 2) * -(-Nn // bn)
    splits = min(2 * NUM_SMS // basec, tiles // 8)
    per_split = gm.Cout * gm.Tw * gm.Cin
    if splits * per_split > ws_floats:
        splits = ws_floats // per_split
    splits = max(splits, 1)
    tps = -(-tiles // splits)
    return tps * KT, -(-tiles // tps)


# ------------------------------------------------------------------ layer tables
# The f16x3 bench's layer shapes (profiles/r2_step_table_f16x3.md): N = 128 images, every distinct
# conv kind / channel pair of ResNet-50 at 256x256.  (name, kind, cin, cout, k, stride, pad, input hw)
C4_LAYERS_SPLIT16 = [
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 64), ("l1_1x1_256_64", "conv", 256, 64, 1, 1, 0, 64),
    ("l1_3x3_64", "conv", 64, 64, 3, 1, 1, 64), ("l2_3x3_s2", "conv", 128, 128, 3, 2, 1, 64),
    ("l2_1x1_s2_down", "conv", 256, 512, 1, 2, 0, 64), ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 16),
    ("l3_1x1_1024_256", "conv", 1024, 256, 1, 1, 0, 16), ("l4_3x3_512", "conv", 512, 512, 3, 1, 1, 8),
    ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 8), ("deconv0", "deconv", 2048, 256, 4, 2, 1, 8),
    ("deconv2", "deconv", 256, 256, 4, 2, 1, 32), ("final", "conv", 256, 1024, 1, 1, 0, 64),
]

# every distinct conv of R50 at 256 x 256 (trunk at 64 / 32 / 16 / 8, deconvs 8 -> 64, the final
# 1 x 1 with bias), the stem as a 1 x 1 conv over its 160-column patch matrix; (name, kind, cin,
# cout, k, stride, pad, input hw, operand, dgrad).  operand "in": a materialised tensor (patch
# matrix, pool or block output); "act": the producer's BatchNorm + ReLU applied on load.
# dgrad "write", "acc" (a downsample adds into the block's input gradient) or None (the stem).
C4_LAYERS_TF32X3 = [
    ("stem_col_160_64", "conv", 160, 64, 1, 1, 0, 128, "in", None),
    ("l1_1x1_64_64", "conv", 64, 64, 1, 1, 0, 64, "in", "write"),
    ("l1_3x3_64", "conv", 64, 64, 3, 1, 1, 64, "act", "write"),
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 64, "act", "write"),
    ("l1_down_64_256", "conv", 64, 256, 1, 1, 0, 64, "in", "acc"),
    ("l1_1x1_256_64", "conv", 256, 64, 1, 1, 0, 64, "in", "write"),
    ("l2_1x1_256_128", "conv", 256, 128, 1, 1, 0, 64, "in", "write"),
    ("l2_3x3_s2_128", "conv", 128, 128, 3, 2, 1, 64, "act", "write"),
    ("l2_1x1_128_512", "conv", 128, 512, 1, 1, 0, 32, "act", "write"),
    ("l2_down_s2_256_512", "conv", 256, 512, 1, 2, 0, 64, "in", "acc"),
    ("l2_1x1_512_128", "conv", 512, 128, 1, 1, 0, 32, "in", "write"),
    ("l2_3x3_128", "conv", 128, 128, 3, 1, 1, 32, "act", "write"),
    ("l3_1x1_512_256", "conv", 512, 256, 1, 1, 0, 32, "in", "write"),
    ("l3_3x3_s2_256", "conv", 256, 256, 3, 2, 1, 32, "act", "write"),
    ("l3_1x1_256_1024", "conv", 256, 1024, 1, 1, 0, 16, "act", "write"),
    ("l3_down_s2_512_1024", "conv", 512, 1024, 1, 2, 0, 32, "in", "acc"),
    ("l3_1x1_1024_256", "conv", 1024, 256, 1, 1, 0, 16, "in", "write"),
    ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 16, "act", "write"),
    ("l4_1x1_1024_512", "conv", 1024, 512, 1, 1, 0, 16, "in", "write"),
    ("l4_3x3_s2_512", "conv", 512, 512, 3, 2, 1, 16, "act", "write"),
    ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 8, "act", "write"),
    ("l4_down_s2_1024_2048", "conv", 1024, 2048, 1, 2, 0, 16, "in", "acc"),
    ("l4_1x1_2048_512", "conv", 2048, 512, 1, 1, 0, 8, "in", "write"),
    ("l4_3x3_512", "conv", 512, 512, 3, 1, 1, 8, "act", "write"),
    ("deconv0_2048_256", "deconv", 2048, 256, 4, 2, 1, 8, "in", "write"),
    ("deconv1_256", "deconv", 256, 256, 4, 2, 1, 16, "act", "write"),
    ("deconv2_256", "deconv", 256, 256, 4, 2, 1, 32, "act", "write"),
    ("final_256_1024", "conv", 256, 16 * 64, 1, 1, 0, 64, "act", "write"),
]

# every distinct conv of R101 at 384 x 384 (trunk at 96 / 48 / 24 / 12, deconvs 12 -> 96), the
# stem's patch-matrix conv; (name, kind, cin, cout, k, stride, pad, input hw)
C5_LAYERS = [
    ("stem_col_192_64", "conv", 192, 64, 1, 1, 0, 192),
    ("l1_1x1_64_64", "conv", 64, 64, 1, 1, 0, 96), ("l1_3x3_64", "conv", 64, 64, 3, 1, 1, 96),
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 96), ("l1_1x1_256_64", "conv", 256, 64, 1, 1, 0, 96),
    ("l2_1x1_256_128", "conv", 256, 128, 1, 1, 0, 96), ("l2_3x3_s2", "conv", 128, 128, 3, 2, 1, 96),
    ("l2_1x1_s2_down", "conv", 256, 512, 1, 2, 0, 96), ("l2_3x3_128", "conv", 128, 128, 3, 1, 1, 48),
    ("l2_1x1_512_128", "conv", 512, 128, 1, 1, 0, 48), ("l3_3x3_s2", "conv", 256, 256, 3, 2, 1, 48),
    ("l3_1x1_s2_down", "conv", 512, 1024, 1, 2, 0, 48), ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 24),
    ("l3_1x1_1024_256", "conv", 1024, 256, 1, 1, 0, 24), ("l3_1x1_256_1024", "conv", 256, 1024, 1, 1, 0, 24),
    ("l4_3x3_s2", "conv", 512, 512, 3, 2, 1, 24), ("l4_1x1_s2_down", "conv", 1024, 2048, 1, 2, 0, 24),
    ("l4_3x3_512", "conv", 512, 512, 3, 1, 1, 12), ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 12),
    ("deconv0", "deconv", 2048, 256, 4, 2, 1, 12), ("deconv1", "deconv", 256, 256, 4, 2, 1, 24),
    ("deconv2", "deconv", 256, 256, 4, 2, 1, 48),
]

# every distinct split-path conv of R50 at 256 x 256 (trunk at 64 / 32 / 16 / 8, deconvs 8 -> 64),
# the stem's patch-matrix conv (K 147 -> 192, whole 64-channel blocks); (name, kind, cin, cout, k,
# stride, pad, input hw).  The final layer (256 -> J with bias) has its own test.
C2_LAYERS = [
    ("stem_col_192_64", "conv", 192, 64, 1, 1, 0, 128),
    ("l1_1x1_64_64", "conv", 64, 64, 1, 1, 0, 64), ("l1_3x3_64", "conv", 64, 64, 3, 1, 1, 64),
    ("l1_1x1_64_256", "conv", 64, 256, 1, 1, 0, 64), ("l1_1x1_256_64", "conv", 256, 64, 1, 1, 0, 64),
    ("l2_1x1_256_128", "conv", 256, 128, 1, 1, 0, 64), ("l2_3x3_s2", "conv", 128, 128, 3, 2, 1, 64),
    ("l2_1x1_128_512", "conv", 128, 512, 1, 1, 0, 32), ("l2_1x1_s2_down", "conv", 256, 512, 1, 2, 0, 64),
    ("l2_1x1_512_128", "conv", 512, 128, 1, 1, 0, 32), ("l2_3x3_128", "conv", 128, 128, 3, 1, 1, 32),
    ("l3_1x1_512_256", "conv", 512, 256, 1, 1, 0, 32), ("l3_3x3_s2", "conv", 256, 256, 3, 2, 1, 32),
    ("l3_1x1_256_1024", "conv", 256, 1024, 1, 1, 0, 16), ("l3_1x1_s2_down", "conv", 512, 1024, 1, 2, 0, 32),
    ("l3_1x1_1024_256", "conv", 1024, 256, 1, 1, 0, 16), ("l3_3x3_256", "conv", 256, 256, 3, 1, 1, 16),
    ("l4_1x1_1024_512", "conv", 1024, 512, 1, 1, 0, 16), ("l4_3x3_s2", "conv", 512, 512, 3, 2, 1, 16),
    ("l4_1x1_512_2048", "conv", 512, 2048, 1, 1, 0, 8), ("l4_1x1_s2_down", "conv", 1024, 2048, 1, 2, 0, 16),
    ("l4_1x1_2048_512", "conv", 2048, 512, 1, 1, 0, 8), ("l4_3x3_512", "conv", 512, 512, 3, 1, 1, 8),
    ("deconv0", "deconv", 2048, 256, 4, 2, 1, 8), ("deconv1", "deconv", 256, 256, 4, 2, 1, 16),
    ("deconv2", "deconv", 256, 256, 4, 2, 1, 32),
]


# ------------------------------------------------------------------ optimiser
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
    """(e_m, e_v, e_upd); Em / Ev carried errors of m0 / v0; k scales the rounding terms;
    torch_ref: (r_c1, r_c2, r_b1, r_b2, r_lr, r_bc1, r_bc2)

    The contract: Adam with lr, beta1, beta2, eps, wd, grad_scale AS STORED in the fp32 `hyper`
    tensor, the bias corrections from those fp32 betas in double.  The kernel rounds g = G gs
    (+ wd P) (e_g <= 2u (|G gs| + |wd P|)), then m = b1 m0 + (1-b1) g and v = b2 v0 + (1-b2) g^2
    (1-b fp32 is exact for b in [0.5, 1]).  m and v cancel, so their bars are on the terms, not on
    the result: e_m = (1-b1) e_g + 3u (|b1 m0| + |(1-b1) g|), e_v = 2 (1-b2) |g| e_g + 4u (b2 v0 +
    (1-b2) g^2).  sqrt moves e_v to e_v / max(sqrt v, sqrt e_v); the denominator sqrt(v) rsqrt_bc2
    + eps adds three roundings (rsqrt_bc2 stored in fp32, the product, + eps), the quotient one,
    lr / bc1 two, the product one, and p - step q rounds once more, to u |p1|.  The update p1 - p0
    is compared, not p1, so that last term is the only one that depends on |p|.  K steps from the
    kernel's own state: m and v errors carry over as E_m <- b1 E_m + e_m, E_v <- b2 E_v + e_v, the
    parameter error adds each step's update bar.

    Against torch.optim.Adam (fp32, same state, torch_ref): torch keeps the betas in double, so
    (1-b1), (1-b2) and the bias corrections differ by their fp32 rounding (r_c1 ~ 2.4e-7, r_c2 ~
    1.3e-5, measured from the stored values) on top of both implementations' roundings (k = 2: 2x
    the kernel's u terms) and both final roundings of p."""
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


def _check_fused_adam(dev, m, opt):
    """FusedAdam steps 1, 2 and 1000 over the model's flat buffer: update / m / v per element
    against the float64 contract of _adam_bar, and the update against torch.optim.Adam"""
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


# ------------------------------------------------------------------ weight split and pack, stem
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
    """pow2_scale: 2^(13 - floor(log2 bound))"""
    if not bound > 0 or not math.isfinite(bound):
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 13 - (math.frexp(bound)[1] - 1))))


def _check_split16_batch(dev, m, opt):
    """split16_batch on the engine's weight jobs (after one Adam step) plus synthetic jobs in the
    same batch: bit-exact with the CPU emulation (tests/emul_ops.py), planes compared as int16,
    both scale words; the scale is pow2_scale(amax), max|hi| <= 2^14."""
    from epipolarpose_b200 import ops
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
        em.split16_batch(em.SplitBatch([(cs, ch, csc)]))
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


def _check_pack_weight_batch(dev, m):
    """pack_weight_batch on the engine's model-scale jobs: bit-exact with the CPU emulation (a
    permutation: no arithmetic)"""
    from epipolarpose_b200 import ops
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
            em.pack_weight_batch(em.PackBatch([(src.detach().cpu(), cdst) + tuple(j[2:])]))
            got = dst.detach().cpu()
            # every element the emulation writes (operand, zero padding) bit for bit
            w_ = ~torch.isnan(cdst)
            assert bool(w_.any()) and not bool(torch.isnan(got[w_]).any()), what
            assert torch.equal(got[w_].view(torch.int32), cdst[w_].view(torch.int32)), what
            njobs += 1
    print("  pack / unpack: %d jobs bit-exact" % njobs)


def _check_im2col_split(dev, kpad, N, H):
    """im2col_split of N images of H x H (7 x 7 / 2, pad 3), bit-exact with the CPU emulation on
    up to five images"""
    from epipolarpose_b200 import ops, net16
    W = H
    Ho = Wo = H // 2
    g = torch.Generator(device=dev).manual_seed(51)
    img = torch.randn(N, 3, H, W, device=dev, generator=g)
    big = min(5, N - 1)
    img[big, :, 0, :] = 4094.0 / net16.IMG_SCALE            # the static scale's largest magnitude
    col = torch.empty(2, N, Ho, Wo, kpad, device=dev, dtype=torch.float16)
    sc = torch.tensor([net16.IMG_SCALE, 1.0 / net16.IMG_SCALE, 65504.0 / net16.IMG_SCALE, 0.0], device=dev)
    ops.im2col_split(img, col, sc, N, 3, H, W, 7, 7, 2, 3, Ho, Wo, kpad)
    torch.cuda.synchronize()
    pick = sorted({0, big, max(0, N // 2 - 1), N // 2, N - 1})
    cimg = img[pick].cpu()
    ccol = torch.empty(2, len(pick), Ho, Wo, kpad, dtype=torch.float16)
    em.im2col_split(cimg, ccol, sc.cpu(), len(pick), 3, H, W, 7, 7, 2, 3, Ho, Wo, kpad)
    got = col[:, pick].cpu()
    assert torch.equal(got.view(torch.int16), ccol.view(torch.int16))
    print("  im2col_split: images %s bit-exact (K pad %d)" % (pick, kpad))


def _check_maxpool_bwd(dev, N, H):
    """maxpool_bwd of the stem's pool over N images of H x H x 64.  Each input element sums at
    most 4 window gradients in (kh, kw) order from 0: <= 3u sum|g| against float64, and bit-equal
    with an fp32 restatement in that order."""
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


# ------------------------------------------------------------------ soft-argmax, joint loss, colsum
def _nhwc_geometry(N, J, D, H, W):
    """epb_softargmax_fwd (NHWC): split count S, pixels per trip ppi, depth d of a term"""
    C4 = J * D // 4
    ppi = max(512 // C4, 1)
    S = 1
    while N * S < 8 * NUM_SMS and (H * W) // (S * 2) >= 16 * ppi:
        S *= 2
    L = -(-(-(-(H * W) // S)) // ppi)
    return S, ppi, L + 2 + (D // 4) * ppi + S


def _check_softargmax_fwd(dev, kind, N, J, D, H, W):
    """epb_softargmax_fwd (NHWC) at one shape against float64 within the merge-depth bar.

    A logit's term exp(v - m) meets d = L + 2 + D4 ppi + S additions (L pixels per thread, the
    quad, the CTA merge of D4 ppi partials, the S-way finalize) and at most as many rescale factors
    exp(m_a - m_b).  With the __expf model of the backward ((6 + 3.5|x|) u) and rescale arguments
    that add up to at most |v - m|, the factor a term carries into s, sx, sy, sz alike is off by
    eps_i <= (6 + 7|v - m| + 6 d) u; on top, each of those positive sums is off by 2 d u relative
    from its own additions and rescale products.  So a coordinate c' = c + 1/2 is off by sum_i p_i
    |pos_i - c'| eps_i + 4 d u c' + 4u, lse[1] = 1 / sum exp(v - m) by sum_i p_i eps_i + 2 d u + 2u,
    and lse[0] is the maximum: exact."""
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
    worst_c, worst_l, maxerr, max_ok = _softargmax_ratios(logits, coords, lse, N, J, D, H, W)
    assert max_ok, "lse[0] is not the maximum"
    print("  softargmax fwd %-8s S %d ppi %d depth %d: coords max err %.3e worst err / bar %.3f, "
          "lse[1] worst err / bar %.3f" % (kind, S, ppi, d, maxerr, worst_c, worst_l))
    assert worst_c <= 1.0 and worst_l <= 1.0


def _softargmax_ratios(logits, coords, lse, N, J, D, H, W):
    """(worst coordinate err / bar, worst lse[1] err / bar, largest coordinate error, lse[0] is the
    maximum exactly) of an NHWC soft-argmax forward over the fp32 volume `logits` [N, H, W, J*D]
    that it read, with the bars of _check_softargmax_fwd"""
    dev = logits.device
    S, ppi, d = _nhwc_geometry(N, J, D, H, W)
    xs = torch.arange(W, device=dev, dtype=torch.float64).view(1, 1, W, 1, 1) / W
    ys = torch.arange(H, device=dev, dtype=torch.float64).view(1, H, 1, 1, 1) / H
    zs = torch.arange(D, device=dev, dtype=torch.float64).view(1, 1, 1, 1, D) / D
    lk = lse.view(N, J, 2)
    worst_c, worst_l, maxerr, max_ok = 0.0, 0.0, 0.0, True
    for n0 in range(0, N, 8):
        B = min(8, N - n0)
        v = logits[n0:n0 + B].double().view(B, H, W, J, D)
        m = v.amax((1, 2, 4), keepdim=True)
        max_ok = max_ok and torch.equal(lk[n0:n0 + B, :, 0].double(), m.view(B, J))
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
    return worst_c, worst_l, maxerr, max_ok


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


def _check_jointloss(dev, kind, norm, N, J):
    """epb_jointloss_fwd_bwd over n = N J 3 elements against float64.

    One CTA of 1024 threads: each thread adds n / 1024 terms, then a 10-level tree: depth dl =
    n / 1024 + 12, |d loss| <= dl u sum|w l| / div.  Without norm x and t are dyadic, d is exact
    and dx rounds at most twice.  With norm, 1 / sum|x| and 1 / sum|t| carry dl + 1 roundings into
    every d (ed = (dl + 3) u (|x_n| + |t_n|)), and the norm term of dx sums g x over all elements
    (3 dl + 6 roundings on sum|g x| / sum|x|^2)."""
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


def _sabwd_ref_bar(v, coords, lse, dco, H, W, D):
    """float64 p (s - s_bar) for logits v [B, H, W, J, D] and its per-element bar from the
    kernel's own coords / lse.

    Soft-argmax backward, fp32 NHWC: p (s - s_bar) per element within the model of the split
    backward's bar (exp ((6 + 3.5 |v - m|) u), the fp32 s and s_bar (6u on their terms, which for
    s_bar are its three products: they cancel where |s_bar| is small), the kernel's s_bar from its
    forward coords + 1/2, its 1 / sum exp from lse) without the plane-rounding term: the output is
    fp32."""
    B, J = v.shape[0], v.shape[3]
    dev = v.device
    xs = torch.arange(W, device=dev, dtype=torch.float64).view(1, 1, W, 1, 1)
    ys = torch.arange(H, device=dev, dtype=torch.float64).view(1, H, 1, 1, 1)
    zs = torch.arange(D, device=dev, dtype=torch.float64).view(1, 1, 1, 1, D)
    m = v.amax((1, 2, 4), keepdim=True)
    ex = torch.exp(v - m)
    tot = ex.sum((1, 2, 4), keepdim=True)
    p = ex / tot
    del ex
    dc = dco.double().view(B, 1, 1, J, 3)
    gx, gy, gz = dc[..., 0:1] / W, dc[..., 1:2] / H, dc[..., 2:3] / D
    s_ = gx * xs + gy * ys + gz * zs
    sbar = (p * s_).sum((1, 2, 4), keepdim=True)
    dl = p * (s_ - sbar)
    cr = coords.double().view(B, 1, 1, J, 3)
    tx, ty, tz = gx * (cr[..., 0:1] + 0.5) * W, gy * (cr[..., 1:2] + 0.5) * H, gz * (cr[..., 2:3] + 0.5) * D
    sbar_k = tx + ty + tz
    sbar_t = tx.abs() + ty.abs() + tz.abs()              # s_bar's terms: they may cancel
    ik = lse.view(B, J, 2)[..., 1].double().view(B, 1, 1, J, 1)
    e_inv = (ik * tot - 1).abs()
    e = p * ((6 + 3.5 * (v - m).abs()) * U * (s_ - sbar).abs()
             + 6 * U * ((gx * xs).abs() + (gy * ys).abs() + (gz * (zs + 3)).abs() + sbar_t)
             + (sbar_k - sbar).abs() + e_inv * (s_ - sbar).abs())
    return dl, e


def _check_softargmax_bwd_fp32(dev, N, J, D, H, W):
    """epb_softargmax_bwd (fp32 NHWC) at one shape against float64 within _sabwd_ref_bar"""
    from epipolarpose_b200 import ops
    C = J * D
    g = torch.Generator(device=dev).manual_seed(93)
    logits = torch.randn(N, H, W, C, device=dev, generator=g) * 3
    dco = torch.randn(N, J * 3, device=dev, generator=g)
    coords, lse = torch.empty(N, J * 3, device=dev), torch.empty(N * J * 2, device=dev)
    ops.softargmax_fwd(logits, 1, N, J, D, H, W, coords, lse)
    dl = torch.empty_like(logits)
    ops.softargmax_bwd(logits, 1, N, J, D, H, W, coords, lse, dco, dl)
    torch.cuda.synchronize()
    ratio, worst = 0.0, 0.0
    B = 8
    for n0 in range(0, N, B):
        v = logits[n0:n0 + B].double().view(B, H, W, J, D)
        ref, e = _sabwd_ref_bar(v, coords[n0:n0 + B], lse.view(N, J * 2)[n0:n0 + B], dco[n0:n0 + B], H, W, D)
        del v
        err = (dl[n0:n0 + B].double().view(B, H, W, J, D) - ref).abs()
        worst = max(worst, float(err.max()))
        ratio = max(ratio, float((err / (e + 1e-300)).max()))
        del ref, e, err
    print("  softargmax bwd fp32 N %d J %d D %d %dx%d: max err %.3e, worst err / bar %.3f" % (N, J, D, H, W, worst, ratio))
    assert ratio <= 1.0


def _check_colsum(dev, M, C):
    """epb_colsum over M x C against float64 column sums; a second run within one fp32 ulp.

    Each thread adds kRowsPerThread = 64 rows in fp32 (<= 64 u sum|x| per column), the CTA's row
    slots and all CTAs add in double (<= (rpi + CTAs) 2^-53 sum|x|), the result rounds once to
    fp32 (u |S|).  Double atomics reorder between runs: two runs agree within one fp32 ulp."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(95)
    x = torch.randn(M, C, device=dev, generator=g) * 1e-3
    x[:, :8] += 1e-3                                            # columns with a consistent sign
    out, out2 = torch.empty(C, device=dev), torch.empty(C, device=dev)
    ops.colsum(x, M, C, out)
    ops.colsum(x, M, C, out2)
    torch.cuda.synchronize()
    ref = torch.zeros(C, device=dev, dtype=torch.float64)
    sab = torch.zeros(C, device=dev, dtype=torch.float64)
    for r0 in range(0, M, 1 << 16):
        xd = x[r0:r0 + (1 << 16)].double()
        ref += xd.sum(0)
        sab += xd.abs().sum(0)
    rpi = max(256 // (C // 4), 1)                               # bn.cu make_rowmap
    ctas = -(-M // (64 * rpi))
    bar = 64 * U * sab + (rpi + ctas) * 2.0 ** -53 * sab + U * ref.abs()
    err = (out.double() - ref).abs()
    ulp = (out.double().abs() * 2.0 ** -23).clamp_min(2.0 ** -149)
    print("  colsum M %d C %d: max err %.3e, worst err / bar %.3f, second run identical %s"
          % (M, C, float(err.max()), float((err / bar).max()), bool(torch.equal(out, out2))))
    assert bool((err <= bar).all())
    assert bool(((out.double() - out2.double()).abs() <= ulp).all())


# ------------------------------------------------------------------ the split-fp16 BatchNorm chain
def _kappa(M):
    """split16.cu channel_bound: fp32 roundings a value meets in the conv16 statistics"""
    return 16 + math.ceil(M / (16.0 * NUM_SMS))


def _bound_def(s1, s2, sc, sh, M):
    """per-channel bound of |sc z + sh| from float64 statistics (split16.cu channel_bound)"""
    mean, q = s1 / M, s2 / M
    var = (q - mean * mean).clamp_min(0)
    ku = _kappa(M) * U
    return (sc * mean + sh).abs() + sc.abs() * (torch.sqrt(M * (var + 4 * ku * q)) + ku * torch.sqrt(q))


def _act_rule(bound):
    """publish_act_scale: the largest power of two s with s * bound < 2^15"""
    if not bound > 0:
        return 1.0
    return math.ldexp(1.0, max(-100, min(100, 15 - math.frexp(bound)[1])))


def _scale_ok(s, bound, rule):
    want = rule(bound)
    edge = bound > 0 and abs(math.log2(bound) - round(math.log2(bound))) < 1e-3
    return s == want or (edge and s in (want / 2, want * 2))


def _tile_runs(M, bm=128):
    """conv16 with statistics (m-fastest order) on a dense [M] grid: the tiles each CTA runs per
    N tile -- the length of the longest run and the number of CTAs per N tile"""
    tiles = -(-M // bm)
    grid = min(tiles, NUM_SMS)
    return -(-tiles // grid), grid


def _stats_depth(M):
    return 13 + _tile_runs(M)[0]


def _bwd_rows(M, C):
    """split16.cu make_rowmap + bn_bwd_workers: rows each partial thread sums, row slots per CTA"""
    C4 = C // 4
    tpr = min(C4, 256)
    rpi = max(256 // tpr, 1)
    chunks = -(-C4 // tpr)
    nblk = -(-M // rpi)
    cap = max(NUM_SMS * 3 // chunks, 1)
    workers = max(min(-(-nblk // 4), cap), 1)
    return -(-nblk // workers), rpi


def _finalize64(s1, s2, M, gamma, beta, rm, rv):
    """bn_finalize_scale in float64 on float64 statistics and the fp32 parameters it reads"""
    eps, mom = float(np.float32(EPS)), float(np.float32(MOM))
    mean = s1 / M
    var = np.maximum(s2 / M - mean * mean, 0)
    inv = 1 / np.sqrt(var + eps)
    g, b = gamma.astype(np.float64), beta.astype(np.float64)
    unb = var * (M / (M - 1.0 if M > 1 else 1.0))
    return dict(mean=mean, invstd=inv, scale=g * inv, shift=b - mean * g * inv,
                rm=(1 - mom) * rm.astype(np.float64) + mom * mean,
                rv=(1 - mom) * rv.astype(np.float64) + mom * unb)


def _ulps(got, ref):
    """|got - ref| in units of the fp32 spacing at ref"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    sp = np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    sp = np.where(sp > 0, sp, np.spacing(np.float32(0)))
    return np.abs(got - ref) / sp


def _no_clamp(planes):
    """no element of the hi plane sits at split2's clamp"""
    return not bool((planes[0].float().abs() >= HALF_MAX).any())


def _contract_act(what, planes, sc, bound, ymax):
    """The scale contract: s is the power of two its rule gives from the bound computed here in
    float64 from its definition (a factor of 2 only within 1e-3 of a power of two), and no element
    of a hi plane is +-65504, the clamp in split2 (a silent clip)."""
    s = float(sc[0])
    print("  %-34s s 2^%d bound %.4e s*max|y| %.1f" % (what, int(math.log2(s)), bound, s * ymax))
    assert _no_clamp(planes), "%s: hi plane at the fp16 clamp" % what
    assert s * ymax < HALF_MAX
    assert _scale_ok(s, bound, _act_rule), "%s: s %g, rule gives %g from %g" % (what, s, _act_rule(bound), bound)
    assert float(sc[1]) == 1 / s


def _stats64(z2d):
    z = z2d.double()
    return torch.cat([z.sum(0), (z * z).sum(0)])


R_TARGETS = (0.0, 1.0, 10.0, 100.0)


def _produce(dev, case):
    """conv16_fprop with statistics at a bench shape; case = (name, kind, cin, cout, k, stride,
    pad, N, hw, offset taps), the offset taps being the weight taps that read the constant input
    channel 0 at every output pixel exactly once (never padding).  Input: relu(randn) with
    channel 0 == 1, so adding o_c to the weights of channel 0 at the offset taps shifts output
    channel c by o_c exactly; o_c targets mean / std = R_TARGETS[c % 4].  Returns (z [M, C], stats,
    stats of a second run, conv); the stem and layer1 outputs the apply and pool checks reuse are
    cached under the case's name."""
    name, kind, cin, cout, k, s, p, N, hw, taps = case
    if name in _CACHE:
        return _CACHE[name]
    from epipolarpose_b200 import net, ops
    conv = net.Conv("t", kind, cin, cout, k, s, p, 0)
    Ho, Wo = conv.out_hw(hw, hw)
    g = torch.Generator(device=dev).manual_seed(17)
    xf = torch.relu(torch.randn(N, hw, hw, cin, device=dev, generator=g))
    xf[..., 0] = 1.0
    x, x_sc, _ = _split_dev(xf)
    del xf
    K = k * k * cin
    w = torch.randn((cout, cin, k, k) if kind == "conv" else (cin, cout, k, k), device=dev, generator=g)
    w *= (2.0 / K) ** 0.5
    wc = w if kind == "conv" else w.transpose(0, 1)             # [cout][cin][k][k] view
    wc[:, 0] = 0
    # z_c ~ sum w x over the taps one pixel meets (all of a conv's, 1/4 of this deconv's);
    # relu(randn) has mean 1/sqrt(2 pi) and variance 1/2 - 1/(2 pi)
    frac = 1.0 if kind == "conv" else 0.25
    sd = torch.sqrt((wc[:, 1:] ** 2).sum((1, 2, 3)) * frac * (0.5 - 0.5 / math.pi))
    mu = wc[:, 1:].sum((1, 2, 3)) * frac / math.sqrt(2 * math.pi)
    rt = torch.tensor([R_TARGETS[c % 4] for c in range(cout)], device=dev)
    off = rt * sd - mu
    for a, b in taps:
        wc[:, 0, a, b] = off
    wf32, _ = conv.pack(ops, w)
    wf, wf_sc, _ = _split_dev(wf32)
    out = torch.empty(N, Ho, Wo, cout, device=dev)
    runs = []
    for _ in range(2):
        st = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
        for gm in conv.fprop_geoms(ops, N, hw, hw, 3):
            if gm is not None:
                gm.in_relu, gm.accumulate = 0, 0
                ops.conv16_fprop(gm, x, x_sc, wf, wf_sc, out, None, st)
        runs.append(st)
    torch.cuda.synchronize()
    M = N * Ho * Wo
    res = (out.view(M, cout), runs[0], runs[1], conv)
    if name.endswith(("stem_col_192_64", "l1_1x1_64_256")):   # reused by the apply / pool tests
        _CACHE[name] = res
    return res


def check_conv16_stats(dev, case):
    """S1 and S2 per channel against float64 sums of the returned z, mean and var within their
    bars and within what channel_bound assumes, two runs bit-identical.

    A value passes through at most d = 13 + T fp32 roundings before its CTA's partial becomes a
    double: 4 (5 with the square) in the 16-row shuffle tree, one per tile the CTA ran for its N
    tile (T, from the tile schedule, `_stats_depth`), 8 in the warp-order flush.  So per channel
    |dS1| <= d u sum|z| and |dS2| <= d u sum z^2.  A warp slice lost from one flush moves a sum by
    ~1 / (8 x CTAs per N tile), at least 100x that.  The variance var = S2/M - mean^2 is then off
    by (eps2 + 2 eps1)(1 + r^2) relative, r = |mean| / std, eps the two relative errors.  Those
    errors are a random walk of roundings, ~u sqrt(T / 3) per CTA, averaged over the CTAs: 1e-8 ..
    3e-8.  VAR_BAR = 1e-7 (1 + r^2) keeps a 3x margin: 1e-5 at r = 10, 1e-3 at r = 100.  The same
    sums bound the error the act scale assumes (split16.cu channel_bound, kappa = 16 + ceil(M /
    (16 * 132))), which is checked too."""
    z, st, st2, conv = _produce(dev, case)
    M, C = z.shape
    assert torch.equal(st, st2), "statistics not run-to-run identical"
    zd = z.double()
    t1, t2, a1 = zd.sum(0), (zd * zd).sum(0), zd.abs().sum(0)
    mu64, var64 = t1 / M, (zd - t1 / M).pow(2).sum(0) / M
    del zd
    s1, s2 = st[:C], st[C:]
    e1, e2 = (s1 - t1).abs() / a1, (s2 - t2).abs() / t2
    # deconv: four phase launches, each with its own (shorter) tile runs; the dense M is the worst
    d = _stats_depth(M)
    bar = d * U
    mk = s1 / M
    vk = (s2 / M - mk * mk).clamp_min(0)
    r = mu64.abs() / var64.sqrt()
    ev = (vk - var64).abs() / var64
    vbar = VAR_COEF * (1 + r * r)
    ku, q = _kappa(M) * U, t2 / M
    for lo, hi in ((0, 0.5), (0.5, 3), (3, 30), (30, 1e9)):
        sel = (r >= lo) & (r < hi)
        if sel.any():
            print("  %-18s r in [%g, %g): eps1 %.2e eps2 %.2e var %.2e (var bar %.2e) bar %.2e"
                  % (case[0], lo, hi, float(e1[sel].max()), float(e2[sel].max()), float(ev[sel].max()),
                     float(vbar[sel].max()), bar))
    assert float(e1.max()) <= bar and float(e2.max()) <= bar, "sum %.3e / squares %.3e (bar %.2e)" % (
        float(e1.max()), float(e2.max()), bar)
    assert bool((ev <= vbar).all()), "var %.3e at r %.1f" % (float((ev / vbar).max()), float(r[(ev / vbar).argmax()]))
    assert bool(((mk - mu64).abs() <= ku * q.sqrt()).all())                     # channel_bound's dmean
    assert bool((var64 - vk <= 4 * ku * q).all())                               # and its var deficit


def _finalize_dev(dev, st, M, C, gamma, beta, rm, rv, group2=(None, None, None), res_sc=None):
    from epipolarpose_b200 import ops
    out = {k: torch.empty(C, device=dev) for k in ("scale", "shift", "mean", "invstd")}
    sc = torch.empty(4, device=dev)
    ops.bn_finalize_scale(st, M, C, gamma, beta, EPS, MOM, rm, rv, out["scale"], out["shift"],
                          out["mean"], out["invstd"], *group2, res_sc, sc)
    out["sc"] = sc
    return out


def check_bn_finalize_scale(dev, M):
    """Every output within 1 fp32 ulp of float64 arithmetic on the same statistics and fp32
    parameters (finalize is float64 arithmetic rounded once to fp32): gamma < 0 and = 0 channels,
    running statistics (unbiased, momentum), a second group and res_sc; the published scale is the
    rule's power of two of the float64 bound."""
    C = 256
    rng = np.random.default_rng(M)
    mean = rng.standard_normal(C) * 3
    var = rng.uniform(0.01, 4, C) if M > 1 else np.zeros(C)
    var[:4] = 0 if M > 1 else var[:4]                        # constant channels
    s1, s2 = mean * M, (var + mean * mean) * M
    g = rng.uniform(0.5, 1.5, C).astype(np.float32)
    g[4:12] *= -1
    g[12:16] = 0
    b = (rng.standard_normal(C) * 0.3).astype(np.float32)
    rm0, rv0 = rng.standard_normal(C).astype(np.float32), rng.uniform(0.5, 2, C).astype(np.float32)
    st2 = torch.tensor(np.concatenate([mean[::-1] * M, (var[::-1] + mean[::-1] ** 2) * M]), device=dev)
    sc2 = torch.tensor(rng.uniform(0.5, 1.5, C).astype(np.float32), device=dev)
    sh2 = torch.tensor((rng.standard_normal(C) * 0.1).astype(np.float32), device=dev)
    res_sc = torch.tensor([4.0, 0.25, 37.5, 0.0], device=dev)
    T = lambda a: torch.tensor(a, device=dev)
    st = torch.tensor(np.concatenate([s1, s2]), device=dev)
    for second in (False, True):
        rm, rv = T(rm0.copy()), T(rv0.copy())
        out = _finalize_dev(dev, st, M, C, T(g), T(b), rm, rv, (st2, sc2, sh2) if second else (None,) * 3,
                            res_sc if second else None)
        torch.cuda.synchronize()
        ref = _finalize64(st[:C].cpu().numpy(), st[C:].cpu().numpy(), M, g, b, rm0, rv0)
        got = dict(mean=out["mean"], invstd=out["invstd"], scale=out["scale"], shift=out["shift"], rm=rm, rv=rv)
        for k in got:
            u = _ulps(got[k].cpu().numpy(), ref[k])
            assert u.max() <= 1, "%s: %.2f ulp at channel %d" % (k, u.max(), u.argmax())
        scd, shd = out["scale"].double(), out["shift"].double()
        bound = float(_bound_def(st[:C], st[C:], scd, shd, M).max())
        if second:
            bound += float(_bound_def(st2[:C], st2[C:], sc2.double(), sh2.double(), M).max())
        bound = bound * 1.001 + (37.5 if second else 0.0)
        s = float(out["sc"][0])
        assert _scale_ok(s, bound, _act_rule) and abs(float(out["sc"][2]) - bound) <= 1e-6 * bound


def check_bn_finalize(dev, M, C=256):
    """epb_bn_finalize (the layers whose post-activation scale comes from elsewhere): every output
    within 1 fp32 ulp of float64 on the same statistics, gamma < 0 and = 0 channels, constant
    channels, running statistics (unbiased, momentum) over C channels."""
    from epipolarpose_b200 import ops
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
    print("  bn_finalize M %d C %d: worst %.2f ulp" % (M, C, worst))


def _apply_bar(zd, scd, shd, res_terms, ymax):
    """The folded affine y = fma(z, sc, sh) (+ q) with sc, sh rounded to fp32 is off by at most
    4u (|z sc| + |sh| + |residual terms|), and the planes hold y to 2^-22 max|y|; against float64
    BatchNorm the statistics' own (measured) error adds |g invstd dmean| + |g xhat| dvar /
    (2 (var + eps))."""
    return 4 * U * ((zd * scd).abs() + shd.abs() + res_terms) + 2.0 ** -22 * ymax


def _check_bn_act_split(dev, res, case):
    """the case's conv16 output -> bn_finalize_scale -> bn_act_split against float64 relu(gamma
    (z - mean64) / sqrt(var64 + eps) + beta (+ residual)); the ReLU bit mask against the float64
    sign (flips only within the bar); the scale contract"""
    from epipolarpose_b200 import ops
    z, st, _, _ = _produce(dev, case)
    M, C = z.shape
    g = torch.Generator(device=dev).manual_seed(23)
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    gamma[::7] *= -1
    beta = torch.randn(C, device=dev, generator=g) * 0.2
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    r = rs = r_sc = rscale = rshift = None
    group2, res_terms, res64 = (None,) * 3, 0.0, 0.0
    if res == "split":
        rs, rsc2, res64 = _split_dev(torch.relu(torch.randn(M, C, device=dev, generator=g)) * 2)
        r_sc = torch.tensor([float(rsc2[0]), float(rsc2[1]), float(res64.abs().max()), 0.0], device=dev)
        res_terms = res64.abs()
    elif res == "affine":
        r = torch.randn(M, C, device=dev, generator=g) * 1.5 + 0.3
        rscale = torch.rand(C, device=dev, generator=g) + 0.5
        rshift = torch.randn(C, device=dev, generator=g) * 0.1
        rst = _stats64(r)
        group2 = (rst, rscale, rshift)
        rd = r.double()
        res64 = rd * rscale.double() + rshift.double()
        res_terms = (rd * rscale.double()).abs() + rshift.double().abs() + res64.abs()
        del rd
    out = _finalize_dev(dev, st, M, C, gamma, beta, rm, rv, group2, r_sc)
    y = torch.empty(2, M, C, device=dev, dtype=torch.float16)
    bits = torch.empty(M * C // 8, device=dev, dtype=torch.uint8)
    ops.bn_act_split(z, out["scale"], out["shift"], r, rscale, rshift, rs, r_sc, 1, M, C, y, out["sc"], bits)
    torch.cuda.synchronize()
    zd = z.double()
    mu64 = zd.mean(0)
    var64 = (zd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    xh = (zd - mu64) * inv64
    pre = gamma.double() * xh + beta.double() + res64
    y64 = pre.clamp_min(0)
    # the statistics' own error, first order (check_conv16_stats bounds it)
    mk = st[:C] / M
    vk = (st[C:] / M - mk * mk).clamp_min(0)
    stat_term = (gamma.double() * inv64 * (mk - mu64)).abs() + \
        (gamma.double() * xh).abs() * (vk - var64).abs() / (2 * (var64 + EPS))
    ymax = float(y64.max())
    bar = _apply_bar(zd, out["scale"].double(), out["shift"].double(), res_terms, ymax) + stat_term
    del xh
    got = _join(y, out["sc"]).view(M, C)
    err = (got - y64).abs()
    print("  apply %-6s max err %.3e, worst err / bar %.3f" % (res, float(err.max()), float((err / bar).max())))
    assert bool((err <= bar).all()), "apply error %.3e over its bar" % float((err - bar).max())
    flips = torch.from_numpy(np.unpackbits(bits.cpu().numpy(), bitorder="little").astype(bool)).to(dev) \
        ^ (pre > 0).view(-1)
    if bool(flips.any()):
        assert bool((pre.view(-1)[flips].abs() <= bar.view(-1)[flips]).all()), "ReLU mask flip outside the bar"
    scd, shd = out["scale"].double(), out["shift"].double()
    zs = _stats64(z)
    bound = float(_bound_def(zs[:C], zs[C:], scd, shd, M).max())
    if res == "affine":
        bound += float(_bound_def(rst[:C], rst[C:], rscale.double(), rshift.double(), M).max())
    bound = bound * 1.001 + (float(r_sc[2]) if r_sc is not None else 0.0)
    _contract_act("apply %s" % res, y, out["sc"], bound, ymax)


def _check_bn_relu_maxpool_split(dev, case):
    """the pool over the stem_col case's conv16 output (N images of hw x hw) -> bn_finalize_scale
    -> bn_relu_maxpool_split against float64 BatchNorm + ReLU + 3x3/2 max pool; argidx may pick
    another window entry only if its value is within the bar of the maximum (ties)"""
    from epipolarpose_b200 import ops
    z, st, _, _ = _produce(dev, case)
    M, C = z.shape
    N, H = case[7], case[8]
    W = H
    Ho, Wo = H // 2, W // 2
    g = torch.Generator(device=dev).manual_seed(29)
    gamma, beta = torch.rand(C, device=dev, generator=g) + 0.5, torch.randn(C, device=dev, generator=g) * 0.2
    out = _finalize_dev(dev, st, M, C, gamma, beta, torch.zeros(C, device=dev), torch.ones(C, device=dev))
    y = torch.empty(2, N, Ho, Wo, C, device=dev, dtype=torch.float16)
    arg = torch.empty(N, Ho, Wo, C, device=dev, dtype=torch.uint8)
    ops.bn_relu_maxpool_split(z, out["scale"], out["shift"], y, out["sc"], arg, N, H, W, C)
    torch.cuda.synchronize()
    zd = z.double()
    mu64 = zd.mean(0)
    var64 = (zd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    mk = st[:C] / M
    vk = (st[C:] / M - mk * mk).clamp_min(0)
    xh = (zd - mu64) * inv64
    a64 = (gamma.double() * xh + beta.double()).clamp_min(0)
    e = 4 * U * ((zd * out["scale"].double()).abs() + out["shift"].double().abs()) + \
        (gamma.double() * inv64 * (mk - mu64)).abs() + (gamma.double() * xh).abs() * (vk - var64).abs() / (2 * (var64 + EPS))
    del zd, xh
    pa = torch.full((N, H + 2, W + 2, C), float("-inf"), device=dev, dtype=torch.float64)
    pa[:, 1:-1, 1:-1] = a64.view(N, H, W, C)
    pe = torch.zeros((N, H + 2, W + 2, C), device=dev, dtype=torch.float64)
    pe[:, 1:-1, 1:-1] = e.view(N, H, W, C)
    del a64, e
    cand = torch.stack([pa[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)])
    ce = torch.stack([pe[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(3) for kw in range(3)])
    del pa, pe
    ref = cand.max(0).values
    ymax = float(ref.max())
    bar = ce.max(0).values + 2.0 ** -22 * ymax
    got = _join(y, out["sc"])
    err = (got - ref).abs()
    print("  maxpool max err %.3e, worst err / bar %.3f" % (float(err.max()), float((err / bar).max())))
    assert bool((err <= bar).all())
    picked = cand.gather(0, arg.long().unsqueeze(0)).squeeze(0)
    assert bool((picked >= ref - 2 * bar).all()), "argidx picks an entry below the window maximum"
    zs = _stats64(z)
    bound = float(_bound_def(zs[:C], zs[C:], out["scale"].double(), out["shift"].double(), M).max()) * 1.001
    _contract_act("stem maxpool", y, out["sc"], bound, ymax)


def check_bn_bwd_split(dev, M, C, mode):
    """bn_bwd_split against float64 autograd of the forward BatchNorm: dgamma, dbeta per channel
    and the joined dz elementwise, with a constant channel (invstd = 316), one huge gradient
    element and a fully masked channel beside ordinary ones; two runs bit-identical; the scale of
    dz from its bound.

    Each bn_bwd_partial thread sums R rows in fp32 (R from bn_bwd_workers, `_bwd_rows`), then the
    rpi row slots of its CTA: depth d = R + rpi + 2, so |d dbeta| <= d u sum|g| and |d dgamma| <=
    (d + 1) u sum|g xhat| + sum|g| e_xhat, e_xhat = 4u (|xhat| + |mean| invstd) the fp32 xhat from
    the fp32 mean / invstd.  Not from max|dgamma|: dgamma cancels."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(M + C)
    mu_c = torch.randn(C, device=dev, generator=g) * 2
    x = torch.randn(M, C, device=dev, generator=g) * (torch.rand(C, device=dev, generator=g) * 2 + 0.2) + mu_c
    x[:, 0] = 0.37                                           # var 0: invstd = 1 / sqrt(eps)
    dy = torch.randn(M, C, device=dev, generator=g) * 1e-4
    dy[M // 2, 1] = 3.0                                      # one huge element
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    beta = torch.randn(C, device=dev, generator=g) * 0.1
    xd = x.double()
    mu64 = xd.mean(0)
    var64 = (xd - mu64).pow(2).mean(0)
    inv64 = 1 / torch.sqrt(var64 + float(np.float32(EPS)))
    mean, invstd = mu64.float(), inv64.float()
    scale, shift = (gamma.double() * inv64).float(), (beta.double() - mu64 * gamma.double() * inv64).float()
    mask = bits = None
    if mode == "relu":
        scale[2], shift[2] = 0.0, -1.0                         # fully masked channel
    elif mode == "mask":
        mask = torch.relu(torch.randn(M, C, device=dev, generator=g)).half()
        mask[:, 2] = 0
    else:
        keep = torch.rand(M, C, device=dev, generator=g) > 0.4
        keep[:, 2] = False
        bits = torch.from_numpy(np.packbits(keep.cpu().numpy().reshape(-1), bitorder="little")).to(dev)
    runs = []
    for _ in range(2):
        dyk = dy.clone()
        dm = dyk if mode == "bits_inplace" else torch.empty_like(dy)
        dz = torch.empty(2, M, C, device=dev, dtype=torch.float16)
        sc = torch.empty(2, device=dev)
        dg, db = torch.empty(C, device=dev), torch.empty(C, device=dev)
        ops.bn_bwd_split(dyk, x, mask, scale, shift, mean, invstd, gamma, int(mode == "relu"), M, C, dz, sc, dm,
                         dg, db, mask_bits=bits)
        torch.cuda.synchronize()
        runs.append((dz, sc, dg, db, dm))
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.float16 else a,
                           b.view(torch.int16) if b.dtype == torch.float16 else b), "not run-to-run identical"
    dz, sc, dg, db, dm = runs[0]
    del runs
    # the gradient the kernel masked: its own mask in relu mode (a fp32 fma at the threshold),
    # which must agree with the float64 sign except within one rounding of zero
    if mode == "relu":
        pre = xd * scale.double() + shift.double()
        keep64 = pre > 0
        flip = (dm != 0) != keep64
        flip &= dy != 0
        if bool(flip.any()):
            assert bool((pre[flip].abs() <= 2 * U * ((xd * scale.double()).abs() + shift.double().abs())[flip]).all())
        g64 = dm.double()
        del pre, keep64, flip
    elif mode == "mask":
        g64 = dy.double() * (mask != 0)
    else:
        g64 = dy.double() * keep
        assert torch.equal(dm, g64.float())
    z64 = xd.clone().requires_grad_(True)
    m = z64.mean(0)
    v = (z64 - m).pow(2).mean(0)
    yref = gamma.double() * (z64 - m) / torch.sqrt(v + float(np.float32(EPS))) + beta.double()
    yref.backward(g64)
    dz64 = z64.grad
    del z64, m, v, yref
    xh = (xd - mu64) * inv64
    dgam64, dbet64 = (g64 * xh).sum(0), g64.sum(0)
    R, rpi = _bwd_rows(M, C)
    d = R + rpi + 2
    ag = g64.abs()
    e_xh = 4 * U * (xh.abs() + mu64.abs() * inv64)
    bar_b = d * U * ag.sum(0)
    bar_g = (d + 1) * U * (ag * xh.abs()).sum(0) + (ag * e_xh).sum(0)
    eb = (db.double() - dbet64).abs() - U * dbet64.abs()
    eg = (dg.double() - dgam64).abs() - U * dgam64.abs()
    print("  bwd %dx%d %-12s R %d dbeta %.2e (bar %.2e) dgamma %.2e (bar %.2e)" % (
        M, C, mode, R, float((eb + U * dbet64.abs()).max()), float(bar_b.max()),
        float((eg + U * dgam64.abs()).max()), float(bar_g.max())))
    assert bool((eb <= bar_b).all()), "dbeta"
    assert bool((eg <= bar_g).all()), "dgamma"
    k1, k2 = dbet64 / M, dgam64 / M
    a = (gamma.double() * inv64).abs()
    dzmax = float(dz64.abs().max())
    bar = a * (4 * U * (ag + k1.abs() + (xh * k2).abs()) + bar_b / M + xh.abs() * (bar_g / M) + k2.abs() * e_xh) \
        + 2 * U * dz64.abs() + 2.0 ** -22 * dzmax
    err = (_join(dz, sc).view(M, C) - dz64).abs()
    print("  bwd %dx%d %-12s dz max err %.3e, worst err / bar %.3f" % (M, C, mode, float(err.max()),
                                                                     float((err / bar).max())))
    assert bool((err <= bar).all()), "dz"
    # the scale of dz: pow2_scale of max_c |gamma invstd| (max|g| + |k1| + max|xhat| |k2|)
    bound = float((a * (ag.max(0).values + k1.abs() + xh.abs().max(0).values * k2.abs())).max())
    s = float(sc[0])
    assert _scale_ok(s, bound, _grad_rule) and float(sc[1]) == 1 / s
    assert _no_clamp(dz) and s * dzmax < HALF_MAX


# ------------------------------------------------------------------ the fp32 BatchNorm chain (bn.cu)
ROWS_PER_THREAD = 64                             # bn.cu kRowsPerThread


def _bn_stats64(x):
    """float64 batch mean and invstd of x [M, C] (the fp32 eps, as bn_finalize adds it)"""
    xd = x.double()
    mu = xd.mean(0)
    var = (xd - mu).pow(2).mean(0)
    return mu, 1 / torch.sqrt(var + float(np.float32(EPS)))


def _bn_bwd_ref_bar(x, dy, keep, gamma, mu, inv):
    """float64 BatchNorm backward of g = dy * keep on x [M, C] with batch statistics (mu, inv),
    and the bars of bn_bwd_reduce + bn_bwd_apply: (dbeta, dgamma, dx, bar_b, bar_g, bar_dx).

    Each thread adds kRowsPerThread = 64 rows in fp32, the CTA's row slots and all CTAs add in
    double, so with d = 64 + 2, |d dbeta| <= d u sum|g| and |d dgamma| <= (d + 1) u sum|g xhat| +
    sum|g| e_xhat, where e_xhat = 4u (|xhat| + |mean| invstd) is the error of the fp32 xhat formed
    from the fp32 mean and invstd.  dgamma and dbeta then round once to fp32 (_bn_bwd_ratios).
    Not from max|dgamma|: dgamma cancels.  k0 = gamma invstd, k1 = sum g / M, k2 = sum g xhat / M
    round to fp32, and dx = k0 (g - k1 - xhat k2) takes four more roundings: |d dx| <= |gamma
    invstd| (4u (|g| + |k1| + |xhat k2|) + bar_b / M + |xhat| bar_g / M + |k2| e_xhat) + 2u |dx|."""
    M = x.shape[0]
    g = dy.double() * keep
    xh = (x.double() - mu) * inv
    sg, sgx = g.sum(0), (g * xh).sum(0)
    d = ROWS_PER_THREAD + 2
    ag = g.abs()
    e_xh = 4 * U * (xh.abs() + mu.abs() * inv)
    bar_b = d * U * ag.sum(0)
    bar_g = (d + 1) * U * (ag * xh.abs()).sum(0) + (ag * e_xh).sum(0)
    k1, k2 = sg / M, sgx / M
    a = gamma.double() * inv
    dx = a * (g - k1 - xh * k2)
    bar = a.abs() * (4 * U * (ag + k1.abs() + (xh * k2).abs()) + bar_b / M + xh.abs() * (bar_g / M)
                     + k2.abs() * e_xh) + 2 * U * dx.abs()
    return sg, sgx, dx, bar_b, bar_g, bar


def _bn_bwd_ratios(dbeta, dgamma, dx, ref):
    """worst err / bar of dbeta, dgamma (each after its one fp32 rounding) and dx"""
    sg, sgx, dx64, bar_b, bar_g, bar = ref
    eb = ((dbeta.double() - sg).abs() - U * sg.abs()).clamp_min(0) / (bar_b + 1e-300)   # a fully masked
    eg = ((dgamma.double() - sgx).abs() - U * sgx.abs()).clamp_min(0) / (bar_g + 1e-300)  # channel: 0 / 0
    ex = (dx.double() - dx64).abs() / (bar + 1e-300)
    return float(eb.max()), float(eg.max()), float(ex.max())


def check_bn_bwd(dev, M, C, mode):
    """bn_bwd_reduce + bn_bwd_apply over M x C against float64 within _bn_bwd_ref_bar: dbeta,
    dgamma per channel and dx per element, with a constant channel (invstd = 316), one huge
    gradient element and a fully masked channel beside ordinary ones.  mode "y_out": g is dy
    masked by y_out > 0; "relu": by the BatchNorm's own ReLU, fma(z, scale, shift) > 0, whose sign
    the float64 z scale + shift gives exactly, so the reference masks alike."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(M + C)
    x = torch.randn(M, C, device=dev, generator=g) * (torch.rand(C, device=dev, generator=g) * 2 + 0.2) \
        + torch.randn(C, device=dev, generator=g) * 2
    x[:, 0] = 0.37                                           # var 0: invstd = 1 / sqrt(eps)
    dy = (torch.randn(M, C, device=dev, generator=g) + torch.randn(C, device=dev, generator=g) * 0.5) * 1e-4
    dy[M // 2, 1] = 3.0                                      # one huge element
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    beta = torch.randn(C, device=dev, generator=g) * 0.1
    mu, inv = _bn_stats64(x)
    mean, invstd = mu.float(), inv.float()
    scale, shift = (gamma.double() * inv).float(), (beta.double() - mu * gamma.double() * inv).float()
    y_out = None
    if mode == "relu":
        scale[2], shift[2] = 0.0, -1.0                       # a fully masked channel
        keep = (x.double() * scale.double() + shift.double()) > 0
    else:
        y_out = torch.relu(torch.randn(M, C, device=dev, generator=g))
        y_out[:, 2] = 0
        keep = y_out > 0
    relu = int(mode == "relu")
    sums = torch.zeros(2 * C, device=dev, dtype=torch.float64)
    dx, dg, db = torch.empty(M, C, device=dev), torch.empty(C, device=dev), torch.empty(C, device=dev)
    ops.bn_bwd_reduce(dy, x, y_out, scale, shift, mean, invstd, relu, M, C, sums)
    ops.bn_bwd_apply(dy, x, y_out, scale, shift, mean, invstd, gamma, relu, sums, M, C, dx, dg, db)
    torch.cuda.synchronize()
    del y_out
    ref = _bn_bwd_ref_bar(x, dy, keep, gamma, mu, inv)
    rb, rg, rx = _bn_bwd_ratios(db, dg, dx, ref)
    print("  bn bwd %7d x %-4d %-5s worst err / bar: dbeta %.3f dgamma %.3f dx %.3f (max dx err %.2e)"
          % (M, C, mode, rb, rg, rx, float((dx.double() - ref[2]).abs().max())))
    assert rb <= 1.0 and rg <= 1.0 and rx <= 1.0


def _bn_act_ref_bar(x, s, b, r, rs, rb):
    """float64 x s + b (+ r rs + rb, or + r) and the bar 4u on its terms: bn_act computes y =
    relu(fma(x, s, b) + q), q = fma(r, rs, rb), r or 0, three roundings on the terms"""
    xd = x.double()
    t = xd * s.double() + b.double()
    terms = (xd * s.double()).abs() + b.double().abs()
    if r is not None:
        rd = r.double()
        if rs is not None:
            t = t + rd * rs.double() + rb.double()
            terms = terms + (rd * rs.double()).abs() + rb.double().abs()
        else:
            t = t + rd
            terms = terms + rd.abs()
    return t, 4 * U * terms


def _bn_act_check(y, t, bar):
    """(worst |y - relu(t)| / bar, elements below -bar that are not exactly 0, negative y)"""
    err = (y.double() - t.clamp_min(0)).abs()
    dead = t < -bar
    return (float((err / (bar + 1e-300)).max()), int((dead & (y != 0)).sum()), int((y < 0).sum()))


def check_bn_act(dev, M, C, res):
    """bn_act with ReLU over M x C: the residual with the downsample BatchNorm's affine ("affine"),
    the identity residual ("identity") or ReLU alone ("relu"); within _bn_act_ref_bar's 4u of the
    terms, exactly 0 where the float64 value is below minus that bar, a guard band untouched."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(M + C + len(res))
    x = torch.randn(M, C, device=dev, generator=g) * 3 + 0.5
    s, b = torch.rand(C, device=dev, generator=g) + 0.2, torch.randn(C, device=dev, generator=g) * 0.5
    r = rs = rb = None
    if res != "relu":
        r = torch.randn(M, C, device=dev, generator=g) * 2
        if res == "identity":
            r = torch.relu(r)                                     # a block output
        else:
            rs, rb = torch.rand(C, device=dev, generator=g) + 0.2, torch.randn(C, device=dev, generator=g) * 0.5
    y, guard = _guarded((M, C), dev, float("nan"))
    guard.fill_(1234.5)
    ops.bn_act(x, s, b, r, rs, rb, 1, y, M, C)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    worst, bad0, neg = 0.0, 0, 0
    step = max((1 << 24) // C, 1)
    for r0 in range(0, M, step):
        sl = slice(r0, r0 + step)
        t, bar = _bn_act_ref_bar(x[sl], s, b, None if r is None else r[sl], rs, rb)
        w_, z_, n_ = _bn_act_check(y[sl], t, bar)
        worst, bad0, neg = max(worst, w_), bad0 + z_, neg + n_
        del t, bar
    print("  bn_act %6d x %-4d %-8s worst err / bar %.3f" % (M, C, res, worst))
    assert worst <= 1.0 and bad0 == 0 and neg == 0, (worst, bad0, neg)


# ------------------------------------------------------------------ conv16 at a layer shape
def _check_conv16_layer(dev, layer, N, wgrad_bar):
    """conv16 fprop (with statistics), dgrad and wgrad of one layer over N images against torch
    float64 on the values the planes hold; returns the three errors"""
    import torch.nn.functional as F
    from epipolarpose_b200 import net, ops
    name, kind, cin, cout, k, s, p, hw = layer
    conv = net.Conv("t", kind, cin, cout, k, s, p, 0)
    Ho, Wo = conv.out_hw(hw, hw)
    T = k * k
    g = torch.Generator(device=dev).manual_seed(7)
    x, x_sc, xv = _split_dev(torch.relu(torch.randn(N, hw, hw, cin, device=dev, generator=g)))
    dz, dz_sc, dzv = _split_dev(torch.randn(N, Ho, Wo, cout, device=dev, generator=g) * 3e-5)
    w = torch.randn((cout, cin, k, k) if kind == "conv" else (cin, cout, k, k), device=dev,
                    generator=g) * (2.0 / (T * cin)) ** 0.5
    wf32, wd32 = conv.pack(ops, w)
    wf, wf_sc, wfv = _split_dev(wf32)
    wd, wd_sc, _ = _split_dev(wd32)
    # the weights the planes hold, back in the state_dict layout (for the float64 reference)
    pk = wfv.view(cout, T, cin)
    wq64 = pk.permute(0, 2, 1).reshape(cout, cin, k, k) if kind == "conv" else \
        pk.permute(2, 0, 1).reshape(cin, cout, k, k)
    xa = xv.permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wt = wq64.contiguous().requires_grad_(True)
    ref = F.conv2d(xa, wt, None, s, p) if kind == "conv" else F.conv_transpose2d(xa, wt, None, s, p)
    ref.backward(dzv.permute(0, 3, 1, 2).contiguous())
    # fprop
    out = torch.zeros(N, Ho, Wo, cout, device=dev)
    stats = torch.zeros(2 * cout, device=dev, dtype=torch.float64)
    for gm in conv.fprop_geoms(ops, N, hw, hw, 3):
        if gm is not None:
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv16_fprop(gm, x, x_sc, wf, wf_sc, out, None, stats)
    r = ref.detach().permute(0, 2, 3, 1)
    e_f = e = float((out.double() - r).abs().max() / r.abs().max())
    assert e <= 5e-5, "fprop %.3e" % e
    # per-channel sums: fp32 partial sums over up to 3584 rows per CTA, then float64 atomics
    assert float((stats[:cout] - r.sum((0, 1, 2))).abs().max() / r.abs().sum((0, 1, 2)).max()) <= 5e-5
    # dgrad: only the dz * w_dgrad-operand product differs from the reference by the weight planes
    din = torch.zeros(N, hw, hw, cin, device=dev)
    for gm in conv.dgrad_geoms(ops, N, hw, hw, 3):
        if gm is not None:
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv16_fprop(gm, dz, dz_sc, wd, wd_sc, din, None, None)
    r = xa.grad.permute(0, 2, 3, 1)
    e_d = e = float((din.double() - r).abs().max() / r.abs().max())
    assert e <= 5e-5, "dgrad %.3e" % e
    # wgrad (packed [cout][T][cin])
    dw = torch.zeros(cout * T * cin, device=dev)
    ws = torch.empty(48 << 20, device=dev)
    for gm in conv.fprop_geoms(ops, N, hw, hw, 3):
        if gm is not None:
            gm.in_relu, gm.accumulate = 0, 0
            ops.conv16_wgrad(gm, x, x_sc, dz, dz_sc, dw, ws)
    gw = wt.grad
    r = (gw.permute(0, 2, 3, 1) if kind == "conv" else gw.permute(1, 2, 3, 0)).reshape(cout, T, cin)
    e = float((dw.view(cout, T, cin).double() - r).abs().max() / r.abs().max())
    assert e <= wgrad_bar, "wgrad %.3e (bar %.2e)" % (e, wgrad_bar)   # C4: fp32 runs over up to 524288 / 74 pixels
    return e_f, e_d, e


# ------------------------------------------------------------------ 3xTF32 conv at a layer shape
def _pad4(c):
    return (c + 3) // 4 * 4


def tf32_wgrad_runs(layer, N):
    """(pixels N Hp Wp, Cin, Cout, taps) of each wgrad geometry of a C4_LAYERS_TF32X3-style row: one
    for a convolution, one per output phase (2 x 2, 4 taps each) for the 4 x 4 / 2 deconvolutions"""
    _, kind, cin, cout, k, s, p, hw, _, _ = layer
    if kind == "conv":
        ho = (hw + 2 * p - k) // s + 1
        return [(N * ho * ho, cin, cout, k * k)]
    return [(N * hw * hw, cin, cout, 4)] * 4


def tf32_wgrad_run(layer, N):
    """the longest pixel run of one CTA over the layer's wgrad geometries"""
    return max(_tf32_wgrad_plan(M, ci, co, T, 3)[0] for M, ci, co, T in tf32_wgrad_runs(layer, N))


def tc_supported(gm, wgrad):
    """conv_tc.cu epb_conv_tc_supported / conv_tc_wgrad.cu epb_conv_wgrad_tc_supported: whether
    epb_conv_fprop / epb_conv_wgrad at precision 1 or 3 run the tensor-core kernels on geometry gm
    (else the fp32 CUDA-core kernels)"""
    fits = gm.N * gm.Hi * gm.Wi * gm.Cin < 1 << 31
    if wgrad:
        return gm.Cin % 32 == 0 and gm.Cout % 4 == 0 and gm.Cout >= 32 and fits and gm.N * gm.Ho * gm.Wo < 1 << 31
    return gm.Cin % 32 == 0 and gm.Cout % 32 == 0 and gm.Cout >= 32 and fits


def check_tf32x3_layer(dev, layer, N, kernels=_all_three_pass, bias_stats=False):
    """3xTF32 fprop (statistics into a zeroed buffer, or the bias for a layer named final* or
    depth_fc*), dgrad (written, or added into the block's input gradient for a downsample) and
    wgrad (into a zeroed dW) of a C4_LAYERS_TF32X3-style row over N images with its operand mode,
    each against torch float64 within its bar: fprop / dgrad _tc_bar(FPROP_BAR, K, 3), K the
    longest taps x Cin of the call's geometries; wgrad _tc_bar(WGRAD_BAR, R, 3), R the pixel run
    of one CTA from the restated planner.  Every output followed by a guard band; the conv
    kernels that ran (_ran's tags) must meet `kernels`: by default every one a three-pass
    instantiation.  kernels=None opens no profiler session: the caller shows which kernels run.

    bias_stats: the bias (zero in the padding columns) and the statistics in the same fprop call,
    as MLPEngine.linear makes it.  The kernels add the bias before they accumulate the sums, so
    the sums must meet STATS_SELF_BAR against the kernel's own output and the fprop bar against
    float64 x W^T + b; the same sums with the bias left out of the reference must miss that bar
    by more than 100x (the check has teeth at these seeds); padding output columns are exactly 0."""
    import torch.nn.functional as F
    from epipolarpose_b200 import ops
    name, kind, cin, cout, k, s, p, hw, operand, dmode = layer
    final = name.startswith(("final", "depth_fc")) and not bias_stats
    conv, Ho, Wo, x, sc, sh, w, gout = _layer(dev, kind, cin, cout, k, s, p, 0, N, hw, hw, 17)
    ci, co, T = conv.cin_p, conv.cout_p, k * k
    act = operand == "act"
    aff = (sc, sh) if act else (None, None)
    wf, wd = conv.pack(ops, w)
    tags, errs = set(), {}
    # ---- fprop
    bias = torch.randn(co, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) * 0.5 \
        if final or bias_stats else None
    if bias_stats:
        bias[cout:] = 0
    geoms = conv.fprop_geoms(ops, N, hw, hw, 3)
    gms = _geoms(geoms, int(act), 0)
    out, guard = _guarded((N, Ho, Wo, co), dev, 0.0 if any(gm is None for gm in geoms) else float("nan"))
    guard.fill_(1234.5)
    stats = sguard = None
    if not final:
        sbuf = torch.zeros(2 * co + 64, device=dev, dtype=torch.float64)
        stats, sguard = sbuf[:2 * co], sbuf[2 * co:]

    def fwd(o, st):
        for gm in gms:
            ops.conv_fprop(gm, x, wf, o, aff[0], aff[1], bias, st)
    if kernels is not None:
        tags |= _ran(lambda: fwd(out.clone(), None if stats is None else stats.clone()))
    fwd(out, stats)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "fprop guard band overwritten"
    a64 = _act64(x, *aff, act)
    with torch.no_grad():
        ref = _fwd64(conv, a64, w.double())
        if bias is not None:
            ref += bias.double()[None, :, None, None]
        ref = ref.permute(0, 2, 3, 1)
        bar_f = _tc_bar(FPROP_BAR, max(gm.T * gm.Cin for gm in gms), 3)
        errs["fprop"] = float((out.double() - ref).abs().max() / ref.abs().max())   # NaN fails
        if stats is not None:
            assert bool((sguard == 0).all()), "statistics guard band overwritten"
            o = out.double().reshape(-1, co)
            s1, s2 = stats[:co], stats[co:]
            errs["st_self"] = max(float(((s1 - o.sum(0)).abs() / o.abs().sum(0).clamp_min(1e-300)).max()),
                                  float(((s2 - (o * o).sum(0)).abs() / (o * o).sum(0).clamp_min(1e-300)).max()))
            del o
            r = ref.reshape(-1, co)
            r2 = (r * r).sum(0)
            errs["st_ref"] = max(float(((s1 - r.sum(0)).abs() / r.abs().sum(0).clamp_min(1e-300)).max()),
                                 float((s2 - r2).abs().max() / r2.abs().max()))
            if bias is not None:
                r = r - bias.double()
                r2n = (r * r).sum(0)
                errs["st_nobias"] = max(float(((s1 - r.sum(0)).abs() / r.abs().sum(0).clamp_min(1e-300)).max()),
                                        float((s2 - r2n).abs().max() / r2n.abs().max()))
                del r2n
            del r, r2
        if bias_stats and cout != co:
            assert bool((out[..., cout:] == 0).all()), "padding output columns are not exactly zero"
            assert bool((stats[cout:co] == 0).all() and (stats[co + cout:] == 0).all()), "padding statistics"
    del out, ref
    # ---- dgrad
    bar_d = None
    if dmode is not None:
        dgeoms = conv.dgrad_geoms(ops, N, hw, hw, 3)
        acc = int(dmode == "acc")
        dgms = _geoms(dgeoms, 0, acc)
        with torch.no_grad():
            g64, w64 = gout.permute(0, 3, 1, 2).double(), w.double()
            if kind == "conv":
                ref = torch.nn.grad.conv2d_input((N, ci, hw, hw), w64, g64, s, p)
            else:
                ref = F.conv2d(g64, w64, None, s, p)
            del g64
            ref = ref.permute(0, 2, 3, 1)
        din, guard = _guarded((N, hw, hw, ci), dev, 0.0 if (acc or any(gm is None for gm in dgeoms)) else float("nan"))
        guard.fill_(1234.5)
        init = None
        if acc:
            init = torch.randn(din.shape, device=dev, generator=torch.Generator(device=dev).manual_seed(9))
            init *= float(ref.abs().max()) / 3
            din.copy_(init)

        def bwd(o):
            for gm in dgms:
                ops.conv_fprop(gm, gout, wd, o, None, None, None, None)
        if kernels is not None:
            tags |= _ran(lambda: bwd(din.clone()))
        bwd(din)
        torch.cuda.synchronize()
        assert bool((guard == 1234.5).all()), "dgrad guard band overwritten"
        base = init.double() if init is not None else 0.0
        errs["dgrad"] = float((din.double() - (base + ref)).abs().max() / ref.abs().max())
        bar_d = _tc_bar(FPROP_BAR, max(gm.T * gm.Cin for gm in dgms), 3)
        del din, ref, init
    # ---- wgrad
    runs = sorted((gm.N * gm.Hp * gm.Wp, gm.Cin, gm.Cout, gm.T) for gm in gms)
    assert runs == sorted((M, _pad4(a), _pad4(b), t) for M, a, b, t in tf32_wgrad_runs(layer, N)), runs
    R = tf32_wgrad_run(layer, N)
    bar_w = _tc_bar(WGRAD_BAR, R, 3)
    w64 = w.double().requires_grad_(True)
    _fwd64(conv, a64, w64).backward(gout.permute(0, 3, 1, 2).double())
    del a64
    gw = w64.grad
    ref = (gw.permute(0, 2, 3, 1) if kind == "conv" else gw.permute(1, 2, 3, 0)).reshape(co, T, ci)
    del w64, gw
    dw, guard = _guarded((co * T * ci,), dev, 0.0)
    guard.fill_(1234.5)

    def wgr(o):
        for gm in gms:
            ops.conv_wgrad(gm, x, gout, o, aff[0], aff[1])
    if kernels is not None:
        tags |= _ran(lambda: wgr(torch.zeros_like(dw)))
    wgr(dw)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "dW guard band overwritten"
    errs["wgrad"] = float((dw.view(co, T, ci).double() - ref).abs().max() / ref.abs().max())
    print("  %-22s %-36s fprop %.2e (bar %.2e)%s%s wgrad %.2e (run %d, bar %.2e)" % (
        name, ",".join(sorted(tags)), errs["fprop"], bar_f,
        " stats %.1e / %.1e" % (errs["st_self"], errs["st_ref"]) if "st_self" in errs else "",
        " dgrad %.2e (bar %.2e)" % (errs["dgrad"], bar_d) if bar_d else "", errs["wgrad"], R, bar_w))
    if bias_stats:
        print("  %-22s worst err / bar: fprop %.3f dgrad %.3f wgrad %.3f stats self %.3f ref %.3f; "
              "stats without the bias %.3g" % (name, errs["fprop"] / bar_f, errs.get("dgrad", 0.0) / (bar_d or 1.0),
                                               errs["wgrad"] / bar_w, errs["st_self"] / STATS_SELF_BAR,
                                               errs["st_ref"] / bar_f, errs["st_nobias"] / bar_f))
    assert kernels is None or kernels(tags), tags
    assert errs["fprop"] <= bar_f, errs
    if "st_self" in errs:
        assert errs["st_self"] <= STATS_SELF_BAR and errs["st_ref"] <= bar_f, errs
    if bias_stats:
        assert errs["st_nobias"] > 100 * bar_f, errs
    if bar_d is not None:
        assert errs["dgrad"] <= bar_d, errs
    assert errs["wgrad"] <= bar_w, errs


# ------------------------------------------------------------------ the VOLUME=False head: pooling, heat-map loss
HM_THREADS, HM_MAX_BLOCKS = 256, 8 * NUM_SMS     # softargmax.cu kHmThreads, kHmMaxBlocks


def _check_avgpool_split(dev, N, HW, C):
    """epb_avgpool_split of trunk planes [N, HW, C] (relu(randn) x 3: block outputs) with their
    scale, against float64 of the joined planes.  The kernel adds the HW (hi + lo) pairs of a
    channel in fp32 in pixel order (one rounding per pair, one per running sum), multiplies by the
    power-of-two scale (exact) and divides by HW (one rounding): |d y| <= (HW + 1) u sum_p |v_p| /
    HW + u |y|, v the joined values."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(101)
    x, x_sc, xv = _split_dev(torch.relu(torch.randn(N, HW, C, device=dev, generator=g)) * 3)
    y, guard = _guarded((N, C), dev, float("nan"))
    guard.fill_(1234.5)
    ops.avgpool_split(x, x_sc, y, N, HW, C)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    ref = xv.mean(1)
    bar = (HW + 1) * U * xv.abs().mean(1) + U * ref.abs()
    err = (y.double() - ref).abs()                              # NaN fails
    print("  avgpool_split [%d, %d, %d] scale 2^%d: max err %.3e, worst err / bar %.3f"
          % (N, HW, C, -int(math.log2(float(x_sc[1]))), float(err.max()), float((err / bar).max())))
    assert bool((err <= bar).all())


def _check_avgpool_bwd(dev, N, HW, C, accumulate):
    """epb_avgpool_bwd bit-exact against fp32 dx + dy / HW (accumulate) or dy / HW restated in
    numpy: the kernel's one IEEE division and one add, in that order (no product to contract, and
    the build does not use fast-math); every element written, a guard band untouched.  Then the
    fp32 engine's epb_avgpool forward over the same [N, HW, C] against float64: a sequential fp32
    sum of HW terms and one division, within HW u mean|x|."""
    from epipolarpose_b200 import ops
    g = torch.Generator(device=dev).manual_seed(103 + HW + C + accumulate)
    dy = torch.randn(N, C, device=dev, generator=g) * 1e-3
    dx0 = torch.randn(N, HW, C, device=dev, generator=g) * 1e-4
    dx, guard = _guarded((N, HW, C), dev, float("nan"))
    guard.fill_(1234.5)
    if accumulate:
        dx.copy_(dx0)
    ops.avgpool_bwd(dy, dx, N, HW, C, accumulate)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "guard band overwritten"
    q = dy.cpu().numpy() / np.float32(HW)
    ref = dx0.cpu().numpy() + q[:, None, :] if accumulate else np.broadcast_to(q[:, None, :], (N, HW, C))
    assert ref.dtype == np.float32
    got = dx.cpu().numpy()
    same = got.view(np.int32) == np.ascontiguousarray(ref).view(np.int32)
    # the fp32 forward
    x = torch.randn(N, HW, C, device=dev, generator=g)
    y, guard = _guarded((N, C), dev, float("nan"))
    guard.fill_(1234.5)
    ops.avgpool(x, y, N, HW, C)
    torch.cuda.synchronize()
    assert bool((guard == 1234.5).all()), "forward guard band overwritten"
    xd = x.double()
    err = (y.double() - xd.mean(1)).abs()
    bar = HW * U * xd.abs().mean(1)
    print("  avgpool_bwd [%d, %d, %d] accumulate %d: %d of %d elements differ; avgpool fwd worst err / bar %.3f"
          % (N, HW, C, accumulate, int((~same).sum()), same.size, float((err / bar).max())))
    assert bool(same.all())
    assert bool((err <= bar).all())


def hm_grid(R, HW):
    """epb_heatmap_joint_loss's launch: (CTAs, trips of the slowest thread): quads of 4 elements
    when HW % 4 == 0 (main loop of four quads per trip, then single quads), else single elements"""
    work = -(-(R * HW) // 4)
    blocks = min(-(-work // HM_THREADS), HM_MAX_BLOCKS)
    per = R * HW // 4 if HW % 4 == 0 else R * HW
    return blocks, -(-per // (blocks * HM_THREADS))


def hm_loss_ref_bar(hm, tg, wr, x, t, w, R, HW, div):
    """float64 heat-map MSE + L1 joint loss with hm_scale = jt_scale = 1, and the bars of the
    kernel's partition: (L_hm, L_jt, L_tot, dhm, dx, bars {hm, jt, tot, dhm, dx}).  hm / tg [R, HW],
    wr [R] (the weight multiplies the difference, so it enters the loss squared).

    Heat-map part: d = wr (h - g) rounds twice, d^2 once (5u relative per element).  With quads
    (HW % 4 == 0) the four squares of a quad add in a two-level tree, each thread adds its quads in
    fp32 over q trips (hm_grid): 7 + q roundings on every term; per element (HW % 4 != 0) the
    squares add in double.  The per-thread partials then add in double (depth < 64) and L_hm
    rounds to fp32: |d L_hm| <= ((7 + q) u + 64 2^-53) L_hm + u L_hm.  Joint part: |x - t| and
    the product with w round once each, the sum is in double (depth < 256): |d L_jt| <= (2u +
    256 2^-53) sum|l w| / div + u L_jt; the total adds them in fp32: + u |L_tot|.
    dhm = gs wr d with gs = 2 / (R HW) (1 / (R HW) rounds once; R HW < 2^24 is exact): the
    reciprocal, gs wr, d (two) and the product: 5 roundings, (5 + 1e-5) u |dhm|.  dx = sign(x - t)
    w / div: the sign of the fp32 difference is exact, so one rounding at most, u |dx|."""
    h, g, wr = hm.double(), tg.double(), wr.double().view(R, 1)
    d = wr * (h - g)
    total = R * HW
    L_hm = float((d * d).sum()) / total
    _, q = hm_grid(R, HW)
    depth = 7 + q if HW % 4 == 0 else 5
    dj = x.double() - t.double()
    lw = dj.abs() * w.double()
    L_jt = float(lw.sum()) / div
    L_tot = L_hm + L_jt
    bars = {"hm": (depth * U + 64 * 2.0 ** -53) * L_hm + U * L_hm,
            "jt": (2 * U + 256 * 2.0 ** -53) * L_jt + U * L_jt}
    bars["tot"] = bars["hm"] + bars["jt"] + U * L_tot
    dhm = 2.0 / total * wr * d
    dx = torch.sign(dj) * w.double() / div
    bars["dhm"] = (5 + 1e-5) * U * dhm.abs()
    bars["dx"] = U * dx.abs()
    return L_hm, L_jt, L_tot, dhm, dx, bars


def hm_case(dev, N, J, H, W, D, seed):
    """The C2(ii) objective's inputs on the device: heat-maps, Gaussian sigma = 2 targets and
    visibility weights from golden_inputs.heatmap_case, the weights of the visible joints scaled
    by dyadic factors in [1/4, 7/4] (so that a weight applied once instead of squared shows); the
    joint part an L1 term on a depth_fc-shaped output [N, J D] against U(-0.5, 0.5) targets,
    weights in {0, 1}."""
    from tests import golden_inputs as gi
    hm, tg, wh, _, _, _ = gi.heatmap_case(N, J, H, W, seed)
    rng = np.random.default_rng(seed + 1)
    wh = (wh * np.round(rng.uniform(0.25, 1.75, wh.shape) * 64) / 64).astype(np.float32)
    n = N * J * D
    x = (rng.standard_normal(n) * 0.5).astype(np.float32)
    t = (rng.random(n) - 0.5).astype(np.float32)
    w = (rng.random(n) > 0.1).astype(np.float32)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return T(hm), T(tg), T(wh.reshape(-1)), T(x), T(t), T(w)


def run_hm_loss(case, N, J, H, W):
    """one epb_heatmap_joint_loss launch (L1, hm_scale = jt_scale = 1, div = N): (loss [3], dhm, dx)"""
    from epipolarpose_b200 import ops
    hm, tg, wh, x, t, w = case
    R, HW = N * J, H * W
    loss = torch.empty(3, device=hm.device)
    dhm = torch.full_like(hm, float("nan"))
    dx = torch.full_like(x, float("nan"))
    ops.heatmap_joint_loss(hm, tg, wh, R, HW, 1.0, x, t, w, x.numel(), 1, float(N), 1.0, loss, dhm, dx)
    return loss, dhm, dx


# ------------------------------------------------------------------ inference: split-K conv16, calibrated models, decode
PATCH = 256.0
# key -> (layers, J, D, image size, init_state seed) of the predictor models: C1 (MPII), the H36M
# model of MultiViewPredictor and save_triangulations, C5
INFER_MODELS = {"c1": (50, 16, 64, 256, 71), "h36m": (50, 17, 64, 256, 72), "c5": (101, 17, 96, 384, 75)}


def _bench_conv(layer):
    """(conv, input size) of a C4_LAYERS_SPLIT16 row"""
    from epipolarpose_b200 import net
    name, kind, cin, cout, k, s, p, hw = layer
    return net.Conv("t", kind, cin, cout, k, s, p, 0), hw


def _splitk_layer(dev, conv, hw, N, seed=7, ref=True):
    """geoms, split operands, bias, the float64 reference [N, Ho, Wo, Cout] with bias (None without
    `ref`) and the joined float64 operands (x NCHW, w as conv2d / conv_transpose2d take it) of conv
    at batch N on hw x hw inputs.  Float64 reads the joined planes: the exact values the kernel reads."""
    import torch.nn.functional as F
    from epipolarpose_b200 import ops
    kind, cin, cout, k, s, p = conv.kind, conv.cin, conv.cout, conv.k, conv.stride, conv.pad
    T = k * k
    g = torch.Generator(device=dev).manual_seed(seed)
    x, x_sc, xv = _split_dev(torch.relu(torch.randn(N, hw, hw, cin, device=dev, generator=g)))
    w = torch.randn((cout, cin, k, k) if kind == "conv" else (cin, cout, k, k), device=dev,
                    generator=g) * (2.0 / (T * cin)) ** 0.5
    wf, wf_sc, wfv = _split_dev(conv.pack(ops, w)[0])
    bias = torch.randn(cout, device=dev, generator=g)
    pk = wfv.view(cout, T, cin)
    wq = pk.permute(0, 2, 1).reshape(cout, cin, k, k) if kind == "conv" else \
        pk.permute(2, 0, 1).reshape(cin, cout, k, k)
    xa = xv.permute(0, 3, 1, 2).contiguous()
    del xv
    out = None
    if ref:
        out = F.conv2d(xa, wq, None, s, p) if kind == "conv" else F.conv_transpose2d(xa, wq, None, s, p, conv.opad)
        out = out.permute(0, 2, 3, 1) + bias.double()
    geoms = [gm for gm in conv.fprop_geoms(ops, N, hw, hw, 3) if gm is not None]
    for gm in geoms:
        gm.in_relu, gm.accumulate = 0, 0
    return geoms, (x, x_sc, wf, wf_sc), bias, out, (xa, wq)


def _splitk_run(geoms, opnds, bias, out, stats, splits):
    """splits: an int (capped at each call's K/64) or None for the planner's count; the workspace
    holds exactly the planner's ws_floats at that count"""
    from epipolarpose_b200 import ops
    from tests import emul_splitk as es
    x, x_sc, w, w_sc = opnds
    for gm in geoms:
        s = ops.conv16_splits(gm)[0] if splits is None else min(splits, es.kblocks(gm))
        ws = torch.empty(max(1, s * es.phase_tiles(gm) * 128 * gm.Cout), device=out.device)
        ops.conv16_fprop_splitk(gm, x, x_sc, w, w_sc, out, bias, stats, s, ws)


def _split_partial64(conv, gm, xw, lo, hi):
    """float64 sum of k-blocks [lo, hi) of a gather conv (k-block = 64 channels of one tap, taps
    outer, as the split ranges of epb_conv16_fprop_splitk cut K): what one split contributes"""
    import torch.nn.functional as F
    xa, wq = xw
    CB = gm.Cin // 64
    mask = torch.zeros_like(wq)
    for kb in range(lo, hi):
        t, cb = divmod(kb, CB)
        r, c = divmod(gm.wt[t], conv.k)
        mask[:, cb * 64:(cb + 1) * 64, r, c] = 1
    return F.conv2d(xa, wq * mask, None, conv.stride, conv.pad).permute(0, 2, 3, 1)


def _coord_bound(dl):
    """largest move (patch px) of a soft-argmax coordinate whose logits each move by <= dl"""
    return PATCH * np.expm1(2.0 * np.asarray(dl, dtype=np.float64)) + 1e-3   # + float32 rounding


def infer_plan(key):
    from epipolarpose_b200.net import PoseNetPlan
    layers, J, D, HW, _ = INFER_MODELS[key]
    return PoseNetPlan(num_layers=layers, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))


def infer_layers(keys):
    """(conv, input size) of every distinct conv16 layer the inference forward of the models `keys`
    runs (emul_splitk.conv16_layers), in call order; the same shape counts once"""
    from tests import emul_splitk as es
    seen, out = set(), []
    for key in keys:
        HW = INFER_MODELS[key][3]
        for conv, h, w in es.conv16_layers(infer_plan(key), HW, HW):
            sig = (conv.kind, conv.cin, conv.cout, conv.k, conv.stride, conv.pad, h, w)
            if sig not in seen:
                seen.add(sig)
                out.append((conv, h))
    return out


def calibrated_state(dev, key, calib=4):
    """The model's init_state weights with calibrated running statistics, as a trained network has:
    one float64 training forward of oracle.restate_net over `calib` seeded images, each
    BatchNorm's running_mean / running_var set to that batch's mean and unbiased variance (momentum
    1, solved from the forward's momentum-0.1 update), then perturbed per channel so that eval and
    batch statistics differ: running_var x U(0.5, 2), running_mean + U(-0.5, 0.5) batch std.
    Cached under "infer_state_" + key."""
    ck = "infer_state_" + key
    if ck not in _CACHE:
        from oracle import restate_net as rn
        layers, J, D, HW, seed = INFER_MODELS[key]
        sd = rn.init_state(rn.param_shapes(num_layers=layers, num_joints=J, volume=True, depth_res=D), seed)
        sd64 = {k: v.to(dev, torch.float64) if v.is_floating_point() else v.to(dev) for k, v in sd.items()}
        x = torch.from_numpy(np.random.default_rng(seed + 1).standard_normal((calib, 3, HW, HW))).to(dev)
        ns = {}
        with torch.no_grad():
            rn.forward(sd64, x, num_layers=layers, image_size=(HW, HW), training=True, new_stats=ns)
        del sd64, x
        rng = np.random.default_rng(seed + 2)
        m = rn.BN_MOMENTUM
        for k in sorted(ns):
            if not k.endswith(".running_mean"):
                continue
            p = k[:-len("running_mean")]
            mean = ((ns[k].cpu() - (1 - m) * sd[k].double()) / m).numpy()
            var = ((ns[p + "running_var"].cpu() - (1 - m) * sd[p + "running_var"].double()) / m).numpy()
            C = mean.size
            sd[p + "running_var"] = torch.from_numpy((var * rng.uniform(0.5, 2.0, C)).astype(np.float32))
            sd[p + "running_mean"] = torch.from_numpy(
                (mean + rng.uniform(-0.5, 0.5, C) * np.sqrt(var)).astype(np.float32))
        _CACHE[ck] = sd
    return _CACHE[ck]


def calibrated_model(dev, key):
    """the f16x3 network of INFER_MODELS[key] on calibrated_state, in eval()"""
    import lib.models as models
    from tools.bench_cfg import make_cfg
    layers, J, D, HW, _ = INFER_MODELS[key]
    cfg = make_cfg(num_layers=layers, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
    model = models.pose3d_resnet.get_pose_net(cfg, False, precision="f16x3")
    model.load_state_dict(calibrated_state(dev, key))
    return model.to(dev).eval()


def _decode64(L, J, D, pairs=None, shift=False):
    """float64 soft-argmax of float64 logits L [B, J*D, H, W]: normalised coordinates [N, J, 3] as
    get_joint_location_coords; with pairs, of the flip-test merge of B = 2N images
    (flip_cases.flip_merge_softargmax)"""
    B, _, H, W = L.shape
    if pairs is not None:
        from lib.core.integral_loss import flip_permutation
        n = B // 2
        fb = L[n:].reshape(n, J, D * H, W).flip(-1)[:, flip_permutation(pairs, J)]
        if shift:
            fb = torch.cat([fb[..., :1], fb[..., :-1]], -1)
        L = 0.5 * (L[:n] + fb.reshape(n, J * D, H, W))
    N = L.shape[0]
    p = torch.softmax(L.reshape(N, J, -1), -1).reshape(N, J, D, H, W)
    ar = lambda k: torch.arange(k, device=L.device, dtype=torch.float64)
    return torch.stack([(p.sum((2, 3)) * ar(W)).sum(-1) / W, (p.sum((2, 4)) * ar(H)).sum(-1) / H,
                        (p.sum((3, 4)) * ar(D)).sum(-1) / D], -1) - 0.5


def _flip_merged32(L2, N, J, D, perm, shift):
    """the fp32 volume [N, H, W, J*D] that epb_softargmax_flip_fwd merges in registers from the
    channels-last logits L2 [2N, H, W, J*D] of [x; flip(x)]: 0.5 * (a + b) with b the mirrored pixel
    of image n + N in the paired joint's channels, read one column to the left under the shift
    (column 0 keeps its own); an fp32 add and an exact halving, as the kernel rounds"""
    _, H, W, C = L2.shape
    out = torch.empty(N, H, W, C, device=L2.device)
    for n0 in range(0, N, 8):
        n1 = min(N, n0 + 8)
        fb = L2[N + n0:N + n1].view(n1 - n0, H, W, J, D).flip(2)[:, :, :, perm]
        if shift:
            fb = torch.cat([fb[:, :, :1], fb[:, :, :-1]], 2)
        out[n0:n1] = (0.5 * (L2[n0:n1].view(n1 - n0, H, W, J, D) + fb)).reshape(n1 - n0, H, W, C)
    return out
