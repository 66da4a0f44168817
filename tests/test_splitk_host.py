"""CPU: the split-K conv16 entry's host rules through the C ABI (split planner epb_conv16_splits,
argument checks of epb_conv16_fprop_splitk) and its CPU emulation (tests/emul_splitk.py), which
sums the splits in the kernel's order."""
import ctypes

import pytest
import torch

from tests import emul_ops as em
from tests import emul_splitk as es

EPB_EINVAL = -1


def _plan():
    from epipolarpose_b200.net import PoseNetPlan
    return PoseNetPlan(num_layers=50, num_joints=16, volume=True, depth_res=64, image_size=(256, 256))


def _planned(g):
    from epipolarpose_b200 import ops
    return ops.conv16_splits(g)


def test_planner_never_splits_the_bench_step():
    """N = 128 (the bench's training batch): every layer already fills the GPU, down to the
    deconv0 phases at 128 tiles."""
    calls = es.conv16_calls(_plan(), 128)
    tiles = {}
    for name, g in calls:
        assert _planned(g) == (1, 0), name
        tiles[name] = es.phase_tiles(g) * es.n_tiles(g)
    assert min(tiles.values()) == 128 and tiles["deconv_layers.0"] == 128


@pytest.mark.parametrize("N", [1, 2, 4, 8, 32])
def test_planner_bounds_and_workspace(N):
    for name, g in es.conv16_calls(_plan(), N):
        s, ws = _planned(g)
        assert (s, ws) == es.splits(g), name
        assert 1 <= s <= es.kblocks(g), name
        tiles = es.phase_tiles(g) * es.n_tiles(g)
        if s > 1:
            assert s * tiles <= es.NUM_SMS and es.kblocks(g) // s >= es.SPLIT_MIN_KB, name
            assert ws == s * es.phase_tiles(g) * 128 * g.Cout, name
        else:
            assert ws == 0


def test_planner_splits_the_small_batch_layers():
    """N = 1: the layers the issue's table lists as filling 2-8 SMs are split."""
    got = {name: _planned(g)[0] for name, g in es.conv16_calls(_plan(), 1)}
    assert got["layer3.0.conv2"] > 1 and got["layer4.0.conv2"] > 1 and got["deconv_layers.0"] > 1
    assert got["final_layer"] == 1                      # 256 tiles


def _geom():
    from epipolarpose_b200.net import Conv
    return Conv("x", "conv", 128, 64, 3, 1, 1).fprop_geoms(em, 1, 8, 8, 3)[0]


def test_splitk_entry_rejects_bad_calls():
    """accumulate, a split count outside [1, K/64] and a short workspace are EPB_EINVAL (checked
    before any device work, so this runs without a GPU)."""
    from epipolarpose_b200 import _lib
    L = _lib.lib()
    g = _geom()                                         # K/64 = 9 * 2 = 18, 1 M tile, Cout 64
    p = ctypes.c_void_p(1 << 20)                        # aligned placeholder, never dereferenced

    def call(splits, ws_floats, accumulate=0):
        g.accumulate = accumulate
        rc = L.epb_conv16_fprop_splitk(ctypes.byref(g), p, p, p, p, None, p, None, splits, p, ws_floats, None)
        g.accumulate = 0
        return rc

    need = 2 * 128 * 64
    assert call(2, need, accumulate=1) == EPB_EINVAL
    assert call(0, need) == EPB_EINVAL
    assert call(19, 19 * need) == EPB_EINVAL
    assert call(2, need - 1) == EPB_EINVAL
    assert call(18, 18 * 128 * 64 - 4) == EPB_EINVAL


def _operands(g, seed=1):
    gen = torch.Generator().manual_seed(seed)
    v = torch.relu(torch.randn(g.N, g.Hi, g.Wi, g.Cin, generator=gen))
    x = torch.empty((2, g.N, g.Hi, g.Wi, g.Cin), dtype=torch.float16)
    em._store_split(x, v, 16.0)
    wv = torch.randn(g.Cout * g.Tw * g.Cin, generator=gen) * 0.05
    w = torch.empty(2 * wv.numel(), dtype=torch.float16)
    w_sc = torch.ones(2)
    em.split16_batch(em.SplitBatch([(wv, w, w_sc)]))
    return x, torch.tensor([16.0, 1 / 16.0]), w, w_sc


def test_split_ranges_cover_k_once():
    for KB in (1, 4, 18, 36, 72, 128):
        for S in range(1, KB + 1):
            r = es.split_ranges(KB, S)
            assert r[0][0] == 0 and r[-1][1] == KB and all(a < b for a, b in r)
            assert all(r[i][1] == r[i + 1][0] for i in range(S - 1))


def test_emulated_splits_match_the_unsplit_product():
    g = _geom()
    x, x_sc, w, w_sc = _operands(g)
    bias = torch.randn(g.Cout, generator=torch.Generator().manual_seed(3))
    ref = torch.zeros(g.N, g.Ho, g.Wo, g.Cout)
    st_ref = torch.zeros(2 * g.Cout, dtype=torch.float64)
    em.conv16_fprop(g, x, x_sc, w, w_sc, ref, bias, st_ref)
    for S in (1, 2, 3, es.kblocks(g)):
        out = torch.zeros_like(ref)
        st = torch.zeros_like(st_ref)
        es.conv16_fprop_splitk(g, x, x_sc, w, w_sc, out, bias, st, S)
        if S == 1:
            assert torch.equal(out, ref)
        e = float((out - ref).abs().max() / ref.abs().max())
        assert e <= 1e-6, (S, e)
        assert float((st - st_ref).abs().max() / st_ref.abs().max()) <= 1e-6


def test_inference_cases_reach_every_split_regime():
    """The split counts the planner gives the cases of test_gpu_infer_step.test_infer_splitk_vs_float64
    (every distinct layer of the R50 inference forward at N = 1, 2, 3, 8, 24 and of C5 at N = 1, 2,
    8): S = 1, S in {2, 3} and S >= 4 all occur, so the float64 test does not silently run S = 1
    only.  At N = 256 (save_triangulations' batch) no call splits, on the H36M model and on C5."""
    from tests import step_cases as sc
    seen = set()
    for keys, Ns in ((["c1", "h36m"], (1, 2, 3, 8, 24)), (["c5"], (1, 2, 8))):
        for N in Ns:
            for conv, hw in sc.infer_layers(keys):
                seen.update(_planned(g)[0] for g in conv.fprop_geoms(em, N, hw, hw, 3) if g is not None)
    assert 1 in seen and seen & {2, 3} and max(seen) >= 4, sorted(seen)
    for key in ("h36m", "c5"):
        HW = sc.INFER_MODELS[key][3]
        assert all(_planned(g) == (1, 0) for _, g in es.conv16_calls(sc.infer_plan(key), 256, HW, HW)), key
