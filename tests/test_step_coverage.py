"""The coverage gate of the training step: every C-ABI entry one step of a composition calls must
have a row in the composition's table naming the tests that hold it to float64 (or bit-exact
against an exact restatement) at that composition's sizes.

Each row of COMPOSITIONS runs one step of its composition at a reduced size and records the
entries it calls: on the CPU through the emulated ABI (tests/emul_ops.py; the labels given, since
the epipolar geometry has no CPU emulation) where the composition has one, and on the device with
online labels.  The inference rows (predict, multiview_h36m, refined, validate_f16x3) run a
predictor or validate_integral instead of a training step, construction included, and reject every
backward, optimiser, loss and training-BatchNorm entry.  A new composition is a new row; its
float64 tests go in its own module, with the shared check bodies of tests/step_cases.py."""
import contextlib
import importlib
import inspect
import math
import re

import pytest
import torch

from tests import step_cases as sc
from tests import tuple_label_cases as tc

gpu = pytest.mark.gpu

# ------------------------------------------------------------------ coverage tables
# C-ABI entry of the step -> tests that check it against float64 (or bit-exact against an exact
# restatement) at the composition's sizes.  C3 (test_c3_selfsup_chain_64_images) runs the geometry
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

S = "test_gpu_c5_step.py::"
COVERAGE_C5 = {
    "epb_im2col_split": [S + "test_c5_im2col_split_bit_exact_at_stem"],
    "epb_conv16_fprop": [S + "test_c5_conv16_layers_vs_torch_float64", S + "test_c5_final_conv16_fprop_vs_float64",
                         S + "test_c5_conv16_stats_vs_float64"],
    "epb_conv16_wgrad": [S + "test_c5_conv16_layers_vs_torch_float64"],
    "epb_bn_finalize_scale": [S + "test_c5_bn_finalize_scale_vs_float64"],
    "epb_bn_finalize": [S + "test_c5_bn_finalize_vs_float64"],
    "epb_bn_act_split": [S + "test_c5_bn_act_split_vs_float64"],
    "epb_bn_relu_maxpool_split": [S + "test_c5_bn_relu_maxpool_split_vs_float64"],
    "epb_maxpool_bwd": [S + "test_c5_maxpool_bwd_vs_float64"],
    "epb_bn_bwd_split": [S + "test_c5_bn_bwd_split_vs_float64"],
    "epb_softargmax_fwd": [S + "test_c5_softargmax_fwd_vs_float64"],
    "epb_softargmax_bwd": [S + "test_c5_softargmax_bwd_fp32_vs_float64"],
    "epb_colsum": [S + "test_c5_colsum_vs_float64"],
    "epb_conv_wgrad": [S + "test_c5_final_tf32_wgrad_vs_float64"],
    "epb_conv_fprop": [S + "test_c5_final_tf32_dgrad_vs_float64"],
    "epb_jointloss_fwd_bwd": [S + "test_c5_jointloss_vs_float64"],
    "epb_split16_batch": [S + "test_c5_split16_batch_bit_exact_on_model_jobs"],
    "epb_pack_weight_batch": [S + "test_c5_pack_weight_batch_bit_exact_on_model_jobs"],
    "epb_adam_step_dev": [S + "test_c5_fused_adam_vs_float64_on_model_buffer"],
    "epb_patch_to_image": [S + "test_c5_selfsup_geometry_j17"],
    "epb_triangulate": [S + "test_c5_selfsup_geometry_j17"],
    "epb_project_labels": [S + "test_c5_selfsup_geometry_j17"],
}
# the head's fp32 backward: entries the C4 step does not call
HEAD_C5 = {"epb_softargmax_bwd", "epb_colsum", "epb_conv_wgrad", "epb_conv_fprop"}

S = "test_gpu_tf32x3_step.py::"
SK = "test_gpu_step_kernels.py::"
COVERAGE_TF32X3 = {
    "epb_nchw_to_nhwc": [S + "test_tf32x3_nchw_to_nhwc_bit_exact"],
    "epb_im2col": [S + "test_tf32x3_im2col_bit_exact_at_stem"],
    "epb_conv_fprop": [S + "test_tf32x3_conv_layers_vs_float64"],
    "epb_conv_wgrad": [S + "test_tf32x3_conv_layers_vs_float64", S + "test_tf32x3_stem_wgrad_through_flat_buffer"],
    "epb_bn_finalize": [S + "test_tf32x3_bn_finalize_vs_float64", SK + "test_bn_finalize_vs_float64_at_bench_M"],
    "epb_bn_relu_maxpool": [S + "test_tf32x3_bn_relu_maxpool_vs_float64"],
    "epb_bn_act": [S + "test_tf32x3_bn_act_vs_float64"],
    "epb_bn_bwd_reduce": [S + "test_tf32x3_bn_bwd_vs_float64", S + "test_tf32x3_bn_bwd_edge_shapes"],
    "epb_bn_bwd_apply": [S + "test_tf32x3_bn_bwd_vs_float64", S + "test_tf32x3_bn_bwd_edge_shapes"],
    "epb_add_masked": [S + "test_tf32x3_add_masked_bit_exact"],
    "epb_maxpool_bwd": [SK + "test_maxpool_bwd_vs_float64_at_stem_bench_size"],
    "epb_softargmax_fwd": [SK + "test_softargmax_fwd_vs_float64_at_bench_shape"],
    "epb_softargmax_bwd": [S + "test_tf32x3_softargmax_bwd_fp32_vs_float64"],
    "epb_colsum": [S + "test_tf32x3_colsum_vs_float64"],
    "epb_jointloss_fwd_bwd": [SK + "test_jointloss_vs_float64_at_bench_shape"],
    "epb_pack_weight_batch": [S + "test_tf32x3_pack_weight_batch_bit_exact_on_model_jobs",
                              S + "test_tf32x3_stem_wgrad_through_flat_buffer"],
    "epb_adam_step_dev": [S + "test_tf32x3_fused_adam_vs_float64_on_model_buffer"],
    "epb_patch_to_image": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
    "epb_triangulate": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
    "epb_project_labels": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
}
# the fp32 engine's own entries: the f16x3 step calls none of them
FP32_ENGINE = {"epb_nchw_to_nhwc", "epb_im2col", "epb_conv_fprop", "epb_conv_wgrad", "epb_bn_finalize",
               "epb_bn_relu_maxpool", "epb_bn_act", "epb_bn_bwd_reduce", "epb_bn_bwd_apply", "epb_add_masked",
               "epb_softargmax_bwd", "epb_colsum"}

COVERAGE_ROBUST = dict(COVERAGE, epb_tuple_labels=["test_gpu_tuple_labels.py::test_kernel_vs_restatement"])
COVERAGE_RELPOSE = dict(COVERAGE, epb_relative_pose=["test_gpu_relpose.py::test_relative_pose_kernel_matches_oracle"])

S = "test_gpu_c2_flat_step.py::"
COVERAGE_C2FLAT = {
    "epb_im2col_split": [S + "test_c2_im2col_split_bit_exact_at_stem"],
    "epb_conv16_fprop": [S + "test_c2_conv16_layers_vs_torch_float64", S + "test_c2_final_conv16_fprop_vs_float64",
                         S + "test_c2_conv16_stats_vs_float64"],
    "epb_conv16_wgrad": [S + "test_c2_conv16_layers_vs_torch_float64"],
    "epb_bn_finalize_scale": [S + "test_c2_bn_finalize_scale_vs_float64"],
    "epb_bn_finalize": [S + "test_c2_bn_finalize_vs_float64"],
    "epb_bn_act_split": [S + "test_c2_bn_act_split_vs_float64"],
    "epb_bn_relu_maxpool_split": [S + "test_c2_bn_relu_maxpool_split_vs_float64"],
    "epb_maxpool_bwd": [S + "test_c2_maxpool_bwd_vs_float64"],
    "epb_bn_bwd_split": [S + "test_c2_bn_bwd_split_vs_float64"],
    "epb_avgpool_split": [S + "test_c2_avgpool_split_vs_float64"],
    "epb_avgpool_bwd": [S + "test_c2_avgpool_bwd_bit_exact"],
    "epb_conv_fprop": [S + "test_c2_head_tf32x3_vs_float64"],
    "epb_conv_wgrad": [S + "test_c2_head_tf32x3_vs_float64"],
    "epb_colsum": [S + "test_c2_colsum_vs_float64"],
    "epb_nhwc_to_nchw": [S + "test_c2_heatmap_layout_bit_exact"],
    "epb_nchw_to_nhwc": [S + "test_c2_heatmap_layout_bit_exact"],
    "epb_heatmap_joint_loss": [S + "test_c2_heatmap_joint_loss_vs_float64",
                               S + "test_c2_heatmap_loss_repeatable_across_grid_sizes"],
    "epb_split16_batch": [S + "test_c2_split16_batch_bit_exact_on_model_jobs"],
    "epb_pack_weight_batch": [S + "test_c2_pack_weight_batch_bit_exact_on_model_jobs"],
    "epb_adam_step_dev": [S + "test_c2_fused_adam_vs_float64_on_model_buffer"],
}
# the VOLUME=False head: entries the C4 step does not call
HEAD_C2FLAT = {"epb_avgpool_split", "epb_avgpool_bwd", "epb_heatmap_joint_loss", "epb_conv_fprop", "epb_conv_wgrad",
               "epb_colsum"}
GEOMETRY = {"epb_patch_to_image", "epb_triangulate", "epb_project_labels", "epb_relative_pose", "epb_tuple_labels"}

S = "test_gpu_refiner_step.py::"
COVERAGE_REFINER = {
    "epb_conv_fprop": [S + "test_refiner_linears_vs_float64"],
    "epb_conv_wgrad": [S + "test_refiner_linears_vs_float64"],
    "epb_pack_weight": [S + "test_refiner_pack_weight_bit_exact"],
    "epb_colsum": [S + "test_refiner_colsum_vs_float64"],
    "epb_bn_finalize": [S + "test_refiner_bn_finalize_vs_float64", S + "test_refiner_training_forward_vs_float64"],
    "epb_bn_act": [S + "test_refiner_bn_act_vs_float64"],
    "epb_bn_bwd_reduce": [S + "test_refiner_bn_bwd_vs_float64"],
    "epb_bn_bwd_apply": [S + "test_refiner_bn_bwd_vs_float64"],
    "epb_bn_eval_affine": [S + "test_refiner_bn_eval_affine_vs_float64", S + "test_refiner_training_forward_vs_float64"],
    "epb_mask_scale": [S + "test_refiner_mask_scale_bit_exact"],
    "epb_add3": [S + "test_refiner_add3_bit_exact"],
    "epb_sumsq": [S + "test_refiner_clip_grad_norm_vs_float64"],
    "epb_clip_scale": [S + "test_refiner_clip_grad_norm_vs_float64"],
    "epb_adam_step": [S + "test_refiner_fused_adam_vs_float64_on_model_buffer"],
}
# the refiner step's entries (refiner/main.py train() and the eval forward of test())
REFINER = set(COVERAGE_REFINER)

# the inference forward: PosePredictor and its subclasses on prepared weights (every conv on the
# split-K entry), and validate_integral's eager eval forward with flip test
S = "test_gpu_infer_step.py::"
SK = "test_gpu_step_kernels.py::"
C2 = "test_gpu_c2_flat_step.py::"
EVAL_CHAIN = [S + "test_infer_eval_chain_vs_float64"]
COVERAGE_PREDICT = {
    "epb_pack_weight_batch": [SK + "test_pack_weight_batch_bit_exact_on_model_jobs",
                              C2 + "test_c2_pack_weight_batch_bit_exact_on_model_jobs"],
    "epb_split16_batch": [SK + "test_split16_batch_bit_exact_on_model_jobs",
                          C2 + "test_c2_split16_batch_bit_exact_on_model_jobs"],
    "epb_bn_eval_affine": [S + "test_infer_bn_eval_affine_within_one_ulp"],
    "epb_im2col_split": [S + "test_infer_im2col_split_bit_exact"],
    "epb_conv16_fprop_splitk": [S + "test_infer_splitk_vs_float64", S + "test_infer_splitk_ragged_final_writes_exactly_its_view",
                                S + "test_infer_splitk_n256_is_the_fused_kernel"],
    "epb_act_scale": EVAL_CHAIN,
    "epb_bn_act_split": EVAL_CHAIN,
    "epb_bn_relu_maxpool_split": EVAL_CHAIN,
    "epb_softargmax_fwd": [S + "test_infer_softargmax_fwd_vs_float64"],
    "epb_softargmax_flip_fwd": [S + "test_infer_softargmax_flip_vs_float64"],
    "epb_patch_to_image": ["test_gpu_sizes.py::test_c3_selfsup_chain_64_images"],
}
COVERAGE_MULTIVIEW = dict(COVERAGE_PREDICT, epb_softargmax_flip_lse_fwd=[S + "test_infer_softargmax_flip_vs_float64"],
                          epb_triangulate_robust=["test_gpu_multiview.py::test_kernel_vs_restatement"])
R = "test_gpu_refiner.py::"
COVERAGE_REFINED = dict(COVERAGE_PREDICT, epb_pose_to_camera=[R + "test_pose_to_camera_is_the_h36m_eval_pred_column"],
                        epb_refiner_prepare=[R + "test_forward_vs_float64_oracle", R + "test_small_width_tails_vs_float64_oracle"],
                        epb_refiner_forward=[R + "test_forward_vs_float64_oracle", R + "test_small_width_tails_vs_float64_oracle"])
COVERAGE_VALIDATE = {k: v for k, v in COVERAGE_PREDICT.items() if k != "epb_conv16_fprop_splitk"}
COVERAGE_VALIDATE.update(
    epb_conv16_fprop=["test_gpu_split16.py::test_conv16_bench_layer_shapes_vs_torch_float64",
                      "test_gpu_bn_chain.py::test_conv16_stats_vs_float64"],
    epb_softargmax_flip_fwd=["test_gpu_flip.py::test_flip_kernel_vs_float64", S + "test_infer_softargmax_flip_vs_float64"])
PREPARED = {"epb_conv16_fprop_splitk", "epb_bn_eval_affine", "epb_split16_batch", "epb_pack_weight_batch",
            "epb_im2col_split", "epb_patch_to_image"}


def _training_entry(e):
    """backward, optimiser, loss and training-BatchNorm entries: no inference forward calls them"""
    return e == "epb_split16" or any(k in e for k in ("bwd", "wgrad", "adam", "loss", "bn_finalize", "colsum",
                                                      "sumsq", "clip_scale"))


def _prepared_only(e):
    """and the prepared forward runs every convolution on the split-K entry"""
    return _training_entry(e) or e == "epb_conv16_fprop"


def _missing_coverage(recorded, table):
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


@contextlib.contextmanager
def _emulated_abi():
    """The model code runs on tests/emul_ops.py: the set of C-ABI entries its wrappers stand for.
    Nested emulations (an emulated entry that calls another) count as their outer entry only."""
    import lib.core.integral_loss as il
    import lib.utils.utils as Ut
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
    il._backend[0], Ut._backend[0] = emul_ops, emul_ops
    try:
        yield rec
    finally:
        for k, f in saved.items():
            setattr(emul_ops, k, f)
        il._backend[0] = Ut._backend[0] = ops


def _three_pass_convs(tags):
    """every conv kernel that ran is a three-pass instantiation, and both an fprop and a wgrad ran"""
    return sc._all_three_pass(tags) and any(t.startswith("fprop") for t in tags) and \
        any(t.startswith("wgrad") for t in tags)


def _fp32_engine(eng):
    from epipolarpose_b200 import net
    return type(eng) is net.Engine and eng.precision == 3 and eng.wgrad_precision == 3


def _refiner_convs(tags):
    """the refiner's linears: every tensor-core kernel a three-pass instantiation, both CUDA-core
    kernels (the 48-channel products) and at least one tensor-core fprop and wgrad"""
    tc = {t for t in tags if "_tc<" in t}
    return sc._all_three_pass(tc) and tags - tc == {"fprop_simt", "wgrad_simt"} and \
        any(t.startswith("fprop") for t in tc) and any(t.startswith("wgrad") for t in tc)


def _mlp_engine(eng):
    from epipolarpose_b200 import mlp
    return type(eng) is mlp.MLPEngine and _fp32_engine(eng.eng)


# ------------------------------------------------------------------ steps
def _eager_step(dev, row):
    """GraphedTrainStep(online=True).eager_step on the bench's cameras, FusedAdam, SmoothL1; with
    the row's estimate_extrinsics, the cameras' extrinsics estimated from the predicted joints"""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.img_utils as iu
    import lib.utils.utils as Ut
    layers, J, D, HW, tuples = row["device"]
    B = 4 * tuples
    est = row.get("estimate_extrinsics", False)
    torch.manual_seed(0)
    m = models.pose3d_resnet.get_pose_net(sc._cfg(layers, J, D, HW), False, precision=row["precision"]).to(dev).train()
    opt = Ut.FusedAdam(list(m.parameters()), lr=1e-3)
    step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J).to(dev), opt, online=True, method=row["method"],
                               estimate_extrinsics=est)
    meta = iu.pack_meta({k: v.to(dev) for k, v in sc._bench_meta(tuples).items()}, B, dev, estimate_extrinsics=est)
    x = torch.randn(B, 3, HW, HW, device=dev)
    return m, lambda: step.eager_step(x, None, None, meta)


def _flat_step(dev, row, shape, ops=None):
    """The VOLUME=False step, eager: forward to (heat-maps, depth_fc output), HeatmapJointLoss
    (L1; Gaussian targets and visibility weights of golden_inputs.heatmap_case, U(-0.5, 0.5)
    depth targets), backward, FusedAdam.step().  shape: (layers, J, D, image size, images)."""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.utils.utils as Ut
    from tests import golden_inputs as gi
    layers, J, D, HW, B = shape
    torch.manual_seed(0)
    m = models.pose3d_resnet.get_pose_net(sc._cfg(layers, J, D, HW, volume=False), False, ops=ops,
                                          precision=row["precision"]).to(dev).train()
    opt = Ut.FusedAdam(list(m.parameters()), lr=1e-3)
    crit = il.HeatmapJointLoss(J, kind="l1")
    _, tg, wh, _, _, _ = gi.heatmap_case(B, J, HW // 4, HW // 4, 5)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, 3, HW, HW, generator=g).to(dev)
    t = (torch.rand(B, J * D, generator=g) - 0.5).to(dev)
    w = torch.ones(B, J * D, device=dev)
    tg, wh = torch.from_numpy(tg).to(dev), torch.from_numpy(wh).to(dev)

    def run():
        loss = crit(m(x), tg, t, w, hm_weight=wh)
        loss.backward()
        opt.step()
        return loss.detach()
    return m, run


def _flat_device_step(dev, row):
    layers, J, D, HW, tuples = row["device"]
    return _flat_step(dev, row, (layers, J, D, HW, 4 * tuples))


def _emulated_graphed_step(row):
    """GraphedTrainStep.eager_step with given labels (R18 trunk or the row's, its J and D, 2 tuples
    x 4 views of 64 x 64), SmoothL1JointLocationLoss, FusedAdam, on the emulated ABI"""
    import lib.models as models
    import lib.core.integral_loss as il
    import lib.core.function as fn
    import lib.utils.utils as Ut
    from tests import emul_ops
    layers, J, D, HW = row["emulated"]
    B = 8
    torch.manual_seed(0)
    m = models.pose3d_resnet.get_pose_net(sc._cfg(layers, J, D, HW), False, ops=emul_ops,
                                          precision=row["precision"]).train()
    opt = Ut.FusedAdam(list(m.parameters()), lr=1e-3)
    step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J), opt, online=False)
    g = torch.Generator().manual_seed(1)
    return m, lambda: step.eager_step(torch.randn(B, 3, HW, HW, generator=g), torch.rand(B, J * 3, generator=g) - 0.5,
                                      torch.ones(B, J * 3), None)


def _emulated_flat_step(row):
    from tests import emul_ops
    layers, J, D, HW = row["emulated"]
    return _flat_step(torch.device("cpu"), row, (layers, J, D, HW, 4), ops=emul_ops)


def _graphed_step(dev, row):
    """GraphedTrainStep(online=True) on a SyntheticH36M tuple batch: warm-up, capture, replay"""
    import lib.core.integral_loss as il
    import lib.core.function as fn
    layers, J, D, HW, tuples = row["device"]
    assert layers == 18
    m, opt = tc.r18(dev, J, D, HW)
    step = fn.GraphedTrainStep(m, il.SmoothL1JointLocationLoss(J).to(dev), opt, online=True, method=row["method"],
                               views=row["views"])
    x, _, _, meta = tc.synthetic_batch(J, HW, tuples, row["views"])

    def run():
        for _ in range(2):
            loss = step(x, meta=meta)
        assert step.graph is not None, "no graph captured"
        return loss
    return m, run


def _refiner_step(dev, shape, ops=None):
    """refiner/main.py train() for one epoch of one batch (LinearModelPG(linear_size, 45 -> 45),
    p_dropout 0.5, FusedAdam, MSELoss on both heads, clip_grad_norm_ to 1), then one eval forward
    of the batch as main.test() runs it; returns the training loss.  shape: (linear_size, rows).
    ops: the model's engine and refiner.utils run on it (the emulated ABI), restored after."""
    import logging
    import types
    import lib.utils.utils as Ut
    from oracle import restate_refiner as rr
    from epipolarpose_b200.refiner import main as rmain, model as rmodel, utils as rutils
    L, N = shape
    m = rmodel.LinearModelPG(linear_size=L, p_dropout=0.5, input_size=45, output_size=45)
    m.load_state_dict(rr.init_state(rr.param_shapes(L, 45, 45), 3))
    m = m.to(dev)
    rmodel.LinearModelPG._backend[0] = ops
    try:
        m._engine()                                  # binds the engine to `ops`
    finally:
        rmodel.LinearModelPG._backend[0] = None
    opt = Ut.FusedAdam(list(m.parameters()), lr=1e-3)
    g = torch.Generator().manual_seed(4)
    x, t = torch.randn(N, 45, generator=g), torch.randn(N, 45, generator=g) * 0.3
    args = types.SimpleNamespace(lr=1e-3, lr_decay=100000, lr_gamma=0.96)
    mse, losses = torch.nn.MSELoss(reduction="mean"), []

    def crit(a, b):
        loss = mse(a, b)
        losses.append(loss.detach())
        return loss

    def run():
        real = rutils._backend[0]
        rutils._backend[0] = ops or real
        try:
            rmain.train(m, [(x, t)], opt, 0, args.lr, crit, args, logging.getLogger("refiner"))
            m.eval()
            with torch.no_grad():
                p2 = m(x.to(dev))[1]
            m.train()
        finally:
            rutils._backend[0] = real
        assert bool(torch.isfinite(p2).all())
        return losses[-2] + losses[-1]
    return m, run


def _refiner_device_step(dev, row):
    return _refiner_step(dev, row["device"])


class _Predictors:
    """the predictors a driver built inside the recorded call; _engine() checks them after it"""

    def __init__(self):
        self.preds = []

    def _engine(self):
        return self.preds


def _prepared_engines(preds):
    """every predictor runs Engine16 on a prepared state"""
    from epipolarpose_b200 import net16
    return bool(preds) and all(type(p.eng) is net16.Engine16 and p.state is not None and
                               {"packed", "w16", "bn", "fbias"} <= set(p.state) for p in preds)


def _images(N, seed, HW=256):
    import numpy as np
    return np.random.default_rng(seed).standard_normal((N, 3, HW, HW)).astype(np.float32)


def _predict_step(dev, row):
    """PosePredictor on the calibrated C1 model at N = 1, without and with flip test: construction
    (prepare_inference), a capture and a replay each"""
    from lib.core.inference import PosePredictor
    from lib.dataset.synthetic import MPII_FLIP_PAIRS
    model, holder, x = sc.calibrated_model(dev, "c1"), _Predictors(), _images(1, 3)

    def run():
        total = 0.0
        for flip in (False, True):
            p = PosePredictor(model, flip_test=flip, shift_heatmap=True, flip_pairs=MPII_FLIP_PAIRS)
            total += float(abs(p(x)).sum())
            holder.preds.append(p)
        return total
    return holder, run


def _multiview_step(dev, row):
    """MultiViewPredictor on the calibrated H36M model, 2 tuples x 4 views, flip test"""
    from lib.core.inference import MultiViewPredictor
    from lib.dataset.synthetic import H36M_FLIP_PAIRS
    from tests import multiview_cases as mc
    model, holder = sc.calibrated_model(dev, "h36m"), _Predictors()
    x, boxes, P = mc.rig_inputs(2, 4, 5)

    def run():
        p = MultiViewPredictor(model, flip_test=True, shift_heatmap=True, flip_pairs=H36M_FLIP_PAIRS)
        holder.preds.append(p)
        return float(abs(p(x, boxes, P)["kps"]).sum())
    return holder, run


def _refined_step(dev, row):
    """RefinedPosePredictor: the calibrated C1 model and a LinearModelPG(1024, 45 -> 45), N = 1"""
    import numpy as np
    from lib.core.inference import RefinedPosePredictor
    from oracle import restate_refiner as rr
    from refiner import model as rmodel
    model, holder, x = sc.calibrated_model(dev, "c1"), _Predictors(), _images(1, 4)
    rnet = rmodel.LinearModelPG(linear_size=1024, input_size=45, output_size=45)
    rnet.load_state_dict(rr.init_state(rr.param_shapes(1024, 45, 45), 43))
    rnet = rnet.to(dev)
    norm = tuple(np.full(45, v, np.float32) for v in (3.0, 120.0, -2.0, 90.0))
    boxes = {"center_x": [500.0], "center_y": [480.0], "width": [300.0], "height": [300.0]}
    cams = {"fl": [[1145.0, 1144.0]], "c_p": [[512.0, 515.0]], "depth": [4500.0]}

    def run():
        p = RefinedPosePredictor(model, rnet, norm, flip_test=False)
        holder.preds.append(p)
        return float(abs(p(x, boxes, cams)["refined"]).sum())
    return holder, run


def _validate_step(dev, row):
    """validate_integral with flip test (shifted) on the calibrated C1 model's eager Engine16 eval
    forward, one batch of 4"""
    import numpy as np
    from lib.core.function import validate_integral
    from lib.dataset.synthetic import MPII_FLIP_PAIRS
    model, x = sc.calibrated_model(dev, "c1"), torch.from_numpy(_images(4, 6))

    class _DS:
        flip_pairs = MPII_FLIP_PAIRS

        def __len__(self):
            return 4

    class _Loader(list):
        dataset = _DS()

    return model, lambda: float(np.abs(validate_integral(_Loader([(x,)]), model, flip_test=True,
                                                         shift_heatmap=True)).sum())


def _emulated_refiner_step(row):
    from tests import emul_ops
    return _refiner_step(torch.device("cpu"), row["emulated"], ops=emul_ops)


# ------------------------------------------------------------------ compositions
# kernel tags a row's predicate accepts (the first) and sets it rejects
TC3 = {"fprop_tc<64,3>", "fprop_tc<128,3>", "wgrad_tc<128,3>"}
REFINER_TAGS = {"fprop_simt", "wgrad_simt", "fprop_tc<128,3>", "wgrad_tc<128,3>"}
# emulated / device: (layers, J, D, image size, and for the device half tuples of 4 views); calls:
# entries every half must call; online: entries the device half (online labels) must call too
COMPOSITIONS = {
    "c4_f16x3": dict(
        table=COVERAGE, precision="f16x3", method="iterative", views=4, driver=_eager_step,
        emulated_driver=_emulated_graphed_step,
        emulated=(18, 16, 64, 64), device=(18, 16, 64, 256, 2),
        calls={"epb_adam_step_dev", "epb_split16_batch"}, online={"epb_triangulate"}, not_called=set(),
        engine=None, tags=None),
    "c5": dict(
        table=COVERAGE_C5, precision="f16x3", method="iterative", views=4, driver=_eager_step,
        emulated_driver=_emulated_graphed_step,
        emulated=(18, 17, 96, 64), device=(101, 17, 96, 384, 2),
        calls=HEAD_C5 | {"epb_adam_step_dev"}, online={"epb_triangulate"}, not_called={"epb_softargmax_bwd_split"},
        engine=lambda eng: not eng.takes_logit_sink(), tags=None),
    "c4_tf32x3": dict(
        table=COVERAGE_TF32X3, precision="tf32x3", method="iterative", views=4, driver=_eager_step,
        emulated_driver=_emulated_graphed_step,
        emulated=(18, 16, 64, 64), device=(50, 16, 64, 256, 2),
        calls=FP32_ENGINE | {"epb_adam_step_dev"}, online={"epb_triangulate"},
        not_called=lambda e: e.endswith("_split") or "conv16" in e,
        engine=_fp32_engine, tags=_three_pass_convs,
        tag_examples=(TC3, [TC3 | {bad} for bad in ("fprop_tc<128,1>", "wgrad_tc<64,1>", "wgrad_simt", "fprop_simt")]
                      + [set()])),
    "robust_tuples": dict(
        table=COVERAGE_ROBUST, precision="f16x3", method="robust", views=4, driver=_graphed_step,
        emulated=None, device=(18, 16, 64, 256, 2),
        calls=set(), online={"epb_tuple_labels"}, not_called={"epb_triangulate"},
        engine=None, tags=None),
    # MODEL.VOLUME: false (SURVEY 8(d) C2(ii)); emulated on R50, since depth_fc takes 2048 inputs
    "c2_flat": dict(
        table=COVERAGE_C2FLAT, precision="f16x3", method=None, views=4, driver=_flat_device_step,
        emulated_driver=_emulated_flat_step, emulated=(50, 17, 4, 64), device=(50, 17, 64, 256, 2),
        calls=HEAD_C2FLAT | {"epb_adam_step_dev"}, online=set(),
        not_called=lambda e: e.startswith("epb_softargmax_") or e == "epb_jointloss_fwd_bwd" or e in GEOMETRY,
        engine=lambda eng: type(eng).__name__ == "Engine16" and not eng.takes_logit_sink(), tags=None),
    # TRAIN.ESTIMATE_EXTRINSICS: each view pair's relative pose from the predicted joints
    "c4_relpose": dict(
        table=COVERAGE_RELPOSE, precision="f16x3", method="iterative", views=4, driver=_eager_step,
        estimate_extrinsics=True, emulated=None, device=(18, 16, 64, 256, 2),
        calls=set(), online={"epb_relative_pose"}, not_called={"epb_tuple_labels"},
        engine=None, tags=None),
    # refiner/main.py train() (LinearModelPG through mlp.MLPEngine on the fp32 engine at 3xTF32)
    # and the eval forward of test(); emulated at linear_size 128, 16 rows
    "refiner": dict(
        table=COVERAGE_REFINER, precision="tf32x3", method=None, views=None, driver=_refiner_device_step,
        emulated_driver=_emulated_refiner_step, emulated=(128, 16), device=(1024, 64),
        calls=REFINER, online=set(),
        not_called=lambda e: e == "epb_adam_step_dev" or e.endswith("_split") or "conv16" in e or
        e.startswith("epb_softargmax_") or e in GEOMETRY,
        engine=_mlp_engine, tags=_refiner_convs,
        tag_examples=(REFINER_TAGS, [REFINER_TAGS | {"fprop_tc<128,1>"}, REFINER_TAGS | {"wgrad_tc<128,1>"}]
                      + [REFINER_TAGS - {t} for t in sorted(REFINER_TAGS)] + [{"fprop_simt", "wgrad_simt"}, set()])),
    # inference (lib/core/inference.py): construction, a capture and a replay inside the recorded call
    "predict": dict(
        table=COVERAGE_PREDICT, precision="f16x3", method=None, views=None, driver=_predict_step,
        emulated=None, device=(50, 16, 64, 256, 1),
        calls=PREPARED | {"epb_softargmax_fwd", "epb_softargmax_flip_fwd"}, online=set(),
        not_called=_prepared_only, engine=_prepared_engines, tags=None),
    "multiview_h36m": dict(
        table=COVERAGE_MULTIVIEW, precision="f16x3", method=None, views=4, driver=_multiview_step,
        emulated=None, device=(50, 17, 64, 256, 2),
        calls=PREPARED | {"epb_softargmax_flip_lse_fwd", "epb_triangulate_robust"}, online=set(),
        not_called=_prepared_only, engine=_prepared_engines, tags=None),
    "refined": dict(
        table=COVERAGE_REFINED, precision="f16x3", method=None, views=None, driver=_refined_step,
        emulated=None, device=(50, 16, 64, 256, 1),
        calls=PREPARED | {"epb_pose_to_camera", "epb_refiner_prepare", "epb_refiner_forward"}, online=set(),
        not_called=_prepared_only, engine=_prepared_engines, tags=None),
    # validate_integral with flip test: the eager eval forward (fused conv16, bn_eval_affine per
    # forward).  Device only: the emulated ABI has no epb_softargmax_flip_fwd
    "validate_f16x3": dict(
        table=COVERAGE_VALIDATE, precision="f16x3", method=None, views=None, driver=_validate_step,
        emulated=None, device=(50, 16, 64, 256, 1),
        calls={"epb_conv16_fprop", "epb_bn_eval_affine", "epb_softargmax_flip_fwd"}, online=set(),
        not_called=lambda e: _training_entry(e) or e == "epb_conv16_fprop_splitk",
        engine=lambda eng: type(eng).__name__ == "Engine16", tags=None),
}
EMULATED = [k for k, row in COMPOSITIONS.items() if row["emulated"] is not None]


def _check_calls(row, calls, required, what):
    print("  %s calls %d entries:" % (what, len(calls)))
    for e in sorted(calls):
        print("    %-28s -> %s" % (e, ", ".join(row["table"].get(e, ["(none)"]))))
    assert required <= calls, "not called: %s" % sorted(required - calls)
    nc = row["not_called"]
    called = sorted(e for e in calls if (nc(e) if callable(nc) else e in nc))
    assert not called, "called: %s" % called
    missing, dangling = _missing_coverage(calls, row["table"])
    assert not missing, "entries without a float64 test at the composition's sizes: %s" % missing
    assert not dangling, dangling


@pytest.mark.parametrize("comp", list(COMPOSITIONS))
def test_gate_has_teeth(comp):
    """Deleting any row, or pointing one at a test that does not exist, fails the gate; the row's
    kernel tag check accepts its good example and rejects each bad one (a single-pass kernel, a
    kernel family that must or must not run, an empty set)."""
    table, tags = COMPOSITIONS[comp]["table"], COMPOSITIONS[comp]["tags"]
    rec = sorted(table)
    assert _missing_coverage(rec, table) == ([], [])
    for k in rec:
        t = dict(table)
        del t[k]
        assert _missing_coverage(rec, t)[0] == [k]
        t[k] = ["test_gpu_step_kernels.py::test_no_such_test"]
        assert _missing_coverage(rec, t)[1]
    if tags is not None:
        good, bads = COMPOSITIONS[comp]["tag_examples"]
        assert tags(good)
        for bad in bads:
            assert not tags(bad), bad


@pytest.mark.parametrize("comp", EMULATED)
def test_gate_emulated_step(comp):
    """One training step of the composition through the emulated ABI, by the row's emulated
    driver: GraphedTrainStep.eager_step with given labels, SmoothL1JointLocationLoss and FusedAdam
    (R18 trunk, its J and D, 2 tuples x 4 views of 64 x 64), or the VOLUME=False step (R50, 4
    images).  Every entry it calls has a row naming existing tests."""
    row = COMPOSITIONS[comp]
    with _emulated_abi() as rec:
        m, run = row["emulated_driver"](row)
        if row["engine"] is not None:
            assert row["engine"](m._engine())
        loss = run()
        assert math.isfinite(float(loss))
    _check_calls(row, rec, row["calls"], "emulated %s step" % comp)


@pytest.fixture(scope="module")
def dev():
    from epipolarpose_b200 import ops
    ops.device_check()
    return torch.device("cuda:0")


@gpu
@pytest.mark.parametrize("comp", list(COMPOSITIONS))
def test_gate_device_step(dev, comp):
    """One step of the composition at a reduced batch (2 tuples x 4 views) with online labels, on
    the device.  Every entry it calls has a row naming existing tests; where the row has a tag
    predicate, the step runs under the profiler and the conv kernels that ran must meet it.  The
    engine predicate is checked after the step, which builds the inference rows' predictors."""
    row = COMPOSITIONS[comp]
    m, run = row["driver"](dev, row)
    losses, tags = [], None
    with sc._record_calls() as names:
        if row["tags"] is None:
            losses.append(float(run()))
        else:
            tags = sc._ran(lambda: losses.append(float(run())))
        torch.cuda.synchronize()
    if row["engine"] is not None:
        assert row["engine"](m._engine())
    assert losses and all(math.isfinite(v) for v in losses)
    if tags is not None:
        print("  conv kernels %s" % sorted(tags))
        assert row["tags"](tags), "conv kernels: %s" % sorted(tags)
    _check_calls(row, names, row["calls"] | row["online"], "%s step" % comp)
