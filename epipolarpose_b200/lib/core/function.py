"""Train / validate / evaluate loops -- host-side mirror of the reference
lib/core/function.py signatures: train_integral(config, train_loader, model,
criterion, optimizer, epoch) (:14-63), validate_integral(val_loader, model)
(:66-110; + the optional flip_test / shift_heatmap keywords), eval_integral(epoch,
preds, val_loader, path, debug) (:113-135).

Differences from the reference body (same observable behaviour):
  * the loss value is kept on the device and read back only when a log line
    is printed (the reference's per-step loss.item() sync, :48, is gone);
  * when config.TRAIN.ONLINE_TRIANGULATION is set the labels are produced per
    batch by the epipolar self-supervision path (lib/utils/img_utils.py
    self_supervision: soft-argmax -> patch->image -> two-view triangulation ->
    re-projection) entirely on the device -- the glue the released reference
    leaves unwired (SURVEY.md section 3.3); with config.TRAIN.ESTIMATE_EXTRINSICS the
    cameras of each view pair are estimated from the predicted 2-D joints (no R, T or
    projection matrix needed: the reference's "without R/t" mode); with
    TRAIN.TRIANGULATION_METHOD robust the batch holds whole tuples of DATASET.TRI_VIEWS views and
    every view's labels come from one robust triangulation of all of them (epb_tuple_labels);
  * the gradient all-reduce for multi-GPU data parallelism happens inside the
    model's backward (one NCCL call on the flat gradient buffer);
  * loader batches of deferred samples (lib/dataset/deferred.py: the h36m / mpii_integral
    datasets indexed in DataLoader workers) are assembled on the device, and a TRI batch
    {'cam_1', 'cam_2'} becomes one batch [cam_1 ; cam_2] (`loader_batch`); the graphed step
    assembles batch i+1 on a side stream while step i replays;
  * validate_integral honours TEST.FLIP_TEST and TEST.SHIFT_HEATMAP (reference
    config.py:118,120, read nowhere by the reference): each batch is one forward of
    [x; flip(x)] and the logits are merged with their flipped-back mirror before the
    soft-argmax (integral_loss.get_joint_location_result_flip);
  * a MODEL.VOLUME = false network, which the reference's result function cannot decode, is
    validated through the heat-map decode (inference.get_heatmap_location_result's rows: the
    get_final_preds argmax and refinement, get_depth_preds as the root-relative depth, the heat-map
    maximum as score), with flip test merged inside the decode; eval_integral scores those rows
    unchanged.
"""
import logging
import time

import numpy as np
import torch

from ..utils.img_utils import (self_supervision_device,
                               trans_coords_from_patch_to_org_3d_batch)
from .integral_loss import get_joint_location_coords_flip, get_result_func, joint_location_result_from_coords
from .inference import check_heatmap_head, heatmap_decode_device, heatmap_rows
from ..utils.utils import AverageMeter
from ..dataset.deferred import assemble_batch, cat_meta, is_deferred, view_keys
from .refine import export_refiner_pairs  # noqa: F401  (public here, next to eval_integral)
from .config import tuple_settings

logger = logging.getLogger(__name__)


def loader_batch(data):
    """(batch_data, label, weight, meta) of a loader batch.  A batch of deferred samples (a
    dataset indexed in DataLoader workers) is assembled on the device; a TRI batch
    {'cam_1', 'cam_2'} becomes one batch [cam_1 ; cam_2], the first-half / second-half pairing
    of online triangulation (reference img_utils.py:194-199); a batch {'cam_1', .., 'cam_V'} of
    whole tuples becomes [cam_1 ; .. ; cam_V], row v*B + t view v of tuple t."""
    if is_deferred(data):
        return assemble_batch(data)
    keys = view_keys(data)
    if keys:
        parts = [data[k] for k in keys]
        return (torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts]), torch.cat([p[2] for p in parts]),
                cat_meta(*[p[3] for p in parts]))
    return data


class _fused_head:
    """Inside the training step nobody but the criterion consumes the logits: let the criterion hand
    their gradient to the network's backward as split planes (_sinks.py).  Off elsewhere, so that
    user code that inspects the logit gradient (retain_grad, hooks, autograd.grad) sees fp32 values."""

    def __init__(self, model):
        net = getattr(model, "module", model)
        self.net = net if hasattr(net, "fused_head_gradient") else None

    def __enter__(self):
        if self.net is not None:
            self.prev, self.net.fused_head_gradient = self.net.fused_head_gradient, True

    def __exit__(self, *exc):
        if self.net is not None:
            self.net.fused_head_gradient = self.prev


def _online_tri(config):
    train = getattr(config, 'TRAIN', None)
    return bool(train is not None and getattr(train, 'ONLINE_TRIANGULATION', False))


def _estimate_extrinsics(config):
    """TRAIN.ESTIMATE_EXTRINSICS: the pair geometry comes from the predicted 2-D joints
    (self-supervision without camera extrinsics); it only applies to online triangulation."""
    train = getattr(config, 'TRAIN', None)
    est = bool(train is not None and getattr(train, 'ESTIMATE_EXTRINSICS', False))
    if est and not _online_tri(config):
        raise ValueError("TRAIN.ESTIMATE_EXTRINSICS needs TRAIN.ONLINE_TRIANGULATION")
    return est


def online_epipolar_loss(criterion, preds, meta, method="iterative", estimate_extrinsics=False, views=2,
                         threshold_px=15.0):
    """criterion(preds, labels(preds), 1) with the labels produced by the epipolar
    self-supervision path from the SAME soft-argmax coordinates the loss uses
    (labels carry no gradient, reference integral_loss.py:88-91).  estimate_extrinsics:
    the cameras of each view pair are estimated from its own 2-D joints, and pairs whose
    estimate failed carry weight 0.  method 'robust': the batch is whole tuples of `views` views,
    view-major (row v*T + t is view v of tuple t), and the labels and weights come from the robust
    triangulation of every view of each tuple (img_utils.tuple_labels_device), each view weighted by
    the peak probability the same soft-argmax pass left in its workspace."""
    from .integral_loss import softmax_integral_tensor, softmax_integral_tensor_lse, _WeightedLossFn
    from ..utils.img_utils import (patch_to_image_device, triangulate_device,
                                   labels_from_global_coords_device,
                                   labels_estimated_extrinsics_device, tuple_labels_device)
    J = criterion.num_joints
    W, H = preds.shape[-1], preds.shape[-2]
    D = preds.shape[-3] // J
    if method == "robust":
        if estimate_extrinsics:
            raise ValueError("the robust online labels need calibrated cameras (no estimate_extrinsics)")
        if preds.shape[0] % views:
            raise ValueError("a batch of %d rows is not whole tuples of %d views" % (preds.shape[0], views))
        coords, lse = softmax_integral_tensor_lse(preds, J, W, H, D)
        with torch.no_grad():
            label, weight = tuple_labels_device(coords.detach(), lse, meta, views, threshold_px)
        return _WeightedLossFn.apply(coords, label, weight, criterion._kind, criterion.size_average,
                                     criterion.norm)
    coords = softmax_integral_tensor(preds, J, True, W, H, D)
    with torch.no_grad():
        kps = patch_to_image_device(coords.detach(), meta)
        if estimate_extrinsics:
            label, weight = labels_estimated_extrinsics_device(kps, meta, method)
        else:
            X = triangulate_device(kps, meta, method)
            label, weight = labels_from_global_coords_device(X, meta)
    return _WeightedLossFn.apply(coords, label, weight, criterion._kind, criterion.size_average,
                                 criterion.norm)


class GraphedTrainStep:
    """One training step (forward, loss, backward incl. the gradient all-reduce, optimiser)
    captured ONCE in a CUDA graph and replayed: the step is ~3000 kernel launches whose
    Python/driver issue time is otherwise comparable to the GPU time.  Inputs are copied
    into static device buffers; hyper-parameters and the step counter live in device
    memory (FusedAdam / FusedSGD), so LR schedules keep working.  The first call runs
    eagerly (sizes workspaces, one-time attributes), the second captures and replays."""

    def __init__(self, model, criterion, optimizer, online=False, method="iterative",
                 estimate_extrinsics=False, views=2, threshold_px=15.0):
        # scripts/train.py:94 wraps the model in nn.DataParallel(device_ids=[k]); with one
        # device id that wrapper only forwards the call (and its scatter is not capturable)
        if isinstance(model, torch.nn.DataParallel) and len(model.device_ids) == 1:
            model = model.module
        self.model, self.criterion, self.optimizer = model, criterion, optimizer
        self.online, self.method = online, method
        if estimate_extrinsics and not online:
            raise ValueError("estimate_extrinsics needs online=True")
        self.estimate_extrinsics = bool(estimate_extrinsics)
        if online and method == "robust" and self.estimate_extrinsics:
            raise ValueError("the robust online labels need calibrated cameras (no estimate_extrinsics)")
        if online and method != "robust" and views != 2:
            raise ValueError("%d views per tuple need method='robust'; the pair triangulators take two" % views)
        self.views, self.threshold_px = int(views), float(threshold_px)
        self.graph = None
        self.key = None
        self.warm_key = None          # shape of the last eager (warm-up) step
        self.failed = False
        self.calls = 0
        self.copy_stream, self.pending, self.stage_next = None, None, 0
        self.assemble_stream, self.staged = None, None
        # eager warm-up and capture share ONE side stream so that the parameters'
        # AccumulateGrad nodes are never bound to the legacy default stream (which
        # may not join a capture)
        self.stream = torch.cuda.Stream() if torch.cuda.is_available() else None

    def eager_step(self, x, label, weight, geom):
        """One un-captured step on the stepper's side stream."""
        if self.stream is None:
            return self._eager(x, label, weight, geom)
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            out = self._eager(x, label, weight, geom)
        cur.wait_stream(self.stream)
        return out

    def _eager(self, x, label, weight, geom):
        self.optimizer.zero_grad()
        with _fused_head(self.model):
            preds = self.model(x)
        if self.online:
            loss = online_epipolar_loss(self.criterion, preds, {"_packed": geom}, self.method,
                                        self.estimate_extrinsics, self.views, self.threshold_px)
        else:
            loss = self.criterion(preds, label, weight)
        loss.backward()
        self.optimizer.step()
        return loss.detach()

    # ---- input staging: the H2D copy of batch i+1 overlaps the replay of step i
    def prefetch(self, batch_data):
        """Start copying a (pinned) host batch into the idle device staging buffer on a copy
        stream; the next __call__ with the SAME tensor object hands it over to the graph's
        static input with a device-side copy (100 MB at HBM speed instead of PCIe speed in
        front of the replay)."""
        if self.graph is None or not torch.cuda.is_available() or batch_data.is_cuda:
            return
        if tuple(batch_data.shape) != tuple(self.sx.shape):
            return
        if self.copy_stream is None:
            self.copy_stream = torch.cuda.Stream()
            self.stage = [torch.empty_like(self.sx) for _ in range(2)]
            self.stage_evt = [torch.cuda.Event() for _ in range(2)]
            self.stage_free = [None, None]
        k = self.stage_next
        with torch.cuda.stream(self.copy_stream):
            if self.stage_free[k] is not None:
                self.copy_stream.wait_event(self.stage_free[k])    # its previous hand-over is done
            self.stage[k].copy_(batch_data, non_blocking=True)
            self.stage_evt[k].record(self.copy_stream)
        self.pending = (batch_data, k)
        self.stage_next = 1 - k

    def stage_batch(self, batch):
        """Assemble a deferred loader batch (lib/dataset/deferred.py) on a side stream, so that
        its decode, crop and labels overlap the replay of the current step; `take` hands it over."""
        if self.graph is None or not torch.cuda.is_available() or not is_deferred(batch):
            return
        if self.assemble_stream is None:
            self.assemble_stream = torch.cuda.Stream()
        with torch.cuda.stream(self.assemble_stream):
            out = assemble_batch(batch)
            ev = torch.cuda.Event()
            ev.record(self.assemble_stream)
        self.staged = (batch, out, ev)

    def take(self, batch):
        """(batch_data, label, weight, meta) of a loader batch; a batch `stage` assembled is
        handed over to the current stream."""
        staged, self.staged = self.staged, None
        if staged is None or staged[0] is not batch:
            return loader_batch(batch)
        cur = torch.cuda.current_stream()
        cur.wait_event(staged[2])
        for t in staged[1][:3]:
            t.record_stream(cur)
        return staged[1]

    def _load_input(self, batch_data):
        if self.pending is not None and self.pending[0] is batch_data:
            k = self.pending[1]
            self.pending = None
            cur = torch.cuda.current_stream()
            cur.wait_event(self.stage_evt[k])
            self.sx.copy_(self.stage[k], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(cur)
            self.stage_free[k] = ev
        else:
            self.sx.copy_(batch_data, non_blocking=True)

    def __call__(self, batch_data, label=None, weight=None, meta=None):
        dev = next(self.model.parameters()).device
        B = batch_data.shape[0]
        geom = None
        if self.online:
            from ..utils.img_utils import pack_meta
            geom = pack_meta(meta, B, dev, self.estimate_extrinsics)
        key = (tuple(batch_data.shape), self.online, self.method, self.views, self.threshold_px,
               self.estimate_extrinsics)
        self.calls += 1
        if self.graph is not None and key == self.key:
            self._load_input(batch_data)
            if self.online:
                for k in self.sgeom:
                    self.sgeom[k].copy_(geom[k], non_blocking=True)
            else:
                self.slabel.copy_(label, non_blocking=True)
                self.sweight.copy_(weight, non_blocking=True)
            if hasattr(self.optimizer, "sync_hyper"):
                self.optimizer.sync_hyper()
            self.graph.replay()
            return self.sloss
        x = batch_data.to(dev, non_blocking=True)
        if not self.online:
            label, weight = label.to(dev, non_blocking=True), weight.to(dev, non_blocking=True)
        # eager when: first call (sizes every scratch buffer), a shape other than the warmed-up
        # one (ragged last batch), no CUDA, or a capture that failed before
        if self.graph is not None or self.failed or not torch.cuda.is_available() \
                or self.warm_key != key:
            self.warm_key = key
            return self.eager_step(x, label, weight, geom)
        # second call with the warmed-up shape: capture, then replay (capture does not execute)
        sx = x.clone()
        sgeom = {k: v.clone() for k, v in geom.items()} if self.online else None
        slabel = label.clone() if not self.online else None
        sweight = weight.clone() if not self.online else None
        if hasattr(self.optimizer, "sync_hyper"):
            self.optimizer.sync_hyper()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        self.optimizer.zero_grad(set_to_none=True)
        try:
            with torch.cuda.graph(graph, stream=self.stream):
                sloss = self._eager(sx, slabel, sweight, sgeom)
        except Exception as e:                     # non-capturable optimiser / wrapper / op
            logger.warning("CUDA-graph capture of the training step failed (%s); running eagerly", e)
            self.failed = True
            torch.cuda.synchronize()
            self.optimizer.zero_grad(set_to_none=True)
            return self.eager_step(x, label, weight, geom)
        # published only after a successful capture
        self.sx, self.sgeom, self.slabel, self.sweight, self.sloss = sx, sgeom, slabel, sweight, sloss
        self.graph, self.key = graph, key
        self.graph.replay()
        return self.sloss


def _graph_capable(model, criterion, optimizer):
    """The captured step needs the fused optimisers (hyper-parameters in device memory) and a
    single-device model: torch.optim.Adam / SGD steps and nn.DataParallel scatter (more than
    one device id: the reference's multi-GPU path, scripts/train.py:94) are not capturable."""
    from ..utils.utils import _FlatOptimizer
    if not hasattr(criterion, '_kind') or not isinstance(optimizer, _FlatOptimizer):
        return False
    if isinstance(model, torch.nn.DataParallel) and len(model.device_ids) != 1:
        return False
    return True


def train_integral(config, train_loader, model, criterion, optimizer, epoch):
    batch_time = AverageMeter()
    data_time = AverageMeter()
    losses = AverageMeter()
    model.train()
    online = _online_tri(config)
    estimate = _estimate_extrinsics(config)
    views, method, thr = tuple_settings(config)
    pending = []           # (device loss, batch size) not yet folded into `losses`
    use_graph = bool(getattr(config.TRAIN, 'CUDA_GRAPH', True)) and \
        _graph_capable(model, criterion, optimizer)
    stepper = getattr(model, '_epb_graphed_step', None)
    if use_graph and (stepper is None or stepper.optimizer is not optimizer
                      or stepper.criterion is not criterion or stepper.online != online
                      or stepper.estimate_extrinsics != estimate or stepper.method != method
                      or stepper.views != views or stepper.threshold_px != thr):
        stepper = GraphedTrainStep(model, criterion, optimizer, online, method, estimate, views, thr)
        model._epb_graphed_step = stepper
    end = time.time()
    it = iter(train_loader)
    nxt = next(it, None)
    i = -1
    while nxt is not None:
        data, i = nxt, i + 1
        nxt = next(it, None)
        data_time.update(time.time() - end)
        batch_data, batch_label, batch_label_weight, meta = \
            stepper.take(data) if use_graph else loader_batch(data)
        batch_size = batch_data.size(0)
        if use_graph:
            if stepper.pending is None and stepper.graph is not None:
                stepper.prefetch(batch_data)              # first replayed batch of this call
            loss = stepper(batch_data, batch_label, batch_label_weight, meta)
            if stepper.graph is not None:
                loss = loss.clone()      # the static loss buffer is overwritten by the next replay
                if nxt is not None:      # H2D / device assembly of the next batch overlaps this step
                    if is_deferred(nxt):
                        stepper.stage_batch(nxt)
                    elif isinstance(nxt, (list, tuple)):
                        stepper.prefetch(nxt[0])
            pending.append((loss, batch_size))
            del loss
        else:
            optimizer.zero_grad()
            batch_data = batch_data.cuda(non_blocking=True)
            with _fused_head(model):
                preds = model(batch_data)
            if online:
                # one soft-argmax pass serves both the epipolar labels and the loss
                loss = online_epipolar_loss(criterion, preds, meta, method, estimate, views, thr)
                batch_label = batch_label_weight = None
            else:
                batch_label = batch_label.cuda(non_blocking=True)
                batch_label_weight = batch_label_weight.cuda(non_blocking=True)
                loss = criterion(preds, batch_label, batch_label_weight)
            del batch_data, batch_label, batch_label_weight, preds
            loss.backward()
            optimizer.step()
            pending.append((loss.detach(), batch_size))
            del loss
        if i % config.PRINT_FREQ == 0:
            for lv, bs in pending:
                losses.update(lv.item(), bs)      # the only device sync of the loop
            pending = []
            batch_time.update(time.time() - end)
            msg = 'Epoch: [{0}][{1}/{2}]\t' \
                  'Time {batch_time.val:.3f}s ({batch_time.avg:.3f}s)\t' \
                  'Speed {speed:.1f} samples/s\t' \
                  'Data {data_time.val:.3f}s ({data_time.avg:.3f}s)\t' \
                  'Loss {loss.val:.5f} ({loss.avg:.5f})'.format(
                      epoch, i, len(train_loader), batch_time=batch_time,
                      speed=batch_size / max(batch_time.val, 1e-9),
                      data_time=data_time, loss=losses)
            logger.info(msg)
        else:
            batch_time.update(time.time() - end)
        end = time.time()
    for lv, bs in pending:
        losses.update(lv.item(), bs)
    return losses.avg


def _flip_pairs(dataset):
    pairs = getattr(dataset, 'flip_pairs', None)
    if pairs is None:
        db = getattr(dataset, 'db', None)
        if db:
            pairs = db[0].get('flip_pairs') if isinstance(db[0], dict) else None
    return pairs


def _validate_flip(val_loader, model, shift_heatmap):
    """Flip-test validation: one forward of the 2B images [x; flip(x, 3)] per batch, merged
    coordinates kept on the device, one copy to the host after the loop."""
    net = getattr(model, 'module', model)
    flat = not getattr(net, 'volume', True)
    if flat:
        check_heatmap_head(net)
    pairs = _flip_pairs(val_loader.dataset)
    if pairs is None:
        raise ValueError("flip test needs the dataset's joint pairs: neither dataset.flip_pairs nor "
                         "dataset.db[0]['flip_pairs'] exists")
    dev = next(model.parameters()).device
    model.eval()
    chunks = []
    with torch.no_grad():
        for data in val_loader:
            x = loader_batch(data)[0]
            B = x.shape[0]
            buf = torch.empty((2 * B,) + tuple(x.shape[1:]), device=dev, dtype=torch.float32)
            buf[:B].copy_(x, non_blocking=True)
            buf[B:] = torch.flip(buf[:B], [3])
            preds = model(buf)
            if flat:
                chunks.append(_heatmap_decode(preds, pairs, shift_heatmap))
            else:
                chunks.append(get_joint_location_coords_flip(preds, pairs, shift_heatmap))
            del preds, buf
    if not chunks:
        return np.zeros((0, 0, 4))
    if flat:
        return heatmap_rows(torch.cat(chunks, dim=0).cpu().numpy(), 256)[0:len(val_loader.dataset)]
    coords = torch.cat(chunks, dim=0).cpu().numpy()
    out = joint_location_result_from_coords(256, 256, coords)     # hard-coded 256 as reference :87
    return out[0:len(val_loader.dataset)]


def _heatmap_decode(preds, flip_pairs=None, shift_heatmap=False):
    """(heatmaps, depth) of a MODEL.VOLUME = false network -> kps [N, J, 4] on the device (patch px,
    root-relative mm, maxval): epb_heatmap_decode with the config's DEPTH_RES, DEPTH_RANGE and
    TEST.POST_PROCESS."""
    from .config import config
    hm, depth = preds
    return heatmap_decode_device(hm, depth, int(config.MODEL.DEPTH_RES), None, 256, 256,
                                 float(config.DATASET.DEPTH_RANGE), bool(config.TEST.POST_PROCESS),
                                 flip_pairs, shift_heatmap)


def _validate_heatmap(val_loader, model):
    """Validation of a MODEL.VOLUME = false network: the heat-map decode of each batch kept on the
    device, one copy to the host after the loop; rows as get_heatmap_location_result."""
    check_heatmap_head(getattr(model, 'module', model))
    model.eval()
    chunks = []
    with torch.no_grad():
        for data in val_loader:
            batch_data = loader_batch(data)[0].cuda(non_blocking=True)
            chunks.append(_heatmap_decode(model(batch_data)))
            del batch_data
    if not chunks:
        return np.zeros((0, 0, 4))
    return heatmap_rows(torch.cat(chunks, dim=0).cpu().numpy(), 256)[0:len(val_loader.dataset)]   # 256 as :87


def validate_integral(val_loader, model, flip_test=None, shift_heatmap=None):
    """flip_test / shift_heatmap default to config.TEST.FLIP_TEST / TEST.SHIFT_HEATMAP of the
    module-global config (filled by update_config)."""
    from .config import config
    if flip_test is None:
        flip_test = bool(config.TEST.FLIP_TEST)
    if shift_heatmap is None:
        shift_heatmap = bool(config.TEST.SHIFT_HEATMAP)
    print("Validation stage")
    if flip_test:
        return _validate_flip(val_loader, model, shift_heatmap)
    if not getattr(getattr(model, 'module', model), 'volume', True):
        return _validate_heatmap(val_loader, model)
    result_func = get_result_func()
    model.eval()
    chunks = []
    with torch.no_grad():
        for i, data in enumerate(val_loader):
            batch_data = loader_batch(data)[0].cuda(non_blocking=True)
            preds = model(batch_data)
            chunks.append(result_func(256, 256, preds))     # hard-coded 256 as reference :87
            del preds, batch_data
    if not chunks:
        return np.zeros((0, 0, 4))
    out = np.concatenate(chunks, axis=0)                   # ragged last batch handled
    return out[0:len(val_loader.dataset)]


def eval_integral(epoch, preds_in_patch_with_score, val_loader, final_output_path, debug=False, with_names=False):
    """perf of the dataset's evaluate, or (perf, [(name, value), ..]) with `with_names`: the values it
    logs, at full precision."""
    print("Evaluation stage")
    imdb_list = val_loader.dataset.db
    imdb = val_loader.dataset
    n = len(val_loader.dataset)
    get = lambda k: np.array([imdb_list[s][k] for s in range(n)], dtype=np.float64)
    preds_in_img_with_score = trans_coords_from_patch_to_org_3d_batch(
        np.asarray(preds_in_patch_with_score)[:n], get('center_x'), get('center_y'), get('width'),
        get('height'), 256, 256, 2000)
    name_value, perf = imdb.evaluate(preds_in_img_with_score.copy(), final_output_path, debug=debug)
    for name, value in name_value:
        logger.info('Epoch[%d] Validation-%s %f', epoch, name, value)
    if with_names:
        return perf, [(name, float(value)) for name, value in name_value]
    return perf


def world_joints_of_record(rec):
    """Ground-truth joints of one H36M record in the world frame [J, 3] (mm).  The records carry no
    world-frame joints: `joints_3d` holds image x, y (px) and the depth relative to the pelvis (mm),
    `pelvis` the camera-frame pelvis, `fl` / `c_p` the intrinsics.  They are back-projected to the
    camera frame as the evaluation does (prep_h36m.py:85-89) and brought to the world frame with the
    record's cam.R, cam.T: X = R^T X_cam + T, the inverse of the X_cam = R (X - T) that
    epb_project_labels applies."""
    j = np.asarray(rec['joints_3d'], dtype=np.float64)
    fl = np.asarray(rec['fl'], dtype=np.float64).reshape(-1)
    cp = np.asarray(rec['c_p'], dtype=np.float64).reshape(-1)
    d = j[:, 2] + np.asarray(rec['pelvis'], dtype=np.float64).reshape(-1)[2]
    xc = np.stack([(j[:, 0] - cp[0]) / fl[0] * d, (j[:, 1] - cp[1]) / fl[1] * d, d], axis=1)
    R = np.asarray(rec['cam'].R, dtype=np.float64).reshape(3, 3)
    T = np.asarray(rec['cam'].T, dtype=np.float64).reshape(1, 3)
    return xc @ R + T


def validate_multiview(dataset, predictor, tuples_per_batch=8):
    """Multi-view inference over every view tuple of `dataset` (H36M_Integral.view_tuples()):
    each frame is read and cropped through the dataset's sample path with augmentation off, the
    views go through `predictor(images [T,V,3,H,W], boxes, P [T,V,3,4])` (a MultiViewPredictor) with
    P from each record's cam.projection_matrix, and the triangulated pose is compared with the
    ground truth in the world frame: world_joints_of_record of every view (see there for the
    fields used), averaged over the views.

    Returns a dict: mpjpe (mm, mean over the joints with status 1), inlier_views (mean number of
    inlier views per joint, a failed joint counting 0), failed (share of joints with status 0),
    tuples, and -- when the records carry `action` -- per_action: {action: the same three}."""
    import copy
    recs = [dataset.tuple_records(r) for r in dataset.view_tuples()]
    was_train, dataset.is_train = dataset.is_train, False        # crop without augmentation
    err, ninl, stat, acts = [], [], [], []
    try:
        for b in range(0, len(recs), max(1, int(tuples_per_batch))):
            chunk = recs[b:b + max(1, int(tuples_per_batch))]
            views = [[dataset.get_data(copy.deepcopy(r)) for r in tup] for tup in chunk]
            images = np.stack([np.stack([v[0] for v in tup]) for tup in views]).astype(np.float32)
            metas = [v[3] for tup in views for v in tup]
            boxes = {k: np.array([float(m[k]) for m in metas])
                     for k in ('center_x', 'center_y', 'width', 'height', 'scale', 'rot')}
            P = np.stack([np.stack([np.asarray(v[3]['projection_matrix'], dtype=np.float64)[0:3, 0:4]
                                    for v in tup]) for tup in views])
            out = predictor(images, boxes, P)
            gt = np.stack([np.mean([world_joints_of_record(r) for r in tup], axis=0) for tup in chunk])
            err.append(np.linalg.norm(out['world'] - gt, axis=2))
            stat.append(np.asarray(out['status']) != 0)
            ninl.append(np.array([[bin(int(m)).count('1') for m in row] for row in out['inliers']]))
            acts.extend(tup[0].get('action') for tup in chunk)
    finally:
        dataset.is_train = was_train
    if not err:
        return {'mpjpe': float('nan'), 'inlier_views': float('nan'), 'failed': float('nan'), 'tuples': 0}
    err, stat, ninl = np.concatenate(err), np.concatenate(stat), np.concatenate(ninl)

    def summary(sel):
        e, s = err[sel], stat[sel]
        return {'mpjpe': float(e[s].mean()) if s.any() else float('nan'),
                'inlier_views': float(ninl[sel].mean()), 'failed': float(1.0 - s.mean())}

    res = summary(np.ones(len(err), dtype=bool))
    res['tuples'] = int(len(err))
    if all(a is not None for a in acts):
        acts = np.array(acts)
        res['per_action'] = {str(a): summary(acts == a) for a in sorted(set(acts.tolist()))}
    return res
