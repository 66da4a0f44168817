"""Hard-argmax keypoint decode -- host-side mirror of the reference
lib/core/inference.py:12-68 (`get_max_preds`, `get_final_preds`), with the
per-(n,j) argmax running in the warp-shuffle kernel epb_argmax2d (first-index
tie-break == numpy.argmax; indices are bit-exact).  numpy in / numpy out like
the reference; `get_max_preds_device` is the tensor-in / tensor-out variant.

Addition: `PosePredictor`, images -> 3-D joints as one CUDA-graph replay per call (the
`model.eval(); get_joint_location_result(W, H, model(img))` of demo.ipynb and scripts/valid.py).
`MultiViewPredictor`: the calibrated views of a rig -> world-frame joints, the same network on
every view followed by the robust V-view triangulation inside the same graph."""
import numpy as np
import torch

from epipolarpose_b200 import net16 as _net16
from epipolarpose_b200 import ops as _ops

_backend = [_ops]


def get_max_preds_device(heatmaps):
    """heatmaps [N,J,H,W] float32 CUDA contiguous -> (preds [N,J,2] f32,
    maxvals [N,J,1] f32, idx [N,J] int32) on the device."""
    ops = _backend[0]
    assert heatmaps.dim() == 4, 'batch_images should be 4-ndim'
    hm = heatmaps.contiguous()
    N, J, H, W = hm.shape
    idx = torch.empty((N, J), device=hm.device, dtype=torch.int32)
    maxvals = torch.empty((N, J, 1), device=hm.device, dtype=torch.float32)
    preds = torch.empty((N, J, 2), device=hm.device, dtype=torch.float32)
    if N * J:
        ops.argmax2d(hm, N * J, H, W, idx, maxvals, preds)
    return preds, maxvals, idx


def get_max_preds(batch_heatmaps):
    """reference :12-40 (numpy [N,J,H,W] -> preds [N,J,2] f32, maxvals [N,J,1])."""
    assert isinstance(batch_heatmaps, np.ndarray), 'batch_heatmaps should be numpy.ndarray'
    assert batch_heatmaps.ndim == 4, 'batch_images should be 4-ndim'
    dev = torch.device("cuda") if _backend[0] is _ops else torch.device("cpu")
    hm = torch.from_numpy(np.ascontiguousarray(batch_heatmaps, dtype=np.float32)).to(dev)
    preds, maxvals, _ = get_max_preds_device(hm)
    return preds.cpu().numpy(), maxvals.cpu().numpy().astype(batch_heatmaps.dtype)


def get_final_preds_device(heatmaps, center, scale, post_process=True):
    """heatmaps [N,J,H,W] float32 (device), center / scale [N,2] -> (preds [N,J,2] f32 image
    coordinates, maxvals [N,J,1] f32) on the device: argmax, +-0.25 px refinement and the
    heat-map -> image affine in ONE launch (epb_final_preds)."""
    ops = _backend[0]
    hm = heatmaps.contiguous()
    N, J, H, W = hm.shape
    dev = hm.device
    c = torch.as_tensor(np.asarray(center, dtype=np.float64).reshape(N, 2)).to(dev)
    sc = torch.as_tensor(np.asarray(scale, dtype=np.float64).reshape(N, 2)).to(dev)
    preds = torch.empty((N, J, 2), device=dev, dtype=torch.float32)
    maxvals = torch.empty((N, J, 1), device=dev, dtype=torch.float32)
    if N * J:
        ops.final_preds(hm, N, J, H, W, c, sc, post_process, preds, maxvals)
    return preds, maxvals


def get_final_preds(config, batch_heatmaps, center, scale):
    """reference :43-68 (numpy in / numpy out)."""
    assert isinstance(batch_heatmaps, np.ndarray), 'batch_heatmaps should be numpy.ndarray'
    dev = torch.device("cuda") if _backend[0] is _ops else torch.device("cpu")
    hm = torch.from_numpy(np.ascontiguousarray(batch_heatmaps, dtype=np.float32)).to(dev)
    scale = np.stack([np.asarray(s_, dtype=np.float64).reshape(-1)[:2] if np.ndim(s_) else
                      np.array([s_, s_], dtype=np.float64) for s_ in scale])
    preds, maxvals = get_final_preds_device(hm, np.asarray(center), scale,
                                            config.TEST.POST_PROCESS)
    return preds.cpu().numpy(), maxvals.cpu().numpy().astype(batch_heatmaps.dtype)


class PosePredictor:
    """Images -> joints at interactive latency: the network, the soft-argmax and the patch -> image
    transform captured as ONE CUDA graph per batch size N (lazily, on the first call with that N)
    and replayed; a call copies the images into the graph's static input, replays, and copies the
    [N, J, 3] result to the host.  The network runs on the split-fp16 engine with the weights
    prepared once and every convolution on the split-K entry (epb_conv16_fprop_splitk), so that
    layers with few tiles at small N still spread over the GPU.

    Snapshot semantics: the weights, the BatchNorm running statistics and the final bias are read
    when the predictor is built and again by refresh(), never in between.  Call refresh() after
    the model changed (training steps, load_state_dict): in-place optimisers such as FusedAdam
    write through raw pointers, so nothing can detect the change.  The predictor always runs eval
    semantics (BatchNorm on running statistics) whatever model.training says.

    pred(images): images float32 [N, 3, H, W] (host or device) -> numpy float64 [N, J, 4], the
    numbers and layout of get_joint_location_result(W, H, model.eval()(images)): (x, y, z) in patch
    pixels and a score of 1.  pred(images, boxes=meta): meta holds center_x, center_y, width,
    height and optionally scale (default 1) and rot (default 0) per image; (x, y, z) are then in
    original-image coordinates (trans_coords_from_patch_to_org_3d, rect_3d_w 2000).
    flip_test / shift_heatmap default to config.TEST.FLIP_TEST / TEST.SHIFT_HEATMAP as in
    validate_integral; with flip test every call replays a 2N graph of [x; flip(x)] merged by
    epb_softargmax_flip_fwd, and flip_pairs (the dataset's joint pairs) is required.
    pred.logits: the static logit buffer of the last call ([N or 2N, J*D, H/4, W/4], channels_last
    memory), overwritten by the next call with the same N."""

    RECT_3D_W = 2000.0              # eval_integral's rect_3d_w

    def __init__(self, model, flip_test=None, shift_heatmap=None, flip_pairs=None):
        from .config import config
        from .integral_loss import flip_permutation
        net = getattr(model, "module", model)
        if not getattr(net, "volume", False):
            raise ValueError("PosePredictor needs the VOLUME head (MODEL.VOLUME: true): it decodes "
                             "the 3-D soft-argmax of the logit volume")
        if getattr(net, "precision", None) != 4:
            raise ValueError("PosePredictor runs the split-fp16 engine (MODEL.PRECISION: f16x3); "
                             "this model runs another precision")
        if not _net16.supported(net._plan):
            raise ValueError("PosePredictor runs the split-fp16 engine, which needs every layer's "
                             "channels in whole 64-channel blocks; this model's plan has others")
        self.flip_test = bool(config.TEST.FLIP_TEST) if flip_test is None else bool(flip_test)
        self.shift_heatmap = bool(config.TEST.SHIFT_HEATMAP) if shift_heatmap is None \
            else bool(shift_heatmap)
        if self.flip_test:
            if flip_pairs is None:
                raise ValueError("flip test needs the dataset's joint pairs (flip_pairs)")
            flip_permutation(flip_pairs, net._plan.num_joints)
        self.flip_pairs = flip_pairs
        self.model = net
        self.dev = next(net.parameters()).device
        self.eng = _net16.Engine16(net._plan, ops=net._ops)
        self.stream = torch.cuda.Stream(self.dev)
        self.graphs = {}
        self.state = None
        self.logits = None
        self.refresh()

    def refresh(self):
        """Re-read the model's weights and BatchNorm buffers into the predictor's snapshot."""
        with torch.no_grad(), torch.cuda.device(self.dev):
            params = {k: v.detach() for k, v in self.model.named_parameters()}
            params.update(dict(self.model.named_buffers()))
            state = self.eng.prepare_inference(params, self.dev, self.state)
        if self.state is not None and state["w16"] is not self.state["w16"]:
            self.graphs.clear()         # the parameters moved: the graphs read the old planes
        self.state = state

    def _forward(self, ent):
        """The captured work: [flip,] network, soft-argmax, patch -> image."""
        from .integral_loss import get_joint_location_coords, get_joint_location_coords_flip
        from ..utils.img_utils import patch_to_image_device
        x, box = ent["x"], ent["box"]
        N, H, W = box.shape[0], x.shape[2], x.shape[3]
        if self.flip_test:
            x[N:] = torch.flip(x[:N], [3])
        logits, _, _ = self.eng.forward(x, None, training=False, save=False, prepared=self.state)
        out = logits.permute(0, 3, 1, 2)
        fin = self.eng.plan.final
        if out.shape[1] != fin.cout:
            out = out[:, :fin.cout]
        if self.flip_test:
            coords = get_joint_location_coords_flip(out, self.flip_pairs, self.shift_heatmap)
        else:
            coords = get_joint_location_coords(out)
        ent["logits"], ent["coords"] = out, coords
        ent["kps"] = patch_to_image_device(coords, {"_packed": {"box": box}}, W, H, self.RECT_3D_W)

    def _capture(self, N, H, W):
        B = 2 * N if self.flip_test else N
        box = torch.tensor([[W / 2.0, H / 2.0, W, H, 1.0, 0.0]], dtype=torch.float64).repeat(N, 1)
        ent = {"x": torch.zeros((B, 3, H, W), device=self.dev), "box": box.to(self.dev)}
        return self._record((N, H, W), ent)

    def _record(self, key, ent):
        """Warm up and capture self._forward(ent) as the graph of `key`."""
        cur = torch.cuda.current_stream(self.dev)
        # warm-up then capture on a side stream (GraphedTrainStep): the eager run sets the
        # kernels' one-time attributes and the geometry caches
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            self._forward(ent)
        torch.cuda.synchronize(self.dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=self.stream):
            self._forward(ent)
        cur.wait_stream(self.stream)
        ent["graph"] = graph
        self.graphs[key] = ent
        return ent

    def __call__(self, images, boxes=None):
        x = torch.as_tensor(images)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected images [N, 3, H, W], got %s" % (tuple(x.shape),))
        if x.dtype != torch.float32:
            raise TypeError("expected float32 images, got %s" % x.dtype)
        N, _, H, W = x.shape
        with torch.cuda.device(self.dev):
            ent = self.graphs.get((N, H, W)) or self._capture(N, H, W)
            ent["x"][:N].copy_(x, non_blocking=x.is_cuda)
            if boxes is not None:
                from ..utils.img_utils import _boxes
                meta = dict(boxes)
                meta.setdefault("scale", np.ones(N))
                meta.setdefault("rot", np.zeros(N))
                ent["box"].copy_(_boxes(meta, N, torch.device("cpu")))
            ent["graph"].replay()
            self.logits = ent["logits"]
            J = ent["kps"].shape[1]
            if boxes is None:
                from .integral_loss import joint_location_result_from_coords
                return joint_location_result_from_coords(W, H, ent["coords"].cpu().numpy())
            out = np.ones((N, J, 4), dtype=np.float64)
            out[:, :, :3] = ent["kps"][:, :, :3].cpu().numpy()
            return out


class MultiViewPredictor(PosePredictor):
    """Calibrated views of one person -> world-frame joints, one CUDA-graph replay per call: the
    network on the T*V images (PosePredictor's engine, snapshot and refresh()), the soft-argmax
    with its per-joint confidence, the patch -> image transform and the robust V-view
    triangulation (epb_triangulate_robust), one graph per (T, V, H, W).  The boxes and the
    projection matrices live in static device buffers that every call fills before the replay.

    pred(images, boxes, P): images float32 [T, V, 3, H, W] (host or device), 2 <= V <= 8; boxes
    holds center_x, center_y, width, height and optionally scale (default 1) and rot (default 0),
    T*V values each in (tuple, view) order; P float64 [T, V, 3, 4] maps world coordinates to
    original-image pixels.  Returns a dict of numpy arrays:
      world   [T, J, 3]    float64, in the frame and unit of P (mm for Human3.6M); 0 where status is 0
      kps     [T, V, J, 4] float64 per view: image x, y, root-relative z (mm), confidence
      inliers [T, J]       int32 bit mask: bit v set <=> view v is in the final fit
      resid   [T, J]       float64 RMS reprojection error (px) over the inlier views
      status  [T, J]       int32 1 = triangulated from at least two agreeing views, else 0
    The confidence is the peak softmax probability of the joint's volume (with flip test, of the
    merged volume).  use_confidence: the confidences weigh the views in the refit (they never decide
    which views agree).  threshold_px: the reprojection error, in original-image pixels, up to which
    a view agrees with a hypothesis; the default is a guess that has not been tuned on real
    predictions.  Constructor refusals as PosePredictor."""

    def __init__(self, model, flip_test=None, shift_heatmap=None, flip_pairs=None, threshold_px=15.0,
                 use_confidence=True):
        if not (np.isfinite(threshold_px) and threshold_px > 0):
            raise ValueError("threshold_px must be a positive number of pixels, got %r" % (threshold_px,))
        super().__init__(model, flip_test, shift_heatmap, flip_pairs)
        self.threshold_px = float(threshold_px)
        self.use_confidence = bool(use_confidence)

    def _forward(self, ent):
        """The captured work: [flip,] network, soft-argmax + confidence, patch -> image, triangulation."""
        from .integral_loss import get_joint_location_coords_peak, get_joint_location_coords_flip_peak
        from ..utils.img_utils import patch_to_image_device
        from ..utils.triangulation import triangulate_views_robust
        x, box, P = ent["x"], ent["box"], ent["P"]
        (T, V), N, H, W = P.shape[:2], box.shape[0], x.shape[2], x.shape[3]
        if self.flip_test:
            x[N:] = torch.flip(x[:N], [3])
        logits, _, _ = self.eng.forward(x, None, training=False, save=False, prepared=self.state)
        out = logits.permute(0, 3, 1, 2)
        fin = self.eng.plan.final
        if out.shape[1] != fin.cout:
            out = out[:, :fin.cout]
        if self.flip_test:
            coords, peak = get_joint_location_coords_flip_peak(out, self.flip_pairs, self.shift_heatmap)
        else:
            coords, peak = get_joint_location_coords_peak(out)
        kps = patch_to_image_device(coords, {"_packed": {"box": box}}, W, H, self.RECT_3D_W)
        conf = peak.double()
        kps[:, :, 3] = conf
        J = kps.shape[1]
        ent["logits"], ent["coords"], ent["kps"] = out, coords, kps
        ent["w"] = conf.reshape(T, V, J).contiguous() if self.use_confidence else None
        if "tri" not in ent:
            ent["tri"] = (torch.empty((T, J, 3), device=self.dev, dtype=torch.float64),
                          torch.empty((T, J), device=self.dev, dtype=torch.int32),
                          torch.empty((T, J), device=self.dev, dtype=torch.int32),
                          torch.empty((T, J), device=self.dev, dtype=torch.float64))
        triangulate_views_robust(kps.view(T, V, J, 4), P, ent["w"], self.threshold_px, out=ent["tri"])

    def __call__(self, images, boxes=None, P=None):
        if boxes is None or P is None:
            raise ValueError("MultiViewPredictor needs the boxes and the projection matrices of every view")
        x = torch.as_tensor(images)
        if x.dim() != 5 or x.shape[2] != 3:
            raise ValueError("expected images [T, V, 3, H, W], got %s" % (tuple(x.shape),))
        if x.dtype != torch.float32:
            raise TypeError("expected float32 images, got %s" % x.dtype)
        T, V, _, H, W = x.shape
        if T < 1 or not 2 <= V <= 8:
            raise ValueError("expected T >= 1 tuples of 2..8 views, got T = %d, V = %d" % (T, V))
        Pm = torch.as_tensor(P)
        if tuple(Pm.shape) != (T, V, 3, 4) or Pm.dtype != torch.float64:
            raise ValueError("expected P float64 [%d, %d, 3, 4], got %s %s" % (T, V, Pm.dtype, tuple(Pm.shape)))
        N = T * V
        from ..utils.img_utils import _boxes
        meta = {k: np.asarray(v, dtype=np.float64).reshape(-1) for k, v in dict(boxes).items()}
        meta.setdefault("scale", np.ones(N))
        meta.setdefault("rot", np.zeros(N))
        for k in ("center_x", "center_y", "width", "height", "scale", "rot"):
            if k not in meta or meta[k].size != N:
                raise ValueError("boxes[%r] must hold T*V = %d values" % (k, N))
        with torch.cuda.device(self.dev):
            key = (T, V, H, W)
            ent = self.graphs.get(key)
            if ent is None:
                B = 2 * N if self.flip_test else N
                box0 = torch.tensor([[W / 2.0, H / 2.0, W, H, 1.0, 0.0]], dtype=torch.float64).repeat(N, 1)
                ent = {"x": torch.zeros((B, 3, H, W), device=self.dev), "box": box0.to(self.dev),
                       "P": torch.zeros((T, V, 3, 4), device=self.dev, dtype=torch.float64)}
                ent["P"].copy_(Pm)             # the warm-up run sees real cameras
                self._record(key, ent)
            ent["x"][:N].copy_(x.reshape(N, 3, H, W), non_blocking=x.is_cuda)
            ent["box"].copy_(_boxes(meta, N, torch.device("cpu")))
            ent["P"].copy_(Pm)
            ent["graph"].replay()
            self.logits = ent["logits"]
            X, status, inliers, resid = ent["tri"]
            J = X.shape[1]
            return {"world": X.cpu().numpy(), "kps": ent["kps"].cpu().numpy().reshape(T, V, J, 4),
                    "inliers": inliers.cpu().numpy(), "resid": resid.cpu().numpy(),
                    "status": status.cpu().numpy()}
