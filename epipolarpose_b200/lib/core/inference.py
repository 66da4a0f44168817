"""Hard-argmax keypoint decode -- host-side mirror of the reference
lib/core/inference.py:12-68 (`get_max_preds`, `get_final_preds`), with the
per-(n,j) argmax running in the warp-shuffle kernel epb_argmax2d (first-index
tie-break == numpy.argmax; indices are bit-exact).  numpy in / numpy out like
the reference; `get_max_preds_device` is the tensor-in / tensor-out variant.

Addition: `PosePredictor`, images -> 3-D joints as one CUDA-graph replay per call (the
`model.eval(); get_joint_location_result(W, H, model(img))` of demo.ipynb and scripts/valid.py).
`MultiViewPredictor`: the calibrated views of a rig -> world-frame joints, the same network on
every view followed by the robust V-view triangulation inside the same graph.
`RefinedPosePredictor`: images, boxes and cameras -> camera-frame poses and their refinement by the
paper's refinement unit, in one graph.
The MODEL.VOLUME = false head: `get_depth_preds` (reference :144-170), `get_heatmap_location_result`
and `HeatmapPredictor`, all on the fused decode epb_heatmap_decode (argmax, refinement, depth
soft-argmax, patch -> image)."""
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


RECT_3D_W = 2000.0                  # eval_integral's rect_3d_w: z (patch units) / patch_w * 2000 = mm


def heatmap_decode_device(heatmaps, depth, depth_res, box=None, patch_width=256, patch_height=256,
                          depth_range=2000.0, post_process=True, flip_pairs=None, shift_heatmap=False,
                          out=None):
    """The MODEL.VOLUME = false head's output -> joints on the device in one launch
    (epb_heatmap_decode).  heatmaps [B, J, H, W] float32 CUDA, either contiguous or the NCHW view of a
    channels-last [B, H, W, C] buffer (C >= J, as the split-fp16 final conv writes it: read in place);
    depth [B, J*depth_res] float32 rows.  box: [N, 6] float64 (c_x, c_y, width, height, scale, rot)
    for image coordinates, None for patch pixels.  flip_pairs: the batch is [x; flip(x)] (B = 2N) and
    each map / depth row is merged with its flipped-back mirror (shifted one column with
    shift_heatmap) before the decode.  -> kps [N, J, 4] float64 = (x, y, root-relative depth mm,
    maxval)."""
    from .integral_loss import flip_permutation
    B, J, H, W = heatmaps.shape
    N = B // 2 if flip_pairs is not None else B
    if flip_pairs is not None and B != 2 * N:
        raise ValueError("flip test needs a batch of 2N rows [x; flip(x)], got %d" % B)
    s = heatmaps.stride()
    if heatmaps.is_contiguous():
        layout, C, store = 0, J, heatmaps
    elif s[1] == 1 and s[3] >= J and s[2] == W * s[3] and s[0] == H * W * s[3]:
        C = s[3]
        layout = 1
        store = heatmaps.as_strided((B, H, W, C), (H * W * C, W * C, C, 1))
        if not store.is_contiguous():
            raise ValueError("channels-last heat-maps must be a dense [B, H, W, C] buffer")
    else:
        raise ValueError("heat-maps must be contiguous NCHW or an NCHW view of a channels-last buffer")
    if depth.dim() != 2 or depth.shape[0] != B or depth.shape[1] < J * depth_res or depth.stride(1) != 1 \
            or depth.stride(0) < J * depth_res:
        raise ValueError("expected depth rows [%d, >= %d], got %s" % (B, J * depth_res, tuple(depth.shape)))
    depth_store = depth.as_strided((B, depth.stride(0)), (depth.stride(0), 1))
    if out is None:
        out = torch.empty((N, J, 4), device=heatmaps.device, dtype=torch.float64)
    perm = flip_permutation(flip_pairs, J) if flip_pairs is not None else None
    _ops.heatmap_decode(store, layout, C, depth_store, depth.stride(0), box, N, J, H, W, depth_res,
                        patch_width, patch_height, depth_range, post_process, perm, bool(shift_heatmap), out)
    return out


def check_heatmap_head(net):
    """ValueError unless `net` is a MODEL.VOLUME = false network whose depth branch can run: depth_fc
    (reference pose3d_resnet.py:126, nn.Linear(2048, J*D)) reads the average-pooled trunk, which has
    2048 channels only for the bottleneck ResNets (50 and deeper).  A basic-block trunk (ResNet-18 / 34,
    512 channels) has no depth for the decode: the reference's forward fails there too, and the depth
    kernels would read past the trunk."""
    plan = net._plan
    if plan.fc is None:
        raise ValueError("the heat-map decode needs the MODEL.VOLUME: false head; for a VOLUME model use "
                         "PosePredictor / the soft-argmax")
    if plan.trunk_channels != plan.fc.cin:
        raise ValueError("MODEL.VOLUME: false needs a %d-channel trunk for depth_fc (ResNet-50 or deeper); this "
                         "network's trunk has %d channels" % (plan.fc.cin, plan.trunk_channels))


def get_depth_preds(cfg, pred):
    """reference :144-166: depth logits [N, J*D] (numpy) -> root-relative depth [N, J] float64 in mm,
    the soft-argmax d = (s / D - 0.5) * DATASET.DEPTH_RANGE (computed with the maximum subtracted, so
    logits above ~88, where the reference's exp overflows, still decode)."""
    J, D = int(cfg.MODEL.NUM_JOINTS), int(cfg.MODEL.DEPTH_RES)
    p = np.ascontiguousarray(np.asarray(pred, dtype=np.float32).reshape(-1, J * D))
    N = p.shape[0]
    if N == 0:
        return np.zeros((0, J))
    dev = torch.device("cuda")
    hm = torch.zeros((N, J, 1, 1), device=dev, dtype=torch.float32)      # the 2-D half has one pixel
    kps = heatmap_decode_device(hm, torch.from_numpy(p).to(dev), D, depth_range=float(cfg.DATASET.DEPTH_RANGE),
                                post_process=False)
    return kps[:, :, 2].cpu().numpy()


def heatmap_rows(kps, patch_width):
    """kps [N, J, 4] (patch px, mm, maxval) -> validate_integral's rows: z in patch units."""
    out = np.asarray(kps, dtype=np.float64).copy()
    out[:, :, 2] = out[:, :, 2] / RECT_3D_W * patch_width
    return out


def get_heatmap_location_result(patch_width, patch_height, preds, depth_res=None, depth_range=None,
                                post_process=None, flip_pairs=None, shift_heatmap=False):
    """The MODEL.VOLUME = false counterpart of get_joint_location_result: preds = (heatmaps [N, J, h, w],
    depth [N, J*D]) -> numpy float64 [N, J, 4] in validate_integral's units: x, y in patch pixels,
    z in patch units (eval_integral's z / patch_width * 2000 is the root-relative depth in mm) and
    the heat-map maximum as score.  depth_res, depth_range and post_process default to the
    config's MODEL.DEPTH_RES, DATASET.DEPTH_RANGE and TEST.POST_PROCESS; flip_pairs / shift_heatmap
    as heatmap_decode_device."""
    from .config import config
    hm, depth = preds
    D = int(config.MODEL.DEPTH_RES if depth_res is None else depth_res)
    rng = float(config.DATASET.DEPTH_RANGE if depth_range is None else depth_range)
    pp = bool(config.TEST.POST_PROCESS) if post_process is None else bool(post_process)
    kps = heatmap_decode_device(hm, depth, D, None, patch_width, patch_height, rng, pp, flip_pairs, shift_heatmap)
    return heatmap_rows(kps.cpu().numpy(), patch_width)


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


class RefinedPosePredictor(PosePredictor):
    """Images -> refined camera-frame 3-D poses, one CUDA-graph replay per (N, H, W): the
    PosePredictor graph (network, soft-argmax, patch -> image), then epb_pose_to_camera (the
    root-relative camera-frame pose, bit-identical to the `pred` column of the H36M evaluation) and
    epb_refiner_forward (refiner.model.Refiner: the hip dropped, the second head denormalised, the
    hip put back at 0).

    refiner: a refiner.model.LinearModelPG; norm: (data_mean, data_std, labels_mean, labels_std) of
    its norm.pkl.  Both the network and the refiner are snapshots: refresh() re-reads both.
    pred(images, boxes, cams): images float32 [N, 3, H, W]; boxes as PosePredictor; cams holds, per
    image, fl [N, 2], c_p [N, 2] and the root (pelvis) depth `depth` [N] in mm, which must be given
    as in the H36M protocol (it is not estimated).  Returns a dict of numpy arrays:
      kps     [N, 16, 4] float64  PosePredictor's output with boxes (image x, y, root-relative z, 1)
      pose    [N, 16, 3] float64  camera-frame mm, root-relative (MPII order, root = joint 6)
      refined [N, 16, 3] float32  the refiner's output, hip at 0
    Constructor refusals: those of PosePredictor, and a network of other than 16 joints."""

    ROOT = 6

    def __init__(self, model, refiner, norm, flip_test=None, shift_heatmap=None, flip_pairs=None):
        from refiner.model import Refiner
        net = getattr(model, "module", model)
        super().__init__(model, flip_test, shift_heatmap, flip_pairs)
        if net._plan.num_joints != 16:
            raise ValueError("RefinedPosePredictor refines 16-joint poses in MPII order, the network has %d "
                             "joints" % net._plan.num_joints)
        self.refiner = Refiner(refiner, norm, device=self.dev)

    def refresh(self):
        super().refresh()
        if getattr(self, "refiner", None) is not None:
            self.refiner.refresh()

    def _forward(self, ent):
        super()._forward(ent)
        N = ent["box"].shape[0]
        kps = ent["kps"][:, :, :3].contiguous()
        _ops.pose_to_camera(kps, ent["cam"], N, 16, self.ROOT, ent["pose"])
        if "ws" not in ent:                 # allocated by the warm-up run, before the capture
            ent["ws"] = self.refiner.workspace(N)
        ent["refined"] = self.refiner.refine(ent["pose"], ws=ent["ws"])

    def __call__(self, images, boxes=None, cams=None):
        if boxes is None or cams is None:
            raise ValueError("RefinedPosePredictor needs the boxes and the cameras (fl, c_p, depth) of every image")
        x = torch.as_tensor(images)
        if x.dim() != 4 or x.shape[1] != 3:
            raise ValueError("expected images [N, 3, H, W], got %s" % (tuple(x.shape),))
        if x.dtype != torch.float32:
            raise TypeError("expected float32 images, got %s" % x.dtype)
        N, _, H, W = x.shape
        fl = np.asarray(cams["fl"], dtype=np.float64).reshape(N, -1)[:, :2]
        cp = np.asarray(cams["c_p"], dtype=np.float64).reshape(N, -1)[:, :2]
        depth = np.asarray(cams["depth"], dtype=np.float64).reshape(N, 1)
        cam = torch.from_numpy(np.ascontiguousarray(np.concatenate([fl, cp, depth], axis=1)))
        from ..utils.img_utils import _boxes
        meta = dict(boxes)
        meta.setdefault("scale", np.ones(N))
        meta.setdefault("rot", np.zeros(N))
        with torch.cuda.device(self.dev):
            key = (N, H, W)
            ent = self.graphs.get(key)
            if ent is None:
                B = 2 * N if self.flip_test else N
                ent = {"x": torch.zeros((B, 3, H, W), device=self.dev),
                       "box": _boxes(meta, N, torch.device("cpu")).to(self.dev),
                       "cam": cam.to(self.dev),
                       "pose": torch.empty((N, 16, 3), device=self.dev, dtype=torch.float64)}
                self._record(key, ent)
            ent["x"][:N].copy_(x, non_blocking=x.is_cuda)
            ent["box"].copy_(_boxes(meta, N, torch.device("cpu")))
            ent["cam"].copy_(cam)
            ent["graph"].replay()
            self.logits = ent["logits"]
            kps = np.ones((N, 16, 4), dtype=np.float64)
            kps[:, :, :3] = ent["kps"][:, :, :3].cpu().numpy()
            return {"kps": kps, "pose": ent["pose"].cpu().numpy(), "refined": ent["refined"].cpu().numpy()}


class HeatmapPredictor(PosePredictor):
    """Images -> joints for the MODEL.VOLUME = false head (2-D heat-maps + depth_fc logits), one
    CUDA-graph replay per (N, H, W): the prepared split-fp16 network (its depth branch on the
    average-pooled trunk) and epb_heatmap_decode (argmax, the get_final_preds refinement,
    get_depth_preds, patch -> image).  Snapshot, refresh() and eval-BatchNorm semantics as
    PosePredictor.

    pred(images): images float32 [N, 3, H, W] (host or device) -> numpy float64 [N, J, 4], the rows
    of get_heatmap_location_result(W, H, model.eval()(images)): x, y in patch pixels, z in patch
    units (z / W * 2000 = root-relative depth in mm) and the heat-map maximum.  pred(images,
    boxes=meta): meta as PosePredictor; rows (image x, image y, root-relative depth mm, maxval).
    flip_test / shift_heatmap / flip_pairs as PosePredictor (the 2N batch [x; flip(x)], merged inside
    the decode); post_process defaults to config.TEST.POST_PROCESS.
    pred.heatmaps [N or 2N, J, h, w] (an NCHW view of the channels-last buffer) and pred.depth
    [N or 2N, J*D]: the static outputs of the last call, overwritten by the next call with the same N."""

    def __init__(self, model, flip_test=None, shift_heatmap=None, flip_pairs=None, post_process=None):
        from .config import config
        from .integral_loss import flip_permutation
        net = getattr(model, "module", model)
        if getattr(net, "volume", True):
            raise ValueError("HeatmapPredictor decodes the 2-D heat-map head (MODEL.VOLUME: false); "
                             "for a VOLUME model use PosePredictor")
        if getattr(net, "precision", None) != 4:
            raise ValueError("HeatmapPredictor runs the split-fp16 engine (MODEL.PRECISION: f16x3); "
                             "this model runs another precision")
        if not _net16.supported(net._plan):
            raise ValueError("HeatmapPredictor runs the split-fp16 engine, which needs every layer's "
                             "channels in whole 64-channel blocks; this model's plan has others")
        check_heatmap_head(net)
        self.flip_test = bool(config.TEST.FLIP_TEST) if flip_test is None else bool(flip_test)
        self.shift_heatmap = bool(config.TEST.SHIFT_HEATMAP) if shift_heatmap is None \
            else bool(shift_heatmap)
        self.post_process = bool(config.TEST.POST_PROCESS) if post_process is None else bool(post_process)
        if self.flip_test:
            if flip_pairs is None:
                raise ValueError("flip test needs the dataset's joint pairs (flip_pairs)")
            flip_permutation(flip_pairs, net._plan.num_joints)
        self.flip_pairs = flip_pairs
        self.depth_range = float(config.DATASET.DEPTH_RANGE)
        self.model = net
        self.dev = next(net.parameters()).device
        self.eng = _net16.Engine16(net._plan, ops=net._ops)
        self.stream = torch.cuda.Stream(self.dev)
        self.graphs = {}
        self.state = None
        self.logits = None
        self.heatmaps = None
        self.depth = None
        self.refresh()

    def _forward(self, ent):
        """The captured work: [flip,] network, heat-map decode."""
        x, box = ent["x"], ent["box"]
        N, H, W = box.shape[0], x.shape[2], x.shape[3]
        if self.flip_test:
            x[N:] = torch.flip(x[:N], [3])
        logits, depth, _ = self.eng.forward(x, None, training=False, save=False, prepared=self.state)
        plan = self.eng.plan
        hm = logits.permute(0, 3, 1, 2)[:, :plan.final.cout]
        depth = depth.reshape(depth.shape[0], -1)
        if "kps" not in ent:
            ent["kps"] = torch.empty((N, plan.num_joints, 4), device=self.dev, dtype=torch.float64)
        heatmap_decode_device(hm, depth, plan.depth_res, box, W, H, self.depth_range, self.post_process,
                              self.flip_pairs if self.flip_test else None, self.shift_heatmap, out=ent["kps"])
        ent["heatmaps"], ent["depth"] = hm, depth

    def _capture(self, N, H, W):
        ent = super()._capture(N, H, W)
        ent["box0"] = ent["box"].clone()            # the identity box: image frame = patch frame
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
            if boxes is None:
                ent["box"].copy_(ent["box0"])
            else:
                from ..utils.img_utils import _boxes
                meta = dict(boxes)
                meta.setdefault("scale", np.ones(N))
                meta.setdefault("rot", np.zeros(N))
                ent["box"].copy_(_boxes(meta, N, torch.device("cpu")))
            ent["graph"].replay()
            self.heatmaps, self.depth = ent["heatmaps"], ent["depth"]
            kps = ent["kps"].cpu().numpy()
            return heatmap_rows(kps, W) if boxes is None else kps
