"""Refiner network -- host-side mirror of the reference refiner/model.py surface
(weight_init :8-12, LinearPG :15-68, LinearModelPG :71-143, get_model :146-150): same class names,
constructor arguments, state_dict keys / shapes / default initialisation (the sub-modules are
torch.nn.Linear / BatchNorm1d objects used as PARAMETER CONTAINERS only), same forward signature
`model(x [N, input_size]) -> (p1, p2)`.  The arithmetic runs through epipolarpose_b200.mlp.MLPEngine
on the libepb.so kernels (SURVEY.md section 8(f) row 4).  Not built: leaky=True, bn=False.

Addition: `Refiner`, the eval-mode forward of a LinearModelPG snapshot as one C-ABI call
(epb_refiner_forward), for refining poses outside the training loop."""
import numpy as np
import torch
import torch.nn as nn

from epipolarpose_b200 import mlp as _mlp


def weight_init(m):
    if isinstance(m, nn.Linear):
        nn.init.kaiming_normal_(m.weight)


class LinearPG(nn.Module):
    """Parameter container of one residual stage (reference :15-37); evaluated by LinearModelPG."""

    def __init__(self, linear_size, p_dropout=0.5, bias=True, bn=True, leaky=False):
        super().__init__()
        if leaky or not bn or not bias:
            raise NotImplementedError("refiner stages are built for bias=True, bn=True, leaky=False")
        self.l_size, self.bn, self.leaky = linear_size, bn, leaky
        for i in (1, 2, 3, 4):
            setattr(self, "w%d" % i, nn.Linear(linear_size, linear_size, bias=bias))
        for i in (1, 2, 3, 4):
            setattr(self, "batch_norm%d" % i, nn.BatchNorm1d(linear_size))

    def forward(self, x):
        raise RuntimeError("LinearPG is evaluated inside LinearModelPG (one fused graph)")


class _RefinerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, x, *params):
        names = module._param_names
        p = dict(zip(names, params))
        p.update(module._buffers_flat())
        eng = module._engine()
        need = any(ctx.needs_input_grad)
        with torch.no_grad():
            p1, p2, record = eng.forward(x.contiguous().float(), p, module.training, module.p_dropout,
                                         want_grad=need)
        ctx.module, ctx.record = module, record
        return p1.clone(), p2.clone()

    @staticmethod
    def backward(ctx, dp1, dp2):
        module = ctx.module
        c = lambda d: None if d is None else d.contiguous()
        with torch.no_grad():
            dx, pg = module._engine().backward(ctx.record, c(dp1), c(dp2))
        return (None, dx) + tuple(pg.get(n) for n in module._param_names)


class LinearModelPG(nn.Module):
    def __init__(self, linear_size=1024, num_stage=2, p_dropout=0.5, input_size=15 * 3,
                 output_size=15 * 3, bias=True, bn=True, leaky=False, precision="tf32x3"):
        super().__init__()
        if leaky or not bn or not bias or num_stage != 2:
            raise NotImplementedError("refiner is built for num_stage=2, bias=True, bn=True, leaky=False")
        if linear_size % 4:
            raise ValueError("linear_size must be a multiple of 4")
        self.linear_size, self.bn, self.leaky = linear_size, bn, leaky
        self.p_dropout, self.num_stage = p_dropout, num_stage
        self.input_size, self.output_size = input_size, output_size
        self.linear_stages = nn.ModuleList([LinearPG(linear_size, p_dropout, bias=bias, bn=bn, leaky=leaky)
                                            for _ in range(num_stage)])
        self.w1 = nn.Linear(input_size, linear_size, bias=bias)
        self.w2 = nn.Linear(linear_size, output_size, bias=bias)
        self.w3 = nn.Linear(output_size, linear_size, bias=bias)
        self.w4 = nn.Linear(linear_size, output_size, bias=bias)
        self.batch_norm1 = nn.BatchNorm1d(linear_size)
        self.batch_norm3 = nn.BatchNorm1d(linear_size)
        self._precision = {"fp32": 0, "tf32": 1, "tf32x3": 3}[precision]
        self._param_names = [n for n, _ in self.named_parameters()]
        self._eng = None

    _backend = [None]      # test hook: an ops module emulating the C ABI on the CPU

    def _engine(self):
        if self._eng is None:
            self._eng = _mlp.MLPEngine(self._precision, ops=self._backend[0])
        return self._eng

    def _buffers_flat(self):
        return dict(self.named_buffers())

    def forward(self, x):
        params = [p for _, p in self.named_parameters()]
        return _RefinerFn.apply(self, x, *params)


# LinearModelPG's linear layers and BatchNorms in the order epb_refiner_prepare takes them
_LAYERS = (["w1"] + ["linear_stages.0.w%d" % i for i in (1, 2, 3, 4)] + ["w2", "w3"] +
           ["linear_stages.1.w%d" % i for i in (1, 2, 3, 4)] + ["w4"])
_BNS = (["batch_norm1"] + ["linear_stages.0.batch_norm%d" % i for i in (1, 2, 3, 4)] + ["batch_norm3"] +
        ["linear_stages.1.batch_norm%d" % i for i in (1, 2, 3, 4)])


class Refiner:
    """Eval-mode refinement with a LinearModelPG: the second head, with dropout the identity and
    BatchNorm on its running statistics, as `model.eval()(x)[1]`.  One epb_refiner_forward call
    per chunk of rows: 12 launches, fp32 FMAs accumulated in input order by one thread per output,
    so each pose's result does not depend on the batch it is refined in.

    Snapshot semantics, as PosePredictor: the weights, the running statistics and `norm` are read
    when the refiner is built and again by refresh(), never in between.

    norm = (data_mean, data_std, labels_mean, labels_std) of norm.pkl (refiner/data.py): inputs are
    normalised and outputs denormalised with them.

    refine(poses): [N, 16, 3] root-relative camera-frame mm in MPII order (the `pred` of the H36M
    evaluation) -> [N, 16, 3] float32: the hip (joint 6) is dropped on the way in and put back at 0,
    as the refiner's training data are.  A torch tensor gives a tensor on the refiner's device,
    anything else a numpy array."""

    HIP = 6
    CHUNK = 8192            # rows per call (the workspace is 4 * linear_size + 48 floats per row)

    def __init__(self, model, norm, device=None):
        from epipolarpose_b200 import ops
        net = getattr(model, "module", model)
        if not isinstance(net, LinearModelPG):
            raise TypeError("Refiner takes a refiner.model.LinearModelPG")
        self.ops = ops
        self.model = net
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.in_size, self.L, self.out_size = net.input_size, net.linear_size, net.output_size
        self._norm_src = norm
        self._ws = None
        self._keep = torch.tensor([j for j in range(16) if j != self.HIP], device=self.device)
        npar, _ = ops.refiner_sizes(self.in_size, self.L, self.out_size, 0)
        self.params = torch.empty(npar, device=self.device)
        self.refresh()

    def refresh(self, norm=None):
        """Re-read the model's parameters and running statistics (and `norm`, if given)."""
        if norm is not None:
            self._norm_src = norm
        if self._norm_src is None:
            norm = (np.zeros(self.in_size), np.ones(self.in_size), np.zeros(self.out_size), np.ones(self.out_size))
        else:
            norm = self._norm_src
        dev = self.device
        f32 = lambda t: (t.detach() if torch.is_tensor(t) else torch.as_tensor(np.asarray(t))).to(
            dev, torch.float32).reshape(-1).contiguous()
        sd = self.model.state_dict()
        src = []
        for n in _LAYERS:
            src += [f32(sd[n + ".weight"]), f32(sd[n + ".bias"])]
        for n in _BNS:
            src += [f32(sd[n + "." + k]) for k in ("weight", "bias", "running_mean", "running_var")]
        src += [f32(a) for a in norm]
        sizes = (self.in_size, self.in_size, self.out_size, self.out_size)
        if any(t.numel() != c for t, c in zip(src[-4:], sizes)):
            raise ValueError("norm arrays must have %d, %d, %d, %d entries" % sizes)
        eps = self.model.batch_norm1.eps
        with torch.cuda.device(dev):
            self.ops.refiner_prepare(self.in_size, self.L, self.out_size, src, eps, self.params)
            torch.cuda.current_stream().synchronize()       # the sources are temporaries
        return self

    def _workspace(self, n):
        _, nws = self.ops.refiner_sizes(self.in_size, self.L, self.out_size, n)
        if self._ws is None or self._ws.numel() < nws:
            self._ws = torch.empty(nws, device=self.device)
        return self._ws

    def forward(self, x, out=None, normalize=True, denormalize=True, force_form=0, ws=None):
        """x [N, in] float32 on the device -> [N, out]: the second head of the snapshot, on x
        normalised with data_mean / data_std (normalize) and denormalised with labels_mean /
        labels_std (denormalize).  ws: a workspace of the caller's (a captured graph keeps its
        own); by default the refiner's, grown as needed."""
        x = x.contiguous()
        N = x.shape[0]
        if x.dim() != 2 or x.shape[1] != self.in_size:
            raise ValueError("expected [N, %d] inputs, got %s" % (self.in_size, tuple(x.shape)))
        if out is None:
            out = torch.empty((N, self.out_size), device=self.device)
        elif tuple(out.shape) != (N, self.out_size) or not out.is_contiguous():
            raise ValueError("out must be a contiguous [%d, %d] tensor, got %s" % (N, self.out_size, tuple(out.shape)))
        with torch.cuda.device(self.device):
            for s in range(0, N, self.CHUNK):
                n = min(self.CHUNK, N - s)
                self.ops.refiner_forward(self.in_size, self.L, self.out_size, self.params, x[s:s + n], n,
                                         normalize, denormalize, out[s:s + n],
                                         self._workspace(n) if ws is None else ws, force_form)
        return out

    def workspace(self, N):
        """A workspace for forward() over up to min(N, CHUNK) rows."""
        return torch.empty(self.ops.refiner_sizes(self.in_size, self.L, self.out_size, min(N, self.CHUNK))[1],
                           device=self.device)

    def refine(self, poses, ws=None):
        as_tensor = torch.is_tensor(poses)
        p = poses if as_tensor else torch.as_tensor(np.asarray(poses))
        if p.dim() != 3 or p.shape[1] != 16 or p.shape[2] != 3 or self.in_size != 45 or self.out_size != 45:
            raise ValueError("refine takes [N, 16, 3] poses and a refiner of 45 inputs and outputs")
        keep = self._keep
        x = p.to(self.device, torch.float32).index_select(1, keep).reshape(-1, 45)
        y = self.forward(x, ws=ws)
        out = torch.zeros((p.shape[0], 16, 3), device=self.device)
        out.index_copy_(1, keep, y.reshape(-1, 15, 3))
        return out if as_tensor else out.cpu().numpy()


def get_model(weights, **kwargs):
    model = LinearModelPG(**kwargs)
    if weights:
        model.load_state_dict(torch.load(weights)['state_dict'])
    return model
