"""Forward / backward engine of the refiner MLP (reference refiner/model.py) over the libepb.so
kernels: every nn.Linear is the 1x1 case of the tap-list implicit GEMM (wgmma path for the
1024-wide layers, CUDA-core path for the 45-wide ends), BatchNorm1d + ReLU are the BatchNorm
kernels of the CNN on [N][C] rows (statistics from the GEMM epilogue), dropout and the residual
sums are the two element-wise kernels epb_mask_scale / epb_add3.  torch only owns memory and
draws the dropout keep masks.

The network is a fixed graph, recorded on a small tape: each forward helper pushes the closure that
turns the gradient of its output into gradients of its inputs / parameters."""
import torch

from . import net, ops as _default_ops

BN_MOMENTUM = 0.1    # torch.nn.BatchNorm1d defaults used by the reference
BN_EPS = 1e-5


class MLPEngine:
    def __init__(self, precision=3, ops=None):
        self.ops = ops or _default_ops
        self.eng = net.Engine(None, precision=precision, ops=self.ops)
        self._convs = {}

    # ---- helpers ---------------------------------------------------------------------------
    def _conv(self, name, cin, cout):
        key = (name, cin, cout)
        if key not in self._convs:
            self._convs[key] = net.Conv(name, "conv", cin, cout, 1, 1, 0, bias=True)
        return self._convs[key]

    def _new(self, *shape, dtype=torch.float32):
        return torch.empty(shape, device=self.dev, dtype=dtype)

    def _acc(self, grads, t, g):
        k = id(t)
        if k in grads:
            s = torch.empty_like(g)
            self.ops.add3(grads[k], g, None, s, g.numel())
            grads[k] = s
        else:
            grads[k] = g

    # ---- forward ops (each records its backward on self.tape) ---------------------------------
    def linear(self, name, x, params, pgrads):
        """y = x W^T + b; x [N][cin_p] (zero padded), returns [N][cout_p]."""
        ops, eng = self.ops, self.eng
        w, b = params[name + ".weight"], params[name + ".bias"]
        cout, cin = w.shape
        conv = self._conv(name, cin, cout)
        N = x.shape[0]
        wf, wd = conv.pack(ops, w.reshape(cout, cin, 1, 1))
        bp = b
        if conv.cout_p != cout:
            bp = torch.zeros(conv.cout_p, device=self.dev)
            bp[:cout] = b
        stats = torch.zeros(2 * conv.cout_p, device=self.dev, dtype=torch.float64)
        y, _, _ = eng._conv_fwd(conv, x, N, 1, 1, wf, bias=bp, stats=stats)
        y = y.reshape(N, conv.cout_p)

        def bwd(grads):
            dy = grads.pop(id(y)).contiguous()
            if pgrads is not None:
                gw = torch.zeros_like(w).reshape(cout, cin, 1, 1)
                eng._conv_wgrad(conv, x.reshape(N, 1, 1, -1), dy.reshape(N, 1, 1, -1), N, 1, 1, gw)
                pgrads[name + ".weight"] = gw.reshape(cout, cin)
                gb = torch.empty(conv.cout_p, device=self.dev)
                ops.colsum(dy, N, conv.cout_p, gb)
                pgrads[name + ".bias"] = gb[:cout].clone()
            dx = eng._conv_dgrad(conv, dy.reshape(N, 1, 1, -1), N, 1, 1, wd).reshape(N, conv.cin_p)
            self._acc(grads, x, dx)
        self.tape.append(bwd)
        return y, stats

    def bn_relu(self, name, z, stats, params, pgrads, training):
        """relu(BatchNorm1d(z)); statistics come from the producing GEMM's epilogue."""
        ops, eng = self.ops, self.eng
        N, C = z.shape
        c_real = params[name + ".weight"].shape[0]
        p = params
        if C != c_real:                       # padded columns: gamma 1 / beta 0 / stats untouched
            raise ValueError("BatchNorm1d width %d must be a multiple of 4" % c_real)
        if training and N == 1:
            # torch.nn.BatchNorm1d refuses a one-row training batch (the reference's loop stops on
            # a last batch of 1); bn_finalize would map it to a zero variance and every output to beta
            raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                             % (tuple(z.shape),))
        st = eng._bn_train(name, C, stats, N, p, None) if training else eng._bn_eval(name, C, p)
        a = torch.empty_like(z)
        ops.bn_act(z, st.scale, st.shift, None, None, None, 1, a, N, C)

        def bwd(grads):
            da = grads.pop(id(a)).contiguous()
            if not training:
                raise RuntimeError("backward through an eval-mode BatchNorm is not built")
            g = {name + ".weight": torch.empty(C, device=self.dev), name + ".bias": torch.empty(C, device=self.dev)}
            dz = eng._bn_bwd(st, da, z, None, 1, p, g)
            if pgrads is not None:
                pgrads.update(g)
            self._acc(grads, z, dz)
        self.tape.append(bwd)
        return a

    def dropout(self, x, p, training):
        if not training or p <= 0.0:
            return x
        ops = self.ops
        keep = (torch.rand(x.shape, device=self.dev) >= p).to(torch.uint8)
        scale = 1.0 / (1.0 - p)
        y = torch.empty_like(x)
        ops.mask_scale(x, keep, scale, y, x.numel())

        def bwd(grads):
            dy = grads.pop(id(y)).contiguous()
            dx = torch.empty_like(dy)
            ops.mask_scale(dy, keep, scale, dx, dy.numel())
            self._acc(grads, x, dx)
        self.tape.append(bwd)
        return y

    def add(self, a, b, c=None):
        out = torch.empty_like(a)
        self.ops.add3(a, b, c, out, a.numel())

        def bwd(grads):
            g = grads.pop(id(out))
            for t in (a, b, c):
                if t is not None:
                    self._acc(grads, t, g)
        self.tape.append(bwd)
        return out

    # ---- the reference graph (refiner/model.py:39-68 and :117-143) --------------------------------
    def _block(self, prefix, x, params, pgrads, training, pdrop, i):
        y, st = self.linear("%s.w%d" % (prefix, i), x, params, pgrads)
        y = self.bn_relu("%s.batch_norm%d" % (prefix, i), y, st, params, pgrads, training)
        return self.dropout(y, pdrop, training)

    def _stage(self, prefix, x, params, pgrads, training, pdrop):
        y = self._block(prefix, x, params, pgrads, training, pdrop, 1)
        y = self._block(prefix, y, params, pgrads, training, pdrop, 2)
        out = self.add(x, y)
        y = self._block(prefix, out, params, pgrads, training, pdrop, 3)
        y = self._block(prefix, y, params, pgrads, training, pdrop, 4)
        return self.add(out, y)

    def forward(self, x, params, training, pdrop, want_grad=True):
        """x [N, input_size] float32 -> (p1, p2) [N, output_size]; records the tape."""
        self.dev = x.device
        self.eng.dev = x.device
        self.tape = []
        self.pgrads = {} if want_grad else None
        pg = self.pgrads
        N, cin = x.shape
        cin_p = (cin + 3) // 4 * 4
        xp = x
        if cin_p != cin:
            xp = torch.zeros((N, cin_p), device=self.dev)
            xp[:, :cin] = x
        y, st = self.linear("w1", xp.contiguous(), params, pg)
        y = self.bn_relu("batch_norm1", y, st, params, pg, training)
        inp = self.dropout(y, pdrop, training)
        s1 = self._stage("linear_stages.0", inp, params, pg, training, pdrop)
        p1, _ = self.linear("w2", s1, params, pg)
        y, st = self.linear("w3", p1, params, pg)
        y = self.bn_relu("batch_norm3", y, st, params, pg, training)
        y = self.dropout(y, pdrop, training)
        y = self.add(s1, y, inp)
        y = self._stage("linear_stages.1", y, params, pg, training, pdrop)
        y = self.add(inp, y)
        p2, _ = self.linear("w4", y, params, pg)
        cout = params["w2.weight"].shape[0]
        # everything the backward needs travels in `record` (several forwards may be alive at once)
        record = {"tape": self.tape, "pgrads": self.pgrads, "outs": (p1, p2), "x_in": xp, "cin": cin}
        self.tape, self.pgrads = [], None
        return p1[:, :cout], p2[:, :cout], record

    def backward(self, record, dp1, dp2):
        """dp1, dp2 [N, output_size] (or None) -> (dx [N, input_size], {param name: grad})."""
        self.dev = record["x_in"].device
        self.eng.dev = self.dev
        grads = {}
        for t, d in zip(record["outs"], (dp1, dp2)):
            g = torch.zeros_like(t)
            if d is not None:
                g[:, :d.shape[1]] = d
            grads[id(t)] = g
        for bwd in reversed(record["tape"]):
            bwd(grads)
        dx = grads.pop(id(record["x_in"]))[:, :record["cin"]]
        record["tape"] = []
        return dx, record["pgrads"]
