"""Per-conv-call timing table of one training step of the bench workload (CUDA events around
each conv call: ops.conv16_fprop / ops.conv16_wgrad of the split-fp16 engine, ops.conv_fprop /
ops.conv_wgrad of the fp32-operand one), next to each row's floor from its shapes.

    python tools/conv_table.py [tuples] [precision] [--peak-tflops P] [--hbm-tbs B]

Floor of a row = max(passes * 2MNK / peak, bytes / bandwidth), with passes = 3 for the split
precisions, and bytes = input + weights + output read once (fp16 hi/lo planes for the split
path, fp32 otherwise; the output is fp32 and read back too when it accumulates)."""
import argparse, os, sys, collections
os.environ.setdefault("EPB_OVERLAP_WGRAD", "0")   # serialise wgrad: clean per-call times
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "epipolarpose_b200"))
from oracle import refshim
from epipolarpose_b200 import ops
import lib.models as models, lib.core.integral_loss as il, lib.utils.utils as U

ap = argparse.ArgumentParser()
ap.add_argument("tuples", nargs="?", type=int, default=32)
ap.add_argument("prec", nargs="?", default="f16x3")
ap.add_argument("--peak-tflops", type=float, default=673.0,
                help="dense fp16 tensor rate (H100 SXM: 132 SMs x 4096 FLOP/clk at 1245 MHz)")
ap.add_argument("--hbm-tbs", type=float, default=3.0, help="HBM bandwidth in TB/s")
args = ap.parse_args()
tuples, prec = args.tuples, args.prec
passes = {"fp32": 1, "tf32": 1, "tf32x3": 3, "f16x3": 3}[prec]
J, D, HW, V = 16, 64, 256, 4
dev = torch.device("cuda:0")
cfg = refshim.make_cfg(num_layers=50, num_joints=J, volume=True, depth_res=D, image_size=(HW, HW))
torch.manual_seed(0)
model = models.pose3d_resnet.get_pose_net(cfg, False, precision=prec).to(dev).train()
crit = il.SmoothL1JointLocationLoss(J)
opt = U.FusedAdam(list(model.parameters()), lr=1e-3)
n = tuples * V
x = torch.randn(n, 3, HW, HW, device=dev)
lab = torch.rand(n, J * 3, device=dev) - 0.5
wt = torch.ones(n, J * 3, device=dev)
rec = []
orig = {f: getattr(ops, f) for f in ("conv_fprop", "conv_wgrad", "conv16_fprop", "conv16_wgrad")}
KIND = {"conv_fprop": "fprop", "conv_wgrad": "wgrad", "conv16_fprop": "fprop16", "conv16_wgrad": "wgrad16"}


def call_bytes(kind, g):
    ab = 4                                     # hi + lo fp16 planes, or one fp32 value
    M = g.N * g.Hp * g.Wp
    src, wts = g.N * g.Hi * g.Wi * g.Cin * ab, g.Cout * g.T * g.Cin * ab
    if kind.startswith("wgrad"):               # reads x and dout, writes dw (fp32)
        return src + M * g.Cout * ab + g.Cout * g.T * g.Cin * 4
    return src + wts + M * g.Cout * 4 * (2 if g.accumulate else 1)


def wrap(f, kind):
    def w(g, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); f(g, *a, **k); e1.record()
        M = g.N * g.Hp * g.Wp
        rec.append(((kind, M, g.Cin, g.Cout, g.T, g.os, g.is_, g.accumulate), call_bytes(kind, g), e0, e1))
    return w


def step():
    opt.zero_grad(); loss = crit(model(x), lab, wt); loss.backward(); opt.step(); return loss
step(); step(); torch.cuda.synchronize()
for f, fn in orig.items():
    setattr(ops, f, wrap(fn, KIND[f]))
t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
t0.record(); step(); t1.record(); torch.cuda.synchronize()
print("step %.2f ms (%s, %d images; floor: %.0f TFLOP/s, %.2f TB/s)"
      % (t0.elapsed_time(t1), prec, n, args.peak_tflops, args.hbm_tbs))
agg = collections.OrderedDict()
for key, by, e0, e1 in rec:
    a = agg.setdefault(key, [0, 0.0, 0]); a[0] += 1; a[1] += e0.elapsed_time(e1); a[2] += by
tot = sum(a[1] for a in agg.values())
print("conv total %.2f ms over %d calls" % (tot, len(rec)))
print("%-7s %8s %5s %5s %3s %2s %2s %3s %4s %8s %8s %8s %6s" % (
    "kind", "M", "Cin", "Cout", "T", "os", "is", "acc", "n", "ms", "TFLOP/s", "floor_ms", "floor%"))
tot_floor = 0.0
for (kind, M, ci, co, T, os_, is_, acc), (cnt, ms, by) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    fl = 2.0 * M * ci * co * T * cnt
    floor = max(passes * fl / (args.peak_tflops * 1e9), by / (args.hbm_tbs * 1e9))
    tot_floor += floor
    print("%-7s %8d %5d %5d %3d %2d %2d %3d %4d %8.3f %8.1f %8.3f %6.1f" % (
        kind, M, ci, co, T, os_, is_, acc, cnt, ms, fl / ms / 1e9, floor, 100.0 * floor / ms))
print("floor total %.2f ms (%.1f %% of the measured conv total)" % (tot_floor, 100.0 * tot_floor / tot))
