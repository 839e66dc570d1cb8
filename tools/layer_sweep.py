"""Per-layer timing of the conv kernels for one BASELINE model (CUDA events, warm, L2 flushed between reps).  The weight gradient
is timed on both entry points: `wgrad` (b2c_conv_backward_filter) and `wsplit` (b2c_conv_backward_filter_split, split pass
included); the `pre` column says whether the latter splits dY first."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi
from caffe_mpi_b200.shapes import MODELS

model = sys.argv[1] if len(sys.argv) > 1 else "resnet50"
N = int(sys.argv[2]) if len(sys.argv) > 2 else 64
math = capi.MATH_TF32 if (len(sys.argv) > 3 and sys.argv[3] == "tf32") else capi.MATH_FP32
reps = 5
only = os.environ.get("B2C_SWEEP_ONLY", "").split()      # e.g. "k1 s2": keep layers whose label contains every token
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
tot = {"fwd": 0.0, "dgrad": 0.0, "wgrad": 0.0, "wsplit": 0.0}
print(f"{'layer':34s} {'op':6s} {'us':>9s} {'TF/s':>7s} {'GB/s(alg)':>10s} {'hbm_us':>7s} {'mma_us':>7s} {'pre':>5s}")
first = True
for (cnt, C, H, O, k, s, p, G, bias) in MODELS[model]:
    label = f"C{C} H{H} O{O} k{k} s{s} g{G}"
    if any(tok not in label.split() for tok in only):
        first = False
        continue
    prm = capi.ConvParams.make(N, C, H, H, O, k, s, p, 1, G, bias)
    d = m.ConvDesc(prm, capi.ENGINE_DEFAULT, math=math)
    x = torch.randn(prm.x_shape(), device="cuda"); w = torch.randn(prm.w_shape(), device="cuda") * 0.05
    b = torch.zeros(O, device="cuda") if bias else None
    y = torch.empty(prm.y_shape(), device="cuda"); dy = torch.randn(prm.y_shape(), device="cuda")
    dx = torch.empty_like(x); dw = torch.zeros_like(w)
    ops = [("fwd", lambda: d.forward(x, w, b, y))]
    if not first:
        ops.append(("dgrad", lambda: d.backward_data(dy, w, dx)))
    ops.append(("wgrad", lambda: d.backward_filter(x, dy, dw)))
    ops.append(("wsplit", lambda: d.backward_filter_split(x, dy, dw)))
    q = d.wgrad_plan()
    pre = "dY" if q["presplit_dy"] else "-"
    first = False
    fl = prm.flops()
    byts = 4 * (x.numel() + w.numel() + y.numel())
    for name, fn in ops:
        fn(); fn()
        ts = []
        for _ in range(reps):
            flush.zero_()
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); e.record(); torch.cuda.synchronize()
            ts.append(a.elapsed_time(e) * 1e3)
        us = sorted(ts)[len(ts) // 2]
        tot[name] += us * cnt
        mma_us = fl * (3 if math == capi.MATH_FP32 else 1) / 847.5e12 * 1e6
        print(f"{cnt}x C{C} H{H} O{O} k{k} s{s} g{G:<12d} {name:6s} {us:9.1f} {fl/us/1e6:7.1f} {byts/us/1e3:10.0f} {byts/6578e9*1e6:7.1f} {mma_us:7.1f} {pre if name == 'wsplit' else '':>5s}", flush=True)
print("totals (us, weighted by layer count):", {k: round(v) for k, v in tot.items()}, "sum", round(sum(tot.values())))
