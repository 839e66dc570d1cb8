"""Transposed-convolution kernels on the GPU: the phase route against the FFMA data-gradient kernels it replaces, and the depthwise
upsampler against the HBM bound.

  python tools/deconv_bench.py [--reps 5] [--iters 10] [--out DIR]

Phase route: the forward of the DCGAN generator's 4x4 / stride 2 / pad 1 layers at batch 64 (b2c_deconv_forward, fp32 math)
against the same product on the FFMA kernels (b2c_conv_backward_data of the dual convolution with ALGO_SIMT), the route such a
layer took before the phase route existed.  Depthwise upsampler: FCN's 64 / 32 bilinear layer (21 channels) and a 4 / 2 one,
forward, data gradient and weight gradient, in GB/s of compulsory traffic (bottom read once, top written once) over 3.35 TB/s, the H100 SXM data-sheet HBM3
bandwidth.  Each number is the median of --reps alternated repetitions of --iters launches timed with CUDA events.  Prints one
JSON line, with the device name and power limit, and writes it to DIR/deconv_bench.json when --out is given.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12

# (name, N, C_in, H, num_output): the generator of DCGAN (Radford et al. 2016) at 64 x 64 output, 4x4 / 2 / pad 1
DCGAN = [("g1 1024->512 4->8", 64, 1024, 4, 512), ("g2 512->256 8->16", 64, 512, 8, 256),
         ("g3 256->128 16->32", 64, 256, 16, 128), ("g4 128->3 32->64", 64, 128, 32, 3)]
# (name, N, C, H, k, s, p)
UPSAMPLERS = [("fcn32 64/32", 8, 21, 16, 64, 32, 16), ("x2 4/2", 32, 64, 64, 4, 2, 1)]


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def device_info():
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        info["power_limit_and_max_sm_clock"] = q[0] if q else "unknown"
    except Exception:  # nvidia-smi missing: say so rather than guess
        info["power_limit_and_max_sm_clock"] = "unknown"
    return info


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("deconv_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    rng = np.random.default_rng(1701)
    res = dict(device_info(), phase=[], depthwise=[])
    for name, N, Cin, H, O in DCGAN:
        p = m.ConvParams.make(N, Cin, H, H, O, 4, 2, 1, 1, 1, False)
        d = capi.DeconvDesc(p)
        assert d.plan(capi.OP_FORWARD)["route"] == "phase"
        Ht, Wt = d.out_shape()
        dual = m.ConvDesc(m.ConvParams.make(N, O, Ht, Wt, Cin, 4, 2, 1, 1, 1, False), algo=capi.ALGO_SIMT)
        x = torch.from_numpy(rng.standard_normal(d.x_shape()).astype(np.float32)).cuda()
        w = torch.from_numpy((rng.standard_normal(d.w_shape()) * 0.05).astype(np.float32)).cuda()
        y1, y2 = torch.empty(d.y_shape(), device="cuda"), torch.empty(d.y_shape(), device="cuda")
        f_phase = lambda: d.forward(x, w, None, y1)  # noqa: E731
        f_ffma = lambda: dual.backward_data(x, w, y2)  # noqa: E731
        f_phase(); f_ffma(); torch.cuda.synchronize()
        rel = float((y1 - y2).abs().max() / y2.abs().max())
        tp, tf = [], []
        for _ in range(args.reps):          # alternated
            tp.append(timed(f_phase, args.iters))
            tf.append(timed(f_ffma, args.iters))
        flops = 2.0 * N * Cin * H * H * O * 16
        mp, mf = float(np.median(tp)), float(np.median(tf))
        res["phase"].append(dict(layer=name, phase_ms=round(mp, 4), ffma_ms=round(mf, 4), speedup=round(mf / mp, 2),
                                 phase_tflops=round(flops / mp / 1e9, 1), max_rel_diff=rel))
    for name, N, Cc, H, k, s, pd in UPSAMPLERS:
        p = m.ConvParams.make(N, Cc, H, H, Cc, k, s, pd, 1, Cc, False)
        d = capi.DeconvDesc(p)
        assert d.plan(capi.OP_FORWARD)["route"] == "depthwise"
        x = torch.randn(d.x_shape(), device="cuda")
        w = torch.randn(d.w_shape(), device="cuda")
        y = torch.empty(d.y_shape(), device="cuda")
        dx, dw = torch.empty_like(x), torch.zeros_like(w)
        nbytes = 4.0 * (x.numel() + y.numel() + w.numel())     # each op reads or writes the bottom and the top once
        for op, fn in (("forward", lambda: d.forward(x, w, None, y)), ("data_gradient", lambda: d.backward_data(y, w, dx)),
                       ("weight_gradient", lambda: d.backward_filter(x, y, dw))):
            fn(); torch.cuda.synchronize()
            ms = float(np.median([timed(fn, args.iters) for _ in range(args.reps)]))
            res["depthwise"].append(dict(layer=name, op=op, shape=list(d.y_shape()), ms=round(ms, 4), gb_s=round(nbytes / ms / 1e6, 1),
                                         share_of_hbm=round(nbytes / ms / 1e-3 / HBM_BYTES_PER_S, 3)))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "deconv_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
