"""The neuron kernels on the GPU against the HBM bound: every elementwise kind both ways, and PReLU at the activation sizes of a
PReLU ResNet-50 at batch 64.

  python tools/neuron_bench.py [--reps 5] [--iters 20] [--out DIR]

Elementwise kinds: one res2-sized activation (64 x 256 x 56 x 56), forward (reads x, writes y) and backward (reads dy and the x / y
its rule needs, writes dx).  PReLU: the stem (64 x 64 x 112 x 112, several CTAs per channel), res2 .. res5 (256 x 56 x 56 down to
2048 x 7 x 7, one CTA per channel), per-channel slopes; forward, backward with dx and the slope gradient (12 B per value) and without
dx (8 B per value), and the stem with a channel-shared slope.  Compulsory bytes come from the shapes.  Each op runs --iters launches
timed with CUDA events, alternated --reps times; GB/s and the share of 3.35 TB/s (the H100 SXM data-sheet HBM3 bandwidth) are of the
median.  Prints one JSON line with the device name, power limit and max SM clock, and writes it to DIR/neuron_bench.json when --out
is given.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from caffe_mpi_b200 import capi  # noqa: E402
from deconv_bench import HBM_BYTES_PER_S, device_info, timed  # noqa: E402

ELEMENTWISE = [  # kind, forward params, backward params, values the backward reads besides dy
    ("ELU", (1.0, 0, 0), (1.0, 0, 0), 2),
    ("POWER", (0.5, 2.0, 1.0), (0.5, 2.0, 1.0), 2),
    ("ABSVAL", (0, 0, 0), (0, 0, 0), 1),
    ("BNLL", (0, 0, 0), (0, 0, 0), 1),
    ("EXP", (1.0, 1.0, 0), (1.0, 1.0, 0), 1),
    ("LOG", (1.0, 2.0, 1.0), (1.0, 2.0, 1.0), 1),
    ("THRESHOLD", (0.0, 0, 0), None, 0),
]
PRELU = [("stem 64x64x112x112", 64, 64, 112 * 112), ("res2 64x256x56x56", 64, 256, 56 * 56), ("res3 64x512x28x28", 64, 512, 28 * 28),
         ("res4 64x1024x14x14", 64, 1024, 14 * 14), ("res5 64x2048x7x7", 64, 2048, 7 * 7)]


def row(times, nbytes):
    ms = float(np.median(times))
    return dict(ms=round(ms, 4), spread_ms=[round(min(times), 4), round(max(times), 4)], mbytes=round(nbytes / 1e6, 1),
                gb_s=round(nbytes / ms / 1e6, 1), share_of_hbm=round(nbytes / ms / 1e-3 / HBM_BYTES_PER_S, 3))


def measure(ops, reps, iters):
    for fn, _ in ops.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in ops}
    for _ in range(reps):                             # alternated
        for k, (fn, _) in ops.items():
            times[k].append(timed(fn, iters))
    return {k: row(times[k], nbytes) for k, (_, nbytes) in ops.items()}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("neuron_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    res = dict(device_info(), elementwise={}, prelu=[])
    g = torch.Generator(device="cuda").manual_seed(1701)
    n = 64 * 256 * 56 * 56
    x = torch.rand(n, device="cuda", generator=g) + 0.5          # inside every kind's domain
    y, dy, dx = torch.empty_like(x), torch.randn(n, device="cuda", generator=g), torch.empty_like(x)
    ops = {}
    for kind, pf, pb, reads in ELEMENTWISE:
        ops[kind + " forward"] = (lambda k=kind, p=pf: capi.neuron_forward(k, x, y, p), 8.0 * n)
        if pb is not None:
            ops[kind + " backward"] = (lambda k=kind, p=pb: capi.neuron_backward(k, x, y, dy, dx, p), (8.0 + 4.0 * reads) * n)
    res["elementwise"] = dict(shape="64x256x56x56", **measure(ops, args.reps, args.iters))
    del x, y, dy, dx
    for name, N, Cc, dim in PRELU + [("stem shared", 64, 64, 112 * 112)]:
        shared = name.endswith("shared")
        m = N * Cc * dim
        x = torch.randn(m, device="cuda", generator=g)
        dy = torch.randn(m, device="cuda", generator=g)
        y, dx = torch.empty_like(x), torch.empty_like(x)
        slope = torch.full((1 if shared else Cc,), 0.25, device="cuda")
        dslope = torch.zeros_like(slope)
        ws = torch.zeros(max(1, capi.prelu_workspace_bytes(N, Cc, dim, shared)), dtype=torch.uint8, device="cuda")
        plan = capi.neuron_plan("prelu_backward", N, Cc, dim, shared=shared, ptrs=(x.data_ptr(), dy.data_ptr(), dx.data_ptr()))
        ops = {
            "forward": (lambda: capi.prelu_forward(N, Cc, dim, shared, x, slope, y), 8.0 * m),
            "backward": (lambda: capi.prelu_backward(N, Cc, dim, shared, x, dy, slope, dx, dslope, ws), 12.0 * m),
            "backward_no_dx": (lambda: capi.prelu_backward(N, Cc, dim, shared, x, dy, slope, None, dslope, ws), 8.0 * m),
        }
        res["prelu"].append(dict(shape=name, plan=plan, **measure(ops, args.reps, args.iters)))
        del x, dy, y, dx
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "neuron_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
