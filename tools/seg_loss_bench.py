"""SoftmaxWithLoss and Accuracy over spatial positions on the GPU, against the HBM bound and against the Softmax pass alone.

  python tools/seg_loss_bench.py [--reps 5] [--iters 20] [--out DIR]

Shapes: a PASCAL-VOC-sized FCN head (N 8, 21 classes, 512 x 512, and 511 x 511: the scalar column route), an ADE20K-sized one (N 16, 150 classes, 128 x 128) and an
ImageNet classifier with ignore_label (N 256, 1000 classes, inner 1: the row route).  Per shape, alternated --reps times,
--iters launches each timed with CUDA events: b2c_softmax_forward on the same bottom (the baseline: the softmax pass alone),
b2c_softmax_loss_forward_ex (VALID, about 10 % of the labels ignored), b2c_softmax_loss_backward_ex and b2c_accuracy_ex with the
per-class top.  Compulsory bytes: softmax and forward read the logits and write prob (+ one label per pixel for the loss), the
backward reads prob and the labels and writes dx, accuracy reads the scores and the labels.  GB/s and the share of 3.35 TB/s, the
H100 SXM data-sheet HBM3 bandwidth, are of the median time.  Prints one JSON line with the device name, power limit and max SM
clock, and writes it to DIR/seg_loss_bench.json when --out is given.
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

# (name, outer, C, inner)
SHAPES = [("voc N8 C21 512x512", 8, 21, 512 * 512), ("voc N8 C21 511x511", 8, 21, 511 * 511), ("ade N16 C150 128x128", 16, 150, 128 * 128),
          ("cls N256 C1000 inner1", 256, 1000, 1)]
IGNORE = 255


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("seg_loss_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    L = capi.lib()
    res = dict(device_info(), shapes=[])
    g = torch.Generator(device="cuda").manual_seed(1701)
    for name, outer, C, inner in SHAPES:
        n, pix = outer * C * inner, outer * inner
        x = torch.randn(n, device="cuda", generator=g)
        lab = torch.randint(0, C, (pix,), device="cuda", generator=g).float()
        lab[torch.rand(pix, device="cuda", generator=g) < 0.1] = IGNORE
        prob, y, dx = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        plan = capi.softmax_loss_plan(outer, C, inner, x.data_ptr(), prob.data_ptr())
        ws = torch.empty(plan["workspace"] // 4, device="cuda")
        loss, nrm, acc, pc = (torch.empty(k, device="cuda") for k in (1, 1, 1, C))
        scratch = torch.empty(2 + 2 * C, dtype=torch.int32, device="cuda")
        st = capi._stream()
        ops = {
            "softmax": (lambda: capi.check(L.b2c_softmax_forward(outer, C, inner, capi._p(x), capi._p(y), st)), 8.0 * n),
            "forward": (lambda: capi.softmax_loss_forward_ex(outer, C, inner, x, lab, prob, loss, nrm, ws, ignore_label=IGNORE),
                        8.0 * n + 4.0 * pix),
            "backward": (lambda: capi.softmax_loss_backward_ex(outer, C, inner, prob, lab, nrm, 1.0, dx, ignore_label=IGNORE),
                         8.0 * n + 4.0 * pix),
            "accuracy": (lambda: capi.accuracy_ex(outer, C, inner, 1, x, lab, acc, pc, scratch, ignore_label=IGNORE), 4.0 * n + 4.0 * pix),
        }
        for fn, _ in ops.values():
            fn()
        torch.cuda.synchronize()
        same = bool(torch.equal(prob.view(torch.int32), y.view(torch.int32)))
        times = {k: [] for k in ops}
        for _ in range(args.reps):                    # alternated
            for k, (fn, _) in ops.items():
                times[k].append(timed(fn, args.iters))
        row = dict(shape=name, route=plan["route"], prob_equals_softmax=same)
        for k, (_, nbytes) in ops.items():
            ms = float(np.median(times[k]))
            row[k] = dict(ms=round(ms, 4), spread_ms=[round(min(times[k]), 4), round(max(times[k]), 4)], mbytes=round(nbytes / 1e6, 1),
                          gb_s=round(nbytes / ms / 1e6, 1), share_of_hbm=round(nbytes / ms / 1e-3 / HBM_BYTES_PER_S, 3))
        row["forward_over_softmax"] = round(row["forward"]["ms"] / row["softmax"]["ms"], 3)
        res["shapes"].append(row)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "seg_loss_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
