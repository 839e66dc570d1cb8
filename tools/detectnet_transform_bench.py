"""Device time of the DetectNetTransformation kernels at KITTI's shape: N = 10 images of 3 x 384 x 1248 in and out, selections
drawn with KITTI's augmentation (scale 0.8-1.2, hue and desaturation on, flips and crops), and a label blob of 50 box rows with
boxes in every image.  Prints one JSON line: the GPU, its power limit and clocks, and per path the median over repetitions of the
mean time per launch, timed with CUDA events over many back-to-back launches.  The image path's bandwidth counts the bytes it must
move: the bottom read and the workspace written (colour + mean), then the workspace read and the top written (sampling).  A
separate profiled run splits the image path's time between its two kernels."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import detectnet_transform_oracle as dto  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return dict(zip(q.split(","), [s.strip() for s in out.split(",")])) if out else {"name": torch.cuda.get_device_name(0)}


def timed(fn, launches, reps):
    """median over `reps` of the mean ms per call across `launches` back-to-back calls"""
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / launches)
    return float(np.median(times)), float(min(times)), float(max(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the device; there is no CPU timing"
    N, H, W, OH, OW, rows = 10, 384, 1248, 384, 1248, 51
    rng = np.random.default_rng(1701)
    x = torch.from_numpy(rng.uniform(0, 255, (N, 3, H, W)).astype(np.float32)).cuda()
    augs = [dto.draw(lambda: float(rng.random()), W, H, dto.KITTI_AUG, OW, OH) for _ in range(N)]
    A = capi.detectnet_augs(augs)
    top = torch.empty((N, 3, OH, OW), device="cuda")
    ws = torch.empty(capi.detectnet_image_workspace_bytes(N, H, W) // 4, device="cuda")
    boxes = [[(rng.uniform(0, W - 200), rng.uniform(0, H - 100), rng.uniform(20, 200), rng.uniform(20, 100), 0, 1)
              for _ in range(int(rng.integers(5, rows)))] for _ in range(N)]
    labels = torch.from_numpy(dto.label_blob(boxes, rows)).cuda()
    gt = capi.DetectNetGT.make(**{k: v for k, v in dto.KITTI_GT.items() if k != "coverage_type"})
    Cc, GH, GW = capi.detectnet_label_shape(gt)
    ltop = torch.empty((N, Cc, GH, GW), device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")

    def image():
        capi.detectnet_image(x, A, top, mean_value=(104.0, 117.0, 123.0), workspace=ws)

    def label():
        capi.detectnet_labels(labels, H, W, A, gt, ltop, status)

    for fn in (image, label):
        for _ in range(20):
            fn()
    torch.cuda.synchronize()
    img_ms = timed(image, args.launches, args.reps)
    lab_ms = timed(label, args.launches, args.reps)
    capi.detectnet_check_status(int(status.item()))
    # per-kernel split of the image path, from a profiled run of its own (tracing is off while the times above are taken)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(50):
            image()
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        for k in ("colour_kernel", "sample_kernel"):
            if k in e.key:
                total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                split[k] = total / max(e.count, 1) / 1e3
    img_bytes = 4 * (2 * N * 3 * H * W + N * 3 * H * W + N * 3 * OH * OW)
    res = dict(gpu=gpu_info(), shape=dict(N=N, C=3, H=H, W=W, OH=OH, OW=OW, label_rows=rows, label_top=[N, Cc, GH, GW]),
               launches=args.launches, reps=args.reps,
               image_ms=dict(median=img_ms[0], min=img_ms[1], max=img_ms[2]),
               image_GBps=img_bytes / (img_ms[0] * 1e-3) / 1e9, image_bytes=img_bytes,
               labels_ms=dict(median=lab_ms[0], min=lab_ms[1], max=lab_ms[2]),
               image_kernel_ms_profiled=split)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
