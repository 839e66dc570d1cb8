#!/usr/bin/env python
"""ResNet-50 TEST-phase measurements on one GPU (the forward-only net `caffe.py test` runs):

  * TEST forward throughput at N = 64 (images / s from CUDA events around the forwards, synthetic source, fp32 math);
  * forward milliseconds per layer type from the per-layer CUDA-event profiler (a separate, instrumented run);
  * b2c_bn_forward_inference on every BatchNorm shape of the net: achieved GB/s from the bytes its shapes require (read x, write y:
    8 B per element) over CUDA-event kernel time, and the share of the H100 SXM's 3.35 TB/s HBM3 bandwidth that is;
  * the device name and power limit, read in the same run.

  python tools/infer_bench.py [--batch 64] [--iters 30] [--warmup 5]

Prints one JSON line.  There is no CPU mode: without a GPU it exits with an error."""
import argparse, ctypes as C, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12         # H100 SXM data sheet
PROTOTXT = os.path.join(ROOT, "tests", "golden", "reference_models", "models", "resnet50", "train_val.prototxt")


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def bn_kernel_rate(torch, L, shapes, reps):
    """(GB/s, total bytes, total ms) of b2c_bn_forward_inference (ReLU form, no residual) over the given [N, C, H, W] shapes"""
    vp = C.c_void_p
    L.b2c_bn_forward_inference.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp, vp, C.c_float, vp, vp, vp, vp, C.c_int, vp]
    total_bytes, total_ms = 0, 0.0
    for shp in shapes:
        N, Cc = shp[0], shp[1]
        S = 1
        for d in shp[2:]:
            S *= d
        x = torch.randn(N, Cc, S, device="cuda")
        y = torch.empty_like(x)
        g, b, m = torch.ones(Cc, device="cuda"), torch.zeros(Cc, device="cuda"), torch.zeros(Cc, device="cuda")
        v = torch.ones(Cc, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        call = lambda: L.b2c_bn_forward_inference(N, Cc, S, x.data_ptr(), g.data_ptr(), b.data_ptr(), 1e-5, m.data_ptr(), v.data_ptr(), None,
                                                  y.data_ptr(), 1, st)
        for _ in range(3):
            assert call() == 0
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            call()
        e.record()
        e.synchronize()
        total_ms += a.elapsed_time(e) / reps
        total_bytes += 8 * N * Cc * S
    return total_bytes / (total_ms / 1e3) / 1e9, total_bytes, total_ms


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("infer_bench.py: no CUDA device (nothing is measured on the CPU)")
    from caffe_mpi_b200 import capi, host_api
    os.environ.setdefault("B2C_DATA", "synthetic")
    t = host_api.Tester(PROTOTXT, batch=args.batch, net_is_text=False)
    t.timed_forwards(args.warmup)
    ms = t.timed_forwards(args.iters)
    prof = t.profile(3)
    layers = t.layers()
    by_type = {}
    for li, m in prof:
        by_type[layers[li][1]] = by_type.get(layers[li][1], 0.0) + m
    bn_shapes = [shp for _, ty, shp in host_api.Net(PROTOTXT, phase="TEST", batch_override=args.batch).layers() if ty == "BatchNorm"]
    gbs, nbytes, bn_ms = bn_kernel_rate(torch, capi.lib(), bn_shapes, 20)
    out = {
        "device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "batch": args.batch, "iters": args.iters,
        "test_forward_ms": ms / args.iters, "img_per_s": args.batch * args.iters / (ms / 1e3),
        "forward_ms_by_layer_type": {k: round(v, 4) for k, v in sorted(by_type.items(), key=lambda kv: -kv[1])},
        "bn_inference": {"layers": len(bn_shapes), "bytes": nbytes, "ms": bn_ms, "GB_per_s": gbs, "share_of_hbm_bound": gbs * 1e9 / HBM_BYTES_PER_S},
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
