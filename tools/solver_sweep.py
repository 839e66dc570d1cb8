#!/usr/bin/env python
"""Time the fused solver updates over ResNet-50's learnable layout (161 blobs, 25 557 032 floats, read from the reference
prototxt), and the ResNet-50 training step with Adam against SGD.

  python tools/solver_sweep.py [--launches 200] [--batch 64] [--steps 10] [--rounds 3] [--out results.json]

Arena update: CUDA events around `--launches` back-to-back b2c_solver_update_arena calls after warm-up, per solver kind.  GB/s
uses the bytes each element must move -- 24 B (g, w, h read and written) for SGD, Nesterov, AdaGrad and RMSProp, 32 B (also h2)
for AdaDelta and Adam -- and is also given as a share of the H100 SXM data-sheet 3.35 TB/s.  Step time: host_api.Trainer on
models.resnet50_prototxt, SGD and Adam alternated `--rounds` times in this one process.  The card name and power limit are read
in the same run.

clip_gradients: CUDA events around `--launches` b2c_arena_sumsq calls over the same arena (4 B read per float), and the ResNet-50
step with RESNET50_SOLVER against the same solver plus `clip_gradients`, alternated `--rounds` times; the median is reported.  A
clipped step does the same work whether or not its norm exceeds the clip, so `--clip` only decides what the last norm line says.
  python tools/solver_sweep.py --clip-only"""
import argparse, json, os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BYTES = {"SGD": 24, "Nesterov": 24, "AdaGrad": 24, "RMSProp": 24, "AdaDelta": 32, "Adam": 32}
PEAK_GBS = 3350.0


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_max_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:                      # the number is still reported, with the reason the limit is missing
        info["power_limit"] = "unknown (%s)" % e
    return info


def arena_sweep(launches):
    import torch
    from caffe_mpi_b200 import capi, host_api
    net = host_api.Net(os.path.join(ROOT, "tests", "golden", "reference_models", "models", "resnet50", "train_val.prototxt"), "TRAIN",
                       batch_override=1)
    counts = [c for _, c, _, _ in net.learnable_params()]
    offsets, off = [], 0
    for c in counts:
        offsets.append(off)
        off += c + (c & 1)                       # arena slots padded to an even element count, like ParamArena
    n = sum(counts)
    rates, decays = [1e-3] * len(counts), [1e-4] * len(counts)
    g, w = torch.zeros(off, device="cuda"), torch.randn(off, device="cuda")
    h, h2 = torch.zeros(off, device="cuda"), torch.zeros(off, device="cuda")
    out = {"blobs": len(counts), "floats": n}
    for kind in BYTES:
        def run():
            capi.solver_update_arena(kind, offsets, counts, rates, decays, g, w, h, h2, momentum=0.0 if kind in ("AdaGrad", "RMSProp")
                                     else 0.9, delta=1e-8, rms_decay=0.9, beta1=0.9, beta2=0.999, clear_grads=True)
        for _ in range(20):
            run()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(launches):
            run()
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b) / launches
        gbs = BYTES[kind] * n / (ms * 1e-3) / 1e9
        out[kind] = {"ms": round(ms, 4), "bytes_per_param": BYTES[kind], "GB_s": round(gbs, 1), "share_of_3350": round(gbs / PEAK_GBS, 3)}
        print(kind, out[kind], flush=True)
    return out


def step_times(batch, steps, rounds):
    from caffe_mpi_b200 import host_api, models
    solvers = {"SGD": models.RESNET50_SOLVER,
               "Adam": 'type: "Adam" base_lr: 0.001 lr_policy: "fixed" momentum: 0.9 momentum2: 0.999 weight_decay: 1e-4 max_iter: 1000'}
    trainers = {k: host_api.Trainer(models.resnet50_prototxt(batch), s, batch=batch) for k, s in solvers.items()}
    for t in trainers.values():
        t.step(3)
        t.sync()
    res = {k: [] for k in solvers}
    for _ in range(rounds):
        for k, t in trainers.items():
            res[k].append(t.timed_steps(steps) / steps)
    out = {k: {"ms_per_step": [round(x, 3) for x in v], "best_ms": round(min(v), 3), "img_s": round(batch / (min(v) / 1e3), 1)}
           for k, v in res.items()}
    out["batch"] = batch
    out["adam_over_sgd"] = round(out["Adam"]["best_ms"] / out["SGD"]["best_ms"], 4)
    print(out, flush=True)
    return out


def sumsq_sweep(launches):
    import torch
    from caffe_mpi_b200 import capi, host_api
    net = host_api.Net(os.path.join(ROOT, "tests", "golden", "reference_models", "models", "resnet50", "train_val.prototxt"), "TRAIN",
                       batch_override=1)
    counts = [c for _, c, _, _ in net.learnable_params()]
    offsets, off = [], 0
    for c in counts:
        offsets.append(off)
        off += c + (c & 1)
    n = sum(counts)
    slots, npart = host_api.clip_slots(counts)
    g = torch.randn(off, device="cuda") * 1e-3
    P = torch.empty(npart, dtype=torch.float64, device="cuda")
    st = torch.zeros(4, device="cuda")

    def run():
        capi.arena_sumsq(offsets, counts, slots, g, P)
    for _ in range(20):
        run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(launches):
        run()
    b.record()
    b.synchronize()
    ms = a.elapsed_time(b) / launches
    a.record()
    for _ in range(launches):
        capi.clip_factor(P, npart, 1.0, 1.0, st)
    b.record()
    b.synchronize()
    fms = a.elapsed_time(b) / launches
    gbs = 4 * n / (ms * 1e-3) / 1e9
    out = {"floats": n, "partials": npart, "sumsq_ms": round(ms, 4), "GB_s": round(gbs, 1), "share_of_3350": round(gbs / PEAK_GBS, 3),
           "clip_factor_ms": round(fms, 4)}
    print("sumsq", out, flush=True)
    return out


def clip_step_times(batch, steps, rounds, clip):
    import statistics
    from caffe_mpi_b200 import host_api, models
    solvers = {"SGD": models.RESNET50_SOLVER, "SGD+clip": models.RESNET50_SOLVER + " clip_gradients: %g" % clip}
    trainers = {k: host_api.Trainer(models.resnet50_prototxt(batch), s, batch=batch) for k, s in solvers.items()}
    for t in trainers.values():
        t.step(3)
        t.sync()
    res = {k: [] for k in solvers}
    for _ in range(rounds):
        for k, t in trainers.items():
            res[k].append(t.timed_steps(steps) / steps)
    out = {k: {"ms_per_step": [round(x, 3) for x in v], "median_ms": round(statistics.median(v), 3)} for k, v in res.items()}
    norm, factor, clipped = trainers["SGD+clip"].clip_state()
    out.update(batch=batch, clip=clip, last_norm=norm, last_factor=factor, clipped_steps=clipped,
               clip_minus_plain_ms=round(out["SGD+clip"]["median_ms"] - out["SGD"]["median_ms"], 3))
    print(out, flush=True)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--clip", type=float, default=1.0, help="clip_gradients of the clipped ResNet-50 run")
    ap.add_argument("--clip-only", action="store_true", help="only the clip_gradients measurements")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("solver_sweep.py: needs a CUDA device")
    res = {"card": card()}
    if not args.clip_only:
        res.update(arena_update=arena_sweep(args.launches), resnet50_step=step_times(args.batch, args.steps, args.rounds))
    res.update(arena_sumsq=sumsq_sweep(args.launches), resnet50_clip_step=clip_step_times(args.batch, args.steps, args.rounds, args.clip))
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
