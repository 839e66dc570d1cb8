"""Where a training step's kernel boundaries go: a few warm steps of a whole net through host_api.Trainer under torch.profiler
(CUDA activities), read back from the trace.  Reports, per step: kernels on the compute stream, the idle time between
consecutive operations on that stream (a kernel, memset or copy ending and the next one starting), the largest boundaries by
kernel pair, and each kernel family's share of the step.  With programmatic dependent launch a kernel may start
before its predecessor ends; such a boundary counts as zero idle time and its overlap is summed separately.

  python tools/step_trace.py [--model resnet50] [--batch 64] [--warmup 5] [--steps 3] [--top 20] [--json PATH]

Run it in a process of its own: the profiler slows the host, so its step times are not the benchmark's."""
import argparse
import collections
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def family(name):
    """Kernel name without its template arguments and parameter list: 'b2c::stg::igemm_stg_kernel'."""
    n = re.sub(r"^void ", "", name)
    n = n.split("(")[0]
    out, depth = [], 0
    for ch in n:
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif depth == 0:
            out.append(ch)
    return "".join(out).strip()


def stream_ops(trace):
    """[(start_us, end_us, kind, name)] of every kernel, memset and copy on the stream that carries the most kernel time."""
    by_stream = collections.defaultdict(list)
    for e in trace["traceEvents"]:
        cat = e.get("cat", "")
        if cat not in ("kernel", "gpu_memset", "gpu_memcpy") or "dur" not in e:
            continue
        st = e.get("args", {}).get("stream")
        by_stream[st].append((float(e["ts"]), float(e["ts"]) + float(e["dur"]), cat, e.get("name", "")))
    busiest = max(by_stream, key=lambda s: sum(b - a for a, b, c, _ in by_stream[s] if c == "kernel"))
    return sorted(by_stream[busiest])


def analyse(ops, steps, top):
    kernels = [o for o in ops if o[2] == "kernel"]
    idle = overlap = 0.0
    pairs = collections.defaultdict(lambda: [0, 0.0])
    for prev, nxt in zip(ops, ops[1:]):
        gap = nxt[0] - prev[1]
        if gap < 0:
            overlap -= gap
            gap = 0.0
        idle += gap
        key = (family(prev[3]) if prev[2] == "kernel" else prev[2], family(nxt[3]) if nxt[2] == "kernel" else nxt[2])
        pairs[key][0] += 1
        pairs[key][1] += gap
    # exposed: how far a kernel extends the stream past the operation before it (its whole duration when nothing overlaps it)
    fam = collections.defaultdict(lambda: [0, 0.0, 0.0])
    prev_end = ops[0][0]
    for a, b, kind, name in ops:
        if kind == "kernel":
            f = fam[family(name)]
            f[0] += 1
            f[1] += b - a
            f[2] += max(0.0, b - max(a, prev_end))
        prev_end = max(prev_end, b)
    busy = sum(b - a for a, b, _, _ in kernels)
    span = ops[-1][1] - ops[0][0]
    return {
        "steps": steps,
        "kernels_per_step": len(kernels) / steps,
        "stream_ops_per_step": len(ops) / steps,
        "span_ms_per_step": span / steps / 1e3,
        "kernel_busy_ms_per_step": busy / steps / 1e3,
        "idle_ms_per_step": idle / steps / 1e3,
        "overlap_ms_per_step": overlap / steps / 1e3,
        "top_boundaries": [{"prev": k[0], "next": k[1], "count_per_step": v[0] / steps, "idle_us_per_step": v[1] / steps}
                           for k, v in sorted(pairs.items(), key=lambda kv: -kv[1][1])[:top]],
        "families": [{"family": k, "launches_per_step": v[0] / steps, "ms_per_step": v[1] / steps / 1e3, "share": v[1] / busy,
                      "exposed_ms_per_step": v[2] / steps / 1e3, "exposed_share": v[2] / span}
                     for k, v in sorted(fam.items(), key=lambda kv: -kv[1][2])],
    }


def report(r):
    print(f"steps traced {r['steps']}: {r['kernels_per_step']:.0f} kernels per step ({r['stream_ops_per_step']:.0f} stream operations)")
    print(f"per step: span {r['span_ms_per_step']:.3f} ms, kernels busy {r['kernel_busy_ms_per_step']:.3f} ms, "
          f"idle between operations {r['idle_ms_per_step']:.3f} ms, overlapped boundaries {r['overlap_ms_per_step']:.3f} ms")
    print(f"\nlargest boundaries (idle us per step, summed by pair):")
    for b in r["top_boundaries"]:
        print(f"  {b['idle_us_per_step']:9.1f} us  x{b['count_per_step']:5.1f}  {b['prev'][:60]} -> {b['next'][:60]}")
    print(f"\nkernel families: exposed time (how far the family's kernels extend the stream past the operation before each) "
          f"and its share of the span; busy time (start to end, including any wait at the start) and its share of all kernels' busy time")
    for f in r["families"]:
        print(f"  exposed {f['exposed_ms_per_step']:8.3f} ms {100 * f['exposed_share']:5.1f}%  busy {f['ms_per_step']:8.3f} ms "
              f"{100 * f['share']:5.1f}%  x{f['launches_per_step']:5.1f}  {f['family'][:90]}")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--model", default="resnet50")
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--top", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    from caffe_mpi_b200 import host_api, models
    if not torch.cuda.is_available():
        sys.exit("step_trace.py needs a GPU")
    torch.cuda.set_device(0)
    defaults = {"resnet50": 64, "alexnet": 256, "vgg16": 32, "googlenet": 128, "lenet": 64}
    N = args.batch or defaults[args.model]
    kw = dict(default_channels=1, default_size=28, num_classes=10) if args.model == "lenet" else {}
    t = host_api.Trainer(models.PROTOTXT[args.model](N), models.SOLVERS[args.model], batch=N, **kw)
    t.step(args.warmup)
    t.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t.step(args.steps)
        t.sync()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    r = analyse(stream_ops(trace), args.steps, args.top)
    r.update(model=args.model, batch=N, device=torch.cuda.get_device_name(0))
    report(r)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
