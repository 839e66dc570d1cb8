#!/usr/bin/env python
"""Command-line shell in the shape of the reference's `caffe` tool (tools/caffe.cpp: train / time / device_query), over the
C++ host layer -- SURVEY 8(f) rank 3.  A Data layer whose data_param.source holds an LMDB (backend: LMDB, raw uint8 datums) reads
it through the parser threads / device transform of host/data_layer.cpp; when the source is not on disk the synthetic in-memory
source stands in (SURVEY 8d).  B2C_DATA=db makes a missing database fatal, as in the reference; B2C_DATA=synthetic ignores it.

  python tools/caffe.py train --solver=models/resnet50/solver.prototxt [--iterations=N] [--batch=B]     (1 GPU)
         [--snapshot=<solverstate to resume from>] [--weights=<caffemodel to fine-tune from>] [--snapshot_prefix=P]
  python -m torch.distributed.run --nproc-per-node N ... tools/caffe.py train --solver=...              (N GPUs, one rank each)
  python tools/caffe.py time --model=models/resnet50/train_val.prototxt [--iterations=50] [--batch=B]
  python tools/caffe.py test --model=models/resnet50/train_val.prototxt --weights=x.caffemodel [--iterations=50] [--batch=B]   (1 GPU)
  python tools/caffe.py device_query
"""
import argparse, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def log(msg, stream=None):
    t = time.localtime()
    print("I%02d%02d %02d:%02d:%02d caffe.py] %s" % (t.tm_mon, t.tm_mday, t.tm_hour, t.tm_min, t.tm_sec, msg), flush=True, file=stream or sys.stdout)


def log_test_net(msg):
    """The test nets' log lines go to stderr -- the stream the reference logs everything to (glog, alsologtostderr) -- so that stdout
    carries the same lines with and without test nets: a script reading the training loss from stdout's `loss = ` never picks up a
    test net's `Test net output #i: loss = ...`."""
    log(msg, sys.stderr)


def cmd_device_query(_):
    from caffe_mpi_b200 import capi
    import ctypes as C
    rt = C.CDLL("libcudart.so")
    n = C.c_int()
    if rt.cudaGetDeviceCount(C.byref(n)) != 0 or n.value == 0:
        sys.exit("caffe.py: no CUDA device (there is no CPU mode)")
    v = capi.lib().b2c_version()
    log("libb2c version %s, %d device(s)" % (v.decode() if isinstance(v, bytes) else v, n.value))


def schedule(it, end, display, snapshot, test_interval=0):
    """The shell's part of Solver::Step (solver.cpp:277-345) as a plan: yields (n, iter_after, show, snap) -- run n iterations,
    after which the iteration counter reads iter_after; print the loss line if `show` (iter % display == 0, or the run is over, or
    display is off and this is the only chunk), write a snapshot if `snap` (iter % snapshot == 0).

    With test_interval > 0 (a solver with test nets) every chunk also says which test pass runs BEFORE its iterations, as a fifth
    element: "initial" (one batch per test net) when the counter reads 0 -- Step's iter_ == 0 branch, whatever test_initialization
    says -- and "full" (test_iter batches) at every later multiple of test_interval except the one a resumed run starts at
    (iterations_last_ = -1 after a restore), else None.  Solve's closing pass (solver.cpp:419-423, when the final counter is a multiple
    of test_interval) comes last as (0, end, False, False, "final"); it is skipped when training stopped early."""
    start = it
    while it < end:
        test = None
        if test_interval > 0:
            test = "initial" if it == 0 else "full" if it > start and it % test_interval == 0 else None
        nxt = end
        for every in (display, snapshot, test_interval):
            if every > 0:
                nxt = min(nxt, (it // every + 1) * every)
        n, it = nxt - it, nxt
        row = (n, it, (display > 0 and it % display == 0) or it == end, snapshot > 0 and it % snapshot == 0)
        yield row + (test,) if test_interval > 0 else row
    if test_interval > 0 and end % test_interval == 0:
        yield 0, end, False, False, "final"


def rank_batch(net, net_is_text, override, solver_count, phase="TRAIN"):
    """Per-solver batch size, or 0 for "what the prototxt says".  P2PSync::divide_batch_size (parallel.cpp:284-316): with more than
    one solver (GPU) on the node, the batch_size of the net's Data layer -- or the --batch override -- is the NODE's batch and each
    solver takes total / solver_count of it, the total first rounded up to a multiple of solver_count.  Nets fed by Input /
    DummyData layers have no data_param and are left alone, as in the reference.  phase="TEST" divides the TEST Data layer's batch
    the same way (Net::Init does it for test nets too)."""
    from caffe_mpi_b200 import host_api
    if solver_count <= 1:
        return override
    total = override
    if not total:
        data = [l for l in host_api.Net(net, phase=phase, is_text=net_is_text).layers() if l[1] == "Data"]
        if not data:
            return 0
        total = data[0][2][0]
    return host_api.divide_batch_size(total, solver_count)


def build_trainer(args, net, net_is_text, solver, solver_is_text):
    from caffe_mpi_b200 import host_api
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    batch = rank_batch(net, net_is_text, args.batch, int(os.environ.get("LOCAL_WORLD_SIZE", world)))
    t = host_api.Trainer(net, solver, batch=batch or 0, num_classes=args.classes, seed=args.seed + rank, net_is_text=net_is_text,
                         solver_is_text=solver_is_text)
    if world > 1:                              # P2PSync: one solver per GPU, rank 0 is the root solver (parallel.cpp:26-60)
        import torch, torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("gloo")
        ids = [t.new_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        t.attach_sync(world, rank, ids[0])
    return t, rank, world


def solver_hparams_text(d):
    """The hyperparameters the solver type reads (solver_describe's dict), for the "Solving" line."""
    keys = {"SGD": ("momentum",), "Nesterov": ("momentum",), "AdaGrad": ("delta",), "RMSProp": ("rms_decay", "delta"),
            "AdaDelta": ("momentum", "delta"), "Adam": ("momentum", "momentum2", "delta")}[d["type"]]
    return " ".join("%s %g" % (k, d[k]) for k in keys)


def test_net_lines(outputs, means, loss, compute_loss):
    """Solver::Test's log lines after a pass (solver.cpp:521-538): `outputs` = [(name, loss_weight, count)] in the net's output order,
    `means` = one value per output element, `loss` = the mean loss, printed only with test_compute_loss."""
    import numpy as np
    lines = ["Test loss: %g" % loss] if compute_loss else []
    i = 0
    for name, w, n in outputs:
        for _ in range(n):
            m = np.float32(means[i])
            lines.append("    Test net output #%d: %s = %g%s" % (i, name, m, " (* %g = %g loss)" % (w, np.float32(w) * m) if w else ""))
            i += 1
    return lines


def cmd_train(args):
    from caffe_mpi_b200 import host_api
    if not args.solver:
        sys.exit("caffe.py train: Need a solver definition to train (--solver=...)")
    if args.snapshot and args.weights:
        sys.exit("caffe.py train: Give a snapshot to resume training or weights to finetune but not both.")   # tools/caffe.cpp:166
    s, net_path = host_api.open_solver(args.solver)
    d = host_api.solver_describe(s)
    net_path = args.model or net_path
    for f in d["test_fields_not_built"]:
        sys.exit("caffe.py train: SolverParameter.%s is not built: test nets are built from the solver's `net` with phase TEST, one per "
                 "test_iter entry" % f)
    if not os.path.exists(net_path):
        sys.exit("caffe.py train: net file %r named by the solver does not exist (paths are relative to the working directory)" % net_path)
    if args.seed < 0:
        args.seed = int(host_api.textproto_scalar(args.solver, "random_seed", "1701"))     # Solver::Init seeds Caffe with it (solver.cpp:63-65)
        if args.seed < 0:
            args.seed = 1701
    t, rank, world = build_trainer(args, net_path, False, args.solver, False)
    if args.snapshot:
        t.restore(args.snapshot)
        if rank == 0:
            log("Resuming from %s at iteration %d" % (args.snapshot, t.iter()))
    elif args.weights:
        n = t.copy_trained_layers_from(args.weights)
        if rank == 0:
            log("Finetuning from %s (%d layers copied)" % (args.weights, n))
    iters = args.iterations or d["max_iter"]
    # SolverParameter fields of the shell (caffe.proto:147-301); command-line flags win where both exist
    sp = lambda key, default: host_api.textproto_scalar(args.solver, key, default)
    display = args.display if args.display > 0 else int(sp("display", "0"))
    snap_every = int(sp("snapshot", "0"))
    snap_prefix = args.snapshot_prefix or sp("snapshot_prefix", "")
    snap_after = sp("snapshot_after_train", "true").lower() in ("true", "1")
    clip = float(sp("clip_gradients", "-1"))
    if rank == 0:
        log("Data layer: %s" % ("reading the LMDB named by data_param.source" if t.database_batches() >= 0 else "synthetic in-memory source"))
        log("Solving %s with %s: %d learnable blobs, lr_policy %s base_lr %g %s weight_decay %g, %d iteration(s) on %d GPU(s)" %
            (net_path, d["type"], t.num_params(), d["lr_policy"], d["base_lr"], solver_hparams_text(d), d["weight_decay"], iters, world))
    try:
        batch = len(t.get_blob("label"))           # images per rank and step, for the img/s figure
    except host_api.HostError:
        batch = 0
    # Solver::InitTestNets (solver.cpp:107-185): one TEST net per test_iter entry, from the solver's net file, sharing the trainer's
    # layers by name; each rank scores its stripe of the validation database at the per-rank TEST batch
    testers = []
    if d["test_iter"]:
        test_batch = rank_batch(net_path, False, 0, int(os.environ.get("LOCAL_WORLD_SIZE", world)), phase="TEST")
        for k, n_iter in enumerate(d["test_iter"]):
            if rank == 0:
                log_test_net("Creating test net (#%d) specified by net file: %s" % (k, net_path))
            te = host_api.Tester(net_path, batch=test_batch, num_classes=args.classes, seed=args.seed + rank, net_is_text=False)
            te.share_trained_layers_with(t)
            testers.append((te, n_iter))
    test_every = d["test_interval"] if testers else 0
    end = t.iter() + args.iterations if args.iterations else max(d["max_iter"], t.iter())   # a resumed run goes on to max_iter
    last_snapshot = -1
    # SignalHandler (src/caffe/util/signal_handler.cpp, tools/caffe.cpp:43-48,209-214): SIGINT = stop (with a snapshot when
    # snapshot_after_train), SIGHUP = snapshot and carry on; both take effect at the next point where the host looks at the device
    import signal
    got = {"stop": False, "snapshot": False}
    signal.signal(signal.SIGINT, lambda *_: got.__setitem__("stop", True))
    if hasattr(signal, "SIGHUP"):
        signal.signal(signal.SIGHUP, lambda *_: got.__setitem__("snapshot", True))

    def between_batches(_):
        # Solver::Test's GetRequestedAction before every batch (solver.cpp:461-475), one GPU only: on several GPUs a rank that left
        # a pass early would leave the others waiting in the score allreduce, so there the flags are read when the pass is over
        nonlocal last_snapshot
        if got["snapshot"] and rank == 0 and snap_prefix:
            log("Snapshotting solver state to binary proto file %s" % t.snapshot(snap_prefix))
            last_snapshot = t.iter()
        got["snapshot"] = False
        return not got["stop"]

    def test_all(it, kind):
        """Solver::TestAll; returns True when a SIGINT ended it ("Test interrupted.")."""
        nonlocal last_snapshot
        for k, (te, n_iter) in enumerate(testers):
            if rank == 0:
                log_test_net("Iteration %d, Testing net (#%d)" % (it, k))
            r = te.test_pass(1 if kind == "initial" else n_iter, between_batches if world == 1 else None)
            if r is None:
                log_test_net("Test interrupted.")
                return True
            if rank == 0:
                for ln in test_net_lines(te.outputs(), r[0], r[1], d["test_compute_loss"]):
                    log_test_net(ln)
        if world > 1:
            if got["snapshot"] and rank == 0 and snap_prefix:
                log("Snapshotting solver state to binary proto file %s" % t.snapshot(snap_prefix))
                last_snapshot = t.iter()
            got["snapshot"] = False
            return got["stop"]
        return False

    mgpu = "[MultiGPU] " if world > 1 else ""
    plan = list(schedule(t.iter(), end, display, snap_every, test_every))
    final_test = bool(plan) and test_every > 0 and plan[-1][4] == "final"
    interrupted = False
    for n, it, show, snap, *test in (plan[:-1] if final_test else plan):
        if test and test[0]:
            t0 = time.time()
            interrupted = test_all(it - n, test[0])
            if interrupted:
                break
            if rank == 0:
                log_test_net(mgpu + ("Initial Test completed" if test[0] == "initial" else "Tests completed in %gs" % (time.time() - t0)))
        ms = max(t.timed_steps(n, copy_input=True), 1e-6)
        assert t.iter() == it
        if got["snapshot"] and rank == 0 and snap_prefix:
            log("Snapshotting solver state to binary proto file %s" % t.snapshot(snap_prefix))
            last_snapshot = it
        got["snapshot"] = False
        if got["stop"]:
            if rank == 0:
                log("Optimization stopped early.")
            break
        if rank == 0 and show:
            log("Iteration %d (%.2f iter/s%s), loss = %.6g" % (it, n / (ms / 1e3), ", %.1f img/s" % (batch * world * n / (ms / 1e3)) if batch else "", t.loss()))
            if clip >= 0:
                # SGDSolver::ClipGradients' line (sgd_solver.cpp:122-125) for the last iteration, at display points only: the norm
                # lives on the device and reading it every iteration would synchronise every step
                import numpy as np
                norm, factor, _ = t.clip_state()
                if np.float32(norm) > np.float32(clip):
                    log("Gradient clipping: scaling down gradients (L2 norm %g > %g) by scale factor %g" % (norm, np.float32(clip), factor),
                        sys.stderr)
        if rank == 0 and snap and snap_prefix:
            log("Snapshotting solver state to binary proto file %s" % t.snapshot(snap_prefix))
            last_snapshot = it
    if rank == 0 and snap_prefix and last_snapshot != t.iter() and (snap_after or args.snapshot_prefix):   # solver.cpp:340-345
        log("Snapshotting solver state to binary proto file %s" % t.snapshot(snap_prefix))
    if interrupted:
        if rank == 0:
            log("Optimization stopped early.")
    elif final_test and not got["stop"]:
        test_all(t.iter(), "final")               # Solve's extra pass after the last iteration (solver.cpp:419-423)
    if rank == 0:
        log("Optimization Done.")


def layer_time_lines(layers, prof):
    """The per-layer table of `caffe time` (tools/caffe.cpp:424-438) from TrainNet's CUDA-event profile: `layers` = [(name, type)],
    `prof` = [(layer index, "fwd" | "bwd" | "wgrad" | "dgrad", ms per iteration)].  Returns (lines, forward ms, backward ms); the
    conv layers' weight- / data-gradient split is nested inside their backward time and listed after it."""
    fwd, bwd, extra = {}, {}, {}
    for li, op, ms in prof:
        if op == "fwd":
            fwd[li] = fwd.get(li, 0.0) + ms
        elif op == "bwd":
            bwd[li] = bwd.get(li, 0.0) + ms
        else:
            extra.setdefault(li, {})[op] = extra.get(li, {}).get(op, 0.0) + ms
    lines = ["Average time per layer: "]
    for i, (name, _) in enumerate(layers):
        lines.append("%10s\tforward: %g ms." % (name, fwd.get(i, 0.0)))
        tail = "".join(" (%s %g)" % (k, v) for k, v in sorted(extra.get(i, {}).items()))
        lines.append("%10s\tbackward: %g ms.%s" % (name, bwd.get(i, 0.0), tail))
    return lines, sum(fwd.values()), sum(bwd.values())


def cmd_time(args):
    from caffe_mpi_b200 import models
    if not args.model:
        sys.exit("caffe.py time: Need a model definition to time (--model=...)")
    if args.seed < 0:
        args.seed = 1701
    t, rank, world = build_trainer(args, args.model, False, models.RESNET50_SOLVER, True)
    iters = args.iterations or 50
    t.step(3)
    t.sync()
    if rank == 0:
        log("*** Benchmark begins ***")
        log("Testing for %d iterations." % iters)
    prof = t.profile(min(iters, 5))                  # CUDA events around every layer call (serialises nothing, but is not free)
    ms = t.timed_steps(iters)                        # the un-instrumented step: forward + backward + exchange + update
    if rank == 0:
        lines, f, b = layer_time_lines(t.layers(), prof)
        for ln in lines:
            log(ln)
        log("Average Forward pass: %g ms." % f)
        log("Average Backward pass: %g ms." % b)
        log("Average Forward-Backward-Update: %.4f ms over %d iterations (%s)." % (ms / iters, iters,
            "per-layer times are device times of single calls; the step overlaps the exchange and update with backward"))
        log("Total Time: %g ms." % ms)
        log("*** Benchmark ends ***")


def score_lines(outputs, per_batch, means, loss):
    """The log lines of `caffe test` (tools/caffe.cpp:261-299): `outputs` = [(name, loss_weight, count)] in the net's output order,
    `per_batch` = [iterations][output elements], `means` = [output elements], `loss` = the mean loss."""
    names, weights = [], []
    for name, w, n in outputs:
        names += [name] * n
        weights += [w] * n
    lines = ["Batch %d, %s = %g" % (i, names[k], v) for i, row in enumerate(per_batch) for k, v in enumerate(row)]
    lines.append("Loss: %g" % loss)
    for k, m in enumerate(means):
        lines.append("%s = %g%s" % (names[k], m, " (* %g = %g loss)" % (weights[k], weights[k] * m) if weights[k] else ""))
    return lines


def cmd_test(args):
    from caffe_mpi_b200 import host_api
    if not args.model:
        sys.exit("caffe.py test: Need a model definition to score.")
    if not args.weights:
        sys.exit("caffe.py test: Need model weights to score.")
    if int(os.environ.get("WORLD_SIZE", 1)) > 1:
        sys.exit("caffe.py test: scoring runs on one GPU (start it without torch.distributed)")
    t = host_api.Tester(args.model, batch=args.batch, num_classes=args.classes, seed=1701 if args.seed < 0 else args.seed, net_is_text=False)
    t.copy_trained_layers_from(args.weights)
    iters = args.iterations or 50
    log("Running for %d iterations." % iters)
    per_batch, means, loss = t.test(iters)
    for ln in score_lines(t.outputs(), per_batch, means, loss):
        log(ln)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("command", choices=["train", "test", "time", "device_query"])
    ap.add_argument("--solver", "-solver", default="")
    ap.add_argument("--model", "-model", default="")
    ap.add_argument("--iterations", "-iterations", type=int, default=0)
    ap.add_argument("--batch", type=int, default=0, help="global batch size override (divided over the ranks like parallel.cpp:284-293)")
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--display", type=int, default=0, help="iterations between loss lines (default: the solver file's `display`)")
    ap.add_argument("--seed", type=int, default=-1, help="default: the solver file's random_seed, else 1701")
    ap.add_argument("--snapshot", "-snapshot", default="", help="solver state (.solverstate) to resume training from")
    ap.add_argument("--weights", "-weights", default="", help="pretrained weights (.caffemodel) to fine-tune from, or to score (test)")
    ap.add_argument("--snapshot_prefix", default="", help="write <prefix>_iter_<N>.caffemodel/.solverstate after the last iteration")
    args = ap.parse_args()
    {"train": cmd_train, "test": cmd_test, "time": cmd_time, "device_query": cmd_device_query}[args.command](args)


if __name__ == "__main__":
    main()
