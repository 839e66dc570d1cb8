"""Periodic testing in `caffe.py train`, the parts that need no GPU: the test points of schedule() against a line-by-line restatement of
Solver::Step / Solve, the solver's testing fields (repeated test_iter, the test_interval check, the fields that are not built, the
reference's five model solver files), and the layout of the test lines."""
import importlib.util
import os

import numpy as np
import pytest

from caffe_mpi_b200 import host_api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "reference_models")
_spec = importlib.util.spec_from_file_location("caffe_cli_periodic", os.path.join(ROOT, "tools", "caffe.py"))
cli = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(cli)


def reference_events(start, end, display, snapshot, test_interval):
    """Solver::Step(end - start) then Solve's tail (solver.cpp:229-345,395-425), line by line, for a run that starts fresh at 0 or
    resumes (iterations_last_ = -1) at `start`.  The loss line follows the shell's convention: after the step that brings the counter
    to a multiple of `display`, and after the last one."""
    ev, it = [], start
    iterations_last = -1 if start > 0 else 0
    while it < end:
        if it == 0:
            ev.append(("test", it, "initial"))                                  # TestAll(1)
        elif test_interval and it % test_interval == 0 and iterations_last >= 0:
            ev.append(("test", it, "full"))                                     # TestAll(0)
        if iterations_last < 0:
            iterations_last = it                                                # first_loop
        ev.append(("step", it))
        it += 1
        if (display and it % display == 0) or it == end:
            ev.append(("show", it))
        if snapshot and it % snapshot == 0:
            ev.append(("snap", it))
    if test_interval and it % test_interval == 0:
        ev.append(("test", it, "final"))                                        # Solve's extra pass
    return ev


def shell_events(plan):
    ev = []
    for n, it, show, snap, test in plan:
        if test == "final":
            ev.append(("test", it, "final"))
            continue
        if test:
            ev.append(("test", it - n, test))
        ev += [("step", i) for i in range(it - n, it)]
        if show:
            ev.append(("show", it))
        if snap:
            ev.append(("snap", it))
    return ev


@pytest.mark.parametrize("start,end,display,snapshot,interval", [
    (0, 10, 0, 0, 2),          # a start at 0: the one-batch pass at 0, full passes at 2, 4, 6, 8, the closing pass at 10
    (4, 12, 0, 0, 2),          # a resume at a multiple of test_interval: no pass at 4
    (6, 11, 0, 0, 4),          # --iterations=5 from a snapshot at 6: a pass at 8, none at the end (11)
    (0, 12, 4, 4, 4),          # display and snapshot on the test points: loss line, snapshot, then the pass
    (0, 12, 3, 6, 4),
    (0, 10, 0, 0, 3),          # test_interval does not divide max_iter: no closing pass
    (0, 10, 7, 5, 3),
    (8, 8, 0, 0, 4),           # nothing left to run: Solve's closing pass only
    (0, 1, 1, 1, 1),
])
def test_schedule_places_the_test_passes_where_solver_step_and_solve_do(start, end, display, snapshot, interval):
    plan = list(cli.schedule(start, end, display, snapshot, interval))
    assert shell_events(plan) == reference_events(start, end, display, snapshot, interval)
    assert list(cli.schedule(start, end, display, snapshot, 0)) == list(cli.schedule(start, end, display, snapshot))   # no test nets: today's plan


def test_test_points_split_the_chunks_without_moving_display_or_snapshot():
    assert list(cli.schedule(0, 6, 3, 0, 2)) == [(2, 2, False, False, "initial"), (1, 3, True, False, "full"), (1, 4, False, False, None),
                                                 (2, 6, True, False, "full"), (0, 6, False, False, "final")]
    assert list(cli.schedule(0, 6, 3, 0)) == [(3, 3, True, False), (3, 6, True, False)]


SOLVER = 'net: "n.prototxt" base_lr: 0.01 lr_policy: "fixed" max_iter: 10 '


def test_solver_reads_repeated_test_iter_and_the_test_fields():
    d = host_api.solver_describe(host_api.open_solver(SOLVER + "test_iter: 5 test_iter: 7 test_interval: 3 test_compute_loss: true", True)[0])
    assert (d["test_iter"], d["test_interval"], d["test_compute_loss"]) == ([5, 7], 3, True)
    d = host_api.solver_describe(host_api.open_solver(SOLVER, True)[0])
    assert (d["test_iter"], d["test_interval"], d["test_compute_loss"]) == ([], 0, False)
    d = host_api.solver_describe(host_api.open_solver(SOLVER + "test_interval: 100", True)[0])    # an interval without test nets
    assert (d["test_iter"], d["test_interval"]) == ([], 100)


@pytest.mark.parametrize("extra", ["test_iter: 5", "test_iter: 5 test_interval: 0", "test_iter: 5 test_interval: -2"])
def test_test_iter_needs_a_positive_test_interval(extra):
    with pytest.raises(host_api.HostError, match="test_interval > 0"):
        host_api.open_solver(SOLVER + extra, True)


@pytest.mark.parametrize("field,name", [('test_net: "t.prototxt"', "test_net"), ('test_net_param { name: "t" }', "test_net_param"),
                                        ('test_state { stage: "val" }', "test_state")])
def test_test_net_files_and_states_are_refused_by_train(field, name, tmp_path):
    """The solver still parses (its hyperparameters are readable, e.g. mnist_autoencoder_solver_*.prototxt with their test_state
    stages), but `caffe.py train` will not build test nets from anything but `net`."""
    d = host_api.solver_describe(host_api.open_solver(SOLVER + "test_iter: 5 test_interval: 3 " + field, True)[0])
    assert d["test_fields_not_built"] == [name]
    s = tmp_path / "solver.prototxt"
    s.write_text(SOLVER + "test_iter: 5 test_interval: 3 " + field)
    import subprocess
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "caffe.py"), "train", "--solver=%s" % s], capture_output=True, text=True,
                       cwd=str(tmp_path), timeout=120)
    assert r.returncode != 0 and ("SolverParameter.%s is not built" % name) in r.stderr


@pytest.mark.parametrize("path,test_iter,interval", [
    ("models/resnet50/solver.prototxt", 1562, 20000), ("models/bvlc_alexnet/solver.prototxt", 1562, 5000),
    ("models/vgg16/solver.prototxt", 1563, 20000), ("models/bvlc_googlenet/solver.prototxt", 10000, 4000),
    ("models/cifar10_nv/cifar10_nv_solver.prototxt", 20, 400)])
def test_reference_solver_files_carry_their_test_schedule(path, test_iter, interval):
    d = host_api.solver_describe(host_api.open_solver(os.path.join(REF, path))[0])
    assert (d["test_iter"], d["test_interval"], d["test_compute_loss"]) == ([test_iter], interval, False)


def test_test_lines_follow_the_reference_layout():
    outputs = [("accuracy", 0.0, 1), ("loss", 1.0, 1), ("loss1/loss1", 0.3, 2)]
    lines = cli.test_net_lines(outputs, np.array([0.5, 2.25, 3.0, 1.5], np.float32), 2.75, True)
    assert lines == ["Test loss: 2.75", "    Test net output #0: accuracy = 0.5", "    Test net output #1: loss = 2.25 (* 1 = 2.25 loss)",
                     "    Test net output #2: loss1/loss1 = 3 (* 0.3 = 0.9 loss)", "    Test net output #3: loss1/loss1 = 1.5 (* 0.3 = 0.45 loss)"]
    assert cli.test_net_lines(outputs[:1], [0.25], 0.0, False) == ["    Test net output #0: accuracy = 0.25"]
