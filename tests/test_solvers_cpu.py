"""The Nesterov, AdaGrad, RMSProp, AdaDelta and Adam solvers without a GPU: the fp32 oracle (tests/solver_oracle.py) against the
double-precision closed form of the reference's solver test, and solver.prototxt parsing (`type`, the legacy `solver_type` enum, the
reference's sanity checks)."""
import os

import numpy as np
import pytest

import solver_oracle as so
from caffe_mpi_b200 import host_api as h

REF = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_models")
HP = dict(momentum=0.9, delta=1e-3, rms_decay=0.95, momentum2=0.999)


def closed_form_step(kind, w, gr, hist, hist2, lr, t, hp):
    """ComputeLeastSquaresUpdate (src/caffe/test/test_gradient_based_solver.cpp:228-364) per element in float64: the update value
    from the regularised gradient `gr` and the solver's histories before the step.  delta is the clamped one."""
    w, gr, hv = (np.asarray(a, np.float64) for a in (w, gr, hist))
    m, d = hp["momentum"], hp["delta"]
    if kind == "SGD":
        u = lr * gr + m * hv
    elif kind == "Nesterov":
        u = (1 + m) * (lr * gr + m * hv) - m * hv
    elif kind == "AdaGrad":
        u = lr * gr / (np.sqrt(hv + gr * gr) + max(d, 1e-3))
    elif kind == "RMSProp":
        rho = hp["rms_decay"]
        u = lr * gr / (np.sqrt(rho * hv + gr * gr * (1 - rho)) + max(d, 1e-4))
    elif kind == "AdaDelta":
        d = max(d, 1e-3)
        u = gr * np.sqrt((np.asarray(hist2, np.float64) + d) / (m * hv + (1 - m) * gr * gr + d)) * lr
    else:
        b2 = hp["momentum2"]
        val_m = (1 - m) * gr + m * hv
        val_v = (1 - b2) * gr * gr + b2 * np.asarray(hist2, np.float64)
        u = lr * np.sqrt(1 - b2 ** t) / (1 - m ** t) * val_m / (np.sqrt(val_v) + max(d, 1e-4))
    return w - u


@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
@pytest.mark.parametrize("iter_size,grad_scale", [(1, 1.0), (3, 0.5)])
def test_oracle_matches_least_squares_closed_form(kind, l2, iter_size, grad_scale):
    """Several iterations of least squares (X w + b ~ y) with weight decay: every step of the oracle equals the closed form on the
    oracle's own histories.  The oracle receives the raw accumulated gradient (iter_size backward passes, before the exchange's
    grad_scale) and must undo both scalings itself."""
    rng = np.random.default_rng(1701)
    N, D = 8, 12
    X = np.concatenate([rng.standard_normal((N, D)), np.ones((N, 1))], 1).astype(np.float32)
    y = rng.standard_normal(N).astype(np.float32)
    w = (rng.standard_normal(D + 1) * 0.5).astype(np.float32)
    hist = np.zeros_like(w)
    hist2 = np.zeros_like(w) if kind in so.TWO_HISTORIES else None
    hp = dict(HP, momentum=0.0 if kind in ("AdaGrad", "RMSProp") else HP["momentum"])
    lr, wd = 0.05, 0.01
    for it in range(4):
        X64 = X.astype(np.float64)
        grad = X64.T @ (X64 @ w.astype(np.float64) - y) / N                      # d/dw of 1/(2N) |Xw - y|^2
        raw = (grad * iter_size / grad_scale).astype(np.float32)
        g1, w1, h1, h21 = so.update(kind, raw, w, hist, hist2, hp, lr, wd, t=it + 1, l2=l2, grad_scale=grad_scale,
                                    iter_size=iter_size, clear_grads=False)
        reg = w.astype(np.float64) if l2 else np.sign(w).astype(np.float64)
        want = closed_form_step(kind, w, grad + wd * reg, hist, hist2, lr, it + 1, hp)
        np.testing.assert_allclose(w1, want, rtol=1e-5, atol=1e-6, err_msg=f"{kind} iteration {it}")
        np.testing.assert_allclose(g1, w.astype(np.float64) - want, rtol=1e-4, atol=1e-6)   # the diff holds the step
        w, hist, hist2 = w1, h1, h21
    assert np.isfinite(w).all()


def test_adam_bias_correction_first_steps():
    # fp32, as the reference computes it: 1 - 0.999f^t loses about 13 bits to cancellation at t = 1
    for t in (1, 2, 3):
        assert so.adam_correction(0.9, 0.999, t) == pytest.approx(np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t), rel=2e-5)
    # t = 1 from zero histories: m = (1-b1) g, v = (1-b2) g^2, so the step is lr * g / (|g| + eps_hat / sqrt(1-b2))
    g = np.array([0.5, -2.0, 1e-3], np.float32)
    _, w, m, v = so.adam_update(g, np.zeros(3, np.float32), np.zeros(3), np.zeros(3), 0.9, 0.999, 1e-8, 0.01, 1, 0.0)
    np.testing.assert_allclose(-w, 0.01 * g / (np.abs(g) + 1e-4 / np.sqrt(1 - 0.999)), rtol=1e-5)


# ------------------------------------------------------------------------------------------------------------------- parsing
FIXTURES = [
    # path, type, {field: value}
    ("examples/solvers/adam/solver.prototxt", "Adam", dict(delta=1.0, momentum=0.9, momentum2=0.99, base_lr=0.1)),
    ("examples/solvers/adagrad/solver.prototxt", "AdaGrad", dict(delta=1.0, momentum=0.0, base_lr=0.1, lr_policy="poly")),
    ("examples/solvers/adadelta/solver.prototxt", "AdaDelta", dict(delta=1.0, momentum=0.9, base_lr=0.1, lr_policy="poly")),
    ("examples/mnist/lenet_solver_adam.prototxt", "Adam", dict(momentum=0.9, momentum2=0.999, base_lr=0.001, delta=1e-8)),
    ("examples/mnist/lenet_solver_rmsprop.prototxt", "RMSProp", dict(rms_decay=0.98, momentum=0.0, base_lr=0.01, lr_policy="inv")),
    ("examples/mnist/lenet_adadelta_solver.prototxt", "AdaDelta", dict(delta=1e-6, momentum=0.95, base_lr=1.0)),
    ("examples/mnist/mnist_autoencoder_solver_nesterov.prototxt", "Nesterov", dict(momentum=0.95, base_lr=0.01, lr_policy="step")),
    ("examples/mnist/mnist_autoencoder_solver_adagrad.prototxt", "AdaGrad", dict(base_lr=0.01)),
    ("examples/mnist/mnist_autoencoder_solver_adadelta.prototxt", "AdaDelta", dict(momentum=0.95, delta=1e-8, base_lr=1.0)),
]


@pytest.mark.parametrize("path,kind,fields", FIXTURES, ids=[os.path.basename(os.path.dirname(f[0])) + "/" + os.path.basename(f[0])
                                                            for f in FIXTURES])
def test_reference_solver_files_parse(path, kind, fields):
    s, net = h.open_solver(os.path.join(REF, path))
    d = h.solver_describe(s)
    assert d["type"] == kind and net.endswith(".prototxt")
    for k, v in fields.items():
        assert d[k] == (v if isinstance(v, str) else pytest.approx(v, rel=1e-6)), k
    # the SGD-only entry refuses them, including the legacy solver_type files it used to read as SGD
    with pytest.raises(h.HostError, match="SGD only"):
        h.solver_from_prototxt(os.path.join(REF, path))


@pytest.mark.parametrize("enum,kind", [("SGD", "SGD"), ("NESTEROV", "Nesterov"), ("ADAGRAD", "AdaGrad"), ("RMSPROP", "RMSProp"),
                                       ("ADADELTA", "AdaDelta"), ("ADAM", "Adam")])
def test_legacy_solver_type_and_type_agree(enum, kind):
    a = h.solver_describe(h.open_solver("base_lr: 0.1 solver_type: %s" % enum, is_text=True)[0])
    b = h.solver_describe(h.open_solver('base_lr: 0.1 type: "%s"' % kind, is_text=True)[0])
    assert a["type"] == b["type"] == kind
    assert a["delta"] == pytest.approx(1e-8) and a["momentum2"] == pytest.approx(0.999) and a["rms_decay"] == 0.0


@pytest.mark.parametrize("text,msg", [
    ('type: "Adam" solver_type: ADAM', "cannot be both"),
    ('type: "Adamax"', "known types: SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam"),
    ("solver_type: LBFGS", "Unknown SolverParameter solver_type"),
    ('type: "AdaGrad" momentum: 0.9', "Momentum cannot be used with AdaGrad"),
    ('type: "RMSProp" momentum: 0.5 rms_decay: 0.9', "Momentum cannot be used with RMSProp"),
    ('type: "RMSProp" rms_decay: 1.0', "rms_decay should lie between 0 and 1"),
    ('type: "RMSProp" rms_decay: -0.1', "rms_decay should lie between 0 and 1"),
])
def test_bad_solver_files_are_fatal(text, msg):
    with pytest.raises(h.HostError, match=msg):
        h.open_solver("base_lr: 0.1 " + text, is_text=True)


def test_typed_solver_constructor_checks():
    assert h.solver_describe(h.SGDSolver(type="Adam", momentum=0.9, momentum2=0.99))["momentum2"] == pytest.approx(0.99)
    with pytest.raises(h.HostError, match="Unknown solver type"):
        h.SGDSolver(type="adam")
    with pytest.raises(h.HostError, match="Momentum cannot be used with AdaGrad"):
        h.SGDSolver(type="AdaGrad", momentum=0.9)
