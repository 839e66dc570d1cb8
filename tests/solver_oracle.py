"""CPU oracle of the Nesterov, AdaGrad, RMSProp, AdaDelta and Adam updates, in fp32 numpy: each function restates the reference's
CPU branch of SGDSolver::ApplyUpdate for one learnable blob -- the scalings the exchange applies first (grad_scale: Net::ReduceBucket's
1/solver_count and Net::ReduceAndUpdate's 1/global_grad_scale, src/caffe/net.cpp:815-817,899-912), Normalize (sgd_solver.cpp:152-158,
x 1/iter_size), Regularize (sgd_solver.cpp:161-192, L2: g += decay*w, L1: g += decay*sign(w)), then the solver's own
ComputeUpdateValue CPU branch, Blob::Update (w -= g, src/caffe/blob.cpp:129-154) and clear_grads (g = 0).  oracle.sgd_update is the
SGD counterpart.  Every array op below is one caffe_cpu_* call of the reference, evaluated in fp32 in the same order.

Each function takes (g, w, h[, h2]) and returns new arrays (g, w, h[, h2]); the inputs are not modified."""
import numpy as np

F = np.float32


def _prologue(g, w, local_decay, l2, grad_scale, iter_size):
    g = np.array(g, np.float32).reshape(-1)
    w = np.array(w, np.float32).reshape(-1)
    if grad_scale != 1.0:
        g = g * F(grad_scale)
    if iter_size != 1:
        g = g * F(F(1.0) / F(iter_size))                                 # Normalize, sgd_solver.cpp:152-158
    if local_decay != 0.0:                                               # Regularize, sgd_solver.cpp:161-192
        reg = w if l2 else np.sign(w).astype(np.float32)
        g = F(local_decay) * reg + g                                     # caffe_axpy(decay, reg, diff)
    return g, w


def _epilogue(g, w, clear_grads):
    w = w - g                                                            # Blob::Update: caffe_axpy(-1, diff, data)
    return (np.zeros_like(g) if clear_grads else g), w


def _h(a):
    return np.array(a, np.float32).reshape(-1)


def nesterov_update(g, w, h, momentum, local_rate, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    """nesterov_solver.cpp:20-38 (CPU branch)."""
    g, w = _prologue(g, w, local_decay, l2, grad_scale, iter_size)
    h = _h(h)
    m = F(momentum)
    update = h.copy()                                                    # caffe_copy(history, update)
    h = F(local_rate) * g + m * h                                        # caffe_cpu_axpby(local_rate, diff, momentum, history)
    update = F(F(1.0) + m) * h + F(-m) * update                          # caffe_cpu_axpby(1+momentum, history, -momentum, update)
    g, w = _epilogue(update, w, clear_grads)                             # caffe_copy(update, diff)
    return g, w, h


def adagrad_update(g, w, h, delta, local_rate, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    """adagrad_solver.cpp:18-42 (CPU branch); delta = max(delta, 1e-3) (:22)."""
    g, w = _prologue(g, w, local_decay, l2, grad_scale, iter_size)
    h = _h(h)
    d = max(F(delta), F(0.001))
    update = g * g                                                       # caffe_powx(diff, 2, update)
    h = update + h                                                       # caffe_add(update, history, history)
    update = np.sqrt(h)                                                  # caffe_powx(history, 0.5, update)
    update = update + d                                                  # caffe_add_scalar(delta, update)
    update = g / update                                                  # caffe_div(diff, update, update)
    g, w = _epilogue(F(local_rate) * update, w, clear_grads)             # caffe_cpu_axpby(local_rate, update, 0, diff)
    return g, w, h


def rmsprop_update(g, w, h, rms_decay, delta, local_rate, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    """rmsprop_solver.cpp:21-48 (CPU branch); delta = max(delta, 1e-4) (:25)."""
    g, w = _prologue(g, w, local_decay, l2, grad_scale, iter_size)
    h = _h(h)
    d = max(F(delta), F(0.0001))
    rho = F(rms_decay)
    update = g * g                                                       # caffe_powx(diff, 2, update)
    h = F(F(1.0) - rho) * update + rho * h                               # caffe_cpu_axpby(1-rms_decay, update, rms_decay, history)
    update = np.sqrt(h) + d                                              # caffe_powx(history, 0.5) + caffe_add_scalar(delta)
    update = g / update                                                  # caffe_div(diff, update, update)
    g, w = _epilogue(F(local_rate) * update, w, clear_grads)             # caffe_cpu_axpby(local_rate, update, 0, diff)
    return g, w, h


def adadelta_update(g, w, h, h2, momentum, delta, local_rate, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    """adadelta_solver.cpp:31-81 (CPU branch); h is the gradient history, h2 the update history; delta = max(delta, 1e-3) (:36)."""
    g, w = _prologue(g, w, local_decay, l2, grad_scale, iter_size)
    h, h2 = _h(h), _h(h2)
    d = max(F(delta), F(0.001))
    m = F(momentum)
    update = g * g                                                       # caffe_powx(diff, 2, update)
    h = F(F(1.0) - m) * update + m * h                                   # caffe_cpu_axpby(1-momentum, update, momentum, history)
    update = d + h2                                                      # caffe_set(delta, temp); caffe_add(temp, update_history, update)
    temp = d + h                                                         # caffe_add(temp, history, temp)
    update = update / temp                                               # caffe_div(update, temp, update)
    update = np.sqrt(update)                                             # caffe_powx(update, 0.5, update)
    g = g * update                                                       # caffe_mul(diff, update, diff)
    update = g * g                                                       # caffe_powx(diff, 2, update)
    h2 = F(F(1.0) - m) * update + m * h2                                 # caffe_cpu_axpby(1-momentum, update, momentum, update_history)
    g, w = _epilogue(F(local_rate) * g, w, clear_grads)                  # caffe_cpu_scale(local_rate, diff, diff)
    return g, w, h, h2


def adam_correction(beta1, beta2, t):
    """adam_solver.cpp:42-43: sqrt(1 - beta2^t) / (1 - beta1^t), t = iter + 1."""
    return F(np.sqrt(F(1.0) - F(beta2) ** F(t)) / (F(1.0) - F(beta1) ** F(t)))


def adam_update(g, w, m, v, beta1, beta2, delta, local_rate, t, local_decay, l2=True, grad_scale=1.0, iter_size=1, clear_grads=True):
    """adam_solver.cpp:25-62 (CPU branch); m, v are history[i] and history[i + np]; t = iter + 1; eps_hat = max(delta, 1e-4) (:45)."""
    g, w = _prologue(g, w, local_decay, l2, grad_scale, iter_size)
    m, v = _h(m), _h(v)
    b1, b2 = F(beta1), F(beta2)
    eps = max(F(delta), F(0.0001))
    m = F(F(1.0) - b1) * g + b1 * m                                      # caffe_cpu_axpby(1-beta1, diff, beta1, val_m)
    val_t = g * g                                                        # caffe_mul(diff, diff, val_t)
    v = F(F(1.0) - b2) * val_t + b2 * v                                  # caffe_cpu_axpby(1-beta2, val_t, beta2, val_v)
    val_t = np.sqrt(v) + eps                                             # caffe_powx(val_v, 0.5) + caffe_add_scalar(eps_hat)
    val_t = m / val_t                                                    # caffe_div(val_m, val_t, val_t)
    rate = F(F(local_rate) * adam_correction(beta1, beta2, t))
    g, w = _epilogue(rate * val_t, w, clear_grads)                       # caffe_cpu_scale(local_rate*correction, val_t, diff)
    return g, w, m, v


def update(kind, g, w, h, h2, hp, local_rate, local_decay, t=1, **kw):
    """One solver step of type `kind` (SGD, Nesterov, AdaGrad, RMSProp, AdaDelta, Adam) -> (g, w, h, h2); h2 is None for the one-history
    solvers.  hp: dict with the SolverParameter fields momentum, delta, rms_decay, momentum2."""
    import oracle
    if kind == "SGD":
        g, w, h = oracle.sgd_update(g, w, h, hp["momentum"], local_rate, local_decay, **kw)
        return g, w, h, None
    if kind == "Nesterov":
        return nesterov_update(g, w, h, hp["momentum"], local_rate, local_decay, **kw) + (None,)
    if kind == "AdaGrad":
        return adagrad_update(g, w, h, hp["delta"], local_rate, local_decay, **kw) + (None,)
    if kind == "RMSProp":
        return rmsprop_update(g, w, h, hp["rms_decay"], hp["delta"], local_rate, local_decay, **kw) + (None,)
    if kind == "AdaDelta":
        return adadelta_update(g, w, h, h2, hp["momentum"], hp["delta"], local_rate, local_decay, **kw)
    if kind == "Adam":
        return adam_update(g, w, h, h2, hp["momentum"], hp["momentum2"], hp["delta"], local_rate, t, local_decay, **kw)
    raise ValueError(kind)


KINDS = ("SGD", "Nesterov", "AdaGrad", "RMSProp", "AdaDelta", "Adam")
TWO_HISTORIES = ("AdaDelta", "Adam")
