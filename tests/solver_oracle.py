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


# ---- the fused kernels' own order (csrc/sgd.cu), for the per-element suites --------------------------------------------------
# hyperparameters as b2c_solver_hparams names them (delta unclamped); Adam's beta1 / beta2 are SolverParameter momentum / momentum2
KERNEL_HP = dict(momentum=0.9, delta=1e-8, rms_decay=0.95, beta1=0.9, beta2=0.999)
DYADIC_HP = dict(momentum=0.875, delta=1e-8, rms_decay=0.875, beta1=0.875, beta2=63 / 64)


def kernel_fp32(kind, g, w, h, h2, hp, lr, decay, l2=True, grad_scale=1.0, clear_grads=True):
    """numpy fp32, one rounding per operation, in the kernel's order: (g, w, h, h2) after the update.  numpy never contracts a
    product into a sum, so on data where every product that meets a sum is exact (dyadic_inputs) this is what any contraction
    of the kernel must store.  Delta is clamped as b2c_solver_update_arena clamps it."""
    g, w, h = (np.array(a, F).reshape(-1) for a in (g, w, h))
    h2 = np.zeros_like(h) if h2 is None else np.array(h2, F).reshape(-1)
    m, rd, b1, b2 = F(hp["momentum"]), F(hp["rms_decay"]), F(hp["beta1"]), F(hp["beta2"])
    d = max(F(hp["delta"]), F(1e-3) if kind in ("AdaGrad", "AdaDelta") else F(1e-4))
    lr, decay, one = F(lr), F(decay), F(1)
    reg = w if l2 else (w > 0).astype(F) - (w < 0).astype(F)               # sign(+-0) = +0, as (0 < w) - (w < 0)
    gr = g * F(grad_scale) + reg * decay
    with np.errstate(all="ignore"):
        if kind == "SGD":
            h = m * h + lr * gr
            u = h
        elif kind == "Nesterov":
            hi, h = h, m * h + lr * gr
            u = (one + m) * h - m * hi
        elif kind == "AdaGrad":
            h = h + gr * gr
            u = (lr * gr) / (np.sqrt(h) + d)
        elif kind == "RMSProp":
            h = rd * h + ((one - rd) * gr) * gr
            u = (lr * gr) / (np.sqrt(h) + d)
        elif kind == "AdaDelta":
            h = m * h + ((one - m) * gr) * gr
            gr = gr * np.sqrt((h2 + d) / (h + d))
            h2 = m * h2 + ((one - m) * gr) * gr
            u = lr * gr
        else:
            h = h * b1 + gr * (one - b1)
            h2 = h2 * b2 + (gr * gr) * (one - b2)
            u = (lr * h) / (np.sqrt(h2) + d)
        w = w - u
    return (np.zeros_like(g) if clear_grads else u.astype(F)), w.astype(F), h.astype(F), h2.astype(F)


def dyadic_inputs(rng, n, kind):
    """(g, w, h, h2) of small integers times powers of two: with DYADIC_HP, grad_scale 1/8, lr = odd/128 (< 16/128) and decay =
    odd/256 (< 16/256), every product that meets a sum in the kernel is exact (at most 24 significant bits), so every contraction
    gives the same bits -- except AdaDelta's h2 and w, which follow a rounded square root.  w holds +-0."""
    g = rng.integers(-64, 65, n).astype(F) / F(64)
    w = rng.integers(-64, 65, n).astype(F) / F(64)
    w[rng.random(n) < 0.05] = F(-0.0)
    lo = -64 if kind in ("SGD", "Nesterov", "Adam") else 0
    h = rng.integers(lo, 65, n).astype(F) / F(256)
    h2 = rng.integers(0, 65, n).astype(F) / F(256)
    return g, w, h, h2


def dyadic_rates(rng, nseg):
    """distinct per-segment (lr, decay) pairs for dyadic_inputs"""
    pairs = [(F(a) / F(128), F(b) / F(256)) for a in range(1, 16, 2) for b in range(1, 16, 2)]
    idx = rng.permutation(len(pairs))
    return [float(pairs[idx[s % len(pairs)]][0]) for s in range(nseg)], [float(pairs[idx[s % len(pairs)]][1]) for s in range(nseg)]


def wide_inputs(rng, n, kind):
    """(g, w, h, h2) over several binades, with +-0 in w and subnormal g, h and w: data on which the contractions of the kernel
    give different bits (test_oracle checks that every pair of forms differs on it)"""
    def wide():
        return (rng.standard_normal(n) * np.exp2(rng.integers(-8, 4, n))).astype(F)
    g, w, h, h2 = wide(), wide(), wide(), np.abs(wide())
    if kind not in ("SGD", "Nesterov", "Adam"):
        h = np.abs(h)
    sub = (rng.integers(1, 1 << 20, n) * np.exp2(-149)).astype(F)        # subnormals: 2^-149 .. 2^-129
    for a, p in ((g, 0.02), (h, 0.02), (w, 0.02)):
        pick = rng.random(n) < p
        a[pick] = sub[pick] * (np.sign(a[pick]) if a is not h or kind in ("SGD", "Nesterov", "Adam") else 1)
    zero = rng.random(n) < 0.03
    w[zero] = np.where(rng.random(int(zero.sum())) < 0.5, F(0.0), F(-0.0))
    return g, w, h, h2
