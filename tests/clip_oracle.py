"""Oracle of SolverParameter.clip_gradients as this project defines it (caffe.proto:241, BVLC Caffe's SGDSolver::ClipGradients): one L2
norm of the whole reduced gradient per iteration, every parameter scaled by the same factor.

- S = sum of g^2 over every parameter, in float64 with one rounding (math.fsum of the exact float64 squares);
- norm = float32(sqrt(s_n^2 * S)), s_n = 1 / (solver_count * global_grad_scale): the scale the net applies before ClipGradients;
- factor = clip / norm in float32 when norm > clip (float32 comparison), else 1 -- so a NaN norm does not scale;
- the update then runs with grad_scale' = float32(grad_scale * factor); weight decay is not scaled (Regularize comes after)."""
import math

import numpy as np

F = np.float32


def _squares(grads, chunk=1 << 20):
    for g in grads:
        g = np.asarray(g, np.float32).reshape(-1)
        for i in range(0, g.size, chunk):
            yield from np.square(g[i:i + chunk].astype(np.float64)).tolist()     # each float32 square is exact in float64


def sumsq(grads):
    """float64 sum of squares over every array in `grads`, rounded once"""
    return math.fsum(_squares(grads))


def clip_factor(grads, clip, s_n=1.0):
    """(norm, factor) as float32 for the float32 gradients `grads` (a list of arrays) and clip_gradients `clip`"""
    S = sumsq(grads)
    norm = F(math.sqrt((s_n * s_n) * S))
    c = F(clip)
    return norm, (c / norm if norm > c else F(1.0))


def clipped_grad_scale(grad_scale, factor):
    """the update's grad_scale under clipping: one float32 product"""
    return F(F(grad_scale) * F(factor))


def replay(kind, spec, params, data, label, steps, base_lr, clip, hp, decay=0.0005, iter_size=1, s_n=1.0):
    """netoracle forward / backward + this clip + the solver oracle, lr_policy fixed: (losses, params, h, h2, norms).  With iter_size
    the diffs of iter_size identical micro-batches accumulate before the clip, as TrainNet::Step accumulates them."""
    import netoracle as no
    import solver_oracle as so
    p = [x.copy() for x in params]
    h = [np.zeros(x.size, F) for x in params]
    h2 = [np.zeros(x.size, F) for x in params]
    losses, norms = [], []
    for it in range(steps):
        loss, grads, _, _ = no.forward_backward(spec, p, data, label)
        losses.append(loss)
        grads = [np.asarray(g, F) for g in grads]
        for _ in range(iter_size - 1):
            grads = [g + g0 for g, g0 in zip(grads, [np.asarray(x, F) for x in no.forward_backward(spec, p, data, label)[1]])]
        norm, factor = clip_factor(grads, clip, s_n)
        norms.append(norm)
        for i, g in enumerate(grads):
            _, w, h[i], b = so.update(kind, g, p[i], h[i], h2[i], hp, base_lr, decay, t=it + 1, grad_scale=float(factor),
                                      iter_size=iter_size)
            p[i] = w.reshape(p[i].shape)
            if b is not None:
                h2[i] = b
    return losses, p, h, h2, norms
