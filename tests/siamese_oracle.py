"""float64 forms of the ContrastiveLoss and Slice layers (contrastive_loss_layer.cpp, slice_layer.cpp) and a siamese-shaped net
(Slice -> two conv towers that share every weight by name -> ContrastiveLoss), the oracles of tests/test_siamese_*.py."""
import numpy as np


def similar(y):
    """the reference's static_cast<int>(y) != 0: truncation toward zero, so 0.7 is dissimilar and -1 similar"""
    return np.trunc(np.asarray(y, np.float64)) != 0


def contrastive_forward(a, b, y, margin=1.0, legacy=False):
    """-> (loss, diff [N, C], dist_sq [N])"""
    a = np.asarray(a, np.float64).reshape(len(a), -1)
    b = np.asarray(b, np.float64).reshape(len(b), -1)
    diff = a - b
    d2 = (diff * diff).sum(axis=1)
    if legacy:
        dis = np.maximum(margin - d2, 0.0)
    else:
        dis = np.maximum(margin - np.sqrt(d2), 0.0) ** 2
    terms = np.where(similar(y), d2, dis)
    return terms.sum() / a.shape[0] / 2.0, diff, d2


def contrastive_backward(diff, d2, y, margin=1.0, legacy=False, loss_weight=1.0):
    """-> (da, db) of Backward_cpu with alpha = loss_weight / N (the 1e-4 in the dissimilar factor is the reference's)"""
    n = diff.shape[0]
    alpha = loss_weight / n
    dist = np.sqrt(d2)
    if legacy:
        coef = np.where(margin - d2 > 0, -alpha, 0.0)
    else:
        md = margin - dist
        coef = np.where(md > 0, -alpha * md / (dist + 1e-4), 0.0)
    coef = np.where(similar(y), alpha, coef)
    da = coef[:, None] * diff
    return da, -da


def slice_forward(x, axis, points):
    """the tops of slice_layer.cpp: split `x` along `axis` at `points` (np.split's indices)"""
    return np.split(x, points, axis=axis)


def slice_backward(top_diffs, axis):
    return np.concatenate(top_diffs, axis=axis)


# ---------------------------------------------------------------------------------------------------------------- siamese net
def siamese_prototxt(N=8, H=12, conv_out=4, ip_out=16, feat=3, margin=1.0, legacy=False, names=True, lr_b=2):
    """Input pair_data [N, 2, H, H] + sim [N] -> Slice(axis 1) -> per half: conv 3x3 -> MAX pool 2 -> InnerProduct -> ReLU ->
    InnerProduct(feat); the _p tower names every blob like the first one -> ContrastiveLoss"""
    def p(nm, lr):
        return 'param { %slr_mult: %g } ' % ('name: "%s" ' % nm if names else "", lr)

    s = ('name: "siamese_mini"\nlayer { name: "pair" type: "Input" top: "pair_data" top: "sim" input_param { shape { dim: %d dim: 2 '
         'dim: %d dim: %d } shape { dim: %d } } }\n' % (N, H, H, N))
    s += 'layer { name: "slice_pair" type: "Slice" bottom: "pair_data" top: "data" top: "data_p" slice_param { slice_dim: 1 slice_point: 1 } }\n'
    for sfx in ("", "_p"):
        s += ('layer { name: "conv1%s" type: "Convolution" bottom: "data%s" top: "conv1%s" %s%s convolution_param { num_output: %d '
              'kernel_size: 3 weight_filler { type: "xavier" } } }\n' % (sfx, sfx, sfx, p("conv1_w", 1), p("conv1_b", lr_b), conv_out))
        s += ('layer { name: "pool1%s" type: "Pooling" bottom: "conv1%s" top: "pool1%s" pooling_param { pool: MAX kernel_size: 2 '
              'stride: 2 } }\n' % (sfx, sfx, sfx))
        s += ('layer { name: "ip1%s" type: "InnerProduct" bottom: "pool1%s" top: "ip1%s" %s%s inner_product_param { num_output: %d '
              'weight_filler { type: "xavier" } } }\n' % (sfx, sfx, sfx, p("ip1_w", 1), p("ip1_b", lr_b), ip_out))
        s += 'layer { name: "relu1%s" type: "ReLU" bottom: "ip1%s" top: "ip1%s" }\n' % (sfx, sfx, sfx)
        s += ('layer { name: "feat%s" type: "InnerProduct" bottom: "ip1%s" top: "feat%s" %s%s inner_product_param { num_output: %d '
              'weight_filler { type: "xavier" } } }\n' % (sfx, sfx, sfx, p("feat_w", 1), p("feat_b", lr_b), feat))
    s += ('layer { name: "loss" type: "ContrastiveLoss" bottom: "feat" bottom: "feat_p" bottom: "sim" top: "loss" '
          'contrastive_loss_param { margin: %g legacy_version: %s } }\n' % (margin, "true" if legacy else "false"))
    return s


def siamese_param_shapes(H=12, conv_out=4, ip_out=16, feat=3):
    P = (H - 2) // 2
    return [(conv_out, 1, 3, 3), (conv_out,), (ip_out, conv_out * P * P), (ip_out,), (feat, ip_out), (feat,)]


def siamese_forward_backward(params, pair, sim, margin=1.0, legacy=False):
    """float64 loss and the gradient of every owner (the sum over both towers) of the siamese_prototxt net: the loss layer's
    gradient as contrastive_backward states it (with its 1e-4), the towers by torch autograd on the CPU"""
    import torch
    import torch.nn.functional as F
    P = [torch.tensor(np.asarray(p, np.float64), requires_grad=True) for p in params]
    x = torch.tensor(np.asarray(pair, np.float64))

    def tower(h):
        h = F.max_pool2d(F.conv2d(h, P[0], P[1]), 2, 2)
        h = F.relu(F.linear(h.reshape(h.shape[0], -1), P[2], P[3]))
        return F.linear(h, P[4], P[5])

    fa, fb = tower(x[:, 0:1]), tower(x[:, 1:2])
    loss, diff, d2 = contrastive_forward(fa.detach().numpy(), fb.detach().numpy(), sim, margin, legacy)
    da, db = contrastive_backward(diff, d2, sim, margin, legacy)
    torch.autograd.backward([fa, fb], [torch.tensor(da), torch.tensor(db)])
    return float(loss), [p.grad.numpy() for p in P], (fa.detach().numpy(), fb.detach().numpy())
