"""b2c_conv_backward_filter_split against b2c_conv_backward_filter, bit for bit.

The split entry point converts dY of 3x3 layers to bf16 hi / lo planes once per call when the staged weight-gradient kernel would
otherwise convert each block in many CTAs (one per 8-channel input tile); the kernel then lands those planes straight in its A tiles.  The
hi / lo values, the MMA order, the 512-pixel promotion and the split-K plan are the same, so dW must keep every bit: each case
runs both entry points on the same inputs, on top of the same non-zero dW0, and compares the int32 views.  Every staged-route
layer of ResNet-50 at N = 64 is covered, and the edge shapes: 64-channel outputs (the second MMA warpgroup's rows are all past O
and it issues no MMAs), O and C off the tile sizes, 7x7 and 14x14 maps, N = 1, one split and several, and the routes that do not
pre-split (few channel tiles, 1x1, both compaction routes), where the split entry point must run the same kernel.  One case per
pre-split regime also meets the float64 oracle at the 1e-4 bar of tests/test_wgrad_schedule_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import oracle as o
from cases import make, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402
from caffe_mpi_b200.shapes import RESNET50  # noqa: E402

TOL = 1e-4


def conv(N, C, H, O, k, s=1):
    return dict(N=N, Cin=C, H=H, W=H, O=O, k=k, s=s, p=k // 2, d=1, G=1, bias=False)


def resnet_cases():
    out = []
    for (_, C, H, O, k, s, p, G, _) in RESNET50:
        c = conv(64, C, H, O, k, s)
        if m.ConvDesc(make(capi, c)).wgrad_plan()["route"] in ("staged_3x3", "staged_3x3_plane", "staged_1x1", "staged_1x1_plane",
                                                                 "compact_staged"):
            out.append((f"r50_C{C}_H{H}_O{O}_k{k}_s{s}", c, None))
    return out


# (id, shape, regime the plan must show: a predicate over ConvDesc.wgrad_plan())
EDGE = [
    ("s3_O64", conv(8, 64, 16, 64, 3), lambda q: q["route"] == "staged_3x3" and q["presplit_dy"] and q["splits"] > 1),
    ("s3_O200_C84", conv(4, 84, 16, 200, 3), lambda q: q["route"] == "staged_3x3" and q["presplit_dy"]),
    ("s3_plane_7x7", conv(6, 72, 7, 96, 3), lambda q: q["route"] == "staged_3x3_plane" and q["presplit_dy"]),
    ("s3_14x14_N1_one_split", conv(1, 64, 14, 72, 3), lambda q: q["route"] == "staged_3x3" and q["splits"] == 1 and q["presplit_dy"]),
    ("s3_few_channel_tiles", conv(4, 40, 16, 64, 3), lambda q: q["route"] == "staged_3x3" and not q["presplit_dy"]),
    ("s1_O64_C200", conv(8, 200, 16, 64, 1), lambda q: q["route"] == "staged_1x1" and not q["presplit_dy"]),
    ("s1_plane_7x7", conv(8, 256, 7, 256, 1), lambda q: q["route"] == "staged_1x1_plane" and not q["presplit_dy"]),
    ("compact_staged", conv(4, 256, 16, 512, 1, 2), lambda q: q["route"] == "compact_staged" and not q["presplit_dy"]),
    ("compact_tma", conv(4, 16, 12, 136, 1, 2), lambda q: q["route"] == "compact_tma" and not q["presplit_dy"]),
]
# one case per pre-split regime that also meets the float64 oracle
ORACLE = {"s3_O64", "s3_O200_C84", "s3_plane_7x7"}


def both(c, dw0, x, dy):
    d = m.ConvDesc(make(capi, c))
    a = dw0.clone()
    b = dw0.clone()
    d.backward_filter(x, dy, a)
    d.backward_filter_split(x, dy, b)
    torch.cuda.synchronize()
    return d, a, b


def inputs(c, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = make(capi, c)
    x = torch.randn(p.x_shape(), device="cuda", generator=g)
    dy = torch.randn(p.y_shape(), device="cuda", generator=g)
    dw0 = torch.randn(p.w_shape(), device="cuda", generator=g)
    return x, dy, dw0


@pytest.mark.parametrize("cid,c,_", resnet_cases(), ids=lambda v: v if isinstance(v, str) else "")
def test_resnet50_layer_bitwise(cid, c, _):
    x, dy, dw0 = inputs(c, 11)
    d, a, b = both(c, dw0, x, dy)
    assert (d.wgrad_split_bytes() > 0) == d.wgrad_plan()["presplit_dy"] == (c["k"] == 3)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not torch.equal(a, dw0)


@pytest.mark.parametrize("cid,c,regime", EDGE, ids=[e[0] for e in EDGE])
def test_edge_shape_bitwise(cid, c, regime):
    d = m.ConvDesc(make(capi, c))
    q = d.wgrad_plan()
    assert regime(q), q
    x, dy, dw0 = inputs(c, 5)
    _, a, b = both(c, dw0, x, dy)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    if cid in ORACLE:
        po = make(o, c)
        want, _, _ = o.conv_backward(po, x.cpu().numpy(), np.zeros(po.w_shape(), np.float32), dy.cpu().numpy(),
                                     dw=dw0.cpu().numpy(), want_dx=False, acc64=True)
        err = rel_err(b.cpu().numpy(), want)
        assert err < TOL, err
    # a second call on top of the first (the split buffer then holds the previous planes)
    d.backward_filter(x, dy, a)
    d.backward_filter_split(x, dy, b)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_no_stuck_waits():
    """after the cases above, no tensor-core kernel recorded an mbarrier timeout"""
    c = conv(8, 256, 7, 256, 1)
    x, dy, dw0 = inputs(c, 3)
    both(c, dw0, x, dy)
    buf = (C.c_uint * 512)()
    assert m.lib().b2c_debug_mbar_timeouts(buf, 512) == 0
