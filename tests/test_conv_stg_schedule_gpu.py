"""Schedule edge cases of the staged forward / data-gradient kernel (csrc/conv_tc_stg.cu) against the CPU oracle.

The kernel is persistent (one CTA per SM, tiles strided by the grid) and its two consumer warpgroups take turns over a CTA's
tiles: warpgroup 0 the even ones, warpgroup 1 the odd ones.  So the tile count per CTA matters: 1 tile (warpgroup 1 idle),
an even or odd number, the grid one short of or one past the SM count.  The other cases cover each epilogue path: the TMA
tensor store (tile inside one image), the 16-byte st.global path (tile spanning two images), plane mode (7x7 maps, a tile
touching four images), the TMA reduce-add store of backward_data_accumulate, the bias, and channel counts that leave the
last N tile partly empty at N_TILE 32 / 64 / 128."""
import numpy as np
import pytest

import oracle as o
from cases import make, tensors, rel_err

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

TOL = 1e-4


def case(N, C, H, W, O, k, bias=True):
    return dict(N=N, Cin=C, H=H, W=W, O=O, k=k, s=1, p=k // 2, d=1, G=1, bias=bias)


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    torch.cuda.synchronize()
    return t.cpu().numpy()


def check_fwd_dgrad(c, rng, dgrad_staged=True):
    """forward and data gradient against the oracle at 1e-4, and each bit-identical on a second run.  The data gradient
    takes the staged kernel only when O % 32 == 0 (its input channels); dgrad_staged=False is a forward-only case."""
    po, pc = make(o, c), make(capi, c)
    x, w, b, dy = tensors(rng, po)
    want_y = o.conv_forward(po, x, w, b, acc64=True)
    _, _, want_dx = o.conv_backward(po, x, w, dy, acc64=True)
    d = m.ConvDesc(pc)
    assert d.backward_data_accumulate_supported() == dgrad_staged
    X, Wt, DY = dev(x), dev(w), dev(dy)
    Bv = dev(b) if b is not None else None
    Y = dev(np.full(po.y_shape(), 3.0, np.float32))
    DX = dev(np.full(po.x_shape(), 3.0, np.float32))
    d.forward(X, Wt, Bv, Y)
    d.backward_data(DY, Wt, DX)
    assert d.algo_used(0) == capi.ALGO_TCGEN05 and d.algo_used(1) == capi.ALGO_TCGEN05
    assert rel_err(host(Y), want_y) < TOL, ("y", rel_err(host(Y), want_y))
    assert rel_err(host(DX), want_dx) < TOL, ("dx", rel_err(host(DX), want_dx))
    Y2, DX2 = torch.empty_like(Y), torch.empty_like(DX)
    d.forward(X, Wt, Bv, Y2)
    d.backward_data(DY, Wt, DX2)
    assert torch.equal(Y, Y2) and torch.equal(DX, DX2)


# H x W = 8 x 16 = 128 pixels: one M tile per image, every tile inside one image; O <= 128: one N tile.  So N images give
# exactly N tiles, and the grid is min(N, SMs).
@pytest.mark.parametrize("tiles", ["1", "sms-1", "sms+1", "2sms+1"])
@pytest.mark.parametrize("C,O,k", [(32, 128, 1), (64, 96, 3)], ids=["1x1_nkb1", "3x3_o96"])
def test_tiles_per_cta(rng, sms, tiles, C, O, k):
    N = {"1": 1, "sms-1": sms - 1, "sms+1": sms + 1, "2sms+1": 2 * sms + 1}[tiles]
    check_fwd_dgrad(case(N, C, 8, 16, O, k), rng)


# 12 x 12 = 144 pixels: most tiles span two images (st.global epilogue); C = 64 with 1x1 is nkb = 1
@pytest.mark.parametrize("C,O,k", [(64, 32, 1), (32, 64, 3), (96, 160, 3), (64, 40, 1)],
                         ids=["1x1_nkb1_nt32", "3x3_nt64", "3x3_nt128_partial", "1x1_nt64_partial_fwd"])
def test_tiles_spanning_two_images(rng, sms, C, O, k):
    check_fwd_dgrad(case(2 * sms // 9 + 3, C, 12, 12, O, k), rng, dgrad_staged=O % 32 == 0)


# 7 x 7 maps: plane mode; the 128-row tile starting at pixel 128 covers images 2..5
@pytest.mark.parametrize("C,O,k,N", [(64, 32, 1, 8), (32, 128, 3, 9), (64, 224, 1, 300)],
                         ids=["1x1_nt32", "3x3_nt128", "1x1_nt128_partial_two_tiles_per_cta"])
def test_plane_mode(rng, C, O, k, N):
    check_fwd_dgrad(case(N, C, 7, 7, O, k), rng)


@pytest.mark.parametrize("N,C,H,W,O,k", [(3, 32, 8, 16, 64, 1), (5, 96, 12, 12, 64, 3), (9, 160, 7, 7, 32, 1),
                                         (4, 64, 16, 16, 32, 3)],
                         ids=["in_image_nt32", "span_nt128_partial", "plane_nt128_partial", "in_image_nt64"])
def test_backward_data_accumulate(rng, N, C, H, W, O, k):
    """dx0 + dgrad through the accumulate path == dx0 + the plain dgrad, bit for bit, and within 1e-4 of the oracle"""
    c = case(N, C, H, W, O, k, bias=False)
    po, pc = make(o, c), make(capi, c)
    x, w, _, dy = tensors(rng, po)
    _, _, want_dx = o.conv_backward(po, x, w, dy, acc64=True)
    dx0 = rng.standard_normal(po.x_shape()).astype(np.float32)
    d = m.ConvDesc(pc)
    assert d.backward_data_accumulate_supported()
    Wt, DY = dev(w), dev(dy)
    DX = torch.empty(po.x_shape(), device="cuda")
    d.backward_data(DY, Wt, DX)
    ACC = dev(dx0)
    d.backward_data_accumulate(DY, Wt, ACC)
    assert torch.equal(ACC, dev(dx0) + DX)
    assert rel_err(host(ACC) - dx0, want_dx) < TOL
