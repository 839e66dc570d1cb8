"""CPU tests of the transposed-convolution and Crop oracles (tests/deconv_oracle.py) and of the host-only parts of the C ABI:
descriptor checks, top extents, and the route plan b2c_debug_deconv_plan reports."""
import ctypes as C
import itertools

import numpy as np
import pytest

import caffe_mpi_b200 as m
from caffe_mpi_b200 import capi
import deconv_oracle as do


def _rand(rng, *shape):
    return rng.standard_normal(shape)


# ---- the oracle's two forward forms, the reference test's shapes and known answers ------------------------------------
@pytest.mark.parametrize("G,O", [(1, 4), (3, 3)])
def test_reference_setup_shapes(G, O):
    # test_deconvolution_layer.cpp TestSetup: bottom 2x3x6x4, kernel 3, stride 2 -> 13 x 9, with and without group
    rng = np.random.default_rng(0)
    x, w = _rand(rng, 2, 3, 6, 4), _rand(rng, 3, O // G, 3, 3)
    y = do.deconv_forward(x, w, None, 3, 2, 0, 1, G)
    assert y.shape == (2, O, 13, 9)
    d = capi.DeconvDesc(m.ConvParams.make(2, 3, 6, 4, O, 3, 2, 0, 1, G))
    assert d.out_shape() == (13, 9)


def test_reference_simple_deconvolution_known_answer():
    # TestSimpleDeconvolution: constant weights 1, bias 0.1, bottom 1: 3.1, +3 where one axis overlaps, +9 where both do
    x = np.ones((2, 3, 6, 4))
    w = np.ones((3, 4, 3, 3))
    y = do.deconv_forward(x, w, np.full(4, 0.1), 3, 2, 0, 1)
    for h, wc in itertools.product(range(13), range(9)):
        ho = h % 2 == 0 and 0 < h < 12
        wo = wc % 2 == 0 and 0 < wc < 8
        want = 3.1 + (9 if ho and wo else 3 if ho or wo else 0)
        assert np.allclose(y[:, :, h, wc], want, atol=1e-12)


CASES = [  # (N, C, H, W, O, k, s, p, d, G)
    (2, 3, 6, 4, 4, 3, 2, 0, 1, 1),
    (2, 4, 5, 3, 6, 4, 2, 1, 1, 2),
    (1, 3, 4, 5, 3, 3, 3, 1, 2, 3),
    (2, 2, 3, 3, 2, (2, 5), (3, 2), (0, 2), (1, 2), 1),
    (1, 2, 4, 4, 3, 1, 3, 0, 1, 1),
]


@pytest.mark.parametrize("case", CASES)
def test_col2im_and_gather_forms_agree(case):
    N, Cc, H, W, O, k, s, p, d, G = case
    rng = np.random.default_rng(1)
    kh, kw = do._pair(k)
    x, w, b = _rand(rng, N, Cc, H, W), _rand(rng, Cc, O // G, kh, kw), _rand(rng, O)
    y1 = do.deconv_forward_col2im(x, w, b, k, s, p, d, G)
    y2 = do.deconv_forward_gather(x, w, b, k, s, p, d, G)
    assert np.abs(y1 - y2).max() < 1e-12


@pytest.mark.parametrize("case", CASES[:4])
def test_gradients_by_finite_differences(case):
    N, Cc, H, W, O, k, s, p, d, G = case
    rng = np.random.default_rng(2)
    kh, kw = do._pair(k)
    x, w, b = _rand(rng, N, Cc, H, W), _rand(rng, Cc, O // G, kh, kw), _rand(rng, O)
    r = _rand(rng, *do.deconv_forward(x, w, b, k, s, p, d, G).shape)
    loss = lambda x_, w_, b_: float((do.deconv_forward(x_, w_, b_, k, s, p, d, G) * r).sum())
    dx, dw, db = do.deconv_backward(x, w, r, k, s, p, d, G)
    eps = 1e-6
    for arr, grad, nm in ((x, dx, "x"), (w, dw, "w"), (b, db, "b")):
        for idx in list(np.ndindex(arr.shape))[:: max(1, arr.size // 12)]:
            a2 = arr.copy(); a2[idx] += eps
            a1 = arr.copy(); a1[idx] -= eps
            args_p = [a2 if a is arr else a for a in (x, w, b)]
            args_m = [a1 if a is arr else a for a in (x, w, b)]
            fd = (loss(*args_p) - loss(*args_m)) / (2 * eps)
            assert abs(fd - grad[idx]) < 1e-6 * max(1.0, abs(fd)), (nm, idx, fd, grad[idx])


# ---- the phase decomposition, restated, over a grid ----------------------------------------------------------------------
GRID = [(k, s, p, d) for k in range(1, 6) for s in range(1, 5) for p in range(0, k + 1) for d in (1, 2)]


@pytest.mark.parametrize("k,s,p,d", GRID)
def test_phase_decomposition_matches_oracle(k, s, p, d):
    H, W = 5, 3                                           # odd sizes
    if do.out_extent(H, k, s, p, d) <= 0 or do.out_extent(W, k, s, p, d) <= 0:
        pytest.skip("non-positive top extent (refused by the descriptor)")
    rng = np.random.default_rng(k * 100 + s * 10 + p + d)
    x, w, b = _rand(rng, 2, 4, H, W), _rand(rng, 4, 3, k, k), _rand(rng, 6)
    ref = do.deconv_forward(x, w, b, k, s, p, d, G=2)
    got = do.phase_forward(x, w, b, k, s, p, d, G=2)
    assert not np.isnan(got).any()                        # every output belongs to exactly one phase
    assert np.abs(got - ref).max() < 1e-12


def test_phase_axis_empty_phases_when_k_below_s():
    # k = 2 < s = 3: the residue no tap reaches holds only the bias
    taps = [do.phase_axis(t0, 10, 2, 3, 0, 1)[1] for t0 in range(3)]
    assert taps == [1, 1, 0]
    # d = 2, s = 4: only even residues are reachable (taps 0, 2, 4 and 1, 3)
    taps = [do.phase_axis(t0, 20, 5, 4, 0, 2)[1] for t0 in range(4)]
    assert taps == [3, 0, 2, 0]


# ---- depthwise float32 restatements: forms of the float64 oracle -------------------------------------------------------
@pytest.mark.parametrize("k,s,p,d", [(4, 2, 1, 1), (3, 2, 0, 1), (64, 32, 16, 1), (3, 3, 1, 2)])
def test_depthwise_restatements_match_oracle(k, s, p, d):
    rng = np.random.default_rng(3)
    Cc, H = 3, 3
    x = rng.integers(-4, 5, (2, Cc, H, H)).astype(np.float32)
    w = rng.integers(-4, 5, (Cc, 1, k, k)).astype(np.float32)
    b = rng.integers(-4, 5, Cc).astype(np.float32)
    y = do.dw_forward_f32(x, w, b, k, s, p, d)
    assert np.array_equal(y, do.deconv_forward(x, w, b, k, s, p, d, G=Cc))     # integer data: exact
    dy = rng.integers(-4, 5, y.shape).astype(np.float32)
    dx = do.dw_dgrad_f32(dy, w, H, H, k, s, p, d)
    assert np.array_equal(dx, do.deconv_backward(x, w, dy, k, s, p, d, G=Cc)[0])


# ---- Crop: every case of the reference's test_crop_layer.cpp ----------------------------------------------------------------
B0, B1 = (2, 4, 5, 4), (2, 3, 4, 2)


def test_crop_setup_shapes():
    assert do.crop_offsets(B0, B1, axis=0)[0] == B1                                    # TestSetupShapeAll
    assert do.crop_offsets(B0, B1)[0] == (2, 4, 4, 2)                                  # TestSetupShapeDefault (axis 2)
    assert do.crop_offsets(B0, B1, axis=-1)[0] == (2, 4, 5, 2)                         # TestSetupShapeNegativeIndexing
    assert do.crop_offsets(B0, (2, 5, 4, 2))[0] == (2, 4, 4, 2)                        # TestDimensionsCheck: axis 1 uncropped


def test_crop_values_and_offsets():
    x = np.arange(np.prod(B0), dtype=np.float32).reshape(B0)
    top, off = do.crop_offsets(B0, B1, axis=0)                                         # TestCropAll
    assert np.array_equal(do.crop_forward(x, top, off), x[:2, :3, :4, :2])
    top, off = do.crop_offsets(B0, B1, axis=0, offset=(0, 1, 1, 2))                    # TestCropAllOffset
    assert np.array_equal(do.crop_forward(x, top, off), x[0:2, 1:4, 1:5, 2:4])
    top, off = do.crop_offsets(B0, B1, axis=2, offset=(1, 2))                          # TestCropHW
    assert np.array_equal(do.crop_forward(x, top, off), x[:, :, 1:5, 2:4])
    b0, b1 = B0 + (2,), B1 + (1,)                                                       # TestCrop5D
    x5 = np.arange(np.prod(b0), dtype=np.float32).reshape(b0)
    top, off = do.crop_offsets(b0, b1, axis=2, offset=(1, 2, 0))
    assert top == (2, 4, 4, 2, 1) and off == (0, 0, 1, 2, 0)
    assert np.array_equal(do.crop_forward(x5, top, off), x5[:, :, 1:5, 2:4, 0:1])
    g = np.ones(top, np.float32)                                                        # the gradient cases: the window, zeros elsewhere
    dx = do.crop_backward(g, b0, off)
    assert dx.sum() == g.size and dx[:, :, 1:5, 2:4, 0:1].all()


def test_crop_refusals():
    with pytest.raises(ValueError, match="invalid crop parameters in dimension: 3"):
        do.crop_offsets(B0, B1, axis=2, offset=(1, 3))
    with pytest.raises(ValueError, match="number of offset values"):
        do.crop_offsets(B0, B1, axis=2, offset=(1, 2, 0))
    with pytest.raises(ValueError, match="out of range"):
        do.crop_offsets(B0, B1, axis=4)


def test_crop_entry_points_refuse_bad_windows_without_a_device():
    L = m.lib()
    arr = lambda v: (C.c_int * len(v))(*v)
    for bs, ts, off in (((2, 4, 5, 4), (2, 4, 4, 2), (0, 0, 2, 0)), ((4,), (2,), (-1,)), ((4,), (5,), (0,))):
        assert L.b2c_crop_forward(len(bs), arr(bs), arr(ts), arr(off), None, None, None) == -1
        assert L.b2c_crop_backward(len(bs), arr(bs), arr(ts), arr(off), None, None, None) == -1
    assert L.b2c_crop_forward(4, arr((2, 4, 5, 4)), arr((2, 4, 4, 2)), arr((0, 0, 2, 0)), None, None, None) == -1
    assert b"invalid crop parameters in dimension: 2" in L.b2c_last_error()
    assert L.b2c_crop_forward(0, arr((1,)), arr((1,)), arr((0,)), None, None, None) == -1


# ---- bilinear weights (filler.hpp BilinearFiller, integer-division f) -----------------------------------------------------
def test_bilinear_weights_values():
    w4 = do.bilinear_weights((1, 1, 4, 4))[0, 0]
    assert np.allclose(w4, np.outer([0.25, 0.75, 0.75, 0.25], [0.25, 0.75, 0.75, 0.25]), atol=0)
    # k = 3: f = 3 // 2 = 1 (BVLC's ceil(3 / 2.) would give 2), c = (2 - 1 - 1) / 2 = 0: taps 1, 0, -1 per axis
    w3 = do.bilinear_weights((2, 1, 3, 3))
    assert np.array_equal(w3[0, 0], np.outer([1, 0, -1], [1, 0, -1]).astype(np.float32))
    assert np.array_equal(w3[1, 0], w3[0, 0])
    with pytest.raises(ValueError, match="square"):
        do.bilinear_weights((1, 1, 3, 4))
    with pytest.raises(ValueError, match="4 dim"):
        do.bilinear_weights((1, 3, 3))


# ---- descriptor and plan (host only) -------------------------------------------------------------------------------------
def test_descriptor_refuses_non_positive_top():
    L = m.lib()
    h = C.c_void_p()
    assert L.b2c_deconv_desc_create(C.byref(m.ConvParams.make(1, 2, 2, 2, 2, 1, 1, 1)), 0, C.byref(h)) == -1   # Ht = 2 - 2 = 0
    assert b"not positive" in L.b2c_last_error()
    assert L.b2c_deconv_desc_create(C.byref(m.ConvParams.make(1, 3, 4, 4, 4, 3, 1, 0, 1, 2)), 0, C.byref(h)) == -1  # C % G


def test_plan_reports_each_route():
    P = m.ConvParams.make
    dcgan = capi.DeconvDesc(P(64, 512, 4, 4, 256, 4, 2, 1, 1, 1, False))
    q = dcgan.plan(capi.OP_FORWARD)
    assert q["route"] == "phase" and q["phases"] == 4 and q["phase_taps"] == [4, 4, 4, 4] and all(t > 0 for t in q["phase_tiles"])
    q = capi.DeconvDesc(P(2, 16, 7, 7, 8, 3, 2, 1)).plan(capi.OP_FORWARD)     # pad 1: even outputs take the odd tap
    assert q["route"] == "phase" and q["phase_taps"] == [1, 2, 2, 4]
    q = capi.DeconvDesc(P(2, 8, 5, 5, 8, 2, 3)).plan(capi.OP_FORWARD)                  # k < s: a third of the phases are empty
    assert q["route"] == "phase" and q["phase_taps"].count(0) == 5 and q["phase_tiles"][2] == 0
    fcn = capi.DeconvDesc(P(1, 21, 16, 16, 21, 64, 32, 16, 1, 21, False))
    assert fcn.y_shape() == (1, 21, 512, 512)
    for op in (0, 1, 2):
        assert fcn.plan(op)["route"] == "depthwise" and fcn.workspace_bytes(op) == 0
    s1 = capi.DeconvDesc(P(2, 16, 8, 8, 32, 3, 1, 1))
    assert s1.plan(0)["route"] == "dual" and capi.CONV_ROUTES[s1.plan(0)["dual_route"]] in ("staged", "gather")
    assert capi.CONV_ROUTES[capi.DeconvDesc(P(2, 16, 8, 8, 32, 1, 2)).plan(0)["dual_route"]] == "gather_scatter"
    assert capi.CONV_ROUTES[capi.DeconvDesc(P(2, 16, 7, 7, 8, 3, 2, 1), capi.ENGINE_CAFFE).plan(0)["dual_route"]] == "caffe"
    assert capi.DeconvDesc(P(2, 16, 7, 7, 8, 3, 2, 1), algo=capi.ALGO_SIMT).plan(0)["route"] == "dual"
    for op in (1, 2):
        assert dcgan.plan(op)["route"] == "dual"


# ---- Net: shapes, learnable parameters, need-backward and refusals of Deconvolution and Crop -----------------------------
from caffe_mpi_b200 import host_api  # noqa: E402


def test_net_shapes_and_params_of_the_encoder_decoder():
    n = host_api.Net(do.encdec_prototxt(2), "TRAIN", is_text=True)
    shapes = {nm: s for nm, ty, s in n.layers()}
    assert shapes["up"] == (2, 3, 10, 10) and shapes["crop"] == (2, 3, 8, 8) and shapes["bil"] == (2, 6, 8, 8)
    counts = [c for _, c, _, _ in n.learnable_params()]
    assert counts == [6 * 3 * 9, 6, 6 * 3 * 16, 3, 6 * 1 * 16, 3 * 6, 3]      # deconv weights [C_in, O/G, k, k]
    lrs = [lr for _, _, lr, _ in n.learnable_params()]
    assert lrs[4] == 0.0                                                      # the frozen bilinear upsampler
    plan = dict(zip([nm for nm, _, _ in n.layers()], n.backward_plan()))
    assert plan["crop"] == (True, [True, False])                              # Crop's reference bottom gets no gradient
    assert [nm for nm, _, _ in n.conv_layers()] == ["conv1", "proj"]          # only Convolution layers are listed as such


def _one(layer, bottom="c1", extra=""):
    return ('layer { name: "data" type: "Input" top: "data" top: "c1" input_param { shape { dim: 2 dim: 3 dim: 8 dim: 8 } '
            'shape { dim: 2 dim: 4 dim: 5 dim: 6 } } }\n' + layer + extra)


@pytest.mark.parametrize("cp,shape", [
    ("num_output: 4 kernel_size: 3 stride: 2", (2, 4, 11, 13)),
    ("num_output: 8 kernel_h: 3 kernel_w: 1 stride_h: 3 stride_w: 1 pad_h: 1 group: 4", (2, 8, 13, 6)),
    ("num_output: 2 kernel_size: 3 dilation: 2 stride: 1 pad: 2", (2, 2, 5, 6)),
])
def test_net_deconvolution_shapes(cp, shape):
    n = host_api.Net(_one('layer { name: "d" type: "Deconvolution" bottom: "c1" top: "d" convolution_param { %s } }' % cp), "TRAIN",
                     is_text=True)
    assert dict((nm, s) for nm, _, s in n.layers())["d"] == shape


@pytest.mark.parametrize("cp,msg", [
    ("num_output: 4 kernel_size: 1 pad: 3", "non-positive output extent"),
    ("num_output: 4 kernel_size: 0", "Filter dimensions must be nonzero."),
    ("num_output: 3 kernel_size: 3 group: 2", "multiples of group"),
    ("num_output: 4 kernel_size: 3 kernel_h: 3 kernel_w: 3", "Either kernel_size or kernel_size_h/w should be specified; not both."),
])
def test_net_deconvolution_refusals(cp, msg):
    with pytest.raises(host_api.HostError, match=msg.replace("(", r"\(").replace(")", r"\)").replace(".", r"\.")):
        host_api.Net(_one('layer { name: "d" type: "Deconvolution" bottom: "c1" top: "d" convolution_param { %s } }' % cp), "TRAIN",
                     is_text=True)


@pytest.mark.parametrize("cp,shape", [("axis: 2 offset: 1", (2, 4, 8, 8)), ("axis: 0", (2, 3, 8, 8)), ("axis: -1 offset: 0", (2, 4, 5, 8))])
def test_net_crop_shapes(cp, shape):
    net = ('layer { name: "data" type: "Input" top: "big" top: "ref" input_param { shape { dim: 2 dim: 4 dim: 10 dim: 9 } '
           'shape { dim: 2 dim: 3 dim: 8 dim: 8 } } }\n'
           'layer { name: "c" type: "Crop" bottom: "big" bottom: "ref" top: "c" crop_param { %s } }' % cp)
    if shape == (2, 4, 5, 8):
        net = net.replace("dim: 10 dim: 9", "dim: 5 dim: 9")
    assert dict((nm, s) for nm, _, s in host_api.Net(net, "TRAIN", is_text=True).layers())["c"] == shape


@pytest.mark.parametrize("cp,msg", [
    ("axis: 2 offset: 3", "invalid crop parameters in dimension: 2"),
    ("axis: 2 offset: 1 offset: 2 offset: 3", "number of offset values specified must be equal to the number of dimensions following axis"),
    ("axis: 4", "out of range"),
])
def test_net_crop_refusals(cp, msg):
    net = ('layer { name: "data" type: "Input" top: "big" top: "ref" input_param { shape { dim: 2 dim: 4 dim: 10 dim: 9 } '
           'shape { dim: 2 dim: 3 dim: 8 dim: 8 } } }\n'
           'layer { name: "c" type: "Crop" bottom: "big" bottom: "ref" top: "c" crop_param { %s } }' % cp)
    with pytest.raises(host_api.HostError, match=msg):
        host_api.Net(net, "TRAIN", is_text=True)


def test_encdec_oracle_gradients_by_finite_differences():
    rng = np.random.default_rng(11)
    shapes = [(6, 3, 3, 3), (6,), (6, 3, 4, 4), (3,), (6, 1, 4, 4), (3, 6, 1, 1), (3,)]
    params = [rng.standard_normal(s) * 0.3 for s in shapes]
    data, target = rng.standard_normal((2, 3, 8, 8)), rng.uniform(0, 1, (2, 192))
    loss, grads, _ = do.encdec_forward_backward(params, data, target)
    eps = 1e-6
    for k, (p, g) in enumerate(zip(params, grads)):
        for idx in list(np.ndindex(p.shape))[:: max(1, p.size // 6)]:
            pp = [a.copy() for a in params]; pp[k][idx] += eps
            pm = [a.copy() for a in params]; pm[k][idx] -= eps
            fd = (do.encdec_forward_backward(pp, data, target)[0] - do.encdec_forward_backward(pm, data, target)[0]) / (2 * eps)
            assert abs(fd - g[idx]) < 1e-6 * max(1.0, abs(fd)), (k, idx, fd, g[idx])
