"""SoftmaxWithLoss and Accuracy over spatial positions without a GPU: the float64 oracle of tests/seg_oracle.py against the closed
forms of the reference's layer tests (test_softmax_with_loss_layer.cpp, test_accuracy_layer.cpp), Net's parsing and shapes of
loss_param / accuracy_param with the reference's messages, and the route plan of b2c_softmax_loss_forward_ex."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import seg_oracle as so
from caffe_mpi_b200 import host_api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bottoms(seed=1701, shape=(10, 5, 2, 3)):
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(shape).astype(np.float32)
    lab = rng.integers(0, shape[1], (shape[0], 1) + tuple(shape[2:])).astype(np.float32)
    return x, lab


# ---- SoftmaxWithLoss: test_softmax_with_loss_layer.cpp ----------------------------------------------------------------------
def test_forward_ignore_label_sums_to_four_times_the_full_loss():
    """TestForwardIgnoreLabel: normalize false (BATCH_SIZE); ignoring each of the 5 labels in turn drops each pixel from exactly
    one run, so the runs sum to 4x the loss with nothing ignored."""
    x, lab = bottoms()
    full = so.loss_only(x, lab, norm="BATCH_SIZE")
    parts = [so.loss_only(x, lab, ignore_label=k, norm="BATCH_SIZE") for k in range(5)]
    assert sum(parts) == pytest.approx(4 * full, rel=1e-12)


@pytest.mark.parametrize("case", ["gradient", "ignore_label", "unnormalized"])
def test_gradient_matches_finite_differences(case):
    """TestGradient (loss_weight 3), TestGradientIgnoreLabel (ignore_label 0) and TestGradientUnnormalized (normalize false) on
    (10, 5, 2, 3): the closed-form dx against central differences of the loss."""
    x, lab = bottoms()
    kw = {"gradient": dict(loss_weight=3.0), "ignore_label": dict(ignore_label=0), "unnormalized": dict(norm="BATCH_SIZE")}[case]
    lw = kw.pop("loss_weight", 1.0)
    _, _, _, dx = so.softmax_loss(x, lab, loss_weight=lw, **kw)
    num = so.numeric_grad(lambda v: lw * so.loss_only(v, lab, **kw), x)
    assert np.abs(dx - num).max() < 1e-5 * max(1.0, np.abs(num).max())
    if case == "ignore_label":
        ign = (lab.reshape(10, 1, 2, 3) == 0)
        assert np.all(dx[np.broadcast_to(ign, dx.shape)] == 0)


def test_normalizers_and_the_floor():
    x, lab = bottoms()
    lab[:] = 2
    _, n, _, _ = so.softmax_loss(x, lab, ignore_label=2)                   # every pixel ignored: VALID counts 0, floored at 1
    assert n == 1.0
    assert so.softmax_loss(x, lab)[1] == 60.0                              # VALID without ignore_label: outer * inner
    assert so.softmax_loss(x, lab, norm="FULL", ignore_label=2)[1] == 60.0
    assert so.softmax_loss(x, lab, norm="BATCH_SIZE")[1] == 10.0
    assert so.softmax_loss(x, lab, norm="NONE")[1] == 1.0
    assert so.softmax_loss(x, lab, ignore_label=2)[0] == 0.0


def test_axis_is_the_class_axis():
    """axis -1 on an NHWC-shaped bottom is the axis-1 loss of the transposed bottom."""
    x, lab = bottoms(shape=(4, 5, 3, 6))
    nhwc = np.ascontiguousarray(x.transpose(0, 2, 3, 1))
    a = so.softmax_loss(x, lab, ignore_label=1)
    b = so.softmax_loss(nhwc, lab, axis=-1, ignore_label=1)
    assert a[0] == pytest.approx(b[0], rel=1e-14)
    assert np.allclose(a[3].transpose(0, 2, 3, 1), b[3], rtol=0, atol=1e-15)


# ---- Accuracy: test_accuracy_layer.cpp -------------------------------------------------------------------------------------
def closed_form(scores, labels, axis=1, top_k=1, ignore=None):
    """The reference tests' own statement: count the classes whose score beats the label's (equal scores: a larger index)."""
    outer, C, inner = so.view(scores.shape, axis)
    z = scores.reshape(outer, C, inner)
    lab = labels.reshape(outer, inner).astype(np.int64)
    hits = count = 0
    hc, nc = np.zeros(C), np.zeros(C)
    for o in range(outer):
        for i in range(inner):
            l = lab[o, i]
            if ignore is not None and l == ignore:
                continue
            count += 1
            nc[l] += 1
            col = z[o, :, i]
            above = sum(1 for k in range(C) if col[k] > col[l] or (col[k] == col[l] and k > l))
            if above < top_k:
                hits += 1
                hc[l] += 1
    return hits / count, np.where(nc == 0, 0, hc / np.maximum(nc, 1))


@pytest.mark.parametrize("case", ["forward", "spatial_axes", "ignore_label", "top_k", "per_class", "per_class_ignore"])
def test_accuracy_cases(case):
    rng = np.random.default_rng(11)
    shape, axis, top_k, ignore = (100, 10), 1, 1, None
    if case == "spatial_axes":
        shape = (2, 10, 4, 5)
    if case == "top_k":
        top_k = 3
    if case in ("ignore_label", "per_class_ignore"):
        ignore = -1
    scores = rng.standard_normal(shape).astype(np.float32)
    labels = rng.integers(0, 10, (shape[0],) + shape[2:]).astype(np.float32)
    if ignore is not None:
        labels[::3] = ignore                                                 # every third label is ignored
    acc, per = so.accuracy(scores, labels, axis, top_k, ignore)
    want, want_pc = closed_form(scores, labels, axis, top_k, ignore)
    assert acc == np.float32(want)
    assert np.array_equal(per, want_pc.astype(np.float32))


def test_accuracy_ties_and_edges():
    s = np.zeros((1, 4, 3), np.float32)                                      # every score equal: the larger index ranks first
    lab = np.array([[3, 2, 0]], np.float32)
    acc, per = so.accuracy(s, lab, top_k=1)
    assert acc == np.float32(1 / 3) and list(per) == [0, 0, 0, 1]
    assert so.accuracy(s, lab, top_k=2)[0] == np.float32(2 / 3)
    all_ign = np.full((1, 3), 7, np.float32)
    assert np.isnan(so.accuracy(s, all_ign, ignore_label=7)[0])              # accuracy / count with count 0
    acc, per = so.accuracy(s, np.array([[9, 3, 3]], np.float32))             # label 9 is out of range: a miss, no class touched
    assert acc == np.float32(2 / 3) and list(per) == [0, 0, 0, 1]


# ---- Net: parsing, top shapes, checks ---------------------------------------------------------------------------------------
def net(loss_extra="", acc_extra="", data=(10, 5, 2, 3), label=(10, 1, 2, 3), loss_tops=("loss",), acc_tops=("acc",)):
    d = " ".join(f"dim: {v}" for v in data)
    lb = " ".join(f"dim: {v}" for v in label)
    lt = " ".join(f'top: "{t}"' for t in loss_tops)
    at = " ".join(f'top: "{t}"' for t in acc_tops)
    return f'''
layer {{ name: "in" type: "Input" top: "data" top: "label" input_param {{ shape {{ {d} }} shape {{ {lb} }} }} }}
layer {{ name: "loss" type: "SoftmaxWithLoss" bottom: "data" bottom: "label" {lt} {loss_extra} }}
layer {{ name: "acc" type: "Accuracy" bottom: "data" bottom: "label" {at} {acc_extra} }}
'''


@pytest.mark.parametrize("text,want", [
    ("", ("VALID", None)),
    ("loss_param { ignore_label: 255 }", ("VALID", 255)),
    ("loss_param { normalization: FULL }", ("FULL", None)),
    ("loss_param { normalization: 2 }", ("BATCH_SIZE", None)),
    ("loss_param { normalization: NONE ignore_label: -1 }", ("NONE", -1)),
    ("loss_param { normalize: false }", ("BATCH_SIZE", None)),
    ("loss_param { normalize: true }", ("VALID", None)),
    ("loss_param { normalization: FULL normalize: false }", ("FULL", None)),        # normalization wins over normalize
    ("loss_param { normalization: 3 normalize: true }", ("NONE", None)),
])
def test_loss_param_parsing(text, want):
    p = host_api.Net(net(loss_extra=text), is_text=True).loss_params(1)
    assert (p["normalization"], p["ignore_label"]) == want


def test_unknown_normalization_is_refused():
    with pytest.raises(host_api.HostError, match="Unknown normalization mode"):
        host_api.Net(net(loss_extra="loss_param { normalization: SOMETIMES }"), is_text=True)


def test_accuracy_param_and_canonical_axes():
    n = host_api.Net(net(loss_extra="softmax_param { axis: -3 }", acc_extra="accuracy_param { axis: -3 top_k: 2 ignore_label: 4 }"),
                     is_text=True)
    assert n.loss_params(1)["softmax_axis"] == 1
    a = n.loss_params(2)
    assert (a["accuracy_axis"], a["top_k"], a["accuracy_ignore_label"]) == (1, 2, 4)
    n = host_api.Net(net(data=(4, 3, 6, 5), label=(4, 3, 6), loss_extra="softmax_param { axis: -1 }",
                         acc_extra="accuracy_param { axis: 3 }"), is_text=True)
    assert n.loss_params(1)["softmax_axis"] == 3 and n.loss_params(2)["accuracy_axis"] == 3


def test_legacy_net_parses_to_the_old_parameters():
    """A classification net with neither sub-message: the parameters every existing net had (axis 1, no ignore_label, VALID,
    top_k 1), and the scalar tops."""
    n = host_api.Net(net(data=(8, 10), label=(8,)), is_text=True)
    assert n.loss_params(1) == {"softmax_axis": 1, "ignore_label": None, "normalization": "VALID", "accuracy_axis": 1, "top_k": 1,
                                "accuracy_ignore_label": None}
    assert n.loss_params(2) == n.loss_params(1)
    assert n.top_shape(1, 0) == () and n.top_shape(2, 0) == ()


def test_second_tops_are_shaped():
    n = host_api.Net(net(loss_tops=("loss", "prob"), acc_tops=("acc", "per_class")), is_text=True)
    assert n.top_shape(1, 1) == (10, 5, 2, 3)
    assert n.top_shape(2, 1) == (5,)


@pytest.mark.parametrize("layer", ["loss", "acc"])
def test_label_count_must_match(layer):
    text = net(label=(10, 1, 2, 2))
    if layer == "acc":                                                       # only the Accuracy layer sees the short label blob
        text = "\n".join(ln for ln in text.splitlines() if "SoftmaxWithLoss" not in ln)
    word = "softmax" if layer == "loss" else "label"
    with pytest.raises(host_api.HostError, match=f"Number of labels must match number of predictions; e.g., if {word} axis == 1"):
        host_api.Net(text, is_text=True)


def test_top_k_must_not_exceed_the_classes():
    with pytest.raises(host_api.HostError, match="top_k must be less than or equal to the number of classes."):
        host_api.Net(net(acc_extra="accuracy_param { top_k: 6 }"), is_text=True)
    host_api.Net(net(acc_extra="accuracy_param { top_k: 5 }"), is_text=True)


# ---- the plan query -------------------------------------------------------------------------------------------------------
def test_softmax_loss_plan_routes_chunks_and_workspace():
    """b2c_debug_softmax_loss_plan is host-only; asked in a subprocess with the device hidden."""
    script = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
from caffe_mpi_b200 import capi
import ctypes as C
P = capi.softmax_loss_plan
S = [P(256, 1000, 1), P(10, 5, 6), P(10, 5, 4, 16, 32), P(10, 5, 4, 16, 36), P(10, 5, 4, 20, 32), P(10, 5, 3, 16, 32),
     P(8, 21, 512 * 512, 256, 512), P(16, 150, 128 * 128, 256, 512), P(1, 2, 1025), P(1, 2, 1024), P(3, 1, 4097),
     capi.softmax_loss_workspace(8, 21, 512 * 512)]
L = capi.lib()
refused = [L.b2c_debug_softmax_loss_plan(0, 5, 6, None, None, (C.c_int * 4)(), 4),
           L.b2c_debug_softmax_loss_plan(1, 0, 6, None, None, (C.c_int * 4)(), 4),
           L.b2c_debug_softmax_loss_plan(1, 5, 6, None, None, (C.c_int * 3)(), 3)]
print(json.dumps([S, refused]))
"""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, "-c", script, ROOT], env=env, capture_output=True, text=True, check=True).stdout
    S, refused = json.loads(out.strip().splitlines()[-1])
    assert refused == [-1, -1, -1]
    routes = [q["route"] for q in S[:11]]
    assert routes == ["row", "column", "column_f4", "column", "column", "column", "column_f4", "column_f4", "column", "column_f4", "column"]
    assert all(q["chunk"] == 1024 for q in S[:11])
    slots = [q["slots"] for q in S[:11]]
    assert slots == [1, 1, 1, 1, 1, 1, 2048, 256, 2, 1, 13]
    # the workspace: one double and one int per chunk, rounded up to 16 bytes
    assert [q["workspace"] for q in S[:11]] == [-(-12 * s // 16) * 16 for s in slots]
    assert S[11] == 2048 * 12
