"""Whole-net parity at the benchmark's real shapes: ResNet-50, GoogLeNet, AlexNet and VGG-16 (caffe_mpi_b200/models.py) built by
TrainNet at 224 x 224 (AlexNet 227) with 1000 classes, checked layer by layer against float64 (tests/fullnet_walker.py).

The mini nets of test_trainer_gpu.py never reach the staged conv kernels (C % 32 == 0), the 7x7 plane mode, the staged and
compact weight-gradient routes, the gather-scatter dgrad, a second filter-prep batch (> 24 prepared layouts), a parameter update
of more than SEG_MAX segments in one call (a second fused solver launch inside one bucket: ResNet-50 with reduce_buckets: 1) or
dropout over 4096-wide blobs; these nets do, and the route inventory below fails first if they stop doing so.  Batch 4
(ResNet-50) and 2 (the others): batch 1 would not reach the tiles that span two images."""
import math
import os
import re
import time

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api, models
import fullnet_walker as fw

pytestmark = pytest.mark.gpu
BATCH = {"resnet50": 4, "googlenet": 2, "alexnet": 2, "vgg16": 2}
CROP = {"resnet50": 224, "googlenet": 224, "alexnet": 227, "vgg16": 224}
LR, WD, MOMENTUM = 0.01, 1e-4, 0.9
SOLVER = f'base_lr: {LR} lr_policy: "fixed" momentum: {MOMENTUM} weight_decay: {WD} max_iter: 100 solver_mode: GPU'
PREP_BATCH = 24             # filter layouts per b2c_conv_prepare_filters launch (csrc/filter_prep.cuh)
SEG_MAX = 96                # segments per fused solver launch (csrc/sgd.cu)


MULTS = ((1.0, 1.0), (2.0, 0.0), (0.5, 2.0))     # (lr_mult, decay_mult) cycled over the one-bucket net's conv and fc layers


def net_text(name, one_bucket=False):
    """models.PROTOTXT[name] with its Data layer replaced by an Input layer of the same shapes: the test owns data and label.
    one_bucket: NetParameter reduce_buckets: 1 (the whole update in one call) and per-layer ParamSpecs cycling through MULTS, so
    that neighbouring segments, on both sides of every SEG_MAX boundary, have different rates and decays."""
    txt = models.PROTOTXT[name](BATCH[name], CROP[name], 1000)
    if one_bucket:
        head, *parts = txt.split("layer {")
        k = 0
        for i, part in enumerate(parts):
            for kind in ("Convolution", "InnerProduct"):
                if f'type: "{kind}"' in part:
                    lm, dm = MULTS[k % len(MULTS)]
                    spec = f" param {{ lr_mult: {lm} decay_mult: {dm} }}" * (1 if "bias_term: false" in part else 2)
                    parts[i] = re.sub(r"(\s)(convolution_param|inner_product_param) \{", lambda m: spec + m.group(1) + m.group(2) + " {",
                                      part, count=1)
                    k += 1
        txt = head + "reduce_buckets: 1\n" + "".join("layer {" + p for p in parts)
    a = txt.index('layer { name: "data" type: "Data"')
    end = "include: { phase: TRAIN } }\n"
    b = txt.index(end, a) + len(end)
    n, c = BATCH[name], CROP[name]
    inp = (f'layer {{ name: "data" type: "Input" top: "data" top: "label" input_param {{ shape {{ dim: {n} dim: 3 dim: {c} dim: {c} }} '
           f'shape {{ dim: {n} }} }} }}\n')
    return txt[:a] + inp + txt[b:]


def make_trainer(name, fuse, data=None, label=None, params=None, one_bucket=False):
    """fuse False: B2C_FUSE=0 (the prototxt's layers one by one); True: the library default.  Weights from the prototxt fillers
    unless `params` (trainable order) is given; data N(0,1), labels uniform in [0, 1000) unless given."""
    old = os.environ.get("B2C_FUSE")
    if not fuse:
        os.environ["B2C_FUSE"] = "0"
    else:
        os.environ.pop("B2C_FUSE", None)
    try:
        t = host_api.Trainer(net_text(name, one_bucket), SOLVER, num_classes=1000)
    finally:
        if old is None:
            os.environ.pop("B2C_FUSE", None)
        else:
            os.environ["B2C_FUSE"] = old
    if params is not None:
        for i, p in enumerate(params):
            t.set_param(i, p)
    rng = np.random.default_rng(20261017)
    n, c = BATCH[name], CROP[name]
    if data is None:
        data = rng.standard_normal((n, 3, c, c)).astype(np.float32)
        label = rng.integers(0, 1000, n).astype(np.float32)
    t.set_blob("data", data)
    t.set_blob("label", label)
    return t, data, label


def param_dict(t, desc):
    out = {}
    for i, (layer, _, _, _) in enumerate(desc.learnable_params()):
        out.setdefault(layer, []).append((t.get_param(i, 0), t.get_param(i, 1)))
    return out


def report(tag, checks, seconds=None):
    worst = fw.summary(checks)
    head = f"[fullnet] {tag}" + (f": {seconds:.1f} s" if seconds is not None else "")
    print(head)
    for (kind, what, bar), err in sorted(worst.items()):
        print(f"[fullnet]   {kind:28s} {what:9s} bar {bar:g}  worst {err:.3g}")


# ------------------------------------------------------------------------------------------------------------ route inventory
def conv_routes(name):
    desc = host_api.Net(net_text(name), is_text=True)
    out = []
    for layer, prm, _ in desc.conv_layers():
        d = capi.ConvDesc(prm, math=capi.MATH_FP32)
        out.append((layer, d.conv_plan(capi.OP_FORWARD)["route"], d.conv_plan(capi.OP_BACKWARD_DATA)["route"], d.wgrad_plan()))
    return out


def bucket_segments(name, one_bucket=False):
    """trainable segments of each reduce bucket: TrainNet's buckets over its parameter arena (every layer blob, BatchNorm's three
    statistics included, as Net::AppendParam lists them); ApplyUpdate leaves the statistics out of its fused launches, which take
    SEG_MAX segments each"""
    desc = host_api.Net(net_text(name, one_bucket), is_text=True)
    types = {nm: ty for nm, ty, _ in desc.layers()}
    counts, trainable, prev = [], [], None
    for layer, cnt, _, _ in desc.learnable_params():
        if types[layer] == "BatchNorm" and layer != prev:
            counts += [cnt, cnt, 1]                     # running mean, running variance, correction
            trainable += [False] * 3
        counts.append(cnt)
        trainable.append(True)
        prev = layer
    return [sum(trainable[f:t + 1]) for f, t, _, _ in host_api.plan_buckets(counts, desc.reduce_buckets())]


CONV_ROUTES_WANTED = {"staged", "staged_plane", "gather", "gather_scatter"}
WGRAD_ROUTES_WANTED = {"staged_3x3", "staged_1x1", "compact_staged", "gather"}


def test_route_inventory():
    """the four nets together reach every forward / dgrad and weight-gradient route this file is meant to guard"""
    fwd, wg, presplit, lines = set(), set(), 0, []
    layouts = 0
    for name in BATCH:
        for layer, rf, rd, w in conv_routes(name):
            fwd |= {rf, rd}
            wg.add(w["route"])
            presplit += int(w["presplit_dy"])
            lines.append(f"[fullnet] {name:9s} {layer:28s} fwd {rf:14s} dgrad {rd:14s} wgrad {w['route']:16s}"
                         f"{' presplit_dy' if w['presplit_dy'] else ''}")
            if name == "resnet50":
                layouts += sum(r in CONV_ROUTES_WANTED for r in (rf, rd))
    print("\n".join(lines))
    print(f"[fullnet] forward/dgrad routes {sorted(fwd)}; wgrad routes {sorted(wg)}; presplit_dy layers {presplit}")
    assert CONV_ROUTES_WANTED <= fwd, CONV_ROUTES_WANTED - fwd
    assert WGRAD_ROUTES_WANTED <= wg, WGRAD_ROUTES_WANTED - wg
    assert wg & {"staged_3x3_plane", "staged_1x1_plane"}, wg
    assert presplit >= 1
    # ResNet-50: its prepared filter layouts (one per tensor-core forward / dgrad route of each conv) take several filter-prep
    # launches; with reduce_buckets: 1 its whole update is one ApplyUpdate call of more than SEG_MAX segments (two fused launches)
    segs, one = bucket_segments("resnet50"), bucket_segments("resnet50", one_bucket=True)
    print(f"[fullnet] resnet50: {layouts} prepared filter layouts; trainable segments per bucket {segs}, with reduce_buckets: 1 {one}")
    assert math.ceil(layouts / PREP_BATCH) >= 3, layouts
    assert one == [161] and max(one) > SEG_MAX, one
    # the multipliers really differ across the first launch's last segment and the second launch's first
    lp = host_api.Net(net_text("resnet50", one_bucket=True), is_text=True).learnable_params()
    assert len({(lr, dc) for _, _, lr, dc in lp[SEG_MAX - 3:SEG_MAX + 3]}) >= 2


# ------------------------------------------------------------------------------------------------------------ layer parity
@pytest.mark.parametrize("name", ["resnet50", "googlenet", "alexnet", "vgg16"])
def test_unfused_layer_parity(name):
    """one forward_backward() of the unfused graph; every layer's tops, every blob diff, every parameter gradient against float64
    recomputed from the product's own inputs (fullnet_walker: teacher forcing, bars per layer kind)"""
    t0 = time.time()
    t, data, label = make_trainer(name, fuse=False)
    desc = host_api.Net(net_text(name), is_text=True)
    t.forward_backward()
    layers = fw.parse_layers(net_text(name))
    shapes = {}
    checks = fw.walk(layers, t.get_blob, param_dict(t, desc), data.shape, label, shapes=shapes)
    if any(L["type"] == "Dropout" for L in layers):
        # a second iteration: every dropout stream moves on by its blob's size (the fc6 / fc7 streams by 8192 per step), so the
        # layers that carry a Dropout are checked again against iteration 1's masks
        t.forward_backward()
        again = fw.walk(layers, t.get_blob, param_dict(t, desc), data.shape, label, iteration=1, forward_only=True,
                        kinds={"InnerProduct", "Pooling"}, shapes=shapes)
        assert any(c.kind == "Dropout" for c in again)
        checks += again
    report(name, checks, time.time() - t0)
    kinds = {c.kind for c in checks}
    assert {"Convolution", "InnerProduct", "SoftmaxWithLoss", "ReLU", "MAX"} <= kinds
    if name == "googlenet":
        assert sum(c.what == "loss" for c in checks) == 3          # loss1/loss1 and loss2/loss1 at 0.3, loss at 1
    bad = fw.failures(checks)
    assert not bad, bad[:20]


# ------------------------------------------------------------------------------------------------------------ fused == unfused
def residual_tail_tops(layers):
    """the BatchNorm tops the fused graph never writes: TrainNet::FuseResidualTails hands each BatchNorm -> Eltwise(SUM) ->
    in-place ReLU tail to the BatchNorm that runs last among the sum's producers, and that BatchNorm writes the sum instead of
    its own top.  Restated from the graph: the sum is followed by an in-place ReLU, the later producer of its two bottoms is an
    out-of-place BatchNorm without a ReLU of its own whose top only the sum reads, nothing between them writes or reads the
    other operand, and the sum is the first backward writer of both bottoms (the last of their consumers to run forward)."""
    def writers(blob, before):
        return [j for j in range(before) if blob in layers[j]["top"]]

    def consumers(blob):
        return [j for j, L in enumerate(layers) if blob in L["bottom"] and not (L["type"] in fw.IN_PLACE and L["top"] == L["bottom"])]

    out = set()
    for i, L in enumerate(layers):
        if L["type"] != "Eltwise" or len(L["bottom"]) != 2 or i + 1 >= len(layers):
            continue
        nxt = layers[i + 1]
        if not (nxt["type"] == "ReLU" and nxt["bottom"] == L["top"] == nxt["top"]):
            continue
        if any(max(consumers(b)) != i for b in L["bottom"]):
            continue
        prod = [max(writers(b, i)) for b in L["bottom"]]
        k = 0 if prod[0] > prod[1] else 1
        j, other = prod[k], L["bottom"][1 - k]
        B = layers[j]
        if B["type"] != "BatchNorm" or B["top"] == B["bottom"] or any(layers[r]["type"] == "ReLU" and layers[r]["bottom"] == B["top"]
                                                                      for r in range(len(layers))):
            continue
        if len(consumers(B["top"][0])) != 1:
            continue
        if any(other in layers[m]["top"] or other in layers[m]["bottom"] for m in range(j + 1, i)):
            continue
        out.add(B["top"][0])
    return out


def test_fused_graph_is_bitwise_the_unfused_graph():
    """ResNet-50 with the library's fusion passes against B2C_FUSE=0, same weights and batch: the loss, every parameter gradient
    and every forward blob the fused graph writes, bit for bit; then a second forward_backward() gives the same bits again"""
    name = "resnet50"
    a, data, label = make_trainer(name, fuse=False)
    params = [a.get_param(i) for i in range(a.num_params())]
    b, _, _ = make_trainer(name, fuse=True, data=data, label=label, params=params)
    la, lb = a.forward_backward(), b.forward_backward()
    assert la == lb, (la, lb)
    grads = []
    for i in range(a.num_params()):
        ga, gb = a.get_param(i, 1), b.get_param(i, 1)
        assert np.array_equal(ga.view(np.uint32), gb.view(np.uint32)), ("gradient", i)
        grads.append(gb)
    layers = fw.parse_layers(net_text(name))
    skipped = residual_tail_tops(layers)
    # one tail per bottleneck block: the projection BatchNorm in each stage's first block (it runs after conv3/bn), conv3/bn after
    assert len(skipped) == 16, sorted(skipped)
    assert all(s.endswith(".1.skipConv/bn") or (s.endswith(".conv3/bn") and ".1." not in s) for s in skipped), sorted(skipped)
    blobs = {tb for L in layers for tb in L["top"]} - skipped
    # The unfused ReLU writes x * 0 = -0.0 for a negative x (the reference's relu_layer.cu: x > 0 ? x : x * negative_slope), the
    # fused BatchNorm + ReLU and Eltwise + ReLU kernels write +0.0.  The two zeros are the same value and every consumer treats them
    # alike (the gradients above are bit-identical); everywhere else the blobs must agree bit for bit.
    for blob in sorted(blobs):
        va, vb = a.get_blob(blob), b.get_blob(blob)
        differ = va.view(np.uint32) != vb.view(np.uint32)
        assert not np.any(differ & ~((va == 0) & (vb == 0))), blob
    # determinism: no atomics anywhere in a step
    b.clear_param_diffs()
    assert b.forward_backward() == lb
    for i in range(b.num_params()):
        assert np.array_equal(b.get_param(i, 1).view(np.uint32), grads[i].view(np.uint32)), ("second run", i)


# ------------------------------------------------------------------------------------------------------------ one solver step
@pytest.mark.parametrize("one_bucket", [False, True], ids=["buckets6", "one_bucket"])
def test_one_sgd_step_then_forward_on_the_new_weights(one_bucket):
    """ResNet-50, fused: Solver::Step on the same batch (its gradient is the forward_backward() one, by determinism) against float64
    w0 - lr * lr_mult * (g + wd * decay_mult * w0); then a forward on the updated weights, every conv against float64 -- a stale or
    misrouted prepared filter cache shows here.  one_bucket: the whole update in one call of 161 segments with per-layer lr_mult /
    decay_mult, so the second fused solver launch and its per-segment rates are checked"""
    name = "resnet50"
    t, data, label = make_trainer(name, fuse=True, one_bucket=one_bucket)
    desc = host_api.Net(net_text(name, one_bucket), is_text=True)
    mults = [(lr, dc) for _, _, lr, dc in desc.learnable_params()]
    assert len(mults) == t.num_params()
    t.forward_backward()
    w0 = [t.get_param(i, 0).astype(np.float64) for i in range(t.num_params())]
    g = [t.get_param(i, 1).astype(np.float64) for i in range(t.num_params())]
    t.clear_param_diffs()
    t.step(1)
    u32 = 2.0 ** -24
    for i, (lm, dm) in enumerate(mults):
        upd = LR * lm * (g[i] + WD * dm * w0[i])
        w1, h1, d1 = t.get_param(i, 0), t.get_param(i, 2), t.get_param(i, 1)
        # w: the update's three roundings (decay product, sum, rate product) and the subtraction, each within 2^-24 of its operands
        assert np.all(np.abs(w1 - (w0[i] - upd)) <= 4 * u32 * (np.abs(w0[i]) + np.abs(upd))), ("weights", i)
        assert np.array_equal(w1, (w0[i].astype(np.float32) - h1).astype(np.float32)), ("w1 != w0 - history", i)
        assert np.all(np.abs(h1 - upd) <= 4 * u32 * LR * lm * (np.abs(g[i]) + WD * dm * np.abs(w0[i]))), ("history", i)
        assert not d1.any(), ("diff not cleared", i)
    t.forward_backward()
    layers = fw.parse_layers(net_text(name, one_bucket))
    checks = fw.walk(layers, t.get_blob, param_dict(t, desc), data.shape, label, forward_only=True, kinds={"Convolution"})
    report(f"resnet50{' one bucket' if one_bucket else ''} after one step (conv forward)", checks)
    assert sum(c.kind == "Convolution" for c in checks) == 53
    bad = fw.failures(checks)
    assert not bad, bad[:20]
