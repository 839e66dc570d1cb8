"""The neuron layers in TrainNet's set-up, on the stream-order model (tests/sim/libtrainsim.so): PReLU's slope blob (filler, default,
learnable id, the 0-axis channel-shared blob in a .caffemodel read back by google.protobuf), and the in-place and Threshold
refusals at build time with their messages."""
import re

import numpy as np
import pytest

from test_snapshot_cpu import _schema
from test_trainer_sim import SOLVER, sim_host  # noqa: F401  (sim_host: the module fixture)

HEAD = ('name: "neuron" '
        'layer { name: "in" type: "Input" top: "data" top: "label" input_param { shape { dim: 2 dim: 4 dim: 3 dim: 3 } shape { dim: 2 } } }\n'
        'layer { name: "c" type: "Convolution" bottom: "data" top: "c" convolution_param { num_output: 5 kernel_size: 1 } }\n')
TAIL = ('layer { name: "ip" type: "InnerProduct" bottom: "%s" top: "ip" inner_product_param { num_output: 3 } }\n'
        'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')


def net(layer, top="x"):
    return HEAD + layer + "\n" + TAIL % top


@pytest.mark.parametrize("shared", [False, True])
@pytest.mark.parametrize("filler", [None, 0.6])
def test_prelu_slope_filler_and_learnable_id(sim_host, shared, filler):
    q = []
    if filler is not None:
        q.append(f'filler {{ type: "constant" value: {filler} }}')
    if shared:
        q.append("channel_shared: true")
    layer = f'layer {{ name: "x" type: "PReLU" bottom: "c" top: "x" prelu_param {{ {" ".join(q)} }} }}'
    t = sim_host.Trainer(net(layer), SOLVER, num_classes=3)
    assert t.num_learnable() == 2 + 1 + 2                  # conv w, b; the slope (learnable id 2); InnerProduct w, b
    np.testing.assert_array_equal(t.get_param(2), np.full(1 if shared else 5, 0.25 if filler is None else filler, np.float32))


def test_channel_shared_slope_in_caffemodel(sim_host, tmp_path):
    layer = 'layer { name: "x" type: "PReLU" bottom: "c" top: "x" prelu_param { channel_shared: true } }'
    t = sim_host.Trainer(net(layer), SOLVER, num_classes=3)
    t.snapshot(str(tmp_path / "snap"))
    model = next(tmp_path.glob("*.caffemodel"))
    m = _schema()["NetParameter"]()
    m.ParseFromString(model.read_bytes())
    pr = [layer for layer in m.layer if layer.name == "x"][0]
    assert pr.type == "PReLU" and len(pr.blobs) == 1
    blob = pr.blobs[0]
    assert list(blob.shape.dim) == []                       # the reference's 0-axis blob
    data = np.frombuffer(blob.raw_data, np.float32) if blob.HasField("raw_data") else np.array(blob.data, np.float32)
    np.testing.assert_array_equal(data, [0.25])
    t2 = sim_host.Trainer(net(layer), SOLVER, num_classes=3)
    t2.set_param(2, np.array([0.5], np.float32))
    assert t2.copy_trained_layers_from(str(model)) >= 1
    np.testing.assert_array_equal(t2.get_param(2), [0.25])


REFUSED = {
    "absval_in_place": ('layer { name: "x" type: "AbsVal" bottom: "c" top: "c" }', "c", "AbsVal Layer does not allow in-place computation."),
    "bnll_in_place": ('layer { name: "x" type: "BNLL" bottom: "c" top: "c" }', "c",
                      "BNLL Layer does not allow in-place computation when it runs backward"),
    "log_in_place": ('layer { name: "x" type: "Log" bottom: "c" top: "c" log_param { shift: 10 } }', "c",
                     "Log Layer does not allow in-place computation when it runs backward"),
    "power_in_place": ('layer { name: "x" type: "Power" bottom: "c" top: "c" power_param { power: 2 } }', "c",
                       "Power Layer does not allow in-place computation when it runs backward"),
    "threshold_backward": ('layer { name: "x" type: "Threshold" bottom: "c" top: "x" }', "x", "Threshold Layer cannot backpropagate"),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_refusals_at_build_time(sim_host, case):
    layer, top, msg = REFUSED[case]
    sim_host.Net(net(layer, top), is_text=True)             # the net description itself is valid
    with pytest.raises(sim_host.HostError, match=re.escape(msg)):
        sim_host.Trainer(net(layer, top), SOLVER, num_classes=3)


@pytest.mark.parametrize("layer", [
    'layer { name: "x" type: "ELU" bottom: "c" top: "c" }',                                  # in place: the top stands in for x
    'layer { name: "x" type: "Exp" bottom: "c" top: "c" }',                                  # reads y only
    'layer { name: "x" type: "Power" bottom: "c" top: "c" power_param { power: 1 scale: 2 shift: 1 } }',   # the constant gradient
    'layer { name: "x" type: "PReLU" bottom: "c" top: "c" }',
])
def test_in_place_layers_that_build(sim_host, layer):
    sim_host.Trainer(net(layer, "c"), SOLVER, num_classes=3)


def test_in_place_bnll_builds_without_a_backward(sim_host):
    """the in-place refusal is about the backward: a frozen branch (nothing below needs a gradient) builds"""
    frozen = ('name: "neuron" '
              'layer { name: "in" type: "Input" top: "data" top: "label" input_param { shape { dim: 2 dim: 4 dim: 3 dim: 3 } shape { dim: 2 } } }\n'
              'layer { name: "x" type: "BNLL" bottom: "data" top: "data" }\n' + TAIL % "data")
    sim_host.Trainer(frozen, SOLVER, num_classes=3)


def test_tanh_and_scale_stay_refused(sim_host):
    for ty in ("TanH", "Scale"):
        with pytest.raises(sim_host.HostError, match=re.escape(f"layer type '{ty}' is not built yet")):
            sim_host.Trainer(net(f'layer {{ name: "x" type: "{ty}" bottom: "c" top: "x" }}'), SOLVER, num_classes=3)
