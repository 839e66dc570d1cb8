"""Layer parameters reaching TrainNet's layers, on the stream-order model (tests/sim/libtrainsim.so): the parameter values the
layers refuse, with their messages, and BatchNorm fillers landing in the learnable blobs they fill."""
import re

import numpy as np
import pytest

from test_trainer_sim import SOLVER, sim_host  # noqa: F401  (sim_host: the module fixture)

HEAD = ('name: "params" '
        'layer { name: "in" type: "Input" top: "data" top: "label" input_param { shape { dim: 2 dim: 4 dim: 3 dim: 3 } shape { dim: 2 } } }\n')
TAIL = ('layer { name: "ip" type: "InnerProduct" bottom: "%s" top: "ip" inner_product_param { num_output: 3 } }\n'
        'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "ip" bottom: "label" top: "loss" }\n')


def net(layer, top="x"):
    return HEAD + layer + "\n" + TAIL % top


REFUSED = {
    "eltwise_prod": ('layer { name: "x" type: "Eltwise" bottom: "data" bottom: "data" top: "x" eltwise_param { operation: PROD } }',
                     "Eltwise PROD / MAX are not built (the BASELINE nets use SUM)"),
    "eltwise_max": ('layer { name: "x" type: "Eltwise" bottom: "data" bottom: "data" top: "x" eltwise_param { operation: MAX } }',
                    "Eltwise PROD / MAX are not built (the BASELINE nets use SUM)"),
    "eltwise_coeff": ('layer { name: "x" type: "Eltwise" bottom: "data" bottom: "data" top: "x" eltwise_param { coeff: 1 coeff: 2 } }',
                      "Eltwise SUM is built for unit coefficients only"),
    "lrn_within": ('layer { name: "x" type: "LRN" bottom: "data" top: "x" lrn_param { norm_region: WITHIN_CHANNEL } }',
                   "LRN WITHIN_CHANNEL is not built (the BASELINE nets use ACROSS_CHANNELS)"),
    "concat_axis0": ('layer { name: "x" type: "Concat" bottom: "data" bottom: "data" top: "x" concat_param { axis: 0 } }',
                     "Concat is built for the channel axis only"),
    "tanh": ('layer { name: "x" type: "TanH" bottom: "data" top: "x" }', "layer type 'TanH' is not built yet"),
    "scale": ('layer { name: "x" type: "Scale" bottom: "data" top: "x" scale_param { bias_term: true } }', "layer type 'Scale' is not built yet"),
}


@pytest.mark.parametrize("case", sorted(REFUSED))
def test_layer_parameters_the_trainer_does_not_build_are_refused_with_their_message(sim_host, case):
    layer, msg = REFUSED[case]
    sim_host.Net(net(layer), is_text=True)                   # the net description itself is valid
    with pytest.raises(sim_host.HostError, match=re.escape(msg)):
        sim_host.Trainer(net(layer), SOLVER, num_classes=3)


def test_batchnorm_fillers_fill_its_scale_and_bias_blobs(sim_host):
    """scale_filler / bias_filler alone imply scale_bias (NVCaffe BatchNormParameter): blobs 3 and 4 exist, are learnable ids 3 and 4
    after the three statistics, and hold the fillers' constants"""
    bn = ('layer { name: "x" type: "BatchNorm" bottom: "data" top: "x" batch_norm_param { '
          'scale_filler { type: "constant" value: 2.5 } bias_filler { type: "constant" value: -0.75 } } }')
    assert [p[:2] for p in sim_host.Net(net(bn), is_text=True).learnable_params()] == [("x", 4), ("x", 4), ("ip", 3 * 36), ("ip", 3)]
    t = sim_host.Trainer(net(bn), SOLVER, num_classes=3)
    assert t.num_learnable() == 5 + 2                        # mean, variance, correction, scale, bias; InnerProduct's weight and bias
    assert t.num_params() == 2 + 2                           # trainable: learnable ids 3 and 4, then InnerProduct's
    t.layer_blob_pointers(1, 4)
    with pytest.raises(sim_host.HostError):
        t.layer_blob_pointers(1, 5)
    np.testing.assert_array_equal(t.get_param(0), np.full(4, 2.5, np.float32))
    np.testing.assert_array_equal(t.get_param(1), np.full(4, -0.75, np.float32))
