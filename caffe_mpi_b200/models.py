"""Prototxt text generators for the BASELINE nets (bench.py builds the architectures of the reference's models/*.prototxt
from here; tests/test_prototxt.py checks that the generated net has exactly the inventory of the reference file, stored
under tests/golden/reference_models).  Layer and blob names follow
models/resnet50/train_val.prototxt (res<stage>.<block>.conv<k>, .../bn, .skipConv, .sum, .relu, pool1/pool2, fc, loss)."""


def _conv(name, bottom, top, num_output, k, stride=1, pad=0):
    extra = (f" stride: {stride}" if stride != 1 else "") + (f" pad: {pad}" if pad else "")
    return (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{top}"\n'
            f'  convolution_param {{ num_output: {num_output} kernel_size: {k}{extra} weight_filler {{ type: "msra" }} bias_term: false }} }}\n')


def _bn(name, bottom, top):
    return (f'layer {{ name: "{name}" type: "BatchNorm" bottom: "{bottom}" top: "{top}"\n'
            f'  batch_norm_param {{ moving_average_fraction: 0.9 eps: 0.0001 scale_bias: true }} }}\n')


def _relu(name, blob):
    return f'layer {{ name: "{name}" type: "ReLU" bottom: "{blob}" top: "{blob}" }}\n'


def resnet50_prototxt(batch=32, crop=224, num_classes=1000):
    s = 'name: "Resnet50"\n'
    s += (f'layer {{ name: "data" type: "Data" top: "data" top: "label" data_param {{ source: "synthetic" batch_size: {batch} backend: LMDB }}\n'
          f'  transform_param {{ crop_size: {crop} mirror: true mean_value: 104 mean_value: 117 mean_value: 123 }} include: {{ phase: TRAIN }} }}\n')
    s += _conv("conv1", "data", "conv1", 64, 7, 2, 3) + _bn("conv1/bn", "conv1", "conv1/bn") + _relu("conv1/relu", "conv1/bn")
    s += 'layer { name: "pool1" type: "Pooling" bottom: "conv1/bn" top: "pool1" pooling_param { pool: MAX kernel_size: 3 stride: 2 } }\n'
    prev = "pool1"
    for stage, (blocks, mid, out) in zip((2, 3, 4, 5), ((3, 64, 256), (4, 128, 512), (6, 256, 1024), (3, 512, 2048))):
        for blk in range(1, blocks + 1):
            p = f"res{stage}.{blk}"
            stride = 2 if (blk == 1 and stage > 2) else 1          # stride sits on the 1x1 convs in this variant
            s += _conv(f"{p}.conv1", prev, f"{p}.conv1", mid, 1, stride) + _bn(f"{p}.conv1/bn", f"{p}.conv1", f"{p}.conv1/bn") + _relu(f"{p}.conv1/relu", f"{p}.conv1/bn")
            s += _conv(f"{p}.conv2", f"{p}.conv1/bn", f"{p}.conv2", mid, 3, 1, 1) + _bn(f"{p}.conv2/bn", f"{p}.conv2", f"{p}.conv2/bn") + _relu(f"{p}.conv2/relu", f"{p}.conv2/bn")
            s += _conv(f"{p}.conv3", f"{p}.conv2/bn", f"{p}.conv3", out, 1) + _bn(f"{p}.conv3/bn", f"{p}.conv3", f"{p}.conv3/bn")
            if blk == 1:
                s += _conv(f"{p}.skipConv", prev, f"{p}.skipConv", out, 1, stride) + _bn(f"{p}.skipConv/bn", f"{p}.skipConv", f"{p}.skipConv/bn")
                short = f"{p}.skipConv/bn"
            else:
                short = prev
            s += (f'layer {{ name: "{p}.sum" type: "Eltwise" bottom: "{p}.conv3/bn" bottom: "{short}" top: "{p}.sum" eltwise_param {{ operation: SUM }} }}\n')
            s += _relu(f"{p}.relu", f"{p}.sum")
            prev = f"{p}.sum"
    s += f'layer {{ name: "pool2" type: "Pooling" bottom: "{prev}" top: "pool2" pooling_param {{ pool: AVE kernel_size: 7 }} }}\n'
    s += (f'layer {{ name: "fc" type: "InnerProduct" bottom: "pool2" top: "fc" inner_product_param {{ num_output: {num_classes}\n'
          f'  weight_filler {{ type: "msra" }} bias_filler {{ type: "constant" value: 0 }} }} }}\n')
    s += 'layer { name: "loss" type: "SoftmaxWithLoss" bottom: "fc" bottom: "label" top: "loss" }\n'
    return s


RESNET50_SOLVER = ('base_lr: 0.001 lr_policy: "poly" power: 2.0 momentum: 0.9 weight_decay: 1e-4 max_iter: 2400000 '
                   'solver_mode: GPU random_seed: 1')    # models/resnet50/solver.prototxt (training hyper-parameters)


# ---- AlexNet / VGG-16 / GoogLeNet / LeNet: the same graphs as the reference's models/*/train_val.prototxt (TRAIN phase) ----
def _data(batch, crop):
    return (f'layer {{ name: "data" type: "Data" top: "data" top: "label" data_param {{ source: "synthetic" batch_size: {batch} backend: LMDB }}\n'
            f'  transform_param {{ crop_size: {crop} mirror: true mean_value: 104 mean_value: 117 mean_value: 123 }} include: {{ phase: TRAIN }} }}\n')


_SPECS = ""     # ParamSpecs emitted by _convb / _ip; set per net (the NVCaffe AlexNet / VGG files carry none)


def _convb(name, bottom, num_output, k, stride=1, pad=0, group=1, wfill='type: "gaussian" std: 0.01', bias=0.0, top=None):
    """Convolution with bias."""
    top = top or name
    extra = (f" stride: {stride}" if stride != 1 else "") + (f" pad: {pad}" if pad else "") + (f" group: {group}" if group != 1 else "")
    return (f'layer {{ name: "{name}" type: "Convolution" bottom: "{bottom}" top: "{top}"{_SPECS}\n'
            f'  convolution_param {{ num_output: {num_output} kernel_size: {k}{extra} weight_filler {{ {wfill} }} bias_filler {{ type: "constant" value: {bias} }} }} }}\n')


def _ip(name, bottom, num_output, wfill='type: "gaussian" std: 0.005', bias=0.1):
    return (f'layer {{ name: "{name}" type: "InnerProduct" bottom: "{bottom}" top: "{name}"{_SPECS}\n'
            f'  inner_product_param {{ num_output: {num_output} weight_filler {{ {wfill} }} bias_filler {{ type: "constant" value: {bias} }} }} }}\n')


def _pool(name, bottom, method, k, stride=1, pad=0):
    return (f'layer {{ name: "{name}" type: "Pooling" bottom: "{bottom}" top: "{name}" pooling_param {{ pool: {method} kernel_size: {k} stride: {stride}'
            + (f" pad: {pad}" if pad else "") + ' } }\n')


def _lrn(name, bottom):
    return f'layer {{ name: "{name}" type: "LRN" bottom: "{bottom}" top: "{name}" lrn_param {{ local_size: 5 alpha: 0.0001 beta: 0.75 }} }}\n'


def _drop(name, blob, ratio=0.5):
    return f'layer {{ name: "{name}" type: "Dropout" bottom: "{blob}" top: "{blob}" dropout_param {{ dropout_ratio: {ratio} }} }}\n'


def _loss(name, bottom, top="loss", weight=None):
    lw = f" loss_weight: {weight}" if weight is not None else ""
    return f'layer {{ name: "{name}" type: "SoftmaxWithLoss" bottom: "{bottom}" bottom: "label" top: "{top}"{lw} }}\n'


def alexnet_prototxt(batch=256, crop=227, num_classes=1000):
    """models/bvlc_alexnet/train_val.prototxt: 5 convs (conv2/4/5 with group 2), 2 LRN, 3 max pools, fc6/fc7 with dropout, fc8."""
    s = 'name: "AlexNet"\n' + _data(batch, crop)
    s += _convb("conv1", "data", 96, 11, 4) + _relu("relu1", "conv1") + _lrn("norm1", "conv1") + _pool("pool1", "norm1", "MAX", 3, 2)
    s += _convb("conv2", "pool1", 256, 5, 1, 2, 2, bias=0.1) + _relu("relu2", "conv2") + _lrn("norm2", "conv2") + _pool("pool2", "norm2", "MAX", 3, 2)
    s += _convb("conv3", "pool2", 384, 3, 1, 1) + _relu("relu3", "conv3")
    s += _convb("conv4", "conv3", 384, 3, 1, 1, 2, bias=0.1) + _relu("relu4", "conv4")
    s += _convb("conv5", "conv4", 256, 3, 1, 1, 2, bias=0.1) + _relu("relu5", "conv5") + _pool("pool5", "conv5", "MAX", 3, 2)
    s += _ip("fc6", "pool5", 4096) + _relu("relu6", "fc6") + _drop("drop6", "fc6")
    s += _ip("fc7", "fc6", 4096) + _relu("relu7", "fc7") + _drop("drop7", "fc7")
    s += _ip("fc8", "fc7", num_classes, 'type: "gaussian" std: 0.01', 0.0) + _loss("loss", "fc8")
    return s


def vgg16_prototxt(batch=32, crop=224, num_classes=1000):
    """models/vgg16/train_val.prototxt: 13 3x3 / pad 1 convs in 5 blocks, max pools, fc6/fc7 with dropout, fc8."""
    s = 'name: "VGG16"\n' + _data(batch, crop)
    prev = "data"
    for blk, (n, ch) in enumerate(((2, 64), (2, 128), (3, 256), (3, 512), (3, 512)), 1):
        for i in range(1, n + 1):
            nm = f"conv{blk}_{i}"
            s += _convb(nm, prev, ch, 3, 1, 1, wfill='type: "xavier"') + _relu(f"relu{blk}_{i}", nm)
            prev = nm
        s += _pool(f"pool{blk}", prev, "MAX", 2, 2)
        prev = f"pool{blk}"
    s += _ip("fc6", prev, 4096, 'type: "xavier"', 0.1) + _relu("relu6", "fc6") + _drop("drop6", "fc6")
    s += _ip("fc7", "fc6", 4096, 'type: "xavier"', 0.1) + _relu("relu7", "fc7") + _drop("drop7", "fc7")
    s += _ip("fc8-5", "fc7", num_classes, 'type: "xavier"', 0.1) + _loss("loss", "fc8-5")
    return s


_INCEPTION = {  # module: (1x1, 3x3_reduce, 3x3, 5x5_reduce, 5x5, pool_proj)
    "3a": (64, 96, 128, 16, 32, 32), "3b": (128, 128, 192, 32, 96, 64),
    "4a": (192, 96, 208, 16, 48, 64), "4b": (160, 112, 224, 24, 64, 64), "4c": (128, 128, 256, 24, 64, 64),
    "4d": (112, 144, 288, 32, 64, 64), "4e": (256, 160, 320, 32, 128, 128),
    "5a": (256, 160, 320, 32, 128, 128), "5b": (384, 192, 384, 48, 128, 128),
}


def googlenet_prototxt(batch=128, crop=224, num_classes=1000):
    """models/bvlc_googlenet/train_val.prototxt: stem, nine inception modules (1x1 / 3x3 / 5x5 / pool-proj branches joined by
    Concat), two auxiliary classifiers with loss_weight 0.3, average pool + dropout + classifier."""
    xav = 'type: "xavier"'
    s = 'name: "GoogleNet"\n' + _data(batch, crop)
    s += _convb("conv1/7x7_s2", "data", 64, 7, 2, 3, wfill=xav, bias=0.2) + _relu("conv1/relu_7x7", "conv1/7x7_s2")
    s += _pool("pool1/3x3_s2", "conv1/7x7_s2", "MAX", 3, 2) + _lrn("pool1/norm1", "pool1/3x3_s2")
    s += _convb("conv2/3x3_reduce", "pool1/norm1", 64, 1, wfill=xav, bias=0.2) + _relu("conv2/relu_3x3_reduce", "conv2/3x3_reduce")
    s += _convb("conv2/3x3", "conv2/3x3_reduce", 192, 3, 1, 1, wfill=xav, bias=0.2) + _relu("conv2/relu_3x3", "conv2/3x3")
    s += _lrn("conv2/norm2", "conv2/3x3") + _pool("pool2/3x3_s2", "conv2/norm2", "MAX", 3, 2)
    prev = "pool2/3x3_s2"

    def aux(tag, bottom):
        t = _pool(f"{tag}/ave_pool", bottom, "AVE", 5, 3)
        t += _convb(f"{tag}/conv", f"{tag}/ave_pool", 128, 1, wfill=xav, bias=0.2) + _relu(f"{tag}/relu_conv", f"{tag}/conv")
        t += _ip(f"{tag}/fc", f"{tag}/conv", 1024, xav, 0.2) + _relu(f"{tag}/relu_fc", f"{tag}/fc") + _drop(f"{tag}/drop_fc", f"{tag}/fc", 0.5)
        t += _ip(f"{tag}/classifier", f"{tag}/fc", num_classes, xav, 0.0) + _loss(f"{tag}/loss", f"{tag}/classifier", f"{tag}/loss1", 0.3)
        return t

    for mod in ("3a", "3b", "4a", "4b", "4c", "4d", "4e", "5a", "5b"):
        c1, r3, c3, r5, c5, pp = _INCEPTION[mod]
        p = f"inception_{mod}"
        s += _convb(f"{p}/1x1", prev, c1, 1, wfill=xav, bias=0.2) + _relu(f"{p}/relu_1x1", f"{p}/1x1")
        s += _convb(f"{p}/3x3_reduce", prev, r3, 1, wfill=xav, bias=0.2) + _relu(f"{p}/relu_3x3_reduce", f"{p}/3x3_reduce")
        s += _convb(f"{p}/3x3", f"{p}/3x3_reduce", c3, 3, 1, 1, wfill=xav, bias=0.2) + _relu(f"{p}/relu_3x3", f"{p}/3x3")
        s += _convb(f"{p}/5x5_reduce", prev, r5, 1, wfill=xav, bias=0.2) + _relu(f"{p}/relu_5x5_reduce", f"{p}/5x5_reduce")
        s += _convb(f"{p}/5x5", f"{p}/5x5_reduce", c5, 5, 1, 2, wfill=xav, bias=0.2) + _relu(f"{p}/relu_5x5", f"{p}/5x5")
        s += _pool(f"{p}/pool", prev, "MAX", 3, 1, 1)
        s += _convb(f"{p}/pool_proj", f"{p}/pool", pp, 1, wfill=xav, bias=0.2) + _relu(f"{p}/relu_pool_proj", f"{p}/pool_proj")
        s += (f'layer {{ name: "{p}/output" type: "Concat" bottom: "{p}/1x1" bottom: "{p}/3x3" bottom: "{p}/5x5" bottom: "{p}/pool_proj" top: "{p}/output" }}\n')
        prev = f"{p}/output"
        if mod == "3b":
            s += _pool("pool3/3x3_s2", prev, "MAX", 3, 2); prev = "pool3/3x3_s2"
        elif mod == "4a":
            s += aux("loss1", prev)
        elif mod == "4d":
            s += aux("loss2", prev)
        elif mod == "4e":
            s += _pool("pool4/3x3_s2", prev, "MAX", 3, 2); prev = "pool4/3x3_s2"
    s += _pool("pool5/7x7_s1", prev, "AVE", 7, 1) + _drop("pool5/drop_7x7_s1", "pool5/7x7_s1", 0.5)
    s += _ip("loss3/classifier", "pool5/7x7_s1", num_classes, xav, 0.0) + _loss("loss", "loss3/classifier", "loss", 1)
    return s


def lenet_prototxt(batch=64, num_classes=10):
    """examples/mnist/lenet_train_test.prototxt (BASELINE configs[0]); 28x28x1 input; weight lr_mult 1, bias lr_mult 2."""
    global _SPECS
    xav = 'type: "xavier"'
    s = 'name: "LeNet"\n'
    _SPECS = " param { lr_mult: 1 } param { lr_mult: 2 }"
    s += f'layer {{ name: "mnist" type: "Input" top: "data" top: "label" input_param {{ shape {{ dim: {batch} dim: 1 dim: 28 dim: 28 }} shape {{ dim: {batch} }} }} }}\n'
    s += _convb("conv1", "data", 20, 5, wfill=xav) + _pool("pool1", "conv1", "MAX", 2, 2)
    s += _convb("conv2", "pool1", 50, 5, wfill=xav) + _pool("pool2", "conv2", "MAX", 2, 2)
    s += _ip("ip1", "pool2", 500, xav, 0.0) + _relu("relu1", "ip1") + _ip("ip2", "ip1", num_classes, xav, 0.0) + _loss("loss", "ip2")
    _SPECS = ""
    return s


# solver hyper-parameters of the reference's models/*/solver.prototxt (the fields the SGD path reads)
SOLVERS = {
    "resnet50": RESNET50_SOLVER,
    "alexnet": 'base_lr: 0.01 lr_policy: "poly" power: 2.0 momentum: 0.9 weight_decay: 0.0005 max_iter: 300000 solver_mode: GPU',
    "vgg16": 'base_lr: 0.005 lr_policy: "poly" power: 2.0 momentum: 0.9 weight_decay: 0.0005 max_iter: 2400000 solver_mode: GPU',
    "googlenet": 'base_lr: 0.01 lr_policy: "poly" power: 2.0 momentum: 0.9 weight_decay: 0.0002 max_iter: 2600 solver_mode: GPU',
    "lenet": 'base_lr: 0.01 lr_policy: "inv" gamma: 0.0001 power: 0.75 momentum: 0.9 weight_decay: 0.0005 max_iter: 10000 solver_mode: GPU',
}
PROTOTXT = {"resnet50": resnet50_prototxt, "alexnet": alexnet_prototxt, "vgg16": vgg16_prototxt, "googlenet": googlenet_prototxt,
            "lenet": lenet_prototxt}
# BASELINE.json configs: per-GPU batch and input size of each model
BASELINE_BATCH = {"resnet50": 64, "alexnet": 256, "vgg16": 32, "googlenet": 128, "lenet": 64}
