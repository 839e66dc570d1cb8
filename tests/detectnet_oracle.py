"""Float64 forms of the pieces of NVCaffe's DetectNet example (examples/kitti/detectnet_network.prototxt) that are built here: the
L1Loss layer (l1_loss_layer.cpp / .cu) and the label databases DIGITS writes for it, whose datums carry float_data.

L1Loss: diff = a - b, loss = sum |diff| / num; backward to bottom i: (+1, -1)[i] * loss_weight / num * sign(diff), sign(0) = 0
(caffe_cpu_sign).  `l1_loss_f32` restates the kernel's float32 operation order for exact-sum inputs.

Label datum layout (DIGITS' KITTI converter; detectnet_transform_layer.cpp:198-223 reads it back): one channel, max_boxes + 1 rows
of 16 floats.  Row 0 is the header [num_boxes, 16, 0, ...]; rows 1..num_boxes hold one box each: x, y, w, h, alpha, class, scenario,
roty, truncated, occluded, 3 dimensions, 3 locations (BboxLabel_, include/caffe/util/detectnet_coverage.hpp:21-50)."""
import numpy as np

LABEL_COLS = 16


def l1_loss(a, b):
    """(loss, diff) in float64; `a`, `b` are [num, ...]."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    diff = a - b
    return np.abs(diff).sum() / a.shape[0], diff


def l1_backward(diff, num, loss_weight=1.0):
    """(gradient to bottom 0, gradient to bottom 1) (l1_loss_layer.cpp:40-52)."""
    g = np.sign(diff) * (loss_weight / num)
    return g, -g


def l1_loss_f32(a, b, num):
    """The kernel's float32 result when the double sum of |a - b| is exact (small dyadic inputs): d = fl(a - b),
    loss = fl(fl(sum |d|) / num)."""
    d = np.float32(a) - np.float32(b)
    s = np.abs(d).astype(np.float64).sum()
    return np.float32(np.float32(s) / np.float32(num)), d


def l1_backward_f32(diff, alpha):
    """alpha * sign(diff) as the kernel writes it: +-alpha exactly, +0 where diff is 0."""
    alpha = np.float32(alpha)
    return np.where(diff > 0, alpha, np.where(diff < 0, -alpha, np.float32(0))).astype(np.float32)


def label_datum(boxes, max_boxes):
    """[1, max_boxes + 1, 16] float32 label array of one image; `boxes` is [k, 16] (k <= max_boxes)."""
    boxes = np.asarray(boxes, np.float32).reshape(-1, LABEL_COLS)
    assert len(boxes) <= max_boxes
    out = np.zeros((1, max_boxes + 1, LABEL_COLS), np.float32)
    out[0, 0, 0], out[0, 0, 1] = len(boxes), LABEL_COLS
    out[0, 1:1 + len(boxes)] = boxes
    return out


def random_boxes(rng, k, width, height, classes=(0,)):
    """k boxes in a width x height image: x, y, w, h in pixels, `class` from `classes`, the other fields arbitrary."""
    b = np.zeros((k, LABEL_COLS), np.float32)
    b[:, 2] = rng.uniform(8, width / 4, k)
    b[:, 3] = rng.uniform(8, height / 4, k)
    b[:, 0] = rng.uniform(0, width - b[:, 2])
    b[:, 1] = rng.uniform(0, height - b[:, 3])
    b[:, 4] = rng.uniform(-np.pi, np.pi, k)
    b[:, 5] = rng.choice(classes, k)
    b[:, 7:] = rng.standard_normal((k, LABEL_COLS - 7))
    return b
