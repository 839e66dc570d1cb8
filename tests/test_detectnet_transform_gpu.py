"""The DetectNetTransformation kernels on the device, in NaN-prefilled guarded buffers (cases.Guarded): b2c_detectnet_image bit for
bit against the float32 / double restatement of tests/detectnet_transform_oracle.py for every case without rotation, rotation
within a stated bound of the float64 layer, b2c_detectnet_labels bit for bit against the float32 restatement, the malformed
header refusal, and the same bits on a second call."""
import numpy as np
import pytest
import torch

import detectnet_transform_oracle as dto
from cases import Guarded
from caffe_mpi_b200 import capi

pytestmark = pytest.mark.gpu


def run_image(x, augs, OH, OW, mean_value=None, mean_image=None):
    N, _, H, W = x.shape
    X = Guarded(x.size, init=x)
    Y = Guarded(N * 3 * OH * OW)
    ws = torch.full((capi.detectnet_image_workspace_bytes(N, H, W) // 4,), float("nan"), device="cuda")
    A = capi.detectnet_augs(augs)
    M = torch.from_numpy(np.ascontiguousarray(mean_image, np.float32)).cuda() if mean_image is not None else None
    mv = (capi.C.c_float * 3)(*(list(mean_value) * 3 if len(mean_value) == 1 else mean_value)) if mean_value is not None else None
    kind = 2 if mean_image is not None else 1 if mean_value is not None else 0
    capi.check(capi.lib().b2c_detectnet_image(N, H, W, OH, OW, X.ptr(), capi._p(A), kind, capi._p(M), mv, capi._p(ws),
                                              ws.numel() * 4, Y.ptr(), None))
    return Y.read().reshape(N, 3, OH, OW).copy()


def aug(W, H, **kw):
    return dict(dto.identity_aug(W, H), **kw)


# (name, N, H, W, OH, OW, per-image augs as a function of (W, H), mean)
IMAGE_CASES = [
    ("identity", 1, 24, 40, 24, 40, lambda W, H: [aug(W, H)], None),
    ("flip", 2, 24, 40, 24, 40, lambda W, H: [aug(W, H, flip=1), aug(W, H)], None),
    ("crop_neg", 1, 31, 45, 20, 30, lambda W, H: [aug(W, H, crop_x=-7, crop_y=-3)], None),
    ("crop_past_edge", 1, 31, 45, 20, 30, lambda W, H: [aug(W, H, crop_x=30, crop_y=25)], None),
    ("scale_down", 1, 40, 64, 24, 40, lambda W, H: [aug(W, H, scale_w=41, scale_h=27, crop_x=1, crop_y=2)], None),
    ("scale_up", 1, 17, 29, 30, 40, lambda W, H: [aug(W, H, scale_w=45, scale_h=33, crop_x=3, crop_y=1, flip=1)], None),
    ("hue", 2, 19, 23, 19, 23, lambda W, H: [aug(W, H, hue_rotation=29.5), aug(W, H, hue_rotation=-170.0)], None),
    ("desaturation", 1, 19, 23, 19, 23, lambda W, H: [aug(W, H, saturation=0.35)], None),
    ("hue_desat_mean3", 1, 19, 23, 19, 23, lambda W, H: [aug(W, H, hue_rotation=12.0, saturation=0.6)], (104.0, 117.0, 123.0)),
    ("mean1", 1, 19, 23, 19, 23, lambda W, H: [aug(W, H, flip=1)], (110.0,)),
    ("hue_beyond_a_turn", 2, 19, 23, 19, 23, lambda W, H: [aug(W, H, hue_rotation=500.0), aug(W, H, hue_rotation=-700.0)], None),
    ("mean3_fractional", 1, 19, 23, 19, 23, lambda W, H: [aug(W, H, saturation=0.5)], (104.3, 116.77, 122.68)),
    ("mean_image", 1, 19, 23, 16, 20, lambda W, H: [aug(W, H, hue_rotation=5.0, crop_x=2, crop_y=1)], "image"),
    ("kitti_like_n10", 10, 48, 96, 40, 80, None, (104.0,)),
]


def kitti_like_augs(W, H, n):
    rng = np.random.default_rng(7)
    out = []
    for _ in range(n):
        a = dto.draw(lambda: float(rng.random()), W, H, dict(dto.KITTI_AUG, shift_x=8, shift_y=8), 80, 40)
        out.append(a)
    return out


@pytest.mark.parametrize("case", IMAGE_CASES, ids=[c[0] for c in IMAGE_CASES])
def test_image_bit_exact(case):
    name, N, H, W, OH, OW, mk, mean = case
    rng = np.random.default_rng(len(name))
    x = rng.uniform(0, 255, (N, 3, H, W)).astype(np.float32)
    x[:, :, 0, 0] = 0.0                                        # black and grey pixels take the s == 0 branches
    x[:, :, 1, 1] = 128.0
    augs = mk(W, H) if mk else kitti_like_augs(W, H, N)
    mean_image = rng.uniform(0, 255, (3, H, W)).astype(np.float32) if mean == "image" else None
    mean_value = mean if isinstance(mean, tuple) else None
    got = run_image(x, augs, OH, OW, mean_value, mean_image)
    ref = dto.image(x, augs, OH, OW, mean_value, mean_image)
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32), err_msg=name)
    again = run_image(x, augs, OH, OW, mean_value, mean_image)
    np.testing.assert_array_equal(again.view(np.uint32), got.view(np.uint32))


@pytest.mark.parametrize("rot", [3.7, -5.0, 30.0])
def test_image_rotation_within_bound(rot):
    """Rotation passes sinf / cosf (1 ulp each, CUDA's documented bound; the float32 restatement rounds the double functions), so
    the source coordinates differ from the float64 layer by a few ulp of the coordinate: |dx| <= 8 ulp(max(W, H)) ~ 4e-5 here.  The
    bicubic's slope is at most 1.5 * 2 * 255 per pixel of coordinate (the kernel's weights sum to 1; a neighbour swing of 255 in a
    0-255 image), and the float32 evaluation adds a few ulp of 255: |got - ref| <= 2 * 1.5 * 255 * 4e-5 + 8 * ulp(255) ~ 0.03."""
    N, H, W = 1, 40, 56
    rng = np.random.default_rng(11)
    x = rng.uniform(0, 255, (N, 3, H, W)).astype(np.float32)
    augs = [aug(W, H, rotation=rot, scale_w=W + 6, scale_h=H + 4, crop_x=4, crop_y=2, hue_rotation=10.0)]
    got = run_image(x, augs, H, W).astype(np.float64)
    ref = dto.image(x, augs, H, W, dt=np.float64)
    assert np.abs(got - ref).max() <= 0.03, np.abs(got - ref).max()
    np.testing.assert_array_equal(run_image(x, augs, H, W).view(np.uint32), got.astype(np.float32).view(np.uint32))


def run_labels(blob, H, W, augs, gt, status=None):
    N, _, rows, _ = blob.shape
    g = capi.DetectNetGT.make(**gt)
    Cc, GH, GW = capi.detectnet_label_shape(g)
    L = Guarded(blob.size, init=blob)
    T = Guarded(N * Cc * GH * GW)
    S = status if status is not None else torch.zeros(1, dtype=torch.int32, device="cuda")
    capi.check(capi.lib().b2c_detectnet_labels(N, rows, H, W, L.ptr(), capi._p(capi.detectnet_augs(augs)), capi.C.byref(g), T.ptr(),
                                               capi._p(S), None))
    return T.read().reshape(N, Cc, GH, GW).copy(), int(S.item())


def random_boxes(rng, n, W, H, classes=(1,)):
    out = []
    for _ in range(n):
        w, h = rng.uniform(4, W / 2), rng.uniform(4, H / 2)
        out.append((rng.uniform(-W / 8, W - w / 2), rng.uniform(-H / 8, H - h / 2), w, h, 0.0, float(rng.choice(classes)), 0, 0,
                    rng.uniform(0, 0.5)))
    return out


LABEL_CASES = [
    ("max_default", dict(stride=4, image_size_x=64, image_size_y=48), 6, (1,)),
    ("min_objnorm", dict(stride=8, image_size_x=96, image_size_y=64, gridbox_type="GRIDBOX_MIN", min_cvg_len=20, obj_norm=True,
                         scale_cvg=0.4), 8, (1,)),
    ("no_crop", dict(stride=16, image_size_x=96, image_size_y=64, crop_bboxes=False, gridbox_type="GRIDBOX_MIN",
                     min_cvg_len=10, scale_cvg=0.4), 8, (1,)),
    ("classes", dict(stride=4, image_size_x=64, image_size_y=48, object_class=[(1, 0), (2, 1), (5, 3), (2, 2)], max_cvg_len=12),
     12, (1, 2, 5, 7)),
    ("odd_grid", dict(stride=16, image_size_x=100, image_size_y=60, obj_norm=True), 5, (1,)),
]


@pytest.mark.parametrize("case", LABEL_CASES, ids=[c[0] for c in LABEL_CASES])
def test_labels_bit_exact(case):
    name, gt, nboxes, classes = case
    H, W = 50, 70
    rng = np.random.default_rng(len(name) + 3)
    N, rows = 4, nboxes + 3
    box_lists = [random_boxes(rng, k, W, H, classes) for k in (0, nboxes, nboxes + 2, 3)]   # zero boxes and the maximum
    blob = dto.label_blob(box_lists, rows)
    ox, oy = gt["image_size_x"], gt["image_size_y"]
    augs = [aug(W, H, crop_x=-3, crop_y=2), aug(W, H, flip=1, scale_w=80, scale_h=61, crop_x=5, crop_y=4),
            aug(W, H, scale_w=60, scale_h=41, crop_x=(60 - ox) // 2, crop_y=(41 - oy) // 2), aug(W, H, flip=1)]
    got, status = run_labels(blob, H, W, augs, gt)
    assert status == 0
    ref = dto.labels(blob, augs, H, W, gt)
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32), err_msg=name)
    assert got[1:, 0].sum() > 0                               # something was drawn
    again, _ = run_labels(blob, H, W, augs, gt)
    np.testing.assert_array_equal(again.view(np.uint32), got.view(np.uint32))


def test_labels_overlap_order_decides():
    gt = dict(stride=4, image_size_x=32, image_size_y=32, object_class=[(1, 0), (2, 1)])
    a = [(0, 0, 16, 16, 0, 1), (4, 4, 16, 16, 0, 2)]
    blob = dto.label_blob([a, a[::-1]], 3)
    got, _ = run_labels(blob, 32, 32, [aug(32, 32)] * 2, gt)
    np.testing.assert_array_equal(got, dto.labels(blob, [aug(32, 32)] * 2, 32, 32, gt))
    assert got[0, 9, 2, 2] == 1 and got[1, 8, 2, 2] == 1     # cell (2, 2) is the one both cover: the later box wins it


def test_labels_rotation_close():
    gt = dict(stride=4, image_size_x=64, image_size_y=48)
    blob = dto.label_blob([[(10.3, 8.2, 20.1, 14.7, 0, 1)]], 2)
    augs = [aug(70, 50, rotation=3.0, crop_x=2, crop_y=1)]
    got, _ = run_labels(blob, 50, 70, augs, gt)
    ref = dto.labels(blob, augs, 50, 70, gt, dt=np.float64)
    fg = (got[0, 0] == 1) & (ref[0, 0] == 1)
    assert fg.sum() >= 0.8 * max((ref[0, 0] == 1).sum(), 1)
    assert np.abs(got[0, 1:5][:, fg] - ref[0, 1:5][:, fg]).max() <= 1e-3


@pytest.mark.parametrize("header,bit,msg", [((1, 15), capi.DETECTNET_BAD_BOX_LENGTH, "bboxLen == 16"),
                                            ((3, 16), capi.DETECTNET_TOO_MANY_BOXES, "numOfBbox <= height")])
def test_malformed_header_raises_the_reference_message(header, bit, msg):
    blob = dto.label_blob([[(1, 1, 10, 10, 0, 1)], [(1, 1, 10, 10, 0, 1)]], 3)
    blob[1, 0, 0, 0], blob[1, 0, 0, 1] = header
    got, status = run_labels(blob, 32, 32, [aug(32, 32)] * 2, dict(stride=4, image_size_x=32, image_size_y=32))
    assert status == bit
    assert not got[1].any() and got[0, 0].any()              # the malformed image is zeroed, the other drawn
    with pytest.raises(capi.B2CError, match=msg.replace("(", r"\(")):
        capi.detectnet_check_status(status)
