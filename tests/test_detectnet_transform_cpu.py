"""DetectNetTransformation on the host: the oracle of tests/detectnet_transform_oracle.py against the closed forms of the
reference's test_detectnet_transform.cpp, the two hue forms, the selection draw with KITTI's parameters, the label map's closed
forms, and the kernels' plan query and label shapes (pure host computation)."""
import math

import numpy as np
import pytest

import detectnet_transform_oracle as dto
from caffe_mpi_b200 import capi

H = W = 32


def bottom(rng, n=1, h=H, w=W):
    return rng.uniform(0, 255, (n, 3, h, w)).astype(np.float32)


def test_no_augmentation_is_identity(rng):
    x = bottom(rng)
    got = dto.image(x, [dto.identity_aug(W, H)], H, W)
    np.testing.assert_array_equal(got, x)


def test_flip_mirrors_columns(rng):
    x = bottom(rng)
    a = dict(dto.identity_aug(W, H), flip=1)
    np.testing.assert_array_equal(dto.image(x, [a], H, W), x[..., ::-1])


@pytest.mark.parametrize("cx,cy", [(5, 3), (-4, -2), (30, 31)])
def test_crop_shifts_with_replicated_border(rng, cx, cy):
    x = bottom(rng)
    a = dict(dto.identity_aug(W, H), crop_x=cx, crop_y=cy)
    got = dto.image(x, [a], H, W)[0]
    ref = np.zeros_like(got)
    for oy in range(H):
        for ox in range(W):
            sy, sx = oy + cy, ox + cx
            sy = 0 if sy == -1 else H - 1 if sy == H else sy
            sx = 0 if sx == -1 else W - 1 if sx == W else sx
            if 0 <= sy < H and 0 <= sx < W:
                ref[:, oy, ox] = x[0, :, sy, sx]
    np.testing.assert_array_equal(got, ref)


@pytest.mark.parametrize("sw,sh", [(16, 16), (48, 40)])
def test_scale_keeps_a_constant_image_and_the_corners(rng, sw, sh):
    x = np.full((1, 3, H, W), 77.0, np.float32)
    a = dict(dto.identity_aug(W, H), scale_w=sw, scale_h=sh)
    np.testing.assert_array_equal(dto.image(x, [a], sh, sw), np.full((1, 3, sh, sw), 77.0, np.float32))
    x = bottom(rng)
    got = dto.image(x, [a], sh, sw, dt=np.float64)[0]
    assert np.allclose(got[:, 0, 0], x[0, :, 0, 0], atol=1e-3)
    assert np.allclose(got[:, -1, -1], x[0, :, -1, -1], atol=1e-3)


def test_rotation_keeps_the_centre_of_a_constant_image():
    x = np.full((1, 3, H, W), 50.0, np.float32)
    a = dict(dto.identity_aug(W, H), rotation=10.0)
    got = dto.image(x, [a], H, W, dt=np.float64)[0]
    assert np.allclose(got[:, 8:24, 8:24], 50.0, atol=1e-9)


def test_full_desaturation_gives_grey(rng):
    x = bottom(rng)
    got = dto.image(x, [dict(dto.identity_aug(W, H), saturation=0.0)], H, W)[0]
    np.testing.assert_array_equal(got[0], x[0].max(axis=0))
    np.testing.assert_array_equal(got[1], got[0])
    np.testing.assert_array_equal(got[2], got[0])


def test_hue_rotation_turns_primaries():
    red = np.zeros((1, 3, 1, 1), np.float32)
    red[0, 0] = 200.0
    # h = 0 - 120 -> 240: blue.  The reference's literal form takes h / 60 = -2 as sector 5 with f = 0: magenta
    got = dto.image(red, [dict(dto.identity_aug(1, 1), hue_rotation=120.0)], 1, 1)[0, :, 0, 0]
    np.testing.assert_array_equal(got, [0.0, 0.0, 200.0])
    lit = dto.colour(red[0], 120.0, 1.0, wrap=False)[:, 0, 0]
    np.testing.assert_array_equal(lit, [200.0, 0.0, 200.0])
    # h = 0 + 120: green, the same in both forms
    got = dto.image(red, [dict(dto.identity_aug(1, 1), hue_rotation=-120.0)], 1, 1)[0, :, 0, 0]
    np.testing.assert_array_equal(got, [0.0, 200.0, 0.0])


@pytest.mark.parametrize("turns", [1, 2, -1, -3])
def test_hue_wraps_by_whole_turns(turns):
    red = np.zeros((3, 1, 1), np.float32)
    red[0] = 200.0
    ref = dto.colour(red, 140.0, 1.0)                     # h = -140 -> 220
    np.testing.assert_array_equal(dto.colour(red, 140.0 + 360.0 * turns, 1.0).view(np.uint32), ref.view(np.uint32))
    np.testing.assert_allclose(ref[:, 0, 0], [0.0, 200 / 3, 200.0], rtol=1e-6)   # sector 3, f = 2/3: (p, q, v)


def test_mean_value_takes_the_reference_round_trip():
    img = np.full((3, 1, 1), 200.0, np.float32)
    got = dto.mean_subtract(img, (104.3, 116.77, 122.68))[:, 0, 0]
    f = np.float32
    want = [f(200) - f(f(f(m) / f(255)) * f(255)) for m in (104.3, 116.77, 122.68)]
    np.testing.assert_array_equal(got, want)
    np.testing.assert_array_equal(dto.mean_subtract(img, (104.0,))[:, 0, 0], [96.0] * 3)   # integer means are unchanged


def test_label_rotation_by_90_degrees_closed_form():
    """A quarter turn of a 100 x 50 image: the rotated frame is 50 x 100 with its corner at (25, -25) of the old one, so a point
    (px, py) goes to (50 - py, px); the box keeps its size and is placed by its centre (20, 10) -> (40, 20)."""
    a = dict(dto.identity_aug(100, 50), rotation=90.0)
    gt = dict(crop_bboxes=False, image_size_x=50, image_size_y=100)
    for dt in (np.float32, np.float64):
        (x, y, w, h, dst), = dto.transform_boxes([(10, 5, 20, 10, 0, 1)], a, 50, 100, gt, dt)
        assert (x, y, w, h) == pytest.approx((30, 15, 20, 10), abs=1e-4)


@pytest.mark.parametrize("rot,sw,sh", [(3.0, 70, 50), (-5.0, 1242, 375), (30.0, 64, 48), (90.0, 100, 50), (-41.5, 33, 71)])
def test_label_rotation_matches_opencv(rot, sw, sh):
    """The label rotation against the reference's getTransformationMatrix, rebuilt from OpenCV itself: the corners of the
    unrotated and of the rotated rectangle (cv::RotatedRect::points), the rotated rectangle shifted by its integer bounding box's
    corner, and cv::getAffineTransform between the two; the box centre is mapped and the box keeps its size."""
    cv2 = pytest.importorskip("cv2")
    c = (sw * 0.5, sh * 0.5)
    src = cv2.boxPoints((c, (sw, sh), 0.0)).astype(np.float32)
    pts = cv2.boxPoints((c, (sw, sh), rot))
    tlx, tly = np.floor(pts[:, 0].min()), np.floor(pts[:, 1].min())
    assert (tlx, tly) == dto.rotated_bounding_tl(sw, sh, rot)[:2]
    dst = cv2.boxPoints(((c[0] - tlx, c[1] - tly), (sw, sh), rot)).astype(np.float32)
    M = cv2.getAffineTransform(src[:3], dst[:3]).astype(np.float32)
    rng = np.random.default_rng(int(sw))
    boxes = [(rng.uniform(0, sw * 0.7), rng.uniform(0, sh * 0.7), rng.uniform(5, sw * 0.3), rng.uniform(5, sh * 0.3), 0, 1)
             for _ in range(6)]
    a = dict(dto.identity_aug(sw, sh), rotation=rot)
    got = dto.transform_boxes(boxes, a, sh, sw, dict(crop_bboxes=False), np.float64)
    for (x, y, w, h, _, _), (gx, gy, gw, gh, _) in zip(boxes, got):
        ctr = M @ np.array([x + w / 2, y + h / 2, 1.0], np.float32)
        assert (gx, gy, gw, gh) == pytest.approx((ctr[0] - w / 2, ctr[1] - h / 2, w, h), abs=2e-3)


@pytest.mark.parametrize("rot", [30.0, -30.0, 15.5, -59.0, 179.0, -180.0, 1e-3])
def test_hue_forms_agree_where_the_reference_is_right(rng, rot):
    img = rng.uniform(0, 255, (3, 64, 64)).astype(np.float32)
    wrapped = dto.colour(img, rot, 0.6, wrap=True)
    literal = dto.colour(img, rot, 0.6, wrap=False)
    h = dto.hue(img) - np.float32(rot)
    inside = (h >= -60) & (h < 360)
    assert inside.any()
    np.testing.assert_array_equal(wrapped.view(np.uint32)[:, inside], literal.view(np.uint32)[:, inside])
    if (~inside).any() and abs(rot) > 60:
        assert not np.array_equal(wrapped[:, ~inside], literal[:, ~inside])


def test_draw_frequencies_with_kitti_parameters():
    """10^5 selections with KITTI's augmentation: each augmentation's frequency within 5 sigma of its probability, the drawn
    values within their ranges, and the crop offsets between -shift/2 and size - out + shift/2."""
    rng = np.random.default_rng(1701)
    u = rng.random(2_000_000)
    it = iter(u)
    p = dto.KITTI_AUG
    n = 100_000
    Wb, Hb = 1242, 375
    hue = sat = flip = scale = 0
    for _ in range(n):
        a = dto.draw(lambda: next(it), Wb, Hb, p)
        hue += a["hue_rotation"] != 0
        sat += a["saturation"] != 1
        flip += a["flip"]
        sc = (a["scale_w"], a["scale_h"]) != (Wb, Hb)
        scale += sc
        assert -30 <= a["hue_rotation"] <= 30
        assert 0.2 - 1e-6 <= a["saturation"] <= 1
        assert round(Wb * 0.8) - 1 <= a["scale_w"] <= round(Wb * 1.2) + 1
        assert a["rotation"] == 0
        for off, size, out in ((a["crop_x"], a["scale_w"], 1248), (a["crop_y"], a["scale_h"], 384)):
            lo, hi = sorted((-16, size - out + 16))       # pct * (size - out + shift) - shift / 2 for pct in [0, 1]
            assert lo <= off <= hi
    for count, prob in ((hue, 0.8), (sat, 0.8), (flip, 0.5), (scale, 0.4)):
        assert abs(count - n * prob) <= 5 * math.sqrt(n * prob * (1 - prob)), (count, prob)


def test_draw_test_phase_is_the_fixed_selection():
    a = dto.draw(lambda: 0.0, 1242, 375, dto.KITTI_AUG, train=False)
    assert a == dict(dto.identity_aug(1248, 384))


def test_draw_rotation_uses_the_rotated_bounding_size():
    vals = iter([1.0, 1.0, 1.0, 1.0, 0.0, 1.0, 0.0, 0.5, 0.5])   # hue off, desat off, no flip, no scale, rotate by +max, crop
    a = dto.draw(lambda: next(vals), 100, 50, dict(max_rotate_degree=10.0, rotation_prob=0.5, crop_prob=1.0), 80, 40)
    assert a["rotation"] == pytest.approx(10.0)
    th = math.radians(10.0)
    bw = 100 * math.cos(th) + 50 * math.sin(th)
    assert abs(a["crop_x"] - 0.5 * (bw - 80)) <= 2


def test_labels_closed_form_single_box():
    gt = dict(stride=4, image_size_x=32, image_size_y=32, scale_cvg=0.5, gridbox_type="GRIDBOX_MAX", max_cvg_len=50)
    blob = dto.label_blob([[(0, 0, 16, 16, 0, 1)]], 2)
    got = dto.labels(blob, [dto.identity_aug(32, 32)], 32, 32, gt)[0]
    assert got.shape == (9, 8, 8)
    fg = np.zeros((8, 8), bool)
    fg[1:3, 1:3] = True                        # coverage: centre (8, 8), 8 x 8 -> cells 1, 2
    np.testing.assert_array_equal(got[0] == 1, fg)
    np.testing.assert_array_equal(got[8], got[0])
    np.testing.assert_array_equal(got[1][fg], [-4, -8, -4, -8])
    np.testing.assert_array_equal(got[3][fg], [12, 8, 12, 8])
    assert np.all(got[5][fg] == np.float32(1 / 16)) and np.all(got[7][fg] == 1)
    # obj_norm: stride^2 / coverage area = 16 / 64
    got = dto.labels(blob, [dto.identity_aug(32, 32)], 32, 32, dict(gt, obj_norm=True))[0]
    assert np.all(got[7][fg] == np.float32(0.25))


def test_labels_drop_unmapped_classes_and_later_boxes_win():
    gt = dict(stride=4, image_size_x=32, image_size_y=32, object_class=[(1, 0), (2, 1)])
    blob = dto.label_blob([[(0, 0, 16, 16, 0, 1), (4, 4, 16, 16, 0, 2), (0, 0, 30, 30, 0, 7)]], 4)
    got = dto.labels(blob, [dto.identity_aug(32, 32)], 32, 32, gt)[0]
    assert got.shape[0] == 10
    assert got[9, 2, 2] == 1 and got[8, 2, 2] == 0          # the class-2 box overwrote the class-1 box where both cover
    assert got[8, 1, 1] == 1


def test_label_shape_matches_kitti_and_rounds_other_sizes():
    g = capi.DetectNetGT.make(**{k: v for k, v in dto.KITTI_GT.items() if k != "coverage_type"})
    assert capi.detectnet_label_shape(g) == (9, 24, 78) == dto.label_shape(dto.KITTI_GT)
    for sx, sy, st in ((100, 60, 16), (104, 72, 16), (33, 17, 4)):
        g = capi.DetectNetGT.make(image_size_x=sx, image_size_y=sy, stride=st, object_class=[(1, 0), (3, 2)])
        assert capi.detectnet_label_shape(g) == dto.label_shape(dict(image_size_x=sx, image_size_y=sy, stride=st,
                                                                     object_class=[(1, 0), (3, 2)]))


def test_plan_query():
    p = capi.detectnet_plan("image", 10, 384, 1248, 384, 1248)
    assert p["launches"] == 2 and p["threads"] == 256
    assert p["workspace"] == 10 * 3 * 384 * 1248 * 4 == capi.detectnet_image_workspace_bytes(10, 384, 1248)
    g = capi.DetectNetGT.make(stride=16)
    p = capi.detectnet_plan("labels", 10, 375, 1242, rows=51, gt=g)
    assert p == dict(ctas=10, threads=256, smem=50 * 64, channels=9, grid_h=24, grid_w=78)
    with pytest.raises(capi.B2CError, match="box rows"):
        capi.detectnet_plan("labels", 10, 375, 1242, rows=2000, gt=g)
    with pytest.raises(capi.B2CError, match="stride"):
        capi.detectnet_plan("labels", 1, 8, 8, rows=2, gt=capi.DetectNetGT.make(stride=0))
