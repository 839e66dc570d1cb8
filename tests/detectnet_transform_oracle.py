"""DetectNetTransformation restated on the host: the image path (colour, mean, bicubic sampling) and the label path (box transform,
pruning, rectangular coverage), each in a dtype the caller picks.  With dt=np.float32 they are the kernels' arithmetic op for op
(float coordinates and HSV, the cubic in double, every product rounded before it is summed), so the GPU results match them bit for
bit wherever sinf / cosf do not enter (no rotation).  With dt=np.float64 they are the layer in double: the yardstick rotation is
held to.  Also the reference's selection draw (get_augmentations) over any uniform stream, and both hue forms."""
import math

import numpy as np

FLT_EPSILON = np.float32(np.finfo(np.float32).eps)

# DetectNetAugmentationParameter / DetectNetGroundTruthParameter defaults (caffe.proto)
AUG_DEFAULTS = dict(crop_prob=1.0, shift_x=0, shift_y=0, scale_prob=0.33, scale_min=0.7, scale_max=1.0, flip_prob=0.33,
                    rotation_prob=0.33, max_rotate_degree=1.0, hue_rotation_prob=0.33, hue_rotation=15.0, desaturation_prob=0.33,
                    desaturation_max=0.5)
GT_DEFAULTS = dict(stride=4, scale_cvg=0.5, gridbox_type="GRIDBOX_MAX", max_cvg_len=50, min_cvg_len=50, image_size_x=1248,
                   image_size_y=384, obj_norm=False, crop_bboxes=True, object_class=())
# examples/kitti/detectnet_network.prototxt
KITTI_AUG = dict(crop_prob=1.0, shift_x=32, shift_y=32, flip_prob=0.5, rotation_prob=0.0, max_rotate_degree=5.0, scale_prob=0.4,
                 scale_min=0.8, scale_max=1.2, hue_rotation_prob=0.8, hue_rotation=30.0, desaturation_prob=0.8,
                 desaturation_max=0.8)
KITTI_GT = dict(stride=16, scale_cvg=0.4, gridbox_type="GRIDBOX_MIN", min_cvg_len=20, coverage_type="RECTANGULAR",
                image_size_x=1248, image_size_y=384, obj_norm=True, crop_bboxes=False)


def identity_aug(W, H):
    return dict(hue_rotation=0.0, saturation=1.0, flip=0, scale_w=W, scale_h=H, rotation=0.0, crop_x=0, crop_y=0)


# ---- colour --------------------------------------------------------------------------------------------------------------------
def colour(img, hue, sat, wrap=True, dt=np.float32):
    """img [3, H, W] -> [3, H, W]: RGB -> HSV -> RGB with h -= hue and s *= sat where the reference applies them.  wrap=False is
    the reference's literal form (hue never wrapped; every sector outside 0..5 taken as 5); wrap=True brings h into [-60, 360)
    by whole turns first, as the kernel does."""
    hue, sat = dt(hue), dt(sat)
    do_hue = abs(np.float32(hue)) > FLT_EPSILON
    do_sat = float(np.float32(sat)) < 1.0 - 1.0 / 255
    r, g, b = (np.asarray(c, dt).copy() for c in img)
    if not (do_hue or do_sat):
        return np.stack([r, g, b])
    with np.errstate(all="ignore"):
        mn, mx = np.minimum(np.minimum(r, g), b), np.maximum(np.maximum(r, g), b)
        delta = mx - mn
        zero = (mx == 0) | (delta == 0)
        h = np.where(r == mx, (g - b) / delta, np.where(g == mx, dt(2) + (b - r) / delta, dt(4) + (r - g) / delta)) * dt(60)
        s = delta / mx
        h = np.where(zero, dt(0), h)
        s = np.where(zero, dt(0), s)
        v = mx
        if do_hue:
            h = h - hue
        if do_sat:
            s = s * sat
        if wrap:
            out_of_range = (h < dt(-60)) | (h >= dt(360))
            h = np.where(out_of_range, np.fmod(h, dt(360)), h)           # exact: whole turns
            h = np.where(out_of_range & (h < dt(-60)), h + dt(360), h)
        h = h / dt(60)
        i = np.floor(h)
        f = h - i
        p = v * (dt(1) - s)
        q = v * (dt(1) - s * f)
        t = v * (dt(1) - s * (dt(1) - f))
    sec = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v)]
    out = []
    for ch in range(3):
        o = (v, p, q)[ch]                              # default: sector 5 (and every sector outside 0..4)
        for k in range(4, -1, -1):
            o = np.where(i == k, sec[k][ch], o)
        out.append(np.where(s == 0, v, o))
    return np.stack(out).astype(dt)


def hue(img, dt=np.float32):
    """the hue the reference's convert_rgb_to_hsv gives each pixel of img [3, H, W] (unwrapped: in [-60, 360))."""
    r, g, b = (np.asarray(c, dt) for c in img)
    with np.errstate(all="ignore"):
        mn, mx = np.minimum(np.minimum(r, g), b), np.maximum(np.maximum(r, g), b)
        delta = mx - mn
        h = np.where(r == mx, (g - b) / delta, np.where(g == mx, dt(2) + (b - r) / delta, dt(4) + (r - g) / delta)) * dt(60)
    return np.where((mx == 0) | (delta == 0), dt(0), h)


def mean_subtract(img, mean_value=None, mean_image=None, dt=np.float32):
    if mean_image is not None:
        return (img - np.asarray(mean_image, dt)).astype(dt)
    if mean_value is not None:
        mv = list(mean_value) * 3 if len(mean_value) == 1 else list(mean_value)
        f = np.float32
        mv = [f(f(f(m) / f(255)) * f(255)) for m in mv]      # the reference's mean_value / 255.f, then * 255 on the GPU path
        return (img - np.asarray(mv, dt)[:, None, None]).astype(dt)
    return img


# ---- spatial sampling ----------------------------------------------------------------------------------------------------------
def _cubic(d, v1, v2, v3, v4):
    """cubic_interpolation in double, each operation rounded, then rounded to float (the reference's Dtype return)."""
    d, v1, v2, v3, v4 = (np.asarray(a, np.float64) for a in (d, v1, v2, v3, v4))
    with np.errstate(all="ignore"):
        c = ((-1.0 * v1 + 3.0 * v2) + -3.0 * v3) + 1.0 * v4
        b = ((3.0 * v1 + -6.0 * v2) + 3.0 * v3) + 0.0 * v4
        b = b + d * c
        a = ((-2.0 * v1 + -3.0 * v2) + 6.0 * v3) + -1.0 * v4
        a = a + d * b
        return v2 + (d * a) / 6.0


def _get(plane, y, x):
    H, W = plane.shape
    x = np.where(x == -1, 0, np.where(x == W, W - 1, x))
    y = np.where(y == -1, 0, np.where(y == H, H - 1, y))
    ok = (x >= 0) & (x < W) & (y >= 0) & (y < H)
    return np.where(ok, plane[np.clip(y, 0, H - 1), np.clip(x, 0, W - 1)], 0).astype(plane.dtype)


def source_coords(aug, H, W, OH, OW, dt=np.float32):
    """the source coordinates (y, x) each output pixel samples: crop, rotate, scale, flip in the kernel's order and types."""
    oy, ox = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
    x = ox.astype(dt) + dt(aug["crop_x"])
    y = oy.astype(dt) + dt(aug["crop_y"])
    if abs(np.float32(aug["rotation"])) > FLT_EPSILON:
        wb, hb = dt(aug["scale_w"] - 1), dt(aug["scale_h"] - 1)
        if dt is np.float32:
            angle = np.float32(np.float32(aug["rotation"]) * np.float32(math.pi)) / np.float32(180)
        else:
            angle = float(aug["rotation"]) * math.pi / 180
        ca, sa = dt(math.cos(angle)), dt(math.sin(angle))
        wa = abs(wb * ca) + abs(hb * sa)
        ha = abs(wb * sa) + abs(hb * ca)
        cx, cy = wa / dt(2), ha / dt(2)
        s, c = dt(math.sin(-angle)), dt(math.cos(-angle))
        tx, ty = x - cx, y - cy
        x = (tx * c - ty * s) + cx
        y = (tx * s + ty * c) + cy
        x = x - (wa - wb) / dt(2)
        y = y - (ha - hb) / dt(2)
    if W != aug["scale_w"]:
        x = x * (dt(W - 1) / dt(aug["scale_w"] - 1))
    if H != aug["scale_h"]:
        y = y * (dt(H - 1) / dt(aug["scale_h"] - 1))
    if aug["flip"]:
        x = (dt(W) - x).astype(np.float64) - 1.0
    return np.asarray(y, dt), np.asarray(x, dt)


def sample(img, aug, OH, OW, dt=np.float32):
    """img [3, H, W] (after colour and mean) -> [3, OH, OW] by the reference's bicubic at source_coords."""
    _, H, W = img.shape
    y, x = source_coords(aug, H, W, OH, OW, dt)
    fx, cx, fy, cy = np.floor(x), np.ceil(x), np.floor(y), np.ceil(y)
    xs = [(fx - 1).astype(np.int64), fx.astype(np.int64), cx.astype(np.int64), (cx + 1).astype(np.int64)]
    ys = [(fy - 1).astype(np.int64), fy.astype(np.int64), cy.astype(np.int64), (cy + 1).astype(np.int64)]
    dx, dy = (x - fx).astype(dt), (y - fy).astype(dt)
    out = np.empty((3, OH, OW), dt)
    for ch in range(3):
        plane = np.asarray(img[ch], dt)
        rows = [_cubic(dx, *[_get(plane, yy, xx) for xx in xs]).astype(dt) for yy in ys]
        out[ch] = _cubic(dy, *rows).astype(dt)
    return out


def image(bottom, augs, OH, OW, mean_value=None, mean_image=None, wrap=True, dt=np.float32):
    """the image top [N, 3, OH, OW] for bottom [N, 3, H, W] and one aug dict per image."""
    out = []
    for n, a in enumerate(augs):
        im = colour(bottom[n], a["hue_rotation"], a["saturation"], wrap, dt)
        im = mean_subtract(im, mean_value, mean_image, dt)
        out.append(sample(im, a, OH, OW, dt))
    return np.stack(out)


# ---- labels --------------------------------------------------------------------------------------------------------------------
def label_shape(gt):
    g = dict(GT_DEFAULTS, **gt)
    dsts = [d for _, d in g["object_class"]] or [0]
    inv = np.float32(1.0 / g["stride"])
    return 8 + max(dsts) + 1, int(np.rint(np.float32(g["image_size_y"]) * inv)), int(np.rint(np.float32(g["image_size_x"]) * inv))


def _rect_and(a, b, dt):
    x1, y1 = max(a[0], b[0]), max(a[1], b[1])
    w = dt(min(dt(a[0] + a[2]), dt(b[0] + b[2])) - x1)
    h = dt(min(dt(a[1] + a[3]), dt(b[1] + b[3])) - y1)
    if w <= 0 or h <= 0:
        return (dt(0), dt(0), dt(0), dt(0))
    return (x1, y1, w, h)


def rotated_bounding_tl(sw, sh, rotation, center=None):
    """cv::RotatedRect(center, (sw, sh), rotation).boundingRect(): (x, y, width, height) with OpenCV's float corners."""
    th = rotation * math.pi / 180
    bh, ah = np.float32(np.float32(math.cos(th)) * np.float32(0.5)), np.float32(np.float32(math.sin(th)) * np.float32(0.5))
    cx, cy = center if center is not None else (np.float32(sw) * np.float32(0.5), np.float32(sh) * np.float32(0.5))
    cx, cy, sw, sh = np.float32(cx), np.float32(cy), np.float32(sw), np.float32(sh)
    p0 = (cx - ah * sh - bh * sw, cy + bh * sh - ah * sw)
    p1 = (cx + ah * sh - bh * sw, cy - bh * sh - ah * sw)
    p2 = (np.float32(2) * cx - p0[0], np.float32(2) * cy - p0[1])
    p3 = (np.float32(2) * cx - p1[0], np.float32(2) * cy - p1[1])
    xs, ys = (p0[0], p1[0], p2[0], p3[0]), (p0[1], p1[1], p2[1], p3[1])
    x0, y0 = math.floor(min(xs)), math.floor(min(ys))
    return x0, y0, math.ceil(max(xs)) - x0 + 1, math.ceil(max(ys)) - y0 + 1


def transform_boxes(boxes, aug, H, W, gt, dt=np.float32):
    """transform_label_cpu then pruneBboxes: [(x, y, w, h, dst)] of the boxes the coverage map draws, in list order."""
    g = dict(GT_DEFAULTS, **gt)
    cmap = {1: 0} if not g["object_class"] else {}
    for s, d in g["object_class"]:
        cmap[s] = d
    out = []
    for row in boxes:
        x, y, w, h = (dt(v) for v in row[:4])
        if aug["flip"]:
            x = dt(dt(dt(W) - x) - w) - dt(1)
        if aug["scale_w"] != W or aug["scale_h"] != H:
            sx, sy = dt(aug["scale_w"]) / dt(W), dt(aug["scale_h"]) / dt(H)
            x, y, w, h = x * sx, y * sy, w * sx, h * sy
        if abs(np.float32(aug["rotation"])) > FLT_EPSILON:
            th = float(np.float32(aug["rotation"])) * math.pi / 180
            tlx, tly, _, _ = rotated_bounding_tl(aug["scale_w"], aug["scale_h"], float(np.float32(aug["rotation"])))
            ccx, ccy = aug["scale_w"] * 0.5, aug["scale_h"] * 0.5
            cx, cy = 0.5 * (float(x) + (float(x) + float(w))), 0.5 * (float(y) + (float(y) + float(h)))
            nx = ((math.cos(th) * (cx - ccx) - math.sin(th) * (cy - ccy)) + ccx) - tlx
            ny = ((math.sin(th) * (cx - ccx) + math.cos(th) * (cy - ccy)) + ccy) - tly
            x, y = dt(nx - 0.5 * float(w)), dt(ny - 0.5 * float(h))
        x, y = x - dt(aug["crop_x"]), y - dt(aug["crop_y"])
        if g["crop_bboxes"]:
            x, y, w, h = _rect_and((x, y, w, h), (dt(0), dt(0), dt(g["image_size_x"]), dt(g["image_size_y"])), dt)
        cls = float(np.float32(row[5]))
        if not (0 <= cls < 2 ** 32) or int(cls) not in cmap:
            continue
        if dt(w * h) < FLT_EPSILON:
            continue
        out.append((x, y, w, h, cmap[int(cls)]))
    return out


def coverage(pruned, gt, dt=np.float32):
    """CoverageGenerator::generate over already pruned boxes: [C, GH, GW]."""
    g = dict(GT_DEFAULTS, **gt)
    C, GH, GW = label_shape(gt)
    out = np.zeros((C, GH, GW), dt)
    stride, box_area = dt(g["stride"]), dt(g["stride"] * g["stride"])
    min_norm = dt(0) if g["obj_norm"] else dt(1)
    for (x, y, w, h, dst) in pruned:
        ctrx, ctry = dt(x + dt(x + w)) * dt(0.5), dt(y + dt(y + h)) * dt(0.5)
        shw, shh = w * dt(g["scale_cvg"]), h * dt(g["scale_cvg"])
        if g["gridbox_type"] in ("GRIDBOX_MIN", 1):
            shw, shh = min(w, max(dt(g["min_cvg_len"]), shw)), min(h, max(dt(g["min_cvg_len"]), shh))
        else:
            shw, shh = min(dt(g["max_cvg_len"]), shw), min(dt(g["max_cvg_len"]), shh)
        hw, hh = shw * dt(0.5), shh * dt(0.5)
        ax, ay, bx, by = ctrx + hw, ctry + hh, ctrx - hw, ctry - hh
        cov = (min(ax, bx), min(ay, by), dt(max(ax, bx) - min(ax, bx)), dt(max(ay, by) - min(ay, by)))
        norm = dt(box_area / dt(cov[2] * cov[3]))
        gx0, gy0 = max(math.floor(cov[0] / stride), 0), max(math.floor(cov[1] / stride), 0)
        gx1, gy1 = min(math.ceil(dt(cov[0] + cov[2]) / stride), GW), min(math.ceil(dt(cov[1] + cov[3]) / stride), GH)
        for gy in range(gy0, gy1):
            for gx in range(gx0, gx1):
                gbx, gby = dt(gx) * stride, dt(gy) * stride
                ix, iy, iw, ih = _rect_and(cov, (gbx, gby, stride, stride), dt)
                if dt(dt(iw * ih) / box_area) > FLT_EPSILON:
                    out[:, gy, gx] = 0
                    out[8 + dst, gy, gx] = 1
                    out[0, gy, gx] = 1
                    out[1, gy, gx] = x - gbx
                    out[2, gy, gx] = y - gby
                    out[3, gy, gx] = dt(x + w) - gbx
                    out[4, gy, gx] = dt(y + h) - gby
                    out[5, gy, gx] = dt(1.0 / float(w))
                    out[6, gy, gx] = dt(1.0 / float(h))
                    out[7, gy, gx] = max(min_norm, norm)
    return out


def labels(label_blob, augs, H, W, gt, dt=np.float32):
    """the label top [N, C, GH, GW] for a DIGITS label blob [N, 1, rows, 16] (headers assumed valid)."""
    out = []
    for n, a in enumerate(augs):
        blk = np.asarray(label_blob[n, 0], np.float32)
        nb = int(blk[0, 0])
        out.append(coverage(transform_boxes(blk[1:1 + nb], a, H, W, gt, dt), gt, dt))
    return np.stack(out)


def label_blob(box_lists, rows):
    """DIGITS layout: [N, 1, rows, 16], row 0 [num_boxes, 16, 0...], then one box per row (x, y, w, h, alpha, class, ...)."""
    out = np.zeros((len(box_lists), 1, rows, 16), np.float32)
    for n, bl in enumerate(box_lists):
        out[n, 0, 0, 0], out[n, 0, 0, 1] = len(bl), 16
        for k, b in enumerate(bl):
            out[n, 0, 1 + k, :len(b)] = b
    return out


# ---- selection draw ------------------------------------------------------------------------------------------------------------
def draw(rand, W, H, aug_param=None, image_size_x=1248, image_size_y=384, train=True):
    """get_augmentations (detectnet_transform_layer.cpp:345-411) with `rand()` giving the reference's randDouble (a float in
    [0, 1]); the conditional draw order is the reference's.  Returns an aug dict."""
    p = dict(AUG_DEFAULTS, **(aug_param or {}))
    f = np.float32
    a = identity_aug(W, H)
    if not train:
        a["scale_w"], a["scale_h"] = image_size_x, image_size_y
        return a
    if f(rand()) <= f(p["hue_rotation_prob"]):
        hue = float(np.float32((float(f(rand())) - 0.5) * 2 * float(f(p["hue_rotation"]))))
        a["hue_rotation"] = max(min(hue, 180.0), -180.0)
    if f(rand()) <= f(p["desaturation_prob"]):
        a["saturation"] = float(np.float32(1.0 - float(f(f(rand()) * f(p["desaturation_max"])))))
    a["flip"] = int(f(rand()) <= f(p["flip_prob"]))
    if f(rand()) <= f(p["scale_prob"]):
        s = f(f(p["scale_min"]) + f(f(f(p["scale_max"]) - f(p["scale_min"])) * f(rand())))
        a["scale_w"], a["scale_h"] = int(_round(float(f(f(W) * s)))), int(_round(float(f(f(H) * s))))
    if f(rand()) <= f(p["rotation_prob"]):
        a["rotation"] = float(np.float32((float(f(rand())) - 0.5) * 2 * float(f(p["max_rotate_degree"]))))
    bw, bh = a["scale_w"], a["scale_h"]
    if abs(np.float32(a["rotation"])) > FLT_EPSILON:
        center = (float(int(0.5 * bw)), float(int(0.5 * bh)))                # cv::Point(0.5 w, 0.5 h) truncates to int
        _, _, bw, bh = rotated_bounding_tl(bw, bh, a["rotation"], center)
    if f(rand()) <= f(p["crop_prob"]):
        px, py = float(f(rand())), float(f(rand()))
        sx, sy = int(p["shift_x"]), int(p["shift_y"])
    else:
        px = py = 0.5
        sx = sy = 0
    a["crop_x"] = int(_round(px * (bw - image_size_x + sx) - sx // 2))
    a["crop_y"] = int(_round(py * (bh - image_size_y + sy) - sy // 2))
    return a


def _round(v):
    """C's round: half away from zero."""
    return math.floor(v + 0.5) if v >= 0 else -math.floor(-v + 0.5)
