"""Generate the convolution fixtures from oracle/_ref, i.e. from the reference's own src/caffe/util/im2col.cpp compiled
verbatim, driven through the per-image / per-group ConvolutionLayer CPU loop with OpenBLAS cblas_sgemm/sgemv (the
reference's BLAS := open):

  conv_ref_golden.npz        small cases, every blob in full
  im2col_ref_sha256.json     SHA-256 of the reference's im2col / col2im (2-D and N-D) outputs on test_oracle.py's
                             IM2COL_SHAPES, inputs from the test's own seed (the test asserts bit-exact equality)
  full_size_ref_golden.npz   the FULL_SIZE_CASES of tests/cases.py (the benchmark's layer shapes and batch sizes): inputs
                             from the test's own seed, outputs stored as a fixed sample of elements per blob (cases.sample_index) (with
                             max|blob|, the denominator of rel_err), bias gradients in full

Needs oracle/_ref, which build() makes only where the reference tree is present:   python tests/golden/make_golden.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle as o  # noqa: E402
from cases import FULL_SIZE_CASES, make, sample_index  # noqa: E402

CASES = [
    ("simple", dict(N=2, Cin=3, H=6, W=4, O=4, k=3, s=2, p=0, d=1, G=1, bias=True)),
    ("group3", dict(N=2, Cin=6, H=6, W=4, O=3, k=3, s=2, p=0, d=1, G=3, bias=True)),
    ("dilated", dict(N=2, Cin=3, H=11, W=9, O=4, k=3, s=1, p=0, d=2, G=1, bias=True)),
    ("one_by_one", dict(N=2, Cin=8, H=6, W=4, O=4, k=1, s=1, p=0, d=1, G=1, bias=True)),
    ("rect", dict(N=2, Cin=4, H=9, W=11, O=5, k=(3, 5), s=(2, 1), p=(1, 2), d=(1, 1), G=1, bias=True)),
    ("res_3x3", dict(N=2, Cin=32, H=14, W=14, O=48, k=3, s=1, p=1, d=1, G=1, bias=False)),
    ("res_1x1_s2", dict(N=2, Cin=32, H=14, W=14, O=24, k=1, s=2, p=0, d=1, G=1, bias=False)),
    ("stem_7x7", dict(N=1, Cin=3, H=30, W=30, O=16, k=7, s=2, p=3, d=1, G=1, bias=False)),
    ("alex_g2", dict(N=2, Cin=16, H=13, W=13, O=24, k=5, s=1, p=2, d=1, G=2, bias=True)),
]


def main():
    assert o.ref() is not None and o.ref_blas_open(1), "oracle/_ref or OpenBLAS unavailable"
    rng = np.random.default_rng(1701)
    out = {}
    for name, c in CASES:
        prm = make(o, c)
        x = rng.standard_normal(prm.x_shape()).astype(np.float32)
        w = (rng.standard_normal(prm.w_shape()) * (2.0 / prm.Kd) ** 0.5).astype(np.float32)
        b = (rng.standard_normal(prm.O) * 0.1).astype(np.float32) if prm.has_bias else None
        dy = rng.standard_normal(prm.y_shape()).astype(np.float32)
        y = np.zeros(prm.y_shape(), np.float32)
        dw = np.zeros(prm.w_shape(), np.float32)
        db = np.zeros(prm.O, np.float32)
        dx = np.zeros(prm.x_shape(), np.float32)
        assert o.ref_conv_fwd_bwd(prm, x, w, b, y=y, dy=dy, dw=dw, db=db if prm.has_bias else None, dx=dx) == 0
        col0 = np.empty((prm.C * prm.kh * prm.kw, prm.Ho, prm.Wo), np.float32)
        o.ref().ref_im2col_cpu(np.ascontiguousarray(x[0]), prm.C, prm.H, prm.W, prm.kh, prm.kw, prm.ph, prm.pw,
                               prm.sh, prm.sw, prm.dh, prm.dw, col0)
        keys = [f for f, _ in o.ConvParams._fields_]
        out[name + "/keys"] = np.array(keys)
        out[name + "/vals"] = np.array([getattr(prm, k) for k in keys], np.int64)
        for k, v in (("x", x), ("w", w), ("dy", dy), ("y", y), ("dw", dw), ("dx", dx), ("col0", col0)):
            out[name + "/" + k] = v
        if prm.has_bias:
            out[name + "/b"] = b
            out[name + "/db"] = db
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "conv_ref_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


def full_size():
    assert o.ref() is not None and o.ref_blas_open(os.cpu_count() or 1), "oracle/_ref or OpenBLAS unavailable"
    out = {}
    for name, c in FULL_SIZE_CASES:
        rng = np.random.default_rng(1701)              # the tests' rng fixture; the draws below are test_full_size_vs_reference_loop's
        po = make(o, c)
        x = rng.standard_normal(po.x_shape(), dtype=np.float32)
        w = rng.standard_normal(po.w_shape(), dtype=np.float32) * np.float32((2.0 / po.Kd) ** 0.5)
        b = (rng.standard_normal(po.O, dtype=np.float32) * np.float32(0.1)) if po.has_bias else None
        dy = rng.standard_normal(po.y_shape(), dtype=np.float32)
        dw0 = rng.standard_normal(po.w_shape(), dtype=np.float32) * np.float32(0.1)
        y = np.empty(po.y_shape(), np.float32)
        dw = dw0.copy()
        db = np.zeros(po.O, np.float32) if po.has_bias else None
        dx = np.empty(po.x_shape(), np.float32)
        assert o.ref_conv_fwd_bwd(po, x, w, b, y=y, dy=dy, dw=dw, db=db, dx=dx) == 0
        for k, v in (("y", y), ("dx", dx), ("dw", dw)):
            v = v.reshape(-1)
            out[f"{name}/{k}"] = v[sample_index(name, k, v.size)]
            out[f"{name}/{k}_absmax"] = np.array(np.abs(v).max(), np.float32)
        if db is not None:
            out[name + "/db"] = db
        print(name, flush=True)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "full_size_ref_golden.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


def im2col_digests():
    import hashlib
    import json
    from test_oracle import IM2COL_SHAPES
    R = o.ref()
    assert R is not None, "oracle/_ref unavailable"
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    out = {}
    for shape in IM2COL_SHAPES:
        Cc, H, W, k, st, p, d = shape
        rng = np.random.default_rng(1701)          # the tests' rng fixture; the draws below are the test's
        im = rng.standard_normal((Cc, H, W)).astype(np.float32)
        col = np.empty_like(o.im2col(im, k, st, p, d))
        R.ref_im2col_cpu(im, Cc, H, W, k[0], k[1], p[0], p[1], st[0], st[1], d[0], d[1], col)
        colr = rng.standard_normal(col.shape).astype(np.float32)
        back = np.empty((Cc, H, W), np.float32)
        R.ref_col2im_cpu(colr, Cc, H, W, k[0], k[1], p[0], p[1], st[0], st[1], d[0], d[1], back)
        ims, cols = np.asarray(im.shape, np.int32), np.asarray(col.shape, np.int32)
        nd = [np.asarray(v, np.int32) for v in (k, p, st, d)]
        coln = np.empty_like(col)
        R.ref_im2col_nd_cpu(im, 2, ims, cols, *nd, coln)
        backn = np.empty_like(back)
        R.ref_col2im_nd_cpu(colr, 2, ims, cols, *nd, backn)
        out[str(shape)] = {"col": sha(col), "back": sha(back), "col_nd": sha(coln), "back_nd": sha(backn)}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "im2col_ref_sha256.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")
    print("wrote", path)


if __name__ == "__main__":
    main()
    im2col_digests()
    full_size()
