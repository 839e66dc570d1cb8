"""Per-element tests of the BatchNorm training kernels (csrc/layers.cu, csrc/layers_fused.cu) against a float64 oracle, on every
launch regime bn_plan picks (include/b2c.h, b2c_debug_bn_plan).

test_layers_gpu.py compares the unfused kernels with the oracle by blob-level rel_err and the fused kernels bit for bit with the
unfused chain; both sides of that comparison share bn_common.cuh, so a slip there passes both.  Here every element is judged on its
own, against the oracle:

* integer data ("int"): x = an integer channel centre + integers of zero sum, integer dy.  Every fp32 partial sum of the
  statistics is then exact, so the mean, the inverse std, the first running mean / variance and dbeta must equal, bit for bit, the
  kernel's own formula evaluated in numpy (IEEE 1.0f / sqrtf: the build has no fast-math); channel 0 takes the second pass.  A unit dropped, counted twice or read
  from the wrong place at a slice or plane boundary fails on its own, not inside a tolerance.
* random data ("normal"): the statistics within worst-case bounds of the summation (gamma_k = k u / (1 - k u) with k the terms a
  thread adds in sequence plus the block and cluster tree); y, x_norm, dx per element within c * 2^-24 * sum|terms| of the
  expression, evaluated from the kernel's own saved statistics and dgamma / dbeta; the second iteration's running averages within
  3 ulp of their operands.

Every input and output lives in a Guarded buffer (NaN-prefilled outputs, sentinel guard bands; dgamma / dbeta start at 9 to show
they are overwritten).  Each call runs twice and must give the same bits.  Before a call, the case's plan at 132 SMs is asserted
through b2c_debug_bn_plan with the call's real pointers; cases marked sm_dep get their cluster size from the SM count (C * cs < SMs)
and are only pinned on a 132-SM part.  Under a B2C_BN_* switch (test_experimental_gpu.py runs this file once per switch) the
expected plan is the switch's documented effect on the table.

test_variance_does_not_depend_on_the_first_value: the variance of a channel whose first value lies 100 sigma from its mean, and of
a channel with mean 50, sigma 1 and first value 0, within the two-pass bound 8 * 2^-24 * log2(N S) * var."""
import math
import os
import zlib

import numpy as np
import pytest

from cases import Guarded

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import caffe_mpi_b200 as m  # noqa: E402
from caffe_mpi_b200 import capi  # noqa: E402

U = 2.0 ** -24
FLT_MIN = float(np.finfo(np.float32).tiny)
EPS, MAF = 1e-5, 0.9
MAF32 = float(np.float32(MAF))
SWITCHES = ["B2C_BN_ONEPASS=0", "B2C_BN_PREFETCH=0", "B2C_BN_PREFETCH_BWD=0", "B2C_BN_CACHE_KB=0", "B2C_BN_CLUSTER=16"]

# (id, N, C, H, W, float offset of every pointer, plan at 132 SMs and default switches:
#  (cs, forward threads, backward threads, forward park, backward park fused, backward park fused_res, float4), sm_dep, variants)
ALL = ("unf_inplace", "unf_noaffine", "fused_relu0", "fused_relu1_noaffine", "res_dres", "res_dy2_noaffine")
CASES = [
    ("bn_conv1_112_park0", 64, 64, 112, 112, 0, (8, 512, 512, 0, 0, 0, True), False, ("fused_relu1_noaffine", "res_dres")),
    ("res2_56_park1_2", 64, 64, 56, 56, 0, (8, 512, 512, 1, 1, 2, True), False, ("unf_inplace", "fused_relu1_noaffine", "res_dy2_noaffine")),
    ("res3_28_cs2", 64, 128, 28, 28, 0, (2, 512, 512, 1, 1, 2, True), False, ALL),
    ("res4_14_256thr_park3", 64, 256, 14, 14, 0, (1, 256, 512, 1, 3, 3, True), False, ALL),
    ("res4_14_off4_scalar", 64, 256, 14, 14, 1, (1, 256, 512, 1, 3, 3, False), False, ("unf_noaffine", "fused_relu1_noaffine", "res_dres")),
    ("res5_7_128thr_scalar", 64, 2048, 7, 7, 0, (1, 128, 128, 1, 3, 3, False), False, ALL),
    ("scalar_s1225_cs4", 64, 40, 35, 35, 0, (4, 512, 512, 1, 1, 2, False), False, ALL),
    ("midplane_37x30x30_cs2", 37, 70, 30, 30, 0, (2, 512, 512, 1, 1, 2, True), False, ALL),
    ("s5_empty_ranks", 1, 3, 1, 5, 0, (8, 128, 128, 1, 3, 3, False), True, ALL),
    ("s1_empty_ranks", 3, 5, 1, 1, 0, (8, 128, 128, 1, 3, 3, False), True, ALL),
    ("s6_midplane", 5, 7, 2, 3, 0, (8, 128, 128, 1, 3, 3, False), True, ALL),
    ("s7_midplane", 4, 9, 1, 7, 0, (8, 128, 128, 1, 3, 3, False), True, ALL),
    ("s4096_cs8", 8, 16, 64, 64, 0, (8, 512, 512, 1, 3, 3, True), True, ALL),
]
VARIANTS = {   # form, relu, affine, in place, d_sum2, d_residual
    "unf_inplace": ("unfused", 0, True, True, False, False),
    "unf_noaffine": ("unfused", 0, False, False, False, False),
    "fused_relu0": ("fused", 0, True, False, False, False),
    "fused_relu1_noaffine": ("fused", 1, False, False, False, False),
    "res_dres": ("fused_res", 1, True, False, False, True),
    "res_dy2_noaffine": ("fused_res", 1, False, False, True, False),
}


def switch():
    on = [s for s in SWITCHES if os.environ.get(s.split("=")[0]) == s.split("=")[1]]
    assert len(on) <= 1, f"one B2C_BN_* switch at a time: {on}"
    return on[0] if on else None


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def expected_plan(case, d, form):
    """the case's plan for direction d and form, under the B2C_BN_* switch in effect; None for what the switch leaves unpinned"""
    _, N, Cc, H, W, off, (cs, tf, tb, pf, pb, pr, vec), sm_dep, _ = case
    launches = 2 if form == "unfused" else 1
    park = 0 if form == "unfused" else (pf if d == 0 else pb if form == "fused" else pr)
    sw = switch()
    if sw == "B2C_BN_ONEPASS=0" and form == "fused":
        launches, park = 2, 0
    if sw == "B2C_BN_CACHE_KB=0":
        park = 0
    prefetch = int(park > 0 and not (sw == "B2C_BN_PREFETCH=0" and d == 0) and not (sw == "B2C_BN_PREFETCH_BWD=0" and d == 1))
    want = dict(launches=launches, cs=cs, threads=tf if d == 0 else tb, park=park, prefetch=prefetch, vec=vec)
    if (sm_dep and sm_count() != 132) or sw == "B2C_BN_CLUSTER=16":
        want.update(cs=None, park=None, prefetch=None)    # the cluster size, hence the slice, depends on the part
    return want


def check_plan(case, d, form, bufs):
    got = capi.bn_plan(d, form, case[1], case[2], case[3] * case[4], [b.ptr().value if b is not None else 0 for b in bufs])
    want = expected_plan(case, d, form)
    for k, v in want.items():
        assert v is None or got[k] == v, f"{case[0]} {form} {'forward' if d == 0 else 'backward'}: plan {got}, the case exists for {want}"
    return got


def st():
    return capi._stream()


def P(b):
    return b.ptr() if b is not None else None


def bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def gam(k):
    return k * U / (1 - k * U)


def within(got, ref, bound, what):
    got64 = got.astype(np.float64)
    assert not np.isnan(got64).any(), f"{what}: NaN (an element never written)"
    err = np.abs(got64 - ref)
    bad = np.argwhere(err > bound)
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: got {got64[tuple(bad[0])]!r}, "
                           f"want {np.broadcast_to(ref, err.shape)[tuple(bad[0])]!r}, bound {np.broadcast_to(bound, err.shape)[tuple(bad[0])]!r}")


def equal(got, ref, what):
    assert not np.isnan(got.astype(np.float64)).any(), f"{what}: NaN (an element never written)"
    bad = np.argwhere(got != ref)
    assert bad.size == 0, f"{what}: {len(bad)} elements differ, first at {tuple(bad[0])}: got {got[tuple(bad[0])]!r}, want {ref[tuple(bad[0])]!r}"


def int_channels(rng, N, Cc, S):
    """x[n, c, s] = centre[c] + v with v integers of zero sum over the channel: the mean is exactly centre[c].  v lies in [-2, 2],
    so pass 1's sums of x - k and (x - k)^2 stay exact up to 2^20 values a channel.  Channel 0 (with 64 values or more) starts with
    v = 12, balanced by a few -2: its first value, pass 1's shift, lies ~8 sigma out, which takes the statistics through pass 2."""
    cnt = N * S
    centre = rng.integers(-2, 3, Cc).astype(np.float64)
    centre[Cc // 2] = 40.0                                  # one channel far from zero: k is then ~40, x - k still small
    v = np.empty((Cc, cnt))
    for c in range(Cc):
        r = rng.integers(-2, 3, cnt // 2)
        v[c] = rng.permutation(np.concatenate([r, -r, np.zeros(cnt % 2, np.int64)]))
    if cnt >= 64:
        d = 12 - v[0, 0]
        v[0, 0] = 12
        z = np.flatnonzero(v[0, 1:] == 0)[:int(d + 1) // 2] + 1
        assert len(z) == int(d + 1) // 2
        v[0, z] = -2
        if d % 2:
            v[0, z[-1]] = -1
    assert (v.sum(axis=1) == 0).all()
    x = (centre[:, None] + v).reshape(Cc, N, S).transpose(1, 0, 2)
    return np.ascontiguousarray(x, np.float32), centre


def terms(cnt, cs, threads):
    """terms a fp32 partial of one channel goes through: a thread's sequential sum, the block tree, the cluster's rank order"""
    return math.ceil(cnt / (cs * threads)) + int(math.log2(threads)) + cs + 2


def forward(case, form, relu, affine, inplace, x, g, b, res, first_calls=(1, 0)):
    """the forward entry point of `form`, twice (first_iteration 1 then 0, same bits); returns what it wrote"""
    _, N, Cc, H, W, off = case[:6]
    S = H * W
    L = m.lib()
    X = Guarded(x.size, off, x)
    Y = X if inplace else Guarded(x.size, off)
    XN = Guarded(x.size, off) if form == "unfused" else None
    R = Guarded(x.size, off, res) if form == "fused_res" else None
    G, B = (Guarded(Cc, 0, g), Guarded(Cc, 0, b)) if affine else (None, None)
    RM, RV, SM, SI = (Guarded(Cc) for _ in range(4))
    check_plan(case, 0, form, [X, Y, XN if form == "unfused" else R])
    outs = []
    for first in first_calls:
        if inplace and outs:
            X = Y = Guarded(x.size, off, x)
        if form == "unfused":
            rc = L.b2c_bn_forward_train(N, Cc, S, X.ptr(), P(G), P(B), EPS, MAF, first, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), XN.ptr(), Y.ptr(), st())
        elif form == "fused":
            rc = L.b2c_bn_forward_train_fused(N, Cc, S, X.ptr(), P(G), P(B), EPS, MAF, first, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), Y.ptr(), relu, st())
        else:
            rc = L.b2c_bn_forward_train_fused_res(N, Cc, S, X.ptr(), P(G), P(B), EPS, MAF, first, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), R.ptr(), Y.ptr(),
                                                  relu, st())
        capi.check(rc)
        outs.append(dict(y=Y.read().reshape(x.shape), xn=XN.read().reshape(x.shape) if XN else None, mean=SM.read().copy(),
                         invstd=SI.read().copy(), rm=RM.read().copy(), rv=RV.read().copy()))
        if not inplace:
            assert np.array_equal(X.read().reshape(x.shape), x), "forward: x changed"
    a, b2 = outs[0], outs[-1]
    for k in ("y", "xn", "mean", "invstd"):
        if a[k] is not None:
            assert np.array_equal(bits(a[k]), bits(b2[k])), f"forward {k}: not bit-identical call to call"
    return outs


def backward(case, form, relu, affine, inplace, x, xn, y, g, b, mean, invstd, dy, dy2, dres):
    """the backward entry point of `form`, twice (same bits); returns dgamma, dbeta, dx, d_residual"""
    _, N, Cc, H, W, off = case[:6]
    S = H * W
    L = m.lib()
    outs = []
    for _ in range(2):
        X = Guarded(x.size, off, x)
        DY = Guarded(x.size, off, dy)
        DX = DY if inplace else Guarded(x.size, off)
        XN = Guarded(x.size, off, xn) if form == "unfused" else None
        YS = Guarded(x.size, off, y) if form == "fused_res" else None
        DY2 = Guarded(x.size, off, dy2) if dy2 is not None else None
        DR = Guarded(x.size, off) if dres else None
        G, B = (Guarded(Cc, 0, g), Guarded(Cc, 0, b)) if affine else (None, None)
        SM, SI = Guarded(Cc, 0, mean), Guarded(Cc, 0, invstd)
        DG, DB = Guarded(Cc, 0, np.full(Cc, 9, np.float32)), Guarded(Cc, 0, np.full(Cc, 9, np.float32))
        if not outs:
            check_plan(case, 1, form, [DY, XN, DX] if form == "unfused" else [DY, DY2, X, DX, YS, DR])
        if form == "unfused":
            rc = L.b2c_bn_backward(N, Cc, S, DY.ptr(), XN.ptr(), P(G), SI.ptr(), DG.ptr(), DB.ptr(), DX.ptr(), st())
        elif form == "fused":
            rc = L.b2c_bn_backward_fused(N, Cc, S, DY.ptr(), X.ptr(), SM.ptr(), SI.ptr(), P(G), P(B), DG.ptr(), DB.ptr(), DX.ptr(), relu, st())
        else:
            rc = L.b2c_bn_backward_fused_res(N, Cc, S, DY.ptr(), P(DY2), YS.ptr(), X.ptr(), SM.ptr(), SI.ptr(), P(G), P(B), DG.ptr(), DB.ptr(),
                                             DX.ptr(), P(DR), st())
        capi.check(rc)
        outs.append((DG.read().copy(), DB.read().copy(), DX.read().reshape(x.shape), DR.read().reshape(x.shape) if DR else None))
    for k, a, c in zip(("dgamma", "dbeta", "dx", "d_residual"), outs[0], outs[1]):
        if a is not None:
            assert np.array_equal(bits(a), bits(c)), f"backward {k}: not bit-identical call to call"
    return outs[0]


def check_statistics(case, data, x, centre, o1, o2, cs, threads):
    """saved mean / invstd and the running averages of the first (copy) and second (average) iteration"""
    N, Cc, S = x.shape[0], x.shape[1], x.shape[2]
    cnt = N * S
    mean, invstd = o1["mean"], o1["invstd"]
    if data == "int":
        xc = x.astype(np.float64).transpose(1, 0, 2).reshape(Cc, cnt)
        v, d = xc - centre[:, None], xc - xc[:, :1]
        assert (v.sum(axis=1) == 0).all()
        # the kernel's two formulas, on exact sums (integers < 2^24): pass 1 about k, pass 2 about pass 1's (exact) mean
        m1 = d.sum(axis=1) / cnt
        one = np.maximum((d * d).sum(axis=1) / cnt - m1 * m1, 0.0).astype(np.float32) + np.float32(EPS)
        two = np.maximum((v * v).sum(axis=1) / cnt, 0.0).astype(np.float32) + np.float32(EPS)
        var_eps = np.where(o1["rv"] == one, one, two)
        if cnt >= 64:
            var_eps[0] = two[0]                            # channel 0's shift lies ~8 sigma out: pass 2 must have run
        equal(mean, centre.astype(np.float32), "mean")
        equal(o1["rv"], var_eps, "running variance (first iteration)")
        equal(invstd, np.float32(1) / np.sqrt(var_eps), "invstd")
        equal(o1["rm"], centre.astype(np.float32), "running mean (first iteration)")
    else:
        k = terms(cnt, cs, threads)
        xc = x.astype(np.float64).transpose(1, 0, 2).reshape(Cc, cnt)
        mu = xc.mean(axis=1)
        var = ((xc - mu[:, None]) ** 2).mean(axis=1)
        d = xc - xc[:, :1]                                 # pass 1 sums about k = the channel's first value
        e0 = gam(k) * np.abs(d).mean(axis=1) + U * np.abs(mu)                          # pass 1's mean
        dev = np.abs(xc - mu[:, None]).mean(axis=1)
        # pass 2 (about pass 1's mean) runs when k lies more than 4 sigma out; nearer, pass 1's sums stand, within 17x its bound
        one = (mu - xc[:, 0]) ** 2 <= 17 * var
        bm = np.maximum(gam(k) * (dev + e0) + U * np.abs(mu), np.where(one, e0, 0)) + FLT_MIN
        within(mean, mu, bm, "mean")
        bv_two = gam(k + 2) * (var + e0 ** 2) + 2 * U * (var + EPS) + (gam(k) * (dev + e0)) ** 2
        bv_one = gam(k + 2) * (d * d).mean(axis=1) + 2 * np.abs(d.mean(axis=1)) * e0 + e0 ** 2 + 2 * U * (var + EPS)
        bv = np.where(one, np.maximum(bv_one, bv_two), bv_two)
        within(o1["rv"], var + EPS, bv, "running variance (first iteration) = var + eps")
        is64 = 1 / np.sqrt(var + EPS)
        within(invstd, is64, is64 * (2.5 * U + 0.5 * bv / (var + EPS)) * 1.01, "invstd")
        equal(o1["rm"], mean, "running mean (first iteration)")
    # second iteration: run = (1 - maf) * batch + maf * run, one rounding per operation (an FMA may fuse two)
    a = float(np.float32(1) - np.float32(MAF))
    for nm, batch in (("rm", o2["mean"]), ("rv", o1["rv"])):
        ref = a * batch.astype(np.float64) + MAF32 * o1[nm].astype(np.float64)
        within(o2[nm], ref, 3 * U * (np.abs(a * batch) + np.abs(MAF32 * o1[nm])) + FLT_MIN, f"running {nm} (second iteration)")


def run_case(case, variant, data, rng):
    cid, N, Cc, H, W, off, plan, sm_dep, _ = case
    form, relu, affine, inplace, two, dres = VARIANTS[variant]
    S = H * W
    shape = (N, Cc, S)
    if data == "int":
        x, centre = int_channels(rng, N, Cc, S)
        dy = rng.integers(-3, 4, shape).astype(np.float32)
        dy2 = rng.integers(-3, 4, shape).astype(np.float32) if two else None
        res = rng.integers(-3, 4, shape).astype(np.float32)
    else:
        centre = None
        x = (rng.standard_normal(shape) * 1.5 + 0.3).astype(np.float32)
        dy = rng.standard_normal(shape).astype(np.float32)
        dy2 = rng.standard_normal(shape).astype(np.float32) if two else None
        res = rng.standard_normal(shape).astype(np.float32)
    g = rng.standard_normal(Cc).astype(np.float32) if affine else None
    b = rng.standard_normal(Cc).astype(np.float32) if affine else None

    o1, o2 = forward(case, form, relu if form != "unfused" else 0, affine, inplace, x, g, b, res)
    fp = capi.bn_plan(0, form, N, Cc, S, ())
    check_statistics(case, data, x, centre, o1, o2, fp["cs"], fp["threads"])

    # elementwise forward from the kernel's own statistics: xn = (x - m) * is (2 roundings), y = fma(xn, g, b) [+ res] [ReLU]
    mean, invstd = o1["mean"][None, :, None].astype(np.float64), o1["invstd"][None, :, None].astype(np.float64)
    xn64 = (x - mean) * invstd
    g64 = g[None, :, None].astype(np.float64) if affine else 1.0
    b64 = b[None, :, None].astype(np.float64) if affine else 0.0
    pre = xn64 * g64 + b64
    bound = 3 * U * (np.abs(xn64 * g64) + np.abs(b64)) + FLT_MIN
    if form == "fused_res":
        pre = pre + res
        bound = bound + U * (np.abs(pre) + np.abs(res))
    y_ref = np.maximum(pre, 0) if (form != "unfused" and relu) else pre
    within(o1["y"], y_ref, bound, "y")
    if form == "unfused":
        within(o1["xn"], xn64, 2 * U * np.abs(xn64) + FLT_MIN, "x_norm")

    # backward: the upstream gradient the kernel sees, masked by the forward's output where a ReLU follows
    d = dy if dy2 is None else (dy + dy2).astype(np.float32)
    if form == "fused_res" or (form == "fused" and relu):
        d = np.where(o1["y"] > 0, d, np.float32(0)).astype(np.float32)
    dg, db, dx, dr = backward(case, form, relu, affine, inplace, x, o1["xn"], o1["y"], g, b, o1["mean"], o1["invstd"], dy, dy2, dres)
    bp = capi.bn_plan(1, form, N, Cc, S, ())
    k = terms(N * S, bp["cs"], bp["threads"])
    xn_used = o1["xn"].astype(np.float64) if form == "unfused" else xn64
    d64 = d.astype(np.float64)
    dg64 = (d64 * xn_used).sum(axis=(0, 2))
    db64 = d64.sum(axis=(0, 2))
    if data == "int":
        equal(db, db64.astype(np.float32), "dbeta (exact: integer gradients)")
    else:
        within(db, db64, gam(k) * np.abs(d64).sum(axis=(0, 2)) + FLT_MIN, "dbeta")
    within(dg, dg64, (gam(k + 1) + 2 * U) * np.abs(d64 * xn_used).sum(axis=(0, 2)) + FLT_MIN, "dgamma")
    cnt = N * S
    gi = (g64 if affine else 1.0) * invstd
    mdy, mdx = db.astype(np.float64)[None, :, None] / cnt, dg.astype(np.float64)[None, :, None] / cnt
    dx_ref = gi * (d64 - mdy - xn_used * mdx)
    within(dx, dx_ref, 6 * U * np.abs(gi) * (np.abs(d64) + np.abs(mdy) + np.abs(xn_used * mdx)) + FLT_MIN, "dx")
    if dres:
        equal(dr, d, "d_residual (the masked gradient)")


# every variant of a case on integer data and on random data, except that the two largest shapes (2^25 values and more) run their
# first variant only on random data
RUNS = [(c, v, d) for c in CASES for v in c[8] for d in ("int", "normal")
        if not (d == "normal" and v != c[8][0] and c[1] * c[2] * c[3] * c[4] >= (1 << 25))]


@pytest.mark.parametrize("case,variant,data", RUNS, ids=[f"{c[0]}-{v}-{d}" for c, v, d in RUNS])
def test_bn_case(case, variant, data):
    run_case(case, variant, data, np.random.default_rng(zlib.crc32(f"{case[0]} {variant} {data}".encode())))


@pytest.mark.parametrize("shape", [(64, 64, 56, 56), (64, 64, 112, 112)], ids=["res2_56_parked", "bn_conv1_112_park0"])
@pytest.mark.parametrize("form", ["unfused", "fused", "fused_res"])
def test_variance_does_not_depend_on_the_first_value(shape, form):
    """channel 0: N(0, 1) with its first value (image 0's top-left pixel, pass 1's shift) at 100; channel 1: mean 50, sigma 1, first
    value 0.  The variance must meet the reference's two-pass level: |var - var64| <= 8 * 2^-24 * log2(N S) * var64"""
    N, Cc, H, W = shape
    S = H * W
    rng = np.random.default_rng(7)
    x = rng.standard_normal((N, Cc, S)).astype(np.float32)
    x[:, 1] += 50
    x[0, 0, 0], x[0, 1, 0] = 100, 0
    L = m.lib()
    X, Y = Guarded(x.size, 0, x), Guarded(x.size)
    XN = Guarded(x.size)
    RM, RV, SM, SI = (Guarded(Cc) for _ in range(4))
    if form == "unfused":
        rc = L.b2c_bn_forward_train(N, Cc, S, X.ptr(), None, None, EPS, MAF, 1, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), XN.ptr(), Y.ptr(), st())
    elif form == "fused":
        rc = L.b2c_bn_forward_train_fused(N, Cc, S, X.ptr(), None, None, EPS, MAF, 1, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), Y.ptr(), 0, st())
    else:
        R = Guarded(x.size, 0, np.zeros_like(x))
        rc = L.b2c_bn_forward_train_fused_res(N, Cc, S, X.ptr(), None, None, EPS, MAF, 1, RM.ptr(), RV.ptr(), SM.ptr(), SI.ptr(), R.ptr(),
                                              Y.ptr(), 0, st())
    capi.check(rc)
    xc = x[:, :2].astype(np.float64).transpose(1, 0, 2).reshape(2, -1)
    var = xc.var(axis=1)
    got = RV.read()[:2].astype(np.float64) - EPS
    rel = np.abs(got - var) / var
    print(f"{form} {shape}: relative variance error {rel[0]:.2e} (first value 100 sigma out), {rel[1]:.2e} (mean 50, first value 0)")
    bound = 8 * U * math.log2(N * S) + 2 * U * (1 + EPS / var)
    assert (rel <= bound).all(), f"relative variance error {rel} beyond the two-pass bound {bound}"
