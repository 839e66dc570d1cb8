"""Numerical checks of the tensor-core convolution routes' operand splits, in numpy (no GPU needed).

In the fp32 math mode the tensor-core kernels split each operand a into a hi and a lo part and form every product as
hi*hi' + hi*lo' + lo*hi'.  Two checks hold a result to that, element by element:

  * the exact split-term probe.  probe_operand() draws a = h + l with h in {1, 2} and l = j * 2^-13, j in 1..7.  Under both
    splits hi == h and lo == l exactly (l < 2^-10 <= the TF32 ulp of h, and l < half a bf16 ulp), every three-term product lies
    on the 2^-13 grid, and three_term() keeps the largest expected value below 2^10, so every partial sum the kernel can form is
    exact in fp32 in any order.  The result must EQUAL E = f(hi, hi') + f(hi, lo') + f(lo, hi').  All terms are positive, so a
    dropped or doubled term always moves the sum (by whole multiples of 2^-13); a lo word paired with the wrong element moves it
    by a scattered pattern.  E also differs from the fp32 product summed exactly, so the probe shows the split route ran.
  * the per-element bound.  On normal data scaled by powers of two per image and channel (pow2_scale: Sum|ab| then spans
    decades across the output, and the splits are scale-invariant), every element must satisfy |got - ref| <= elem_bound().

The split restatements cite the tc_common.cuh lines they restate."""
import numpy as np

BF16X3, TF32X3, TF32 = "bf16x3", "3xtf32", "tf32"

# c_split of elem_bound: the relative error of one split product, before accumulation.
#   bf16x3: split_pack_bf16 rounds to 8 significant bits twice: a = hi + lo + r with |lo| <= u |a|, |r| <= u |lo|, u = 2^-8.
#           The missing terms lo*lo' + hi*r' + r*hi' + lo*r' + r*lo' + r*r' total <= u^2 (3 + 4u + u^2) |ab| < 3.02 * 2^-16 |ab|.
#           (test_gemm_schedule_gpu.py's docstring argues the same way from |a - hi| <= 2^-9 |a|, which would give 2^-16; one
#           rounding to 8 significant bits can leave 2^-8 |a|, e.g. a = 1 + 2^-8 - 2^-20.)
#   3xTF32: truncation leaves |a - hi| < 2^-10 |a|, the TF32 read of lo loses < 2^-20 |a|; the three missing terms total
#           < 3 * 2^-20 < 2^-18 |ab|.
#   TF32 math: round-to-nearest to TF32 costs <= 2^-11 per operand, so <= 2^-10 + 2^-22 per product.
C_SPLIT = {BF16X3: 3.02 * 2.0 ** -16, TF32X3: 2.0 ** -18, TF32: 1.001 * 2.0 ** -10}
# accumulator additions per MMA k-step and the k-step width of each split's wgmma (bf16: k16, tf32: k8)
TERMS = {BF16X3: 3, TF32X3: 3, TF32: 1}
KSTEP = {BF16X3: 16, TF32X3: 8, TF32: 8}

GRID = 2.0 ** -13            # the probe's lo unit
BUDGET = 2.0 ** 10           # max E: every partial sum on the 2^-13 grid below it spans at most 23 bits


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _float(u):
    return np.asarray(u, np.uint32).view(np.float32)


def bf16_rn(a):
    """fp32 -> bf16 (round to nearest even), returned as the fp32 value it stands for (NaN and Inf not handled)"""
    u = _bits(a)
    return _float((u + (np.uint32(0x7FFF) + ((u >> 16) & 1))) & np.uint32(0xFFFF0000))


def split_pack_bf16(a):
    """(hi, lo) of tc_common.cuh:219-226 split_pack_bf16: hi = bf16_rn(a), lo = bf16_rn(a - hi), a - hi exact in fp32"""
    a = np.asarray(a, np.float32)
    hi = bf16_rn(a)
    return hi, bf16_rn(a - hi)


def split_tf32(a):
    """(hi, lo) of tc_common.cuh:178-181 split_tf32: hi = a with the 13 low mantissa bits cleared, lo = a - hi (exact), and lo
    as the tensor core reads it (its top 19 bits: the same truncation; the TMA-fed 1x1 kernel's raw hi tile is read that way too,
    conv_tc_wgrad.cu:356-357)"""
    a = np.asarray(a, np.float32)
    hi = _float(_bits(a) & np.uint32(0xFFFFE000))
    lo = (a - hi).astype(np.float32)
    return hi, _float(_bits(lo) & np.uint32(0xFFFFE000))


def to_tf32(a):
    """tc_common.cuh:175-177 to_tf32: round to nearest, ties away, on the integer pipe ((bits + 0x1000) & ~0x1fff)"""
    return _float((_bits(a) + np.uint32(0x1000)) & np.uint32(0xFFFFE000))


def split(kind, a):
    """(hi, lo) the tensor cores multiply for operand a under `kind`; TF32 math has one term (lo = 0)"""
    if kind == BF16X3:
        return split_pack_bf16(a)
    if kind == TF32X3:
        return split_tf32(a)
    if kind == TF32:
        return to_tf32(a), np.zeros_like(np.asarray(a, np.float32))
    raise ValueError(kind)


def probe_operand(rng, shape, hmax=2, jmax=7):
    """a = h + j * 2^-13, h in 1..hmax, j in 1..jmax (all positive).  jmax = 3 keeps to_tf32(a) == h (TF32 math mode)."""
    h = rng.integers(1, hmax + 1, shape)
    j = rng.integers(1, jmax + 1, shape)
    return (h + j * GRID).astype(np.float32)


def thin(a, keep):
    """a with a deterministic fraction 1 - keep of its elements zeroed (a fixed hash of the flat index)"""
    idx = np.arange(a.size, dtype=np.uint64)
    h = (idx * np.uint64(2654435761)) % np.uint64(1 << 32)
    mask = (h.astype(np.float64) / 2.0 ** 32 < keep).reshape(a.shape)
    return np.where(mask, a, np.float32(0)).astype(np.float32)


def three_term(f, a, b, kind, budget=BUDGET):
    """E = f(hi_a, hi_b) + f(hi_a, lo_b) + f(lo_a, hi_b) in float64, where f is a float64-accumulating oracle of the operation
    (bilinear in its two operands).  When max E reaches `budget`, a deterministic fraction of `a` is zeroed until it does not
    (zeros are exact; positive data makes E its own budget).  Returns (E, a as used)."""
    keep = 1.0
    a0 = a
    for _ in range(20):
        ha, la = split(kind, a)
        hb, lb = split(kind, b)
        E = np.asarray(f(ha, hb), np.float64) + np.asarray(f(ha, lb), np.float64) + np.asarray(f(la, hb), np.float64)
        top = float(E.max()) if E.size else 0.0
        if top < budget:
            assert np.all(E == np.round(E / GRID) * GRID), "E is not on the 2^-13 grid: the probe data is not exact"
            return E, a
        keep *= 0.9 * budget / top
        a = thin(a0, keep)
    raise AssertionError("could not bring the probe under its budget")


def pow2_scale(rng, arr, axis, lo=-12, hi=12):
    """arr times 2^e, e drawn per index along `axis` (an int or a tuple of ints, one exponent set per axis) in [lo, hi]"""
    out = np.asarray(arr, np.float32)
    for ax in ((axis,) if isinstance(axis, int) else axis):
        shape = [1] * out.ndim
        shape[ax] = out.shape[ax]
        out = out * np.exp2(rng.integers(lo, hi + 1, out.shape[ax])).reshape(shape).astype(np.float32)
    return out.astype(np.float32)


def chain(kind, K, splits=1, extra=1):
    """n of elem_bound: fp32 accumulator additions along one element's chain -- TERMS per MMA k-step over a reduction of K
    (per split), one per split in the fixed-order reduction, and `extra` (bias, dx0 or dW0, or an accumulator fold)"""
    return TERMS[kind] * -(-int(K) // KSTEP[kind]) + (splits if splits > 1 else 0) + extra


def elem_bound(kind, n, mag, ref):
    """(c_split + n * 2^-23) * mag + 2^-23 * |ref|; mag: the oracle on |operands|.  Each of the n additions is off by at most one
    ulp (2^-23 relative) of a partial sum bounded by mag; the last term covers the final rounding and the oracle's fp32 output."""
    return (C_SPLIT[kind] + n * 2.0 ** -23) * np.asarray(mag, np.float64) + 2.0 ** -23 * np.abs(np.asarray(ref, np.float64))


def probe_mismatch(got, want):
    """None when got == want element by element, else a message: the count, the first index, got, want and the difference in
    2^-13 units (a whole number points to a dropped or doubled term; a scattered pattern to a lo word paired with the wrong
    element)"""
    got = np.asarray(got, np.float64)
    bad = np.argwhere(got != want)
    if bad.size == 0:
        return None
    i = tuple(int(v) for v in bad[0])
    units = (got - want)[got != want] / GRID
    whole = np.mean(units == np.round(units))
    return (f"{len(bad)} of {got.size} elements differ from the three-term sum, first at {i}: got {got[i]!r}, want {want[i]!r}, "
            f"difference {(got[i] - want[i]) / GRID:.4g} units of 2^-13 (a whole number of units on {whole:.0%} of them)")


def bound_report(got, ref, bnd):
    """(max err / bound, message or None)"""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64))
    ratio = err / bnd
    worst = float(np.nanmax(ratio)) if ratio.size else 0.0
    bad = np.argwhere(~(err <= bnd))
    if bad.size == 0:
        return worst, None
    i = tuple(int(v) for v in bad[0])
    return worst, (f"{len(bad)} of {err.size} elements over the per-element bound, first at {i}: got {got[i]!r}, "
                   f"ref {ref[i]!r}, bound {bnd[i]:.3g}")
