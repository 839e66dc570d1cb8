"""The checks of test_conv_precision_gpu.py have teeth: a numpy emulation of a correct tensor-core convolution passes both, and
each way of mishandling the lo half of the split is rejected by at least one of them, where the suites' 1e-4 blob-level bar lets
the localized ones through.

The emulated kernel is the forward convolution as the gather and staged kernels compute it: per image, im2col (o.im2col) times
the filter over the restated splits (tests/tc_precision.py), one fp32 rounding per MMA k-step and term (16-wide K steps for
bf16x3, 8-wide for 3xTF32 and TF32), optionally split along K with the partials added in split order, then the bias."""
import numpy as np
import pytest

import oracle as o
from cases import make, rel_err
import tc_precision as tp

CASE = dict(N=2, Cin=32, H=6, W=6, O=40, k=3, s=1, p=1, d=1, G=1, bias=True)   # K = 288; O = 40: a ragged last N tile of 8
N_TILE = 32
K_BLOCK = 64
SMALL = np.float32(2.0 ** -8)


def emulate(kind, po, x, w, b, splits=1, mutant=None):
    """the fp32 result of a tensor-core forward under `kind`, with one of the mutants below applied"""
    cols = np.stack([o.im2col(x[n], po.kh, po.sh, po.ph, po.dh).reshape(po.Kd, -1) for n in range(po.N)])   # [N, K, P]
    wm = w.reshape(po.O, po.Kd)
    wh, wl = (t.astype(np.float64) for t in tp.split(kind, wm))
    ch, cl = (t.astype(np.float64) for t in tp.split(kind, cols))
    if mutant == "swap_lo_pairs":                        # the e / o halves of each packed lo word exchanged
        cl = cl.copy()
        cl[:, 0::2], cl[:, 1::2] = cl[:, 1::2].copy(), cl[:, 0::2].copy()
    ragged = np.arange(po.O) >= (po.O // N_TILE) * N_TILE
    if mutant == "ragged_tile_lo_zero":                  # the last, partial N tile runs hi * hi' alone
        wl = np.where(ragged[:, None], 0.0, wl)
    ks = tp.KSTEP[kind]
    per = -(-po.Kd // splits)
    parts = []
    for s in range(splits):
        acc = np.zeros((po.N, po.O, cols.shape[2]), np.float32)
        for k0 in range(s * per, min(po.Kd, (s + 1) * per), ks):
            k = slice(k0, min(k0 + ks, po.Kd))
            terms = [("hh", wh, ch), ("hl", wh, cl), ("lh", wl, ch)] if tp.TERMS[kind] == 3 else [("hh", wh, ch)]
            for name, A, B in terms:
                if name == "hl" and (mutant == "drop_hilo_all" or (mutant == "drop_hilo_block" and k0 // K_BLOCK == 0)):
                    continue
                if name == "lh" and mutant == "ragged_tile_lo_zero":
                    t = np.einsum("ok,nkp->nop", A[:, k], B[:, k])
                    t[:, ragged] = 0.0
                else:
                    t = np.einsum("ok,nkp->nop", A[:, k], B[:, k])
                acc = (acc.astype(np.float64) + t).astype(np.float32)
        parts.append(acc)
    if mutant == "splitk_partial_twice":
        parts.insert(1, parts[0])
    y = parts[0]
    for p in parts[1:]:
        y = (y + p).astype(np.float32)
    if b is not None:
        y = (y + b[None, :, None]).astype(np.float32)
    return y.reshape(po.y_shape())


def probe_check(kind, po, rng, **kw):
    """None when the emulation equals the three-term sum exactly on probe data, else the mismatch"""
    jmax = 3 if kind == tp.TF32 else 7
    x, w = tp.probe_operand(rng, po.x_shape(), jmax=jmax), tp.probe_operand(rng, po.w_shape(), jmax=jmax)
    b = rng.integers(-4, 5, po.O).astype(np.float32)
    E, x = tp.three_term(lambda a, c: o.conv_forward(po, a, c, None, acc64=True), x, w, kind)
    got = emulate(kind, po, x, w, b, **kw)
    return tp.probe_mismatch(got, E + b[None, :, None, None])


def float_data(rng, po, localized=False):
    """normal data; pow2-scaled per image and channel, or (localized) with the weights of the ragged N tile and the input
    channels of the first K block scaled by 2^-8, the elements a localized mistake touches"""
    x = rng.standard_normal(po.x_shape()).astype(np.float32)
    w = (rng.standard_normal(po.w_shape()) * (2.0 / po.Kd) ** 0.5).astype(np.float32)
    b = (rng.standard_normal(po.O) * 0.1).astype(np.float32)
    if localized:
        x[:, :-(-K_BLOCK // (po.kh * po.kw))] *= SMALL
        w[(po.O // N_TILE) * N_TILE:] *= SMALL
        b[(po.O // N_TILE) * N_TILE:] *= SMALL
    else:
        x = tp.pow2_scale(rng, x, (0, 1))
        w = tp.pow2_scale(rng, w, (0, 1))
    return x, w, b


def bound_check(kind, po, x, w, b, splits=1, **kw):
    """(max err / bound, message or None, blob-level error)"""
    ref = o.conv_forward(po, x, w, b, acc64=True)
    mag = o.conv_forward(po, np.abs(x), np.abs(w), np.abs(b), acc64=True)
    got = emulate(kind, po, x, w, b, splits=splits, **kw)
    bnd = tp.elem_bound(kind, tp.chain(kind, -(-po.Kd // splits), splits), mag, ref)
    worst, msg = tp.bound_report(got, ref, bnd)
    return worst, msg, rel_err(got, ref)


@pytest.fixture(scope="module")
def po():
    return make(o, CASE)


# ---- the restated splits on probe data ------------------------------------------------------------------------------------
@pytest.mark.parametrize("hmax", [1, 2])
def test_probe_splits_exactly(hmax):
    rng = np.random.default_rng(3)
    a = tp.probe_operand(rng, 4096, hmax)
    h = np.floor(a)
    l = (a - h).astype(np.float32)
    assert set(np.unique(h)) <= set(range(1, hmax + 1)) and (l > 0).all() and (l <= 7 * tp.GRID).all()
    for kind in (tp.BF16X3, tp.TF32X3):
        hi, lo = tp.split(kind, a)
        assert np.array_equal(hi, h) and np.array_equal(lo, l), kind
    a3 = tp.probe_operand(rng, 4096, hmax, jmax=3)          # TF32 math: round to nearest drops l
    assert np.array_equal(tp.to_tf32(a3), np.floor(a3))


def test_split_restatements_on_normal_data():
    a = np.random.default_rng(4).standard_normal(1 << 16).astype(np.float32)
    # the per-operand errors C_SPLIT is derived from: bf16 keeps 8 significant bits (round to nearest), TF32 11 (truncated)
    for kind, u in ((tp.BF16X3, 2.0 ** -8), (tp.TF32X3, 2.0 ** -10)):
        hi, lo = tp.split(kind, a)
        assert (np.abs(a.astype(np.float64) - hi) <= u * np.abs(a)).all(), kind
        assert (np.abs(a.astype(np.float64) - hi - lo) <= u * u * np.abs(a)).all(), kind
    t = tp.to_tf32(a)
    assert (np.abs(a.astype(np.float64) - t) <= 2.0 ** -11 * np.abs(a)).all()
    assert tp.to_tf32(np.float32(1 + 2.0 ** -11))[()] == np.float32(1 + 2.0 ** -10)     # the tie rounds away


def test_three_term_thins_to_its_budget():
    """K = 4608: E would reach ~10^4; a deterministic fraction of x is zeroed until max E < 2^10"""
    po = make(o, dict(N=1, Cin=512, H=5, W=5, O=8, k=3, s=2, p=1, d=1, G=1, bias=False))
    rng = np.random.default_rng(5)
    x, w = tp.probe_operand(rng, po.x_shape()), tp.probe_operand(rng, po.w_shape())
    E, xt = tp.three_term(lambda a, c: o.conv_forward(po, a, c, None, acc64=True), x, w, tp.BF16X3)
    assert E.max() < tp.BUDGET and E.max() > tp.BUDGET / 4
    assert 0 < (xt == 0).mean() < 1 and np.array_equal(xt[xt != 0], x[xt != 0])


# ---- a correct kernel passes both checks ------------------------------------------------------------------------------------
@pytest.mark.parametrize("splits", [1, 3])
@pytest.mark.parametrize("kind", [tp.BF16X3, tp.TF32X3, tp.TF32])
def test_correct_kernel_passes(po, kind, splits):
    rng = np.random.default_rng(6)
    assert probe_check(kind, po, rng, splits=splits) is None
    worst, msg, blob = bound_check(kind, po, *float_data(rng, po), splits=splits)
    print(f"[emulated {kind}, {splits} splits] max err / bound {worst:.3g}, blob err {blob:.3g}")
    assert msg is None, msg
    assert blob < (1e-3 if kind == tp.TF32 else 1e-4)


# ---- each mutant is rejected; the localized ones get past the blob-level bar ---------------------------------------------
MUTANTS = [  # (mutant, splits, localized)
    ("drop_hilo_all", 1, False),
    ("drop_hilo_block", 1, True),
    ("ragged_tile_lo_zero", 1, True),
    ("swap_lo_pairs", 1, False),
    ("splitk_partial_twice", 3, False),
]


@pytest.mark.parametrize("kind", [tp.BF16X3, tp.TF32X3])
@pytest.mark.parametrize("mutant,splits,localized", MUTANTS, ids=[m[0] for m in MUTANTS])
def test_mutant_is_rejected(po, kind, mutant, splits, localized):
    rng = np.random.default_rng(7)
    probe = probe_check(kind, po, rng, splits=splits, mutant=mutant)
    worst, msg, _ = bound_check(kind, po, *float_data(rng, po), splits=splits, mutant=mutant)
    print(f"[{mutant}, {kind}] probe: {probe}; bound: max err / bound {worst:.3g}")
    assert probe is not None or msg is not None, f"{mutant} passes both checks"
    assert probe is not None, f"{mutant} passes the exact probe"
    if localized:
        # the gap the two checks close: on data where the mistake touches only small elements, the blob-level bar passes it
        _, _, blob = bound_check(kind, po, *float_data(rng, po, localized=True), splits=splits, mutant=mutant)
        assert blob < 1e-4, blob
