"""The fused solver updates (csrc/sgd.cu) element by element against the oracle, on every launch regime b2c_debug_solver_plan
reports.  Every case asserts its plan first, writes into arenas whose gaps between segments hold a NaN sentinel that must survive,
and runs twice from the same inputs, which must give the same bits.

- Bit-exact tier: on data over several binades (with +-0 and subnormals) every element of g, w, h and h2 must equal the fp32
  oracle (oracle.solver_fp32) under the contraction form of its path -- the float4 body's or the scalar loops', which differ in
  one product (SCALAR_FORM, BODY_FORM) -- on the float4 path, the scalar path and, for SGD, the legacy b2c_sgd_update.  On dyadic
  data every product that meets a sum is exact, so the kernel must equal the plain numpy restatement (solver_oracle.kernel_fp32)
  bit for bit, whatever it contracts (AdaDelta's h2 and w keep the per-path form check).
- Layouts: the counts and starts of every head / body / tail split, zero-count segments, 0 / 96 / 97 / 192 / 193 segments, one
  segment of 2^26 + 3 elements, the legacy kernel over several grid-stride passes.
- Float64 tier: the ResNet-50 arena with realistic magnitudes, every kind, within oracle.solver_f64's derived bound.
- Refusals: nothing is written by a call the library refuses."""
import os

import numpy as np
import pytest

import oracle as o
import solver_oracle as so
from caffe_mpi_b200 import capi, host_api

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESNET50 = os.path.join(ROOT, "tests", "golden", "reference_models", "models", "resnet50", "train_val.prototxt")
SEG_MAX, BLOCK = 96, 4096
SENTINEL = np.array([0x7fc0dead], np.int32).view(np.float32)[0]      # a quiet NaN with a payload: gaps must keep these bits
F = np.float32
# The contraction nvcc chooses for each rule, as oracle.solver_fp32 forms.  The scalar loops (head, tail, and spans whose arrays
# do not share their offset within 16 bytes) fuse decay*reg into gr = fma(reg, decay, g*s) (bit 1); the unrolled float4 body
# fuses g*s instead, gr = fma(g, s, decay*reg) (bit 0).  The rest is the same on both paths:
#   SGD       h = fma(m, h, lr*gr)                                          bit 2
#   Nesterov  h' = fma(lr, gr, m*h), u = fma(1+m, h', -(m*h))               bits 3, 4
#   AdaGrad   h = fma(gr, gr, h)                                            bit 2
#   RMSProp   h = fma(rd, h, (1-rd)*gr*gr)                                  bit 2
#   AdaDelta  h = fma(m, h, (1-m)*gr*gr), h2 likewise, w = w - lr*gr        bits 2, 4
#   Adam      m = fma(m, b1, gr*(1-b1)), v = fma(v, b2, gr*gr*(1-b2))       bits 2, 4
# So one element's bits depend on whether it falls in a float4 unit; the suite pins both forms element by element.
SCALAR_FORM = {"SGD": 0b110, "Nesterov": 0b11010, "AdaGrad": 0b110, "RMSProp": 0b110, "AdaDelta": 0b10110, "Adam": 0b10110}
BODY_FORM = {k: f ^ 0b11 for k, f in SCALAR_FORM.items()}
# AdaDelta with clear_grads: the step u = lr*gr is not stored, and nvcc fuses w - lr*gr into fma(-lr, gr, w) (bit 6) in some of
# the scalar loops it specialises for clear and not in others, so a scalar element's w may take either result.
def scalar_alternative(kind, clear):
    return 0b1000000 if kind == "AdaDelta" and clear else 0

def _bits(a):
    return np.ascontiguousarray(a, F).view(np.int32)


def layout(counts, mods=None, gap=2):
    """offsets of `counts` in order, segment s starting at an element offset = mods[s] (mod 4), a sentinel gap of >= `gap`
    elements between neighbours; -> (offsets, total)"""
    offs, off = [], 5
    for s, c in enumerate(counts):
        off += gap
        if mods is not None:
            off += (mods[s] - off) % 4
        offs.append(off)
        off += c
    return offs, off + 7


def hp_for(kind, base=so.KERNEL_HP, **kw):
    hp = dict(base, **kw)
    if kind in ("AdaGrad", "RMSProp"):
        hp["momentum"] = 0.0
    return hp


class Arena:
    """g, w, h, h2 device arenas of `total` elements: segment data at the offsets, the sentinel elsewhere.  shift: None (all four
    arrays at 16-byte-aligned bases), "all" (all four 4 bytes on: float4 path, other heads), "g" or "h2" (that array alone 4 bytes
    on: the scalar path, for h2 only where the kind reads it)."""

    def __init__(self, total, offsets, counts, arrays, shift=None):
        import torch
        self.total, self.offsets, self.counts, self.shift = total, offsets, counts, shift
        self.host = []
        for a in arrays:
            full = np.full(total, SENTINEL, F)
            for o_, c in zip(offsets, counts):
                full[o_:o_ + c] = a[o_:o_ + c]
            self.host.append(full)
        self.bufs, self.views = [], []
        for k, full in enumerate(self.host):
            lead = 1 if shift == "all" or (shift == "g" and k == 0) or (shift == "h2" and k == 3) else 0
            buf = torch.empty(total + 4, dtype=torch.float32, device="cuda")
            buf.fill_(float("nan"))
            self.bufs.append(buf)
            self.views.append(buf[lead:lead + total])
        self.reset()

    def reset(self):
        import torch
        for v, full in zip(self.views, self.host):
            v.copy_(torch.from_numpy(full))

    def ptrs(self):
        return [v.data_ptr() for v in self.views]

    def fetch(self):
        import torch
        torch.cuda.synchronize()
        return [v.cpu().numpy() for v in self.views]


def seg_mask(total, offsets, counts):
    m = np.zeros(total, bool)
    for o_, c in zip(offsets, counts):
        m[o_:o_ + c] = True
    return m


def check_plan(kind, ar, vec):
    """the plan of this call: launches of at most 96 non-empty segments, the blocks of every segment, the head / body / tail split
    of the path `vec` expects (None: whatever the offsets give)"""
    g, w, h, h2 = ar.ptrs()
    q = capi.solver_plan(kind, ar.offsets, ar.counts, g, w, h, h2)
    nonempty = [s for s, c in enumerate(ar.counts) if c]
    assert [n for n, _ in q["launches"]] == [min(SEG_MAX, len(nonempty) - i) for i in range(0, len(nonempty), SEG_MAX)]
    for s, c in enumerate(ar.counts):
        d = q["segs"][s]
        if not c:
            assert d["launch"] == -1 and d["blocks"] == 0
            continue
        assert d["launch"] == nonempty.index(s) // SEG_MAX and d["blocks"] == -(-c // BLOCK)
        assert d["head"] + 4 * d["body4"] + d["tail"] == c
        if vec is not None:
            assert d["vec"] == vec, (s, d)
        if not d["vec"]:
            assert d["tail"] == c
    return q


def launch(kind, ar, rates, decays, hp, l2, gs, clear):
    import torch
    G, W, H, H2 = ar.views
    capi.solver_update_arena(kind, ar.offsets, ar.counts, rates, decays, G, W, H, H2 if kind in so.TWO_HISTORIES else None,
                             momentum=hp["momentum"], delta=hp["delta"], rms_decay=hp["rms_decay"], beta1=hp["beta1"],
                             beta2=hp["beta2"], l2=l2, grad_scale=gs, clear_grads=clear)
    torch.cuda.synchronize()


def run_twice(kind, ar, rates, decays, hp, l2, gs, clear, call=launch):
    call(kind, ar, rates, decays, hp, l2, gs, clear)
    first = ar.fetch()
    ar.reset()
    call(kind, ar, rates, decays, hp, l2, gs, clear)
    second = ar.fetch()
    for k in range(4):
        assert np.array_equal(_bits(first[k]), _bits(second[k])), f"{kind}: array {k} differs between two identical calls"
    gaps = ~seg_mask(ar.total, ar.offsets, ar.counts)
    for k in range(4):
        assert np.all(_bits(first[k])[gaps] == _bits(SENTINEL)), f"{kind}: array {k} written outside its segments"
    return first


def outputs_checked(kind, clear):
    """indices of (g, w, h, h2) that carry information: g only when kept, h2 only for the two-history kinds"""
    return [k for k in range(4) if not (k == 0 and clear) and not (k == 3 and kind not in so.TWO_HISTORIES)]


def float4_mask(kind, ar, block=BLOCK):
    """elements the float4 body updates: in each span of `block` elements of a segment (None: the whole segment, as
    b2c_sgd_update's one grid-stride span) those after the head that peels the span to a 16-byte boundary, in whole float4 units;
    none when g, w, h (and h2 where the kind reads it) differ in their offset within 16 bytes or sit off 4-byte alignment"""
    m = np.zeros(ar.total, bool)
    g, w, h, h2 = ar.ptrs()
    mods = {p % 16 for p in ((g, w, h, h2) if kind in so.TWO_HISTORIES else (g, w, h))}
    if len(mods) != 1 or next(iter(mods)) % 4:
        return m
    for o_, c in zip(ar.offsets, ar.counts):
        step = block or max(c, 1)
        for b in range(0, c, step):
            n = min(step, c - b)
            hd = min((16 - (g + 4 * (o_ + b)) % 16) % 16 // 4, n)
            m[o_ + b + hd:o_ + b + hd + 4 * ((n - hd) // 4)] = True
    return m


def kernel_expected(kind, ar, inputs, rates, decays, hp, l2, gs, clear, block=BLOCK, forms=None):
    """what the kernel stores, per element: oracle.solver_fp32 under BODY_FORM on float4_mask's elements, SCALAR_FORM elsewhere"""
    scalar, body = forms or (SCALAR_FORM[kind], BODY_FORM[kind])
    mask = float4_mask(kind, ar, block)
    out = [a.copy() for a in ar.host]
    for s, (o_, c) in enumerate(zip(ar.offsets, ar.counts)):
        if not c:
            continue
        sl = slice(o_, o_ + c)
        a = o.solver_fp32(kind, scalar, *(x[sl] for x in inputs), hp, rates[s], decays[s], l2, gs, clear)
        b = o.solver_fp32(kind, body, *(x[sl] for x in inputs), hp, rates[s], decays[s], l2, gs, clear)
        for k in range(4):
            out[k][sl] = np.where(mask[sl], b[k], a[k])
    return out, mask


def assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, l2, gs, clear, block=BLOCK):
    """every element of every output equals kernel_expected bit for bit (a scalar element also scalar_alternative's result)"""
    want, mask = kernel_expected(kind, ar, inputs, rates, decays, hp, l2, gs, clear, block)
    alt = want
    if scalar_alternative(kind, clear):
        alt, _ = kernel_expected(kind, ar, inputs, rates, decays, hp, l2, gs, clear, block,
                                 forms=(SCALAR_FORM[kind] | scalar_alternative(kind, clear), BODY_FORM[kind]))
    seg = seg_mask(ar.total, ar.offsets, ar.counts)
    for k in outputs_checked(kind, clear):
        bad = np.flatnonzero((_bits(got[k]) != _bits(want[k])) & (_bits(got[k]) != _bits(alt[k])) & seg)
        if bad.size:
            i = bad[0]
            s = int(np.searchsorted(ar.offsets, i, side="right")) - 1
            raise AssertionError(f"{kind}: array {'gwhH'[k]}, {bad.size} elements differ; first: segment {s} element "
                                 f"{i - ar.offsets[s]} ({'float4 body' if mask[i] else 'scalar'}): got {got[k][i]!r}, "
                                 f"want {want[k][i]!r}")


def matching_forms(kind, got, ar, rates, decays, hp, l2, gs, clear, inputs, select, also=0):
    """the forms of oracle.solver_fp32 that reproduce every element of `select` (a mask over the arena) in every output; with
    `also`, an element may instead match the form with those bits set"""
    ks = outputs_checked(kind, clear)
    good = []
    for form in o.solver_forms(kind):
        if form & also:
            continue
        want, _ = kernel_expected(kind, ar, inputs, rates, decays, hp, l2, gs, clear, forms=(form, form))
        alt = kernel_expected(kind, ar, inputs, rates, decays, hp, l2, gs, clear, forms=(form | also,) * 2)[0] if also else want
        if all(np.all(((_bits(got[k]) == _bits(want[k])) | (_bits(got[k]) == _bits(alt[k])))[select]) for k in ks):
            good.append(form)
    return good


# ---- layouts and data -----------------------------------------------------------------------------------------------------------
EDGE_COUNTS = [1, 2, 3, 4, 4095, 4096, 4097, 3 * 4096 + 1]


def edge_layout():
    """every edge count at every start mod 4 (heads 0-3, segments shorter than their head), with empty segments between"""
    counts, mods = [], []
    for c in EDGE_COUNTS:
        for m in range(4):
            counts += [c, 0] if m == 1 else [c]
            mods += [m, 0] if m == 1 else [m]
    return counts, mods


def distinct_rates(rng, nseg):
    lr = rng.uniform(0.05, 0.5, nseg).astype(F)
    dc = rng.uniform(0.1, 0.9, nseg).astype(F)
    lr[: nseg] += np.arange(nseg, dtype=F) * F(1e-3)           # all distinct, and distinct from every neighbour's
    return [float(x) for x in lr], [float(x) for x in dc]


def wide_case(kind, counts, mods, seed):
    rng = np.random.default_rng(seed)
    offs, total = layout(counts, mods)
    inputs = so.wide_inputs(rng, total, kind)
    rates, decays = distinct_rates(rng, len(counts))
    return offs, total, inputs, rates, decays


# ---- bit-exact tier -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
@pytest.mark.parametrize("clear", [True, False], ids=["clear", "keep"])
def test_forms_bit_exact(kind, l2, clear):
    """every element is reproduced bit for bit by its path's pinned form -- the float4 body's or the scalar loops' -- on the float4
    path (two different heads), the scalar path (g alone, and h2 alone, 4 bytes off) and, for SGD, the legacy kernel; and of all
    the forms, the pinned ones are among those that match each path's elements"""
    import torch
    counts, mods = edge_layout()
    offs, total, inputs, rates, decays = wide_case(kind, counts, mods, 1701)
    hp, gs = hp_for(kind), 1 / 3
    seen = {"scalar": set(o.solver_forms(kind)), "body": set(o.solver_forms(kind))}
    for shift in (None, "all", "g", "h2"):
        ar = Arena(total, offs, counts, inputs, shift)
        vec = 0 if shift == "g" or (shift == "h2" and kind in so.TWO_HISTORIES) else 1
        q = check_plan(kind, ar, vec)
        mask = float4_mask(kind, ar)
        for s, (o_, c) in enumerate(zip(offs, counts)):      # the elements the suite treats as float4 units are the query's
            assert int(mask[o_:o_ + c].sum()) == 4 * q["segs"][s]["body4"], (shift, s)
        got = run_twice(kind, ar, rates, decays, hp, l2, gs, clear)
        assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, l2, gs, clear)
        seg = seg_mask(total, offs, counts)
        for path, sel in (("scalar", seg & ~mask), ("body", seg & mask)):
            if sel.any():
                also = scalar_alternative(kind, clear) if path == "scalar" else 0
                seen[path] &= set(matching_forms(kind, got, ar, rates, decays, hp, l2, gs, clear, inputs, sel, also))
    if kind == "SGD":
        # the legacy entry point, one call (one grid-stride span) per segment
        ar = Arena(total, offs, counts, inputs)

        def legacy(kind_, ar_, rates_, decays_, hp_, l2_, gs_, clear_):
            G, W, H, _ = ar_.views
            for s, (o_, c) in enumerate(zip(ar_.offsets, ar_.counts)):
                if c:
                    capi.sgd_update(G[o_:o_ + c], W[o_:o_ + c], H[o_:o_ + c], hp_["momentum"], rates_[s], decays_[s], l2_, gs_, clear_)
            torch.cuda.synchronize()
        got = run_twice(kind, ar, rates, decays, hp, l2, gs, clear, call=legacy)
        assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, l2, gs, clear, block=None)
    print(f"[solver forms] {kind} L2={l2} clear={clear}: scalar loops match forms {sorted(seen['scalar'])}, "
          f"float4 body {sorted(seen['body'])}")
    assert SCALAR_FORM[kind] in seen["scalar"] and BODY_FORM[kind] in seen["body"], (kind, seen)


@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
@pytest.mark.parametrize("clear", [True, False], ids=["clear", "keep"])
def test_dyadic_bit_exact(kind, l2, clear):
    """dyadic data: the kernel equals the numpy fp32 restatement bit for bit, whatever it contracts (AdaDelta's h2 and w: a form)"""
    rng = np.random.default_rng(29)
    counts, mods = edge_layout()
    offs, total = layout(counts, mods)
    inputs = so.dyadic_inputs(rng, total, kind)
    rates, decays = so.dyadic_rates(rng, len(counts))
    hp = hp_for(kind, so.DYADIC_HP)
    for shift in (None, "g"):
        ar = Arena(total, offs, counts, inputs, shift)
        check_plan(kind, ar, 0 if shift == "g" else 1)
        got = run_twice(kind, ar, rates, decays, hp, l2, 0.125, clear)
        for s, (o_, c) in enumerate(zip(offs, counts)):
            sl = slice(o_, o_ + c)
            want = so.kernel_fp32(kind, *(a[sl] for a in inputs), hp, rates[s], decays[s], l2, 0.125, clear)
            for k in outputs_checked(kind, clear):
                if kind == "AdaDelta" and k in (1, 3):
                    continue
                bad = np.flatnonzero(_bits(got[k][sl]) != _bits(want[k]))
                assert bad.size == 0, (kind, shift, s, "gwhH"[k], bad[:4], got[k][sl][bad[:4]], want[k][bad[:4]])
        if kind == "AdaDelta":
            assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, l2, 0.125, clear)


# ---- values ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["AdaGrad", "RMSProp", "AdaDelta", "Adam"])
@pytest.mark.parametrize("delta", ["below", "at", "above"])
def test_delta_clamp(kind, delta):
    """delta below its clamp (1e-8: the clamp is used), at it, and above it (1e-2)"""
    clamp = 1e-3 if kind in ("AdaGrad", "AdaDelta") else 1e-4
    d = {"below": 1e-8, "at": clamp, "above": 1e-2}[delta]
    counts, mods = [4097, 3, 130], [1, 2, 0]
    offs, total, inputs, rates, decays = wide_case(kind, counts, mods, 3)
    hp = hp_for(kind, delta=d)
    ar = Arena(total, offs, counts, inputs)
    check_plan(kind, ar, 1)
    got = run_twice(kind, ar, rates, decays, hp, True, 1.0, False)
    assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, True, 1.0, False)
    # the clamp changes the result: the same call with delta = the clamp gives the same bits exactly when d <= clamp
    hp_c = dict(hp, delta=clamp)
    ref = o.solver_fp32(kind, 0, *(a[offs[0]:offs[0] + counts[0]] for a in inputs), hp_c, rates[0], decays[0], True, 1.0, False)
    mine = o.solver_fp32(kind, 0, *(a[offs[0]:offs[0] + counts[0]] for a in inputs), hp, rates[0], decays[0], True, 1.0, False)
    assert np.array_equal(_bits(ref[1]), _bits(mine[1])) == (d <= clamp)


@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("gs", [1.0, 0.125, 1 / 3], ids=["gs1", "gs1_8", "gs1_3"])
def test_grad_scale(kind, gs):
    """the folded grad_scale: exact (1, 1/8) and rounding (1/3: three ranks, iter_size 3 or global_grad_scale 3)"""
    counts, mods = [4096 + 5, 7, 1000], [3, 0, 2]
    offs, total, inputs, rates, decays = wide_case(kind, counts, mods, 5)
    hp = hp_for(kind)
    ar = Arena(total, offs, counts, inputs)
    check_plan(kind, ar, 1)
    got = run_twice(kind, ar, rates, decays, hp, True, gs, False)
    assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, True, gs, False)


@pytest.mark.parametrize("kind", so.KINDS)
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
def test_zero_rate_is_the_identity(kind, l2):
    """lr = decay = 0 with g = h = h2 = 0 leaves every bit of w as it was, -0 and subnormals included: ApplyUpdate relies on it
    to leave the BatchNorm statistics out of the launch"""
    rng = np.random.default_rng(41)
    counts, mods = edge_layout()
    offs, total = layout(counts, mods)
    _, w, _, _ = so.wide_inputs(rng, total, kind)
    w[::7] = F(-0.0)
    z = np.zeros(total, F)
    for shift in (None, "g"):
        ar = Arena(total, offs, counts, [z, w, z, z], shift)
        check_plan(kind, ar, 0 if shift == "g" else 1)
        got = run_twice(kind, ar, [0.0] * len(counts), [0.0] * len(counts), hp_for(kind), l2, 1.0, False)
        m = seg_mask(total, offs, counts)
        assert np.array_equal(_bits(got[1])[m], _bits(w)[m]), kind
        for k in (0, 2, 3):
            assert np.all(_bits(got[k])[m] == 0), (kind, k)


# ---- layouts --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["SGD", "Adam"])
@pytest.mark.parametrize("nseg", [0, 96, 97, 192, 193, "zeros_at_boundary"])
def test_segment_counts(kind, nseg):
    """0, 96, 97, 192 and 193 segments (one, two and three launches), and zero-count segments at the 96th / 97th non-empty
    position; every segment with its own lr and decay, so a segment given a neighbour's constants is caught"""
    rng = np.random.default_rng(17)
    if nseg == "zeros_at_boundary":
        counts = [int(c) for c in rng.integers(1, 40, 95)] + [0, 33, 0, 0, 21] + [int(c) for c in rng.integers(1, 40, 100)] + [0]
    else:
        counts = [int(c) for c in rng.integers(1, 40, nseg)]
    mods = [int(m) for m in rng.integers(0, 4, len(counts))]
    offs, total, inputs, rates, decays = wide_case(kind, counts, mods, 19)
    hp = hp_for(kind)
    ar = Arena(total, offs, counts, inputs)
    q = check_plan(kind, ar, None)
    assert len(q["launches"]) == -(-sum(1 for c in counts if c) // SEG_MAX)
    got = run_twice(kind, ar, rates, decays, hp, True, 1 / 3, False)
    if counts:
        assert_kernel_bits(kind, got, ar, inputs, rates, decays, hp, True, 1 / 3, False)


def test_largest_segment():
    """one segment of 2^26 + 3 elements starting at 1 mod 4 (Adam: four arrays, ~1 GB), dyadic data against numpy bit for bit"""
    kind, n = "Adam", (1 << 26) + 3
    rng = np.random.default_rng(23)
    offs, total = layout([n], [1])
    inputs = so.dyadic_inputs(rng, total, kind)
    hp = hp_for(kind, so.DYADIC_HP)
    ar = Arena(total, offs, [n], inputs)
    q = check_plan(kind, ar, 1)
    assert q["segs"][0]["blocks"] == -(-n // BLOCK) and q["segs"][0]["head"] == 3 * q["segs"][0]["blocks"]
    got = run_twice(kind, ar, [3 / 128], [5 / 256], hp, True, 0.125, False)
    sl = slice(offs[0], offs[0] + n)
    want = so.kernel_fp32(kind, *(a[sl] for a in inputs), hp, 3 / 128, 5 / 256, True, 0.125, False)
    for k in range(4):
        assert np.array_equal(_bits(got[k][sl]), _bits(want[k])), "gwhH"[k]


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, (1 << 22) + 3])
@pytest.mark.parametrize("l2", [True, False], ids=["L2", "L1"])
def test_legacy_sgd_update(n, l2):
    """b2c_sgd_update at n = 1..5 and at 2^22 + 3 (several grid-stride passes at 132 SMs), starting at every offset mod 4: every
    element as its path's pinned form gives it -- one head for the whole span, where the arena kernel peels one per 4096-element
    block -- and the arena kernel on the same segment likewise"""
    import torch
    hp = hp_for("SGD")
    for mod in range(4):
        offs, total = layout([n], [mod])
        inputs = so.wide_inputs(np.random.default_rng(n + mod), total, "SGD")
        ar = Arena(total, offs, [n], inputs)
        check_plan("SGD", ar, 1)

        def legacy(kind_, ar_, rates_, decays_, hp_, l2_, gs_, clear_):
            G, W, H, _ = ar_.views
            sl = slice(offs[0], offs[0] + n)
            capi.sgd_update(G[sl], W[sl], H[sl], hp_["momentum"], rates_[0], decays_[0], l2_, gs_, clear_)
            torch.cuda.synchronize()
        got = run_twice("SGD", ar, [0.03], [0.4], hp, l2, 1 / 3, False, call=legacy)
        assert_kernel_bits("SGD", got, ar, inputs, [0.03], [0.4], hp, l2, 1 / 3, False, block=None)
        ar.reset()
        got = run_twice("SGD", ar, [0.03], [0.4], hp, l2, 1 / 3, False)
        assert_kernel_bits("SGD", got, ar, inputs, [0.03], [0.4], hp, l2, 1 / 3, False)


# ---- float64 tier ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", so.KINDS)
def test_resnet50_arena_within_float64_bound(kind):
    """the ResNet-50 learnable layout (161 segments, padded to even counts as ParamArena pads them) with realistic magnitudes,
    every element within oracle.solver_f64's derived bound"""
    lp = host_api.Net(open(RESNET50).read(), is_text=True).learnable_params()
    counts = [c for _, c, _, _ in lp]
    offs, off = [], 0
    for c in counts:
        offs.append(off)
        off += c + (c & 1)
    total = off
    rng = np.random.default_rng(31)
    g = (rng.standard_normal(total) * 1e-3).astype(F)
    w = (rng.standard_normal(total) * 0.05).astype(F)
    h = (rng.standard_normal(total) * 1e-3).astype(F)
    h2 = (np.abs(rng.standard_normal(total)) * 1e-6).astype(F)
    if kind not in ("SGD", "Nesterov", "Adam"):
        h = np.abs(h) * F(1e-3)
    rates = [float(F(0.1 * lr * (1 + s / 1000))) for s, (_, _, lr, _) in enumerate(lp)]
    decays = [float(F(1e-4 * dc * (1 + s / 1000))) for s, (_, _, _, dc) in enumerate(lp)]
    hp = hp_for(kind)
    ar = Arena(total, offs, counts, [g, w, h, h2])
    q = check_plan(kind, ar, 1)
    assert [n for n, _ in q["launches"]] == [96, 65]
    got = run_twice(kind, ar, rates, decays, hp, True, 1 / 3, False)
    worst = 0.0
    for s, (o_, c) in enumerate(zip(offs, counts)):
        sl = slice(o_, o_ + c)
        vals, bounds = o.solver_f64(kind, g[sl], w[sl], h[sl], h2[sl], hp, rates[s], decays[s], True, 1 / 3, False)
        for k in outputs_checked(kind, False):
            err = np.abs(got[k][sl].astype(np.float64) - vals[k])
            r = err / np.maximum(bounds[k], 1e-300)
            assert np.all(err <= bounds[k] * (1 + 2.0 ** -20)), (kind, s, "gwhH"[k], float(r.max()))
            worst = max(worst, float(r.max()))
    print(f"[solver f64] {kind}: ResNet-50 arena, worst |kernel - f64| / bound = {worst:.3f}")


# ---- refusals -------------------------------------------------------------------------------------------------------------------
def test_refused_call_writes_nothing():
    """100 segments, the 99th over 2^32 - 1 elements: refused before any launch, so every arena byte is unchanged (the packing of
    the first 96 segments must not run ahead of the check).  Null h2 for AdaDelta and Adam and an unknown kind: refused, nothing
    written."""
    counts = [11] * 100
    offs, total, inputs, rates, decays = wide_case("SGD", counts, None, 43)
    big = list(counts)
    big[98] = 1 << 32
    for kind in so.KINDS:
        ar = Arena(total, offs, counts, inputs)
        with pytest.raises(capi.B2CError, match="segment 98 too large"):
            capi.solver_plan(kind, offs, big, *ar.ptrs())
        G, W, H, H2 = ar.views
        with pytest.raises(capi.B2CError, match="segment 98 too large"):
            capi.solver_update_arena(kind, offs, big, rates, decays, G, W, H, H2, momentum=0.9, delta=1e-3, rms_decay=0.9)
        if kind in so.TWO_HISTORIES:
            with pytest.raises(capi.B2CError):
                capi.solver_update_arena(kind, offs, counts, rates, decays, G, W, H, None, momentum=0.9)
        got = ar.fetch()
        for k in range(4):
            assert np.array_equal(_bits(got[k]), _bits(ar.host[k])), (kind, "gwhH"[k])
    ar = Arena(total, offs, counts, inputs)
    G, W, H, H2 = ar.views
    with pytest.raises(capi.B2CError, match="segment 98 too large"):
        capi.sgd_update_arena(offs, big, rates, decays, G, W, H, 0.9)
    for bad in (-1, 6):
        with pytest.raises(capi.B2CError, match="unknown solver kind"):
            capi.solver_update_arena(bad, offs, counts, rates, decays, G, W, H, H2)
    got = ar.fetch()
    for k in range(4):
        assert np.array_equal(_bits(got[k]), _bits(ar.host[k])), "gwhH"[k]
