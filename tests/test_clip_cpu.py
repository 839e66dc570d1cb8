"""clip_gradients without a GPU: the float64 clip oracle against hand-computed norms and factors, the launch plan of the norm's
partials (b2c_debug_sumsq_plan), the entry points' refusals, and solver files that set the field."""
import ctypes as C
import math

import numpy as np
import pytest

from caffe_mpi_b200 import capi, host_api
import clip_oracle as co

F = np.float32
A = 1 << 20                                               # a 16-byte aligned arena base (never dereferenced)


def test_oracle_known_answers():
    g = [np.array([3, 0], F), np.array([[4]], F)]         # ||g|| = 5
    assert co.sumsq(g) == 25.0
    assert co.clip_factor(g, 10.0) == (F(5), F(1))
    assert co.clip_factor(g, 5.0) == (F(5), F(1))         # norm == clip: not clipped
    assert co.clip_factor(g, 2.5) == (F(5), F(0.5))
    assert co.clip_factor(g, 2.5, s_n=0.5) == (F(2.5), F(1))   # the clip sees the gradient after 1/(solver_count * global_grad_scale)
    assert co.clip_factor(g, 1.0, s_n=0.25) == (F(1.25), F(0.8))
    assert co.clip_factor(g, 0.0) == (F(5), F(0))         # clip 0: the gradient term vanishes
    assert co.clip_factor([np.zeros(7, F)], 0.0) == (F(0), F(1))
    norm, factor = co.clip_factor([np.array([1, np.nan], F)], 1.0)
    assert math.isnan(norm) and factor == F(1)            # a NaN norm is not > clip: no scaling
    norm, factor = co.clip_factor([np.array([2e38, 2e38], F)], 1.0)
    assert norm == F(math.sqrt(2 * float(F(2e38)) ** 2)) and factor == F(1) / norm      # float32 squares overflow, the float64 sum does not
    assert co.clip_factor([np.array([1.0, 1.0, 1.0], F)], 1.0)[1] == F(1) / F(math.sqrt(3))
    assert co.clipped_grad_scale(0.5, F(1)) == F(0.5) and co.clipped_grad_scale(1 / 3, F(1)) == F(1 / 3)
    assert co.clipped_grad_scale(F(1 / 3), F(0.3)) == F(F(1 / 3) * F(0.3))


def test_oracle_sum_is_rounded_once():
    # 2^60 + many small squares: a float64 running sum drops every 1.0; fsum keeps them
    g = [np.array([2.0 ** 30], F), np.ones(4096, F)]
    assert co.sumsq(g) == 2.0 ** 60 + 4096
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(20000) * np.exp2(rng.integers(-20, 20, 20000))).astype(F)
    assert co.sumsq([x[:7000], x[7000:]]) == math.fsum(float(v) ** 2 for v in x)


def test_entry_points_refuse_to_launch_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    L = capi.lib()
    one = C.c_void_p(A)
    sz = lambda *v: (C.c_size_t * len(v))(*v)
    assert L.b2c_arena_sumsq(1, sz(0), sz(5000), sz(0), one, one, None) == -2
    assert L.b2c_clip_factor(one, 2, 1.0, 1.0, one, None) == -2
    hp = capi.SolverHParams(0.9, 1e-8, 0.0, 0.9, 0.999)
    for kind in range(6):
        assert L.b2c_solver_update_arena_scaled(kind, 1, sz(0), sz(5000), (C.c_float * 1)(0.1), (C.c_float * 1)(0.0), one, one, one,
                                                one, hp, 1, 1.0, one, 1, None) == -2
    # nothing to do is not an error
    assert L.b2c_arena_sumsq(0, None, None, None, None, None, None) == 0


def test_entry_points_refuse_bad_arguments():
    """refused before any launch, so the same with or without a device"""
    L = capi.lib()
    one = C.c_void_p(A)
    sz = lambda *v: (C.c_size_t * len(v))(*v)
    big = 1 << 32
    assert L.b2c_arena_sumsq(-1, sz(0), sz(1), sz(0), one, one, None) == -1
    for args in ((None, sz(1), sz(0), one, one), (sz(0), None, sz(0), one, one), (sz(0), sz(1), None, one, one),
                 (sz(0), sz(1), sz(0), None, one), (sz(0), sz(1), sz(0), one, None)):
        assert L.b2c_arena_sumsq(1, *args, None) == -1
    # a too-large segment past the first launch: refused whole
    counts = [7] * 100 + [big]
    assert L.b2c_arena_sumsq(101, sz(*range(0, 808, 8)), sz(*counts), sz(*range(101)), one, one, None) == -1
    assert b"too large" in L.b2c_last_error()
    assert L.b2c_clip_factor(None, 2, 1.0, 1.0, one, None) == -1
    assert L.b2c_clip_factor(one, 2, 1.0, 1.0, None, None) == -1
    for s_n, clip in ((1.0, -1.0), (1.0, float("nan")), (0.0, 1.0), (-1.0, 1.0), (float("inf"), 1.0), (float("nan"), 1.0)):
        assert L.b2c_clip_factor(one, 2, s_n, clip, one, None) == -1, (s_n, clip)
    hp = capi.SolverHParams(0.9, 1e-8, 0.0, 0.9, 0.999)
    rate, decay = (C.c_float * 1)(0.1), (C.c_float * 1)(0.0)
    assert L.b2c_solver_update_arena_scaled(0, 1, sz(0), sz(5), rate, decay, one, one, one, one, hp, 1, 1.0, None, 1, None) == -1
    assert L.b2c_solver_update_arena_scaled(6, 1, sz(0), sz(5), rate, decay, one, one, one, one, hp, 1, 1.0, one, 1, None) == -1
    assert L.b2c_solver_update_arena_scaled(5, 1, sz(0), sz(5), rate, decay, one, one, one, None, hp, 1, 1.0, one, 1, None) == -1
    assert L.b2c_solver_update_arena_scaled(0, 1, sz(0), sz(big), rate, decay, one, one, one, one, hp, 1, 1.0, one, 1, None) == -1


def _layout(counts, start=0):
    offs, off = [], start
    for c in counts:
        offs.append(off)
        off += c + (c & 1)                                # arena slots at even stride
    return offs


def test_slots_are_contiguous_in_arena_order():
    counts = [1, 4096, 4097, 0, 3 * 4096 + 5, 2, 64 * 4096, 7]
    slots, total = host_api.clip_slots(counts)
    blocks = [-(-c // 4096) for c in counts]
    assert slots == [sum(blocks[:i]) for i in range(len(counts))] and total == sum(blocks)
    q = capi.sumsq_plan(_layout(counts), counts, slots, A)
    assert q["npartials"] == total
    assert [s["blocks"] for s in q["segs"]] == blocks and [s["slot"] for s in q["segs"]] == slots
    assert host_api.clip_slots([]) == ([], 0)


@pytest.mark.parametrize("nseg", [0, 96, 97, 193])
def test_segment_plan_is_the_same_alone_in_a_bucket_or_in_the_whole_arena(nseg):
    """each segment's path, blocks, split and slot do not depend on which call carries it -- so neither do its partials"""
    rng = np.random.default_rng(nseg)
    counts = [int(c) for c in rng.integers(0, 3 * 4096, nseg)]
    for i in range(0, nseg, 11):
        counts[i] = 0                                     # zero counts: no launch position, no block
    offs = _layout(counts, start=3)                       # odd start: every segment peels a head
    slots, total = host_api.clip_slots(counts)
    whole = capi.sumsq_plan(offs, counts, slots, A)
    assert whole["npartials"] == total
    nonempty = sum(1 for c in counts if c)
    assert [n for n, _ in whole["launches"]] == [min(96, nonempty - 96 * i) for i in range(-(-nonempty // 96))]
    for s, c in enumerate(counts):
        w = whole["segs"][s]
        alone = capi.sumsq_plan([offs[s]], [c], [slots[s]], A)["segs"][0]
        assert {k: v for k, v in alone.items() if k != "launch"} == {k: v for k, v in w.items() if k != "launch"}, s
        assert (w["launch"] < 0) == (c == 0) and w["blocks"] == -(-c // 4096) and w["slot"] == slots[s]
        assert w["head"] + 4 * w["body4"] + w["tail"] == c
    # the buckets the scheduler flushes (reduce_buckets 6 and one per parameter)
    for rb in (6, max(1, nseg)):
        if not nseg:
            break
        for f, t, _, _ in host_api.plan_buckets([max(c, 1) for c in counts], rb):
            b = capi.sumsq_plan(offs[f:t + 1], counts[f:t + 1], slots[f:t + 1], A)
            for k, s in enumerate(range(f, t + 1)):
                want = {kk: v for kk, v in whole["segs"][s].items() if kk != "launch"}
                assert {kk: v for kk, v in b["segs"][k].items() if kk != "launch"} == want, (rb, s)


def test_plan_splits_and_misaligned_starts():
    def seg(off, cnt, g=A):
        s = capi.sumsq_plan([off], [cnt], [5], g)["segs"][0]
        return s["vec"], s["blocks"], s["slot"], s["head"], s["body4"], s["tail"]
    assert seg(8, 1) == (1, 1, 5, 0, 0, 1)
    assert seg(8, 4096) == (1, 1, 5, 0, 1024, 0)
    assert seg(9, 4096) == (1, 1, 5, 3, 1023, 1)
    assert seg(10, 4097) == (1, 2, 5, 3, 1023, 2)         # every block peels its own head (2, then 1 of 1)
    assert seg(11, 2) == (1, 1, 5, 1, 0, 1)
    assert seg(0, (1 << 26) + 3) == (1, (1 << 14) + 1, 5, 0, 1 << 24, 3)
    assert seg(0, 9, g=A + 2) == (0, 1, 5, 0, 0, 9)        # an address no float lives at: one float at a time
    assert seg(8, 0) == (0, 0, 5, 0, 0, 0)
    assert capi.sumsq_plan([], [], [], A) == dict(launches=[], segs=[], npartials=0)
    assert capi.sumsq_plan([0], [4097], [10], A)["npartials"] == 12


def test_plan_refuses_what_the_entry_point_refuses():
    L = capi.lib()
    sz = lambda *v: (C.c_size_t * len(v))(*v)
    lo, nl, seg, npart = (C.c_int * 8)(), C.c_int(), (C.c_longlong * 7000)(), C.c_longlong()
    g = C.c_void_p(A)
    plan = lambda n, o, c, s, gg: L.b2c_debug_sumsq_plan(n, o, c, s, gg, lo, 4, C.byref(nl), seg, C.byref(npart))
    assert plan(-1, sz(0), sz(1), sz(0), g) == -1
    for args in ((None, sz(1), sz(0), g), (sz(0), None, sz(0), g), (sz(0), sz(1), None, g), (sz(0), sz(1), sz(0), None)):
        assert plan(1, *args) == -1
    counts = [7] * 100 + [1 << 32]
    assert plan(101, sz(*range(0, 808, 8)), sz(*counts), sz(*range(101)), g) == -1
    assert plan(101, sz(*range(0, 808, 8)), sz(*counts[:100], (1 << 32) - 1), sz(*range(101)), g) == 0
    assert nl.value == 2 and npart.value == 100 + (1 << 20)           # the last segment: 2^20 blocks from slot 100
    # and only the outputs it needs
    assert L.b2c_debug_sumsq_plan(1, sz(0), sz(1), sz(0), g, lo, 4, None, seg, C.byref(npart)) == -1
    assert L.b2c_debug_sumsq_plan(1, sz(0), sz(1), sz(0), g, lo, 4, C.byref(nl), seg, None) == -1
    assert L.b2c_debug_sumsq_plan(1, sz(0), sz(1), sz(0), g, lo, 0, C.byref(nl), seg, C.byref(npart)) == -1


@pytest.mark.parametrize("value,clips", [("1.5", True), ("0", True), ("1e30", True), ("-1", False), ("-0.5", False), (None, False)])
def test_solver_files_with_clip_gradients_parse(value, clips):
    text = 'net: "n.prototxt" base_lr: 0.01 lr_policy: "fixed" momentum: 0.9 max_iter: 10 type: "Adam"'
    if value is not None:
        text += " clip_gradients: " + value
    s, net = host_api.open_solver(text, is_text=True)
    assert net == "n.prototxt"
    with pytest.raises(host_api.HostError, match="has no parameters yet" if clips else "does not clip"):
        s.clip_state()
    assert float(host_api.textproto_scalar(text, "clip_gradients", -1.0, is_text=True)) == (float(value) if value else -1.0)


def test_clip_gradients_is_set_before_the_parameters():
    s = host_api.SGDSolver(clip_gradients=2.0)
    with pytest.raises(host_api.HostError, match="has no parameters yet"):
        s.clip_state()
    with pytest.raises(host_api.HostError, match="does not clip"):
        host_api.SGDSolver().clip_state()
