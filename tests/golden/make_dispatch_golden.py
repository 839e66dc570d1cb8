"""Pin the host-side convolution dispatch: which kernel family each op takes, the workspace and filter-cache sizes it asks
for, and the weight-gradient route with its split-K plan (b2c_debug_wgrad_plan); and, in a file of their own, the forward
and data-gradient routes with their tile plans (b2c_debug_conv_plan).  All of these are host-only queries of libb2c.so, so
they are answered without a GPU; the device is hidden from the process, so sm_count() takes its no-device value of 132 (the
SM count of an H100 SXM) and the split plans and grids are those of that card.

The switches are read once per process, so each setting is swept in a subprocess of its own.

    python tests/golden/make_dispatch_golden.py          writes tests/golden/dispatch_golden.json and conv_plan_golden.json
    python tests/golden/make_dispatch_golden.py --one    prints the sweep of this process's environment as JSON
    python tests/golden/make_dispatch_golden.py --plans  prints the conv plan sweep of this process's environment as JSON

tests/test_dispatch_cpu.py replays the sweeps and compares them with the files."""
import ctypes as C
import itertools
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
GOLDEN = os.path.join(ROOT, "tests", "golden", "dispatch_golden.json")
PLAN_GOLDEN = os.path.join(ROOT, "tests", "golden", "conv_plan_golden.json")

# (name, environment additions); "default" sets nothing
SETTINGS = [
    ("default", {}),
    ("conv_staged_0", {"B2C_CONV_STAGED": "0"}),
    ("conv_staged_plane_0", {"B2C_CONV_STAGED_PLANE": "0"}),
    ("wgrad_staged_0", {"B2C_WGRAD_STAGED": "0"}),
    ("wgrad_staged_plane_0", {"B2C_WGRAD_STAGED_PLANE": "0"}),
    ("wgrad_tma_0", {"B2C_WGRAD_TMA": "0"}),
    ("wgrad_compact_0", {"B2C_WGRAD_COMPACT": "0"}),
    ("wgrad_compact_2", {"B2C_WGRAD_COMPACT": "2"}),
]
SWITCHES = sorted({k for _, env in SETTINGS for k in env})
# the settings whose switches the forward / data-gradient planners read
PLAN_SETTINGS = [s for s in SETTINGS if s[0] in ("default", "conv_staged_0", "conv_staged_plane_0")]

ENGINES = (0, 1)     # DEFAULT, CAFFE
MATHS = (0, 1, 2)    # FP32, TF32, FP32_3XTF32
ALGOS = (0, 1)       # AUTO, SIMT


def shapes():
    """[(N, C, H, W, O, G, kh, kw, sh, sw, ph, pw, dh, dw, bias)]: tests/cases.py's lists, then a grid over the edges of
    each kernel's eligibility (H*W of 36 / 49 / 64 / 128+, C % 4 and C % 32, k of 1 / 3 / 5 / 7, stride 1 / 2, groups 1 / 2,
    O up to and past 128)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from cases import ALL_CASES, FULL_SIZE_CASES

    def pair(v):
        return (v, v) if isinstance(v, int) else tuple(v)

    out = []
    for _, c in ALL_CASES + FULL_SIZE_CASES:
        kh, kw = pair(c["k"])
        sh, sw = pair(c["s"])
        ph, pw = pair(c["p"])
        dh, dw = pair(c["d"])
        out.append((c["N"], c["Cin"], c["H"], c["W"], c["O"], c["G"], kh, kw, sh, sw, ph, pw, dh, dw, int(c["bias"])))
    for (H, W), Cin, k, s, G, O in itertools.product(((6, 6), (7, 7), (8, 8), (12, 11), (14, 14), (56, 56)), (30, 32, 36, 96),
                                                      (1, 3, 5, 7), (1, 2), (1, 2), (64, 192)):
        out.append((16, Cin, H, W, O, G, k, k, s, s, k // 2, k // 2, 1, 1, 0))
    return out


def packed(rows):
    """[index string, distinct rows...]: character i of the index string names the distinct row of combination i (most
    shapes answer alike for several combinations; this keeps the file small)."""
    distinct, idx = [], ""
    for r in rows:
        if r not in distinct:
            distinct.append(r)
        idx += str(distinct.index(r))
    return [idx] + distinct


def sweep():
    """{shape key: packed rows, one row per (engine, math, algo)} for the switches of this process's environment.  A row is
    algo_used x 3 ops, workspace_bytes x 3 ops, filter_cache_bytes, then the six b2c_debug_wgrad_plan values."""
    sys.path.insert(0, ROOT)
    from caffe_mpi_b200 import capi
    L = capi.lib()
    L.b2c_conv_filter_cache_bytes.restype = C.c_size_t
    L.b2c_conv_filter_cache_bytes.argtypes = [C.c_void_p]
    res = {}
    plan = (C.c_int * 6)()
    for shp in shapes():
        prm = capi.ConvParams(*shp)
        rows = []
        for eng, math, algo in itertools.product(ENGINES, MATHS, ALGOS):
            h = C.c_void_p()
            capi.check(L.b2c_conv_desc_create(C.byref(prm), eng, C.byref(h)))
            try:
                capi.check(L.b2c_conv_desc_set_math(h, math))
                capi.check(L.b2c_conv_desc_set_algo(h, algo))
                row = [int(L.b2c_conv_algo_used(h, op)) for op in range(3)]
                row += [int(L.b2c_conv_workspace_bytes(h, op)) for op in range(3)]
                row.append(int(L.b2c_conv_filter_cache_bytes(h)))
                capi.check(L.b2c_debug_wgrad_plan(h, plan, 6))
                row += list(plan)
            finally:
                L.b2c_conv_desc_destroy(h)
            rows.append(row)
        res[",".join(map(str, shp))] = packed(rows)
    return res


def plan_sweep():
    """[one string per shape of shapes(), in order] for the switches of this process's environment: the eight
    b2c_debug_conv_plan values of the forward, then of the data gradient, in the FP32 math mode of engine DEFAULT / algo
    AUTO; then "|" and the same in TF32 where that differs.  The other combinations answer by rule, checked here: engine
    CAFFE reports the CAFFE route, algo SIMT the SIMT route (all other values 0), and FP32_3XTF32 reports what TF32 does."""
    sys.path.insert(0, ROOT)
    from caffe_mpi_b200 import capi
    L = capi.lib()
    out = (C.c_int * 8)()
    res = []
    for shp in shapes():
        prm = capi.ConvParams(*shp)
        plans = {}
        for eng, math, algo in itertools.product(ENGINES, MATHS, ALGOS):
            h = C.c_void_p()
            capi.check(L.b2c_conv_desc_create(C.byref(prm), eng, C.byref(h)))
            try:
                capi.check(L.b2c_conv_desc_set_math(h, math))
                capi.check(L.b2c_conv_desc_set_algo(h, algo))
                row = []
                for op in (0, 1):
                    capi.check(L.b2c_debug_conv_plan(h, op, out, 8))
                    row += list(out)
            finally:
                L.b2c_conv_desc_destroy(h)
            plans[eng, math, algo] = ".".join(map(str, row))
        for (eng, math, algo), p in plans.items():
            if eng == 1 or algo == 1:                        # route CAFFE (0) or SIMT (1), the plan all zeros, for both ops
                one = ".".join([str(0 if eng == 1 else 1)] + ["0"] * 7)
                assert p == one + "." + one, (shp, eng, math, algo, p)
        assert plans[0, 2, 0] == plans[0, 1, 0], (shp, plans[0, 2, 0], plans[0, 1, 0])
        fp32, tf32 = plans[0, 0, 0], plans[0, 1, 0]
        res.append(fp32 if tf32 == fp32 else fp32 + "|" + tf32)
    return res


def run_setting(env_add, mode="--one"):
    """sweep() (or plan_sweep() with mode "--plans") in a fresh process with the switches set as `env_add` says (every other
    switch unset, B2C_NTILE too) and no visible GPU."""
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES and k != "B2C_NTILE"}
    env.update(env_add)
    env["CUDA_VISIBLE_DEVICES"] = ""
    out = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=env, capture_output=True, text=True,
                         check=True).stdout
    return json.loads(out.strip().splitlines()[-1])


def collect():
    """{"default": sweep, "overrides": {setting: {shape key: rows that differ from the default}}}"""
    base = run_setting({})
    over = {}
    for name, env in SETTINGS[1:]:
        got = run_setting(env)
        assert got.keys() == base.keys(), name
        over[name] = {k: v for k, v in got.items() if v != base[k]}
    return {"default": base, "overrides": over}


def collect_plans():
    """{"default": plan_sweep, "overrides": {setting: {shape index: plans that differ from the default}}}"""
    base = run_setting({}, "--plans")
    over = {}
    for name, env in PLAN_SETTINGS[1:]:
        got = run_setting(env, "--plans")
        assert len(got) == len(base), name
        over[name] = {str(i): v for i, v in enumerate(got) if v != base[i]}
    return {"default": base, "overrides": over}


def main():
    if "--one" in sys.argv:
        print(json.dumps(sweep(), separators=(",", ":")))
        return
    if "--plans" in sys.argv:
        print(json.dumps(plan_sweep(), separators=(",", ":")))
        return
    with open(GOLDEN, "w") as f:
        json.dump(collect(), f, separators=(",", ":"))
        f.write("\n")
    with open(PLAN_GOLDEN, "w") as f:
        json.dump(collect_plans(), f, separators=(",", ":"))
        f.write("\n")


if __name__ == "__main__":
    main()
