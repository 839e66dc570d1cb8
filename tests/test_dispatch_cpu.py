"""Host dispatch is pinned: for every shape of tests/golden/make_dispatch_golden.py's sweep, under every switch setting, the
kernel family, workspace and filter-cache sizes and the weight-gradient route and split-K plan equal
tests/golden/dispatch_golden.json, and the forward and data-gradient routes and tile plans equal
tests/golden/conv_plan_golden.json.  These are host-only queries: no GPU is used."""
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_dispatch_golden as mdg  # noqa: E402


@pytest.fixture(scope="module")
def golden():
    with open(mdg.GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name,env", mdg.SETTINGS, ids=[n for n, _ in mdg.SETTINGS])
def test_dispatch_matches_golden(golden, name, env):
    want = dict(golden["default"])
    if name != "default":
        want.update(golden["overrides"][name])
    got = mdg.run_setting(env)
    assert got.keys() == want.keys()
    bad = [k for k in want if got[k] != want[k]]
    assert not bad, f"{len(bad)} shapes differ under {name}; first {bad[0]}: got {got[bad[0]]}, want {want[bad[0]]}"


@pytest.mark.parametrize("name,env", mdg.PLAN_SETTINGS, ids=[n for n, _ in mdg.PLAN_SETTINGS])
def test_conv_plans_match_golden(name, env):
    with open(mdg.PLAN_GOLDEN) as f:
        golden = json.load(f)
    want = list(golden["default"])
    for i, v in golden["overrides"].get(name, {}).items():
        want[int(i)] = v
    got = mdg.run_setting(env, "--plans")
    assert len(got) == len(want)
    bad = [i for i in range(len(want)) if got[i] != want[i]]
    keys = mdg.shapes()
    assert not bad, f"{len(bad)} shapes differ under {name}; first {keys[bad[0]]}: got {got[bad[0]]}, want {want[bad[0]]}"
