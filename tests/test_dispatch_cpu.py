"""Host dispatch is pinned: for every shape of tests/golden/make_dispatch_golden.py's sweep, under every switch setting, the
kernel family, workspace and filter-cache sizes and the weight-gradient route and split-K plan equal
tests/golden/dispatch_golden.json.  These are host-only queries: no GPU is used."""
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
