"""Non-default kernel selections (DESIGN.md "Switches"): every eligible strided 1x1 weight gradient through the compaction
path, the gather weight-gradient kernel instead of the TMA one, the gather forward / dgrad kernel instead of the staged one, the
BatchNorm launch variants, and the TrainNet fusions of the residual tail turned off.  Skipped unless B2C_RUN_EXPERIMENTAL=1; each
runs, in a subprocess with the switch set (switches are read once per process), the tests that reach what it switches: the conv
parity cases, the BatchNorm regime cases (whose plan assertions follow the switch), or the TrainNet cases."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONV = ("test_gpu_parity.py", "s2 or 1x1 or 3x3 or 5x5 or full_size")
BN = ("test_bn_schedule_gpu.py", "bn_case or variance")
TRAINER = ("test_trainer_gpu.py", "fusion or forward_backward")
TARGET = {"B2C_WGRAD_COMPACT=2": CONV, "B2C_WGRAD_TMA=0": CONV, "B2C_CONV_STAGED=0": CONV, "B2C_CONV_STAGED_PLANE=0": CONV,
          "B2C_WGRAD_STAGED=0": CONV, "B2C_WGRAD_STAGED_PLANE=0": CONV, "B2C_BN_CLUSTER=16": BN, "B2C_FUSE_SPLIT=0": TRAINER,
          "B2C_BN_ONEPASS=0": BN, "B2C_BN_PREFETCH=0": BN, "B2C_BN_PREFETCH_BWD=0": BN, "B2C_BN_CACHE_KB=0": BN, "B2C_FUSE_RES=0": TRAINER}


@pytest.mark.skipif(os.environ.get("B2C_RUN_EXPERIMENTAL") != "1", reason="experimental variants run only on request")
@pytest.mark.parametrize("switch", list(TARGET))
def test_variant_passes_the_parity_cases(switch):
    name, val = switch.split("=")
    env = dict(os.environ, **{name: val})
    env.pop("B2C_RUN_EXPERIMENTAL")
    test, sel = TARGET[switch]
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", test), "-m", "gpu", "-q", "-x", "-rs", "-k", sel],
                       env=env, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:]
    if TARGET[switch] is BN:                                # every regime case ran under the switch, none skipped
        skipped = [ln for ln in r.stdout.splitlines() if ln.startswith("SKIPPED")]
        assert " passed" in r.stdout and not skipped, (skipped, r.stdout[-500:])
