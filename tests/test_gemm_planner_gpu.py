"""The launch planner of the GEMM back ends (engine.gemm_plan: plan_gemm / tc_plan in the library) against its restatement
(scripts/profile_gemms.py gemm_plan) on backends 0, 1 and 2, for fprop / dgrad / wgrad with one and two sources, over a dense grid of
geometries: once at the default switches and once per non-default setting of a switch the plans depend on (the library reads them
once per process, hence a subprocess each).  Nothing is launched; the GPU is needed for the driver's tensor-map entry points, which
decide whether the TMA producers exist."""
import itertools
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

import profile_gemms as P  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402

BATCH = (1, 2, 8, 32)
SPATIAL = (1, 2, 3, 7, 14, 28, 56)
CHANNELS = (3, 4, 16, 32, 64, 96, 128, 512, 2048)
FILTERS = (1, 3, 7)
STRIDES = (1, 2, 3, 10)
SETTINGS = [{"BRE_TC_TMA": "0"}, {"BRE_TC_NARROW": "0"}, {"BRE_TC_STREAM": "0"}, {"BRE_TC_STAGES": "8"}, {"BRE_TC_MAX_SPLITS": "2"},
            {"BRE_LINEAR_SMALL": "0", "BRE_LINEAR_SMALL_ROWS": "1"}]


def geometries():
    """(N, H, W, Ci, Co, R, stride, pad): convolutions with no and with 'same' padding, and linear layers on 1-32 rows up to the token
    decoder's 50304 outputs."""
    for N, H, Ci, Co, R, st in itertools.product(BATCH, SPATIAL, CHANNELS, CHANNELS, FILTERS, STRIDES):
        for pd in sorted({0, R // 2}):
            if H + 2 * pd >= R:
                yield (N, H, H, Ci, Co, R, st, pd)
    for N, Ci, Co in itertools.product(range(1, 33), CHANNELS, CHANNELS + (50304,)):
        yield (N, 1, 1, Ci, Co, 1, 1, 0)


def mismatches():
    """[(mode, geometry, nsrc, backend, library plan, restated plan)] over the whole grid, and the number of plans compared."""
    bad, n = [], 0
    for g in geometries():
        N, H, W, Ci, Co, R, st, pd = g
        for mode, nsrc, backend in itertools.product(range(3), (1, 2), range(3)):
            got = E.gemm_plan(mode, backend, N, H, W, Ci, Co, R, R, st, pd, nsrc)
            want = P.gemm_plan(mode, g, nsrc, backend)
            n += 1
            if not (got["family"] is None if want is None else got == want):   # None: backend 1 refuses the shape
                bad.append((mode, g, nsrc, backend, got, want))
    return bad, n


def report(bad, n):
    for row in bad[:20]:
        print(row)
    assert n > 10 ** 5, n
    assert not bad, f"{len(bad)} of {n} plans differ"


def test_planner_matches_the_restatement_at_the_defaults():
    for name in ("BRE_TC_TMA", "BRE_TC_NARROW", "BRE_TC_STRIDED_TMA", "BRE_TC_STREAM", "BRE_TC_STAGES", "BRE_TC_SHORTK_STAGES",
                 "BRE_TC_MAX_SPLITS", "BRE_TC_TARGET_CTAS", "BRE_LINEAR_SMALL", "BRE_LINEAR_SMALL_ROWS", "BRE_LINEAR_TALL"):
        assert name not in os.environ, name
    report(*mismatches())


@pytest.mark.parametrize("env", SETTINGS, ids=[",".join(f"{k}={v}" for k, v in s.items()) for s in SETTINGS])
def test_planner_matches_the_restatement_under_a_switch(env, tmp_path):
    path = str(tmp_path / "planner.json")
    code = (f"import sys, json; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_gemm_planner_gpu as t; "
            f"json.dump(t.mismatches(), open({path!r}, 'w'))")
    res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    with open(path) as f:
        report(*json.load(f))
