"""The GEMM launch-plan table (tests/gemm_plan_cases.py) against the restatement of the launch rules (scripts/profile_gemms.py): every
case's plan is the one the rules give, the table holds every shape it is built from, and it reaches every plan the launchers can
choose.  No GPU needed; tests/test_gemm_plans_gpu.py checks the same plans against what the launchers record."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import gemm_plan_cases as T  # noqa: E402
import profile_gemms as P  # noqa: E402

PLAN_ENV = ("BRE_TC_TMA", "BRE_TC_NARROW", "BRE_TC_STRIDED_TMA", "BRE_TC_STREAM", "BRE_TC_STAGES", "BRE_TC_SHORTK_STAGES", "BRE_TC_MAX_SPLITS",
            "BRE_LINEAR_SMALL", "BRE_LINEAR_SMALL_ROWS", "BRE_LINEAR_TALL")


@pytest.fixture(autouse=True)
def default_rules(monkeypatch):
    for name in PLAN_ENV:
        monkeypatch.delenv(name, raising=False)


@pytest.mark.parametrize("case", T.CASES, ids=[T.label(c) for c in T.CASES])
def test_table_plan_is_the_restated_plan(case):
    mode, geom, nsrc, backend, _ = case
    assert P.gemm_plan(mode, geom, nsrc, backend) == T.plan(case)


def test_table_holds_every_shape_it_is_built_from():
    keys = [(mode, geom, nsrc, backend) for mode, geom, nsrc, backend, _ in T.CASES]
    assert len(keys) == len(set(keys))
    want = [(m, g, nsrc, b) for m, g, b in T.shape_list() for nsrc in (1, 2) if P.gemm_plan(m, g, nsrc, b) is not None]
    assert sorted(set(want)) == sorted(keys)


def test_table_reaches_every_plan():
    covered = set()
    for case in T.CASES:
        covered |= T.features(case)
    for fam, mode, nsrc, prop in sorted(covered, key=str):
        print(f"{fam:15s} {T.MODES[mode]} nsrc {nsrc}: {prop}")
    missing = T.required() - covered
    assert not missing, sorted(missing, key=str)


def test_64_row_tiles_need_the_tma_producer():
    """A fprop of M <= 64 that no tensor map covers (stride 10) runs 128-row cp.async tiles, as tc_plan decides."""
    g = (1, 20, 20, 64, 64, 1, 10, 0)
    assert P.gemm_shape(0, g)[0] == 4
    assert P.ring_plan(0, g, 1) == (128, 4)
    assert P.tc_plan(0, g, 1)["producer"] == "cp.async"
    assert P.ring_plan(0, (1, 20, 20, 64, 64, 1, 8, 0), 1) == (64, 4)   # stride 8: still a tensor map


def test_tma_switch_is_honoured(monkeypatch):
    """BRE_TC_TMA=0: every contraction on the cp.async producer with 128 x 64 tiles; widths that are only a multiple of 32 are refused."""
    monkeypatch.setenv("BRE_TC_TMA", "0")
    for case in T.CASES:
        mode, geom, nsrc, backend, _ = case
        if backend != 1:
            continue
        p = P.gemm_plan(mode, geom, nsrc, 1)
        if T.gemm_dims(mode, geom)[1] % 64:
            assert p is None, T.label(case)
        else:
            assert (p["producer"], p["tile_rows"], p["tile_width"]) == ("cp.async", 128, 64), T.label(case)
