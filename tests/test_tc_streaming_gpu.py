"""64-row tiles for m-tiles of <= 64 GEMM rows (csrc/igemm_tc.cu, tc_plan): at batch 1 every 7 x 7 layer-4 launch of ResNet-18
stages a 64-pixel im2col box instead of a 128-pixel one whose upper 79 rows lie past the end of the tensor, and the launches that are
one wave or less and walk >= 16 k-blocks per CTA spend the freed shared memory on an 8-deep ring.  Every output element keeps its
k-ranges, MMA instruction sequence and cluster reduction order, so the results must be bitwise those of 128-row tiles
(BRE_TC_STREAM=0, read once per process, hence a subprocess) and within the GEMM bound of float64."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import test_tc_narrow_tiles_gpu as narrow  # noqa: E402
from profile_gemms import ring_plan, split_plan  # noqa: E402

U = 2.0 ** -23

# (label, mode, (N, H, W, Ci, Co, R, stride, pad), nsrc): mode 0 fprop, 1 dgrad
CASES = [
    ("layer4 fprop", 0, (1, 7, 7, 512, 512, 3, 1, 1), 1),            # 128 x 64 -> 64 x 64, 8 stages
    ("layer4 tangent fprop", 0, (1, 7, 7, 512, 512, 3, 1, 1), 2),
    ("layer4 dgrad", 1, (1, 7, 7, 512, 512, 3, 1, 1), 1),            # 128 x 32 -> 64 x 32, 8 stages, 64-slot cluster reduction
    ("layer4 tangent dgrad", 1, (1, 7, 7, 512, 512, 3, 1, 1), 2),
    ("layer4.0 fprop, stride 2", 0, (1, 14, 14, 256, 512, 3, 2, 1), 1),   # 9 k-blocks per CTA: 64 rows, 4 stages
    ("2 x 4 x 4 fprop", 0, (2, 4, 4, 64, 128, 3, 1, 1), 1),          # M = 32 over two images
    ("2 x 4 x 4 dgrad, dual source", 1, (2, 4, 4, 128, 64, 3, 1, 1), 2),
    ("8 x 8 fprop, 96 wide", 0, (1, 8, 8, 96, 96, 1, 1, 0), 2),       # M = 64 exactly, 64 x 32 tiles (width not a multiple of 64)
]


def results():
    return {label: narrow.launch(mode, geom, nsrc, narrow.operands(mode, geom, nsrc)).cpu() for label, mode, geom, nsrc in CASES}


@pytest.mark.parametrize("label,mode,geom,nsrc", CASES, ids=[c[0] for c in CASES])
def test_matches_float64_within_the_gemm_bound(label, mode, geom, nsrc):
    _, bn, splits, kb = split_plan(mode, geom, nsrc)
    bm, stages = ring_plan(mode, geom, nsrc)
    assert bm == 64, (bm, stages)
    ops = narrow.operands(mode, geom, nsrc)
    out = narrow.launch(mode, geom, nsrc, ops).double()
    ref, mag = narrow.reference(mode, geom, nsrc, ops), narrow.reference(mode, geom, nsrc, ops, absolute=True)
    N, H, W, Ci, Co, R, st, pd = geom
    K = {0: R * R * Ci, 1: R * R * Co}[mode] * nsrc
    ratio = ((out - ref).abs() / ((K + 2) * U * mag).clamp_min(1e-300)).max().item()
    print(f"{label}: {bm} x {bn} tiles, {stages} stages, split {splits}, {kb} k-blocks per CTA, max |err| / bound = {ratio:.3g}")
    assert torch.isfinite(out).all() and ratio <= 1.0, ratio
    assert torch.equal(narrow.launch(mode, geom, nsrc, ops).double(), out)   # run to run


def test_layer4_plan():
    """The config-2 layer-4 launches keep their tile width and split and take the 8-deep ring."""
    for mode, nsrc, bn in ((0, 1, 64), (0, 2, 64), (1, 1, 32), (1, 2, 32)):
        g = (1, 7, 7, 512, 512, 3, 1, 1)
        _, width, splits, kb = split_plan(mode, g, nsrc)
        assert (width, splits, kb) == (bn, 8, 18 * nsrc) and ring_plan(mode, g, nsrc) == (64, 8)
    assert ring_plan(0, (1, 14, 14, 256, 256, 3, 1, 1), 1) == (128, 4)   # layer 3 (M = 196) is left alone


def in_subprocess(func, env, tmp_path):
    path = str(tmp_path / f"{func}.pt")
    code = (f"import sys, torch; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'tests')!r}]; import test_tc_streaming_gpu as t; "
            f"torch.save(t.{func}(), {path!r})")
    res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    return torch.load(path)


def test_streaming_tiles_are_bitwise_the_128_row_result(tmp_path):
    wide, rows64 = in_subprocess("results", {"BRE_TC_STREAM": "0"}, tmp_path), results()
    for label in wide:
        assert torch.equal(wide[label], rows64[label]), label


def engine_outputs():
    """Candidate, best-so-far and objective history after a few iterations of config 2 (ResNet-18, 224 x 224, batch 1) and of
    config 4 (FedAvg: the local steps rewrite the weights, so no weight load is issued ahead of the dependency wait)."""
    import bench

    torch.manual_seed(0)
    out = {}
    for config in (2, 4):
        runner = bench.EngineRunner(config, bench.build_case(config), torch.device("cuda:0"), "tc", 0)
        runner.warm(4)
        out.update({f"config {config} {k}": torch.from_numpy(v) for k, v in runner.outputs().items()})
        runner.eng.close()
    return out


def test_engine_iterations_are_bitwise_the_128_row_result(tmp_path):
    wide, rows64 = in_subprocess("engine_outputs", {"BRE_TC_STREAM": "0"}, tmp_path), engine_outputs()
    assert wide.keys() == rows64.keys()
    for k in wide:
        assert torch.equal(wide[k], rows64[k]), k
