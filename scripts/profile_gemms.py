#!/usr/bin/env python
"""Per-launch profile of the conv / linear GEMMs of one config-2 iteration (ResNet-18, 224x224, batch 1, tensor-core back end).

    python scripts/profile_gemms.py --out DIR [--repeats 200]

1. Every GEMM launch of one iteration (per layer: fprop, wgrad, dgrad, dual-source tangent fprop, dual-source tangent dgrad --
   the list bench.py's GEMM-family roofline replays) is issued through the C ABI (`bre_conv_gemm`, the engine's dispatch rule),
   captured `--repeats` times back to back into one CUDA graph and timed with CUDA events over the replay, after a warm-up
   replay.  Printed per launch: GEMM M x N x K, output tiles and their width, split-K factor, k-blocks per CTA, us.
2. One torch.profiler trace of the engine's captured iteration (a few iterations of the real trial), reduced to a per-kernel
   table (launches, total and mean device time per iteration).

Both tables go to DIR/gemm_launches.json and DIR/iteration_kernels.json.  The split plan is computed here from the shapes by
the same rules as tc_plan in breaching_b200/csrc/igemm_tc.cu (honouring BRE_TC_MAX_SPLITS); it is a label of the rows, the times are
measured.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NUM_SMS, BM, BK, MAX_CLUSTER = 132, 128, 32, 8


def gemm_shape(mode, g):
    N, H, W, Ci, Co, R, st, pd = g
    Ho, Wo = (H + 2 * pd - R) // st + 1, (W + 2 * pd - R) // st + 1
    if mode == 0:
        return N * Ho * Wo, Co, R * R * Ci
    if mode == 1:
        return N * H * W, Ci, R * R * Co
    return Co, R * R * Ci, N * Ho * Wo


def _env(name, default):
    return int(os.environ.get(name, str(default)))


def tma_ok(mode, g):
    """tma_eligible in igemm_tc.cu: the TMA producer covers this contraction (BRE_TC_TMA=0 turns it off everywhere)."""
    N, H, W, Ci, Co, R, st, pd = g
    if not _env("BRE_TC_TMA", 1) or st > 8 or pd > 127 or R - 1 - pd > 127 or R > 128:
        return False
    if mode == 1:
        return st == 1
    if mode == 2:
        return Ci % 32 == 0
    return True


def narrow_ok(mode, g):
    """narrow_tiles_ok in igemm_tc.cu: 128 x 32 / 64 x 32 tiles exist for the TMA producer of fprop, stride-1 dgrad and wgrad."""
    return bool(_env("BRE_TC_NARROW", 1)) and tma_ok(mode, g)


def classes_ok(mode, g):
    """cls_eligible in igemm_tc.cu (stride-2 dgrad as per-parity-class TMA gathers; the tap-corner range check never binds here)."""
    N, H, W, Ci, Co, R, st, pd = g
    return mode == 1 and st == 2 and bool(_env("BRE_TC_STRIDED_TMA", 1)) and bool(_env("BRE_TC_TMA", 1)) and R <= 16


def tc_supported(mode, g):
    """igemm_tc_supported in igemm_tc.cu for NHWC / OHWI operands on 16-byte aligned buffers."""
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    if Nc % 64 != 0 and not (Nc % 32 == 0 and narrow_ok(mode, g)):
        return False
    if R * R > 64:
        return False
    return {0: Ci % BK == 0, 1: Co % BK == 0, 2: Co % 4 == 0 and Ci % 4 == 0}[mode]


def _tc_split(mode, g, nsrc):
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    kb = -(-K // BK) * nsrc
    tm = -(-M // BM)
    cls = classes_ok(mode, g)
    if cls:   # strided dgrad: one m-tile range per parity class, k extent of the largest class
        tm, kmax = 0, 0
        for ey in range(2):
            for ex in range(2):
                y0, x0 = (ey - pd) % 2, (ex - pd) % 2
                if y0 >= H or x0 >= W:
                    continue
                hc, wc = -(-(H - y0) // 2), -(-(W - x0) // 2)
                tm += -(-(N * hc * wc) // BM)
                ty = -(-(R - ey) // 2) if ey < R else 0
                tx = -(-(R - ex) // 2) if ex < R else 0
                kmax = max(kmax, ty * tx)
        kb = max(kmax * (Co // BK) * nsrc, 1)
    underfilled = mode != 0 and not cls and Nc % 64 == 0 and tm * (Nc // 64) * 16 <= NUM_SMS and kb >= 64 and narrow_ok(mode, g)
    bn = 32 if Nc % 64 != 0 or underfilled else 64
    tiles = tm * (Nc // bn)
    splits = 1
    while splits < MAX_CLUSTER and tiles * splits < NUM_SMS and kb // (splits * 2) >= 2:
        splits *= 2
    cap = _env("BRE_TC_MAX_SPLITS", 0)
    if cap > 0:
        splits = min(splits, cap)
    p = 1
    while p * 2 <= splits and p < MAX_CLUSTER:
        p *= 2
    splits = p
    while splits > 1 and splits > kb:
        splits //= 2
    return tiles, bn, splits, -(-kb // splits), kb, cls


def split_plan(mode, g, nsrc):
    """(tiles, tile width, split-K factor, k-blocks per CTA) as tc_plan in igemm_tc.cu chooses them."""
    return _tc_split(mode, g, nsrc)[:4]


def ring_plan(mode, g, nsrc):
    """(tile rows, ring depth) as tc_plan in igemm_tc.cu chooses them (honouring BRE_TC_STREAM and BRE_TC_STAGES)."""
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    tiles, bn, splits, kbc = split_plan(mode, g, nsrc)
    # 64-row tiles are im2col boxes of the TMA producer: a fprop the producer does not cover (stride > 8) keeps 128-row cp.async tiles
    bm = 64 if _env("BRE_TC_STREAM", 1) and M <= 64 and mode in (0, 1) and tma_ok(mode, g) else BM
    shortk = _env("BRE_TC_SHORTK_STAGES", 2) == 2 and kbc <= 6 and tiles == Nc // bn and tiles * splits > 2 * NUM_SMS
    deep = bm == 64 and tiles * splits <= NUM_SMS and kbc >= 16
    forced = _env("BRE_TC_STAGES", 0)
    return bm, forced if forced in (2, 4, 8) else (2 if shortk else 8 if deep else 4)


def tc_plan(mode, g, nsrc):
    """The whole tensor-core launch plan (tc_plan in igemm_tc.cu), in the form engine.last_gemm_plan() reports it."""
    tiles, bn, splits, kbc, kb, cls = _tc_split(mode, g, nsrc)
    bm, stages = ring_plan(mode, g, nsrc)
    producer = "classes" if cls else "tma" if bm == 64 or bn == 32 or tma_ok(mode, g) else "cp.async"
    return dict(family="tc", mode=mode, nsrc=nsrc, tile_rows=bm, tile_width=bn, splits=splits, stages=stages, producer=producer,
                total_kblocks=kb, kblocks_per_split=kbc, vec=0)


SIMT_BM, SIMT_BN, SIMT_BK, SIMT_WS_TILES, SC_PX, SC_KCH = 64, 64, 16, 1024, 4, 4


def _linear(g):
    N, H, W, Ci, Co, R, st, pd = g
    return R == 1 and H == 1 and W == 1 and st == 1 and pd == 0


def linear_tall_ok(mode, g, nsrc):
    """linear_tall_supported in linear_small.cu (with bre_conv_gemm's 1024-tile workspace)."""
    N, H, W, Ci, Co, R, st, pd = g
    if not _env("BRE_LINEAR_TALL", 1) or mode != 1 or not _linear(g) or not 1 <= N <= 32 or Ci % 32 or Ci > 128 or Co < 8192:
        return False
    return -(-Co // _tall_chunk(Co)) * 32 * Ci <= SIMT_WS_TILES * SIMT_BM * SIMT_BN


def _tall_chunk(Co):
    c = -(-Co // (4 * NUM_SMS))
    c += c & 1
    return min(max(c, 32), 96)


def linear_small_preferred(mode, g, nsrc):
    N, H, W, Ci, Co, R, st, pd = g
    if not _env("BRE_LINEAR_SMALL_ROWS", 0) or mode == 2 or not (_linear(g) and 1 <= N <= 32):
        return False
    return (Ci if mode == 0 else Co) * nsrc <= 512


def linear_small_plan(mode, g, nsrc):
    """linear_small_plan in linear_small.cu for 16-byte aligned operands."""
    N, H, W, Ci, Co, R, st, pd = g
    nb = next(b for b in (1, 2, 4, 8, 16, 32) if N <= b)
    return dict(family="linear_small", mode=mode, nsrc=nsrc, tile_rows=nb, tile_width=0, splits=1, stages=0, producer=None, total_kblocks=0,
                kblocks_per_split=0, vec=int(mode == 0 and Ci % 4 == 0))


def simt_plan(mode, g, nsrc):
    """The fp32 kernels of plan_gemm in igemm_simt.cu (linear_small / dgrad_small_ci / the SIMT implicit GEMM) for NHWC / OHWI operands
    on 16-byte aligned buffers, in the form engine.last_gemm_plan() reports it."""
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    base = dict(mode=mode, nsrc=nsrc, tile_rows=0, tile_width=0, splits=1, stages=0, producer=None, total_kblocks=0, kblocks_per_split=0,
                vec=0)
    if _env("BRE_LINEAR_SMALL", 1) and _linear(g) and 1 <= N <= 16:
        return linear_small_plan(mode, g, nsrc)
    if mode == 1 and Ci <= 4 and Co <= 16 * SC_KCH and nsrc * -(-R // st) * R * Co * Ci * 4 <= 200 * 1024:
        return dict(base, family="dgrad_small_ci", tile_rows=32 * SC_PX, tile_width=Ci, vec=int(Co % 4 == 0))
    total = -(-K // SIMT_BK) * nsrc
    x_vec = Ci % 4 == 0
    vec_a, vec_b, vec_out = {0: (x_vec, K % 4 == 0, Nc % 4 == 0), 1: (Co % 4 == 0, Ci % 4 == 0, x_vec),
                             2: (Co % 4 == 0, x_vec, Nc % 4 == 0)}[mode]
    tiles = -(-M // SIMT_BM) * -(-Nc // SIMT_BN)
    splits = 1
    if tiles < 2 * NUM_SMS:
        splits = min(-(-2 * NUM_SMS // tiles), max(total // 4, 1))
    splits = min(splits, total)
    if splits > 1 and tiles * splits > SIMT_WS_TILES:
        splits = max(SIMT_WS_TILES // tiles, 1)
    per = -(-total // splits)
    return dict(base, family="igemm_simt", tile_rows=SIMT_BM, tile_width=SIMT_BN, splits=-(-total // per), stages=2, total_kblocks=total,
                kblocks_per_split=per, vec=int(vec_a) | 2 * int(vec_b) | 4 * int(vec_out))


def gemm_plan(mode, g, nsrc, backend):
    """plan_gemm in igemm_simt.cu: the plan bre_conv_gemm launches for `backend` (0 SIMT, 1 tensor cores, 2 the engine's dispatch), None
    if it refuses the shape.  Family order: linear_tall, linear_small where preferred (not on backend 1), the tensor cores where they
    cover the shape (not on backend 0), then the fp32 kernels."""
    if linear_tall_ok(mode, g, nsrc):
        N, H, W, Ci, Co, R, st, pd = g
        chunk = _tall_chunk(Co)
        return dict(family="linear_tall", mode=mode, nsrc=nsrc, tile_rows=32, tile_width=Ci, splits=-(-Co // chunk), stages=0, producer=None,
                    total_kblocks=Co, kblocks_per_split=chunk, vec=0)
    if backend != 1 and linear_small_preferred(mode, g, nsrc):
        return linear_small_plan(mode, g, nsrc)
    if backend != 0 and tc_supported(mode, g):
        return tc_plan(mode, g, nsrc)
    if backend == 1:
        return None
    return simt_plan(mode, g, nsrc)


def launches_of(prog, dev):
    """(label, mode, geometry, nsrc, thunk, keep-alive tensors) for every GEMM launch of one iteration, in bench.py's order."""
    import bench

    out = []
    for li, o in enumerate(bench.gemm_ops(prog, "tc")):
        out += layer_launches(li, o, dev)
    return out


def layer_launches(li, o, dev):
    """The launches of one layer (a function of its own so that every thunk binds this layer's tensors)."""
    import torch

    from breaching_b200 import engine as E

    out = []
    N, H, W, Ci, Co, R, st, pd = g = o["geom"]
    Ho, Wo = o["Ho"], o["Wo"]
    x, x2 = (torch.randn(N, H, W, Ci, device=dev) for _ in range(2))
    w, w2 = (torch.randn(Co, R, R, Ci, device=dev) for _ in range(2))
    dy, dy2 = (torch.randn(N, Ho, Wo, Co, device=dev) for _ in range(2))
    of, od, ow = torch.empty(N, Ho, Wo, Co, device=dev), torch.empty(N, H, W, Ci, device=dev), torch.empty(Co, R, R, Ci, device=dev)
    keep = (x, x2, w, w2, dy, dy2, of, od, ow)
    a = (N, H, W, Ci, Co, R, R, st, pd)
    tag = f"op{li}" + (" (candidate-fed, columns)" if o["first"] else "")
    rows = [("fprop", 0, 1, lambda: E.conv_gemm(0, x, w, of, *a, backend=2)),
            ("wgrad", 2, 1, lambda: E.conv_gemm(2, x, dy, ow, *a, backend=2))]
    if not o["first"]:
        rows += [("dgrad", 1, 1, lambda: E.conv_gemm(1, dy, w, od, *a, backend=2)),
                 ("tangent fprop", 0, 2, lambda: E.conv_gemm(0, x, w, of, *a, a2=x2, w2=w2, backend=2))]
    else:
        rows += [("tangent fprop", 0, 1, lambda: E.conv_gemm(0, x, w, of, *a, backend=2))]
    rows += [("tangent dgrad", 1, 2, lambda: E.conv_gemm(1, dy, w, od, *a, a2=dy2, w2=w2, backend=2))]
    for kind, mode, nsrc, fn in rows:
        out.append((f"{tag} {kind}", mode, g, nsrc, fn, keep))
    return out


def time_launch(fn, dev, repeats):
    import torch

    fn()
    torch.cuda.synchronize(dev)
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            for _ in range(repeats):
                fn()
    graph.replay()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(3):   # best of three replays: other work on a shared host shows up as outliers, not as a shift
        e0.record()
        graph.replay()
        e1.record()
        e1.synchronize()
        best = min(best, 1e3 * e0.elapsed_time(e1) / repeats)
    return best


def iteration_trace(dev, iters):
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench

    runner = bench.EngineRunner(2, bench.build_case(2), dev, "tc", 0)
    runner.warm(20)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        runner.eng.run(iters)
        runner.eng.sync()
    torch.cuda.synchronize(dev)
    launches = runner.eng.launches_per_iteration()
    runner.eng.close()
    table = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        row = table.setdefault(ev.name, [0, 0.0])
        row[0] += 1
        row[1] += ev.device_time
    rows = [dict(kernel=k, launches_per_iteration=c / iters, us_per_iteration=t / iters, us_mean=t / c) for k, (c, t) in table.items()]
    rows.sort(key=lambda r: -r["us_per_iteration"])
    return dict(iterations=iters, engine_launches_per_iteration=launches, kernels=rows,
                gemm_us_per_iteration=sum(r["us_per_iteration"] for r in rows if "igemm" in r["kernel"] or "linear_" in r["kernel"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=200)
    ap.add_argument("--trace-iters", type=int, default=10)
    args = ap.parse_args()
    import torch

    from breaching_b200 import build as bbuild

    if not torch.cuda.is_available():
        raise SystemExit("profile_gemms.py: no CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    bbuild.build()
    torch.manual_seed(0)
    os.makedirs(args.out, exist_ok=True)
    gpu = dict(name=torch.cuda.get_device_name(dev), BRE_TC_MAX_SPLITS=os.environ.get("BRE_TC_MAX_SPLITS"),
               BRE_TC_STREAM=os.environ.get("BRE_TC_STREAM"))

    import bench

    prog = bench.EngineRunner(2, bench.build_case(2), dev, "tc", 0).prog
    rows = []
    print(f"{'launch':38s} {'M x N x K':>20s} {'tiles':>10s} {'stages':>6s} {'splits':>6s} {'kb/CTA':>6s} {'us':>8s}")
    for label, mode, g, nsrc, fn, _keep in launches_of(prog, dev):
        M, Nc, K = gemm_shape(mode, g)
        us = time_launch(fn, dev, args.repeats)
        if g[1] == 1 and g[2] == 1:   # the classification head: linear_small kernels, not the tensor-core GEMM
            tiles = bm = bn = stages = splits = kbc = 0
        else:
            tiles, bn, splits, kbc = split_plan(mode, g, nsrc)
            bm, stages = ring_plan(mode, g, nsrc)
        rows.append(dict(launch=label, mode=mode, geom=list(g), nsrc=nsrc, M=M, N=Nc, K=K * nsrc, tiles=tiles, tile_m=bm, tile_n=bn,
                         stages=stages, splits=splits, kblocks_per_cta=kbc, us=us))
        print(f"{label:38s} {f'{M} x {Nc} x {K * nsrc}':>20s} {f'{tiles}x{bm}x{bn}':>10s} {stages:6d} {splits:6d} {kbc:6d} {us:8.2f}",
              flush=True)
    total = sum(r["us"] for r in rows)
    print(f"sum over {len(rows)} launches: {total:.1f} us")
    with open(os.path.join(args.out, "gemm_launches.json"), "w") as f:
        json.dump(dict(gpu=gpu, repeats=args.repeats, sum_us=total, launches=rows), f, indent=1)
    trace = iteration_trace(dev, args.trace_iters)
    trace["gpu"] = gpu
    with open(os.path.join(args.out, "iteration_kernels.json"), "w") as f:
        json.dump(trace, f, indent=1)
    print(f"iteration trace: {trace['engine_launches_per_iteration']} launches, GEMM kernels {trace['gemm_us_per_iteration']:.1f} us "
          f"per iteration; top kernels:")
    for r in trace["kernels"][:8]:
        print(f"  {r['us_per_iteration']:8.1f} us  {r['launches_per_iteration']:6.1f} x  {r['kernel'][:100]}")


if __name__ == "__main__":
    main()
