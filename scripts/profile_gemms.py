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
the same rules as launch_igemm_tc / launch_tc in breaching_b200/csrc/igemm_tc.cu (honouring BRE_TC_MAX_SPLITS); it is a label of the rows, the
times are measured.
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


def split_plan(mode, g, nsrc):
    """(tiles, tile width, split-K factor, k-blocks per CTA) as launch_igemm_tc / launch_tc choose them."""
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    kb = -(-K // BK) * nsrc
    tm = -(-M // BM)
    cls = mode == 1 and st == 2
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
    narrow_ok = mode != 0 and not cls and (mode != 2 or Ci % 32 == 0)
    underfilled = Nc % 64 == 0 and tm * (Nc // 64) * 16 <= NUM_SMS and kb >= 64 and narrow_ok
    bn = 32 if Nc % 64 != 0 or underfilled else 64
    tiles = tm * (Nc // bn)
    splits = 1
    while splits < MAX_CLUSTER and tiles * splits < NUM_SMS and kb // (splits * 2) >= 2:
        splits *= 2
    cap = int(os.environ.get("BRE_TC_MAX_SPLITS", "0"))
    if cap > 0:
        splits = min(splits, cap)
    p = 1
    while p * 2 <= splits and p < MAX_CLUSTER:
        p *= 2
    splits = p
    while splits > 1 and splits > kb:
        splits //= 2
    return tiles, bn, splits, -(-kb // splits)


def ring_plan(mode, g, nsrc):
    """(tile rows, ring depth) as launch_igemm_tc / launch_tc choose them (honouring BRE_TC_STREAM and BRE_TC_STAGES)."""
    N, H, W, Ci, Co, R, st, pd = g
    M, Nc, K = gemm_shape(mode, g)
    tiles, bn, splits, kbc = split_plan(mode, g, nsrc)
    stream = int(os.environ.get("BRE_TC_STREAM", "1")) != 0
    bm = 64 if stream and M <= 64 and (mode == 0 or (mode == 1 and st == 1)) else BM
    shortk = kbc <= 6 and tiles == Nc // bn and tiles * splits > 2 * NUM_SMS
    deep = bm == 64 and tiles * splits <= NUM_SMS and kbc >= 16
    forced = int(os.environ.get("BRE_TC_STAGES", "0"))
    return bm, forced if forced in (2, 4, 8) else (2 if shortk else 8 if deep else 4)


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
