#!/usr/bin/env python
"""Where a k-block of the batch-1 layer-3 / layer-4 GEMM launches goes (ResNet-18, 224x224, batch 1, config 2).

    python scripts/trace_gemm_phases.py --out DIR [--repeats 100]

1. Phase trace.  A second copy of the library is compiled with -DBRE_TC_TRACE into DIR (the flags and sources of
   breaching_b200/build.py; the in-tree library is left alone) and loaded with engine.load_library.  Every fprop / dgrad launch of
   the layer-3 and layer-4 convolutions (the thunks of profile_gemms.launches_of) runs once and reads back the clock64 marks of
   CTA (0,0,0) (bre_debug_tc_trace): prologue (marks 0 -> 2), first-stage latency (2 -> 4), k-loop per k-block ((5 - 4) / k-blocks
   per CTA) and split-K epilogue (5 -> 10), in SM cycles.  Run with BRE_TC_STREAM=0 (128-row tiles, 4 stages) and =1.
2. Timing matrix.  The same launches on the normal library, CUDA events over a graph of back-to-back launches as
   profile_gemms.time_launch, for BRE_TC_STAGES = 2, 4, 8 x BRE_TC_PRODUCERS = 1, 2, 4 x BRE_TC_STREAM = 0, 1, with the weights
   L2-hot (the same tensors every launch) and cold (rotating copies totalling more than the 50 MB L2).  The kernel runs at most
   one producer lane per ring stage, so 4 producers on a 2-deep ring run as 2.

Every switch is read once per process, so each setting runs in a subprocess of this script.  Results: DIR/phases.json and
DIR/timing.json, with the card's name, power limit and SM clocks read in the same run.
"""
import argparse
import concurrent.futures
import itertools
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

COLD_BYTES = 64 << 20


def build_traced(out_dir):
    from breaching_b200 import build as bbuild

    libdir = os.path.join(out_dir, "traced")
    os.makedirs(libdir, exist_ok=True)
    flags = [f for f in bbuild.NVCC_FLAGS if f != "--use_fast_math=false"] + ["-DBRE_TC_TRACE"]

    def compile_one(src):
        obj = os.path.join(libdir, src.replace(".cu", ".o"))
        res = subprocess.run([bbuild._nvcc(), *flags, "-c", os.path.join(bbuild.CSRC, src), "-o", obj], capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{res.stderr[-4000:]}")
        return obj

    with concurrent.futures.ThreadPoolExecutor(max_workers=len(bbuild.SOURCES)) as pool:
        objs = list(pool.map(compile_one, bbuild.SOURCES))
    lib = os.path.join(libdir, "libbreaching_b200_trace.so")
    res = subprocess.run([bbuild._nvcc(), "-shared", "-o", lib, *objs, "-lcudart", "-lcuda"], capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("link failed:\n" + res.stderr[-4000:])
    return lib


def deep_layers(dev):
    """(index, bench.gemm_ops entry) of the config-2 conv layers whose output is 14 x 14 or 7 x 7."""
    import bench

    prog = bench.EngineRunner(2, bench.build_case(2), dev, "tc", 0).prog
    return [(li, o) for li, o in enumerate(bench.gemm_ops(prog, "tc")) if o["Ho"] in (7, 14) and o["geom"][1] > 1]


def deep_launches(layers, dev):
    """(label, mode, geometry, nsrc, thunk, keep-alive) of their fprop / dgrad launches (the thunks of profile_gemms.launches_of)."""
    import profile_gemms as P

    out = []
    for li, o in layers:
        out += [row for row in P.layer_launches(li, dict(o, geom=tuple(o["geom"])), dev) if row[1] != 2]
    return out


def cold_thunk(mode, g, nsrc, dev):
    """A launch of the same shape whose weight operand rotates over copies totalling more than the L2."""
    import torch

    from breaching_b200 import engine as E

    N, H, W, Ci, Co, R, st, pd = g
    Ho, Wo = (H + 2 * pd - R) // st + 1, (W + 2 * pd - R) // st + 1
    a = [torch.randn(N, *((H, W, Ci) if mode == 0 else (Ho, Wo, Co)), device=dev) for _ in range(nsrc)]
    wbytes = Co * R * R * Ci * 4 * nsrc
    copies = max(2, -(-COLD_BYTES // wbytes))
    ws = [[torch.randn(Co, R, R, Ci, device=dev) for _ in range(nsrc)] for _ in range(copies)]
    out = torch.empty(*((N, Ho, Wo, Co) if mode == 0 else (N, H, W, Ci)), device=dev)
    args = (N, H, W, Ci, Co, R, R, st, pd)
    it = itertools.cycle(ws)

    def fn():
        w = next(it)
        E.conv_gemm(mode, a[0], w[0], out, *args, a2=a[1] if nsrc == 2 else None, w2=w[1] if nsrc == 2 else None, backend=2)

    return fn, (a, ws, out)


def worker(kind, lib, repeats, layers_path):
    import torch

    import profile_gemms as P
    from breaching_b200 import engine as E

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    torch.manual_seed(0)
    if lib:
        E.load_library(lib)
    with open(layers_path) as f:
        layers = json.load(f)
    rows = []
    for label, mode, g, nsrc, fn, _keep in deep_launches(layers, dev):
        tiles, bn, splits, kbc = P.split_plan(mode, g, nsrc)
        bm, stages = P.ring_plan(mode, g, nsrc)
        row = dict(launch=label, mode=mode, geom=list(g), nsrc=nsrc, tiles=tiles, tile_m=bm, tile_n=bn, stages=stages, splits=splits,
                   kblocks_per_cta=kbc)
        if kind == "trace":
            import ctypes

            trace = (ctypes.c_longlong * 16)()
            fn()
            torch.cuda.synchronize(dev)
            fn()
            torch.cuda.synchronize(dev)
            if E.load_library().bre_debug_tc_trace(trace) != 0:
                raise SystemExit("bre_debug_tc_trace failed")
            m = list(trace)
            row.update(prologue=m[2] - m[0], first_stage=m[4] - m[2], kloop_per_kblock=(m[5] - m[4]) / kbc, epilogue=m[10] - m[5],
                       total=m[10] - m[0])
        else:
            row["us_hot"] = P.time_launch(fn, dev, repeats)
            cfn, _ckeep = cold_thunk(mode, g, nsrc, dev)
            row["us_cold"] = P.time_launch(cfn, dev, repeats)
            del _ckeep
        rows.append(row)
    return rows


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        res = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=60)
        return dict(zip(q.split(","), (s.strip() for s in res.stdout.splitlines()[0].split(","))))
    except (OSError, IndexError, subprocess.SubprocessError) as e:
        return dict(error=str(e))


def run_worker(kind, env, lib, repeats, out_dir):
    path = os.path.join(out_dir, f"worker_{os.getpid()}.json")
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", kind, "--out", path, "--repeats", str(repeats),
           "--layers", os.path.join(out_dir, "layers.json")] + (["--lib", lib] if lib else [])
    res = subprocess.run(cmd, env=dict(os.environ, **env), capture_output=True, text=True)
    if res.returncode != 0:
        raise SystemExit(f"worker {kind} {env} failed:\n{res.stdout[-2000:]}{res.stderr[-4000:]}")
    with open(path) as f:
        rows = json.load(f)
    os.remove(path)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=100)
    ap.add_argument("--worker", choices=("trace", "time"))
    ap.add_argument("--lib", default=None)
    ap.add_argument("--layers", default=None)
    args = ap.parse_args()
    if args.worker:
        with open(args.out, "w") as f:
            json.dump(worker(args.worker, args.lib, args.repeats, args.layers), f)
        return
    import torch

    from breaching_b200 import build as bbuild

    if not torch.cuda.is_available():
        raise SystemExit("trace_gemm_phases.py: no CUDA device")
    os.makedirs(args.out, exist_ok=True)
    bbuild.build()
    with concurrent.futures.ThreadPoolExecutor(max_workers=1) as pool:   # the traced library compiles while the layers are listed
        traced = pool.submit(build_traced, args.out)
        with open(os.path.join(args.out, "layers.json"), "w") as f:
            json.dump(deep_layers(torch.device("cuda:0")), f)
        lib = traced.result()
    gpu = gpu_info()
    phases = {}
    for stream in (0, 1):
        rows = run_worker("trace", {"BRE_TC_STREAM": str(stream)}, lib, args.repeats, args.out)
        phases[f"BRE_TC_STREAM={stream}"] = rows
        print(f"-- phases (SM cycles, CTA (0,0,0)), BRE_TC_STREAM={stream}")
        for r in rows:
            print(f"{r['launch']:32s} {r['tile_m']:4d}x{r['tile_n']:<3d} {r['stages']} st  kb {r['kblocks_per_cta']:3d}  prologue {r['prologue']:6d}  "
                  f"first {r['first_stage']:6d}  per-kb {r['kloop_per_kblock']:7.0f}  epilogue {r['epilogue']:6d}", flush=True)
    with open(os.path.join(args.out, "phases.json"), "w") as f:
        json.dump(dict(gpu=gpu, cycles="SM clock64", phases=phases), f, indent=1)
    timing = {}
    for stream, stages, prod in itertools.product((0, 1), (2, 4, 8), (1, 2, 4)):
        key = f"stream={stream} stages={stages} producers={prod}"
        rows = run_worker("time", {"BRE_TC_STREAM": str(stream), "BRE_TC_STAGES": str(stages), "BRE_TC_PRODUCERS": str(prod)}, None,
                          args.repeats, args.out)
        timing[key] = rows
        print(f"-- {key}: sum hot {sum(r['us_hot'] for r in rows):.1f} us, cold {sum(r['us_cold'] for r in rows):.1f} us", flush=True)
        with open(os.path.join(args.out, "timing.json"), "w") as f:   # rewritten after every setting: a partial run keeps its rows
            json.dump(dict(gpu=gpu, repeats=args.repeats, timing=timing), f, indent=1)
    for stream in (0, 1):   # the depth each launch gets by default
        key = f"stream={stream} default"
        timing[key] = run_worker("time", {"BRE_TC_STREAM": str(stream)}, None, args.repeats, args.out)
        print(f"-- {key}: sum hot {sum(r['us_hot'] for r in timing[key]):.1f} us, cold {sum(r['us_cold'] for r in timing[key]):.1f} us")
    gpu_after = gpu_info()
    with open(os.path.join(args.out, "timing.json"), "w") as f:
        json.dump(dict(gpu=gpu, gpu_after=gpu_after, repeats=args.repeats, timing=timing), f, indent=1)
    print(json.dumps(dict(gpu=gpu, gpu_after=gpu_after)))


if __name__ == "__main__":
    main()
