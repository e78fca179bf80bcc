"""L-BFGS trials on the host loop (attacks/lbfgs.py: two-loop recursion in Python, one eager engine evaluation per closure) against
the device loop (one captured graph per optimizer.step, the inner loop under conditional nodes), on three workloads:

  wei          the `wei` preset on the reference ConvNet (width 64) at CIFAR-10 shape, batch 1
  deepleakage  the `deepleakage` preset (joint data + label optimisation) on the same network
  ig_resnet18  `invertinggradients` with optim.optimizer=L-BFGS on ResNet-18 at 224 x 224 (a 150 528-value candidate)

Both paths run the attacker's own trial entry on the same engine from the same start, alternately, ``--repeats`` times, for
``--steps`` recorded iterations each (after one warm-up trial of each, which includes the graph capture).  Reported per path:
recorded iterations and closure evaluations per second, closures per recorded iteration; for the device path also the time its
L-BFGS kernels take per inner iteration (torch.profiler, a separate short run).  The card's name and power limit are read in the
same process.  Writes ``OUTDIR/bench_lbfgs.json`` and prints it.

    python scripts/bench_lbfgs.py OUTDIR [--steps 20] [--repeats 2] [--workloads wei,deepleakage,ig_resnet18]
"""
import argparse
import copy
import json
import os
import statistics
import sys
import time
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

WORKLOADS = {
    "wei": (dict(model_name="convnet", data="cifar", batch=1, seed=16, bn_random=True), "wei", {}),
    "deepleakage": (dict(model_name="convnet", data="cifar", batch=1, seed=21, bn_random=True), "deepleakage", {}),
    "ig_resnet18": (dict(model_name="resnet18", data="imagenet", batch=1, seed=233, bn_random=True), "invertinggradients",
                    {"optim.optimizer": "L-BFGS"}),
}


def card_info(dev):
    import subprocess

    import torch

    info = dict(name=torch.cuda.get_device_name(dev), power_limit_w=None)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(dev.index or 0)],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out)
    except Exception:  # noqa: BLE001
        pass
    return info


class Counting:
    """The engine with its host closure entry counted (the host path's closures)."""

    def __init__(self, engine):
        self.engine, self.calls = engine, 0

    def __getattr__(self, name):
        return getattr(self.engine, name)

    def objective_and_gradient(self, x):
        self.calls += 1
        return self.engine.objective_and_gradient(x)


def setup(name, steps, dev):
    import torch

    from breaching_b200 import get_attack_config, synthetic
    from breaching_b200.attacks import prepare_attack

    case, attack, overrides = WORKLOADS[name]
    joint = attack == "deepleakage"
    model, loss_fn, payload, shared, true = synthetic.make_case(**case, provide_labels=not joint)
    cfg = get_attack_config(attack, {**overrides, "optim.max_iterations": steps, "optim.callback": 0})
    attacker = prepare_attack(model, loss_fn, cfg, dict(device=dev, dtype=torch.float))
    rec_models, labels, stats, shared2 = attacker.prepare_attack(payload, copy.deepcopy(shared))
    engine = attacker._get_engine(rec_models, shared2, torch.zeros(labels.shape[0], dtype=torch.long) if joint else labels)
    gen = torch.Generator().manual_seed(0)
    x0 = torch.randn(true["data"].shape, generator=gen).to(dev)
    l0 = torch.randn(labels.shape, generator=gen).to(dev) if joint else None
    return attacker, engine, joint, x0, l0


def run(attacker, engine, joint, x0, l0, device_path):
    """One trial through the attacker's entry; returns (seconds, recorded iterations, closures)."""
    import torch

    from breaching_b200.attacks import lbfgs
    from breaching_b200.schedule import lr_table

    stats = defaultdict(list)
    counted = Counting(engine)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if joint:
        attacker.host_driven = not device_path
        attacker._run_joint_trial(engine if device_path else counted, x0, l0, stats, 0)
    elif device_path:
        attacker._run_trial(engine, x0, stats, 0)
    else:
        opt = attacker.cfg.optim
        table = lr_table(opt.step_size, opt.step_size_decay, opt.warmup, int(opt.max_iterations))
        dm, ds = attacker.dm.to(x0.device), attacker.ds.to(x0.device)
        _, hist = lbfgs.run_trial(counted, x0, attacker.cfg, table, -dm / ds, (1 - dm) / ds)
        stats["Trial_0_Val"] = hist
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    closures = engine.lbfgs_counters()["closures"] if device_path else counted.calls
    return seconds, len(stats["Trial_0_Val"]), closures, list(stats["Trial_0_Val"])


def kernel_time(attacker, engine, joint, x0, l0):
    """Device time of the L-BFGS kernels per inner iteration (torch.profiler over one device trial)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(attacker, engine, joint, x0, l0, True)
    us = sum(e.device_time_total for e in prof.key_averages() if "lbfgs_" in e.key)
    direction_us = sum(e.device_time_total for e in prof.key_averages()
                       if any(k in e.key for k in ("lbfgs_gram", "lbfgs_recurrence", "lbfgs_dvec")))
    inner = max(engine.lbfgs_counters()["inner_iterations"], 1)
    return dict(lbfgs_kernels_us_per_inner=us / inner, direction_kernels_us_per_inner=direction_us / inner, inner_iterations=inner)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch

    dev = torch.device("cuda:0")
    result = dict(card=card_info(dev), steps=args.steps, repeats=args.repeats, workloads={})
    for name in args.workloads.split(","):
        attacker, engine, joint, x0, l0 = setup(name, args.steps, dev)
        run(attacker, engine, joint, x0, l0, False)   # warm-up of both paths (the device one captures its graph)
        run(attacker, engine, joint, x0, l0, True)
        per = {"host": [], "device": []}
        hist = {}
        for _ in range(args.repeats):
            for path in ("host", "device"):
                s, recorded, closures, h = run(attacker, engine, joint, x0, l0, path == "device")
                per[path].append((s, recorded, closures))
                hist[path] = h
        out = {}
        for path, rows in per.items():
            s = statistics.median(r[0] for r in rows)
            recorded, closures = rows[-1][1], rows[-1][2]
            out[path] = dict(seconds=s, recorded_iterations=recorded, closures=closures,
                             recorded_iterations_per_s=recorded / s, closures_per_s=closures / s,
                             closures_per_recorded_iteration=closures / max(recorded, 1))
        out["device"].update(kernel_time(attacker, engine, joint, x0, l0))
        out["speedup_recorded_iterations"] = out["device"]["recorded_iterations_per_s"] / out["host"]["recorded_iterations_per_s"]
        out["history_host"], out["history_device"] = hist["host"], hist["device"]
        result["workloads"][name] = out
        engine.close()
        print(name, json.dumps({k: v for k, v in out.items() if not k.startswith("history")}), flush=True)
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "bench_lbfgs.json"), "w") as handle:
        json.dump(result, handle, indent=1)
    print(json.dumps(dict(card=result["card"])))


if __name__ == "__main__":
    main()
