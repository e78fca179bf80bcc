"""Cost of train-mode BatchNorm in FedAvg attacks: BASELINE config 4 (torchvision ResNet-18 at 224 x 224, a FedAvg update of 4
points in 4 local steps x 1 image, lr 1e-3, `modern` without the features prior) timed in two arms:

  (a) eval-mode BN with the server's public buffers (the workload ``bench.py --config 4`` times),
  (b) no BN buffers anywhere: every local step normalises with its own batch statistics (train mode).

Each arm is one engine with its captured CUDA graph; after a warm-up (capture included) the arms are timed in turn, ``--repeats``
rounds of ``--steps`` iterations each, with CUDA events on the engine's stream around the graph launches (``Engine.run_timed``).
The card's name and power limit are read in the same process.  Writes ``OUTDIR/bench_fedavg_trainbn.json`` and prints it.

    python scripts/bench_fedavg_trainbn.py OUTDIR [--steps 300] [--warmup 30] [--repeats 3]
"""
import argparse
import copy
import json
import math
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ARMS = {"a_eval_bn": False, "b_train_bn": True}   # arm -> no_buffers
OVERRIDES = {"regularization.features.scale": 0.0}


def card_info(dev):
    import torch

    info = dict(name=torch.cuda.get_device_name(dev), power_limit_w=None)
    try:
        import pynvml

        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(dev.index or 0)
        info["power_limit_w"] = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception as exc:  # noqa: BLE001
        info["power_limit_error"] = repr(exc)
    return info


def make_engine(case, no_buffers, dev, backend, n_lr):
    import torch

    from breaching_b200 import get_attack_config
    from breaching_b200.engine import Engine
    from breaching_b200.schedule import lr_table

    model, loss_fn, payload, shared, true = case
    cfg = get_attack_config("modern", dict(OVERRIDES))
    local = shared[0]["metadata"]["local_hyperparams"]
    meta = payload[0]["metadata"]
    model = copy.deepcopy(model).to(dev).train(no_buffers)
    for m in model.modules():   # the attacker's model without buffers (base_attack.py:192-197)
        if no_buffers and hasattr(m, "track_running_stats"):
            m.track_running_stats = False
    eng = Engine(model, (int(local["data_per_step"]), *meta.shape), cfg, dev, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(dev) for g in shared[0]["gradients"]], local["labels"][0], mean=meta.mean, std=meta.std)
    n = shared[0]["metadata"]["num_data_points"]
    eng.set_local_steps(n, int(local["steps"]), float(local["lr"]), local["labels"])
    x0 = torch.randn(n, *meta.shape, generator=torch.Generator().manual_seed(0))
    opt = cfg.optim
    eng.begin_trial(x0.to(dev), lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations, n_lr))
    return eng


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--backend", default="tc", choices=["tc", "simt"])
    args = ap.parse_args()

    import torch

    from breaching_b200 import synthetic

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the H100 and has no CPU fallback")
    dev = torch.device("cuda:0")
    n_lr = args.warmup + args.repeats * args.steps
    engines = {}
    for name, no_buffers in ARMS.items():
        case = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-3, seed=233,
                                          no_buffers=no_buffers)
        engines[name] = make_engine(case, no_buffers, dev, args.backend, n_lr)
    for eng in engines.values():
        eng.run(args.warmup)
        eng.sync()
    times = {name: [] for name in engines}
    for _ in range(args.repeats):            # the arms alternate, so drifts of clock or temperature hit all of them
        for name, eng in engines.items():
            times[name].append(eng.run_timed(args.steps))
    result = dict(workload="BASELINE config 4: ResNet-18 224x224, FedAvg 4 points, 4 local steps x 1 image, lr 1e-3, modern "
                           "(features prior off)", backend=args.backend, steps=args.steps, warmup=args.warmup, repeats=args.repeats,
                  timing="CUDA events around the captured-graph launches on the engine stream", card=card_info(dev), arms={})
    base = None
    for name, eng in engines.items():
        its = [args.steps / (ms / 1000.0) for ms in times[name]]
        hist = eng.history().tolist()
        arm = dict(train_mode_bn=ARMS[name], it_per_s=its, it_per_s_median=statistics.median(its),
                   launches_per_iteration=eng.launches_per_iteration(), history_finite=all(math.isfinite(h) for h in hist),
                   last_objective=hist[-1] if hist else None)
        if base is None:
            base = arm["it_per_s_median"]
        arm["relative_to_a"] = arm["it_per_s_median"] / base
        result["arms"][name] = arm
        eng.close()
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "bench_fedavg_trainbn.json"), "w") as handle:
        json.dump(result, handle, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
