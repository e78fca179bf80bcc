"""Cost of the shape-changing augmentations: invertinggradients on a torchvision ResNet-18 (synthetic ImageNet case, batch 1) timed in three arms:

  (a) a 224 x 224 candidate without augmentations,
  (b) a 112 x 112 candidate with ``zoom: {out_size: 224}`` (the model runs at 224; RESAMPLE view and pull-back),
  (c) a 224 x 224 candidate with ``antialias: {width: 5}`` (BLUR view and pull-back),
  (d) - (g) a 224 x 224 candidate with ``continuous_shift: {shift: 8}`` sampled bilinearly with the module's default reflection padding,
      bicubically with reflection padding, nearest with reflection padding, and bilinearly with the circular wrap of multiscale_ghiasi.

Each arm is one engine with its captured CUDA graph; after a warm-up (capture included) the arms are timed in turn, ``--repeats``
rounds of ``--steps`` iterations each, with CUDA events on the engine's stream around the graph launches (``Engine.run_timed``).
The card's name and power limit are read in the same process.  Writes ``OUTDIR/bench_augment_views.json`` and prints it.

    python scripts/bench_augment_views.py OUTDIR [--steps 300] [--warmup 30] [--repeats 3] [--backend tc]
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

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_fedavg_priors import card_info  # noqa: E402

ARMS = {   # name: (candidate size, augmentations)
    "a_224_plain": (224, None),
    "b_112_zoom_224": (112, {"zoom": {"out_size": 224}}),
    "c_224_antialias5": (224, {"antialias": {"width": 5}}),
    "d_224_cshift_reflection_bilinear": (224, {"continuous_shift": {"shift": 8}}),
    "e_224_cshift_reflection_bicubic": (224, {"continuous_shift": {"shift": 8, "mode": "bicubic"}}),
    "f_224_cshift_reflection_nearest": (224, {"continuous_shift": {"shift": 8, "mode": "nearest"}}),
    "g_224_cshift_circular_bilinear": (224, {"continuous_shift": {"shift": 8, "padding": "circular"}}),
}


def make_engine(case, size, augs, dev, backend, n_lr):
    import torch

    from breaching_b200 import get_attack_config
    from breaching_b200.attacks import augment
    from breaching_b200.engine import Engine
    from breaching_b200.schedule import lr_table

    model, loss_fn, payload, shared, true = case
    over = {} if augs is None else {"augmentations": augs, "differentiable_augmentations": True}
    cfg = get_attack_config("invertinggradients", over)
    meta = payload[0]["metadata"]
    cand = (1, 3, size, size)
    eng = Engine(copy.deepcopy(model).to(dev).eval(), augment.view_shape(cfg, cand), cfg, dev, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(dev) for g in shared[0]["gradients"]], true["labels"].to(dev), mean=meta.mean, std=meta.std)
    if augs is not None:
        torch.manual_seed(0)
        eng.set_augmentations(augment.build_plan(cfg, 1, 3, dict(device=dev, dtype=torch.float), spatial=(size, size)))
    x0 = torch.randn(cand, generator=torch.Generator().manual_seed(0))
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
    case = synthetic.make_case("resnet18", "imagenet", batch=1, seed=233, bn_random=True)
    n_lr = args.warmup + args.repeats * args.steps
    engines = {name: make_engine(case, size, augs, dev, args.backend, n_lr) for name, (size, augs) in ARMS.items()}
    for eng in engines.values():
        eng.run(args.warmup)
        eng.sync()
    times = {name: [] for name in engines}
    for _ in range(args.repeats):            # the arms alternate, so drifts of clock or temperature hit all of them
        for name, eng in engines.items():
            times[name].append(eng.run_timed(args.steps))
    result = dict(workload="invertinggradients, torchvision ResNet-18 on the synthetic ImageNet case, batch 1", backend=args.backend, steps=args.steps,
                  warmup=args.warmup, repeats=args.repeats, timing="CUDA events around the captured-graph launches on the engine stream",
                  card=card_info(dev), arms={})
    base = None
    for name, eng in engines.items():
        its = [args.steps / (ms / 1000.0) for ms in times[name]]
        hist = eng.history().tolist()
        size, augs = ARMS[name]
        arm = dict(candidate=size, augmentations=augs, model_input=list(eng.prog.tensors[0].__dict__[k] for k in "NCHW"), it_per_s=its,
                   it_per_s_median=statistics.median(its), launches_per_iteration=eng.launches_per_iteration(),
                   history_finite=all(math.isfinite(h) for h in hist), last_objective=hist[-1] if hist else None)
        if base is None:
            base = arm["it_per_s_median"]
        arm["relative_to_a"] = arm["it_per_s_median"] / base
        result["arms"][name] = arm
        eng.close()
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "bench_augment_views.json"), "w") as handle:
        json.dump(result, handle, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
