"""TAG on the reference's text presets at 32 positions with the GPT-2 vocabulary of 50 257 tokens: transformer3 (learnable
positions, BASELINE config 5), transformer3f (fixed positions, 8 heads of 12), transformer1 (one head of 200) and transformerS (one
head of 512).  Two measurements:

  * iterations per second of the captured joint iteration (``Engine.run_timed``: CUDA events on the engine's stream), ``--repeats``
    rounds of ``--steps`` iterations after ``--warmup``;
  * device time of each attention sweep of each preset's head shape on every kernel that holds it: the resident-head kernel where
    it fits and the cluster-split kernel on each cluster size from the automatic choice to 8 (CUDA events around ``--launches``
    launches of the stand-alone entry point).

The card's name and power limit are read in the same process.  Writes ``OUTDIR/bench_fixed_transformers.json`` and prints it.

    python scripts/bench_fixed_transformers.py OUTDIR [--steps 200] [--warmup 20] [--repeats 3] [--backend tc]
"""
import argparse
import copy
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

sys.path.insert(0, os.path.join(ROOT, "scripts"))
from bench_fedavg_priors import card_info  # noqa: E402

PRESETS = {   # name: (d, heads, nhid, layers, positional)  -- cases/models/model_preparation.py:42-84
    "transformer3": (96, 8, 1536, 3, "learnable"),
    "transformer3f": (96, 8, 1536, 3, "fixed"),
    "transformer1": (200, 1, 200, 1, "fixed"),
    "transformerS": (512, 1, 512, 1, "fixed"),
}
T, VOCAB = 32, 50257


def make_engine(preset, dev, backend):
    import torch

    from breaching_b200 import compiler, get_attack_config, synthetic
    from breaching_b200.attacks import host
    from breaching_b200.engine import Engine
    from breaching_b200.schedule import lr_table

    d, heads, nhid, layers, positional = PRESETS[preset]
    model, _, _, shared, _ = synthetic.make_text_case(batch=1, seq_len=T, seed=233, ntokens=VOCAB, ninp=d, nhead=heads, nhid=nhid,
                                                      nlayers=layers, positional=positional)
    cfg = get_attack_config("tag", {})
    m = copy.deepcopy(model).to(dev).eval()
    sh = [dict(shared[0], gradients=[g.to(dev) for g in shared[0]["gradients"]])]
    host.prepare_for_text_data([m], sh, "run-embedding")
    eng = Engine(None, (T, d, 1, 1), cfg, dev, backend=backend, program=compiler.compile_transformer(m, 1, T))
    eng.load_model(params=[p.detach() for p in m.parameters()])
    L = len(sh[0]["gradients"])
    eng.load_targets(sh[0]["gradients"], torch.zeros(T, dtype=torch.long), tensor_weights=torch.arange(L, 0, -1, dtype=torch.float32) / L)
    opt = cfg.optim
    gen = torch.Generator().manual_seed(0)
    eng.begin_joint_trial((0.1 * torch.randn(T, d, 1, 1, generator=gen)).clamp(-0.1, 0.1),
                          (0.1 * torch.randn(1, T, VOCAB, generator=gen)).clamp(-0.1, 0.1),
                          lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations))
    return eng


def attention_times(dh, heads, launches, dev):
    """{kernel: [ms per launch of sweep 0, 1, 2, 3]} for the head shape (T, heads, dh)."""
    import torch

    from breaching_b200 import engine as E

    d = heads * dh
    gen = torch.Generator().manual_seed(1)
    r = lambda *s: torch.randn(*s, generator=gen).to(dev)  # noqa: E731
    qkv, qkvd, dO, dOd = r(T, 3 * d), r(T, 3 * d), r(T, d), r(T, d)
    P, Pd = torch.empty(1, heads, T, T, device=dev), torch.empty(1, heads, T, T, device=dev)
    ins = {0: {}, 1: dict(in1=dO), 2: dict(in1=qkvd), 3: dict(in1=dOd, in2=dO, in3=qkvd)}
    kernels = ([1] if E.token_attention_plan(T, dh, 1) == 1 else []) + \
        [c for c in range(2, 9) if c <= dh and E.token_attention_plan(T, dh, c) == c]
    out = {}
    for c in kernels:
        times = []
        for sweep in range(4):
            for _ in range(10):
                E.token_attention(sweep, qkv, 1, T, heads, P, Pd, cluster=c, **ins[sweep])
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(launches):
                E.token_attention(sweep, qkv, 1, T, heads, P, Pd, cluster=c, **ins[sweep])
            end.record()
            end.synchronize()
            times.append(start.elapsed_time(end) / launches)
        out["resident" if c == 1 else f"cluster{c}"] = times
    return out, E.token_attention_plan(T, dh, 0)


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--backend", default="tc", choices=["simt", "tc"])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fixed_transformers needs a CUDA device")
    dev = torch.device("cuda:0")
    result = dict(card=card_info(dev), backend=args.backend, seq_len=T, vocab=VOCAB, steps=args.steps, repeats=args.repeats, presets={})
    engines = {name: make_engine(name, dev, args.backend) for name in PRESETS}
    for eng in engines.values():
        eng.run(args.warmup)
        eng.sync()
    rates = {name: [] for name in PRESETS}
    for _ in range(args.repeats):   # the presets alternate within every round
        for name, eng in engines.items():
            rates[name].append(args.steps / (eng.run_timed(args.steps) / 1000.0))
    for name, (d, heads, _, _, positional) in PRESETS.items():
        att, auto = attention_times(d // heads, heads, args.launches, dev)
        result["presets"][name] = dict(positional=positional, heads=heads, dh=d // heads,
                                       launches_per_iteration=engines[name].launches_per_iteration(),
                                       it_per_s=rates[name], it_per_s_median=statistics.median(rates[name]),
                                       attention_ctas_auto=auto, attention_ms_per_sweep=att)
        engines[name].close()
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "bench_fixed_transformers.json"), "w") as handle:
        json.dump(result, handle, indent=1)
    print(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
