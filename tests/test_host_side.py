"""Host-side pieces that need no GPU: compiler, C-ABI library symbols, multi-rank selection over gloo."""
import ctypes
import math
import os
import re
import subprocess
import sys

import pytest
import torch

from breaching_b200 import compiler, synthetic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_compile_resnet18_program():
    model = synthetic.build_model("resnet18", 397).eval()
    prog = compiler.compile_model(model, (1, 3, 224, 224))
    kinds = [op.kind for op in prog.ops]
    assert kinds.count(compiler.OP_CONV) == 20 and kinds.count(compiler.OP_BNACT) == 20
    assert kinds.count(compiler.OP_LINEAR) == 1 and kinds.count(compiler.OP_MAXPOOL) == 1
    assert len(prog.params) == 62 and sum(p.numel for p in prog.params) == 11_380_173  # SURVEY.md section 0 fact 5
    assert prog.tensors[prog.logits].C == 397
    # residual blocks: block input is consumed twice -> second writer accumulates in the reverse sweeps
    assert any(op.acc_in or op.acc_res for op in prog.ops)


def test_compile_rejects_unsupported_graphs():
    class Odd(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.c = torch.nn.Conv2d(3, 4, 3)
            self.f = torch.nn.Linear(4, 2)

        def forward(self, x):
            return self.f(torch.sigmoid(self.c(x)).mean(dim=(2, 3)))

    with pytest.raises(compiler.UnsupportedModelError):
        compiler.compile_model(Odd().eval(), (1, 3, 8, 8))
    # train-mode BatchNorm (no buffers, base_attack.py:192-197) is lowered to batch-statistics BN ops
    train_bn = synthetic.build_model("convnet-tiny", 10).train()
    prog = compiler.compile_model(train_bn, (2, 3, 32, 32))
    assert all(op.bn_train for op in prog.ops if op.kind == compiler.OP_BNACT and op.has_bn)
    assert not any(op.bn_train for op in compiler.compile_model(train_bn.eval(), (2, 3, 32, 32)).ops)


def test_linear_model_on_the_candidate_keeps_torch_column_order():
    """The reference's `linear` model (Flatten -> Linear on the image itself): the candidate stays NCHW in the engine, so the
    weight must NOT be permuted to HWC columns (ADVICE round 1); a Linear behind a feature map is."""
    lin = synthetic.build_model("linear", 10)
    prog = compiler.compile_model(lin, (2, 3, 32, 32))
    assert [op.kind for op in prog.ops] == [compiler.OP_LINEAR] and prog.ops[0].tin == 0
    assert prog.params[prog.ops[0].w].perm == compiler.PERM_NONE
    conv = synthetic.build_model("convnet-tiny", 10)
    prog2 = compiler.compile_model(conv, (2, 3, 32, 32))
    head = [op for op in prog2.ops if op.kind == compiler.OP_LINEAR][-1]
    assert prog2.params[head.w].perm == compiler.PERM_LINEAR_CHW_TO_HWC


def test_reshapes_other_than_flatten_are_rejected_and_eval_dropout_is_identity():
    class ViewNet(torch.nn.Module):
        def __init__(self, how):
            super().__init__()
            self.conv = torch.nn.Conv2d(3, 4, 3, padding=1)
            self.drop = torch.nn.Dropout(0.5)
            self.fc = torch.nn.Linear(4 * 8 * 8, 5)
            self.how = how

        def forward(self, x):
            h = self.drop(self.conv(x))
            if self.how == "view":
                h = h.view(h.size(0), -1)
            elif self.how == "bad-view":
                h = h.view(-1, 4 * 8 * 8 // 2).view(-1, 4 * 8 * 8)
            elif self.how == "flatten0":
                h = torch.flatten(h, 0).view(2, -1)
            else:
                h = h.flatten(1)
            return self.fc(h)

    for how in ("view", "flatten"):
        prog = compiler.compile_model(ViewNet(how).eval(), (2, 3, 8, 8))   # Dropout(0.5) in eval mode is the identity
        assert [op.kind for op in prog.ops] == [compiler.OP_CONV, compiler.OP_LINEAR]
    with pytest.raises(compiler.UnsupportedModelError):
        compiler.compile_model(ViewNet("view").train(), (2, 3, 8, 8))      # ... in train mode it is not
    for how in ("bad-view", "flatten0"):
        with pytest.raises(compiler.UnsupportedModelError):
            compiler.compile_model(ViewNet(how).eval(), (2, 3, 8, 8))


def test_reference_style_container_and_scripted_loss_are_accepted():
    class VisionContainer(torch.nn.Module):  # same shape as cases/models/model_preparation.py:152-160
        def __init__(self, model):
            super().__init__()
            self.model = model

        def forward(self, inputs, **kwargs):
            return self.model(inputs)

    model = VisionContainer(synthetic.build_model("resnet18", 10)).eval()
    prog = compiler.compile_model(model, (1, 3, 64, 64))
    assert len(prog.params) == 62
    from breaching_b200.attacks.optimization_attack import _loss_name

    assert _loss_name(torch.jit.script(torch.nn.CrossEntropyLoss())) == "CrossEntropyLoss"


def test_shared_library_exports_every_declared_symbol():
    from breaching_b200 import build, engine

    lib_path = build.build()
    lib = ctypes.CDLL(lib_path)
    header = open(os.path.join(ROOT, "include", "breaching_b200.h")).read()
    declared = set(re.findall(r"\b(bre_[a-z_0-9]+)\s*\(", header))
    declared -= {"bre_engine"}  # the opaque struct tag
    assert declared == set(engine.EXPORTS), declared ^ set(engine.EXPORTS)
    for name in declared:
        assert hasattr(lib, name), name
    engine.load_library(lib_path)
    assert b"sm_90a" in engine.load_library().bre_version()


def test_product_never_imports_the_oracle():
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "breaching_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, re.M):
                    bad.append(f)
    assert not bad, bad


def test_engine_refuses_cpu_device():
    from breaching_b200 import get_attack_config
    from breaching_b200.attacks import prepare_attack
    from breaching_b200.engine import EngineError

    model = synthetic.build_model("convnet-tiny", 10)
    with pytest.raises(EngineError):
        prepare_attack(model, torch.nn.CrossEntropyLoss(), get_attack_config("invertinggradients"),
                       dict(device=torch.device("cpu"), dtype=torch.float))
    cfg = get_attack_config("invertinggradients")
    cfg.attack_type = "nonsense"
    with pytest.raises(ValueError):
        prepare_attack(model, torch.nn.CrossEntropyLoss(), cfg, dict(device=torch.device("cpu"), dtype=torch.float))
    cfg = get_attack_config("invertinggradients", {"objective.type": "nonsense"})
    with pytest.raises(ValueError):
        prepare_attack(model, torch.nn.CrossEntropyLoss(), cfg, dict(device=torch.device("cuda:0"), dtype=torch.float))


def test_key_packing_orders_like_torch_min():
    from breaching_b200 import dist as bd

    scores = [0.5, float("inf"), 0.25, 0.25, float("nan"), 1e-30, 3.0]
    keys = [bd.pack_key(s, i) for i, s in enumerate(scores)]
    val, idx = bd.unpack_key(min(keys))
    assert (val, idx) == (float(torch.tensor(1e-30, dtype=torch.float32)), 5)
    val, idx = bd.unpack_key(min(bd.pack_key(s, i) for i, s in enumerate([0.25, 0.25])))
    assert idx == 0  # first index wins on ties, like torch.min
    val, idx = bd.unpack_key(min(bd.pack_key(s, i) for i, s in enumerate([float("nan"), float("inf")])))
    assert val == float("inf") and idx == 0
    assert bd.unpack_key(bd.pack_key(-2.0, 3)) == (-2.0, 3) and bd.pack_key(-2.0, 3) < bd.pack_key(-1.0, 0)


_WORKER = r"""
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, sys.argv[1])
from breaching_b200 import dist as bd
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=int(sys.argv[3]), world_size=2)
rank = dist.get_rank()
num_trials = 5
scores = torch.full((num_trials,), float("inf"))
sols = [None] * num_trials
table = [0.9, 0.4, 0.7, 0.4, float("nan")]
for k in range(num_trials):
    if k % 2 == rank:
        scores[k] = table[k] if table[k] == table[k] else float("inf")
        sols[k] = torch.full((1, 3, 4, 4), float(k))
val, idx = bd.select_best(scores)
sol = bd.fetch_solution(sols, idx, (1, 3, 4, 4), dict(device=torch.device("cpu"), dtype=torch.float))
assert idx == 1 and abs(val - 0.4) < 1e-6, (val, idx)
assert torch.all(sol == 1.0)
dist.destroy_process_group()
print("rank", rank, "ok")
"""


def test_trial_selection_over_two_gloo_ranks(tmp_path):
    script = tmp_path / "worker.py"
    script.write_text(_WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = [subprocess.Popen([sys.executable, str(script), ROOT, port, str(r)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(2)]
    outs = [p.communicate(timeout=180)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o


def test_device_lbfgs_restates_torch_lbfgs():
    """breaching_b200/attacks/lbfgs.py against the optimiser the reference constructs (common.py:18:
    ``torch.optim.LBFGS(params, lr)``, torch defaults) on a smooth non-quadratic test function: same loss sequence,
    same iterate, across several ``step`` calls (the optimiser state persists between them) and a changing lr."""
    from breaching_b200.attacks.lbfgs import DeviceLBFGS

    gen = torch.Generator().manual_seed(0)
    A = torch.randn(40, 24, generator=gen)
    b = torch.randn(40, generator=gen)

    def f(z):
        r = A @ z - b
        return 0.5 * (r * r).sum() / 40 + 0.1 * torch.log1p(z * z).sum()

    x_ref = torch.nn.Parameter(torch.randn(24, generator=gen))
    x_dev = x_ref.detach().clone()
    ref_opt = torch.optim.LBFGS([x_ref], lr=1.0)
    dev_opt = DeviceLBFGS(x_dev)

    def ref_closure():
        ref_opt.zero_grad()
        loss = f(x_ref)
        loss.backward()
        return loss

    def dev_closure():
        z = x_dev.detach().clone().requires_grad_(True)
        loss = f(z)
        (g,) = torch.autograd.grad(loss, z)
        return float(loss), g

    for lr in (0.05, 0.3, 1.0, 1.0, 0.5):
        ref_opt.param_groups[0]["lr"] = lr
        a = float(ref_opt.step(ref_closure))
        c = dev_opt.step(dev_closure, lr)
        assert math.isclose(a, c, rel_tol=1e-4, abs_tol=1e-6), (a, c)
        assert (x_ref.detach() - x_dev).abs().max().item() < 1e-3 * (1 + x_ref.detach().abs().max().item())
    # at convergence the `directional derivative > -1e-9` exit is taken on a float32 rounding difference: one evaluation apart
    assert abs(dev_opt.func_evals - ref_opt.state[x_ref]["func_evals"]) <= 1
    assert dev_opt.total_iters == ref_opt.state[x_ref]["n_iter"]


@pytest.mark.parametrize("name", ["adam", "adam-safe", "bert-adam", "momgd", "gd"])
def test_leaf_optimizer_restates_torch_optimisers(name):
    """breaching_b200/attacks/host_optim.py (host-driven loops of the joint and multi-query attackers) against the torch
    optimisers the reference's ``optimizer_lookup`` constructs (common.py:5-18), two leaves, changing step size."""
    from breaching_b200.attacks.host_optim import LeafOptimizer

    gen = torch.Generator().manual_seed(1)
    a0, b0 = torch.randn(5, 7, generator=gen), torch.randn(3, generator=gen)
    ra, rb = torch.nn.Parameter(a0.clone()), torch.nn.Parameter(b0.clone())
    if name == "adam":
        ref = torch.optim.Adam([ra, rb], lr=0.1)
    elif name == "adam-safe":
        ref = torch.optim.Adam([ra, rb], lr=0.1, betas=(0.5, 0.99), eps=1e-4)
    elif name == "bert-adam":
        ref = torch.optim.AdamW([ra, rb], lr=0.1, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01)
    else:
        ref = torch.optim.SGD([ra, rb], lr=0.1, momentum=0.9 if name == "momgd" else 0.0, nesterov=name == "momgd")
    da, db = a0.clone(), b0.clone()
    dev = LeafOptimizer([da, db], name)
    for step, lr in enumerate([0.0, 0.05, 0.1, 0.1, 0.02, 0.3]):
        ga, gb = torch.randn(5, 7, generator=gen), torch.randn(3, generator=gen)
        ref.param_groups[0]["lr"] = lr
        ra.grad, rb.grad = ga.clone(), gb.clone()
        ref.step()
        dev.step([ga, gb], lr)
        assert (ra.detach() - da).abs().max().item() < 1e-6, (name, step)
        assert (rb.detach() - db).abs().max().item() < 1e-6, (name, step)
