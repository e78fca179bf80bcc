"""Every buffer of the four sweeps of a token program (``compiler.compile_transformer``: positional embedding, LayerNorm,
multi-head attention, linears, residual adds, next-token loss with soft targets over a padded vocabulary) against a float64
restatement of its own op (oracle/sweep_check.py), on both GEMM back ends; plus the label gradient, the padded logit columns
(exactly zero), and the TF32 grid of every tensor-core operand on the tensor-core back end.  A soft-label vision case runs the
same seed and label-gradient checks on a CNN.  One joint data + label iteration (``iteration_joint``) is checked end to end: the
soft targets q = softmax(label logits), every sweep buffer on that q, the un-chained label gradient and its softmax chain."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import compiler  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine  # noqa: E402
from helpers import EngineSource, case_from_fixture, cfg_from_fixture, load_golden, sweep_objective  # noqa: E402
from oracle.sweep_check import SweepChecker  # noqa: E402

DEV = torch.device("cuda:0")

MULTI_SEQ = dict(batch=3, seq_len=12, seed=19, ntokens=3000, ninp=96, nhead=8, nhid=384, nlayers=2)
TEXT_CASES = {
    "tag-mini": None,                                     # the fixture model: d = 16, V = 50 (64 padded), SIMT linears
    "multi-seq": (MULTI_SEQ, {}),                         # sequence boundaries, pos_grad over B, tensor-core linears on 36 rows
    "long-seq": (dict(MULTI_SEQ, batch=1, seq_len=72), {}),   # T > 64: several lane strides per softmax row
    "task-reg": (MULTI_SEQ, {"objective.task_regularization": 0.2}),
    "config5": "config5",                                 # full size: V = 50 257 -> 50 304, cluster CE kernels, tall decoder dgrad
}
# one vocabulary per plan of the cluster row kernels not reached above: 2 and 4 CTAs per row, BERT's 30 522 on 8, and 65 500 (65 536
# padded) streaming its segments
WIDE_VOCAB = dict(batch=2, seq_len=8, seed=23, ninp=16, nhead=2, nhid=32, nlayers=1)
for _V in (5000, 12000, 30522, 65500):
    TEXT_CASES[f"vocab-{_V}"] = (dict(WIDE_VOCAB, ntokens=_V), {})


def text_case(name):
    """(model, batch, seq_len, target gradients in program order, attack config)."""
    spec = TEXT_CASES[name]
    if spec is None or spec == "config5":
        fx = load_golden("trial_joint_tag_transformer.pt" if spec is None else "trial_joint_tag_config5.pt")
        model, _, _, shared, _ = case_from_fixture(fx)
        cfg = cfg_from_fixture(fx)
        B, T = fx["case"]["batch"], fx["case"]["seq_len"]
    else:
        case, over = spec
        model, _, _, shared, _ = synthetic.make_text_case(**case)
        cfg = get_attack_config("tag", over)
        B, T = case["batch"], case["seq_len"]
    names = [n for n, _ in model.named_parameters()]
    grads = list(shared[0]["gradients"])
    grads.pop(names.index("encoder.weight"))
    return model, B, T, grads, cfg


def report(chk, tag):
    print(f"\n[{tag}] " + ", ".join(f"{k}/{s}: {r:.3g}" for (k, s), r in sorted(chk.ratios.items())) +
          f"; tensor-core ops reading an off-grid activation: {sorted(chk.off_grid)}")


def check_text(name, backend):
    model, B, T, grads, cfg = text_case(name)
    params = [p.detach() for n, p in model.named_parameters() if n != "encoder.weight"]
    d, V = model.decoder.in_features, model.decoder.out_features
    prog = compiler.compile_transformer(model, B, T)
    eng = Engine(None, (B * T, d, 1, 1), cfg, DEV, backend=backend, program=prog)
    try:
        eng.load_model(params=params)
        L = len(grads)
        eng.load_targets([g.to(DEV) for g in grads], torch.zeros(B * T, dtype=torch.long),
                         tensor_weights=torch.arange(L, 0, -1, dtype=torch.float32) / L)
        gen = torch.Generator().manual_seed(29)
        x = torch.randn(B * T, d, 1, 1, generator=gen)
        q = torch.randn(B * T, V, generator=gen).softmax(dim=-1)
        eng.load_soft_labels(q.to(DEV))
        eng.objective_and_gradient(x.to(DEV))
        lg = eng.label_gradient((B * T, V)).cpu()
        chk = SweepChecker(prog, params, [None] * len(prog.ops), grads, q, sweep_objective(cfg), EngineSource(eng))
        try:
            chk.check(raise_on_failure=False)
            chk.check_label_gradient(lg, raise_on_failure=False)
        finally:
            report(chk, f"{name} / {backend}")
    finally:
        eng.close()
    return chk, prog


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", list(TEXT_CASES))
def test_every_token_sweep_buffer_is_locally_exact(name, backend):
    chk, prog = check_text(name, backend)
    assert not chk.findings, "\n".join(repr(f) for f in chk.findings[:20])
    kinds = {k for k, _ in chk.ratios}
    assert {"posadd", "layernorm", "attention", "linear", "bnact", "label"} <= kinds
    assert {s for _, s in chk.ratios} == {"F", "B", "V", "TF", "TB", "L"}
    assert prog.tensors[prog.logits].C > prog.logits_valid   # the padded logit columns exist (and were checked to be zero)
    if backend == "tc":   # every tensor-core operand the token kernels store is on the TF32 grid
        assert chk.off_grid == set()
    if name == "task-reg":
        assert ("posadd", "B") in chk.ratios


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_soft_label_vision_seed_and_label_gradient(backend):
    """convnet-tiny with class-probability targets (joint DLG / Adam): the soft cross-entropy seed, every sweep and the label
    gradient, with and without the task term."""
    cfg = get_attack_config("invertinggradients", {"objective.task_regularization": 0.3})
    model, _, _, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=2, seed=17, bn_random=True, image_size=32, classes=10)
    model.eval()
    shape = (2, 3, 32, 32)
    grads = shared[0]["gradients"]
    eng = Engine(copy.deepcopy(model).to(DEV), shape, cfg, DEV, backend=backend)
    try:
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in grads], true["labels"].to(DEV))
        gen = torch.Generator().manual_seed(5)
        q = torch.randn(2, 10, generator=gen).softmax(dim=-1)
        eng.load_soft_labels(q.to(DEV))
        eng.objective_and_gradient(torch.randn(shape, generator=gen).to(DEV))
        lg = eng.label_gradient((2, 10)).cpu()
        bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
              for m in compiler.bn_modules(model, eng.prog)]
        chk = SweepChecker(eng.prog, list(model.parameters()), bn, grads, q, sweep_objective(cfg), EngineSource(eng))
        try:
            chk.check()
            chk.check_label_gradient(lg)
        finally:
            report(chk, f"soft-label convnet-tiny / {backend}")
    finally:
        eng.close()
    assert ("label", "L") in chk.ratios and ("linear", "F") in chk.ratios


class JointSource(EngineSource):
    """The engine's buffers after one joint iteration.  Tensor 0's value is the candidate buffer itself, which the step has
    already moved: the iteration evaluated ``x0``."""

    def __init__(self, eng, x0):
        super().__init__(eng)
        self.x0 = x0.detach().double().cpu()

    def tensor(self, which, tid):
        if tid == 0 and which == "val":
            return self.x0.view(self.eng.debug_tensor("val", 0).shape)
        return super().tensor(which, tid)


def check_joint_iteration(eng, params, bn, grads, cfg, x0, ell0, tag):
    """begin_joint_trial(x0, l0), run(1); then q, the chained label gradient the step read, and last the un-chained gradient
    (``label_gradient`` recomputes it into the same buffer)."""
    eng.begin_joint_trial(x0.to(DEV), ell0.to(DEV), [1e-2])
    eng.run(1)
    eng.sync()
    q = eng.debug_step_state("soft_q")
    g_chained = eng.debug_step_state("label_grad")
    g_pre = eng.label_gradient(tuple(ell0.shape)).cpu()
    moved = not torch.equal(eng.debug_tensor("val", 0).view(-1), x0.cpu().view(-1))
    chk = SweepChecker(eng.prog, params, bn, grads, q, sweep_objective(cfg), JointSource(eng, x0))
    try:
        chk.check(raise_on_failure=False)
        chk.check_label_gradient(g_pre, raise_on_failure=False)
        chk.check_label_leaf(ell0, q, g_pre, g_chained, raise_on_failure=False)
        if not eng.prog.seq_len:
            chk.check_terms(eng.last_terms(), raise_on_failure=False)
    finally:
        report(chk, f"joint {tag}; candidate moved by the step: {moved}")
    assert not chk.findings, "\n".join(repr(f) for f in chk.findings[:20])
    assert {("row_softmax", "L"), ("softmax_chain", "L"), ("label", "L")} <= set(chk.ratios)
    return chk


JOINT_TEXT = ["tag-mini", "vocab-5000", "vocab-12000", "vocab-30522", "vocab-65500", "config5"]


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", JOINT_TEXT)
def test_joint_iteration_label_leaf_and_sweeps(name, backend):
    if name == "config5" and backend == "simt":
        pytest.skip("full size on the tensor-core back end, as bench.py --config 5 runs it")
    model, B, T, grads, cfg = text_case(name)
    params = [p.detach() for n, p in model.named_parameters() if n != "encoder.weight"]
    d, V = model.decoder.in_features, model.decoder.out_features
    prog = compiler.compile_transformer(model, B, T)
    eng = Engine(None, (B * T, d, 1, 1), cfg, DEV, backend=backend, program=prog)
    try:
        eng.load_model(params=params)
        L = len(grads)
        eng.load_targets([g.to(DEV) for g in grads], torch.zeros(B * T, dtype=torch.long),
                         tensor_weights=torch.arange(L, 0, -1, dtype=torch.float32) / L)
        gen = torch.Generator().manual_seed(31)
        x0, ell0 = torch.randn(B * T, d, 1, 1, generator=gen), torch.randn(B * T, V, generator=gen)
        check_joint_iteration(eng, params, [None] * len(prog.ops), grads, cfg, x0, ell0, f"{name} / {backend}")
    finally:
        eng.close()


@pytest.mark.parametrize("backend", ["simt", "tc"])
def test_joint_iteration_vision_fixture(backend):
    """The joint Adam fixture's ConvNet (10 classes): ``ce_label_grad`` under the chain."""
    fx = load_golden("trial_joint_adam_convnet.pt")
    model, _, _, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    model.eval()
    x0, ell0 = fx["x0"].float(), fx["l0"].float()
    grads = shared[0]["gradients"]
    eng = Engine(copy.deepcopy(model).to(DEV), tuple(x0.shape), cfg, DEV, backend=backend)
    try:
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in grads], true["labels"].to(DEV))
        bn = [None if m is None or m.running_mean is None else (m.running_mean.double(), m.running_var.double())
              for m in compiler.bn_modules(model, eng.prog)]
        check_joint_iteration(eng, list(model.parameters()), bn, grads, cfg, x0, ell0, f"joint_adam_convnet / {backend}")
    finally:
        eng.close()
