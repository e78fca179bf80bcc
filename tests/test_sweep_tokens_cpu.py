"""The layer-local sweep checker (oracle/sweep_check.py) on token programs (``compiler.compile_transformer``: positional
embedding, LayerNorm, multi-head attention, next-token loss with soft targets) fed with the float64 interpreter's buffers:
every relation holds to rounding level, and a buffer corrupted the way a faulty token kernel would corrupt it is reported at
exactly the op and sweep that produced it."""
import copy

import pytest
import torch

from breaching_b200 import compiler, get_attack_config, synthetic
from helpers import case_from_fixture, load_golden, sweep_objective
from oracle import program_interp as PI
from oracle.sweep_check import InterpreterSource, SweepChecker


def text_case(name):
    """(model, batch, seq_len, target gradients in program order, attack config)."""
    if name == "tag-fixture":
        fx = load_golden("trial_joint_tag_transformer.pt")
        model, _, _, shared, _ = case_from_fixture(fx)
        cfg = get_attack_config("tag", dict(fx["overrides"]))
        B, T = fx["case"]["batch"], fx["case"]["seq_len"]
    else:   # three sequences, odd head size (15 = 3 heads of 5)
        model, _, _, shared, _ = synthetic.make_text_case(batch=3, seq_len=5, seed=7, ntokens=37, ninp=15, nhead=3, nhid=20, nlayers=2)
        treg = {"objective.task_regularization": 0.2} if name == "multi-seq-task-reg" else {}
        cfg = get_attack_config("tag", treg)
        B, T = 3, 5
    names = [n for n, _ in model.named_parameters()]
    grads = list(shared[0]["gradients"])
    grads.pop(names.index("encoder.weight"))
    return model, B, T, grads, cfg


class _Params:   # the interpreter reads parameters in program order (token embedding removed)
    def __init__(self, model):
        self.model = model

    def parameters(self):
        return [p for n, p in self.model.named_parameters() if n != "encoder.weight"]

    def named_modules(self):
        return self.model.named_modules()


def run_interpreter(name, tamper=None, seed=3):
    """float64 four sweeps of the un-padded token program; returns (checker fed with the interpreter's buffers, program,
    interpreter)."""
    model, B, T, grads, cfg = text_case(name)
    m64 = copy.deepcopy(model).double()
    prog = compiler.compile_transformer(m64, B, T, pad_vocab=False)
    it = PI.ProgramInterpreter(_Params(m64), prog)
    it.tamper = tamper
    gen = torch.Generator().manual_seed(seed)
    d, V = m64.decoder.in_features, m64.decoder.out_features
    x = torch.randn(B, T, d, generator=gen, dtype=torch.float64)
    q = torch.randn(B, T, V, generator=gen, dtype=torch.float64).softmax(dim=-1)
    obj = sweep_objective(cfg)
    g64 = [g.double() for g in grads]
    kw = {k: obj[k] for k in ("tag_scale", "scale_scheme") if k in obj}
    _, dx, _, _ = it.matching_gradient(x, q, g64, obj["kind"], scale=obj["scale"], task_regularization=obj["task_regularization"], **kw)
    chk = SweepChecker(prog, it.P, it.bn, g64, q.reshape(B * T, V), obj, InterpreterSource(it, dx))
    return chk, prog, it


def label_gradient(it, tau):
    """d objective / d q of the interpreter run: the matching term's ``dq`` plus the task term ``tau dL/dq``."""
    z = it.a[it.prog.logits].flatten(1)
    lsm = torch.log_softmax(z, dim=1)
    task = torch.zeros_like(lsm)
    task[1:] = -lsm[:-1] / it.M
    task[torch.arange(z.shape[0]) % it.prog.seq_len == 0] = 0.0
    return it.dq.reshape(z.shape) + tau * task


CASES = ["tag-fixture", "multi-seq", "multi-seq-task-reg"]


@pytest.mark.parametrize("name", CASES)
def test_interpreter_buffers_satisfy_every_token_relation(name):
    chk, prog, it = run_interpreter(name)
    chk.check()
    chk.check_label_gradient(label_gradient(it, chk.obj["task_regularization"]))
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]
    kinds = {k for k, _ in chk.ratios}
    assert {"posadd", "layernorm", "attention", "linear", "bnact", "label"} <= kinds
    assert {s for _, s in chk.ratios} == {"F", "B", "V", "TF", "TB", "L"}
    if name == "multi-seq-task-reg":   # the task-loss gradient of the candidate (delta of tensor 0) is checked
        assert ("posadd", "B") in chk.ratios and chk.obj["task_regularization"] == 0.2


def _flagged(chk):
    return {(f.op, f.sweep) for f in chk.check(raise_on_failure=False)}


def _ops(prog, kind):
    return [i for i, op in enumerate(prog.ops) if op.kind == kind]


@pytest.mark.parametrize("name", ["tag-fixture", "multi-seq"])
def test_scaled_attention_head_tangent_is_reported_at_the_attention(name):
    """The columns of one head of an attention tangent scaled by 1.001."""
    _, prog, _ = run_interpreter(name)
    target = _ops(prog, compiler.OP_ATTENTION)[-1]
    op = prog.ops[target]
    dh = prog.tensors[op.tout].C // op.R

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "TF" and i == target:
            stored = stored.clone()
            stored[:, dh:2 * dh] *= 1.001
        return stored

    chk, _, _ = run_interpreter(name, tamper=tamper)
    assert _flagged(chk) == {(target, "TF")}


def test_layernorm_delta_rows_swapped_across_a_sequence_boundary():
    _, prog, _ = run_interpreter("multi-seq")
    target = _ops(prog, compiler.OP_LAYERNORM)[1]
    t = prog.ops[target].tin
    assert min(i for i, op in enumerate(prog.ops) if t in (op.tin, op.res)) == target   # its write makes the delta final
    T = prog.seq_len

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "B" and i == target and tid == t:
            stored = stored.clone()
            assert not torch.equal(stored[T - 1], stored[T])
            stored[[T - 1, T]] = stored[[T, T - 1]]
        return stored

    chk, _, _ = run_interpreter("multi-seq", tamper=tamper)
    assert _flagged(chk) == {(target, "B")}


@pytest.mark.parametrize("sweep", ["B", "TB"])
def test_dropped_accumulation_on_a_layernorm_output_is_reported(sweep):
    """The output of the first LayerNorm feeds linear1 and the second residual add; linear1 runs last in the reverse sweeps and
    overwrites its delta instead of accumulating into it."""
    _, prog, _ = run_interpreter("multi-seq")
    n1 = prog.ops[_ops(prog, compiler.OP_LAYERNORM)[0]].tout
    consumers = [i for i, op in enumerate(prog.ops) if n1 in (op.tin, op.res)]
    assert [prog.ops[i].kind for i in consumers] == [compiler.OP_LINEAR, compiler.OP_BNACT] and prog.ops[consumers[1]].res == n1
    last = consumers[0]

    def tamper(sweep_, i, tid, stored, contribution=None):
        return contribution if (sweep_ == sweep and i == last and tid == n1) else stored

    chk, _, _ = run_interpreter("multi-seq", tamper=tamper)
    assert _flagged(chk) == {(last, sweep)}


def test_task_loss_gradient_of_the_candidate_is_required():
    """A program that drops the task-loss gradient of the candidate (delta of tensor 0 left zero) is reported at the positional
    embedding, sweep B."""
    chk, prog, it = run_interpreter("multi-seq-task-reg")
    it.d_B[0] = torch.zeros_like(it.d_B[0])
    assert {(f.op, f.sweep) for f in chk.check(raise_on_failure=False)} >= {(0, "B")}


def test_label_gradient_with_a_wrong_source_row_is_reported():
    chk, prog, it = run_interpreter("multi-seq")
    chk.check()
    lg = label_gradient(it, 0.0)
    assert not chk.check_label_gradient(lg, raise_on_failure=False)
    shifted = torch.roll(lg, 1, dims=0)
    assert {(f.kind, f.sweep) for f in chk.check_label_gradient(shifted, raise_on_failure=False)} == {("label", "L")}
