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


# ---- the row kernels of the label leaf and of the seeds (csrc/cluster_rows.cuh), emulated in fp32 -----------------------------------
# The register path of a cluster row kernel: the row is cut into one segment per CTA, thread t of a CTA holds elements c0 + k 256 + t
# (k < 26), max and expf per thread, expf summed in fp32 runs of four folded into a double, the (m, s) pairs merged over the lanes
# (butterfly), the 8 warps and the CTAs in order.  The relations of oracle/sweep_check.py must hold for it, and each corrupted result
# below must be reported at its kernel, output and element.
from oracle.sweep_check import check_row_kernel  # noqa: E402

SEG, THREADS = 26, 256
FMAX = torch.finfo(torch.float32).max


def cluster_size(C):   # row_cluster_size
    cs = 1
    while cs < 8 and C // (cs * 2) >= 2048:
        cs *= 2
    return cs


def segments(C, cs):   # row_segment
    per = (((C + cs - 1) // cs) + 3) & ~3
    out = []
    for r in range(cs):
        c0 = min(r * per, C)
        out.append((c0, min(c0 + per, C)))
    return out


def merge(m, s, m2, s2):   # merge_softmax
    M = torch.maximum(m, m2)
    return M, s * torch.exp(m - M).double() + s2 * torch.exp(m2 - M).double()


def cta_pair(zseg):
    """(m, s) of one CTA's segment [rows, L] after the lane and warp merges."""
    rows, L = zseg.shape
    grid = torch.full((rows, SEG * THREADS), -FMAX, dtype=torch.float32)
    grid[:, :L] = zseg
    grid = grid.view(rows, SEG, THREADS)
    m = grid.amax(dim=1)
    e = torch.exp(grid - m.unsqueeze(1))
    s = torch.zeros(rows, THREADS, dtype=torch.float64)
    for k0 in range(0, SEG, 4):
        acc = torch.zeros(rows, THREADS, dtype=torch.float32)
        for k in range(k0, min(k0 + 4, SEG)):
            acc = acc + e[:, k]
        s = s + acc.double()
    m, s = m.view(rows, 8, 32), s.view(rows, 8, 32)
    for o in (16, 8, 4, 2, 1):
        perm = torch.arange(32) ^ o
        m, s = merge(m, s, m[..., perm], s[..., perm])
    tm, ts = m[:, 0, 0], s[:, 0, 0]
    for w in range(1, 8):
        tm, ts = merge(tm, ts, m[:, w, 0], s[:, w, 0])
    return tm, ts


def softmax_stats(z, local=False):
    """Row (max, sum) of the register path; ``local``: every CTA keeps its own pair (the cluster reduction skipped)."""
    C = z.shape[1]
    pairs = [cta_pair(z[:, c0:c1]) for c0, c1 in segments(C, cluster_size(C))]
    if local:
        return pairs
    tm, ts = pairs[0]
    for m2, s2 in pairs[1:]:
        tm, ts = merge(tm, ts, m2, s2)
    return [(tm, ts)] * len(pairs)


def emu_softmax(z, local=False, drop=None):
    C = z.shape[1]
    q = torch.empty_like(z)
    for (c0, c1), (m, s) in zip(segments(C, cluster_size(C)), softmax_stats(z, local)):
        inv = (1.0 / s).float().unsqueeze(1)
        q[:, c0:c1] = torch.exp(z[:, c0:c1] - m.unsqueeze(1)) * inv
    if drop is not None:
        q[:, drop] = 0.0
    return q


def cluster_dot(a, b, local=False):
    """<a, b> per row as the cluster kernels form it (double products and sums, rounded to fp32), per segment."""
    C = a.shape[1]
    parts = [(a[:, c0:c1].double() * b[:, c0:c1].double()).sum(dim=1) for c0, c1 in segments(C, cluster_size(C))]
    tot = sum(parts)
    return [(p if local else tot).float().unsqueeze(1) for p in parts]


def emu_chain(q, g, local=False):
    out = torch.empty_like(g)
    for (c0, c1), d in zip(segments(q.shape[1], cluster_size(q.shape[1])), cluster_dot(q, g, local)):
        out[:, c0:c1] = q[:, c0:c1] * (g[:, c0:c1] - d)
    return out


def emu_token_ce_fwd(z, q, T, score_last=False):
    rows, C = z.shape
    scored = torch.arange(rows) % T != T - 1
    if score_last:
        scored[:] = True
    invM = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(max(rows - rows // T, 1)), dtype=torch.float32)
    m, s = softmax_stats(z)[0]
    fsum = s.float().unsqueeze(1)
    lse = m.unsqueeze(1) + torch.log(fsum)
    p = torch.exp(z - m.unsqueeze(1)) / fsum
    qn = torch.cat([q[1:], torch.zeros_like(q[:1])])
    d = torch.where(scored.view(-1, 1), (p - qn) * invM, torch.zeros_like(p))
    lt = -(qn.double() * (z - lse).double()).sum(dim=1)
    loss = torch.where(scored, (lt * rows * invM.double()).float(), torch.zeros(rows))
    return p, loss, d


def emu_token_tan_bwd(p, zd, T):
    rows = p.shape[0]
    invM = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(max(rows - rows // T, 1)), dtype=torch.float32)
    dt = cluster_dot(p, zd)[0]
    g = p * (zd - dt) * invM
    return torch.where((torch.arange(rows) % T != T - 1).view(-1, 1), g, torch.zeros_like(g))


def emu_label_grad(z, p, zd, tau, T=None, shift=1):
    """ce_label_grad (T None: mean over the N rows) or token_label_grad (row (b, t) from logits row (b, t - shift))."""
    rows = z.shape[0]
    M = rows if T is None else max(rows - rows // T, 1)
    iM = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(M), dtype=torch.float32)
    dt = cluster_dot(p, zd)[0]
    mx = z.amax(dim=1, keepdim=True)
    lse = mx + torch.log(torch.exp(z - mx).double().sum(dim=1, keepdim=True).float())
    v = -(zd - dt) * iM
    if tau:
        v = v - tau * (z - lse) * iM
    if T is None:
        return v
    out = torch.zeros_like(v)
    src = torch.arange(rows) - shift
    ok = (torch.arange(rows) % T != 0) & (src >= 0)
    out[ok] = v[src[ok]]
    return out


def _rows(rows, C, seed, scale=1.0):
    gen = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, C, generator=gen) * scale
    return z, torch.randn(rows, C, generator=gen).softmax(dim=1), torch.randn(rows, C, generator=gen), torch.randn(rows, C, generator=gen)


@pytest.mark.parametrize("C", [3, 257, 5000, 12000, 30522])
@pytest.mark.parametrize("scale", [1.0, 40.0])
def test_fp32_emulated_row_kernels_satisfy_their_relations(C, scale):
    T = 4
    z, q, g, zd = _rows(2 * T, C, C, scale)
    p = z.double().softmax(dim=1).float()
    rel = dict(z=z.double(), q=q.double(), g=g.double(), p=p.double(), zd=zd.double(), T=T)
    pp, loss, d = emu_token_ce_fwd(z, q, T)
    results = {
        "softmax": {"q": emu_softmax(z)},
        "softmax_chain": {"g": emu_chain(q, g)},
        "token_ce_fwd": {"p": pp, "loss": loss, "dlogits": d},
        "token_ce_tan_bwd": {"tdlogits": emu_token_tan_bwd(p, zd, T)},
        "token_label_grad": {"out": emu_label_grad(z, p, zd, 0.3, T)},
        "ce_label_grad": {"out": emu_label_grad(z, p, zd, 0.3)},
    }
    for kernel, outs in results.items():
        findings, ratios = check_row_kernel(kernel, outs, **dict(rel, coef=0.3 if "label" in kernel else 0.0))
        assert not findings, findings
        assert max(ratios.values()) < 0.5, (kernel, ratios)


def _reported(kernel, outs, **rel):
    findings, _ = check_row_kernel(kernel, outs, **rel)
    return [(f.kind, f.sweep, f.index) for f in findings]


def test_element_dropped_at_a_segment_boundary_is_reported():
    C = 16384
    assert cluster_size(C) == 8
    z, q, g, zd = _rows(3, C, 1)
    c = segments(C, 8)[2][1] - 1   # the last element of rank 2's segment
    found = _reported("softmax", {"q": emu_softmax(z, drop=c)}, z=z.double())
    assert [f[:2] for f in found] == [("softmax", "q")] and found[0][2][1] == c


@pytest.mark.parametrize("local", ["sum", "pair"])
def test_softmax_over_one_rank_only_is_reported(local):
    """The sum of rank 0's segment only (max right), or every CTA normalising by its own (max, sum)."""
    C = 16384
    z, q, g, zd = _rows(2, C, 2)
    if local == "pair":
        bad = emu_softmax(z, local=True)
    else:
        (m, _), = softmax_stats(z)[:1]
        s0 = cta_pair(z[:, :segments(C, 8)[0][1]])[1] * torch.exp(cta_pair(z[:, :segments(C, 8)[0][1]])[0] - m).double()
        bad = torch.exp(z - m.unsqueeze(1)) * (1.0 / s0).float().unsqueeze(1)
    found = _reported("softmax", {"q": bad}, z=z.double())
    assert [f[:2] for f in found] == [("softmax", "q")]


def test_chain_with_a_cta_local_dot_is_reported():
    C = 30522
    z, q, g, zd = _rows(2, C, 3)
    assert not _reported("softmax_chain", {"g": emu_chain(q, g)}, q=q.double(), g=g.double())
    found = _reported("softmax_chain", {"g": emu_chain(q, g, local=True)}, q=q.double(), g=g.double())
    assert [f[:2] for f in found] == [("softmax_chain", "g")]


def test_unscored_last_row_left_nonzero_is_reported():
    C, T = 5000, 4
    z, q, g, zd = _rows(2 * T, C, 4)
    p, loss, d = emu_token_ce_fwd(z, q, T)
    _, _, bad = emu_token_ce_fwd(z, q, T, score_last=True)
    rel = dict(z=z.double(), q=q.double(), T=T)
    assert not _reported("token_ce_fwd", {"p": p, "loss": loss, "dlogits": d}, **rel)
    found = _reported("token_ce_fwd", {"p": p, "loss": loss, "dlogits": bad}, **rel)
    assert [f[:2] for f in found] == [("token_ce_fwd", "dlogits")] and found[0][2][0] % T == T - 1


def test_label_gradient_from_the_wrong_source_row_is_reported():
    C, T = 12000, 4
    z, q, g, zd = _rows(2 * T, C, 5)
    p = z.double().softmax(dim=1).float()
    rel = dict(z=z.double(), p=p.double(), zd=zd.double(), T=T, coef=0.3)
    assert not _reported("token_label_grad", {"out": emu_label_grad(z, p, zd, 0.3, T)}, **rel)
    found = _reported("token_label_grad", {"out": emu_label_grad(z, p, zd, 0.3, T, shift=0)}, **rel)
    assert [f[:2] for f in found] == [("token_label_grad", "out")] and found[0][2][0] % T != 0
