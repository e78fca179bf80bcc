"""The row kernels of the label leaf and of the cross-entropy seeds, alone (``engine.row_op``: the engine's own launchers), element
by element against their float64 relations (oracle/sweep_check.py, ``check_row_kernel``).

  * widths C from 1 to 65 536 reach every plan of the five cluster kernels (row softmax, softmax chain, token cross-entropy, its
    tangent, token label gradient): 1, 2, 4 and 8 CTAs per row with the segment in registers, and 8 CTAs streaming it (53 248 is
    the last register width, 53 249 the first streamed one); the block-per-row kernels (``ce_fwd`` with class indices and soft
    targets, ``ce_label_grad``, ``ce_tan_bwd`` with and without the labelled seed) run at the same widths;
  * rows 1, 5, 32; token kernels on B x T rows with T in {1, 2, 8, 32} (T = 1: no row is scored), row stride C and C rounded
    up to 64; logits randn, randn x 40, constant rows (exact ties), one logit of +80, all near -80; targets random softmax rows,
    one-hot rows, sparse rows with exact zeros; task_reg 0 and 0.3; TF32-rounded outputs on and off;
  * guards: every buffer sits inside 4096 NaNs on each side and the padding columns [C, Vs) of every logits-shaped buffer hold
    NaN; afterwards both are still NaN bit for bit (the engine relies on padded logit columns staying untouched) and the outputs
    hold no NaN where a value is due;
  * a second launch gives the same bits."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import engine as E  # noqa: E402
from oracle.sweep_check import check_row_kernel  # noqa: E402

DEV = "cuda:0"
GUARD = 4096
WIDTHS = [1, 2, 3, 10, 255, 256, 257, 1000, 4095, 4096, 4097, 8191, 8192, 16383, 16384, 30522, 50257, 53248, 53249, 65536]
CLUSTER_KERNELS = ("softmax", "softmax_chain", "token_ce_fwd", "token_ce_tan_bwd", "token_label_grad")
BLOCK_KERNELS = ("ce_fwd", "ce_fwd_soft", "ce_label_grad", "ce_tan_bwd", "ce_tan_bwd_seeded")
PLANS = {(1, True), (2, True), (4, True), (8, True), (8, False)}
LOGITS = ("randn", "x40", "const", "spike", "neg80")
TARGETS = ("softmax", "onehot", "sparse")
SEQS = [(1, 1), (3, 2), (1, 8), (3, 8), (1, 32), (3, 32)]   # (B, T) of the token kernels
ROWS = (1, 5, 32)
RATIOS = {}     # (kernel, plan) -> worst error / bound over every case run
REACHED = set()


def expected_plan(C):
    cs = 1 if C < 4096 else 2 if C < 8192 else 4 if C < 16384 else 8
    return cs, C <= 53248


def plan_name(kernel, C):
    if kernel not in CLUSTER_KERNELS:
        return "block"
    cs, fits = E.row_plan(C)
    return f"cs{cs}/{'reg' if fits else 'stream'}"


def _nan_bits():
    return torch.full((1,), float("nan"), device=DEV).view(torch.int32)


class Buf:
    """A [rows, width] fp32 buffer with GUARD NaNs on each side; columns [C, width) are NaN padding."""

    def __init__(self, rows, width, C, values=None):
        self.rows, self.width, self.C = rows, width, C
        self.flat = torch.full((2 * GUARD + rows * width,), float("nan"), device=DEV)
        self.t = self.flat[GUARD:GUARD + rows * width].view(rows, width)
        if values is not None:
            self.t[:, :C] = values

    def intact(self):
        bits, nan = self.flat.view(torch.int32), _nan_bits()
        ok = bool((bits[:GUARD] == nan).all()) and bool((bits[-GUARD:] == nan).all())
        return ok and bool((self.t[:, self.C:].contiguous().view(torch.int32) == nan).all())

    def val(self):
        return self.t[:, :self.C].double()


def logits(kind, rows, C, gen):
    z = torch.randn(rows, C, generator=gen, device=DEV)
    if kind == "x40":
        return z * 40
    if kind == "const":
        return torch.randn(rows, 1, generator=gen, device=DEV).expand(rows, C).contiguous()
    if kind == "spike":
        z = z * 0.1
        z[torch.arange(rows, device=DEV), torch.randint(0, C, (rows,), generator=gen, device=DEV)] = 80.0
        return z
    if kind == "neg80":
        return -80.0 + 0.01 * z
    return z


def targets(kind, rows, C, gen):
    s = torch.randn(rows, C, generator=gen, device=DEV).double().softmax(dim=1)
    if kind == "onehot":
        return torch.nn.functional.one_hot(torch.randint(0, C, (rows,), generator=gen, device=DEV), C).float()
    if kind == "sparse":
        keep = torch.rand(rows, C, generator=gen, device=DEV) < 0.5
        keep[torch.arange(rows, device=DEV), s.argmax(dim=1)] = True
        s = s * keep
        s = s / s.sum(dim=1, keepdim=True)
    return s.float()


def run_case(kernel, C, v, gen):
    """One kernel at width C, variant v: returns (worst ratio per output, findings)."""
    zkind, qkind = LOGITS[v % len(LOGITS)], TARGETS[v % len(TARGETS)]
    tau, round_out = (0.0, 0.3)[(v // 2) % 2], bool((v // 3) % 2)
    token = kernel.startswith("token")
    B, T = SEQS[v % len(SEQS)]
    rows = B * T if token else ROWS[v % len(ROWS)]
    Vs = C if (not token or v % 2 == 0) else (C + 63) // 64 * 64
    z = logits(zkind, rows, C, gen)
    p = z.double().softmax(dim=1).float()
    zd, g = torch.randn(rows, C, generator=gen, device=DEV), torch.randn(rows, C, generator=gen, device=DEV)
    q = targets(qkind, rows, C, gen)
    labels = torch.randint(0, C, (rows,), generator=gen, device=DEV)
    coef = -3.0

    def launch():
        ins, outs = [], {}
        if kernel == "softmax":
            ins = [Buf(rows, C, C, z)]
            outs = {"q": Buf(rows, C, C)}
            E.row_op("softmax", ins[0].t, out0=outs["q"].t)
        elif kernel == "softmax_chain":
            ins = [Buf(rows, C, C, q)]
            outs = {"g": Buf(rows, C, C, g)}
            E.row_op("softmax_chain", ins[0].t, out0=outs["g"].t)
        elif kernel in ("token_ce_fwd", "ce_fwd", "ce_fwd_soft"):
            W = Vs if token else C
            ins = [Buf(rows, W, C, z), Buf(rows, C, C, q)]
            outs = {"p": Buf(rows, W, C), "loss": Buf(rows, 1, 1), "dlogits": Buf(rows, W, C)}
            lab = labels if kernel == "ce_fwd" else None
            E.row_op("token_ce_fwd" if token else "ce_fwd", ins[0].t, in1=None if lab is not None else ins[1].t, labels=lab, C=C, T=T,
                     round_out=round_out and token, out0=outs["p"].t, out1=outs["loss"].t.view(-1), out2=outs["dlogits"].t)
        elif kernel in ("token_ce_tan_bwd", "ce_tan_bwd", "ce_tan_bwd_seeded"):
            W = Vs if token else C
            ins = [Buf(rows, W, C, p), Buf(rows, W, C, zd)]
            outs = {"tdlogits": Buf(rows, W, C)}
            seeded = kernel == "ce_tan_bwd_seeded"
            E.row_op("token_ce_tan_bwd" if token else "ce_tan_bwd", ins[0].t, in1=ins[1].t, labels=labels if seeded else None, C=C, T=T,
                     coef=coef, round_out=round_out and (token or seeded), out0=outs["tdlogits"].t)
        else:   # label gradients
            W = Vs if token else C
            ins = [Buf(rows, W, C, z), Buf(rows, W, C, p), Buf(rows, W, C, zd)]
            outs = {"out": Buf(rows, C, C)}
            E.row_op(kernel, ins[0].t, in1=ins[1].t, in2=ins[2].t, C=C, T=T, coef=tau, out0=outs["out"].t)
        torch.cuda.synchronize()
        return ins, outs

    ins, outs = launch()
    ins2, outs2 = launch()
    for b in ins + list(outs.values()):
        assert b.intact(), f"{kernel} C={C} variant {v}: a guard band or padding column was written"
    for name in outs:
        a, b = outs[name].t.contiguous().view(torch.int32), outs2[name].t.contiguous().view(torch.int32)
        assert torch.equal(a, b), f"{kernel} C={C} variant {v}: {name} differs between two launches"
    rel = dict(z=z.double(), q=q.double(), g=g.double(), p=p.double(), zd=zd.double(), T=T)
    name = {"ce_fwd_soft": "ce_fwd", "ce_tan_bwd_seeded": "ce_tan_bwd"}.get(kernel, kernel)
    if kernel == "ce_fwd":
        rel["labels"] = labels
    if kernel == "ce_tan_bwd_seeded":
        rel.update(labels=labels, coef=coef)
    if kernel in ("token_label_grad", "ce_label_grad"):
        rel["coef"] = tau
    rel["round_out"] = round_out and (token or kernel == "ce_tan_bwd_seeded")
    got = {k: (b.t[:, :1] if k == "loss" else b.t[:, :C]) for k, b in outs.items()}
    if "loss" in got:
        got["loss"] = got["loss"].reshape(-1)
    findings, ratios = check_row_kernel(name, got, **rel)
    tag = f"{kernel} C={C} rows={rows} T={T} Vs={Vs} logits={zkind} targets={qkind} tau={tau} round={rel['round_out']}"
    return ratios, [f"{tag}: {f!r}" for f in findings]


@pytest.mark.parametrize("C", WIDTHS)
def test_row_kernels_against_float64(C):
    plan = E.row_plan(C)
    assert plan == expected_plan(C), (C, plan)
    gen = torch.Generator(device=DEV).manual_seed(1000 + C)
    failures, worst = [], {}
    for kernel in CLUSTER_KERNELS + BLOCK_KERNELS:
        for v in range(6):
            ratios, found = run_case(kernel, C, v, gen)
            failures += found
            worst[kernel] = max([worst.get(kernel, 0.0)] + list(ratios.values()))
        key = (kernel, plan_name(kernel, C))
        RATIOS[key] = max(RATIOS.get(key, 0.0), worst[kernel])
        if kernel in CLUSTER_KERNELS:
            REACHED.add((kernel, plan))
    print(f"\n[row kernels C={C} plan {plan}] " + ", ".join(f"{k}: {r:.3g}" for k, r in worst.items()))
    assert not failures, "\n".join(failures[:20])


def test_every_cluster_kernel_reaches_every_plan():
    assert {expected_plan(C) for C in WIDTHS} == PLANS
    assert {E.row_plan(C) for C in WIDTHS} == PLANS
    if not REACHED:
        pytest.skip("run with the width cases")
    assert REACHED == {(k, p) for k in CLUSTER_KERNELS for p in PLANS}
    print("\n[row kernels: worst error / bound per (kernel, plan)]\n" +
          "\n".join(f"  {k:18s} {p:10s} {r:.3g}" for (k, p), r in sorted(RATIOS.items())))
