"""The reference's fixed-position transformers (transformer3f, transformer1, transformerS: the sinusoidal ``PositionalEmbedding``
buffer of language_models.py:89-130) on the CPU: the synthetic model against the reference's ``TransformerModel``, the constant
positional add of ``compiler.compile_transformer``, and the float64 four-sweep statement against the reference's TAG closure
(tests/golden/fixed_transformers.pt)."""
import os
import sys
import types

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from helpers import load_golden  # noqa: E402
from breaching_b200 import compiler, synthetic  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.transformer_interp import TransformerFourSweep  # noqa: E402

FIXTURES = ["transformer3f", "transformer1", "transformerS"]
needs_reference = pytest.mark.skipif(not refshim.reference_available(), reason="the reference tree is not available here")


class FixedPositionFourSweep(TransformerFourSweep):
    """The float64 four sweeps with the constant table: TransformerFourSweep over the model with ``pe[0]`` in place of the learnable
    table, whose gradient entry is dropped (the table is no parameter) and whose direction is zero (TF passes the zero tangent of
    x through the constant add)."""

    def __init__(self, model, dtype=torch.float64):
        view = types.SimpleNamespace(pos_embedding=types.SimpleNamespace(weight=model.pos_encoder.pe[0]), layers=model.layers,
                                     decoder=model.decoder)
        super().__init__(view, dtype)

    def backward(self):
        self.G = super().backward()[1:]
        return self.G

    def tangent_forward(self, V):
        return super().tangent_forward([torch.zeros_like(self.pos)] + list(V))


def _relerr(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-300)).item()


def _case(name):
    fx = load_golden("fixed_transformers.pt")[name]
    model, loss_fn, payload, shared, true = synthetic.make_text_case(**fx["case"])
    checksum = float(sum(p.detach().double().sum() for p in model.parameters()))
    assert abs(checksum - fx["weight_checksum"]) <= 1e-6 * max(1.0, abs(fx["weight_checksum"]))
    return fx, model, shared


@needs_reference
@pytest.mark.parametrize("d,heads,nhid,nlayers", [(96, 8, 1536, 3), (200, 1, 200, 1), (512, 1, 512, 1)])
def test_synthetic_fixed_model_equals_the_reference_transformer(d, heads, nhid, nlayers):
    refshim.import_reference()
    from breaching.cases.models.language_models import TransformerModel

    torch.manual_seed(5)
    ours = synthetic.TransformerLM(30, d, heads, nhid, nlayers, positional="fixed").eval()
    ref = TransformerModel(30, d, heads, nhid, nlayers, dropout=0.0, positional_embedding="fixed").eval()
    assert torch.equal(ours.pos_encoder.pe, ref.pos_encoder.pe)                 # the same float32 table, bit for bit
    assert [n for n, _ in ours.named_parameters()] == [n for n, _ in ref.named_parameters()]
    assert [n for n, _ in ours.named_buffers()] == [n for n, _ in ref.named_buffers()]
    ref.load_state_dict(ours.state_dict())
    x = torch.randn(2, 9, d)
    with sdpa_kernel(SDPBackend.MATH):
        yo, yr = ours(inputs_embeds=x), ref(None, inputs_embeds=x)
        assert torch.equal(yo, yr)
        q = torch.randn(2, 9, 30).softmax(-1)
        attacked = lambda m: [p for n, p in m.named_parameters() if n != "encoder.weight"]  # noqa: E731
        go = torch.autograd.grad(synthetic.causal_loss(yo, q), attacked(ours))
        gr = torch.autograd.grad(synthetic.causal_loss(yr, q), attacked(ref))
    assert len(go) == len(gr) and all(torch.equal(a, b) for a, b in zip(go, gr))


@pytest.mark.parametrize("name", FIXTURES)
def test_program_adds_the_reference_table_as_a_constant(name):
    fx, model, _ = _case(name)
    B, T = fx["case"]["batch"], fx["case"]["seq_len"]
    prog = compiler.compile_transformer(model, B, T)
    op = prog.ops[0]
    assert op.kind == compiler.OP_POSCONST and op.w == -1 and op.tin == 0 and op.S == T
    assert op.table.dtype == torch.float32 and torch.equal(op.table, fx["pe"])   # the reference's pe[0, :T], bit for bit
    names = [n for n, _ in model.named_parameters() if n != "encoder.weight"]
    assert len(prog.params) == len(names) and [p.shape for p in prog.params] == [tuple(p.shape) for n, p in model.named_parameters()
                                                                                  if n != "encoder.weight"]
    assert all(o.kind != compiler.OP_POSADD for o in prog.ops)


def test_learnable_program_is_unchanged():
    model = synthetic.make_text_case()[0]
    prog = compiler.compile_transformer(model, 1, 8)
    assert prog.ops[0].kind == compiler.OP_POSADD and prog.ops[0].table is None
    assert prog.ops[0].w == [n for n, _ in model.named_parameters() if n != "encoder.weight"].index("pos_encoder.embedding.weight")
    assert all(op.kind != compiler.OP_POSCONST for op in prog.ops)


@pytest.mark.parametrize("name", FIXTURES)
def test_float64_sweeps_reproduce_the_reference_tag_closure(name):
    """The float64 sweeps with the constant table against the reference attacker's closure on its own fixed-position model."""
    from helpers import cfg_from_fixture
    from oracle.program_interp import objective_direction

    fx, model, shared = _case(name)
    cfg = cfg_from_fixture(fx)
    names = [n for n, _ in model.named_parameters()]
    g = [t.double() for t in shared[0]["gradients"]]
    g.pop(names.index("encoder.weight"))
    fs = FixedPositionFourSweep(model.double())
    q = fx["l0"].double().softmax(dim=-1)
    fs.forward(fx["x0"].double(), q)
    G = fs.backward()
    assert len(G) == len(g)
    o = cfg.objective
    val, V = objective_direction(o.type, G, g, scale=o.scale, tag_scale=o.tag_scale, scale_scheme=o.scale_scheme)
    assert abs(float(val) - fx["objective0"]) < 1e-5 * abs(fx["objective0"]), (float(val), fx["objective0"])
    fs.tangent_forward(V)
    dx, dq = fs.tangent_backward()
    dl = q * (dq - (q * dq).sum(dim=-1, keepdim=True))
    assert _relerr(dx, fx["raw_grad_x0"]) < 1e-4, _relerr(dx, fx["raw_grad_x0"])
    assert _relerr(dl, fx["raw_grad_l0"]) < 1e-4, _relerr(dl, fx["raw_grad_l0"])


def test_tied_weights_and_positional_dropout_are_refused():
    model = synthetic.TransformerLM(20, 16, 2, 24, 1, positional="fixed").eval()
    model.decoder.weight = model.encoder.weight                    # transformer3t
    with pytest.raises(compiler.UnsupportedModelError, match="tied"):
        compiler.compile_transformer(model, 1, 8)
    model = synthetic.TransformerLM(20, 16, 2, 24, 1, positional="fixed").eval()
    model.pos_encoder.dropout.p = 0.1
    with pytest.raises(compiler.UnsupportedModelError, match="dropout"):
        compiler.compile_transformer(model, 1, 8)
    with pytest.raises(compiler.UnsupportedModelError, match="does not cover"):
        compiler.compile_transformer(synthetic.TransformerLM(20, 16, 2, 24, 1, max_positions=4, positional="fixed"), 1, 8)
