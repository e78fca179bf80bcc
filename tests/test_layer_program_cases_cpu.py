"""The layer-geometry table (tests/layer_program_cases.py) on the CPU: every case compiles, its float64 four-sweep formulation
(oracle/program_interp.py) equals autograd's double backward, and the table reaches every engine rule it is meant to reach -- each
case reaching at least one rule no other case does."""
import pytest
import torch

from breaching_b200 import compiler, config
from layer_program_cases import CASES, REQUIRED, build, reached
from oracle import program_interp as PI
from oracle import restate


def _oracle(name, kind, treg):
    model, shape, labels, grads, _ = build(name)
    model = model.double()
    x = torch.randn(shape, dtype=torch.double, generator=torch.Generator().manual_seed(5))
    cfg = config.get_attack_config("invertinggradients", {"objective.type": kind, "objective.task_regularization": treg,
                                                           "regularization": None})
    g = [t.double() for t in grads]
    dm, ds = torch.zeros(1, shape[1], 1, 1), torch.ones(1, shape[1], 1, 1)
    return model, x, labels, g, restate.TrialOracle(model, torch.nn.CrossEntropyLoss(), cfg, g, labels, dm, ds, dtype=torch.double)


@pytest.mark.parametrize("name", list(CASES))
def test_case_compiles(name):
    model, shape, *_ = build(name)
    prog = compiler.compile_model(model, shape)
    assert prog.tensors[prog.logits].C == 10 and prog.tensors[0].N == shape[0]


@pytest.mark.parametrize("kind,treg", [("cosine-similarity", 0.3), ("euclidean", 0.0)])
@pytest.mark.parametrize("name", list(CASES))
def test_four_sweeps_match_double_backward(name, kind, treg):
    model, x, labels, g, orc = _oracle(name, kind, treg)
    phi, _, raw, _ = orc.closure_gradient(x, 0, 0.1)
    it = PI.ProgramInterpreter(model, compiler.compile_model(model, x.shape))
    val, dx, _, G = it.matching_gradient(x, labels, g, kind, scale=1.0, task_regularization=treg)
    assert abs(float(val) - float(phi)) < 1e-10 * max(1.0, abs(float(phi)))
    assert ((dx - raw).norm() / raw.norm()).item() < 1e-10
    Gref, _ = orc.param_gradient(x, False)
    scale = max(b.abs().max().item() for b in Gref)   # conv biases in front of a train-mode BN have an exactly-zero gradient
    for a, b in zip(G, Gref):
        assert (a - b).abs().max().item() <= 1e-10 * b.abs().max().item() + 1e-13 * scale


def test_table_reaches_every_rule():
    got = {name: reached(name, "simt") | reached(name, "tc") for name in CASES}
    missing = REQUIRED - set().union(*got.values())
    assert not missing, sorted(missing, key=repr)
    for name in CASES:   # no entry is redundant: dropping any one loses a rule
        others = set().union(*(r for n, r in got.items() if n != name))
        assert REQUIRED & got[name] - others, f"{name} reaches no rule that another case does not"
