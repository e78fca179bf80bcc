"""Every sweep buffer of every network of tests/layer_program_cases.py against float64 (oracle/sweep_check.py), on both GEMM back ends:
the column path of the candidate-fed conv with 1-4 channels, candidate-fed convs off it, strided inner convs of every parity-class
shape, max-pools whose windows skip, overlap, pad or tie, two-layer heads and batches 1-64.  Also: the engine takes the column path
exactly where the restated rule says, and its GEMM planner agrees with scripts/profile_gemms.gemm_plan on every GEMM of the case.
A few cases go through two FedAvg local steps (oracle/sweep_check.MultiStepChecker): the column path re-pads the weights every step."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

import test_sweep_multistep_gpu as MS  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402
from breaching_b200 import get_attack_config  # noqa: E402
from layer_program_cases import CASES, MULTISTEP, build, gemm_plans, stem_columns  # noqa: E402
from test_sweep_local_gpu import candidate, check_evaluation, make_engine, pool_fed  # noqa: E402


def attack_config(shape):
    """invertinggradients; its total-variation prior is defined for 3-channel images only."""
    return get_attack_config("invertinggradients", {} if shape[1] == 3 else {"regularization": None})


def check_plans(prog, backend, options):
    for (i, mode, nsrc), (be, g, want) in gemm_plans(prog, backend, options).items():
        N, H, W, Ci, Co, R, st, pd = g
        got = E.gemm_plan(mode, 0 if be == "nchw" else be, N, H, W, Ci, Co, R, R, st, pd, nsrc)
        if be == "nchw":   # the NCHW candidate operand: the planner's NHWC form decides the family, not the vector loaders
            got, want = got["family"], want["family"]
        assert got == want, (i, mode, nsrc, be, g, got, want)


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", list(CASES))
def test_every_sweep_buffer_of_the_case(name, backend):
    model, shape, labels, grads, options = build(name)
    cfg = attack_config(shape)
    eng = make_engine(model, shape, cfg, labels, grads, backend, options=options)
    try:
        chk = check_evaluation(eng, candidate(shape), model, grads, labels, cfg, None, f"{name} / {backend}")
        assert chk.stem == [i for i in range(len(eng.prog.ops)) if stem_columns(eng.prog, i, backend, options)]
        check_plans(eng.prog, backend, options)
    finally:
        eng.close()


def fedavg_case(name, steps=2, lr=1e-2, model_shape=None):
    """The case as a FedAvg update: ``steps`` SGD steps on consecutive slices of twice the case's batch (synthetic.make_fedavg_case),
    in MS.build_case's form.  ``model_shape``: (model, input shape) of another network instead of the named case's."""
    model, shape = model_shape or build(name)[:2]
    dps, n = shape[0], 2 * shape[0]
    gen = torch.Generator().manual_seed(23)
    x = torch.randn((n, *shape[1:]), generator=gen)
    y = torch.randint(0, 10, (n,), generator=gen)
    server = [p.detach().clone() for p in model.parameters()]
    m = copy.deepcopy(model).eval()
    opt = torch.optim.SGD(m.parameters(), lr=lr)
    labels = []
    for k in range(steps):
        sl = slice((k * dps) % n, (k * dps) % n + dps)
        labels.append(y[sl].sort()[0])
        opt.zero_grad()
        torch.nn.functional.cross_entropy(m(x[sl]), y[sl]).backward()
        opt.step()
    shared = [dict(gradients=[(a - b).detach() for a, b in zip(m.parameters(), server)], buffers=None)]
    hyper = dict(lr=lr, steps=steps, data_per_step=dps, labels=labels)
    cand = torch.randn((n, *shape[1:]), generator=torch.Generator().manual_seed(4))
    return model, shared, hyper, attack_config(shape), cand, ((0.0,) * shape[1], (1.0,) * shape[1])


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", MULTISTEP)
def test_every_step_buffer_of_the_case(name, backend):
    chk = MS.check_engine(name, backend, case=fedavg_case(name))
    assert {i for _, i in chk.off_grid} <= pool_fed(chk.prog), sorted(chk.off_grid)
    assert chk.stem == [i for i in range(len(chk.prog.ops)) if stem_columns(chk.prog, i, backend)]
