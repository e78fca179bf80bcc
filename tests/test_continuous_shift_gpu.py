"""continuous_shift with every option of the reference's RandomTransform on the engine: the device view and its pull-back against the
unmodified module's float64 views and vector-Jacobian products (tests/golden/continuous_shift.pt), the adjoint identity, one closure
evaluation against the float64 trial oracle with the draws read back from the device, the draws and launches of the options accepted
before, and an attack end to end with the module's default reflection padding."""
import copy
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import load_golden  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.attacks import augment  # noqa: E402
from cshift_oracle import ShiftTrialOracle, apply, continuous_shift, randgen_from_draws  # noqa: E402
from oracle import restate  # noqa: E402

DEV = torch.device("cuda:0")
ULP = 2.0 ** -24


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _device_kwargs(c):
    r = c["randgen"]
    lr = [int(c["fliplr"] and v > 0.5) for v in r[:, 2].tolist()]
    ud = [int(c["flipud"] and v > 0.5) for v in r[:, 3].tolist()]
    return dict(continuous_shift=float(c["shift"]), circular=c["padding"] == "circular", uniforms=(r[:, 0].tolist(), r[:, 1].tolist()),
                mode=c["mode"], padding="zeros" if c["padding"] == "circular" else c["padding"], flips=(lr, ud))


def _case_id(c):
    return f"{c['mode']}-{c['padding']}-lr{int(c['fliplr'])}-ud{int(c['flipud'])}-S{c['S']}-shift{c['shift']}"


FIXTURE = load_golden("continuous_shift.pt")


@pytest.mark.parametrize("case", FIXTURE["cases"], ids=_case_id)
def test_view_and_pullback_against_the_reference_module(case):
    inp = FIXTURE["inputs"][case["S"]]
    x, g = inp["x"], inp["probe"]
    kw = _device_kwargs(case)
    view = E.augment_view(x.float().to(DEV), **kw).double().cpu()
    pulled = E.augment_view(g.float().to(DEV), transpose=True, **kw).double().cpu()
    # the Jacobian of the float64 restatement: |J| |x| and |J|^T |g| bound the fp32 rounding of every element
    f = lambda t: continuous_shift(t, case["shift"], case["randgen"], case["mode"], case["padding"], case["fliplr"], case["flipud"])  # noqa: E731
    J = torch.autograd.functional.jacobian(f, x).reshape(x.numel(), x.numel()).abs()
    xf, gf = x.float().double().reshape(-1), g.float().double().reshape(-1)
    bound_view = (8 * ULP * (J @ xf.abs())).reshape(x.shape)
    bound_pull = (8 * ULP * (J.T @ gf.abs())).reshape(x.shape)
    if case["mode"] == "nearest":
        assert torch.equal(view.float(), case["view"].float()), (view - case["view"]).abs().max().item()
    else:
        err = (view - case["view"]).abs()
        assert (err <= bound_view + 1e-300).all(), (err - bound_view).max().item()
    err = (pulled - case["vjp"]).abs()
    assert (err <= bound_pull + 1e-300).all(), (err - bound_pull).max().item()
    # adjoint identity in float64 of the device's own view and pull-back, relative to the size of its terms (sum |w| |x| |g|: the
    # bicubic weights have both signs, so the inner product itself may cancel)
    lhs = (view * gf.reshape(x.shape)).sum().item()
    rhs = (xf.reshape(x.shape) * pulled).sum().item()
    scale = ((J @ xf.abs()) * gf.abs()).sum().item()
    assert abs(lhs - rhs) <= 1e-6 * scale, (lhs, rhs, scale)
    assert torch.equal(pulled, E.augment_view(g.float().to(DEV), transpose=True, **kw).double().cpu())   # fixed-order gathers


def test_unknown_modes_are_refused_by_the_stand_alone_view():
    x = torch.zeros(1, 1, 8, 8, device=DEV)
    with pytest.raises(ValueError):
        E.augment_view(x, continuous_shift=2.0, uniforms=([0.5], [0.5]), mode="area")
    with pytest.raises(E.EngineError):     # circular wraps the grid and pads with zeros
        E.augment_view(x, continuous_shift=2.0, circular=True, uniforms=([0.5], [0.5]), padding="reflection")


CLOSURES = {
    "shape_keeping": {"discrete_shift": {"lim": 3},
                      "continuous_shift": {"shift": 5, "padding": "reflection", "mode": "bicubic", "fliplr": True, "flipud": True},
                      "colorjitter": {"mean": 0.1, "std": 0.3}},
    "staged": {"continuous_shift": {"shift": 6, "padding": "reflection", "mode": "bicubic", "fliplr": True, "flipud": True},
               "flip": {"p": 0.5}},
}


@pytest.mark.parametrize("differentiable", [True, False])
@pytest.mark.parametrize("name", sorted(CLOSURES))
def test_closure_matches_the_float64_oracle(name, differentiable):
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=2, seed=8, bn_random=True)
    cfg = get_attack_config("invertinggradients", {"augmentations": CLOSURES[name], "differentiable_augmentations": differentiable,
                                                   "objective.task_regularization": 0.2})
    meta = payload[0]["metadata"]
    torch.manual_seed(5)
    plan = augment.build_plan(cfg, 2, 3, dict(device=DEV, dtype=torch.float), spatial=(32, 32))
    assert (len(plan.stages) == 2) == (name == "staged")
    eng = E.Engine(copy.deepcopy(model).to(DEV).eval(), (2, 3, 32, 32), cfg, DEV, backend="simt")
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], true["labels"].to(DEV), mean=meta.mean, std=meta.std)
    eng.set_augmentations(plan)
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(4))
    val, grad = eng.objective_and_gradient(x.to(DEV))
    draws, flips = eng.augmentation_draws(), eng.augmentation_flips()
    opts = CLOSURES[name]["continuous_shift"]
    shift_kw = lambda k: dict(shift=float(opts["shift"]), mode=opts["mode"], padding=opts["padding"], fliplr=True, flipud=True,  # noqa: E731
                              randgen=randgen_from_draws(draws[k]["sx"], draws[k]["sy"], flips[k]["fliplr"], flips[k]["flipud"]))
    if name == "staged":
        entries = [("continuous_shift", {}, shift_kw(0)), ("pixel", {}, dict(steps=[(2, 0.5)], offsets=[(draws[1]["o1"][0], 0)]))]
    else:
        st = plan
        std = (1 / st.colour_scale).double().cpu().view(2, 3, 1, 1)
        mean = (-st.colour_shift / st.colour_scale).double().cpu().view(2, 3, 1, 1)
        entries = [("pixel", {}, dict(steps=st.steps, offsets=[(draws[0]["o1"][0], draws[0]["o2"][0])])),
                   ("continuous_shift", {}, shift_kw(0)),
                   ("pixel", {}, dict(colour_mean=mean, colour_std=std))]
    dm, ds = torch.tensor(meta.mean)[None, :, None, None].double(), torch.tensor(meta.std)[None, :, None, None].double()
    orc = ShiftTrialOracle(copy.deepcopy(model).double().eval(), loss_fn, cfg, [g.double() for g in shared[0]["gradients"]], true["labels"],
                           dm, ds, dtype=torch.float64, entries=entries)
    xd = x.double().requires_grad_(True)
    if differentiable:
        total, terms = orc.objective_terms(xd)
        (gref,) = torch.autograd.grad(total, xd)
    else:     # the candidate is replaced by its view, and the gradient is taken there
        xa = apply(xd, entries).detach().requires_grad_(True)
        assert (eng.candidate().cpu().double() - xa.detach()).abs().max().item() < 2e-5
        total, terms = restate.TrialOracle.objective_terms(orc, xa)
        (gref,) = torch.autograd.grad(total, xa)
    assert math.isclose(val, float(total), rel_tol=2e-4), (val, float(total), terms, eng.last_terms())
    assert _relerr(grad, gref) < 2e-3, _relerr(grad, gref)
    eng.close()
    orc.close()


def test_plans_accepted_before_draw_and_view_as_the_parameterless_entry_points():
    """The extended entry points with the default options against the original ones, side by side: the same draws, the same view and
    gradient bit for bit, and the launches of the original pipeline (draw, view, two continuous-shift gathers, permutation pull)."""
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=2, seed=8, bn_random=True)
    aug = {"discrete_shift": {"lim": 5}, "flip": {"p": 0.5}, "continuous_shift": {"shift": 6, "padding": "circular"},
           "colorjitter": {"mean": 0.1, "std": 0.3}}
    cfg = get_attack_config("invertinggradients", {"augmentations": aug, "differentiable_augmentations": True})
    meta = payload[0]["metadata"]
    torch.manual_seed(5)
    plan = augment.build_plan(cfg, 2, 3, dict(device=DEV, dtype=torch.float))
    from breaching_b200.schedule import lr_table

    table = lr_table(0.1, "step-lr", 0, 10)
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(4)).to(DEV)
    results = []
    for extended in (False, True):
        eng = E.Engine(copy.deepcopy(model).to(DEV).eval(), (2, 3, 32, 32), cfg, DEV, backend="simt")
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], true["labels"].to(DEV), mean=meta.mean, std=meta.std)
        eng.begin_trial(x, table)
        eng.run(1)
        plain = eng.launches_per_iteration()
        if extended:
            eng.set_augmentations(plan)
        else:
            n = len(plan.steps)
            kinds = (ctypes.c_int32 * n)(*[k for k, _ in plan.steps])
            params = (ctypes.c_float * n)(*[float(p) for _, p in plan.steps])
            sc, sh = plan.colour_scale.to(DEV).contiguous(), plan.colour_shift.to(DEV).contiguous()
            torch.cuda.synchronize()
            E._check(eng.lib, eng.lib.bre_engine_set_augmentations(eng.h, n, kinds, params, 1, 6.0, 1, sc.data_ptr(), sh.data_ptr(), 1, plan.seed),
                     "bre_engine_set_augmentations")
        val, grad = eng.objective_and_gradient(x)
        draws = eng.last_augmentation()
        view = eng.debug_tensor("val", 0).clone()
        eng.begin_trial(x, table)
        eng.run(1)
        results.append((val, grad.cpu(), draws, view.cpu(), eng.launches_per_iteration() - plain, eng.augmentation_flips()))
        eng.close()
    (v0, g0, d0, w0, l0, f0), (v1, g1, d1, w1, l1, f1) = results
    assert d0 == d1 and torch.equal(w0, w1) and torch.equal(g0, g1) and v0 == v1
    assert l0 == l1
    assert all(not any(f["fliplr"]) and not any(f["flipud"]) for f in f0 + f1)
    # the stand-alone view: bre_augment_view against bre_augment_view_ex with the default options
    lib = E.load_library()
    xs = torch.randn(2, 3, 18, 18, generator=torch.Generator().manual_seed(11)).to(DEV)
    outs = []
    for fn in ("old", "new"):
        out = torch.empty_like(xs)
        sx, sy = (ctypes.c_float * 2)(0.31, 0.5), (ctypes.c_float * 2)(0.97, 0.02)
        kinds, o1, o2 = (ctypes.c_int32 * 1)(1), (ctypes.c_int32 * 1)(2), (ctypes.c_int32 * 1)(-1)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        if fn == "old":
            rc = lib.bre_augment_view(xs.data_ptr(), out.data_ptr(), 2, 3, 18, 18, 1, kinds, o1, o2, 20.0, 1, sx, sy, None, None, 0, None, stream)
        else:
            rc = lib.bre_augment_view_ex(xs.data_ptr(), out.data_ptr(), 2, 3, 18, 18, 1, kinds, o1, o2, 20.0, 1, 0, 0, sx, sy, None, None, None,
                                         None, 0, None, stream)
        assert rc == 0
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])


def test_multiscale_preset_with_reflection_padding_runs():
    """multiscale_ghiasi.yaml with the module's default padding (reflection) instead of the preset's circular one."""
    from breaching_b200.attacks import prepare_attack

    model, loss_fn, payload, shared, true = synthetic.make_case("resnet18", "imagenet", batch=1, seed=4, bn_random=True, image_size=64, classes=10)
    cfg = get_attack_config("multiscale_ghiasi", {"num_stages": 2, "scale_pyramid": "log", "optim.max_iterations": 5, "optim.callback": 5,
                                                  "augmentations.continuous_shift.padding": "reflection"})
    assert cfg.augmentations.continuous_shift.padding == "reflection"
    torch.manual_seed(1)
    rec, stats = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == (1, 3, 64, 64) and torch.isfinite(rec["data"]).all() and len(stats["Trial_0_Val"]) == 10
    assert all(math.isfinite(v) for v in stats["Trial_0_Val"])
