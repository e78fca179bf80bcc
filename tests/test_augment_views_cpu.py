"""Shape-changing augmentations (zoom, centerzoom, focus, antialias) without a GPU: the float64 restatements of oracle/augment_views.py
against the reference modules' outputs and vector-Jacobian products (tests/golden/augment_views.pt), the oracle closure and trajectory
with a centerzoom + antialias view against the reference attack, and the plan / shape / refusal logic of attacks/augment.py."""
import copy
import math

import pytest
import torch

from helpers import case_from_fixture, cfg_from_fixture, load_golden
from breaching_b200 import get_attack_config
from breaching_b200.attacks import augment
from oracle import augment_views as AV
from oracle import restate

SETUP = dict(device=torch.device("cpu"), dtype=torch.float)


def _restated(entry, x):
    kw = entry["kwargs"]
    if entry["name"] == "Zoom":
        return AV.zoom(x, kw["out_size"])
    if entry["name"] == "CenterZoom":
        return AV.centerzoom(x, kw["initial_fov"], kw["out_size"])
    if entry["name"] == "Focus":
        return AV.focus(x, kw["size"], pert=entry["pert"])
    return AV.antialias(x, kw["width"], kw["stride"], kw["channels"])


def test_restatements_equal_the_reference_modules():
    fx = load_golden("augment_views.pt")["modules"]
    assert {e["name"] for e in fx} == {"Zoom", "CenterZoom", "Focus", "AntiAlias"}
    assert {e["kwargs"]["width"] for e in fx if e["name"] == "AntiAlias"} == set(range(1, 8))
    for entry in fx:
        x = entry["x"].clone().requires_grad_(True)
        y = _restated(entry, x)
        assert y.shape == entry["y"].shape, entry["name"]
        assert (y.detach() - entry["y"]).abs().max().item() < 1e-12, entry["name"]
        (vjp,) = torch.autograd.grad((y * entry["g"]).sum(), x)
        assert (vjp - entry["vjp"]).abs().max().item() < 1e-12, entry["name"]


def _trial_oracle(fx):
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    m = copy.deepcopy(model)
    if shared[0]["buffers"] is not None:
        for buf, src in zip(m.buffers(), shared[0]["buffers"]):
            buf.data.copy_(src)
    m.eval()
    meta = payload[0]["metadata"]
    dm, ds = torch.tensor(meta.mean)[None, :, None, None], torch.tensor(meta.std)[None, :, None, None]
    labels = restate.recover_labels(cfg.label_strategy, shared, shared[0]["metadata"]["num_data_points"])
    aug = cfg.augmentations
    entries = [(k, dict(aug[k]), None) for k in aug.keys()]
    return AV.ViewTrialOracle(m, loss_fn, cfg, shared[0]["gradients"], labels, dm, ds, entries=entries), labels


def test_view_oracle_reproduces_the_reference_closure_and_trajectory():
    fx = load_golden("augment_views.pt")["trial"]
    orc, labels = _trial_oracle(fx)
    assert labels.tolist() == fx["labels"].tolist()
    phi0, _, raw, _ = orc.closure_gradient(fx["x0"], 0, 0.0)
    assert math.isclose(float(phi0), fx["objective0"], rel_tol=1e-5, abs_tol=1e-7)
    assert ((raw - fx["raw_grad0"]).norm() / fx["raw_grad0"].norm()).item() < 1e-4
    best, hist, trace = orc.run(fx["x0"], iterations=fx["iters"], record=True)
    assert len(hist) == len(fx["history"])
    for a, b in zip(hist, fx["history"]):
        assert math.isclose(a, b, rel_tol=2e-4, abs_tol=1e-6), (hist, fx["history"])
    assert (trace[0]["candidate"] - fx["candidate_after_1"]).abs().max().item() < 1e-4
    assert (trace[-1]["candidate"] - fx["candidate_final"]).abs().mean().item() < 2e-3
    assert math.isclose(orc.score(best, fx["scoring"]), fx["score"], rel_tol=5e-2, abs_tol=1e-5)
    # the view matters: without it the closure is a different function
    plain = restate.TrialOracle(orc.model, orc.loss_fn, orc.cfg, orc.g, orc.labels, orc.dm, orc.ds)
    assert not math.isclose(float(plain.closure_gradient(fx["x0"], 0, 0.0)[0]), fx["objective0"], rel_tol=1e-3)
    orc.close()


def _cfg(augs, differentiable=True):
    return get_attack_config("invertinggradients", {"augmentations": augs, "differentiable_augmentations": differentiable})


@pytest.mark.parametrize("augs, shape, want", [
    ({"zoom": {"out_size": 24}}, (2, 3, 12, 10), (2, 3, 24, 24)),
    ({"zoom": {"out_size": 6}}, (2, 3, 12, 10), (2, 3, 6, 6)),
    ({"centerzoom": {"initial_fov": 8, "out_size": 20}}, (1, 3, 12, 16), (1, 3, 20, 20)),
    ({"focus": {"size": 7, "std": 1.0}}, (1, 3, 12, 16), (1, 3, 7, 7)),
    ({"antialias": {"width": 5}}, (1, 3, 12, 16), (1, 3, 12, 16)),
    ({"antialias": {"width": 4}}, (1, 3, 12, 16), (1, 3, 13, 17)),
    ({"antialias": {"width": 3, "stride": 2}}, (1, 3, 12, 15), (1, 3, 6, 8)),
    ({"flip": {}, "centerzoom": {"initial_fov": 8, "out_size": 16}, "antialias": {"width": 2}}, (1, 3, 12, 12), (1, 3, 17, 17)),
    ({"discrete_shift": {"lim": 2}, "flip": {}}, (1, 3, 12, 10), (1, 3, 12, 10)),
])
def test_view_shape_follows_each_stage(augs, shape, want):
    cfg = _cfg(augs)
    assert augment.view_shape(cfg, shape) == want
    plan = augment.build_plan(cfg, shape[0], shape[1], SETUP, spatial=shape[2:])
    if augment.has_view_stages(cfg):
        assert plan.candidate_shape == shape and plan.stages[-1].out_hw == want[2:]
        for a, b in zip(plan.stages, plan.stages[1:]):
            assert a.out_hw == b.in_hw
    else:
        assert plan.stages == [] and plan.candidate_shape is None


def test_stage_geometry():
    plan = augment.build_plan(_cfg({"discrete_shift": {"lim": 3}, "colorjitter": {"mean": 0.1, "std": 0.2}, "centerzoom": {"initial_fov": 7, "out_size": 16},
                                    "flip": {"p": 0.5}, "focus": {"size": 10, "std": 2.0}, "antialias": {"width": 5, "stride": 2}}),
                              2, 3, SETUP, spatial=(13, 12))
    kinds = [s.kind for s in plan.stages]
    assert kinds == [augment.PIXEL, augment.RESAMPLE, augment.PIXEL, augment.RESAMPLE, augment.BLUR]
    p0, cz, p1, fo, bl = plan.stages
    assert p0.steps == [(augment.SHIFT, 3.0)] and p0.colour_scale.shape == (2, 3) and p1.steps == [(augment.FLIP, 0.5)]
    assert cz.corner == (3, 2) and cz.window == (7, 7) and cz.out_hw == (16, 16) and cz.focus_std is None
    assert fo.window == (10, 10) and fo.focus_std == 2.0 and fo.in_hw == (16, 16)
    assert bl.width == 5 and bl.stride == 2 and bl.out_hw == (5, 5)


def test_view_shape_draws_nothing_and_plain_plans_are_unchanged():
    cfg = _cfg({"colorjitter": {"mean": 0.1, "std": 0.2}, "zoom": {"out_size": 32}, "focus": {"size": 16}})
    torch.manual_seed(3)
    state = torch.get_rng_state()
    assert augment.view_shape(cfg, (2, 3, 16, 16)) == (2, 3, 16, 16)
    assert augment.has_view_stages(cfg)
    assert torch.equal(torch.get_rng_state(), state)
    # a config of the shape-keeping kinds draws what it always drew, in the same order, and fills the same fields
    plain = _cfg({"discrete_shift": {"lim": 4}, "colorjitter": {"mean": 0.1, "std": 0.3}, "continuous_shift": {"shift": 3, "padding": "zeros"}})
    torch.manual_seed(9)
    plan = augment.build_plan(plain, 2, 3, SETUP)
    torch.manual_seed(9)
    m = (torch.rand((2, 3, 1, 1)) - 0.5) * 2 * 0.1
    sd = ((torch.rand((2, 3, 1, 1)) - 0.5) * 2 * 0.3).exp()
    seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item())
    assert plan.seed == seed and plan.steps == [(augment.SHIFT, 4.0)] and plan.continuous_shift == 3.0 and not plan.circular
    assert torch.equal(plan.colour_scale, (1 / sd).view(2, 3)) and torch.equal(plan.colour_shift, (-m / sd).view(2, 3))
    assert plan.stages == []


@pytest.mark.parametrize("augs, differentiable, error, match", [
    ({"zoom": {"out_size": 8}}, False, ValueError, "differentiable_augmentations"),
    ({"antialias": {"width": 4}}, False, ValueError, "differentiable_augmentations"),
    ({"focus": {"size": 20}}, True, ValueError, "window does not fit"),
    ({"centerzoom": {"initial_fov": 17, "out_size": 8}}, True, ValueError, "does not fit"),
    ({"antialias": {"channels": 1}}, True, ValueError, "channels"),
    ({"antialias": {"width": 8}}, True, ValueError, "filter bank"),
    ({"antialias": {"width": 0}}, True, ValueError, "filter bank"),
    ({"median": {}}, True, NotImplementedError, "median"),
])
def test_refusals(augs, differentiable, error, match):
    cfg = _cfg(augs, differentiable)
    with pytest.raises(error, match=match):
        augment.view_shape(cfg, (1, 3, 16, 16)) if "median" not in augs else None
        augment.build_plan(cfg, 1, 3, SETUP, spatial=(16, 16))


def test_shape_keeping_stages_run_without_the_differentiable_mode():
    """antialias of odd width at stride 1 keeps the shape, so the reference's non-differentiable mode (the candidate becomes its view)
    stays well defined and is allowed, as it is for the shift / flip / colour kinds."""
    cfg = _cfg({"antialias": {"width": 3}}, False)
    assert augment.view_shape(cfg, (1, 3, 16, 16)) == (1, 3, 16, 16)
    plan = augment.build_plan(cfg, 1, 3, SETUP, spatial=(16, 16))
    assert not plan.differentiable and [s.kind for s in plan.stages] == [augment.BLUR]


def test_a_plan_for_another_resolution_keeps_its_draws_and_draws_nothing():
    """Multi-scale stages reuse the attacker's plan: colour constants and seed drawn once (the reference's ColorJitter keeps its
    constants for the whole attacker), stage geometry recomputed for each stage's candidate."""
    cfg = _cfg({"colorjitter": {"mean": 0.1, "std": 0.2}, "focus": {"size": 12, "std": 1.0}, "flip": {}, "zoom": {"out_size": 32}})
    torch.manual_seed(4)
    plan = augment.build_plan(cfg, 2, 3, SETUP, spatial=(32, 32))
    state = torch.get_rng_state()
    small = augment.with_spatial(plan, cfg, (16, 16))
    assert torch.equal(torch.get_rng_state(), state)
    assert small.seed == plan.seed and small.candidate_shape == (2, 3, 16, 16) and plan.candidate_shape == (2, 3, 32, 32)
    assert [s.kind for s in small.stages] == [s.kind for s in plan.stages]
    assert small.stages[0].colour_scale is plan.stages[0].colour_scale and small.stages[0].in_hw == (16, 16)
    assert small.stages[1].window == (12, 12) and small.stages[1].in_hw == (16, 16) and small.stages[2].in_hw == (12, 12)
    assert small.stages[-1].out_hw == (32, 32)
    torch.manual_seed(4)
    direct = augment.build_plan(cfg, 2, 3, SETUP, spatial=(16, 16))
    for a, b in zip(small.stages, direct.stages):
        assert (a.kind, a.in_hw, a.out_hw, a.corner, a.window, a.steps) == (b.kind, b.in_hw, b.out_hw, b.corner, b.window, b.steps)
    with pytest.raises(ValueError, match="does not fit"):
        augment.with_spatial(plan, cfg, (8, 8))


def test_scoring_engines_go_through_the_multiscale_override(monkeypatch):
    """The scoring engine of a resizing view is built through ``_get_engine``; the multi-scale attacker's override must pass the
    request on (compiled at the candidate's shape, no noise seed drawn), and the engine is built once per shape."""
    from types import SimpleNamespace

    from breaching_b200.attacks import optimization_attack as OA
    from breaching_b200.attacks.multiscale_attack import MultiScaleOptimizationAttacker

    calls = []

    def fake_get_engine(self, rec_models, shared_data, labels, index=0, cfg=None, data_shape=None, primary=True, for_scoring=False):
        calls.append(dict(data_shape=data_shape, primary=primary, for_scoring=for_scoring))
        return SimpleNamespace(prog=SimpleNamespace(tensors=[SimpleNamespace(N=1, C=3, H=data_shape[1], W=data_shape[2])]))

    monkeypatch.setattr(OA.OptimizationBasedAttacker, "_get_engine", fake_get_engine)
    att = MultiScaleOptimizationAttacker.__new__(MultiScaleOptimizationAttacker)
    att._score_context = ([object()], [{}], None)
    trial_engine = SimpleNamespace(prog=SimpleNamespace(tensors=[SimpleNamespace(N=1, C=3, H=65, W=65)]))
    cand = torch.zeros(1, 3, 64, 64)
    eng = att._scoring_engine(trial_engine, cand)
    assert eng is not trial_engine and calls == [dict(data_shape=(3, 64, 64), primary=False, for_scoring=True)]
    assert att._scoring_engine(trial_engine, cand) is eng and len(calls) == 1
    same = SimpleNamespace(prog=SimpleNamespace(tensors=[SimpleNamespace(N=1, C=3, H=64, W=64)]))
    assert att._scoring_engine(same, cand) is same
