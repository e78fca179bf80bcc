"""Shape-changing augmentations on the engine (zoom, centerzoom, focus, antialias; reference attacks/auxiliaries/augmentations.py, closure
at optimization_based_attack.py:149-162 with differentiable_augmentations): the RESAMPLE / BLUR kernels and their pull-backs against the
float64 restatements of oracle/augment_views.py, one closure evaluation with every buffer that crosses the view checked in float64,
the trajectory against the reference fixture, and the attacker paths (scoring at the candidate's shape, multi-scale stages at the
view's shape)."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from helpers import case_from_fixture, cfg_from_fixture, load_golden  # noqa: E402
from breaching_b200 import engine as E  # noqa: E402
from breaching_b200 import get_attack_config, synthetic  # noqa: E402
from breaching_b200.attacks import augment  # noqa: E402
from oracle import augment_views as AV  # noqa: E402
from oracle import restate  # noqa: E402

DEV = torch.device("cuda:0")


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


RESAMPLE_CASES = [   # (input shape, corner, window, output)
    ((2, 3, 11, 14), (0, 0), (11, 14), (17, 17)),     # zoom up, non-square input
    ((2, 3, 11, 14), (0, 0), (11, 14), (5, 6)),       # zoom down
    ((1, 3, 13, 10), (3, 1), (7, 7), (19, 19)),       # centerzoom-like window, up
    ((1, 3, 13, 10), (2, 2), (9, 6), (4, 4)),         # window, down
    ((2, 2, 15, 12), (4, 5), (6, 6), (6, 6)),         # focus: exact copy of the window
]


@pytest.mark.parametrize("shape, corner, window, out", RESAMPLE_CASES)
def test_resample_view_and_pullback_against_float64(shape, corner, window, out):
    gen = torch.Generator().manual_seed(sum(shape) + sum(out))
    x = torch.randn(shape, generator=gen)
    g = torch.randn((*shape[:2], *out), generator=gen)
    xd = x.double().requires_grad_(True)
    crop = xd[:, :, corner[0]:corner[0] + window[0], corner[1]:corner[1] + window[1]]
    want = torch.nn.functional.interpolate(crop, size=out, mode="bilinear", align_corners=False)
    (gwant,) = torch.autograd.grad((want * g.double()).sum(), xd)
    got = E.augment_resample(x.to(DEV), corner, window, out)
    assert (got.cpu().double() - want.detach()).abs().max().item() < 2e-5
    pulled = E.augment_resample(g.to(DEV), corner, window, out, transpose=True, in_hw=shape[2:])
    assert _relerr(pulled, gwant) < 1e-5, _relerr(pulled, gwant)
    # adjoint identity and run-to-run bitwise reproducibility of the gather
    lhs = (got.double() * g.to(DEV).double()).sum().item()
    rhs = (x.to(DEV).double() * pulled.double()).sum().item()
    assert math.isclose(lhs, rhs, rel_tol=1e-5, abs_tol=1e-5), (lhs, rhs)
    again = E.augment_resample(g.to(DEV), corner, window, out, transpose=True, in_hw=shape[2:])
    assert torch.equal(pulled, again)


@pytest.mark.parametrize("width", range(1, 8))
@pytest.mark.parametrize("stride", [1, 2])
def test_blur_view_and_pullback_against_float64(width, stride):
    gen = torch.Generator().manual_seed(10 * width + stride)
    x = torch.randn(2, 3, 9, 12, generator=gen)
    xd = x.double().requires_grad_(True)
    want = AV.antialias(xd, width, stride, 3)
    g = torch.randn(want.shape, generator=gen)
    (gwant,) = torch.autograd.grad((want * g.double()).sum(), xd)
    got = E.augment_blur(x.to(DEV), width, stride)
    assert got.shape == want.shape
    assert (got.cpu().double() - want.detach()).abs().max().item() < 2e-5
    pulled = E.augment_blur(g.to(DEV), width, stride, transpose=True, in_hw=(9, 12))
    assert _relerr(pulled, gwant) < 1e-5, _relerr(pulled, gwant)
    lhs = (got.double() * g.to(DEV).double()).sum().item()
    rhs = (x.to(DEV).double() * pulled.double()).sum().item()
    assert math.isclose(lhs, rhs, rel_tol=1e-5, abs_tol=1e-5), (lhs, rhs)
    assert torch.equal(pulled, E.augment_blur(g.to(DEV), width, stride, transpose=True, in_hw=(9, 12)))


def test_multiscale_resize_and_the_resample_stage_share_the_index_rule():
    x = torch.randn(2, 3, 13, 9, generator=torch.Generator().manual_seed(2)).to(DEV)
    for out in ((26, 18), (5, 4), (13, 9)):
        assert torch.equal(E.resize_bilinear(x, out), E.augment_resample(x, (0, 0), (13, 9), out))


def _resnet_case(seed=8, image=32):
    return synthetic.make_case("resnet18", "imagenet", batch=1, seed=seed, bn_random=True, image_size=image, classes=10)


def _engine(model, cfg, shared, labels, meta, view, backend):
    eng = E.Engine(copy.deepcopy(model).to(DEV).eval(), view, cfg, DEV, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], labels.to(DEV), mean=meta.mean, std=meta.std)
    return eng


def _entries(plan, draws, aug_cfg):
    """The oracle's view entries for a plan and the engine's read-back draws."""
    keys = [k for k in aug_cfg.keys()]
    entries, k_iter = [], iter(keys)
    for i, st in enumerate(plan.stages):
        if st.kind == augment.PIXEL:
            kw = dict(steps=[], offsets=[], continuous_shift=st.continuous_shift, circular=st.circular,
                      uniforms=(draws[i]["sx"], draws[i]["sy"]) if st.continuous_shift is not None else None)
            if st.colour_scale is not None:
                kw["colour_std"] = (1 / st.colour_scale).double().cpu().view(-1, 3, 1, 1)
                kw["colour_mean"] = (-st.colour_shift / st.colour_scale).double().cpu().view(-1, 3, 1, 1)
            entries.append(("pixel", {}, kw))
            continue
        key = next(k for k in k_iter if k in ("zoom", "centerzoom", "focus", "antialias"))
        draw = {"corner": (draws[i]["o1"][0], draws[i]["o2"][0])} if key == "focus" else None
        entries.append((key, dict(aug_cfg[key]), draw))
    return entries


CLOSURE_VIEWS = {
    "centerzoom_antialias_cs_cj": {"centerzoom": {"initial_fov": 20, "out_size": 24}, "antialias": {"width": 3},
                                   "continuous_shift": {"shift": 3, "padding": "circular"}, "colorjitter": {"mean": 0.1, "std": 0.3}},
    "cs_cj_centerzoom_antialias": {"continuous_shift": {"shift": 3, "padding": "zeros"}, "colorjitter": {"mean": 0.1, "std": 0.3},
                                   "centerzoom": {"initial_fov": 20, "out_size": 24}, "antialias": {"width": 4, "stride": 1}},
    "focus_antialias_stride2": {"focus": {"size": 26, "std": 2.0}, "colorjitter": {"mean": 0.1, "std": 0.3}, "antialias": {"width": 5, "stride": 2}},
}


@pytest.mark.parametrize("backend", ["simt", "tc"])
@pytest.mark.parametrize("name", sorted(CLOSURE_VIEWS))
def test_closure_through_a_resizing_view_matches_float64(name, backend):
    model, loss_fn, payload, shared, true = _resnet_case()
    meta = payload[0]["metadata"]
    cfg = get_attack_config("invertinggradients", {"augmentations": CLOSURE_VIEWS[name], "differentiable_augmentations": True,
                                                   "objective.task_regularization": 0.2})
    cand_shape = (1, 3, 32, 32)
    view = augment.view_shape(cfg, cand_shape)
    torch.manual_seed(5)
    plan = augment.build_plan(cfg, 1, 3, dict(device=DEV, dtype=torch.float), spatial=(32, 32))
    eng = _engine(model, cfg, shared, true["labels"], meta, view, backend)
    assert eng.prog.tensors[0].H == view[2] and eng.prog.tensors[0].W == view[3]
    eng.set_augmentations(plan)
    assert eng.input_shape == cand_shape
    x = torch.randn(cand_shape, generator=torch.Generator().manual_seed(4))
    val, grad = eng.objective_and_gradient(x.to(DEV))
    assert grad.shape == cand_shape
    draws = eng.augmentation_draws()
    for st, d in zip(plan.stages, draws):
        if st.kind == augment.RESAMPLE and st.focus_std is not None:     # Focus: clamp(trunc(pert + H // 2 - size // 2))
            c = (32 - st.window[0]) // 2
            assert all(0 <= v <= 32 - st.window[0] and abs(v - c) <= math.ceil(st.focus_std) for v in (d["o1"][0], d["o2"][0])), d
    entries = _entries(plan, draws, cfg.augmentations)
    dm, ds = torch.tensor(meta.mean)[None, :, None, None].double(), torch.tensor(meta.std)[None, :, None, None].double()
    orc = restate.TrialOracle(copy.deepcopy(model).double().eval(), loss_fn, cfg, [g.double() for g in shared[0]["gradients"]],
                              true["labels"], dm, ds, dtype=torch.float64)
    xd = x.double().requires_grad_(True)
    vd = AV.apply(xd, entries)
    # the view buffer (program tensor 0)
    assert (eng.debug_tensor("val", 0).double() - vd.detach()).abs().max().item() < 2e-5
    vleaf = vd.detach().requires_grad_(True)
    total, terms = orc.objective_terms(vleaf)
    (gview,) = torch.autograd.grad(total, vleaf)
    (gx_ref,) = torch.autograd.grad(AV.apply(xd, entries), xd, grad_outputs=gview)
    tol_val, tol_grad = (2e-4, 2e-3) if backend == "simt" else (2e-3, 5e-2)
    assert math.isclose(val, float(total), rel_tol=tol_val), (val, float(total), terms, eng.last_terms())
    assert _relerr(grad, gx_ref) < tol_grad, _relerr(grad, gx_ref)
    if plan.stages[-1].kind != augment.PIXEL or plan.stages[-1].continuous_shift is None:
        # (a last PIXEL stage with a continuous shift uses the view gradient as its pull-back scratch)
        g_eng = eng.debug_tensor("tangent_delta", 0)
        assert _relerr(g_eng, gview) < tol_grad, _relerr(g_eng, gview)
        # the pull-back alone: the float64 VJP of the view applied to the engine's own view gradient
        (pulled_ref,) = torch.autograd.grad(AV.apply(xd, entries), xd, grad_outputs=g_eng.double())
        assert _relerr(grad, pulled_ref) < 1e-5, _relerr(grad, pulled_ref)
    if view != cand_shape:     # the score is taken on the candidate, which this program cannot take
        with pytest.raises(E.EngineError, match="candidate's shape"):
            eng.score(x.to(DEV), "euclidean")
    eng.close()
    orc.close()


def test_trajectory_matches_the_reference_fixture_graph_and_eager():
    fx = load_golden("augment_views.pt")["trial"]
    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    labels = restate.recover_labels(cfg.label_strategy, shared, shared[0]["metadata"]["num_data_points"])
    shape = tuple(fx["x0"].shape)
    from breaching_b200.schedule import lr_table

    opt = cfg.optim
    table = lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations)
    runs = []
    for use_graph in (1, 0):
        eng = _engine(model, cfg, shared, labels, payload[0]["metadata"], augment.view_shape(cfg, shape), "simt")
        eng.set_option("use_graph", use_graph)
        eng.set_augmentations(augment.build_plan(cfg, shape[0], shape[1], dict(device=DEV, dtype=torch.float), spatial=shape[2:]))
        eng.begin_trial(fx["x0"].to(DEV), table)
        eng.run(fx["iters"])
        eng.sync()
        runs.append((eng.history().tolist(), eng.candidate().cpu()))
        eng.close()
    hist, final = runs[0]
    assert len(hist) == fx["iters"]
    for a, b in zip(hist, fx["history"]):
        assert math.isclose(a, b, rel_tol=5e-3, abs_tol=1e-5), (hist, fx["history"])
    assert (final - fx["candidate_final"]).abs().mean().item() < 2e-3
    assert runs[0][0] == runs[1][0] and torch.equal(runs[0][1], runs[1][1])     # captured graph == eager, bitwise


@pytest.mark.parametrize("view", [{"centerzoom": {"initial_fov": 20, "out_size": 24}}, {"focus": {"size": 24, "std": 2.0}}])
def test_reconstruct_returns_the_candidate_shape_and_scores_it_there(view):
    from breaching_b200.attacks import prepare_attack

    model, loss_fn, payload, shared, true = _resnet_case(seed=9)
    cfg = get_attack_config("invertinggradients", {"augmentations": view, "differentiable_augmentations": True, "optim.max_iterations": 4,
                                                   "optim.callback": 4})
    torch.manual_seed(2)
    att = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    rec, stats = att.reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == (1, 3, 32, 32) and torch.isfinite(rec["data"]).all()
    assert att._engine.prog.tensors[0].H == 24 and att._engine.input_shape == (1, 3, 32, 32)
    meta = payload[0]["metadata"]
    dm, ds = torch.tensor(meta.mean)[None, :, None, None], torch.tensor(meta.std)[None, :, None, None]
    orc = restate.TrialOracle(copy.deepcopy(model).eval(), loss_fn, cfg, shared[0]["gradients"], rec["labels"].cpu(), dm, ds)
    want = orc.score(rec["data"].cpu(), cfg.restarts.scoring)
    assert math.isclose(float(stats["opt_value"]), float(want), rel_tol=1e-3), (stats["opt_value"], want)
    orc.close()


def test_scoring_a_resized_view_on_a_fixed_input_model_is_refused():
    """A 16 x 16 candidate zoomed to the 32 x 32 a ConvNet takes: the attack's program exists, the score at the candidate's own
    shape needs one the network's fixed Linear cannot take (the reference's _score_trial fails there as well)."""
    from breaching_b200.attacks import prepare_attack
    from breaching_b200.compiler import UnsupportedModelError

    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=1, seed=3, bn_random=True)
    cfg = get_attack_config("invertinggradients", {"augmentations": {"zoom": {"out_size": 32}}, "differentiable_augmentations": True,
                                                   "optim.max_iterations": 2})
    att = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float))
    rec_models, labels, _, shared_data = att.prepare_attack(payload, copy.deepcopy(shared))
    att._score_context = (rec_models, shared_data, labels)
    eng = att._get_engine(rec_models, shared_data, labels, data_shape=(3, 16, 16))
    assert eng.prog.tensors[0].H == 32
    with pytest.raises(UnsupportedModelError):
        att._scoring_engine(eng, torch.zeros(1, 3, 16, 16, device=DEV))


def test_multiscale_stages_run_the_model_at_the_zoomed_resolution():
    from breaching_b200.attacks import prepare_attack

    model, loss_fn, payload, shared, true = _resnet_case(seed=4, image=64)
    cfg = get_attack_config("multiscale_ghiasi", {"num_stages": 2, "scale_pyramid": "log", "optim.max_iterations": 3, "optim.callback": 3,
                                                  "augmentations": {"zoom": {"out_size": 64}}})
    torch.manual_seed(1)
    att = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float))
    rec, stats = att.reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == (1, 3, 64, 64) and torch.isfinite(rec["data"]).all()
    engines = [att._engine, *att._stage_engines.values()]
    assert len(engines) == 2 and all(e.prog.tensors[0].H == 64 and e.prog.tensors[0].W == 64 for e in engines)
    assert sorted(e.input_shape[2] for e in engines) == [32, 64]
    cfg_bad = get_attack_config("multiscale_ghiasi", {"num_stages": 2, "scale_pyramid": "log", "optim.max_iterations": 2,
                                                      "augmentations": {"focus": {"size": 48}, "zoom": {"out_size": 64}}})
    with pytest.raises(ValueError, match="stage 1/2"):
        prepare_attack(model, loss_fn, cfg_bad, dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})


def test_multiscale_with_a_view_off_the_data_shape_scores_at_the_candidate_shape():
    """multiscale_ghiasi (continuous shift + colour jitter) with an even-width antialias: every stage's view is one pixel larger than
    its candidate, so the trial's score needs the scoring engine at the data's shape.  The colour constants and seed are drawn once
    for all stages."""
    from breaching_b200.attacks import prepare_attack

    model, loss_fn, payload, shared, true = _resnet_case(seed=12, image=64)
    cfg = get_attack_config("multiscale_ghiasi", {"num_stages": 2, "scale_pyramid": "log", "optim.max_iterations": 3, "optim.callback": 3,
                                                  "augmentations": {"antialias": {"width": 4}}})
    torch.manual_seed(3)
    att = prepare_attack(model, loss_fn, cfg, dict(device=DEV, dtype=torch.float, backend="simt"))
    rec, stats = att.reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == (1, 3, 64, 64) and torch.isfinite(rec["data"]).all()
    assert att._engine.prog.tensors[0].H == 65 and sorted(e.prog.tensors[0].H for e in att._stage_engines.values()) == [33]
    assert list(att._aug_plans) == [(1, 3)] and list(att._score_engines) == [(1, 3, 64, 64)]
    meta = payload[0]["metadata"]
    dm, ds = torch.tensor(meta.mean)[None, :, None, None], torch.tensor(meta.std)[None, :, None, None]
    orc = restate.TrialOracle(copy.deepcopy(model).eval(), loss_fn, cfg, shared[0]["gradients"], rec["labels"].cpu(), dm, ds)
    want = orc.score(rec["data"].cpu(), cfg.restarts.scoring)
    assert math.isclose(float(stats["opt_value"]), float(want), rel_tol=1e-3), (stats["opt_value"], want)
    orc.close()


def test_host_driven_and_joint_paths_refuse_resizing_views():
    from breaching_b200.attacks import prepare_attack

    model, loss_fn, payload, shared, true = _resnet_case(seed=6)
    view = {"augmentations": {"zoom": {"out_size": 24}}, "differentiable_augmentations": True, "optim.max_iterations": 2}
    with pytest.raises(NotImplementedError, match="L-BFGS"):
        prepare_attack(model, loss_fn, get_attack_config("invertinggradients", {**view, "optim.optimizer": "L-BFGS"}),
                       dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})
    with pytest.raises(NotImplementedError, match="joint"):
        prepare_attack(model, loss_fn, get_attack_config("invertinggradients", {**view, "attack_type": "joint-optimization"}),
                       dict(device=DEV, dtype=torch.float)).reconstruct(payload, copy.deepcopy(shared), {})


def test_launches_without_augmentations_are_unchanged_by_a_stage_plan():
    model, loss_fn, payload, shared, true = _resnet_case()
    cfg = get_attack_config("invertinggradients", {"augmentations": {"antialias": {"width": 3}}, "differentiable_augmentations": True})
    eng = _engine(model, cfg, shared, true["labels"], payload[0]["metadata"], (1, 3, 32, 32), "tc")
    from breaching_b200.schedule import lr_table

    table = lr_table(0.1, "step-lr", 0, 10)
    eng.begin_trial(torch.zeros(1, 3, 32, 32, device=DEV), table)
    eng.run(1)
    plain = eng.launches_per_iteration()
    eng.set_augmentations(augment.build_plan(cfg, 1, 3, dict(device=DEV, dtype=torch.float), spatial=(32, 32)))
    eng.begin_trial(torch.zeros(1, 3, 32, 32, device=DEV), table)
    eng.run(1)
    assert eng.launches_per_iteration() == plain + 3        # draw, blur view, blur pull-back
    eng.set_augmentations(None)
    eng.begin_trial(torch.zeros(1, 3, 32, 32, device=DEV), table)
    eng.run(1)
    assert eng.launches_per_iteration() == plain
    eng.close()
