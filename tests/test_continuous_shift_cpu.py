"""continuous_shift with every option of the reference's RandomTransform, without a GPU: the float64 restatement (tests/cshift_oracle.py)
against the unmodified module's views and vector-Jacobian products (tests/golden/continuous_shift.pt), and the plans of
attacks/augment.py: configs of the options accepted before keep their plans and draws, the new orderings split into PIXEL stages, and
unknown modes / paddings are refused as grid_sample refuses them."""
import pytest
import torch

from helpers import load_golden
from breaching_b200 import get_attack_config
from breaching_b200.attacks import augment
from cshift_oracle import continuous_shift, source_coordinates

SETUP = dict(device=torch.device("cpu"), dtype=torch.float)


def _cfg(augs, differentiable=True):
    return get_attack_config("invertinggradients", {"augmentations": augs, "differentiable_augmentations": differentiable})


def test_restatement_equals_the_reference_module():
    fx = load_golden("continuous_shift.pt")
    cases = fx["cases"]
    combos = {(c["mode"], c["padding"], c["fliplr"], c["flipud"]) for c in cases}
    assert len(combos) == 3 * 4 * 4 == len(cases)
    for c in cases:
        inp = fx["inputs"][c["S"]]
        x = inp["x"].clone().requires_grad_(True)
        y = continuous_shift(x, c["shift"], c["randgen"], c["mode"], c["padding"], c["fliplr"], c["flipud"])
        assert (y.detach() - c["view"]).abs().max().item() < 1e-12, c["mode"]
        (vjp,) = torch.autograd.grad((y * inp["probe"]).sum(), x)
        assert (vjp - c["vjp"]).abs().max().item() < 1e-12, c["mode"]
        assert torch.equal(c["randgen"][:, :2], c["randgen"][:, :2].float().double())      # the device receives them exactly
        if c["mode"] == "nearest":
            for p in source_coordinates(c["S"], c["shift"], c["randgen"], c["padding"], c["fliplr"], c["flipud"]):
                assert (p - p.floor() - 0.5).abs().min().item() > 1e-5


def _draws(augs_in_order, batch):
    """The random numbers the parent plan builder drew for a config: colour constants in config order, then the seed."""
    colour = []
    for key, opts in augs_in_order:
        if key == "colorjitter":
            m = (torch.rand((batch, 3, 1, 1)) - 0.5) * 2 * opts.get("mean", 0.0)
            sd = ((torch.rand((batch, 3, 1, 1)) - 0.5) * 2 * opts.get("std", 1.0)).exp()
            colour.append((m.view(batch, 3), sd.view(batch, 3)))
    return colour, int(torch.randint(0, 2 ** 31 - 1, (1,)).item())


PLAIN = [   # configs accepted before: (augmentations, steps, continuous_shift, circular)
    ({"discrete_shift": {"lim": 4}}, [(augment.SHIFT, 4.0)], None, False),
    ({"flip": {"p": 0.3}, "discrete_shift": {}}, [(augment.FLIP, 0.3), (augment.SHIFT, 32.0)], None, False),
    ({"continuous_shift": {"shift": 5, "padding": "zeros"}}, [], 5.0, False),
    ({"discrete_shift": {"lim": 2}, "continuous_shift": {"shift": 7, "padding": "circular", "mode": "bilinear"},
      "colorjitter": {"mean": 0.1, "std": 0.3}}, [(augment.SHIFT, 2.0)], 7.0, True),
    ({"colorjitter": {"mean": 0.2}, "flip": {}, "continuous_shift": {"shift": 224, "padding": "circular", "fliplr": False}},
     [(augment.FLIP, 0.5)], 224.0, True),
]


@pytest.mark.parametrize("augs, steps, cs, circular", PLAIN)
def test_configs_accepted_before_build_the_same_plan(augs, steps, cs, circular):
    torch.manual_seed(17)
    plan = augment.build_plan(_cfg(augs), 2, 3, SETUP, spatial=(16, 16))
    after = torch.get_rng_state()
    torch.manual_seed(17)
    colour, seed = _draws(list(augs.items()), 2)
    assert torch.equal(torch.get_rng_state(), after)
    assert plan.seed == seed and plan.steps == steps and plan.continuous_shift == cs and plan.circular == circular
    assert plan.stages == [] and plan.candidate_shape is None and plan.differentiable
    assert (plan.cs_mode, plan.cs_padding, plan.fliplr, plan.flipud) == ("bilinear", "zeros", False, False)
    if colour:
        scale, shift = torch.ones(2, 3), torch.zeros(2, 3)
        for m, sd in colour:
            scale, shift = scale / sd, (shift - m) / sd
        assert torch.equal(plan.colour_scale, scale) and torch.equal(plan.colour_shift, shift)
    else:
        assert plan.colour_scale is None


def test_staged_configs_accepted_before_build_the_same_stages():
    augs = {"discrete_shift": {"lim": 3}, "continuous_shift": {"shift": 3, "padding": "zeros"}, "colorjitter": {"mean": 0.1, "std": 0.3},
            "centerzoom": {"initial_fov": 12, "out_size": 16}, "flip": {"p": 0.5}, "antialias": {"width": 3}}
    torch.manual_seed(5)
    plan = augment.build_plan(_cfg(augs), 1, 3, SETUP, spatial=(16, 16))
    after = torch.get_rng_state()
    torch.manual_seed(5)
    colour, seed = _draws(list(augs.items()), 1)
    assert torch.equal(torch.get_rng_state(), after) and plan.seed == seed
    assert [s.kind for s in plan.stages] == [augment.PIXEL, augment.RESAMPLE, augment.PIXEL, augment.BLUR]
    p0, p1 = plan.stages[0], plan.stages[2]
    assert p0.steps == [(augment.SHIFT, 3.0)] and p0.continuous_shift == 3.0 and not p0.circular
    assert p1.steps == [(augment.FLIP, 0.5)] and p1.continuous_shift is None
    for st in (p0, p1):
        assert (st.cs_mode, st.cs_padding, st.fliplr, st.flipud) == ("bilinear", "zeros", False, False)
    m, sd = colour[0]
    assert torch.equal(p0.colour_scale, 1 / sd) and torch.equal(p0.colour_shift, (0 - m) / sd)


def test_the_module_defaults_and_every_option_reach_the_plan():
    plan = augment.build_plan(_cfg({"continuous_shift": {"shift": 8}}), 1, 3, SETUP, spatial=(16, 16))
    assert plan.continuous_shift == 8.0 and (plan.cs_mode, plan.cs_padding, plan.circular) == ("bilinear", "reflection", False)
    plan = augment.build_plan(_cfg({"continuous_shift": {"shift": 2, "mode": "bicubic", "padding": "border", "fliplr": True, "flipud": True}}),
                              1, 3, SETUP, spatial=(16, 16))
    assert (plan.cs_mode, plan.cs_padding, plan.fliplr, plan.flipud) == ("bicubic", "border", True, True) and plan.stages == []
    plan = augment.build_plan(_cfg({"continuous_shift": {"mode": "nearest", "padding": "circular"}}), 1, 3, SETUP, spatial=(16, 16))
    assert (plan.cs_mode, plan.cs_padding, plan.circular) == ("nearest", "zeros", True)


@pytest.mark.parametrize("augs, want", [
    ({"continuous_shift": {}, "flip": {}}, [[], [(augment.FLIP, 0.5)]]),
    ({"continuous_shift": {}, "discrete_shift": {"lim": 2}, "colorjitter": {}}, [[], [(augment.SHIFT, 2.0)]]),
    ({"flip": {}, "continuous_shift": {}, "colorjitter": {}, "discrete_shift": {"lim": 1}},
     [[(augment.FLIP, 0.5)], [(augment.SHIFT, 1.0)]]),
    ({"continuous_shift": {}, "colorjitter": {}}, None),                      # colour after the shift: one plain plan
    ({"continuous_shift": {}, "zoom": {"out_size": 20}, "flip": {}}, [[], "resample", [(augment.FLIP, 0.5)]]),
])
def test_steps_after_a_continuous_shift_open_a_pixel_stage(augs, want):
    cfg = _cfg(augs)
    torch.manual_seed(3)
    plan = augment.build_plan(cfg, 2, 3, SETUP, spatial=(16, 16))
    if want is None:
        assert plan.stages == [] and plan.continuous_shift == 8.0
        return
    got = [st.steps if st.kind == augment.PIXEL else st.kind for st in plan.stages]
    assert got == want
    assert plan.candidate_shape == (2, 3, 16, 16) and augment.view_shape(cfg, (2, 3, 16, 16)) == (2, 3, 16, 16) or "zoom" in augs
    pixel = [st for st in plan.stages if st.kind == augment.PIXEL]
    assert pixel[0].continuous_shift == 8.0 and pixel[0].cs_padding == "reflection"
    assert all(st.continuous_shift is None for st in pixel[1:])
    colour = [st for st in pixel if st.colour_scale is not None]
    assert len(colour) == (1 if "colorjitter" in augs else 0)
    # a plan for another resolution splits the same way and keeps the draws
    if "zoom" not in augs:
        small = augment.with_spatial(plan, cfg, (8, 8))
        assert [st.steps for st in small.stages] == want and small.seed == plan.seed and small.stages[0].in_hw == (8, 8)


def test_new_orderings_need_the_spatial_shape():
    with pytest.raises(ValueError, match="spatial shape"):
        augment.build_plan(_cfg({"continuous_shift": {}, "flip": {}}), 1, 3, SETUP)


@pytest.mark.parametrize("opts, match", [
    ({"mode": "cubic"}, "mode"),
    ({"mode": "area"}, "mode"),
    ({"padding": "reflect"}, "padding"),
    ({"padding": "constant"}, "padding"),
])
def test_unknown_modes_and_paddings_are_refused(opts, match):
    with pytest.raises(ValueError, match=match):
        augment.build_plan(_cfg({"continuous_shift": opts}), 1, 3, SETUP, spatial=(16, 16))
