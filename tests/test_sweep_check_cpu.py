"""The layer-local sweep checker (oracle/sweep_check.py) on the float64 four-sweep interpreter: every relation it checks holds
to rounding level on the interpreter's own buffers, and a buffer corrupted the way a faulty kernel would corrupt it (the
ops that read it see the corrupted value) is reported at exactly the op and sweep that produced it."""
import copy

import pytest
import torch

from breaching_b200 import compiler, get_attack_config, synthetic
from helpers import masked_targets, odd_case, sweep_objective
from oracle import program_interp as PI
from oracle import restate
from oracle.sweep_check import TERMS, InterpreterSource, SweepChecker, f32, tag_weights


def _synthetic(name, size, no_buffers=False, seed=11):
    data = "cifar" if size == 32 else "imagenet"
    model, _, _, shared, true = synthetic.make_case(name, data, batch=2, seed=seed, bn_random=True, image_size=size, classes=10,
                                                    no_buffers=no_buffers)
    return model, (2, 3, size, size), true["labels"], shared[0]["gradients"]


def _case(name):
    if name == "odd":
        return odd_case()
    if name == "convnet-tiny":
        return _synthetic("convnet-tiny", 32)
    if name == "trainbn-convnet-tiny":
        return _synthetic("convnet-tiny", 32, no_buffers=True)
    return _synthetic(name, 32)


def run_interpreter(model, shape, labels, grads, obj, seed=3, tamper=None):
    """float64 four sweeps + priors; returns the checker fed with the interpreter's buffers."""
    m64 = copy.deepcopy(model).double()
    prog = compiler.compile_model(m64, shape)
    it = PI.ProgramInterpreter(m64, prog)
    it.tamper = tamper
    x = torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64)

    def inject_fn(it_):
        inj = {}
        parts = []
        if obj.get("di") is not None:
            parts.append(it_.deep_inversion(obj["di"]["scale"], obj["di"]["first_bn_multiplier"])[1])
        if obj.get("features") is not None:
            parts.append(it_.feature_regularization(obj["features"]["measured"], obj["features"]["scale"])[1])
        for p in parts:
            for k, v in p.items():
                inj[k] = inj.get(k, 0) + v
        return inj or None

    g64 = [g.double() for g in grads]
    _, dx, _, _ = it.matching_gradient(x, labels, g64, obj["kind"], scale=obj["scale"], task_regularization=obj["task_regularization"],
                                       inject_fn=inject_fn)
    from oracle import restate

    xd = x.clone().requires_grad_(True)
    prior = xd.sum() * 0
    if obj.get("tv") is not None:
        prior = prior + restate.total_variation(xd, scale=obj["tv"]["scale"])
    if obj.get("norm") is not None:
        prior = prior + restate.norm_regularization(xd, scale=obj["norm"]["scale"], pnorm=obj["norm"]["p"])
    (gp,) = torch.autograd.grad(prior, xd)
    chk = SweepChecker(prog, it.P, it.bn, g64, labels, obj, InterpreterSource(it, dx + gp))
    chk.interp, chk.x0 = it, x
    return chk, prog


def _objective(name):
    if name == "resnet18":   # every prior the checker knows
        cfg = get_attack_config("invertinggradients", {"objective.task_regularization": 0.1, "regularization.norm.scale": 1e-3,
                                                        "regularization.deep_inversion.scale": 1e-3,
                                                        "regularization.features.scale": 0.1})
        feats = torch.randn(2, 512, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
        return sweep_objective(cfg, features=feats)
    return sweep_objective(get_attack_config("invertinggradients"))


CASES = ["convnet-tiny", "resnet18", "resnet50", "trainbn-convnet-tiny", "odd"]


@pytest.mark.parametrize("name", CASES)
def test_interpreter_buffers_satisfy_every_relation(name):
    model, shape, labels, grads = _case(name)
    chk, prog = run_interpreter(model, shape, labels, grads, _objective(name))
    chk.check()
    # float64 buffers against fp32 rounding bounds: every relation holds far below its bound (~1e-12 relative)
    worst = max(chk.ratios.values())
    assert worst < 1e-6, sorted(chk.ratios.items(), key=lambda kv: -kv[1])[:5]
    kinds = {k for k, _ in chk.ratios}
    assert {"conv", "bnact", "linear"} <= kinds
    sweeps = {s for _, s in chk.ratios}
    assert sweeps == {"F", "B", "V", "TF", "TB"}


def _flagged(chk):
    return {(f.op, f.sweep) for f in chk.check(raise_on_failure=False)}


@pytest.mark.parametrize("name", ["convnet-tiny", "odd", "resnet18"])
def test_scaled_tangent_channel_is_reported_at_its_producer(name):
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    target = [i for i, op in enumerate(prog.ops) if op.kind == compiler.OP_CONV][2]

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "TF" and i == target:
            stored = stored.clone()
            stored[:, 1] *= 1.001
        return stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(target, "TF")}


@pytest.mark.parametrize("name", ["convnet-tiny", "odd", "resnet18"])
def test_swapped_delta_pixels_are_reported_where_the_delta_is_final(name):
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    t = [op.tout for op in prog.ops if op.kind == compiler.OP_BNACT][1]
    last = min(i for i, op in enumerate(prog.ops) if t in (op.tin, op.res))

    def tamper(sweep, i, tid, stored, contribution=None):
        if sweep == "B" and i == last and tid == t:
            stored = stored.clone()
            flat = stored[0, 0].flatten()
            nz = flat.nonzero().flatten()
            j, k = int(nz[0]), int(nz[-1])
            assert flat[j] != flat[k]
            flat[j], flat[k] = flat[k].clone(), flat[j].clone()
            stored[0, 0] = flat.view_as(stored[0, 0])
        return stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(last, "B")}


def _branch_point(prog, kind):
    """(op index, tensor) of an accumulation: ``conv``: the residual branch point of the first residual op (a conv accumulates into
    its delta); ``bnact-in`` / ``bnact-res``: a BN / ReLU / add op with ``acc_in`` / ``acc_res``, ``-scalar`` on C % 4 != 0 channels
    (scalar kernels), ``-vec`` on C % 4 == 0 (float4 kernels)."""
    consumers = lambda t: [i for i, op in enumerate(prog.ops) if t in (op.tin, op.res)]  # noqa: E731
    if kind == "conv":
        first_res = next(op for op in prog.ops if op.res >= 0)
        t = next(t for t in (first_res.res, first_res.tin) if len(consumers(t)) == 2)
        return min(consumers(t)), t
    field, width = kind.split("-")[1:]
    for i, op in enumerate(prog.ops):
        vec = prog.tensors[op.tout].C % 4 == 0
        if op.kind == compiler.OP_BNACT and getattr(op, f"acc_{field}") and vec == (width == "vec"):
            t = op.tin if field == "in" else op.res
            assert min(consumers(t)) == i   # this op's write makes the buffer final
            return i, t
    raise AssertionError(f"no {kind} accumulation in the program")


@pytest.mark.parametrize("name,kind", [("resnet18", "conv"), ("odd", "conv"), ("odd", "bnact-in-scalar"), ("odd", "bnact-res-scalar"),
                                       ("odd", "bnact-in-vec"), ("odd", "bnact-res-vec")])
@pytest.mark.parametrize("sweep", ["B", "TB"])
def test_dropped_accumulation_is_reported(name, kind, sweep):
    """The last consumer of a tensor with two consumers overwrites the delta instead of accumulating into it."""
    model, shape, labels, grads = _case(name)
    prog = compiler.compile_model(copy.deepcopy(model).double(), shape)
    last, t = _branch_point(prog, kind)

    def tamper(sweep_, i, tid, stored, contribution=None):
        return contribution if (sweep_ == sweep and i == last and tid == t) else stored

    chk, _ = run_interpreter(model, shape, labels, grads, _objective(name), tamper=tamper)
    assert _flagged(chk) == {(last, sweep)}


KINDS = ["euclidean", "l1", "tag-euclidean", "cosine-similarity", "angular", "fast-cosine-similarity", "masked-cosine-similarity"]


@pytest.mark.parametrize("kind", KINDS)
def test_other_objectives_direction(kind):
    model, shape, labels, grads = _case("convnet-tiny")
    if kind == "masked-cosine-similarity":
        grads = masked_targets(grads)
    obj = sweep_objective(get_attack_config("invertinggradients", {"objective.type": kind, "objective.scale": 0.5}))
    chk, _ = run_interpreter(model, shape, labels, grads, obj)
    chk.check()
    assert chk.ratios[("objective", "V")] < 1e-6


# ---------------------------------------------------------------------------------------------------- objective terms
def _terms_objective(kind, scheme="linear"):
    """Every term on, with configuration scalars that fp32 holds exactly (the checker reads them at their fp32 values, the
    interpreter in float64)."""
    cfg = get_attack_config("invertinggradients", {
        "objective.type": kind, "objective.scale": 0.5, "objective.tag_scale": 0.125, "objective.scale_scheme": scheme,
        "objective.task_regularization": 0.125, "regularization.total_variation.scale": 0.25,
        "regularization.norm.scale": 2.0 ** -10, "regularization.deep_inversion.scale": 2.0 ** -10,
        "regularization.features.scale": 0.125})
    feats = torch.randn(2, 512, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    return sweep_objective(cfg, features=feats)


def interpreter_terms(chk, obj, weights=None):
    """The six terms of ``Engine.last_terms()`` and the objective as the engine assembles it, from the float64 interpreter."""
    it, x = chk.interp, chk.x0
    kw = {k: obj[k] for k in ("tag_scale", "scale_scheme") if k in obj}
    if obj["kind"] == "tag-euclidean":
        kw["weights"] = tag_weights(len(chk.g), obj["scale_scheme"]) if weights is None else weights
    match, _ = PI.objective_direction(obj["kind"], it.G, chk.g, scale=obj["scale"], **kw)
    tv = obj["tv"]
    terms = dict(match=float(match), task_loss=float(it.loss),
                 total_variation=float(restate.total_variation(x, scale=tv["scale"], eps=tv["eps"])),
                 norm=float(restate.norm_regularization(x, scale=obj["norm"]["scale"], pnorm=obj["norm"]["p"])),
                 deep_inversion=float(it.deep_inversion(obj["di"]["scale"], obj["di"]["first_bn_multiplier"])[0]),
                 features=float(it.feature_regularization(obj["features"]["measured"], obj["features"]["scale"])[0]))
    return terms, assemble(terms, obj)


def assemble(terms, obj):
    """``bre_engine_objective_and_gradient``: the terms summed in this order in double, the task term at fp32 tau."""
    phi = terms["match"] + terms["total_variation"] + terms["norm"] + terms["deep_inversion"] + terms["features"]
    return phi + f32(obj["task_regularization"]) * terms["task_loss"]


_RUNS = {}


def _terms_run(kind, scheme="linear"):
    key = (kind, scheme)
    if key not in _RUNS:
        model, shape, labels, grads = _case("resnet18")
        if kind == "masked-cosine-similarity":
            grads = masked_targets(grads)
        obj = _terms_objective(kind, scheme)
        chk, _ = run_interpreter(model, shape, labels, grads, obj)
        _RUNS[key] = (chk, obj)
    chk, obj = _RUNS[key]
    chk.findings, chk.ratios = [], {}
    return chk, obj


def _terms_flagged(chk, terms, value):
    return {f.sweep for f in chk.check_terms(terms, value, raise_on_failure=False)}


@pytest.mark.parametrize("kind,scheme", [(k, "linear") for k in KINDS] + [("tag-euclidean", "exp")])
def test_interpreter_terms_satisfy_the_terms_relation(kind, scheme):
    chk, obj = _terms_run(kind, scheme)
    terms, value = interpreter_terms(chk, obj)
    assert all(terms[k] != 0 for k in TERMS), terms
    chk.check_terms(terms, value)
    assert {s for k, s in chk.ratios if k == "terms"} == set(TERMS) | {"value"}
    assert max(chk.ratios.values()) < 1e-6, chk.ratios


@pytest.mark.parametrize("term", TERMS + ("value",))
@pytest.mark.parametrize("kind", ["euclidean", "angular"])
def test_perturbed_term_is_reported_at_that_term(kind, term):
    """A term 1e-5 off (relative) -- and the objective assembled from it, as the engine would -- is reported there alone.
    DeepInversion's bound covers the fp32 batch statistics, TRAIN_C (M + 8) u kap relative (1.3e-4 here: M = 512 at the first BN
    layer), so its perturbation is 1e-3."""
    chk, obj = _terms_run(kind)
    terms, value = interpreter_terms(chk, obj)
    rel = 1e-3 if term == "deep_inversion" else 1e-5
    if term == "value":
        value *= 1 + rel
    else:
        terms[term] *= 1 + rel
        value = assemble(terms, obj)
    assert _terms_flagged(chk, terms, value) == {term}


def test_swapped_tag_weights_are_reported_at_the_match_term():
    """tag-euclidean with one tensor's weight swapped for its neighbour's (the chunk-weight map of load_targets off by one tensor)."""
    chk, obj = _terms_run("tag-euclidean")
    w = tag_weights(len(chk.g), "linear").clone()
    l1 = [float((a - b).abs().sum()) for a, b in zip(chk.interp.G, chk.g)]
    j = max(range(len(w) - 1), key=lambda k: abs(l1[k] - l1[k + 1]))
    w[j], w[j + 1] = w[j + 1].clone(), w[j].clone()
    terms, value = interpreter_terms(chk, obj, weights=w)
    assert _terms_flagged(chk, terms, value) == {"match"}


def test_unmasked_cosine_is_reported_at_the_match_term():
    chk, obj = _terms_run("masked-cosine-similarity")
    terms, _ = interpreter_terms(chk, obj)
    terms["match"] = float(PI.objective_direction("cosine-similarity", chk.interp.G, chk.g, scale=obj["scale"])[0])
    assert _terms_flagged(chk, terms, assemble(terms, obj)) == {"match"}


@pytest.mark.parametrize("kind", ["euclidean", "cosine-similarity"])
def test_score_relation(kind):
    """``Engine.score``: the fp32-rounded match with scale 1; a 1e-5 relative error is reported."""
    chk, obj = _terms_run("euclidean")
    ref = float(PI.objective_direction(kind, chk.interp.G, chk.g)[0])
    assert not chk.check_score(f32(ref), kind)
    assert chk.ratios[("score", kind)] < 1.0
    assert [f.sweep for f in chk.check_score(ref * (1 + 1e-5), kind, raise_on_failure=False)] == [kind]


@pytest.mark.parametrize("kind", ["euclidean", "tag-euclidean"])
def test_direction_bound_covers_the_fma_form_where_G_and_g_agree(kind):
    """make_v_kernel forms s (G - g) as fma(-s, g, fma(s, G, c3 w sign(G - g))): where G and g agree to 1e-6 its rounding is
    relative to s (|G| + |g|), far above s |G - g|.  An fp32 emulation of that kernel passes the direction relation."""
    model, shape, labels, grads = _case("convnet-tiny")
    obj = sweep_objective(get_attack_config("invertinggradients", {"objective.type": kind, "objective.scale": 1e-4}))
    chk, _ = run_interpreter(model, shape, labels, grads, obj)
    gen = torch.Generator().manual_seed(0)
    r32 = lambda t: t.to(torch.float32).double()  # noqa: E731
    G = [r32(chk.Pm("G", j)) for j in range(len(chk.P))]
    chk.g = [r32(a * (1 + 1e-6 * torch.randn(a.shape, generator=gen, dtype=torch.float64))) for a in G]
    s = f32(obj["scale"])
    c3 = f32(0.5 * s * f32(obj.get("tag_scale", 0.1))) if kind == "tag-euclidean" else 0.0
    w = tag_weights(len(G), "linear") if kind == "tag-euclidean" else torch.ones(len(G))
    for j, (a, b) in enumerate(zip(G, chk.g)):
        w3 = f32(c3 * float(w[j]))
        inner = r32(s * a + w3 * torch.sign(r32(a - b)))   # fma: one rounding of the exact s a + w3 sign
        chk._cache[("p", "G", j)] = a
        chk._cache[("p", "v_operand", j)] = r32(-s * b + inner)
    chk.findings, chk.ratios = [], {}
    chk.direction()
    assert not chk.findings, chk.findings[:3]
