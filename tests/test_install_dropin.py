"""Drop-in mounting: ``breaching_b200.install.install()`` rebinds ``breaching.attacks.prepare_attack`` of the (unmodified)
reference package, so reference entry points keep calling ``breaching.attacks.prepare_attack(...)`` unchanged.
What the reference computes or composes is pinned by ``tests/golden/dropin.pt`` and ``tests/golden/attack_configs.pt``
(``tests/golden/make_golden.py``), so these tests need no reference installation."""
import sys
import types

import torch

from oracle import refshim


def _ref_cfg(plain):
    """A composed reference config as the reference's YAML loader hands it over (attribute + item access)."""
    return refshim._coerce(plain)


def test_install_rebinds_prepare_attack_and_delegates_other_attack_types(golden):
    """A stand-in ``breaching`` package (its ``attacks.prepare_attack`` returns an object of a ``breaching.attacks`` class)
    is mounted and unmounted; the attack type outside the accelerated path is delegated to it."""
    import breaching_b200
    from breaching_b200 import install as inst
    from breaching_b200 import synthetic
    from breaching_b200.engine import EngineError

    class AnalyticAttacker:
        pass

    AnalyticAttacker.__module__ = "breaching.attacks.analytic_attack"

    def original(model, loss, cfg_attack, setup):
        return AnalyticAttacker()

    original.__module__ = "breaching.attacks"
    pkg, sub = types.ModuleType("breaching"), types.ModuleType("breaching.attacks")
    sub.prepare_attack = original
    pkg.attacks = sub
    saved = {k: sys.modules.get(k) for k in ("breaching", "breaching.attacks")}
    sys.modules.update({"breaching": pkg, "breaching.attacks": sub})
    inst._ORIGINAL = None
    try:
        returned = inst.install()
        assert returned is original
        assert sub.prepare_attack.__module__.startswith("breaching_b200")
        model = synthetic.build_model("convnet-tiny", 10)
        loss = torch.nn.CrossEntropyLoss()
        setup = dict(device=torch.device("cpu"), dtype=torch.float)
        # optimisation attacks go to the engine: on a CPU "device" it refuses loudly (no fallback) ...
        try:
            sub.prepare_attack(model, loss, breaching_b200.get_attack_config("invertinggradients"), setup)
            raise AssertionError("the engine accepted a CPU device")
        except EngineError:
            pass
        # ... while the attack types outside the accelerated path are delegated to the reference's own classes
        cfg = _ref_cfg(golden("dropin.pt")["analytic_cfg"])
        attacker = sub.prepare_attack(model, loss, cfg, setup)
        assert type(attacker).__module__.startswith("breaching.attacks")
        inst.uninstall()
        assert sub.prepare_attack is original
    finally:
        inst._ORIGINAL = None
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def test_reference_yaml_config_objects_are_accepted_by_the_engine_config_flattening(golden):
    """cfg objects composed from the reference's own YAML (attribute + item access) flatten to the same C struct as ours."""
    import ctypes

    import breaching_b200
    from breaching_b200.engine import make_cfg

    composed = golden("attack_configs.pt")
    for name in ["invertinggradients", "modern", "seethroughgradients", "clsattack", "legacy"]:
        a = make_cfg(_ref_cfg(composed[name]))
        b = make_cfg(breaching_b200.get_attack_config(name))
        assert bytes(ctypes.string_at(ctypes.addressof(a), ctypes.sizeof(a))) == bytes(ctypes.string_at(ctypes.addressof(b), ctypes.sizeof(b))), name


def test_text_prologue_and_token_recovery_match_the_reference(golden):
    """host.prepare_for_text_data / postprocess_text_data against what the reference attacker's own methods
    (base_attack.py:76-167) produced on the miniature causal-LM case."""
    import copy

    from breaching_b200 import synthetic
    from breaching_b200.attacks import host

    fx = golden("dropin.pt")["text"]
    model, loss_fn, payload, shared, true = synthetic.make_text_case(batch=2, seq_len=6, seed=77)
    mine = copy.deepcopy(model)
    sh_mine = copy.deepcopy(shared)
    emb, dim = host.prepare_for_text_data([mine], sh_mine, golden("attack_configs.pt")["tag"]["text_strategy"])
    assert dim == fx["embedding_dim"] == fx["data_shape"][-1]
    assert len(sh_mine[0]["gradients"]) == len(fx["gradients"])
    for a, b in zip(sh_mine[0]["gradients"], fx["gradients"]):
        assert torch.equal(a, b)
    assert torch.equal(emb[0]["grads"], fx["embedding_grads"])
    assert isinstance(mine.encoder, torch.nn.Identity) and fx["encoder_is_identity"]
    assert [n for n, _ in mine.named_parameters()] == fx["parameter_names"]
    # token recovery from reconstructed embeddings: noisy true embeddings must map back to the tokens, identically to the reference
    gen = torch.Generator().manual_seed(5)
    tokens = true["data"]
    rec = dict(data=model.encoder.weight.detach()[tokens] + 0.01 * torch.randn(2, 6, dim, generator=gen), labels=tokens.clone())
    assert torch.equal(rec["data"], fx["rec_data"]) and torch.equal(rec["labels"], fx["labels"])
    for mode in ("from-embedding", "from-labels", "from-limited-embedding"):
        got = host.postprocess_text_data(dict(data=rec["data"].clone(), labels=rec["labels"].clone()), emb[0]["weight"].detach(), mode)
        assert torch.equal(got["data"], fx["recovered"][mode]), mode


def test_compile_transformer_accepts_the_reference_model_class(golden):
    """``compiler.compile_transformer`` on a model with the parameters of an instance of the reference's own
    ``TransformerModel`` (cases/models/language_models.py:150-205): same attribute names and parameter order as
    ``synthetic.TransformerLM``; the lowered program, run by the four-sweep interpreter, reproduces the gradients autograd
    computed through the reference module."""
    from breaching_b200 import compiler, synthetic
    from oracle import program_interp as PI

    fx = golden("dropin.pt")["transformer"]
    model = synthetic.TransformerLM(40, 16, 4, 24, 2).double().eval()
    assert [n for n, _ in model.named_parameters()] == fx["parameter_names"]
    B, T = 2, 6
    pos = "pos_encoder.embedding.weight"       # the fixture holds the T positional rows the sequence reads
    state = dict(fx["state_dict"])
    state[pos] = torch.cat([state[pos], model.state_dict()[pos][T:]])
    model.load_state_dict(state)
    prog = compiler.compile_transformer(model, B, T, pad_vocab=False)   # the torch interpreter runs the un-padded program
    model.encoder = torch.nn.Identity()                     # what the attack does (base_attack.py:100-110)
    params = [p for p in model.parameters()]

    class _Params:
        def parameters(self):
            return params

        def named_modules(self):
            return model.named_modules()

    it = PI.ProgramInterpreter(_Params(), prog)
    assert abs(float(it.forward(fx["x"], fx["q"])) - fx["loss"]) < 1e-12
    names = [n for n in fx["parameter_names"] if n != "encoder.weight"]
    for name, a, b in zip(names, it.backward(), fx["grads"], strict=True):
        if name == pos:
            assert not a[T:].any()
            a = a[:T]
        assert ((a - b).norm() / (b.norm() + 1e-300)).item() < 1e-10
