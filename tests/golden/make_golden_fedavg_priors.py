"""Generate the FedAvg-with-priors fixtures in this directory (``trial_fedavg_taskreg_convnet.pt``, ``trial_fedavg_di_convnet.pt``,
``trial_fedavg_di_resnet18.pt``) by running the reference, the way ``make_golden.py`` produces the others.

Run where the reference is importable (``BREACHING_REFERENCE_ROOT``, see oracle/refshim.py):
``python tests/golden/make_golden_fedavg_priors.py [fixture names]``

Task-loss regularisation with FedAvg runs in the unmodified reference: ``GradientLoss.forward`` adds ``task_regularization`` times
the last local step's loss (objectives.py:30-31, 71-72).  DeepInversion with FedAvg does not (SURVEY.md fact 9); those cases run
with the forward hooks kept on the functional copy, see ``deep_inversion_hooks_survive_functional_copy``.
"""
import contextlib
import importlib
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository root on sys.path)
from oracle import refshim  # noqa: E402

CASES = {
    # name: (case kwargs, attack yaml, overrides, iterations)
    "fedavg_taskreg_convnet": (dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05,
                                    seed=41, bn_random=True), "modern",
                               {"regularization.features.scale": 0.0, "objective.task_regularization": 0.1}, 6),
    "fedavg_di_convnet": (dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, seed=42,
                               bn_random=True), "modern",
                          {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01,
                           "objective.task_regularization": 0.1}, 6),
    "fedavg_di_resnet18": (dict(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=0.01, seed=43,
                                bn_random=True, image_size=64, classes=10), "modern",
                           {"regularization.features.scale": 0.0, "regularization.deep_inversion.scale": 0.01,
                            "objective.task_regularization": 0.1}, 4),
}


@contextlib.contextmanager
def deep_inversion_hooks_survive_functional_copy():
    """The reference's FedAvg objective evaluates the model through ``make_functional_with_buffers``, which deep-copies the module
    (``FunctionalModuleWithBuffers._create_from`` / ``with_state``).  The copy takes the DeepInversion forward hooks with it, so the
    hooks that fire write ``r_feature`` on copies of the hook objects, and the regulariser, which reads the originals, fails
    (SURVEY.md fact 9).  SURVEY section 8(c) fixes the semantics instead: the hooks act on the functional copy, so the statistics of
    the last forward of the iteration -- the last local step -- win.  While this context is active, every ``copy.deepcopy`` that
    ``breaching.attacks.auxiliaries.make_functional`` performs starts from a memo pre-seeded ``{id(h): h}`` for every
    ``DeepInversionFeatureHook`` registered on the module being copied (those of the attackers' regularisers), so the copied
    modules call the original hook objects.  The reference tree itself is not modified."""
    from breaching.attacks.auxiliaries.deepinversion import DeepInversionFeatureHook

    mf = importlib.import_module("breaching.attacks.auxiliaries.make_functional")   # the module (the package exports a function of that name)
    real = mf.copy

    class _SeededCopy:
        @staticmethod
        def deepcopy(obj, memo=None):
            memo = {} if memo is None else memo
            for mod in obj.modules():
                for fn in mod._forward_hooks.values():
                    hook = getattr(fn, "__self__", None)
                    if isinstance(hook, DeepInversionFeatureHook):
                        memo[id(hook)] = hook
            return real.deepcopy(obj, memo)

    mf.copy = _SeededCopy
    try:
        yield
    finally:
        mf.copy = real


def main():
    ref = refshim.import_reference()
    only = sys.argv[1:]
    for name, (case_kwargs, attack, overrides, iters) in CASES.items():
        if only and name not in only:
            continue
        torch.manual_seed(0)
        di = overrides.get("regularization.deep_inversion.scale", 0.0) > 0   # task regularisation alone: the unmodified reference
        with deep_inversion_hooks_survive_functional_copy() if di else contextlib.nullcontext():
            fx = make_golden.run_reference(ref, case_kwargs, attack, overrides, iters)
        torch.save(fx, os.path.join(HERE, f"trial_{name}.pt"))
        print(name, "history", [round(h, 5) for h in fx["history"]], "score", fx["score"])


if __name__ == "__main__":
    main()
