"""Drop-in for ``breaching.attacks`` (reference ``attacks/__init__.py:12-37``)."""
import torch

from .joint_attack import OptimizationJointAttacker
from .multiscale_attack import MultiScaleOptimizationAttacker
from .optimization_attack import OptimizationBasedAttacker, _loss_name

_OTHER_ATTACKS = (
    "analytic", "april-analytic", "imprint-readout", "decepticon-readout", "recursive",
    "joint-optimization", "permutation-optimization",
)


def prepare_attack(model, loss, cfg_attack, setup=dict(dtype=torch.float, device=torch.device("cpu"))):
    """Same signature and error behaviour as the reference's ``prepare_attack``.

    ``attack_type == "optimization"`` is served by the sm_90a engine.  Other attack types are outside the
    accelerated hot path; when the original ``breaching`` package is importable they are delegated to it,
    otherwise a ``NotImplementedError`` names what is missing (never a silent fallback).
    """
    if cfg_attack.attack_type == "optimization":
        return OptimizationBasedAttacker(model, loss, cfg_attack, setup)
    if cfg_attack.attack_type == "joint-optimization" and _loss_name(loss) in ("CrossEntropyLoss", "CausalLoss"):
        # classification models (deepleakage.yaml) and causal language models (tag.yaml, BASELINE config 5)
        return OptimizationJointAttacker(model, loss, cfg_attack, setup)
    if cfg_attack.attack_type == "multiscale":
        return MultiScaleOptimizationAttacker(model, loss, cfg_attack, setup)
    if cfg_attack.attack_type in _OTHER_ATTACKS:
        from ..install import reference_prepare_attack

        ref = reference_prepare_attack()
        if ref is not None:
            return ref(model, loss, cfg_attack, setup)
        raise NotImplementedError(
            f"attack_type={cfg_attack.attack_type} is not part of the accelerated path and the reference package "
            "`breaching` is not importable to delegate to."
        )
    raise ValueError(f"Invalid type of attack {cfg_attack.attack_type} given.")


__all__ = ["prepare_attack", "OptimizationBasedAttacker", "OptimizationJointAttacker", "MultiScaleOptimizationAttacker"]
