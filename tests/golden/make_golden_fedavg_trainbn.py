"""Generate the FedAvg fixtures of train-mode BatchNorm networks in this directory (``trial_fedavg_trainbn_convnet.pt``,
``trial_fedavg_trainbn_taskreg_convnet.pt``, ``trial_fedavg_trainbn_resnet18.pt``) by running the reference, the way
``make_golden.py`` produces the others.

Run where the reference is importable (``BREACHING_REFERENCE_ROOT``, see oracle/refshim.py):
``python tests/golden/make_golden_fedavg_trainbn.py [fixture names]``

Neither the server nor the user ships BN buffers (``synthetic.make_fedavg_case(no_buffers=True)``): the user trains every local
step in train mode and the unmodified reference attacker evaluates its FedAvg objective the same way (base_attack.py:192-197,
objectives.py:48-72).
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository root on sys.path)
from oracle import refshim  # noqa: E402

CONVNET = dict(model_name="convnet-tiny", data="cifar", num_data_points=4, steps=3, data_per_step=2, lr=0.05, bn_random=True,
               no_buffers=True)
CASES = {
    # name: (case kwargs, attack yaml, overrides, iterations)
    "fedavg_trainbn_convnet": (dict(CONVNET, seed=51), "modern", {"regularization.features.scale": 0.0}, 6),
    "fedavg_trainbn_taskreg_convnet": (dict(CONVNET, seed=52), "modern",
                                       {"regularization.features.scale": 0.0, "objective.task_regularization": 0.1}, 3),
    "fedavg_trainbn_resnet18": (dict(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=0.01, seed=53,
                                     bn_random=True, image_size=64, classes=10, no_buffers=True), "modern",
                                {"regularization.features.scale": 0.0}, 2),
}
# Iterations: batch statistics over two images (or over 2 x 2 pixels in ResNet-18's last stage) make these attacks badly
# conditioned, and fp32 rounding soon dominates the recorded history.  Against a float64 run of the same attack the fixtures
# deviate by 2e-3 to 5e-3 at ConvNet iterations 5-6, by 3.5e-2 at the task-loss ConvNet's iteration 3 and by 7.6e-3 already at
# ResNet-18's first objective.  Beyond their first iterations they therefore record fp32 rounding rather than the attack: an
# implementation that runs the reference's own torch ops (the CPU oracle) reproduces them to 2e-4, another one only over the first
# iterations.


def main():
    ref = refshim.import_reference()
    only = sys.argv[1:]
    for name, (case_kwargs, attack, overrides, iters) in CASES.items():
        if only and name not in only:
            continue
        torch.manual_seed(0)
        fx = make_golden.run_reference(ref, case_kwargs, attack, overrides, iters)
        torch.save(fx, os.path.join(HERE, f"trial_{name}.pt"))
        print(name, "history", [round(h, 5) for h in fx["history"]], "score", fx["score"])


if __name__ == "__main__":
    main()
