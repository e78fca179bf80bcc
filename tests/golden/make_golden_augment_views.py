"""Generate ``augment_views.pt`` in this directory by running the reference's shape-changing augmentations
(``attacks/auxiliaries/augmentations.py``: ``Zoom``, ``CenterZoom``, ``Focus``, ``AntiAlias``) and one attack with a
``centerzoom`` + ``antialias`` view, the way ``make_golden.py`` produces the other fixtures.

Run where the reference is importable (``BREACHING_REFERENCE_ROOT``, see oracle/refshim.py):
``python tests/golden/make_golden_augment_views.py``

Contents:
- ``modules``: float64 output and vector-Jacobian product of each module on seeded inputs (non-square, up- and down-sampling
  zoom, every antialias width at strides 1 and 2, focus with its drawn ``pert`` recorded);
- ``trial``: the closure at x0 and a short trajectory of ``invertinggradients`` on a small ResNet-18 with
  ``differentiable_augmentations: True`` and the deterministic view ``centerzoom`` (fov < H, out = H) then ``antialias``.
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the repository root on sys.path)
from oracle import refshim  # noqa: E402

SHAPES = [(2, 3, 9, 13), (1, 3, 12, 10)]
MODULE_CASES = (
    [("Zoom", dict(out_size=s), shape) for s in (16, 5) for shape in SHAPES]
    + [("CenterZoom", dict(initial_fov=6, out_size=15), shape) for shape in SHAPES]
    + [("CenterZoom", dict(initial_fov=8, out_size=4), shape) for shape in SHAPES]
    + [("Focus", dict(size=6, std=2.0), shape) for shape in SHAPES]
    + [("Focus", dict(size=9, std=3.0), (2, 3, 9, 13))]                  # window = full height: the row corner clamps to 0
    + [("AntiAlias", dict(channels=3, width=w, stride=s), SHAPES[i % 2]) for i, (w, s) in
       enumerate((w, s) for w in range(1, 8) for s in (1, 2))]
)
TRIAL = (dict(model_name="resnet18", data="imagenet", batch=1, seed=71, bn_random=True, image_size=32, classes=10), "invertinggradients",
         {"augmentations": {"centerzoom": {"initial_fov": 16, "out_size": 32}, "antialias": {"channels": 3, "width": 3, "stride": 1}},
          "differentiable_augmentations": True, "optim.signed": "soft"}, 5)


def module_fixtures(ref):
    aug = ref.attacks.auxiliaries.augmentations
    out = []
    for i, (name, kwargs, shape) in enumerate(MODULE_CASES):
        gen = torch.Generator().manual_seed(100 + i)
        x = torch.randn(shape, generator=gen, dtype=torch.float64)
        mod = getattr(aug, name)(**kwargs).double()
        entry = dict(name=name, kwargs=kwargs, x=x)
        xr = x.clone().requires_grad_(True)
        if name == "Focus":                                  # the module draws pert from torch's global generator
            torch.manual_seed(500 + i)
            entry["pert"] = (torch.rand(2) * 2 - 1) * kwargs["std"]
            torch.manual_seed(500 + i)
        y = mod(xr)
        g = torch.randn(y.shape, generator=gen, dtype=torch.float64)
        (vjp,) = torch.autograd.grad((y * g).sum(), xr)
        entry.update(y=y.detach(), g=g, vjp=vjp)
        out.append(entry)
    return out


def main():
    ref = refshim.import_reference()
    case, attack, overrides, iters = TRIAL
    fx = dict(modules=module_fixtures(ref), trial=make_golden.run_reference(ref, case, attack, overrides, iters))
    torch.save(fx, os.path.join(HERE, "augment_views.pt"))
    print("augment_views history", [round(h, 5) for h in fx["trial"]["history"]], "score", fx["trial"]["score"])


if __name__ == "__main__":
    main()
