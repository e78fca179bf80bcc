"""The steps either side of the hot path on the engine (SURVEY section 8 f-2 / f-3): user-side update production
(``cases/users.py:107-200``) and the reconstruction-quality report (``analysis/analysis.py:204-283``, ``metrics.py:108-130``)
against plain PyTorch restatements of the reference formulas on the CPU."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import analysis, synthetic  # noqa: E402
from breaching_b200.users import UserSingleStep  # noqa: E402

DEV = torch.device("cuda:0")
SETUP = dict(device=DEV, dtype=torch.float)


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _update_error(got, want):
    """(rel. l2 error of the whole update, worst per-tensor error measured against max(|tensor|, 1e-3 |update|)): a conv bias in
    front of a train-mode BN has an exactly-zero gradient, whose own norm is pure rounding noise."""
    total = torch.cat([w.double().flatten().cpu() for w in want]).norm().item()
    diff = torch.cat([(g.double().cpu() - w.double().cpu()).flatten() for g, w in zip(got, want)]).norm().item()
    worst = max((g.double().cpu() - w.double().cpu()).norm().item() / max(w.double().norm().item(), 1e-3 * total) for g, w in zip(got, want))
    return diff / total, worst


@pytest.mark.parametrize("arch,size,batch", [("convnet-tiny", 32, 3), ("resnet18", 64, 2)])
def test_user_gradient_matches_autograd(arch, size, batch):
    data = "cifar" if size == 32 else "imagenet"
    model, loss_fn, payload, shared, true = synthetic.make_case(arch, data, batch=batch, seed=11, bn_random=True, image_size=size, classes=10,
                                                                provide_labels=True)
    user = UserSingleStep(model, loss_fn, dict(SETUP), batch, backend="simt")
    sd, tud = user.compute_local_updates(payload[0], dict(inputs=true["data"], labels=true["labels"]))
    assert sd["buffers"] is None and sd["metadata"]["num_data_points"] == batch
    assert sd["metadata"]["labels"].tolist() == true["labels"].sort()[0].tolist()
    assert all(g.shape == w.shape for g, w in zip(sd["gradients"], shared[0]["gradients"]))
    rel, worst = _update_error(sd["gradients"], shared[0]["gradients"])   # make_case computed them with torch.autograd (eval-mode BN)
    assert rel < 1e-4 and worst < 2e-4, (rel, worst)
    # the TF32 tensor-core back end: same update to TF32 accuracy (per tensor: a few per cent on the small BN vectors, as for
    # cuDNN's TF32 path, tests/test_bench_workload_gpu.py prints both)
    user_tc = UserSingleStep(model, loss_fn, dict(SETUP), batch, backend="tc")
    sd_tc, _ = user_tc.compute_local_updates(payload[0], dict(inputs=true["data"], labels=true["labels"]))
    rel, worst = _update_error(sd_tc["gradients"], shared[0]["gradients"])
    # typical: ResNet-18 ~2e-2 / ~6e-2; ConvNet-tiny ~1e-3 overall, ~0.2 on its smallest-norm tensor
    assert rel < 4e-2 and worst < 0.5, (rel, worst)


def test_user_per_example_clipping_and_noise():
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=3, seed=5, bn_random=True, provide_labels=True)
    clip = 0.5
    user = UserSingleStep(model, loss_fn, dict(SETUP), 3, per_example_clipping=clip, backend="simt")
    sd, _ = user.compute_local_updates(payload[0], dict(inputs=true["data"], labels=true["labels"]))
    m = copy.deepcopy(model).eval()
    params = list(m.parameters())
    want = [torch.zeros_like(p) for p in params]
    clipped = 0
    for i in range(3):                                                     # users.py:158-165, :190-194
        g = torch.autograd.grad(loss_fn(m(true["data"][i:i + 1]), true["labels"][i:i + 1]), params)
        norm = torch.norm(torch.stack([torch.norm(t, 2) for t in g]), 2)
        if norm > clip:
            g = [t * (clip / (norm + 1e-6)) for t in g]
            clipped += 1
        want = [a + b for a, b in zip(want, g)]
    want = [t / 3 for t in want]
    assert clipped > 0
    assert _update_error(sd["gradients"], want)[1] < 5e-4
    noisy = UserSingleStep(model, loss_fn, dict(SETUP), 3, gradient_noise=1e-2, backend="simt")
    torch.manual_seed(0)
    sdn, _ = noisy.compute_local_updates(payload[0], dict(inputs=true["data"], labels=true["labels"]))
    diff = torch.cat([(a.cpu() - b).flatten() for a, b in zip(sdn["gradients"], shared[0]["gradients"])])
    assert 0.8e-2 < diff.std().item() < 1.2e-2                             # users.py:196-200: N(0, scale) on every entry


def test_user_train_mode_ships_buffers():
    """No public buffers: the user runs in train mode with momentum None and ships its BN buffers (users.py:140-143,174)."""
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=4, seed=9, user_buffers=True, provide_labels=True)
    assert payload[0]["buffers"] is None and shared[0]["buffers"] is not None
    user = UserSingleStep(model, loss_fn, dict(SETUP), 4, backend="simt")
    sd, tud = user.compute_local_updates(payload[0], dict(inputs=true["data"], labels=true["labels"]))
    rel, worst = _update_error(sd["gradients"], shared[0]["gradients"])
    assert rel < 2e-4 and worst < 5e-4, (rel, worst)
    assert len(sd["buffers"]) == len(shared[0]["buffers"])
    for got, want in zip(sd["buffers"], shared[0]["buffers"]):
        if want.dtype == torch.long:
            assert int(got) == int(want)
        else:
            assert _relerr(got, want) < 1e-4, _relerr(got, want)


def test_report_mse_psnr_label_accuracy():
    model, loss_fn, payload, shared, true = synthetic.make_case("convnet-tiny", "cifar", batch=3, seed=2, bn_random=True, provide_labels=True)
    meta = payload[0]["metadata"]
    gen = torch.Generator().manual_seed(1)
    rec = true["data"] + 0.3 * torch.randn(true["data"].shape, generator=gen)
    rec[0, :, :4] += 5.0   # saturates: exercises the clamp
    out = analysis.report(dict(data=rec.to(DEV), labels=true["labels"].to(DEV)), dict(data=true["data"], labels=true["labels"], buffers=None),
                          payload, model, setup=SETUP)
    dm = torch.tensor(meta.mean)[None, :, None, None]
    ds = torch.tensor(meta.std)[None, :, None, None]
    a = torch.clamp(rec * ds + dm, 0, 1)
    b = torch.clamp(true["data"] * ds + dm, 0, 1)
    mse = (a - b).pow(2).mean(dim=[1, 2, 3])                                # analysis.py:236-238
    psnr = 10 * torch.log10(1.0 / mse)                                      # metrics.py:108-130
    assert math.isclose(out["mse"], mse.mean().item(), rel_tol=1e-5) and math.isclose(out["max_mse"], mse.max().item(), rel_tol=1e-5)
    assert math.isclose(out["psnr"], psnr.mean().item(), rel_tol=1e-5) and math.isclose(out["max_psnr"], psnr.max().item(), rel_tol=1e-5)
    assert out["label_acc"] == 1.0 and out["parameters"] == sum(p.numel() for p in model.parameters())
    m = copy.deepcopy(model).eval()
    with torch.no_grad():
        want = (m(rec) - m(true["data"]))[..., true["labels"].view(-1)].pow(2).mean().item()
    assert math.isclose(out["feat_mse"], want, rel_tol=2e-3), (out["feat_mse"], want)   # the report runs its forward passes in fp32
    mean_psnr, max_psnr = analysis.psnr_compute(a.to(DEV), b.to(DEV), factor=1.0)
    assert math.isclose(mean_psnr, psnr.mean().item(), rel_tol=1e-5) and math.isclose(max_psnr, psnr.max().item(), rel_tol=1e-5)


@pytest.mark.parametrize("shape,size", [((2, 3, 16, 16), 32), ((1, 3, 32, 32), 20), ((2, 3, 9, 13), (17, 7)), ((1, 1, 7, 7), 7)])
def test_bilinear_resize_equals_interpolate(shape, size):
    from breaching_b200.engine import resize_bilinear

    x = torch.randn(shape, generator=torch.Generator().manual_seed(3))
    want = torch.nn.functional.interpolate(x, size=size, mode="bilinear", align_corners=False)
    got = resize_bilinear(x.to(DEV), size)
    assert got.shape == want.shape and (got.cpu() - want).abs().max().item() < 1e-5


def test_multiscale_attack_runs_its_stages_on_the_engine():
    """MultiScaleOptimizationAttacker (multiscale_optimization_attack.py:18-122; preset multiscale_ghiasi.yaml without its
    augmentations): two stages of a log pyramid on a ResNet-18 -- every stage is a trial of a layer program compiled for that
    resolution, candidates move between stages through bre_resize_bilinear, the history concatenates the stages, and a
    one-stage `trivial` pyramid equals the plain attacker's trial from the same initial candidate."""
    from breaching_b200 import get_attack_config
    from breaching_b200.attacks import prepare_attack
    from breaching_b200.attacks.multiscale_attack import scale_pyramid

    assert scale_pyramid("linear", 7, 224) == [32, 64, 96, 128, 160, 192, 224]      # :32-33
    assert scale_pyramid("log", 3, 64) == [16, 32, 64] and scale_pyramid("trivial", 2, 8) == [8, 8]
    model, loss_fn, payload, shared, true = synthetic.make_case("resnet18", "imagenet", batch=1, seed=4, bn_random=True, image_size=64, classes=10)
    over = {"augmentations": None, "num_stages": 2, "scale_pyramid": "log", "resize": "upsampling", "optim.max_iterations": 6, "optim.callback": 3}
    cfg = get_attack_config("multiscale_ghiasi", over)
    attacker = prepare_attack(model, loss_fn, cfg, dict(SETUP, backend="simt"))
    assert type(attacker).__name__ == "MultiScaleOptimizationAttacker"
    torch.manual_seed(0)
    rec, stats = attacker.reconstruct(payload, copy.deepcopy(shared), {})
    assert rec["data"].shape == (1, 3, 64, 64) and torch.isfinite(rec["data"]).all()
    hist = stats["Trial_0_Val"]
    assert len(hist) == 12 and hist[5] < hist[0] and hist[11] < hist[6]                # two stages of 6 iterations, each optimising
    assert sorted(attacker._stage_engines) == [32]                                     # the 64x64 stage runs on the attacker's main engine
    # `focus` pasting and a trivial pyramid
    cfg2 = get_attack_config("multiscale_ghiasi", dict(over, resize="focus", scale_pyramid="trivial", num_stages=1))
    rec2, stats2 = prepare_attack(model, loss_fn, cfg2, dict(SETUP, backend="simt")).reconstruct(payload, copy.deepcopy(shared), {})
    assert len(stats2["Trial_0_Val"]) == 6 and rec2["data"].shape == (1, 3, 64, 64)
