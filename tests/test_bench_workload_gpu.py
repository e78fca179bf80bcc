"""Parity of the paths ``bench.py`` times, at the sizes it times them (VERDICT round 1, item 1).

* config 2 (``bench.py`` default): tensor-core back end, torchvision ResNet-18, 397 classes, 1x3x224x224, seed 233 -- one closure
  evaluation against the CPU oracle in float32 and float64, with the *reference's own* GPU numerics (eager PyTorch, cuDNN TF32
  convolutions = torch's default) as the yardstick for the TF32 gradient; a 50-iteration trajectory; and
* a long-run quality test (>= 1000 iterations, 64x64, 3 seeds): final objective and PSNR against the ground truth
  (``analysis/metrics.py:108-130`` via ``bre_image_mse``) inside the spread of the reference algorithm run on the same GPU;
* config 4 (FedAvg, 4 local steps, ResNet-18 224^2, `modern` + TV double opponents): closure at full size.

Tolerances are stated next to each assertion together with what they were measured against.
"""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from breaching_b200 import analysis, get_attack_config, synthetic  # noqa: E402
from breaching_b200.engine import Engine  # noqa: E402
from breaching_b200.schedule import lr_table  # noqa: E402

DEV = torch.device("cuda:0")


def _relerr(a, b):
    return ((a.double().cpu() - b.double().cpu()).norm() / (b.double().cpu().norm() + 1e-30)).item()


def _sign_agreement(a, b):
    return (torch.sign(a.cpu()) == torch.sign(b.cpu())).float().mean().item()


class _tf32:
    """torch's GPU default for the reference: cuDNN convolutions in TF32 (SURVEY section 8c)."""

    def __enter__(self):
        self.old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = True
        torch.backends.cuda.matmul.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = self.old


def _oracle(model, loss_fn, cfg, shared, labels, meta, device="cpu", dtype=torch.float32, local=None):
    from oracle import restate

    dev = torch.device(device)
    dm = torch.tensor(meta.mean, device=dev, dtype=dtype)[None, :, None, None]
    ds = torch.tensor(meta.std, device=dev, dtype=dtype)[None, :, None, None]
    m = copy.deepcopy(model).to(dev, dtype).eval()
    if local is not None:
        local = dict(local, labels=[l.to(dev) for l in local["labels"]])
    return restate.TrialOracle(m, loss_fn, cfg, [g.to(dev, dtype) for g in shared[0]["gradients"]], labels.to(dev), dm, ds, dtype=dtype,
                               local_hyperparams=local)


def _engine(model, cfg, shared, labels, meta, shape, backend):
    eng = Engine(copy.deepcopy(model).to(DEV).eval(), shape, cfg, DEV, backend=backend)
    eng.load_model()
    eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], labels.to(DEV), mean=meta.mean, std=meta.std)
    return eng


def _config2():
    torch.manual_seed(234)   # bench.build_case: utils.py:159-167 seeding recipe with cfg.seed = 233
    model, loss_fn, payload, shared, true = synthetic.make_case("resnet18", "imagenet", batch=1, seed=233)
    return model, loss_fn, payload, shared, true, get_attack_config("invertinggradients")


def test_config2_tc_closure_at_the_benchmarked_size():
    model, loss_fn, payload, shared, true, cfg = _config2()
    meta = payload[0]["metadata"]
    from oracle import restate

    labels = restate.recover_labels(cfg.label_strategy, shared, 1)
    assert labels.tolist() == true["labels"].tolist()                      # label recovery: bit-exact
    x = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(8))
    o64 = _oracle(model, loss_fn, cfg, shared, labels, meta, dtype=torch.double)
    phi64, _, raw64, terms64 = o64.closure_gradient(x.double(), 0, 0.1)
    G64, _ = o64.param_gradient(x.double(), False)
    o32 = _oracle(model, loss_fn, cfg, shared, labels, meta)
    phi32, _, raw32, _ = o32.closure_gradient(x, 0, 0.1)
    with _tf32():                                                           # the reference on this GPU, as shipped
        ogpu = _oracle(model, loss_fn, cfg, shared, labels, meta, device=DEV)
        phig, _, rawg, _ = ogpu.closure_gradient(x.to(DEV), 0, 0.1)
        Gg, _ = ogpu.param_gradient(x.to(DEV), False)
    dev_fp32, dev_tf32 = _relerr(raw32, raw64), _relerr(rawg, raw64)
    worstG_tf32 = max(_relerr(a, b) for a, b in zip(Gg, G64))
    res = {}
    for backend in ("simt", "tc"):
        eng = _engine(model, cfg, shared, labels, meta, (1, 3, 224, 224), backend)
        val, grad = eng.objective_and_gradient(x.to(DEV))
        worstG = max(_relerr(eng.debug_param("G", i), G64[i]) for i in range(len(G64)))
        res[backend] = (val, _relerr(grad, raw64), _sign_agreement(grad, raw64), worstG)
        eng.close()
    print(f"config 2 closure: phi64 {float(phi64):.6f}; d(phi)/dx rel-l2 to float64: reference fp32 CPU {dev_fp32:.2e}, reference cuDNN-TF32 "
          f"GPU {dev_tf32:.2e} (objective {float(phig):.6f}, sign agreement {_sign_agreement(rawg, raw64):.4f}, worst-G {worstG_tf32:.2e}); engine "
          + "; ".join(f"{b}: value {v:.6f} rel {r:.2e} sign {s:.4f} worst-G {g:.2e}" for b, (v, r, s, g) in res.items()))
    # fp32 back end: the algorithm, to fp32 noise (SURVEY 7.4(3)(ii): 1e-3 / 99 %)
    v, r, s, g = res["simt"]
    assert math.isclose(v, float(phi64), rel_tol=2e-4) and r < max(1e-3, 2 * dev_fp32) and s > 0.99 and g < 1e-3, res["simt"]
    # tensor-core back end: objective to 2e-3; gradient no further from float64 than 1.5x the reference's own TF32 GPU path
    v, r, s, g = res["tc"]
    assert math.isclose(v, float(phi64), rel_tol=2e-3), (v, float(phi64))
    assert r < 1.5 * max(dev_tf32, 2e-3), (r, dev_tf32)
    assert s > min(0.985, _sign_agreement(rawg, raw64) - 0.01), (s, _sign_agreement(rawg, raw64))
    assert g < 1.5 * max(worstG_tf32, 2e-2), (g, worstG_tf32)   # per-tensor parameter gradients: same yardstick
    for o in (o64, o32, ogpu):
        o.close()


def test_config2_tc_trajectory_50_iterations():
    """50 signed-Adam iterations from the same initial candidate: the objective history of the tensor-core engine against the CPU
    oracle (fp32) and against the reference's GPU numerics.  A hard sign() turns numerically-zero gradient entries into +-lr
    jumps, so two correct implementations drift apart pixel-wise; the yardstick is how far the reference's own TF32 GPU run
    drifts from its CPU run."""
    model, loss_fn, payload, shared, true, cfg = _config2()
    meta = payload[0]["metadata"]
    labels = true["labels"]
    x0 = torch.randn(1, 3, 224, 224, generator=torch.Generator().manual_seed(9))
    n = 50
    ocpu = _oracle(model, loss_fn, cfg, shared, labels, meta)
    _, hcpu, _ = ocpu.run(x0, iterations=n)
    with _tf32():
        ogpu = _oracle(model, loss_fn, cfg, shared, labels, meta, device=DEV)
        _, hgpu, _ = ogpu.run(x0.to(DEV), iterations=n)
    eng = _engine(model, cfg, shared, labels, meta, (1, 3, 224, 224), "tc")
    opt = cfg.optim
    eng.begin_trial(x0.to(DEV), lr_table(opt.step_size, opt.step_size_decay, opt.warmup, opt.max_iterations))
    eng.run(n)
    eng.sync()
    heng = eng.history().tolist()
    assert len(heng) == n
    dev_ref = max(abs(a - b) / abs(b) for a, b in zip(hgpu, hcpu))
    dev_eng = max(abs(a - b) / abs(b) for a, b in zip(heng, hcpu))
    print(f"config 2 trajectory ({n} it): objective {hcpu[0]:.4f} -> {hcpu[-1]:.4f} (CPU oracle), {hgpu[-1]:.4f} (reference on GPU, TF32), "
          f"{heng[-1]:.4f} (engine tc); max rel. deviation from the CPU history: reference-GPU {dev_ref:.3e}, engine {dev_eng:.3e}")
    assert math.isclose(heng[0], hcpu[0], rel_tol=2e-3)
    # (measured over several runs: reference-GPU 1.8e-2 .. 2.5e-2 -- cuDNN picks algorithms per run --, engine 2.5e-2 .. 4.4e-2 depending on
    # the summation order of the BN reductions; a hard-sign trajectory amplifies either)
    assert dev_eng < max(3.0 * dev_ref, 5e-2), (dev_eng, dev_ref)
    assert heng[-1] < 0.8 * heng[0]                                          # and it optimises
    eng.close()
    ocpu.close()
    ogpu.close()


def _psnr(rec, true, meta):
    mse = analysis.E.image_mse(rec.to(DEV), true.to(DEV), meta.mean, meta.std, clamp=True)
    return sum(10 * math.log10(1.0 / m) for m in mse) / len(mse)


def test_long_run_quality_inside_the_reference_spread():
    """1200 iterations of `invertinggradients` on a 64x64 ResNet-18 case, three initialisations: final objective and PSNR
    against the ground truth for the engine (tensor-core and fp32 back ends) and for the reference algorithm run in eager PyTorch
    on the same GPU.  Different summation orders + hard sign = different trajectories; the claim is statistical: the engine's
    results lie inside the reference's spread."""
    model, loss_fn, payload, shared, true = synthetic.make_case("resnet18", "imagenet", batch=1, seed=233, bn_random=True, image_size=64,
                                                                classes=10)
    T = 1200
    cfg = get_attack_config("invertinggradients", {"optim.max_iterations": T, "optim.callback": T})
    meta = payload[0]["metadata"]
    labels = true["labels"]
    opt = cfg.optim
    table = lr_table(opt.step_size, opt.step_size_decay, opt.warmup, T)
    seeds = (0, 1, 2)
    ref_obj, ref_psnr = [], []
    with _tf32():
        ogpu = _oracle(model, loss_fn, cfg, shared, labels, meta, device=DEV)
        for s in seeds:
            x0 = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(s))
            best, hist, _ = ogpu.run(x0.to(DEV), iterations=T)
            ref_obj.append(min(hist))
            ref_psnr.append(_psnr(best, true["data"], meta))
        ogpu.close()
    out = {}
    for backend in ("tc", "simt"):
        eng = _engine(model, cfg, shared, labels, meta, (1, 3, 64, 64), backend)
        objs, psnrs = [], []
        for s in seeds:
            x0 = torch.randn(1, 3, 64, 64, generator=torch.Generator().manual_seed(s))
            eng.begin_trial(x0.to(DEV), table)
            eng.run(T)
            eng.sync()
            st = eng.status()
            assert st["recorded"] == T and not st["stopped"]
            objs.append(st["min_objective"])
            psnrs.append(_psnr(eng.best(), true["data"], meta))
        out[backend] = (objs, psnrs)
        eng.close()
    mean = lambda v: sum(v) / len(v)  # noqa: E731
    spread_o = max(ref_obj) - min(ref_obj)
    spread_p = max(ref_psnr) - min(ref_psnr)
    print(f"long run ({T} it, 64x64, seeds {seeds}): reference-on-GPU final objective {ref_obj} PSNR {ref_psnr}; "
          + "; ".join(f"engine {b}: objective {o} PSNR {p}" for b, (o, p) in out.items()))
    for backend, (objs, psnrs) in out.items():
        # final objective: the engine's mean within the reference's range widened by its spread (and 10 %)
        assert mean(objs) < max(ref_obj) + spread_o + 0.1 * mean(ref_obj), (backend, objs, ref_obj)
        # PSNR: not worse than the reference's mean by more than its spread (or 1 dB)
        assert mean(psnrs) > mean(ref_psnr) - max(spread_p, 1.0), (backend, psnrs, ref_psnr)


def test_config4_fedavg_closure_at_full_size():
    """BASELINE config 4: `modern` (cosine, soft sign, TV double opponents; features prior off: the reference crashes with it
    under FedAvg, SURVEY fact 9) on a ResNet-18 multi-step update (4 points, 4 local steps, lr 1e-3), 224x224.  FedAvg
    Hessian-vector products are ill-conditioned under TF32 in the reference as well; both back ends are measured against
    float64 with the reference's fp32 CPU / TF32 GPU deviations as yardsticks."""
    model, loss_fn, payload, shared, true = synthetic.make_fedavg_case("resnet18", "imagenet", num_data_points=4, steps=4, data_per_step=1,
                                                                       lr=1e-3, seed=233)
    cfg = get_attack_config("modern", {"regularization.features.scale": 0.0})
    meta = payload[0]["metadata"]
    local = shared[0]["metadata"]["local_hyperparams"]
    labels = torch.cat(local["labels"])
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(3))
    o64 = _oracle(model, loss_fn, cfg, shared, labels, meta, dtype=torch.double, local=local)
    phi64, _, raw64, _ = o64.closure_gradient(x.double(), 0, 0.0)
    o32 = _oracle(model, loss_fn, cfg, shared, labels, meta, local=local)
    _, _, raw32, _ = o32.closure_gradient(x, 0, 0.0)
    with _tf32():
        ogpu = _oracle(model, loss_fn, cfg, shared, labels, meta, device=DEV, local=local)
        _, _, rawg, _ = ogpu.closure_gradient(x.to(DEV), 0, 0.0)
    dev_fp32, dev_tf32 = _relerr(raw32, raw64), _relerr(rawg, raw64)
    res = {}
    for backend in ("simt", "tc"):
        eng = Engine(copy.deepcopy(model).to(DEV).eval(), (1, 3, 224, 224), cfg, DEV, backend=backend)
        eng.load_model()
        eng.load_targets([g.to(DEV) for g in shared[0]["gradients"]], local["labels"][0], mean=meta.mean, std=meta.std)
        eng.set_local_steps(4, local["steps"], local["lr"], local["labels"])
        val, grad = eng.objective_and_gradient(x.to(DEV))
        res[backend] = (val, _relerr(grad, raw64), eng.launches_per_iteration())
        eng.close()
    print(f"config 4 closure: phi64 {float(phi64):.6f}; rel-l2 to float64: reference fp32 CPU {dev_fp32:.2e}, reference TF32 GPU {dev_tf32:.2e}; "
          + "; ".join(f"engine {b}: value {v:.6f} rel {r:.2e}" for b, (v, r, _) in res.items()))
    assert math.isclose(res["simt"][0], float(phi64), rel_tol=1e-3) and res["simt"][1] < max(3 * dev_fp32, 2e-3), (res, dev_fp32)
    assert math.isclose(res["tc"][0], float(phi64), rel_tol=1e-2) and res["tc"][1] < 1.5 * max(dev_tf32, 3 * dev_fp32, 2e-3), (res, dev_tf32)
    for o in (o64, o32, ogpu):
        o.close()
