"""Shared helpers for the parity tests."""
import copy
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from breaching_b200 import config as bcfg  # noqa: E402
from breaching_b200 import synthetic  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def load_golden(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cfg_from_fixture(fx):
    return bcfg.get_attack_config(fx["attack"], dict(fx["overrides"]))


def case_from_fixture(fx):
    if "seq_len" in fx["case"]:
        model, loss_fn, payload, shared, true = synthetic.make_text_case(**fx["case"])
    elif "steps" in fx["case"]:
        model, loss_fn, payload, shared, true = synthetic.make_fedavg_case(**fx["case"])
    elif "queries" in fx["case"]:
        model, loss_fn, payload, shared, true = synthetic.make_multi_query_case(**fx["case"])
    else:
        model, loss_fn, payload, shared, true = synthetic.make_case(**fx["case"])
    checksum = float(sum(p.double().sum() for p in model.parameters()))
    assert abs(checksum - fx["weight_checksum"]) <= 1e-6 * max(1.0, abs(fx["weight_checksum"])), \
        "synthetic case differs from the one the fixture was generated with"
    return model, loss_fn, payload, shared, true


def oracle_for_fixture(fx):
    """TrialOracle (CPU restatement) set up exactly like the reference attacker was for this fixture."""
    from oracle import restate

    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    shared = copy.deepcopy(shared)
    m = copy.deepcopy(model)
    if shared[0]["buffers"] is not None:
        for buf, src in zip(m.buffers(), shared[0]["buffers"]):
            buf.data.copy_(src)
    m.eval()
    if shared[0]["buffers"] is None and payload[0]["buffers"] is None:  # base_attack.py:192-197: no buffers anywhere -> train mode
        m.train()
        for mod in m.modules():
            if hasattr(mod, "track_running_stats"):
                mod.track_running_stats = False
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean)[None, :, None, None]
    ds = torch.tensor(meta.std)[None, :, None, None]
    labels = restate.recover_labels(cfg.label_strategy, shared, shared[0]["metadata"]["num_data_points"])
    return restate.TrialOracle(m, loss_fn, cfg, shared[0]["gradients"], labels, dm, ds,
                               local_hyperparams=shared[0]["metadata"]["local_hyperparams"]), cfg, labels


TRIAL_FIXTURES = ["ig_convnet", "ig_resnet18", "stg_resnet18", "modern_convnet", "tag_clip_convnet", "l1_sgd_convnet"]
FEDAVG_FIXTURES = ["fedavg_convnet", "fedavg_resnet18"]
LBFGS_FIXTURES = ["lbfgs_convnet", "lbfgs_wei_convnet", "lbfgs_cosine_convnet"]
JOINT_FIXTURES = ["joint_dlg_convnet", "joint_adam_convnet", "joint_tag_transformer"]
MULTI_QUERY_FIXTURES = ["multiquery_convnet"]
TRAIN_BN_FIXTURES = ["trainbn_convnet", "trainbn_resnet18"]


def joint_oracle_for_fixture(fx):
    """JointTrialOracle (CPU restatement of OptimizationJointAttacker) for a joint-optimisation fixture."""
    from oracle import restate

    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    m = copy.deepcopy(model).eval()
    meta = payload[0]["metadata"]
    grads = list(shared[0]["gradients"])
    if getattr(meta, "modality", "vision") == "text":
        # base_attack.py:76-128 ("run-embedding"): optimise in embedding space -- drop the token-embedding gradient and bypass
        # the embedding layer; no input normalisation
        names = [n for n, _ in m.named_parameters()]
        grads.pop(names.index("encoder.weight"))
        m.encoder = torch.nn.Identity()
        dm, ds = torch.tensor(0.0), torch.tensor(1.0)
    else:
        dm = torch.tensor(meta.mean)[None, :, None, None]
        ds = torch.tensor(meta.std)[None, :, None, None]
    return restate.JointTrialOracle(m, loss_fn, cfg, grads, None, dm, ds), cfg


def multi_query_oracle_for_fixture(fx):
    """MultiQueryOracle: one TrialOracle per (model, update) pair, regularisers only on the first."""
    from oracle import restate

    model, loss_fn, payload, shared, true = case_from_fixture(fx)
    cfg = cfg_from_fixture(fx)
    no_priors = copy.deepcopy(cfg)
    if no_priors.get("regularization") is not None:
        for key in no_priors["regularization"].keys():
            no_priors["regularization"][key]["scale"] = 0.0
    meta = payload[0]["metadata"]
    dm = torch.tensor(meta.mean)[None, :, None, None]
    ds = torch.tensor(meta.std)[None, :, None, None]
    labels = restate.recover_labels(cfg.label_strategy, copy.deepcopy(shared), shared[0]["metadata"]["num_data_points"])
    oracles = []
    for i, (pl, sh) in enumerate(zip(payload, shared)):
        m = copy.deepcopy(model)
        with torch.no_grad():
            for p, src in zip(m.parameters(), pl["parameters"]):
                p.copy_(src)
            for b, src in zip(m.buffers(), pl["buffers"]):
                b.copy_(src)
        m.eval()
        oracles.append(restate.TrialOracle(m, loss_fn, cfg if i == 0 else no_priors, sh["gradients"], labels, dm, ds))
    return restate.MultiQueryOracle(oracles), cfg, labels


class OddNet(torch.nn.Module):
    """A network that reaches the scalar (non-float4) element-wise and pooling kernels and the accumulation paths of the BN / ReLU /
    residual kernels.  A 6-channel branch (C % 4 != 0: scalar kernels) with a conv without bias, BN without ReLU, ReLU without
    BN and residual adds without BN; maxpool 3/2/1 on odd sizes; a 10-channel conv + BN + ReLU; an 8-channel branch (float4
    kernels) with the same shapes of reuse; a linear head on a spatial map.  In both branches a BN / ReLU / add op reads a tensor
    that a later op also reads (``acc_in``) and takes as residual a tensor that a later op also reads (``acc_res``).  Meant for
    15 x 13 inputs."""

    def __init__(self, classes=5):
        super().__init__()
        self.conv1 = torch.nn.Conv2d(3, 6, 3, padding=1)
        self.bn1 = torch.nn.BatchNorm2d(6)
        self.conv2 = torch.nn.Conv2d(6, 6, 3, padding=1, bias=False)
        self.relu = torch.nn.ReLU()
        self.pool = torch.nn.MaxPool2d(3, 2, 1)
        self.conv3 = torch.nn.Conv2d(6, 10, 3, padding=1, bias=False)
        self.bn3 = torch.nn.BatchNorm2d(10)
        self.conv5 = torch.nn.Conv2d(10, 8, 3, padding=1)
        self.bn5 = torch.nn.BatchNorm2d(8)
        self.conv6 = torch.nn.Conv2d(8, 8, 3, padding=1, bias=False)
        self.conv7 = torch.nn.Conv2d(8, 8, 1)
        self.fc = torch.nn.Linear(8 * 8 * 7, classes)

    def forward(self, x):
        a = self.bn1(self.conv1(x))          # BN without ReLU
        r = self.relu(a)                     # ReLU without BN; conv2 reads `a` later -> acc_in
        b = self.relu(self.conv2(a))
        s = r + b                            # residual add without BN; the next add reads `b` later -> acc_res
        c = self.pool(s + b)
        d = self.relu(self.bn3(self.conv3(c)))
        e = self.bn5(self.conv5(d))
        g = self.relu(e)                     # 8 channels: conv6 reads `e` later -> acc_in (float4)
        h = self.conv6(e)
        k = g + h                            # conv7 reads `h` later -> acc_res (float4)
        u = self.conv7(h) + k
        return self.fc(torch.flatten(u, 1))


def odd_case(seed=5, batch=3):
    """(model in eval mode with random BN, input shape, labels, target gradients) for :class:`OddNet`."""
    torch.manual_seed(seed)
    model = synthetic.randomize_bn(OddNet(), seed + 1).eval()
    gen = torch.Generator().manual_seed(seed + 7)
    x = torch.randn(batch, 3, 15, 13, generator=gen)
    y = torch.randint(0, 5, (batch,), generator=gen)
    grads = torch.autograd.grad(torch.nn.functional.cross_entropy(model(x), y), list(model.parameters()))
    return model, (batch, 3, 15, 13), y, [g.detach() for g in grads]


class BNRegisteredLate(torch.nn.Module):
    """conv -> BN -> ReLU -> conv -> BN -> ReLU -> avg-pool -> Linear, with the second BN registered before the first: the first
    registered BatchNorm2d, which the reference's DeepInversion prior weights by ``first_bn_multiplier``, is not the first that
    runs.  ``in_order``: the same layers registered in the order they run (same parameter and buffer names)."""

    def __init__(self, in_order=False):
        super().__init__()
        if not in_order:
            self.bn2 = torch.nn.BatchNorm2d(16)
        self.conv1 = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.bn1 = torch.nn.BatchNorm2d(8)
        self.conv2 = torch.nn.Conv2d(8, 16, 3, stride=2, padding=1)
        if in_order:
            self.bn2 = torch.nn.BatchNorm2d(16)
        self.pool = torch.nn.AdaptiveAvgPool2d(1)
        self.fc = torch.nn.Linear(16, 10)

    def forward(self, x):
        x = torch.relu(self.bn1(self.conv1(x)))
        x = torch.relu(self.bn2(self.conv2(x)))
        return self.fc(torch.flatten(self.pool(x), 1))


class LinearRegisteredLast(torch.nn.Module):
    """conv -> ReLU -> avg-pool -> proj (Linear 16 -> 16) -> ReLU -> fc (Linear 16 -> 10), with proj registered after fc: the last
    registered Linear, whose input the reference's features prior reads (and whose weight / bias gradients are the last two
    entries the feature targets are derived from), is not the last that runs.  ``in_order``: registered in the order they run."""

    def __init__(self, in_order=False):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 16, 3, stride=2, padding=1)
        self.pool = torch.nn.AdaptiveAvgPool2d(1)
        if in_order:
            self.proj = torch.nn.Linear(16, 16)
        self.fc = torch.nn.Linear(16, 10)
        if not in_order:
            self.proj = torch.nn.Linear(16, 16)

    def forward(self, x):
        x = torch.flatten(self.pool(torch.relu(self.conv(x))), 1)
        return self.fc(torch.relu(self.proj(x)))


def registration_case(cls, in_order=False, seed=3, batch=2, size=12):
    """(model in eval mode with random BN, input shape, labels, target gradients) of a :class:`BNRegisteredLate` /
    :class:`LinearRegisteredLast`; the ``in_order`` twin has exactly the same parameters and buffers."""
    torch.manual_seed(seed)
    model = synthetic.randomize_bn(cls(), seed + 1).eval()
    if in_order:
        twin = cls(in_order=True)
        twin.load_state_dict(model.state_dict())
        model = twin.eval()
    gen = torch.Generator().manual_seed(seed + 7)
    x = torch.randn(batch, 3, size, size, generator=gen)
    y = torch.randint(0, 10, (batch,), generator=gen)
    grads = torch.autograd.grad(torch.nn.functional.cross_entropy(model(x), y), list(model.parameters()))
    return model, (batch, 3, size, size), y, [g.detach() for g in grads]


def sweep_objective(cfg, features=None):
    """The objective dict of ``oracle.sweep_check.SweepChecker`` for an attack config."""
    reg = cfg.get("regularization") or {}

    def on(key):
        return key in reg and reg[key]["scale"] > 0

    obj = dict(kind=cfg.objective.type, scale=float(cfg.objective.get("scale", 1.0)),
               task_regularization=float(cfg.objective.get("task_regularization", 0.0) or 0.0))
    if cfg.objective.type == "tag-euclidean":
        obj.update(tag_scale=float(cfg.objective.get("tag_scale", 0.1)), scale_scheme=cfg.objective.get("scale_scheme", "linear"))
    if on("total_variation"):
        r = reg["total_variation"]
        obj["tv"] = dict(scale=r["scale"], inner_exp=r.get("inner_exp", 1), outer_exp=r.get("outer_exp", 1), eps=r.get("eps", 1e-8),
                         double_opponents=bool(r.get("double_opponents", False)))
    if on("norm"):
        obj["norm"] = dict(scale=reg["norm"]["scale"], p=reg["norm"].get("pnorm", 2.0))
    if on("deep_inversion"):
        obj["di"] = dict(scale=reg["deep_inversion"]["scale"], first_bn_multiplier=reg["deep_inversion"].get("first_bn_multiplier", 10))
    if on("features") and features is not None:
        obj["features"] = dict(scale=reg["features"]["scale"], measured=features)
    if on("orthogonality"):   # the reference never multiplies this term by its scale (engine.make_cfg)
        obj["orthogonality"] = True
    return obj


def tensor_weights(cfg, L):
    """Per-tensor weights the attack hands to ``Engine.load_targets`` for tag-euclidean (optimization_attack.py), else None."""
    from oracle.sweep_check import tag_weights

    if cfg.objective.type != "tag-euclidean":
        return None
    return tag_weights(L, cfg.objective.get("scale_scheme", "linear"))


def masked_targets(grads):
    """Target gradients that reach both sides of masked-cosine's strict ``|g| > float32(1e-6)``: in the largest tensor exact zeros,
    +-float32(1e-6) and its two fp32 neighbours; one other tensor of at least 1024 elements zeroed whole (fully masked chunks)."""
    g = [t.detach().clone().float() for t in grads]
    big = max(range(len(g)), key=lambda j: g[j].numel())
    m = torch.tensor(1e-6, dtype=torch.float32)
    edge = torch.stack([m, torch.nextafter(m, torch.tensor(0.0)), torch.nextafter(m, torch.tensor(1.0))])
    edge = torch.cat([edge, -edge, torch.zeros(3)])
    flat = g[big].view(-1)
    n = (flat.numel() // (2 * edge.numel())) * edge.numel()
    flat[:n] = edge.repeat(n // edge.numel())
    whole = next(j for j in range(len(g)) if j != big and g[j].numel() >= 1024)
    g[whole].zero_()
    return g


def unwritten_tangents(eng):
    """Tensors whose tangent the last evaluation did not store (fuse_bnact: a conv output whose only consumer is the BN op that ran
    in the conv's epilogue), as the engine reports them."""
    return {op.tin for i, op in enumerate(eng.prog.ops) if eng.debug_op(i)["tangent_in_unwritten"]}


class EngineSource:
    """The sweep checker's buffer source (oracle/sweep_check.py): the engine's debug read-back (NCHW / torch layout).  Build it
    after the evaluation."""

    def __init__(self, eng):
        self.eng = eng
        self.unwritten = unwritten_tangents(eng)
        self.stem = {i for i in range(len(eng.prog.ops)) if eng.debug_op(i)["stem_columns"]}

    def rounds_operands(self, i):
        return i in self.stem   # the candidate-fed conv on the tensor-core column path rounds x, W and v itself

    def tensor(self, which, tid):
        if tid == 0 and which == "tangent":
            return None
        return self.eng.debug_tensor(which, tid).double()

    def param(self, which, idx):
        return self.eng.debug_param(which, idx).double()
