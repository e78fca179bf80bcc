"""Small networks that reach the layer geometries compiler.compile_model accepts beyond the benchmarked ones: the column path of the
candidate-fed convolution with 1-4 input channels, candidate-fed convolutions off that path, strided inner convolutions with every
filter size the parity-class dgrad distinguishes, max-pools whose windows skip, overlap, pad or tie, two-layer heads and batches on
both sides of the small-linear kernels.  tests/test_layer_program_cases_cpu.py checks the float64 four-sweep formulation of every case
against autograd and that the table reaches every rule listed in ``REQUIRED``; tests/test_layer_programs_gpu.py checks every sweep
buffer of every case against float64 on both GEMM back ends.

``reached(case, backend)`` restates, from the program alone, which engine rules a case takes: the stem column path
(csrc/engine.cu: a convolution reading the candidate with at most 4 channels, ``Co % 64 == 0`` and ``R * S <= 64``, on the
tensor-core back end unless the layer is kept precise), the vector (``C % 4 == 0``) or scalar element-wise and pooling kernels, and
the GEMM families and tensor-core plans of scripts/profile_gemms.gemm_plan."""
import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "scripts")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from breaching_b200 import compiler as C  # noqa: E402

CLASSES = 10
TIE_BETA = -4.0   # BN shift of every other channel of the tie cases: after the ReLU all its max-pool windows are zero ties


def bn(c, train=False):
    return nn.BatchNorm2d(c, track_running_stats=not train)


class TwoBranch(nn.Module):
    """stem -> BN(strongly negative shift) -> ReLU -> max-pool 3/1/1, read by a tensor-core 3x3 conv and by a 9x9 conv (R * S > 64:
    fp32 kernels) whose outputs are added."""

    def __init__(self):
        super().__init__()
        self.stem = nn.Conv2d(3, 128, 2, stride=3)
        self.bn = bn(128)
        self.relu = nn.ReLU()
        self.pool = nn.MaxPool2d(3, 1, 1)
        self.tc = nn.Conv2d(128, 64, 3, padding=1)
        self.simt = nn.Conv2d(128, 64, 9, padding=4, bias=False)
        self.head = nn.Sequential(nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(64, CLASSES))

    def forward(self, x):
        p = self.pool(self.relu(self.bn(self.stem(x))))
        return self.head(self.tc(p) + self.simt(p))


def _head(c):
    return [nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(c, CLASSES)]


def _stem1():
    return nn.Sequential(nn.Conv2d(1, 64, 3), bn(64), nn.ReLU(), nn.MaxPool2d(2, 2, 0), nn.Conv2d(64, 32, 3, 2, 2), *_head(32))


# name -> (purpose, model factory, input shape, engine options)
CASES = {
    "stem1-k3s1p0": ("1-channel column-path stem 3x3/1/0 on an odd 17x15 image; max-pool 2/2/0 into a 32-wide tensor-core conv "
                     "3x3/2/2 (pad > R/2)",
                     _stem1, (2, 1, 17, 15), ()),
    "stem2-k4s4p0": ("2-channel column-path stem 4x4/4/0 with 128 outputs (the last image row has no tap); 2x2/2/0 conv with "
                     "unequal parity classes (5 x 4 input); linear on a spatial map",
                     lambda: nn.Sequential(nn.Conv2d(2, 128, 4, 4), nn.ReLU(), nn.Conv2d(128, 64, 2, 2), nn.ReLU(), nn.Flatten(),
                                 nn.Linear(64 * 2 * 2, CLASSES)),
                     (3, 2, 21, 18), ()),
    "stem3-k5s2p2": ("3-channel column-path stem 5x5/2/2 at batch 1; max-pool 3/2/1; 5x5/2/2 and 1x1/2/0 strided convs, 160 wide",
                     lambda: nn.Sequential(nn.Conv2d(3, 64, 5, 2, 2), bn(64), nn.ReLU(), nn.MaxPool2d(3, 2, 1), nn.Conv2d(64, 64, 5, 2, 2), nn.ReLU(),
                                 nn.Conv2d(64, 160, 1, 2), *_head(160)),
                     (1, 3, 19, 23), ()),
    "stem4-k8s8p0": ("4-channel column-path stem 8x8/8/0 (K padded to 256, the unfold table's limit); max-pool 2/3/0 (k < stride) "
                     "into a tensor-core conv",
                     lambda: nn.Sequential(nn.Conv2d(4, 64, 8, 8), nn.ReLU(), nn.MaxPool2d(2, 3, 0), nn.Conv2d(64, 64, 3, 1, 1), nn.ReLU(),
                                 nn.Flatten(), nn.Linear(64 * 3 * 3, CLASSES)),
                     (2, 4, 72, 64), ()),
    "stem3-k2s3p0-ties": ("column-path stem 2x2/3/0 (stride > R: pixels no tap reaches); BN with a strongly negative shift, so the "
                          "overlapping padded max-pool 3/1/1 sees tied all-zero windows, read by a tensor-core and an fp32 conv",
                          TwoBranch, (2, 3, 16, 17), ()),
    "cand-co32": ("candidate-fed conv with 32 outputs (off the column path, NCHW operand strides) at batch 3; 3x3/3/0 conv; "
                  "max-pool 5/2/2; AdaptiveAvgPool -> Linear -> ReLU -> Linear without bias",
                  lambda: nn.Sequential(nn.Conv2d(3, 32, 3, 1, 1), nn.ReLU(), nn.Conv2d(32, 32, 3, 3), nn.ReLU(), nn.MaxPool2d(5, 2, 2),
                              nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(32, 16), nn.ReLU(), nn.Linear(16, CLASSES, bias=False)),
                  (3, 3, 15, 13), ()),
    "cand-co96": ("4-channel candidate-fed conv 3x3/2/1 with 96 outputs (off the column path); 96-wide 4x4/4/0 conv",
                  lambda: nn.Sequential(nn.Conv2d(4, 96, 3, 2, 1), bn(96), nn.ReLU(), nn.Conv2d(96, 64, 4, 4), nn.ReLU(), nn.Flatten(),
                              nn.Linear(64 * 2 * 2, CLASSES)),
                  (2, 4, 18, 18), ()),
    "cand-k11s4": ("AlexNet's 11x11/4/2 stem (R * S > 64: off the column path); tensor-core 3x3/4/1 conv (stride-4 dgrad)",
                   lambda: nn.Sequential(nn.Conv2d(3, 64, 11, 4, 2), nn.ReLU(), nn.Conv2d(64, 64, 3, 4, 1), nn.ReLU(), nn.Flatten(),
                               nn.Linear(64 * 3 * 2, CLASSES)),
                   (2, 3, 41, 37), ()),
    "widths-b17": ("batch 17 (the head leaves the small-linear kernel): 48-wide candidate-fed conv, max-pool 3/3/0, 4x4/2/1 conv "
                   "48 -> 96, two-layer head",
                   lambda: nn.Sequential(nn.Conv2d(3, 48, 3, 1, 1), nn.ReLU(), nn.MaxPool2d(3, 3, 0), nn.Conv2d(48, 96, 4, 2, 1), nn.ReLU(),
                               nn.Conv2d(96, 64, 1), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(64, 32), nn.ReLU(),
                               nn.Linear(32, CLASSES, bias=False)),
                   (17, 3, 12, 12), ()),
    "scalar-ties-b1": ("6 and 10 channels (scalar kernels) at batch 1: BN with a strongly negative shift, max-pool 3/2/1 of tied "
                       "zero windows into an fp32 conv, max-pool 2/2/0, linear on a 10-channel map",
                       lambda: nn.Sequential(nn.Conv2d(3, 6, 3, 1, 1), bn(6), nn.ReLU(), nn.MaxPool2d(3, 2, 1), nn.Conv2d(6, 10, 3, 2, 1), nn.ReLU(),
                                   nn.MaxPool2d(2, 2, 0), nn.Flatten(), nn.Linear(10 * 2 * 1, CLASSES)),
                       (1, 3, 13, 11), ()),
    "cifar-b64": ("a CIFAR-sized batch of 64: column-path stem, max-pool 3/3/0, 4x4/2/1 and 3x3/2/1 convs (5 x 5: unequal parity "
                  "classes)",
                  lambda: nn.Sequential(nn.Conv2d(3, 64, 3, 1, 1), bn(64), nn.ReLU(), nn.MaxPool2d(3, 3, 0), nn.Conv2d(64, 128, 4, 2, 1), bn(128),
                              nn.ReLU(), nn.Conv2d(128, 64, 3, 2, 1), *_head(64)),
                  (64, 3, 32, 32), ()),
    "trainbn": ("train-mode BN on 64 (float4) and 6 (scalar) channels; tensor-core 3x3/3/1 conv (stride-3 dgrad)",
                lambda: nn.Sequential(nn.Conv2d(3, 64, 3, 1, 1), bn(64, True), nn.ReLU(), nn.Conv2d(64, 64, 3, 3, 1), bn(64, True), nn.ReLU(),
                            nn.Conv2d(64, 6, 3, 2, 1), bn(6, True), nn.ReLU(), nn.Flatten(), nn.Linear(6 * 3 * 3, CLASSES)),
                (3, 3, 16, 16), ()),
    "precise-first": ("the stem1-k3s1p0 network with its first layer on the fp32 kernels (precise_first = 1): the 1-channel stem "
                      "leaves the column path",
                      _stem1, (2, 1, 17, 15), (("precise_first", 1),)),
}

MULTISTEP = ["stem2-k4s4p0", "cand-k11s4", "stem3-k2s3p0-ties"]   # checked through 2 FedAvg local steps as well


def build(name, seed=11):
    """(model in eval mode with random BN, input shape, labels, target gradients, engine options)."""
    _, factory, shape, options = CASES[name]
    torch.manual_seed(seed)
    model = factory().eval()
    gen = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():   # non-trivial BN parameters and running statistics (synthetic.randomize_bn, also for train-mode BN)
        for m in model.modules():
            if isinstance(m, nn.BatchNorm2d):
                m.weight.copy_(1.0 + 0.2 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=gen))
                if "ties" in name:   # the other channels are shifted by -0.5: partly tied windows
                    m.bias[0::2], m.bias[1::2] = TIE_BETA, -0.5
                if m.running_mean is not None:
                    m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=gen))
                    m.running_var.copy_(1.0 + 0.3 * torch.rand(m.running_var.shape, generator=gen))
    gen = torch.Generator().manual_seed(seed + 7)
    x = torch.randn(shape, generator=gen)
    y = torch.randint(0, CLASSES, (shape[0],), generator=gen)
    grads = torch.autograd.grad(nn.functional.cross_entropy(model(x), y), list(model.parameters()))
    return model, shape, y, [g.detach() for g in grads], options


# ---- restated engine rules ---------------------------------------------------------------------------------------------------
def stem_columns(prog, i, backend, options=()):
    """csrc/engine.cu: the candidate-fed convolution runs on the column path (stem_cols.cu) on the tensor-core back end when the
    candidate has at most 4 channels, Co % 64 == 0 and R * S <= 64, unless precise_first keeps it on the fp32 kernels."""
    op, t = prog.ops[i], prog.tensors
    if backend != "tc" or op.kind != C.OP_CONV or op.tin != 0 or dict(options).get("precise_first", 0) > 0:
        return False
    return t[0].C <= 4 and t[op.tout].C % 64 == 0 and op.R * op.S <= 64


def gemm_geom(prog, op):
    """(N, H, W, Ci, Co, R, stride, pad) of a conv / linear op as the engine hands it to the GEMM planner."""
    ti, to = prog.tensors[op.tin], prog.tensors[op.tout]
    if op.kind == C.OP_LINEAR:
        return (ti.N, 1, 1, ti.C * ti.H * ti.W, to.C, 1, 1, 0)
    return (ti.N, ti.H, ti.W, ti.C, to.C, op.R, op.stride, op.pad)


def gemm_plans(prog, backend, options=()):
    """{(op, mode, nsrc): (planner backend, geometry, plan)} by scripts/profile_gemms.gemm_plan for every GEMM of the program, with the
    planner backend the engine passes (2 on the tensor-core back end, 0 on the SIMT back end and for layers kept precise).  On the
    column path the candidate-fed conv's GEMMs are 1x1 convolutions over the unfolded candidate [N, Ho, Wo, Kp] (one source each);
    off it the candidate's NCHW strides keep it off the tensor cores, and its geometry is listed with backend 0 under ``nchw``."""
    from profile_gemms import gemm_plan

    precise = dict(options).get("precise_first", 0)
    gemms = [i for i, op in enumerate(prog.ops) if op.kind in (C.OP_CONV, C.OP_LINEAR)]
    out = {}
    for rank, i in enumerate(gemms):
        op = prog.ops[i]
        be, g, srcs = (2 if backend == "tc" and rank >= precise else 0), gemm_geom(prog, op), (1, 2)
        if op.kind == C.OP_CONV and op.tin == 0:
            if stem_columns(prog, i, backend, options):
                to = prog.tensors[op.tout]
                g, srcs = (to.N, to.H, to.W, -(-op.R * op.S * prog.tensors[0].C // 64) * 64, to.C, 1, 1, 0), (1,)
            else:
                be = "nchw"
        for mode in range(3):
            for nsrc in srcs:
                out[(i, mode, nsrc)] = (be, g, gemm_plan(mode, g, nsrc, 0 if be == "nchw" else be))
    return out


def _parity_classes(H, pad):
    return sorted({len(range((e - pad) % 2, H, 2)) for e in range(2)})


def reached(name, backend):
    """The rules of ``REQUIRED`` that case ``name`` takes on ``backend`` ("simt" / "tc")."""
    _, factory, shape, options = CASES[name]
    model, *_ = build(name)
    prog = C.compile_model(model, shape)
    ops, t = prog.ops, prog.tensors
    out = {("batch", shape[0]) if shape[0] in (1, 3, 17) else ("batch", "cifar") if 64 <= shape[0] <= 100 else ("batch", "other")}
    producer = {op.tout: op for op in ops}
    bn_mods = C.bn_modules(model, prog)
    for i, op in enumerate(ops):
        ti, to = t[op.tin], t[op.tout]
        if op.kind == C.OP_CONV and op.tin == 0:
            if stem_columns(prog, i, backend, options):
                out |= {("stem", "C", ti.C), ("stem", "geom", op.R, op.stride, op.pad), ("stem", "Co", to.C)}
                if ti.H % 2 and ti.W % 2:
                    out.add(("stem", "odd"))
                if op.R * op.S * ti.C == 256:
                    out.add(("stem", "K256"))
            elif backend == "tc" and dict(options).get("precise_first", 0) == 0:
                out.add(("candidate-fed off the columns", "R*S>64" if op.R * op.S > 64 else f"Co={to.C}"))
        elif op.kind == C.OP_CONV:
            if op.stride == 2:
                out.add(("inner s2", "R", op.R))
                if len(_parity_classes(ti.H, op.pad)) > 1 or len(_parity_classes(ti.W, op.pad)) > 1:
                    out.add(("inner s2", "unequal parity classes"))
            if op.stride in (3, 4):
                out.add(("inner stride", op.stride))
            if op.pad == 0 and op.R > 1:
                out.add(("inner pad", 0))
            if 2 * op.pad > op.R:
                out.add(("inner pad", "> R/2"))
            for w in (ti.C, to.C):
                if w in (32, 48, 96, 160):
                    out.add(("inner width", w))
        elif op.kind == C.OP_MAXPOOL:
            out |= {("maxpool", op.R, op.stride, op.pad), ("maxpool", "C%4==0", ti.C % 4 == 0)}
            src = producer.get(op.tin)
            if src is not None and src.kind == C.OP_BNACT and src.has_bn and src.relu and \
                    float(model.get_submodule(src.bn_module).bias.detach().min()) <= TIE_BETA:
                out.add(("maxpool", "tied zero windows"))
        elif op.kind == C.OP_LINEAR:
            if ti.H * ti.W > 1 and ti.C % 4:
                out.add(("head", "linear on a spatial map, C % 4 != 0"))
            src = producer.get(op.tin)
            if op.b < 0 and src is not None and src.kind == C.OP_BNACT and src.relu and not src.has_bn and \
                    producer.get(src.tin) is not None and producer[src.tin].kind == C.OP_LINEAR and \
                    producer[producer[src.tin].tin].kind == C.OP_AVGPOOL:
                out.add(("head", "avgpool-linear-relu-linear(bias=False)"))
        elif op.kind == C.OP_BNACT and op.has_bn and op.bn_train:
            out.add(("train-mode BN", "C%4==0", to.C % 4 == 0))
    if dict(options).get("precise_first", 0):
        out.add(("option", "precise_first"))
    pooled = {i for i, op in enumerate(ops) if op.tin in {o.tout for o in ops if o.kind == C.OP_MAXPOOL}}
    for (i, mode, nsrc), (be, g, p) in gemm_plans(prog, backend, options).items():
        out.add(("family", p["family"]))
        if p["family"] == "tc":
            out |= {("tc producer", p["producer"]), ("tc tile", p["tile_rows"], p["tile_width"])}
            if p["splits"] > 1:
                out.add(("tc split-K",))
        if i in pooled:
            out.add(("maxpool feeds", "tc" if p["family"] == "tc" and mode == 0 else "simt"))
    return out


REQUIRED = (
    {("stem", "C", c) for c in (1, 2, 3, 4)} | {("stem", "geom", *g) for g in ((3, 1, 0), (4, 4, 0), (5, 2, 2), (8, 8, 0), (2, 3, 0))}
    | {("stem", "Co", 64), ("stem", "Co", 128), ("stem", "odd"), ("stem", "K256")}
    | {("candidate-fed off the columns", k) for k in ("Co=32", "Co=96", "R*S>64")}
    | {("inner s2", "R", r) for r in (1, 2, 3, 4, 5)} | {("inner s2", "unequal parity classes"), ("inner stride", 3), ("inner stride", 4)}
    | {("inner pad", 0), ("inner pad", "> R/2")} | {("inner width", w) for w in (32, 48, 96, 160)}
    | {("maxpool", *g) for g in ((2, 2, 0), (3, 3, 0), (3, 2, 1), (3, 1, 1), (2, 3, 0), (5, 2, 2))}
    | {("maxpool", "C%4==0", True), ("maxpool", "C%4==0", False), ("maxpool", "tied zero windows"), ("maxpool feeds", "tc"),
       ("maxpool feeds", "simt")}
    | {("head", "avgpool-linear-relu-linear(bias=False)"), ("head", "linear on a spatial map, C % 4 != 0")}
    | {("batch", b) for b in (1, 3, 17, "cifar")}
    | {("train-mode BN", "C%4==0", True), ("train-mode BN", "C%4==0", False), ("option", "precise_first")}
    | {("family", f) for f in ("igemm_simt", "dgrad_small_ci", "linear_small", "tc")}
    | {("tc producer", p) for p in ("tma", "cp.async", "classes")} | {("tc tile", 128, 64), ("tc tile", 128, 32), ("tc tile", 64, 64)}
    | {("tc split-K",)}
)
