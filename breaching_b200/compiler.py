"""Lower an ``nn.Module`` to the static layer program the sm_90a engine executes.

The reference runs the attacked model through the PyTorch autograd engine twice per iteration
(``attacks/auxiliaries/objectives.py:40-46`` forward + ``autograd.grad(create_graph=True)``,
``attacks/optimization_based_attack.py:165`` second backward).  The engine instead executes four
sweeps of one static program (forward, backward, tangent-forward, tangent-backward; DESIGN.md section 3),
so the model has to be known as a list of typed layer records with explicit tensor ids.

Supported graph vocabulary (everything the BASELINE vision configs need -- torchvision ResNet
BasicBlock/Bottleneck nets and the reference's ConvNet/ConvNetSmall, SURVEY.md appendix C):

    Conv2d (groups=1, dilation=1, zeros padding) . BatchNorm2d (eval mode) . ReLU . residual add
    MaxPool2d . AdaptiveAvgPool2d(1) . Flatten . Linear . Identity/Dropout(p=0)

Anything else raises :class:`UnsupportedModelError` -- there is deliberately no eager/CPU fallback.
"""
import operator
from dataclasses import dataclass, field
from typing import List, Optional

import torch
import torch.fx

OP_CONV, OP_BNACT, OP_MAXPOOL, OP_AVGPOOL, OP_LINEAR = 1, 2, 3, 4, 5
# token-sequence models (the TAG / transformer path, SURVEY section 8 rows a15 / a16): tensors are [rows = batch x seq_len, C, 1, 1]
OP_POSADD, OP_LAYERNORM, OP_ATTENTION = 6, 7, 8
OP_POSCONST = 9   # + a constant positional table (the fixed sinusoidal positions): no parameter, ``Op.table`` [seq_len, C]
OP_NAMES = {OP_CONV: "conv", OP_BNACT: "bnact", OP_MAXPOOL: "maxpool", OP_AVGPOOL: "avgpool", OP_LINEAR: "linear",
            OP_POSADD: "posadd", OP_LAYERNORM: "layernorm", OP_ATTENTION: "attention", OP_POSCONST: "posconst"}

# how a parameter tensor is laid out in the engine arena relative to torch's layout
PERM_NONE, PERM_OIHW_TO_OHWI, PERM_LINEAR_CHW_TO_HWC = 0, 1, 2


class UnsupportedModelError(RuntimeError):
    pass


@dataclass
class TensorDesc:
    tid: int
    N: int
    C: int
    H: int
    W: int

    @property
    def numel(self):
        return self.N * self.C * self.H * self.W


@dataclass
class ParamDesc:
    index: int  # position in model.parameters()
    shape: tuple
    perm: int = PERM_NONE
    perm_c: int = 0  # for PERM_LINEAR_CHW_TO_HWC: (C, H*W) of the flattened feature map
    perm_hw: int = 0
    alloc_numel: int = 0  # > numel: the engine reserves this many elements (zero tail), e.g. rows of a padded vocabulary

    @property
    def numel(self):
        n = 1
        for s in self.shape:
            n *= s
        return n


@dataclass
class Op:
    kind: int
    tin: int
    tout: int
    # conv / linear / pool geometry
    R: int = 1
    S: int = 1
    stride: int = 1
    pad: int = 0
    w: int = -1  # parameter indices (model.parameters() order), -1 = absent
    b: int = -1
    # bnact
    has_bn: bool = False
    bn_train: bool = False      # BN normalises with the batch statistics of its input (train mode without buffers)
    relu: bool = False
    res: int = -1  # residual tensor id
    gamma: int = -1
    beta: int = -1
    eps: float = 1e-5
    bn_module: Optional[str] = None  # qualified module name (running stats are read from it)
    module: Optional[str] = None     # linear: qualified module name
    table: Optional[torch.Tensor] = None   # posconst: the float32 table the op adds, a copy of the model's buffer
    # gradient accumulation flags for the reverse sweeps (set by finalize())
    acc_in: bool = False
    acc_res: bool = False


@dataclass
class Program:
    tensors: List[TensorDesc] = field(default_factory=list)
    ops: List[Op] = field(default_factory=list)
    params: List[ParamDesc] = field(default_factory=list)
    logits: int = -1  # tensor id of the network output
    num_classes: int = 0
    seq_len: int = 0  # > 0: token-sequence program (rows = batch * seq_len), causal next-token loss over rows
    logits_valid: int = 0  # > 0: number of real classes when the logits tensor is padded to the GEMM tile width
    # the layers the reference's priors single out by module *registration* order (regularizers.py): the BN op of the first
    # registered BatchNorm2d (DeepInversion's first_bn_multiplier) and the op of the last registered Linear (the features prior);
    # -1 where the program has none or does not record it
    di_first_op: int = -1
    feature_op: int = -1

    def describe(self):
        lines = []
        for op in self.ops:
            ti, to = self.tensors[op.tin], self.tensors[op.tout]
            extra = ""
            if op.kind == OP_CONV:
                extra = f" {op.R}x{op.S}/s{op.stride}/p{op.pad} w={op.w} b={op.b}"
            elif op.kind == OP_BNACT:
                extra = f" bn={op.has_bn} relu={op.relu} res={op.res}"
            elif op.kind == OP_MAXPOOL:
                extra = f" k{op.R}/s{op.stride}/p{op.pad}"
            lines.append(
                f"{OP_NAMES[op.kind]:8s} t{op.tin}[{ti.N},{ti.C},{ti.H},{ti.W}] -> t{op.tout}[{to.N},{to.C},{to.H},{to.W}]{extra}"
            )
        return "\n".join(lines)


def _pair(v):
    if isinstance(v, (tuple, list)):
        if len(v) != 2 or v[0] != v[1]:
            raise UnsupportedModelError(f"non-square geometry {v} is not supported")
        return int(v[0])
    return int(v)


class _Tracer(torch.fx.Tracer):
    """Treat every leaf layer type we know as a leaf (default behaviour) and trace through containers."""

    def is_leaf_module(self, m, qualname):
        return m.__module__.startswith("torch.nn") and not isinstance(m, torch.nn.Sequential)


def _trace(model):
    try:
        graph = _Tracer().trace(model)
    except Exception as exc:  # noqa: BLE001
        raise UnsupportedModelError(f"model could not be traced into a static layer program: {exc}") from exc
    return graph


def _check_flatten_args(node, first):
    """``flatten(x, 1)`` / ``x.flatten(1)`` (optionally ``end_dim=-1``) is the only flatten the layer program can express."""
    args = list(node.args[first:])
    start = args[0] if len(args) > 0 else node.kwargs.get("start_dim", 0)
    end = args[1] if len(args) > 1 else node.kwargs.get("end_dim", -1)
    if start != 1 or end not in (-1, 3):
        raise UnsupportedModelError(f"{node.name}: only flatten(start_dim=1, end_dim=-1) is supported (got {start}, {end})")


def _check_view_args(node, ti):
    """``x.view(N, -1)`` / ``x.view(x.size(0), -1)`` / ``x.reshape(N, features)``: anything else would silently be mis-lowered."""
    shape = node.args[1:]
    if len(shape) == 1 and isinstance(shape[0], (tuple, list)):
        shape = tuple(shape[0])
    if len(shape) != 2:
        raise UnsupportedModelError(f"{node.name}: only a reshape to [N, -1] is supported")
    n, f = shape
    ok_n = isinstance(n, torch.fx.Node) or n in (ti.N, -1)
    ok_f = isinstance(f, torch.fx.Node) or f in (-1, ti.C * ti.H * ti.W)
    if not (ok_n and ok_f) or (n == -1 and f == -1):
        raise UnsupportedModelError(f"{node.name}: reshape to {shape} is not [N, -1]")


def compile_model(model, input_shape):
    """Return the :class:`Program` for ``model`` applied to a batch of shape ``input_shape`` (N, C, H, W)."""
    N, C0, H0, W0 = [int(s) for s in input_shape]
    graph = _trace(model)
    modules = dict(model.named_modules())
    param_index = {id(p): i for i, p in enumerate(model.parameters())}

    prog = Program()
    prog.tensors.append(TensorDesc(0, N, C0, H0, W0))
    prog.params = [ParamDesc(i, tuple(p.shape)) for i, p in enumerate(model.parameters())]

    # --- pass 1: primitive ops -----------------------------------------------------------------
    prim = []  # dicts: kind, in(s), out, attrs
    env = {}  # fx node -> tensor id
    flat_of = {}  # tensor id -> tensor id it is a flattened view of

    def new_tensor(n, c, h, w):
        t = TensorDesc(len(prog.tensors), n, c, h, w)
        prog.tensors.append(t)
        return t.tid

    def pidx(p):
        return -1 if p is None else param_index[id(p)]

    seen_input = False
    out_tid = None
    for node in graph.nodes:
        if node.op == "placeholder":
            if not seen_input:
                env[node] = 0
                seen_input = True
            continue  # extra (**kwargs) placeholders are ignored
        if node.op == "output":
            res = node.args[0]
            if isinstance(res, (tuple, list, dict)):
                raise UnsupportedModelError("model must return a single logits tensor")
            out_tid = env[res]
            continue
        if node.op == "get_attr":
            raise UnsupportedModelError(f"free tensor attribute {node.target} in forward is not supported")

        def arg_tid(a):
            if a not in env:
                raise UnsupportedModelError(f"cannot resolve input of node {node.name}")
            return env[a]

        if node.op == "call_module":
            mod = modules[node.target]
            tin = arg_tid(node.args[0])
            ti = prog.tensors[tin]
            if isinstance(mod, torch.nn.Conv2d):
                if mod.groups != 1 or _pair(mod.dilation) != 1 or mod.padding_mode != "zeros" or isinstance(mod.padding, str):
                    raise UnsupportedModelError(f"conv {node.target}: groups/dilation/padding mode unsupported")
                R, S = mod.kernel_size
                if R != S:
                    raise UnsupportedModelError("non-square kernels unsupported")
                st, pd = _pair(mod.stride), _pair(mod.padding)
                Ho = (ti.H + 2 * pd - R) // st + 1
                Wo = (ti.W + 2 * pd - S) // st + 1
                tout = new_tensor(ti.N, mod.out_channels, Ho, Wo)
                prim.append(dict(kind="conv", tin=tin, tout=tout, R=R, S=S, stride=st, pad=pd,
                                 w=pidx(mod.weight), b=pidx(mod.bias)))
                prog.params[pidx(mod.weight)].perm = PERM_OIHW_TO_OHWI
                env[node] = tout
            elif isinstance(mod, torch.nn.BatchNorm2d):
                if mod.weight is None:
                    raise UnsupportedModelError("BatchNorm without affine parameters unsupported")
                tout = new_tensor(ti.N, ti.C, ti.H, ti.W)
                # train mode (no server / user buffers: base_attack.py:192-197 puts the model in .train() with
                # track_running_stats = False): normalisation by the statistics of the candidate batch itself
                prim.append(dict(kind="bn", tin=tin, tout=tout, gamma=pidx(mod.weight), beta=pidx(mod.bias),
                                 eps=float(mod.eps), module=node.target, train=bool(mod.training or mod.running_mean is None)))
                env[node] = tout
            elif isinstance(mod, torch.nn.ReLU):
                tout = new_tensor(ti.N, ti.C, ti.H, ti.W)
                prim.append(dict(kind="relu", tin=tin, tout=tout))
                env[node] = tout
            elif isinstance(mod, torch.nn.MaxPool2d):
                k, st, pd = _pair(mod.kernel_size), _pair(mod.stride), _pair(mod.padding)
                if _pair(mod.dilation) != 1 or mod.ceil_mode:
                    raise UnsupportedModelError("maxpool dilation/ceil_mode unsupported")
                Ho = (ti.H + 2 * pd - k) // st + 1
                Wo = (ti.W + 2 * pd - k) // st + 1
                tout = new_tensor(ti.N, ti.C, Ho, Wo)
                prim.append(dict(kind="maxpool", tin=tin, tout=tout, R=k, stride=st, pad=pd))
                env[node] = tout
            elif isinstance(mod, torch.nn.AdaptiveAvgPool2d):
                osz = mod.output_size
                if osz not in (1, (1, 1)):
                    raise UnsupportedModelError("only AdaptiveAvgPool2d(1) supported")
                tout = new_tensor(ti.N, ti.C, 1, 1)
                prim.append(dict(kind="avgpool", tin=tin, tout=tout))
                env[node] = tout
            elif isinstance(mod, torch.nn.Flatten):
                if mod.start_dim != 1 or mod.end_dim not in (-1, 3):
                    raise UnsupportedModelError(f"Flatten({mod.start_dim}, {mod.end_dim}) is not [N, -1]")
                env[node] = tin  # layout handled by the consuming Linear
            elif isinstance(mod, (torch.nn.Identity,)) or (isinstance(mod, torch.nn.Dropout) and (mod.p == 0 or not mod.training)):
                env[node] = tin
            elif isinstance(mod, torch.nn.Linear):
                feat = ti.C * ti.H * ti.W
                if feat != mod.in_features:
                    raise UnsupportedModelError(f"linear {node.target}: {feat} features arrive, {mod.in_features} expected")
                tout = new_tensor(ti.N, mod.out_features, 1, 1)
                prim.append(dict(kind="linear", tin=tin, tout=tout, w=pidx(mod.weight), b=pidx(mod.bias), module=node.target))
                if ti.H * ti.W > 1 and tin != 0:
                    # internal activations are NHWC: permute the weight columns once.  The candidate itself (tensor 0) stays
                    # NCHW, so a Linear fed directly by it (the reference's `linear` model, model_preparation.py:238,313)
                    # keeps torch's CHW column order.
                    pd_ = prog.params[pidx(mod.weight)]
                    pd_.perm, pd_.perm_c, pd_.perm_hw = PERM_LINEAR_CHW_TO_HWC, ti.C, ti.H * ti.W
                env[node] = tout
            else:
                raise UnsupportedModelError(f"layer type {type(mod).__name__} ({node.target}) is not supported by the engine")
        elif node.op == "call_function":
            fn = node.target
            if fn in (operator.add, torch.add, operator.iadd):
                a, b = node.args[0], node.args[1]
                if not (isinstance(a, torch.fx.Node) and isinstance(b, torch.fx.Node)):
                    raise UnsupportedModelError("add with a constant unsupported")
                ta, tb = arg_tid(a), arg_tid(b)
                A = prog.tensors[ta]
                tout = new_tensor(A.N, A.C, A.H, A.W)
                prim.append(dict(kind="add", tin=ta, tin2=tb, tout=tout))
                env[node] = tout
            elif fn is torch.flatten:
                _check_flatten_args(node, 1)
                env[node] = arg_tid(node.args[0])
            elif fn in (torch.relu, torch.nn.functional.relu):
                tin = arg_tid(node.args[0])
                ti = prog.tensors[tin]
                tout = new_tensor(ti.N, ti.C, ti.H, ti.W)
                prim.append(dict(kind="relu", tin=tin, tout=tout))
                env[node] = tout
            else:
                raise UnsupportedModelError(f"function {getattr(fn, '__name__', fn)} is not supported by the engine")
        elif node.op == "call_method":
            if node.target in ("flatten", "view", "reshape", "contiguous"):
                if node.target == "flatten":
                    _check_flatten_args(node, 1)
                elif node.target in ("view", "reshape"):
                    _check_view_args(node, prog.tensors[arg_tid(node.args[0])])
                env[node] = arg_tid(node.args[0])
            elif node.target == "size":
                pass  # x.size(0) as an argument of view / reshape (checked there)
            else:
                raise UnsupportedModelError(f"tensor method {node.target} is not supported by the engine")
    if out_tid is None:
        raise UnsupportedModelError("no output found")

    # --- pass 2: fuse bn / add / relu chains into BNACT ----------------------------------------
    consumers = {}
    for p in prim:
        for key in ("tin", "tin2"):
            if key in p:
                consumers.setdefault(p[key], []).append(p)
    consumers.setdefault(out_tid, []).append(None)

    used = set()

    def single_next(t, kind):
        cs = consumers.get(t, [])
        if len(cs) == 1 and cs[0] is not None and cs[0]["kind"] == kind and id(cs[0]) not in used:
            return cs[0]
        return None

    order = {id(p): i for i, p in enumerate(prim)}
    keyed = []  # (position of the last fused primitive, op)
    for p in prim:
        if id(p) in used:
            continue
        k = p["kind"]
        last = p
        if k == "conv":
            op = Op(OP_CONV, p["tin"], p["tout"], R=p["R"], S=p["S"], stride=p["stride"], pad=p["pad"], w=p["w"], b=p["b"])
        elif k == "linear":
            op = Op(OP_LINEAR, p["tin"], p["tout"], w=p["w"], b=p["b"], module=p["module"])
        elif k == "maxpool":
            op = Op(OP_MAXPOOL, p["tin"], p["tout"], R=p["R"], S=p["R"], stride=p["stride"], pad=p["pad"])
        elif k == "avgpool":
            op = Op(OP_AVGPOOL, p["tin"], p["tout"])
        elif k in ("bn", "add", "relu"):
            op = Op(OP_BNACT, p["tin"], p["tout"])
            cur = p
            if cur["kind"] == "bn":
                op.has_bn, op.gamma, op.beta, op.eps, op.bn_module = True, cur["gamma"], cur["beta"], cur["eps"], cur["module"]
                op.bn_train = cur.get("train", False)
                nxt = single_next(cur["tout"], "add")
                if nxt is not None:
                    used.add(id(nxt))
                    op.res = nxt["tin2"] if nxt["tin"] == cur["tout"] else nxt["tin"]
                    cur = nxt
            elif cur["kind"] == "add":
                op.res = cur["tin2"]
            if cur["kind"] != "relu":
                nxt = single_next(cur["tout"], "relu")
                if nxt is not None:
                    used.add(id(nxt))
                    cur = nxt
            op.relu = cur["kind"] == "relu"
            op.tout = cur["tout"]
            last = cur
        else:
            raise AssertionError(k)
        used.add(id(p))
        keyed.append((order[id(last)], len(keyed), op))
    prog.ops = [op for _, _, op in sorted(keyed, key=lambda t: (t[0], t[1]))]

    # the residual operand of a fused BN+add must already exist when the op runs (true for ResNets);
    # ops are emitted in fx (topological) order keyed on their first primitive, so verify.
    produced = {0}
    for op in prog.ops:
        for t in (op.tin, op.res):
            if t >= 0 and t not in produced:
                raise UnsupportedModelError("residual operand is produced after its consumer; unsupported topology")
        produced.add(op.tout)

    prog.logits = out_tid
    lt = prog.tensors[out_tid]
    if lt.H * lt.W != 1:
        raise UnsupportedModelError("model output must be [N, classes]")
    prog.num_classes = lt.C

    # --- gradient-accumulation flags for the reverse sweeps --------------------------------------
    written = set()
    for op in reversed(prog.ops):
        op.acc_in = op.tin in written
        written.add(op.tin)
        if op.res >= 0:
            op.acc_res = op.res in written
            written.add(op.res)
    _registered_prior_layers(model, prog)
    _compact_tensors(prog)
    return prog


def _registered_prior_layers(model, prog):
    """``prog.di_first_op`` / ``prog.feature_op``: the op of the first BatchNorm2d and of the last Linear in ``model.modules()``
    order, which is the order the reference's DeepInversion and feature priors hook them in.  A network may register its modules
    in another order than it runs them; the engine refuses the priors on such a network (engine.Engine)."""
    rank, order = {}, {}
    for name, m in model.named_modules(remove_duplicate=False):   # a module registered under two names ranks where modules() lists it
        order[name] = rank.setdefault(id(m), len(rank))
    bn = [i for i, op in enumerate(prog.ops) if op.kind == OP_BNACT and op.has_bn]
    lin = [i for i, op in enumerate(prog.ops) if op.kind == OP_LINEAR]
    if bn:
        prog.di_first_op = min(bn, key=lambda i: (order[prog.ops[i].bn_module], i))
    if lin:
        prog.feature_op = max(lin, key=lambda i: (order[prog.ops[i].module], i))


def _compact_tensors(prog):
    """Drop tensor ids that no op references after fusion and renumber densely (tensor 0 stays the input)."""
    live = {0, prog.logits}
    for op in prog.ops:
        live.update(t for t in (op.tin, op.tout, op.res) if t >= 0)
    remap, tensors = {}, []
    for t in prog.tensors:
        if t.tid in live:
            remap[t.tid] = len(tensors)
            tensors.append(TensorDesc(len(tensors), t.N, t.C, t.H, t.W))
    for op in prog.ops:
        op.tin, op.tout = remap[op.tin], remap[op.tout]
        if op.res >= 0:
            op.res = remap[op.res]
    prog.logits = remap[prog.logits]
    prog.tensors = tensors


def bn_modules(model, prog):
    """Map each BNACT op with BN to its module (for running statistics)."""
    modules = dict(model.named_modules())
    return [modules[op.bn_module] if (op.kind == OP_BNACT and op.has_bn) else None for op in prog.ops]


def _fixed_positions(pos, T, d):
    """The table ``pe[0, :T]`` of a fixed positional module (a ``pe`` buffer [1, max_len, d], no parameters, dropout 0)."""
    pe = getattr(pos, "pe", None)
    if not isinstance(pe, torch.Tensor) or any(True for _ in pos.parameters()):
        raise UnsupportedModelError("pos_encoder must be a learnable embedding or a constant `pe` buffer without parameters")
    for m in pos.modules():
        if isinstance(m, torch.nn.Dropout) and m.p > 0:
            raise UnsupportedModelError(f"dropout p = {m.p} on the positional encoding is not lowered (the engine adds the table as it is)")
    if pe.dim() != 3 or pe.shape[0] != 1 or pe.shape[2] != d or pe.shape[1] < T:
        raise UnsupportedModelError(f"positional table of shape {tuple(pe.shape)} does not cover [1, {T}, {d}]")
    return pe[0, :T].detach().to(device="cpu", dtype=torch.float32).contiguous().clone()


def compile_transformer(model, batch, seq_len, pad_vocab=True):
    """Lower the reference's ``TransformerModel`` (cases/models/language_models.py:150-205) *as the attack runs it* -- token
    embedding bypassed, the candidate is the embedding sequence [batch, seq_len, d] (base_attack.py:76-128) -- to the layer
    program: positional embedding added, post-norm encoder layers (self-attention without mask, ReLU FFN), linear decoder.
    ``model`` needs ``pos_encoder``, ``transformer_encoder.layers`` and ``decoder`` (``synthetic.TransformerLM`` has the
    reference's attribute names).  A learnable ``pos_encoder.embedding`` (LearnablePositionalEmbedding) lowers to OP_POSADD; a
    ``pos_encoder`` with a ``pe`` buffer and no parameters (the fixed sinusoidal PositionalEmbedding, language_models.py:89-130)
    lowers to OP_POSCONST, which adds the model's own float32 values ``pe[0, :seq_len]``.  Parameter indices follow
    ``model.parameters()`` with the token embedding removed, i.e. the order of the shared gradient list after base_attack.py:88-95.

    The program is the contract between this lowering and the sweeps: ``csrc/engine.cu`` executes it on the GPU (token ops in
    ``csrc/tokens.cu``), ``oracle/program_interp.py`` on the CPU (float64-verified against autograd and the reference's TAG
    closure).
    """
    names = [n for n, _ in model.named_parameters() if n != "encoder.weight"]
    shapes = {n: tuple(p.shape) for n, p in model.named_parameters()}
    prog = Program(seq_len=int(seq_len))
    prog.params = [ParamDesc(i, shapes[n]) for i, n in enumerate(names)]
    pidx = {n: i for i, n in enumerate(names)}
    rows = int(batch) * int(seq_len)
    d = model.decoder.in_features

    def new_tensor(C):
        prog.tensors.append(TensorDesc(len(prog.tensors), rows, C, 1, 1))
        return len(prog.tensors) - 1

    enc = getattr(model, "encoder", None)
    if isinstance(enc, torch.nn.Embedding) and model.decoder.weight is enc.weight:
        raise UnsupportedModelError("tied token embedding and decoder weights (transformer3t) are not lowered: the attack's run-embedding "
                                    "prologue removes the gradient entry they share")
    x = new_tensor(d)   # tensor 0: the candidate embeddings
    cur = new_tensor(d)
    pos = model.pos_encoder
    if hasattr(pos, "embedding"):
        prog.ops.append(Op(OP_POSADD, x, cur, w=pidx["pos_encoder.embedding.weight"], S=int(seq_len)))
    else:
        prog.ops.append(Op(OP_POSCONST, x, cur, S=int(seq_len), table=_fixed_positions(pos, int(seq_len), d)))
    for li, layer in enumerate(model.transformer_encoder.layers):
        if getattr(layer, "norm_first", False) or not getattr(layer.self_attn, "batch_first", True):
            raise UnsupportedModelError("only post-norm, batch-first encoder layers (the reference's configuration) are lowered")
        pre = f"transformer_encoder.layers.{li}."
        heads = layer.self_attn.num_heads
        qkv = new_tensor(3 * d)
        prog.ops.append(Op(OP_LINEAR, cur, qkv, w=pidx[pre + "self_attn.in_proj_weight"], b=pidx[pre + "self_attn.in_proj_bias"]))
        att = new_tensor(d)
        prog.ops.append(Op(OP_ATTENTION, qkv, att, R=heads, S=int(seq_len)))
        proj = new_tensor(d)
        prog.ops.append(Op(OP_LINEAR, att, proj, w=pidx[pre + "self_attn.out_proj.weight"], b=pidx[pre + "self_attn.out_proj.bias"]))
        r1 = new_tensor(d)
        prog.ops.append(Op(OP_BNACT, proj, r1, res=cur))                       # residual add
        n1 = new_tensor(d)
        prog.ops.append(Op(OP_LAYERNORM, r1, n1, gamma=pidx[pre + "norm1.weight"], beta=pidx[pre + "norm1.bias"], eps=float(layer.norm1.eps)))
        f1 = new_tensor(layer.linear1.out_features)
        prog.ops.append(Op(OP_LINEAR, n1, f1, w=pidx[pre + "linear1.weight"], b=pidx[pre + "linear1.bias"]))
        hid = new_tensor(layer.linear1.out_features)
        prog.ops.append(Op(OP_BNACT, f1, hid, relu=True))
        f2 = new_tensor(d)
        prog.ops.append(Op(OP_LINEAR, hid, f2, w=pidx[pre + "linear2.weight"], b=pidx[pre + "linear2.bias"]))
        r2 = new_tensor(d)
        prog.ops.append(Op(OP_BNACT, f2, r2, res=n1))
        cur = new_tensor(d)
        prog.ops.append(Op(OP_LAYERNORM, r2, cur, gamma=pidx[pre + "norm2.weight"], beta=pidx[pre + "norm2.bias"], eps=float(layer.norm2.eps)))
    # the vocabulary is padded to the GEMM tile width (50 257 -> 50 304) so that the decoder -- the contraction that dominates this
    # model (SURVEY section 8 a15) -- runs on the tensor-core kernels: extra logit columns exist in the logits-shaped tensors only
    # (zero weight rows / bias entries, never read by the loss: ``logits_valid``); labels stay [rows, vocabulary]
    V = model.decoder.out_features
    Vp = ((V + 63) // 64) * 64 if pad_vocab else V
    logits = new_tensor(Vp)
    prog.ops.append(Op(OP_LINEAR, cur, logits, w=pidx["decoder.weight"], b=pidx["decoder.bias"]))
    prog.logits, prog.num_classes, prog.logits_valid = logits, V, V
    if Vp != V:
        prog.params[pidx["decoder.weight"]].alloc_numel = Vp * d
        if "decoder.bias" in pidx:
            prog.params[pidx["decoder.bias"]].alloc_numel = Vp
    written = set()
    for op in reversed(prog.ops):
        op.acc_in = op.tin in written
        written.add(op.tin)
        if op.res >= 0:
            op.acc_res = op.res in written
            written.add(op.res)
    return prog
