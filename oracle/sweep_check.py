"""Layer-local check of the engine's four sweeps.  TEST INFRASTRUCTURE ONLY.

The closure-level tests compare one number and one image-sized gradient at the end of some two hundred launches, so their
tolerances have to absorb the conditioning of the whole network.  This checker judges every kernel on its own: for every op
and every sweep it recomputes, in float64, *that op's output from the engine's own inputs to that op* (the rules of
``oracle/program_interp.py`` applied locally) and compares it element by element with what the engine stored, against a
rounding-error bound derived for that element:

  * GEMM outputs (conv / linear, one or two sources): ``(K + 2) 2^-23 (|A| * |B|)`` with ``|A| * |B|`` the same op on
    absolute values and K the reduction length (Higham's summation bound with 2u, which also covers accumulation that does
    not round to nearest).  The reference uses the operands the kernel read: activations and deltas as stored (the engine
    stores tensor-core operands on the TF32 grid), weights / direction in operand form (``W_operand`` / ``v_operand``),
    and the candidate and weights rounded to TF32 for an op whose kernel rounds them itself (the stem column path).
    TF32 x TF32 products are exact in fp32, so no TF32 term is needed.
  * element-wise ops: a few fp32 ulps of the magnitudes involved;
  * reductions (bias sums, BN gamma / beta gradients, pooling): ``(P + 4) 2^-23 sum |terms|``;
  * train-mode BN and the DeepInversion adjoints (composites of per-channel batch statistics and element-wise terms):
    ``TRAIN_C (P + 8) 2^-24`` times the magnitudes, with the conditioning of the variance / norm differences as a factor;
  * a tensor-core layer (weights read from the TF32 shadow) whose activation operand is stored off the TF32 grid has that
    operand truncated by the tensor core: its bound is widened by 2^-10 of the magnitudes and the op is listed in
    ``off_grid`` (this contradicts the intent of the engine's rounding flags; today: GEMMs fed by a max-pool, and linear
    layers fed by an average pool whose weight gradient runs on the tensor cores);
  * a stored tensor whose every element lies on the TF32 grid (13 low mantissa bits zero) was rounded on store: half a
    TF32 ulp of the reference (per accumulation for deltas summed over several consumers) is added.

Token programs (``compiler.compile_transformer``: tensors are [rows = B x T, C, 1, 1]):

  * ``posadd``: F and TF are one fp32 add / a copy (``2u`` of the magnitudes; the tangent is ``v_pos`` of row mod T exactly); the
    positional-table gradient of B is a sum over the B sequences, ``(B + 4) 2^-23 sum |terms|``, its rows >= T exactly zero; the
    delta passes to the candidate unchanged (task-loss gradient in B, candidate gradient in TB);
  * ``layernorm`` (statistics over the C features of a row): composite bounds as for train-mode BN, ``TRAIN_C (C + 8) 2^-24``
    times the magnitudes with the conditioning ``1 + mean(x^2) / var`` of the row as a factor; in those magnitudes ``xh`` counts
    as ``|xh| + inv (|x| + |mean|)`` (the error of ``x - mean``); gamma / beta gradients are sums over rows, ``(rows + 4) 2^-23``
    plus the composite term of ``xh``;
  * ``attention``, per (sequence, head), recomputed in float64 from the stored ``qkv`` (and its tangent, the output delta and
    tangent delta): a first-order running error bound.  Dot products over dh (scores) or T (P V, dS K, ...) cost
    ``(n + 2) 2^-23`` of their magnitudes; the softmax adds ``(T + 2) 2^-23 + 3u + u |S - max S|`` relative to P plus the
    P-weighted mean of the score errors; each product / difference one more ``u``; these errors are propagated through P V,
    dS K / Q and their tangents (the kernel's stored P / P' carry exactly these errors);
  * the next-token loss seed (sweep B) and its tangent (TB): row (b, t) is scored against the target row (b, t + 1) of the soft
    targets, each sequence's last row is exactly zero, the mean runs over ``M = rows - rows / T``; only the first
    ``logits_valid`` columns are real: the padded columns of the logits value, delta, tangent and tangent delta must be exactly
    zero (the decoder's tangent dgrad would read a nonzero one through v);
  * ``check_label_gradient``: d objective / d target probabilities, ``-(zdot - <p, zdot>) / M - tau (z - lse) / M`` of the
    source row (row (b, t - 1) for tokens, 0 at t = 0), bounded like the seeds.

The label leaf of a joint iteration (``check_label_leaf``; the row kernels ``row_softmax`` and ``softmax_chain``), and the row
kernels alone (``check_row_kernel``; every relation is a module function that ``SweepChecker`` uses as well):

  * row softmax ``q = softmax(l)``: the kernel takes the exact fp32 row max m, forms ``expf(l_c - m)`` (the argument rounded
    once, ``u |l_c - m|``, and CUDA's ``expf`` within 2 ulp, ``4u``), sums them -- on the register path in runs of four fp32
    adds folded into a double (``4u`` of the run), on the streamed path in double -- and merges the per-thread (m, s) pairs as
    ``s e^(m - M)`` over lanes, warps and CTAs: a partial is rescaled at most ``SOFTMAX_MERGES = 19`` times (5 lane steps, 7 warps,
    7 CTAs), each rescale one ``expf`` (``4u``) of a rounded difference (the differences along one chain add up to at most the
    row range ``R = max l - min l``, ``u R``).  So the sum carries ``e_S = (8 + 4 SOFTMAX_MERGES) u + u R`` relative, and
    ``q_c = expf(l_c - m) (1 / S)`` (the reciprocal rounded to fp32, the product rounded) is within
    ``q_c ((6 + |l_c - m|) u + e_S)`` plus ``2^-147`` for results that underflow to subnormals;
  * chain ``g <- q (g - <q, g>)`` on the engine's own fp32 q and un-chained g: the products are exact in double, the double
    sum costs ``n 2^-53 sum |q g|`` and its rounding to fp32 ``u |<q, g>|``; the difference and the product one ``u`` each:
    ``|q| (u |g - d| + u |d| + n 2^-53 sum |q g|) + u |ref|``, doubled;
  * the cross-entropy forward (vision ``ce_fwd`` with class indices or soft targets, token ``token_ce_fwd``): p by the softmax
    relation, the seed by the seed bound above, each row's loss by the per-row task-loss bound below (tokens: times
    ``rows / M`` through the fp32 ``1 / M``, ``2u`` more); the tangent seeds (``ce_tan_bwd``, ``token_ce_tan_bwd``, the
    labelled ``ce_tan_bwd_seed`` with ``coef (p - y) / N`` fused in) by the tangent-seed bound of sweep TB, evaluated on the
    p the kernel read; the label gradients (``ce_label_grad``, ``token_label_grad``) by the label-gradient bound.  Outputs
    stored on the TF32 grid add half a TF32 ulp.  Unscored token rows (each sequence's last row; every row when T = 1) and
    label-gradient rows at t = 0 must be exactly zero.

Multi-step (FedAvg) evaluations (``MultiStepChecker``; the engine's ``evaluate_multistep``, ``MultiStepInterpreter``): every
local step k is checked as a single step, with W_k as the parameters (the BN constants follow from it), step k's labels, the
direction u_{k+1} that step k used as ``v``, and no priors or task term in its candidate-gradient relation (that buffer is the
step's own input gradient).  In addition:

  * sweep ``TG`` (steps k > 0): the tangent parameter gradients ``H_k u_{k+1}``.  Conv / linear weights
    ``wgrad(a, d_T) + wgrad(a', d_B)`` (one source for the candidate-fed layer) with the GEMM bound ``(K_total + 2) 2^-23`` of
    ``|A| * |B|`` summed over both sources, on the operands the kernel read (stored values; the candidate rounded to TF32 on the
    stem column path; an off-grid activation or tangent of a tensor-core layer widened as for sweep B); biases ``sum d_T`` and the
    eval-mode BN tangents (gamma ``sum (du_T xh + du_B x' inv)``, beta ``sum du_T``, ``du`` the ReLU-masked deltas, ``x'`` the
    pre-BN tangent) with the reduction bound ``(P + 4) 2^-23 sum |terms|`` (2P terms for gamma);
  * the glue, each one rounding of an fp32 axpby with the step size the engine applied (its fp32 value):
    ``W_{k+1} = W_k - lr G_k``, ``D_{k+1} = D_k - lr G_k`` and the adjoint update ``u_k = u_{k+1} - lr TG_k``, each within
    ``2u (|a| + |lr b|)``; the TF32 operand forms of W_k and u_k equal ``rna`` of their fp32 values exactly (shadowed weights) or
    the values themselves; ``v = make_v(D_K, g)`` is the direction relation above with ``G := D_K``;
  * the final candidate gradient: ``sum_k -lr gradx_step_k`` scattered onto step k's slice (the slices of steps that wrap
    around the images accumulate), ``(n + 2) 2^-23 sum |terms|`` for n contributions to an element, plus the TV / norm priors on
    the whole candidate with the prior bound of the single-step relation.

``delta[t]`` / ``tangent_delta[t]`` are checked as the sum over *all* consumers of ``t`` (residual branches included), which
judges the accumulation flags; such a failure is reported at the consumer that runs last in the reverse sweep (the one with
the lowest op index), where the buffer becomes final.

The vision cross-entropy seed takes soft targets (a float ``labels`` tensor [N, classes]) as well as class indices.

Objective terms (``check_terms``; the six scalars of ``Engine.last_terms()`` and the returned objective).  Every term is
recomputed in float64 from the engine's own inputs to it (the stored G, the stored logits, the stored candidate / view, the
stored BN and feature inputs), with the configuration scalars at the fp32 values the kernels read; the bounds are first order:

  * ``match``: ``match_reduce_kernel`` forms the five sums dot = sum G g, nG = sum G^2, ng = sum g^2, sq = sum (G - g)^2 and
    l1w = sum w |G - g| (w: the tensor's tag-euclidean weight, 1 otherwise; masked-cosine drops every element with
    ``|g| <= float32(1e-6)`` from all five) over groups of 4 elements in fp32 before a double reduction, and rounds G - g once:
    each sum S_k is off by at most ``e_k = (4 2^-23 + n 2^-53) A_k`` (A_k = the sum of its |terms|; n terms in the double
    reduction), sq and l1w by ``2u A`` / ``u A`` more for the rounded difference.  ``finalize_objective`` in double: euclidean
    ``s sq / 2`` (bound ``|s| e_sq / 2``), l1 ``s l1w / 2``, tag-euclidean ``s (sq + t l1w) / 2``, the cosine kinds
    ``s (1 - c)`` with ``c = dot / sqrt(nG ng)``, ``|dc| <= e_dot / sqrt(nG ng) + |c| (e_nG / nG + e_ng / ng) / 2``, angular
    ``s acos(c) / pi`` with the chain factor ``1 / (pi sqrt(1 - c^2))`` (c clamped to the fudge interval; zero outside it);
  * ``task_loss``: the mean over rows of ``-sum_c q_c (z_c - lse)`` (q one-hot for class indices): per row the fp32 max,
    ``expf`` of the shifted logits summed in double, ``logf`` and a few roundings cost
    ``sum_c |q_c| ((16 + 2 rng) u + 4 u (|z_c - max| + |max| + |log sum|)) + 2 u |l_n|`` (rng = the row's logit range, as for
    the seeds), and the mean is rounded to fp32 (``u |L|``);
  * ``total_variation`` / ``norm``: per point the fp32 differences (exact for plain channels by Sterbenz up to one rounding;
    the double-opponent planes carry the rounding of their own difference), ``|d| + eps``, the powers and the sum
    ``(A^p + B^p)^q``; every power other than an exponent of 1 costs ``POW_C u`` relative (``POW_C = 8``: CUDA's ``powf`` is
    within 4 ulp; squares and square roots are within it), every add / subtract one ``u``; propagated to first order
    through p and q and summed with the double reduction's ``n 2^-53``; the norm ``s / p mean(x^p)`` costs ``POW_C u |x|^p``
    per element;
  * orthogonality (``obj["orthogonality"]``, ``orthogonality_relation``): ``(1/D) sum_k (S_k^2 - Q_k)`` from the fp32 batch sums
    S_k / Q_k of x^2 / x^4 at each of the D positions, added into the ``norm`` term; its candidate gradient
    ``(4/D) x_ik (S_k - x_ik^2)`` joins the candidate-gradient relation of sweep TB; 0 with fewer than two images;
  * ``deep_inversion``: per BN layer ``mult (||rv - var|| + ||rm - mean||)`` from the batch mean and biased variance of the
    stored BN input (``mult = float32(scale x first_bn_multiplier)`` at the first BN layer), with the bound of the fp32
    statistics used for the DeepInversion adjoint: ``|mult| TRAIN_C (M + 8) u (nm kap_m + nv kap_v)``;
  * ``features``: ``s mean((f - m)^2)`` from the stored input of the last linear layer, the difference rounded to fp32 and
    squared and summed in double: ``|s| (2u + n 2^-53) mean((f - m)^2)``;
  * the returned objective: exactly ``match + tv + norm + di + features (+ float32(tau) task_loss)``, summed in that order in
    double (``bre_engine_objective_and_gradient``).

``check_score(score, kind)``: ``Engine.score`` returns the fp32 rounding of the match term with scale 1 of the G it left
(``D`` for a multi-step engine), within the match bound plus ``u |match|``.

A buffer source provides ``tensor(which, tid)`` (``which`` in val / delta / tangent / tangent_delta, NCHW, ``None`` where a
tensor has no such buffer), ``param(which, index)`` (G / v_operand / W_operand, torch layout; multi-step steps also v and TG), ``unwritten`` (tensor ids whose
tangent is not stored because the BN op reading it ran in the producing GEMM's epilogue; that pair is then checked as one)
and ``rounds_operands(op_index)``.
"""
import torch
import torch.nn.functional as F

from breaching_b200 import compiler as C
from oracle.program_interp import objective_direction
from oracle import restate

U = 2.0 ** -24          # fp32 unit roundoff
U2 = 2.0 ** -23         # 2u per accumulation step
TF32_HALF = 2.0 ** -11  # half a TF32 ulp, relative
TINY = 1e-30
TRAIN_C = 8.0           # stated constant of the composite train-mode BN / DeepInversion bounds
POW_C = 8.0             # stated constant of one fp32 power (powf: 4 ulp), in units of u
D53 = 2.0 ** -53        # one double rounding
MASK_VALUE = float(torch.tensor(1e-6, dtype=torch.float32))   # masked-cosine threshold as the kernels compare it
SOFTMAX_MERGES = 19     # rescales of one (m, s) partial in the cluster softmax: 5 lane steps, 7 warps, 7 CTAs
SUBNORMAL = 2.0 ** -147  # absolute error of an fp32 result that underflows to a subnormal
TERMS = ("match", "task_loss", "total_variation", "norm", "deep_inversion", "features")


def f32(v):
    """The fp32 value of a configuration scalar, as the kernels read it."""
    return float(torch.tensor(float(v), dtype=torch.float32))


def tag_weights(L, scheme):
    """Per-tensor weights of tag-euclidean as the attack hands them to the engine (fp32; objectives.py:115-124)."""
    if scheme == "linear":
        return torch.arange(L, 0, -1, dtype=torch.float32) / L
    if scheme == "exp":
        w = torch.arange(L, 0, -1, dtype=torch.float32).softmax(dim=0)
        return w / w[0]
    return torch.ones(L)


def match_sums(G, g, kind, weights=None):
    """The five sums of ``match_reduce_kernel`` in float64 and their error bounds: ({dot, nG, ng, sq, l1w}, {same: bound})."""
    masked = kind == "masked-cosine-similarity"
    S = dict(dot=0.0, nG=0.0, ng=0.0, sq=0.0, l1w=0.0)
    A = dict(S)
    n = 0
    for j, (a, b) in enumerate(zip(G, g)):
        a, b = a.double().flatten(), b.double().flatten()
        if masked:
            keep = (b.to(torch.float32).abs() > MASK_VALUE).double()
            a, b = a * keep, b * keep
        w = 1.0 if weights is None else float(weights[j])
        d = a - b
        terms = dict(dot=a * b, nG=a * a, ng=b * b, sq=d * d, l1w=w * d.abs())
        for k, t in terms.items():
            S[k] += float(t.sum())
            A[k] += float(t.abs().sum())
        n += a.numel()
    rel = 4 * U2 + n * D53
    E = {k: rel * A[k] for k in S}
    E["sq"] += 2 * U * A["sq"]
    E["l1w"] += U * A["l1w"]
    return S, E


def match_value(kind, S, E, scale, tag_scale=0.1, fudge=1e-7):
    """``finalize_objective`` in float64 on the sums ``S`` and its first-order bound from the sum errors ``E``."""
    s = abs(scale)
    if kind == "euclidean":
        return 0.5 * scale * S["sq"], 0.5 * s * E["sq"]
    if kind == "l1":
        return 0.5 * scale * S["l1w"], 0.5 * s * E["l1w"]
    if kind == "tag-euclidean":
        return 0.5 * scale * (S["sq"] + tag_scale * S["l1w"]), 0.5 * s * (E["sq"] + abs(tag_scale) * E["l1w"])
    den = (S["nG"] * S["ng"]) ** 0.5
    c = S["dot"] / den
    dc = E["dot"] / den + abs(c) * 0.5 * (E["nG"] / S["nG"] + E["ng"] / S["ng"])
    if kind == "angular":
        lo, hi = -1.0 + fudge, 1.0 - fudge
        cc = min(max(c, lo), hi)
        inside = lo < c < hi
        return torch.acos(torch.tensor(cc, dtype=torch.float64)).item() / torch.pi * scale, \
            (s * dc / (torch.pi * (1.0 - cc * cc) ** 0.5) if inside else 0.0)
    return (1.0 - c) * scale, s * dc


def rna(t):
    """float64 tensor -> its fp32 value rounded to the TF32 grid, ties away from zero (``cvt.rna.tf32.f32``)."""
    f = t.to(torch.float32).contiguous()
    r = torch.bitwise_and(f.view(torch.int32) + 0x1000, -0x2000).view(torch.float32)
    return r.to(torch.float64)


def on_grid(t):
    """True if every element of ``t`` (fp32 values) has its 13 low mantissa bits zero."""
    f = t.to(torch.float32).contiguous()
    return bool((torch.bitwise_and(f.view(torch.int32), 0x1FFF) == 0).all())


def softmax_relation(z):
    """q = softmax(z) per row as the row kernels form it: (float64 reference, per-element bound); see the module docstring."""
    m = z.max(dim=1, keepdim=True).values
    d = (z - m).abs()
    R = (z.max(dim=1, keepdim=True).values - z.min(dim=1, keepdim=True).values)
    q = torch.softmax(z, dim=1)
    e_s = (8 + 4 * SOFTMAX_MERGES) * U + U * R
    return q, q * ((6 + d) * U + e_s) + SUBNORMAL


def chain_relation(q, g):
    """Softmax chain ``q (g - <q, g>)`` per row on the fp32 q and g the kernel read: (reference, bound)."""
    dot = (q * g).sum(dim=1, keepdim=True)
    ref = q * (g - dot)
    n = q.shape[1]
    A = (q * g).abs().sum(dim=1, keepdim=True)
    return ref, 2 * (q.abs() * (U * (g - dot).abs() + U * dot.abs() + n * D53 * A) + U * ref.abs())


def seed_relation(z, t, M, keep=1.0):
    """Cross-entropy seed ``(softmax(z) - t) / M`` on scored rows (``keep``) against the aligned targets t: (reference, bound)."""
    p = torch.softmax(z, dim=1)
    rng = (z - z.max(dim=1, keepdim=True).values).abs()
    return (p - t) * keep / M, (16 + 2 * rng) * U * (p + t.abs()) * keep / M


def tangent_seed_relation(p, zd, rng, M, keep=1.0):
    """Tangent of the cross-entropy seed ``p (zd - <p, zd>) / M`` on scored rows: (reference, bound).  ``rng``: |z - max z| when
    p is the float64 softmax of the stored logits (the kernel read its own fp32 p), 0 when p is what the kernel read."""
    ref = (p * zd - p * (p * zd).sum(dim=1, keepdim=True)) * keep / M
    mag = (p * zd.abs() + p * (p * zd.abs()).sum(dim=1, keepdim=True)) * keep / M
    return ref, (16 + 2 * rng) * U * mag


def label_gradient_relation(z, zd, p, p_rng, tau, M):
    """d objective / d target probabilities of each logits row, ``-(zd - <p, zd>) / M - tau (z - lse) / M``: (reference, bound).
    ``p``: the probabilities the kernel read (``p_rng`` as for ``tangent_seed_relation``)."""
    lse = torch.logsumexp(z, dim=1, keepdim=True)
    rng = (z - z.max(dim=1, keepdim=True).values).abs()
    dot = (p * zd).sum(dim=1, keepdim=True)
    ref = -(zd - dot) / M - tau * (z - lse) / M
    # <p, zdot> from the stored fp32 p (softmax bound) in double; lse in fp32 from a double sum of expf; a few roundings each
    bound = (4 * U * (zd.abs() + (p * zd.abs()).sum(dim=1, keepdim=True)) + ((16 + 2 * p_rng) * U * p * zd.abs()).sum(dim=1, keepdim=True)
             + abs(tau) * (8 * U * (z.abs() + lse.abs()) + (4 + 2 * rng.amax(dim=1, keepdim=True)) * U)) / M + U * ref.abs()
    return ref, bound


def to_target_rows(t, seq):
    """Token programs: the relation of logits row (b, t - 1) belongs to target row (b, t); rows at t = 0 are exactly zero."""
    first = (torch.arange(t.shape[0], device=t.device) % seq == 0).view(-1, 1)
    return torch.cat([torch.zeros_like(t[:1]), t[:-1]]).masked_fill(first, 0.0)


def task_loss_rows(z, q):
    """Per-row cross-entropy ``-sum_c q_c (z_c - lse)`` against targets q [rows, C] (one-hot for class indices): (loss, bound)."""
    mx = z.max(dim=1, keepdim=True).values
    lse = torch.logsumexp(z, dim=1, keepdim=True)
    rng = (z - mx).abs().amax(dim=1, keepdim=True)
    ln = -(q * (z - lse)).sum(dim=1)
    en = (q.abs() * ((16 + 2 * rng) * U + 4 * U * ((z - mx).abs() + mx.abs() + (lse - mx).abs()))).sum(dim=1) + 2 * U * ln.abs()
    return ln, en


def token_rows(rows, seq, device=None):
    """Token programs: (scored-row mask [rows, 1], M = rows - rows / T; 1 when no row is scored)."""
    keep = ((torch.arange(rows, device=device) % seq) != seq - 1).double().view(-1, 1)
    return keep, max(rows - rows // seq, 1)


def row_kernel_relations(kernel, z=None, q=None, g=None, p=None, zd=None, labels=None, T=1, coef=0.0, round_out=False):
    """(reference, bound) of every output of one row kernel (``engine.row_op``) from float64 inputs [rows, C]: ``z`` logits, ``q``
    soft targets / probabilities of the chain, ``g`` un-chained gradient, ``p`` probabilities the kernel read, ``zd`` logits
    tangent, ``labels`` class indices.  Returns {output name: (reference, bound)}."""
    tf = TF32_HALF if round_out else 0.0
    if kernel == "softmax":
        return {"q": softmax_relation(z)}
    if kernel == "softmax_chain":
        return {"g": chain_relation(q, g)}
    rows, C = (z if z is not None else p).shape
    if kernel in ("token_ce_fwd", "ce_fwd"):
        token = kernel == "token_ce_fwd"
        t = q if labels is None else F.one_hot(labels.view(-1).long(), C).to(z.dtype)
        keep, M = token_rows(rows, T, z.device) if token else (1.0, rows)
        if token:
            t = torch.cat([t[1:], torch.zeros_like(t[:1])]) * keep   # row (b, t) is scored against target row (b, t + 1)
        d, db = seed_relation(z, t, M, keep)
        ln, en = task_loss_rows(z, t)
        if token:
            ln, en = ln * keep.view(-1) * rows / M, (en * rows / M + 2 * U * ln.abs() * rows / M) * keep.view(-1)
        return {"p": softmax_relation(z), "loss": (ln, en), "dlogits": (d, db + tf * (d.abs() + db))}
    if kernel in ("token_ce_tan_bwd", "ce_tan_bwd"):
        keep, M = token_rows(rows, T, p.device) if kernel == "token_ce_tan_bwd" else (1.0, rows)
        ref, bound = tangent_seed_relation(p, zd, 0.0, M, keep)
        if labels is not None:   # the labelled tangent seed: coef (p - y) / N fused in
            y = F.one_hot(labels.view(-1).long(), C).to(p.dtype)
            ref = ref + coef * (p - y) / M
            bound = bound + 4 * U * abs(coef) * (p + y) / M + 2 * U * ref.abs()
        return {"tdlogits": (ref, bound + tf * (ref.abs() + bound))}
    if kernel in ("token_label_grad", "ce_label_grad"):
        token = kernel == "token_label_grad"
        M = token_rows(rows, T)[1] if token else rows
        ref, bound = label_gradient_relation(z, zd, p, 0.0, coef, M)
        if token:
            ref, bound = to_target_rows(ref, T), to_target_rows(bound, T)
        return {"out": (ref, bound)}
    raise ValueError(kernel)


def orthogonality_relation(x):
    """OrthogonalityRegularization (regularizers.py:169-178) as ``orthogonality_kernel`` forms it on the candidate x [N, ...]:
    (value, value bound, candidate gradient, gradient bound).  Per position k of the D = numel / N, the kernel sums S_k = sum_j x_jk^2
    and Q_k = sum_j x_jk^4 over the batch in fp32 (every term >= 0: S_k within ``(N + 2) u S_k``, Q_k within ``(N + 3) u Q_k``), the
    value ``(1/D) sum_k (S_k^2 - Q_k)`` in double (``2 S e_S + e_Q`` per position and the double reduction's ``(D + 4) 2^-53``), the
    gradient ``(4/D) x_ik (S_k - x_ik^2)`` in fp32 (the difference carries ``e_S + u x^2 + u |S - x^2|``, the three products
    one u each).  With fewer than two images the term is exactly 0."""
    N = x.shape[0]
    if N < 2:
        return 0.0, 0.0, torch.zeros_like(x), torch.zeros_like(x)
    xf = x.reshape(N, -1)
    D = xf.shape[1]
    x2 = xf * xf
    S, Q = x2.sum(dim=0), (x2 * x2).sum(dim=0)
    eS, eQ = (N + 2) * U * S, (N + 3) * U * Q
    val = float((S * S - Q).sum()) / D
    bound = float((2 * S * eS + eQ).sum() + (D + 4) * D53 * (S * S + Q).sum()) / D
    c = 4.0 / D
    diff = S - x2
    grad = c * xf * diff
    egrad = c * xf.abs() * (eS + U * x2 + U * diff.abs()) + 3 * U * grad.abs()
    return val, bound, grad.view_as(x), egrad.view_as(x)


def worst_element(y, ref, bound):
    """(worst error / bound ratio, flat index of that element); NaN counts as infinitely wrong, an exact match as 0."""
    err = (y - ref).abs()
    ratio = err / bound.clamp_min(TINY) if torch.is_tensor(bound) else err / max(bound, TINY)
    ratio = torch.where(err == 0, torch.zeros_like(ratio), ratio)
    ratio = torch.nan_to_num(ratio, nan=float("inf"))
    if not ratio.numel():
        return 0.0, 0
    j = int(ratio.flatten().argmax())
    return float(ratio.flatten()[j]), j


def check_row_kernel(kernel, outputs, **inputs):
    """Findings (kind = the kernel, sweep = the output name, index = the worst element) of one row kernel's ``outputs`` (dict of
    fp32 or float64 tensors keyed like ``row_kernel_relations``) against its relations; also returns {output: worst ratio}."""
    findings, ratios = [], {}
    for name, (ref, bound) in row_kernel_relations(kernel, **inputs).items():
        y = outputs[name].double().reshape(ref.shape)
        worst, j = worst_element(y, ref, bound)
        ratios[name] = worst
        if not worst <= 1.0:
            idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(j), y.shape))
            b = bound.expand_as(ref).flatten()[j] if torch.is_tensor(bound) else torch.tensor(bound)
            e = (y - ref).abs().flatten()[j]
            findings.append(Finding(-1, kernel, name, f"{kernel} {name}", idx, float(y.flatten()[j]), float(ref.flatten()[j]), float(e), float(b)))
    return findings, ratios


class Finding:
    def __init__(self, op, kind, sweep, what, index, value, ref, err, bound, step=None):
        self.op, self.kind, self.sweep, self.what = op, kind, sweep, what
        self.index, self.value, self.ref, self.err, self.bound = index, value, ref, err, bound
        self.step = step   # local step of a multi-step evaluation (None: single step, or a relation over all steps)

    def __repr__(self):
        at = "" if self.step is None else f"step {self.step}, "
        return (f"{at}op {self.op} ({self.kind}), sweep {self.sweep}, {self.what}: worst element {self.index} = {self.value:.9g}, "
                f"reference {self.ref:.9g}, error {self.err:.3g} > bound {self.bound:.3g}")


class SweepCheckError(AssertionError):
    pass


class SweepChecker:
    """``params``: float64 parameters in ``model.parameters()`` order (what the engine loaded); ``bn``: per op (rm, rv) or None;
    ``g``: target gradients; ``objective``: dict(kind, scale, task_regularization, tv=dict(scale, inner_exp, outer_exp, eps,
    double_opponents) | None, norm=dict(scale, p) | None, di=dict(scale, first_bn_multiplier) | None,
    features=dict(scale, measured) | None, and optionally orthogonality=True (the term is added into the ``norm`` slot, as the
    engine accumulates it there)).  DeepInversion's ``first_bn_multiplier`` goes to the first *registered* BN layer and the
    features prior reads the last *registered* Linear (``prog.di_first_op`` / ``prog.feature_op``, the reference's rule), not
    to the first / last one that runs."""

    def __init__(self, prog, params, bn, g, labels, objective, source):
        self.prog, self.src = prog, source
        self.P = [p.detach().double() for p in params]
        self.bn = bn
        self.g = [t.detach().double() for t in g]
        self.labels = labels
        self.obj = dict(scale=1.0, task_regularization=0.0, tv=None, norm=None, di=None, features=None)
        self.obj.update(objective)
        self.findings, self.ratios, self.off_grid = [], {}, set()
        self.seq = getattr(prog, "seq_len", 0)
        self.Vv = getattr(prog, "logits_valid", 0) or prog.tensors[prog.logits].C   # real classes
        ops = prog.ops
        self.first_consumer = {}
        for i, op in enumerate(ops):
            for t in (op.tin, op.res):
                if t >= 0 and t not in self.first_consumer:
                    self.first_consumer[t] = i
        self._cache = {}

    # ------------------------------------------------------------------ buffers
    def T(self, which, tid):
        """Buffer ``which`` of tensor ``tid`` in float64; logits-shaped tensors without their padded columns."""
        key = (which, tid)
        if key not in self._cache:
            v = self.src.tensor(which, tid)
            if v is not None and tid == self.prog.logits and v.shape[1] > self.Vv:
                v = v[:, :self.Vv]
            self._cache[key] = None if v is None else v.double()
        return self._cache[key]

    def _padding(self, which, op, sweep):
        """The padded logit columns of buffer ``which`` must be exactly zero."""
        v = self.src.tensor(which, self.prog.logits)
        if v is not None and v.shape[1] > self.Vv:
            pad = v[:, self.Vv:].double()
            self._cmp(op, sweep, f"{which}[t{self.prog.logits}] padded columns", pad, torch.zeros_like(pad), 0.0)

    def Pm(self, which, idx):
        key = ("p", which, idx)
        if key not in self._cache:
            self._cache[key] = self.src.param(which, idx).double()
        return self._cache[key]

    # ------------------------------------------------------------------ comparison
    def _cmp(self, i, sweep, what, y, ref, bound, kind=None):
        kind = kind or ("objective" if i < 0 else C.OP_NAMES[self.prog.ops[i].kind])
        err = (y - ref).abs()
        worst, j = worst_element(y, ref, bound)
        key = (kind, sweep)
        self.ratios[key] = max(self.ratios.get(key, 0.0), worst)
        if not worst <= 1.0:   # also catches NaN
            idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(j), y.shape)) if y.dim() else ()
            b = bound.expand_as(ref).flatten()[j] if torch.is_tensor(bound) else torch.tensor(bound)
            self.findings.append(Finding(i, kind, sweep, what, idx, float(y.flatten()[j]), float(ref.flatten()[j]),
                                         float(err.flatten()[j]), float(b)))

    @staticmethod
    def _rounded(y, ref):
        """Half a TF32 ulp of the reference where the engine stored ``y`` on the TF32 grid."""
        return TF32_HALF * ref.abs() if on_grid(y) else 0.0

    # ------------------------------------------------------------------ GEMM helpers
    def _gemm_fwd(self, op, act, wgt):
        if op.kind == C.OP_CONV:
            return F.conv2d(act, wgt, None, stride=op.stride, padding=op.pad)
        return F.linear(act.reshape(act.shape[0], -1), wgt).view(act.shape[0], -1, 1, 1)

    def _gemm_dgrad(self, op, shape, wgt, dout):
        if op.kind == C.OP_CONV:
            return torch.nn.grad.conv2d_input(shape, wgt, dout, stride=op.stride, padding=op.pad)
        return (dout.reshape(dout.shape[0], -1) @ wgt).view(shape)

    def _gemm_wgrad(self, op, act, shape, dout):
        if op.kind == C.OP_CONV:
            return torch.nn.grad.conv2d_weight(act, shape, dout, stride=op.stride, padding=op.pad)
        return dout.reshape(dout.shape[0], -1).t() @ act.reshape(act.shape[0], -1)

    def _K(self, op, mode):
        ti, to = self.prog.tensors[op.tin], self.prog.tensors[op.tout]
        if op.kind == C.OP_LINEAR:
            return {"fprop": ti.C * ti.H * ti.W, "dgrad": to.C, "wgrad": ti.N}[mode]
        return {"fprop": ti.C * op.R * op.S, "dgrad": to.C * op.R * op.S + op.R * op.S, "wgrad": to.N * to.H * to.W}[mode]

    def _operands(self, i, op):
        """(activation, W, v) as the kernels of op i read them."""
        a = self.T("val", op.tin)
        W, V = self.Pm("W_operand", op.w), self.Pm("v_operand", op.w)
        if self.src.rounds_operands(i):
            a, W, V = rna(a), rna(W), rna(V)
        return a, W, V

    def _truncation(self, i, op, a):
        """Relative widening for a tensor-core layer (its weights are read from the TF32 shadow) whose activation operand is
        stored off the TF32 grid: the tensor core truncates it (up to 2^-10 relative).  Recorded in ``off_grid``."""
        if self.src.rounds_operands(i) or not on_grid(self.Pm("W_operand", op.w)) or on_grid(a) or on_grid(self.P[op.w]):
            return 0.0
        self.off_grid.add(i)
        return 2.0 ** -10

    # ------------------------------------------------------------------ BN helpers
    def _bn_eval(self, i, op):
        rm, rv = self.bn[i]
        inv = 1.0 / torch.sqrt(rv + op.eps)
        gam, bet = self.P[op.gamma], self.P[op.beta]
        v = lambda t: t.view(1, -1, 1, 1)  # noqa: E731
        return v(rm), v(inv), v(gam), v(bet)

    @staticmethod
    def _m(t):
        return t.mean(dim=(0, 2, 3), keepdim=True)

    def _bn_train(self, op, x):
        mean = self._m(x)
        var = ((x - mean) ** 2).mean(dim=(0, 2, 3), keepdim=True)
        inv = 1.0 / torch.sqrt(var + op.eps)
        xh = (x - mean) * inv
        # conditioning of the fp32 batch statistics: E[x^2] / var (variance by differences) and the pixel count
        Pch = x.shape[0] * x.shape[2] * x.shape[3]
        cond = 1.0 + self._m(x * x) / var.clamp_min(TINY)
        return mean, var, inv, xh, TRAIN_C * (Pch + 8) * U * cond

    # ------------------------------------------------------------------ token helpers
    @staticmethod
    def _mc(t):
        return t.mean(dim=1, keepdim=True)

    def _ln(self, op, x):
        """Row statistics of a LayerNorm input [rows, C]: mean, inv, xh, A (magnitude of xh with the error of x - mean), c."""
        x = x.flatten(1)
        mean = self._mc(x)
        var = self._mc((x - mean) ** 2)
        inv = 1.0 / torch.sqrt(var + op.eps)
        xh = (x - mean) * inv
        cond = 1.0 + self._mc(x * x) / var.clamp_min(TINY)
        return mean, inv, xh, xh.abs() + inv * (x.abs() + mean.abs()), TRAIN_C * (x.shape[1] + 8) * U * cond

    def _heads(self, t, op, width):
        """[rows, width * d] -> ``width`` tensors [B, heads, T, dh]."""
        rows = t.shape[0]
        T_ = self.seq
        parts = t.flatten(1).split(t.shape[1] // width, dim=1)
        return [p.reshape(rows // T_, T_, op.R, -1).transpose(1, 2) for p in parts]

    @staticmethod
    def _merge(*ts):
        return torch.cat([t.transpose(1, 2).reshape(t.shape[0] * t.shape[2], -1) for t in ts], dim=1)

    @staticmethod
    def _mm(pairs, n):
        """sum of products A @ B over ``pairs`` = [(A, eA, B, eB)] (e: absolute error bound or None) with n terms in all:
        (value, error bound)."""
        val, err = 0.0, 0.0
        mag = 0.0
        for A, eA, B, eB in pairs:
            val = val + A @ B
            mag = mag + A.abs() @ B.abs()
            if eA is not None:
                err = err + eA @ B.abs()
            if eB is not None:
                err = err + A.abs() @ eB
        return val, err + (n + 2) * U2 * mag

    def _attention(self, op, qkv):
        """Scores and probabilities of every (sequence, head) with their error bounds."""
        Q, K, Vv = self._heads(qkv, op, 3)
        dh, T_ = Q.shape[-1], self.seq
        s = 1.0 / dh ** 0.5
        S0, eS0 = self._mm([(Q, None, K.transpose(-1, -2), None)], dh)
        S = S0 * s
        eS = eS0 * s + 3 * U * S.abs()
        P = torch.softmax(S, dim=-1)
        rho = eS + U * (S - S.amax(dim=-1, keepdim=True)).abs() + 2 * U
        eP = P * (rho + (P * rho).sum(dim=-1, keepdim=True) + (T_ + 2) * U2 + 2 * U)
        return Q, K, Vv, s, P, eP

    def _att_tangent_probs(self, op, Q, K, s, P, eP):
        """Tangent of the probabilities from the stored tangent of qkv: (Q', K', V', P', error of P')."""
        Qd, Kd, Vd = self._heads(self.T("tangent", op.tin), op, 3)
        dh, T_ = Q.shape[-1], self.seq
        Sd0, eSd0 = self._mm([(Qd, None, K.transpose(-1, -2), None), (Q, None, Kd.transpose(-1, -2), None)], 2 * dh)
        Sd = Sd0 * s
        eSd = eSd0 * s + 3 * U * Sd.abs()
        acc = (P * Sd).sum(dim=-1, keepdim=True)
        eacc = (T_ + 2) * U2 * (P * Sd.abs()).sum(dim=-1, keepdim=True) + (eP * Sd.abs() + P * eSd).sum(dim=-1, keepdim=True)
        diff = Sd - acc
        Pd = P * diff
        ePd = eP * diff.abs() + P * (eSd + eacc + U * diff.abs()) + U * Pd.abs()
        return Qd, Kd, Vd, Pd, ePd

    def _seed_rows(self, rows):
        """Token programs: (scored-row mask [rows, 1], M)."""
        return token_rows(rows, self.seq)

    def _targets(self, n):
        """Soft targets [n, classes] (float64) or the one-hot of class-index labels."""
        if self.labels.is_floating_point():
            return self.labels.double().reshape(n, -1)
        return F.one_hot(self.labels.view(-1).long(), self.Vv).double()

    # ------------------------------------------------------------------ sweeps
    def check(self, raise_on_failure=True):
        self.forward()
        self.backward()
        self.direction()
        self.tangent_forward()
        self.tangent_backward()
        if getattr(self.src, "has_tangent_G", False):
            self.tangent_G()
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def tangent_G(self):
        """Sweep TG: the tangent parameter gradients ``param("TG", j)`` of a multi-step step k > 0 (see module docstring).
        Run after ``tangent_forward`` (a tangent the engine did not store is taken from its reference)."""
        for i, op in enumerate(self.prog.ops):
            dT = self.T("tangent_delta", op.tout)
            if op.kind in (C.OP_CONV, C.OP_LINEAR):
                a, _, _ = self._operands(i, op)
                TGw = self.Pm("TG", op.w)
                ref, mag = self._gemm_wgrad(op, a, TGw.shape, dT), self._gemm_wgrad(op, a.abs(), TGw.shape, dT.abs())
                K, trunc = self._K(op, "wgrad"), self._truncation(i, op, a)
                if op.tin != 0:
                    ad = self._tangent_in(op)
                    if self.src.rounds_operands(i):
                        ad = rna(ad)
                    dB = self.T("delta", op.tout)
                    ref = ref + self._gemm_wgrad(op, ad, TGw.shape, dB)
                    mag = mag + self._gemm_wgrad(op, ad.abs(), TGw.shape, dB.abs())
                    K, trunc = 2 * K, max(trunc, self._truncation(i, op, ad))
                self._cmp(i, "TG", f"TG[{op.w}] (tangent weight gradient)", TGw, ref, ((K + 2) * U2 + trunc) * mag)
                if op.b >= 0:
                    P_ = dT.shape[0] * dT.shape[2] * dT.shape[3]
                    self._cmp(i, "TG", f"TG[{op.b}] (tangent bias gradient)", self.Pm("TG", op.b), dT.sum(dim=(0, 2, 3)),
                              (P_ + 4) * U2 * dT.abs().sum(dim=(0, 2, 3)))
            elif op.kind == C.OP_BNACT and op.has_bn:
                if op.bn_train:
                    raise NotImplementedError("tangent parameter gradients of train-mode BN")
                x = self.T("val", op.tin)
                mask = (self.T("val", op.tout) > 0).double() if op.relu else torch.ones_like(dT)
                duT, duB = dT * mask, self.T("delta", op.tout) * mask
                rm, inv, _, _ = self._bn_eval(i, op)
                xh, xhm = (x - rm) * inv, (x * inv).abs() + (rm * inv).abs()
                xd = self._tangent_in(op)
                Pch = x.shape[0] * x.shape[2] * x.shape[3]
                s = (duT.abs() * xhm + duB.abs() * xd.abs() * inv).sum(dim=(0, 2, 3))
                self._cmp(i, "TG", f"TG[{op.gamma}] (BN gamma tangent)", self.Pm("TG", op.gamma),
                          (duT * xh + duB * xd * inv).sum(dim=(0, 2, 3)), (2 * Pch + 4) * U2 * s)
                self._cmp(i, "TG", f"TG[{op.beta}] (BN beta tangent)", self.Pm("TG", op.beta), duT.sum(dim=(0, 2, 3)),
                          (Pch + 4) * U2 * duT.abs().sum(dim=(0, 2, 3)))

    def _tangent_in(self, op):
        """The stored tangent of op's input (its reference where the engine did not store it)."""
        if op.tin in self.src.unwritten:
            return self._tf_override[op.tin][0]
        return self.T("tangent", op.tin)

    def forward(self):
        prog = self.prog
        for i, op in enumerate(prog.ops):
            y = self.T("val", op.tout)
            x = self.T("val", op.tin)
            if op.kind in (C.OP_CONV, C.OP_LINEAR):
                a, W, _ = self._operands(i, op)
                ref = self._gemm_fwd(op, a, W)
                mag = self._gemm_fwd(op, a.abs(), W.abs())
                if op.b >= 0:
                    b = self.P[op.b].view(1, -1, 1, 1)
                    ref, mag = ref + b, mag + b.abs()
                bound = ((self._K(op, "fprop") + 2) * U2 + self._truncation(i, op, a)) * mag
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
            elif op.kind == C.OP_BNACT:
                u, mag = x, x.abs()
                if op.has_bn and op.bn_train:
                    mean, var, inv, xh, c = self._bn_train(op, x)
                    gam, bet = self.P[op.gamma].view(1, -1, 1, 1), self.P[op.beta].view(1, -1, 1, 1)
                    u = gam * xh + bet
                    mag = c * (gam.abs() * inv * (x.abs() + mean.abs())) / U + bet.abs()
                elif op.has_bn:
                    rm, inv, gam, bet = self._bn_eval(i, op)
                    u = gam * inv * x + (bet - gam * rm * inv)
                    mag = (gam * inv * x).abs() + bet.abs() + (gam * rm * inv).abs()
                if op.res >= 0:
                    r = self.T("val", op.res)
                    u, mag = u + r, mag + r.abs()
                ref = torch.relu(u) if op.relu else u
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, 8 * U * mag + self._rounded(y, ref))
            elif op.kind == C.OP_MAXPOOL:
                ref = F.max_pool2d(x, op.R, op.stride, op.pad)
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, 0.0)
            elif op.kind == C.OP_AVGPOOL:
                hw = x.shape[2] * x.shape[3]
                ref = x.mean(dim=(2, 3), keepdim=True)
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, (hw + 2) * U2 * x.abs().mean(dim=(2, 3), keepdim=True))
            elif op.kind == C.OP_POSADD:
                pos = self._pos_rows(self.P[op.w], x)
                ref = x + pos
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, 2 * U * (x.abs() + pos.abs()) + self._rounded(y, ref))
            elif op.kind == C.OP_LAYERNORM:
                mean, inv, xh, A, c = self._ln(op, x)
                gam, bet = self.P[op.gamma].view(1, -1), self.P[op.beta].view(1, -1)
                ref = (gam * xh + bet).view_as(y)
                bound = (c * gam.abs() * inv * (x.flatten(1).abs() + mean.abs()) + 4 * U * (gam * xh).abs() + 4 * U * bet.abs()).view_as(y)
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
            elif op.kind == C.OP_ATTENTION:
                _, _, Vv, _, P, eP = self._attention(op, x)
                O, eO = self._mm([(P, eP, Vv, None)], self.seq)
                ref, bound = self._merge(O).view_as(y), self._merge(eO).view_as(y)
                self._cmp(i, "F", f"val[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
        z = self.T("val", prog.logits).flatten(1)
        self._padding("val", len(prog.ops) - 1, "F")
        if self.seq:   # the next-token seed is checked with sweep B
            return
        # cross-entropy seed of sweep B (class indices or soft targets)
        n = z.shape[0]
        ref, bound = seed_relation(z, self._targets(n), n)
        d = self.T("delta", prog.logits).flatten(1)
        self._cmp(len(prog.ops) - 1, "F", f"delta[t{prog.logits}] (cross-entropy seed)", d, ref, bound)

    def _pos_rows(self, pos, like):
        rows = like.shape[0]
        return pos[:self.seq].repeat(rows // self.seq, 1).view_as(like)

    def _token_seed(self):
        """Next-token loss seed of sweep B: (p - q of the next row) / M on scored rows, exactly 0 on each sequence's last row."""
        prog = self.prog
        z = self.T("val", prog.logits).flatten(1)
        rows = z.shape[0]
        keep, M = self._seed_rows(rows)
        q = self._targets(rows)
        qn = torch.zeros_like(q)
        qn[:-1] = q[1:]
        ref, bound = seed_relation(z, qn * keep, M, keep)
        d = self.T("delta", prog.logits).flatten(1)
        self._cmp(len(prog.ops) - 1, "B", f"delta[t{prog.logits}] (next-token loss seed)", d, ref, bound + self._rounded(d, ref))
        self._padding("delta", len(prog.ops) - 1, "B")

    def _reverse(self, sweep):
        """Contributions of every op to the deltas (B) or tangent deltas (TB) of its inputs; returns {tid: [(i, ref, bound, mag)]}."""
        prog = self.prog
        tang = sweep == "TB"
        dn = "tangent_delta" if tang else "delta"
        contrib = {}

        def add(tid, i, ref, bound, mag):
            contrib.setdefault(tid, []).append((i, ref, bound, mag))

        for i in reversed(range(len(prog.ops))):
            op = prog.ops[i]
            x = self.T("val", op.tin)
            dout = self.T(dn, op.tout)
            if op.kind in (C.OP_CONV, C.OP_LINEAR):
                a, W, V = self._operands(i, op)
                want_in = op.tin != 0 or tang or self.obj["task_regularization"] != 0
                if want_in:
                    K = self._K(op, "dgrad")
                    ref = self._gemm_dgrad(op, x.shape, W, dout)
                    mag = self._gemm_dgrad(op, x.shape, W.abs(), dout.abs())
                    if tang:
                        dB = self.T("delta", op.tout)
                        ref = ref + self._gemm_dgrad(op, x.shape, V, dB)
                        mag = mag + self._gemm_dgrad(op, x.shape, V.abs(), dB.abs())
                        K = 2 * K
                    add(op.tin, i, ref, (K + 2) * U2 * mag, mag)
                if tang and self.obj["features"] is not None and op.kind == C.OP_LINEAR and i == self._feature_op():
                    fs = self.obj["features"]
                    diff = x.reshape(x.shape[0], -1) - fs["measured"].double().reshape(x.shape[0], -1)
                    adj = (2.0 * fs["scale"] / diff.numel() * diff).view_as(x)
                    add(op.tin, i, adj, 8 * U * (adj.abs() + 2.0 * fs["scale"] / diff.numel() * fs["measured"].double().abs().view_as(x)), adj.abs())
                if not tang:   # parameter gradients
                    Gw = self.Pm("G", op.w)
                    ref = self._gemm_wgrad(op, a, Gw.shape, dout)
                    mag = self._gemm_wgrad(op, a.abs(), Gw.shape, dout.abs())
                    self._cmp(i, "B", f"G[{op.w}] (weight gradient)", Gw, ref,
                              ((self._K(op, "wgrad") + 2) * U2 + self._truncation(i, op, a)) * mag)
                    if op.b >= 0:
                        Gb = self.Pm("G", op.b)
                        P_ = dout.shape[0] * dout.shape[2] * dout.shape[3]
                        self._cmp(i, "B", f"G[{op.b}] (bias gradient)", Gb, dout.sum(dim=(0, 2, 3)),
                                  (P_ + 4) * U2 * dout.abs().sum(dim=(0, 2, 3)))
            elif op.kind == C.OP_BNACT:
                y = self.T("val", op.tout)
                mask = (y > 0).double() if op.relu else torch.ones_like(y)
                du = dout * mask
                if op.res >= 0:
                    add(op.res, i, du, 0.0, du.abs())
                if op.has_bn and op.bn_train:
                    mean, var, inv, xh, c = self._bn_train(op, x)
                    gam = self.P[op.gamma].view(1, -1, 1, 1)
                    m = self._m
                    duB = self.T("delta", op.tout) * mask
                    if not tang:
                        ref = gam * inv * (du - m(du) - xh * m(du * xh))
                        mag = gam.abs() * inv * (du.abs() + m(du.abs()) + xh.abs() * m((du * xh).abs()))
                        self._bn_param_grads(i, op, du, xh, xh.abs())
                    else:
                        xd = self.T("tangent", op.tin) if op.tin not in self.src.unwritten else self._tf_override[op.tin]
                        xhd = inv * (xd - m(xd) - xh * m(xh * xd))
                        vg = self.Pm("v_operand", op.gamma).view(1, -1, 1, 1)
                        invd = -inv * inv * m(xh * xd)
                        w = duB - m(duB) - xh * m(duB * xh)
                        wd = du - m(du) - xhd * m(duB * xh) - xh * m(du * xh + duB * xhd)
                        ref = (vg * inv + gam * invd) * w + gam * inv * wd
                        A = lambda t: t.abs()  # noqa: E731
                        wm = A(duB) + m(A(duB)) + A(xh) * m(A(duB * xh))
                        xhdm = inv * (A(xd) + m(A(xd)) + A(xh) * m(A(xh * xd)))
                        wdm = A(du) + m(A(du)) + xhdm * m(A(duB * xh)) + A(xh) * m(A(du * xh) + A(duB) * xhdm)
                        mag = (A(vg) * inv + A(gam) * inv * inv * m(A(xh * xd))) * wm + A(gam) * inv * wdm
                    add(op.tin, i, ref, c * mag, mag)
                elif op.has_bn:
                    rm, inv, gam, bet = self._bn_eval(i, op)
                    xh = (x - rm) * inv
                    xhm = (x * inv).abs() + (rm * inv).abs()
                    ref, mag = gam * inv * du, (gam * inv * du).abs()
                    if tang:
                        vg = self.Pm("v_operand", op.gamma).view(1, -1, 1, 1)
                        duB = self.T("delta", op.tout) * mask
                        ref, mag = ref + vg * inv * duB, mag + (vg * inv * duB).abs()
                    else:
                        self._bn_param_grads(i, op, du, xh, xhm)
                    add(op.tin, i, ref, 8 * U * mag, mag)
                    if tang and self.obj["di"] is not None:
                        adj, bnd = self._di_adjoint(i, op, x)
                        add(op.tin, i, adj, bnd, adj.abs())
                else:
                    add(op.tin, i, du, 0.0, du.abs())
            elif op.kind == C.OP_MAXPOOL:
                _, idx = F.max_pool2d(x, op.R, op.stride, op.pad, return_indices=True)
                N_, Cc, H, W_ = x.shape
                ref = torch.zeros(N_, Cc, H * W_, dtype=torch.float64).scatter_add_(2, idx.flatten(2), dout.flatten(2)).view_as(x)
                mag = torch.zeros(N_, Cc, H * W_, dtype=torch.float64).scatter_add_(2, idx.flatten(2), dout.abs().flatten(2)).view_as(x)
                add(op.tin, i, ref, op.R * op.R * U * mag, mag)
            elif op.kind == C.OP_AVGPOOL:
                hw = x.shape[2] * x.shape[3]
                ref = (dout / hw).expand_as(x)
                add(op.tin, i, ref, 2 * U * ref.abs(), ref.abs())
            elif op.kind == C.OP_POSADD:
                add(op.tin, i, dout, 0.0, dout.abs())
                if not tang:   # positional-table gradient: sum over the sequences, rows >= T untouched
                    d2 = dout.flatten(1).reshape(-1, self.seq, dout.shape[1])
                    Gp = self.Pm("G", op.w)
                    ref, mag = torch.zeros_like(Gp), torch.zeros_like(Gp)
                    ref[:self.seq], mag[:self.seq] = d2.sum(dim=0), d2.abs().sum(dim=0)
                    self._cmp(i, "B", f"G[{op.w}] (positional table gradient)", Gp, ref, (d2.shape[0] + 4) * U2 * mag)
            elif op.kind == C.OP_LAYERNORM:
                ref, bound, mag = self._ln_reverse(i, op, x, dout, tang)
                add(op.tin, i, ref.view_as(x), bound.view_as(x), mag.view_as(x))
            elif op.kind == C.OP_ATTENTION:
                ref, bound = self._att_reverse(op, x, dout, tang)
                add(op.tin, i, ref.view_as(x), bound.view_as(x), (ref.abs() + bound).view_as(x))
        return contrib

    def _ln_reverse(self, i, op, x, dout, tang):
        """LayerNorm input delta (B) or tangent delta (TB): (reference, bound, magnitude) as [rows, C]; B also checks gamma / beta."""
        m = self._mc
        mean, inv, xh, A, c = self._ln(op, x)
        gam = self.P[op.gamma].view(1, -1)
        dy = dout.flatten(1)
        if not tang:
            t = dy * gam
            ref = inv * (t - m(t) - xh * m(t * xh))
            mag = inv * (t.abs() + m(t.abs()) + A * m(t.abs() * A))
            rows = dy.shape[0]
            s = (dy.abs() * xh.abs()).sum(dim=0)
            bound = (rows + 4) * U2 * s + (c * dy.abs() * inv * (x.flatten(1).abs() + mean.abs())).sum(dim=0)
            self._cmp(i, "B", f"G[{op.gamma}] (LayerNorm gamma gradient)", self.Pm("G", op.gamma), (dy * xh).sum(dim=0), bound)
            self._cmp(i, "B", f"G[{op.beta}] (LayerNorm beta gradient)", self.Pm("G", op.beta), dy.sum(dim=0),
                      (rows + 4) * U2 * dy.abs().sum(dim=0))
            return ref, c * mag, mag
        dyB = self.T("delta", op.tout).flatten(1)
        xd = self.T("tangent", op.tin).flatten(1)
        vg = self.Pm("v_operand", op.gamma).view(1, -1)
        xhd = inv * (xd - m(xd) - xh * m(xh * xd))
        t, td = dyB * gam, dy * gam + dyB * vg
        u = t - m(t) - xh * m(t * xh)
        ud = td - m(td) - xhd * m(t * xh) - xh * m(td * xh + t * xhd)
        ref = inv * ud - u * m(xh * xd) * inv * inv
        At, Atd = t.abs(), dy.abs() * gam.abs() + dyB.abs() * vg.abs()
        Axhd = inv * (xd.abs() + m(xd.abs()) + A * m(A * xd.abs()))
        Au = At + m(At) + A * m(At * A)
        Aud = Atd + m(Atd) + Axhd * m(At * A) + A * m(Atd * A + At * Axhd)
        mag = inv * Aud + Au * m(A * xd.abs()) * inv * inv
        return ref, c * mag, mag

    def _att_reverse(self, op, qkv, dout, tang):
        """Attention: delta (B) or tangent delta (TB) of qkv, (reference, bound) as [rows, 3 d]."""
        T_ = self.seq
        Q, K, Vv, s, P, eP = self._attention(op, qkv)
        dh = Q.shape[-1]
        tr = lambda t: t.transpose(-1, -2)  # noqa: E731
        (dO,) = self._heads(self.T("delta", op.tout), op, 1)
        dP, edP = self._mm([(dO, None, tr(Vv), None)], dh)
        r = (dP * P).sum(dim=-1, keepdim=True)
        er = (T_ + 2) * U2 * (dP.abs() * P).sum(dim=-1, keepdim=True) + (edP * P + dP.abs() * eP).sum(dim=-1, keepdim=True)
        diff = dP - r
        ediff = edP + er + U * diff.abs()
        dS = P * diff
        edS = eP * diff.abs() + P * ediff + U * dS.abs()
        if not tang:
            dQ, edQ = self._mm([(dS, edS, K, None)], T_)
            dK, edK = self._mm([(tr(dS), tr(edS), Q, None)], T_)
            dV, edV = self._mm([(tr(P), tr(eP), dO, None)], T_)
            grads = [(dQ * s, edQ * s + 3 * U * (dQ * s).abs()), (dK * s, edK * s + 3 * U * (dK * s).abs()), (dV, edV)]
        else:
            (dOd,) = self._heads(dout, op, 1)
            Qd, Kd, Vd, Pd, ePd = self._att_tangent_probs(op, Q, K, s, P, eP)
            dPd, edPd = self._mm([(dOd, None, tr(Vv), None), (dO, None, tr(Vd), None)], 2 * dh)
            rd = (dPd * P + dP * Pd).sum(dim=-1, keepdim=True)
            erd = (2 * T_ + 2) * U2 * (dPd.abs() * P + dP.abs() * Pd.abs()).sum(dim=-1, keepdim=True) + \
                (edPd * P + dPd.abs() * eP + edP * Pd.abs() + dP.abs() * ePd).sum(dim=-1, keepdim=True)
            diff2 = dPd - rd
            ediff2 = edPd + erd + U * diff2.abs()
            dSd = Pd * diff + P * diff2
            edSd = ePd * diff.abs() + Pd.abs() * ediff + eP * diff2.abs() + P * ediff2 + 2 * U * ((Pd * diff).abs() + (P * diff2).abs())
            dQ, edQ = self._mm([(dSd, edSd, K, None), (dS, edS, Kd, None)], 2 * T_)
            dK, edK = self._mm([(tr(dSd), tr(edSd), Q, None), (tr(dS), tr(edS), Qd, None)], 2 * T_)
            dV, edV = self._mm([(tr(Pd), tr(ePd), dO, None), (tr(P), tr(eP), dOd, None)], 2 * T_)
            grads = [(dQ * s, edQ * s + 3 * U * (dQ * s).abs()), (dK * s, edK * s + 3 * U * (dK * s).abs()), (dV, edV)]
        return self._merge(*[g for g, _ in grads]), self._merge(*[e for _, e in grads])

    def _bn_param_grads(self, i, op, du, xh, xhm):
        Pch = du.shape[0] * du.shape[2] * du.shape[3]
        s = (du.abs() * xhm).sum(dim=(0, 2, 3))
        bound = (Pch + 4) * U2 * s
        if op.bn_train:   # xh itself comes from the fp32 batch statistics
            bound = bound + self._bn_train(op, self.T("val", op.tin))[4].view(-1) * s
        self._cmp(i, "B", f"G[{op.gamma}] (BN gamma gradient)", self.Pm("G", op.gamma), (du * xh).sum(dim=(0, 2, 3)), bound)
        self._cmp(i, "B", f"G[{op.beta}] (BN beta gradient)", self.Pm("G", op.beta), du.sum(dim=(0, 2, 3)),
                  (Pch + 4) * U2 * du.abs().sum(dim=(0, 2, 3)))

    def _first_bn(self):
        """The BN op whose DeepInversion term carries ``first_bn_multiplier``: the first registered BatchNorm2d (the first BN op
        when the program does not record registration order, e.g. token programs)."""
        first = getattr(self.prog, "di_first_op", -1)
        return first if first >= 0 else min(j for j, o in enumerate(self.prog.ops) if o.kind == C.OP_BNACT and o.has_bn)

    def _feature_op(self):
        """The Linear op whose input the features prior reads: the last registered Linear (else the last Linear op)."""
        last = getattr(self.prog, "feature_op", -1)
        return last if last >= 0 else max(j for j, o in enumerate(self.prog.ops) if o.kind == C.OP_LINEAR)

    def _di_layer(self, i, z):
        """Batch statistics of the BN input ``z`` of op i against the running statistics: (M, mean, var, nm, nv, kap_m, kap_v),
        kap_m / kap_v the conditioning of the fp32 statistics (P = M terms) and of the norms of their differences."""
        rm, rv = self.bn[i]
        M = z.shape[0] * z.shape[2] * z.shape[3]
        mean = z.mean(dim=(0, 2, 3))
        var = z.var(dim=(0, 2, 3), unbiased=False)
        nv, nm = torch.norm(rv - var, 2), torch.norm(rm - mean, 2)
        kap_m = 1.0 + (mean.abs().norm() + rm.norm()) / nm
        kap_v = 1.0 + ((z * z).mean(dim=(0, 2, 3)).norm() + rv.norm()) / nv
        return M, mean, var, nm, nv, kap_m, kap_v

    def _di_adjoint(self, i, op, z):
        """DeepInversion adjoint at the input of BN op i (program_interp.deep_inversion, engine statistics of ``z``)."""
        di = self.obj["di"]
        mult = di["scale"] * (di.get("first_bn_multiplier", 10.0) if i == self._first_bn() else 1.0)
        rm, rv = self.bn[i]
        M, mean, var, nm, nv, kap_m, kap_v = self._di_layer(i, z)
        cm = (mean - rm) / nm / M
        cv = (var - rv) / nv * 2.0 / M
        v = lambda t: t.view(1, -1, 1, 1)  # noqa: E731
        adj = mult * (v(cm) + v(cv) * (z - v(mean)))
        mag = abs(mult) * (v(cm.abs()) * kap_m + v(cv.abs()) * kap_v * ((z - v(mean)).abs() + v(mean.abs()) + z.abs()))
        return adj, TRAIN_C * (M + 8) * U * mag

    def _check_deltas(self, sweep, contrib):
        dn = "tangent_delta" if sweep == "TB" else "delta"
        for tid, parts in contrib.items():
            if tid == 0:
                continue
            y = self.T(dn, tid)
            ref = sum(p[1] for p in parts)
            mag = sum(p[3] for p in parts)
            bound = sum(p[2] for p in parts) + len(parts) * U * mag
            if on_grid(y):
                bound = bound + len(parts) * TF32_HALF * mag
            self._cmp(self.first_consumer[tid], sweep, f"{dn}[t{tid}] (sum over {len(parts)} consumer(s))", y, ref, bound)
        return contrib

    def backward(self):
        if self.seq:
            self._token_seed()
        contrib = self._check_deltas("B", self._reverse("B"))
        if self.obj["task_regularization"] != 0 and 0 in contrib:
            parts = contrib[0]
            ref, mag = sum(p[1] for p in parts), sum(p[3] for p in parts)
            self._cmp(self.first_consumer[0], "B", "delta[t0] (task-loss gradient)", self.T("delta", 0), ref,
                      sum(p[2] for p in parts) + U * mag)

    def direction(self):
        o = self.obj
        n = len(self.P)
        G = [self.Pm("G", j) for j in range(n)]
        kw = {k: o[k] for k in ("tag_scale", "scale_scheme") if k in o}
        _, v = objective_direction(o["kind"], G, self.g, scale=o["scale"], **kw)
        s = abs(o["scale"])
        if o["kind"] in ("cosine-similarity", "angular", "fast-cosine-similarity", "masked-cosine-similarity"):
            Gs, gs = G, self.g
            if o["kind"] == "masked-cosine-similarity":   # the kernels' coefficients come from the masked sums
                keep = [(b.to(torch.float32).abs() > MASK_VALUE).double() for b in self.g]
                Gs, gs = [a * k for a, k in zip(G, keep)], [b * k for b, k in zip(self.g, keep)]
            nG = sum(a.pow(2).sum() for a in Gs).sqrt()
            ng = sum(b.pow(2).sum() for b in gs).sqrt()
            al, be = 1.0 / (nG * ng), abs(sum((a * b).sum() for a, b in zip(Gs, gs))) / (nG.pow(3) * ng)
            if o["kind"] == "angular":   # chain factor d acos(c) / dc
                c = float(sum((a * b).sum() for a, b in zip(G, self.g)) / (nG * ng))
                al, be = al / (torch.pi * max(1.0 - c * c, 1e-14) ** 0.5), be / (torch.pi * max(1.0 - c * c, 1e-14) ** 0.5)
            mags = [s * (al * b.abs() + be * a.abs()) for a, b in zip(G, self.g)]
        elif o["kind"] == "l1":    # 0.5 s sign(G - g): exact in fp32
            mags = [0.5 * s * torch.ones_like(a) for a in G]
        else:
            # euclidean s (G - g) and tag-euclidean s ((G - g) + tag_scale / 2 w_l sign(G - g)): make_v_kernel evaluates
            # fma(-s, g, fma(s, G, c3 w sign(G - g))) -- the difference G - g is never rounded on its own, so each of the two
            # roundings is relative to s (|G| + |g|) + c3 w, not to s |G - g| (which vanishes where G and g agree)
            L = len(G)
            w = [0.0] * L
            if o["kind"] == "tag-euclidean":
                scheme = o.get("scale_scheme", "linear")
                if scheme == "linear":
                    w = (torch.arange(L, 0, -1, dtype=torch.float64) / L).tolist()
                elif scheme == "exp":
                    e = torch.arange(L, 0, -1, dtype=torch.float64).softmax(dim=0)
                    w = (e / e[0]).tolist()
                else:
                    w = [1.0] * L
                w = [0.5 * o.get("tag_scale", 0.1) * wl for wl in w]
            mags = [s * (a.abs() + b.abs() + wl) for a, b, wl in zip(G, self.g, w)]
        for j in range(n):
            y = self.Pm("v_operand", j)
            bound = 16 * U * mags[j] + (TF32_HALF * v[j].abs() if on_grid(y) else 0.0)
            self._cmp(-1, "V", f"v[{j}] (direction, operand form)", y, v[j], bound)

    def tangent_forward(self):
        self._tf_override = {}
        prog = self.prog
        for i, op in enumerate(prog.ops):
            x = self.T("val", op.tin)
            tin, tin_bound = None, 0.0
            if op.tin != 0:
                if op.tin in self.src.unwritten:
                    tin, tin_bound = self._tf_override[op.tin]
                else:
                    tin = self.T("tangent", op.tin)
            if op.kind in (C.OP_CONV, C.OP_LINEAR):
                a, W, V = self._operands(i, op)
                ref, mag = self._gemm_fwd(op, a, V), self._gemm_fwd(op, a.abs(), V.abs())
                K = self._K(op, "fprop")
                if tin is not None:
                    ref = ref + self._gemm_fwd(op, tin, W)
                    mag = mag + self._gemm_fwd(op, tin.abs(), W.abs())
                    K = 2 * K
                if op.b >= 0:
                    vb = self.Pm("v_operand", op.b).view(1, -1, 1, 1)
                    ref, mag = ref + vb, mag + vb.abs()
                bound = ((K + 2) * U2 + self._truncation(i, op, a)) * mag
                if op.tout in self.src.unwritten:
                    self._tf_override[op.tout] = (ref, bound)
                    continue
                y = self.T("tangent", op.tout)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
                continue
            y = self.T("tangent", op.tout)
            if op.kind == C.OP_BNACT:
                u = tin if tin is not None else torch.zeros_like(x)
                mag, extra = u.abs(), tin_bound
                if op.has_bn and op.bn_train:
                    mean, var, inv, xh, c = self._bn_train(op, x)
                    m = self._m
                    gam = self.P[op.gamma].view(1, -1, 1, 1)
                    vg, vb = (self.Pm("v_operand", k).view(1, -1, 1, 1) for k in (op.gamma, op.beta))
                    xhd = inv * (u - m(u) - xh * m(xh * u))
                    u = vg * xh + gam * xhd + vb
                    mag = c / U * (vg.abs() * xh.abs() + gam.abs() * inv * (mag + m(mag) + xh.abs() * m((xh * mag).abs()))) + vb.abs()
                    extra = gam.abs() * inv * 3 * (tin_bound if torch.is_tensor(tin_bound) else torch.tensor(tin_bound)).amax() \
                        if tin is not None else 0.0
                elif op.has_bn:
                    rm, inv, gam, bet = self._bn_eval(i, op)
                    vg, vb = (self.Pm("v_operand", k).view(1, -1, 1, 1) for k in (op.gamma, op.beta))
                    xh = (x - rm) * inv
                    u = gam * inv * u + vg * xh + vb
                    mag = (gam * inv).abs() * mag + vg.abs() * ((x * inv).abs() + (rm * inv).abs()) + vb.abs()
                    extra = (gam * inv).abs() * tin_bound
                if op.res >= 0:
                    r = self.T("tangent", op.res)
                    u, mag = u + r, mag + r.abs()
                if op.relu:
                    mask = (self.T("val", op.tout) > 0).double()
                    u, mag, extra = u * mask, mag * mask, extra * mask
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, u, 8 * U * mag + extra + self._rounded(y, u))
            elif op.kind == C.OP_MAXPOOL:
                _, idx = F.max_pool2d(x, op.R, op.stride, op.pad, return_indices=True)
                ref = tin.flatten(2).gather(2, idx.flatten(2)).view_as(idx)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, ref, 0.0)
            elif op.kind == C.OP_AVGPOOL:
                hw = tin.shape[2] * tin.shape[3]
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, tin.mean(dim=(2, 3), keepdim=True),
                          (hw + 2) * U2 * tin.abs().mean(dim=(2, 3), keepdim=True))
            elif op.kind == C.OP_POSADD:   # the candidate's tangent is zero: v of the positional table, copied
                ref = self._pos_rows(self.Pm("v_operand", op.w), y)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, ref, self._rounded(y, ref))
            elif op.kind == C.OP_LAYERNORM:
                m = self._mc
                mean, inv, xh, A, c = self._ln(op, x)
                gam = self.P[op.gamma].view(1, -1)
                vg, vb = (self.Pm("v_operand", k).view(1, -1) for k in (op.gamma, op.beta))
                xd = tin.flatten(1)
                xhd = inv * (xd - m(xd) - xh * m(xh * xd))
                ref = (vg * xh + gam * xhd + vb).view_as(y)
                Axhd = inv * (xd.abs() + m(xd.abs()) + A * m(A * xd.abs()))
                bound = (c * (vg.abs() * A + gam.abs() * Axhd) + 4 * U * vb.abs()).view_as(y)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
            elif op.kind == C.OP_ATTENTION:
                Q, K, Vv, s, P, eP = self._attention(op, x)
                _, _, Vd, Pd, ePd = self._att_tangent_probs(op, Q, K, s, P, eP)
                Od, eOd = self._mm([(Pd, ePd, Vv, None), (P, eP, Vd, None)], 2 * self.seq)
                ref, bound = self._merge(Od).view_as(y), self._merge(eOd).view_as(y)
                self._cmp(i, "TF", f"tangent[t{op.tout}]", y, ref, bound + self._rounded(y, ref))
        self._padding("tangent", len(prog.ops) - 1, "TF")

    def tangent_backward(self):
        prog = self.prog
        # seed: tangent of the cross-entropy delta (token programs: scored rows, mean over M)
        z = self.T("val", prog.logits).flatten(1)
        zd = self.T("tangent", prog.logits).flatten(1)
        n = z.shape[0]
        keep, M = self._seed_rows(n) if self.seq else (1.0, n)
        rng = (z - z.max(dim=1, keepdim=True).values).abs()
        ref, bound = tangent_seed_relation(torch.softmax(z, dim=1), zd, rng, M, keep)
        y = self.T("tangent_delta", prog.logits).flatten(1)
        self._cmp(len(prog.ops) - 1, "TB", f"tangent_delta[t{prog.logits}] (cross-entropy seed)", y, ref, bound + self._rounded(y, ref))
        self._padding("tangent_delta", len(prog.ops) - 1, "TB")
        contrib = self._check_deltas("TB", self._reverse("TB"))
        # the candidate gradient: first op's contribution + image priors + task term
        parts = contrib.get(0, [])
        x = self.T("val", 0)
        ref = sum(p_[1] for p_ in parts)
        mag = sum(p_[3] for p_ in parts)
        bound = sum(p_[2] for p_ in parts) + 2 * U * mag
        o = self.obj
        xd = x.clone().requires_grad_(True)
        prior = torch.zeros((), dtype=torch.float64)
        if o["tv"] is not None:
            tv = o["tv"]
            prior = prior + restate.total_variation(xd, scale=tv["scale"], inner_exp=tv.get("inner_exp", 1), outer_exp=tv.get("outer_exp", 1),
                                                    double_opponents=tv.get("double_opponents", False), eps=tv.get("eps", 1e-8))
        if o["norm"] is not None:
            prior = prior + restate.norm_regularization(xd, scale=o["norm"]["scale"], pnorm=o["norm"].get("p", 2.0))
        if prior.requires_grad:
            (gp,) = torch.autograd.grad(prior, xd)
            ref = ref + gp
            tvs = o["tv"]["scale"] if o["tv"] is not None else 0.0
            bound = bound + 64 * U * (gp.abs() + 4 * tvs / x.numel())
        if o.get("orthogonality"):   # added into the candidate gradient after the other priors: one more rounding of the sum
            _, _, og, eog = orthogonality_relation(x)
            ref = ref + og
            bound = bound + eog + 2 * U * (ref.abs() + og.abs())
        if o["task_regularization"] != 0:
            dt = self.T("delta", 0)
            ref = ref + o["task_regularization"] * dt
            bound = bound + 2 * U * abs(o["task_regularization"]) * dt.abs()
        self._cmp(self.first_consumer[0], "TB", "tangent_delta[t0] (candidate gradient)", self.T("tangent_delta", 0), ref, bound)

    def check_label_gradient(self, lg, raise_on_failure=True):
        """d objective / d (target probabilities) as ``bre_engine_label_gradient`` returns it ([rows or N, classes]):
        ``-(zdot - <p, zdot>) / M - tau (z - lse) / M`` of the source row -- the row itself for vision programs (M = N), row
        (b, t - 1) for token programs (exactly 0 at t = 0).  Run after ``check()`` (or ``forward()``)."""
        z = self.T("val", self.prog.logits).flatten(1)
        zd = self.T("tangent", self.prog.logits).flatten(1)
        n = z.shape[0]
        M = n - n // self.seq if self.seq else n
        rng = (z - z.max(dim=1, keepdim=True).values).abs()
        ref, bound = label_gradient_relation(z, zd, torch.softmax(z, dim=1), rng, self.obj["task_regularization"], M)
        if self.seq:
            ref, bound = to_target_rows(ref, self.seq), to_target_rows(bound, self.seq)
        y = lg.double().reshape(n, -1)
        self._cmp(len(self.prog.ops) - 1, "L", "label gradient", y, ref, bound, kind="label")
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def check_label_leaf(self, ell, q, g_pre, g_chained, raise_on_failure=True):
        """The label leaf of a joint iteration: ``q`` (the soft targets the evaluation read, ``debug_step_state("soft_q")``)
        against softmax of the label logits ``ell`` the iteration started from, and ``g_chained`` (``debug_step_state("label_grad")``)
        against the softmax chain of the engine's own q and un-chained gradient ``g_pre`` (``label_gradient``).  Reported with
        the kernel's name as the kind, sweep "L"."""
        n = ell.shape[0]
        q64, g64 = q.double().reshape(n, -1), g_pre.double().reshape(n, -1)
        ref, bound = softmax_relation(ell.double().reshape(n, -1))
        self._cmp(-1, "L", "soft targets q = softmax(label logits)", q64, ref, bound, kind="row_softmax")
        ref, bound = chain_relation(q64, g64)
        self._cmp(-1, "L", "label-logit gradient q (g - <q, g>)", g_chained.double().reshape(n, -1), ref, bound, kind="softmax_chain")
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    # ------------------------------------------------------------------ objective terms
    def _match_term(self, G, kind, scale):
        o = self.obj
        w = tag_weights(len(G), o.get("scale_scheme", "linear")) if kind == "tag-euclidean" else None
        S, E = match_sums(G, self.g, kind, w)
        val, bound = match_value(kind, S, E, f32(scale), f32(o.get("tag_scale", 0.1)), f32(1e-7))
        return val, bound + 16 * D53 * (abs(val) + abs(scale))

    def _task_loss_term(self):
        z = self.T("val", self.prog.logits).flatten(1)
        ln, en = task_loss_rows(z, self._targets(z.shape[0]))
        L = float(ln.mean())
        return L, float(en.mean()) + U * abs(L)

    def _tv_term(self, x):
        t = self.obj["tv"]
        p, q, eps, s = (f32(t.get(k, d)) for k, d in (("inner_exp", 1), ("outer_exp", 1), ("eps", 1e-8), ("scale", 0.0)))
        X, Xe = x, torch.zeros_like(x)
        if t.get("double_opponents", False):   # planes x_a - x_b, each carrying the rounding of its own difference
            d = torch.cat([x[:, 0:1] - x[:, 1:2], x[:, 0:1] - x[:, 2:3], x[:, 1:2] - x[:, 2:3]], dim=1)
            X, Xe = torch.cat([x, d], dim=1), torch.cat([Xe, U * d.abs()], dim=1)
        nb_h = lambda t_: F.pad(t_, (0, 0, 0, 1))[:, :, 1:, :]  # noqa: E731  (neighbour below / right, 0 past the edge)
        nb_w = lambda t_: F.pad(t_, (0, 1, 0, 0))[:, :, :, 1:]  # noqa: E731
        cp, cq = (0.0 if e == 1.0 else POW_C for e in (p, q))
        parts = []
        for nb in (nb_h, nb_w):
            dd = nb(X) - X
            A = dd.abs() + eps
            eA = U * dd.abs() + Xe + nb(Xe) + U * A
            Ap = A.pow(p)
            parts.append((A, eA, Ap))
        (A, eA, Ap), (B, eB, Bp) = parts
        ssum = Ap + Bp
        es = abs(p) * (A.pow(p - 1) * eA + B.pow(p - 1) * eB) + cp * U * ssum + U * ssum
        f = ssum.pow(q)
        ef = abs(q) * ssum.pow(q - 1) * es + cq * U * f
        n = f.numel()
        val = s * float(f.sum()) / n
        return val, abs(s) * float(ef.sum() + n * D53 * f.abs().sum()) / n + 4 * D53 * abs(val)

    def _norm_term(self, x):
        nr = self.obj["norm"]
        s, p = f32(nr["scale"]), f32(nr.get("p", 2.0))
        xp = x.pow(p)
        val = s / p * float(xp.mean())
        return val, abs(s / p) * ((0.0 if p == 1.0 else POW_C * U) + xp.numel() * D53) * float(xp.abs().mean()) + 4 * D53 * abs(val)

    def _di_term(self):
        di = self.obj["di"]
        first = self._first_bn()
        val, bound = 0.0, 0.0
        for i, op in enumerate(self.prog.ops):
            if op.kind != C.OP_BNACT or not op.has_bn:
                continue
            mult = f32(f32(di["scale"]) * (f32(di.get("first_bn_multiplier", 10.0)) if i == first else 1.0))
            M, _, _, nm, nv, kap_m, kap_v = self._di_layer(i, self.T("val", op.tin))
            val += mult * float(nv + nm)
            bound += abs(mult) * TRAIN_C * (M + 8) * U * float(nm * kap_m + nv * kap_v)
        return val, bound + 4 * D53 * abs(val)

    def _features_term(self):
        fs = self.obj["features"]
        x = self.T("val", self.prog.ops[self._feature_op()].tin)
        diff = x.reshape(x.shape[0], -1) - fs["measured"].double().reshape(x.shape[0], -1)
        n, s = diff.numel(), f32(fs["scale"])
        sq = float(diff.pow(2).sum())
        return s * sq / n, abs(s) * (2 * U + n * D53) * sq / n + 4 * D53 * abs(s * sq / n)

    def check_terms(self, terms, value=None, G=None, x=None, raise_on_failure=True):
        """The objective terms ``terms`` (``Engine.last_terms()``) and the returned objective ``value`` of the last evaluation (see
        the module docstring).  ``G``: the matched gradient (default: the stored G); ``x``: what the image priors act on (default:
        the stored candidate / view, tensor 0).  Findings are reported with kind "terms" and the term's name as the sweep."""
        if self.seq:
            raise NotImplementedError("objective terms of token programs")
        o = self.obj
        G = G if G is not None else [self.Pm("G", j) for j in range(len(self.P))]
        x = x.double() if x is not None else self.T("val", 0)
        ref = {k: (0.0, 0.0) for k in TERMS}
        ref["match"] = self._match_term(G, o["kind"], o["scale"])
        ref["task_loss"] = self._task_loss_term()
        if o["tv"] is not None:
            ref["total_variation"] = self._tv_term(x)
        if o["norm"] is not None:
            ref["norm"] = self._norm_term(x)
        if o.get("orthogonality"):   # accumulated into the norm slot (after the norm prior, in double)
            v, b = orthogonality_relation(x)[:2]
            ref["norm"] = (ref["norm"][0] + v, ref["norm"][1] + b + D53 * abs(ref["norm"][0] + v))
        if o["di"] is not None:
            ref["deep_inversion"] = self._di_term()
        if o["features"] is not None:
            ref["features"] = self._features_term()
        for k in TERMS:
            r, b = ref[k]
            self._cmp(-1, k, k, torch.tensor(float(terms[k]), dtype=torch.float64), torch.tensor(r, dtype=torch.float64), b, kind="terms")
        if value is not None:   # assembled in double in this order: no rounding of its own to allow for
            phi = terms["match"] + terms["total_variation"] + terms["norm"] + terms["deep_inversion"] + terms["features"]
            tau = f32(o["task_regularization"])
            if tau != 0.0:
                phi += tau * terms["task_loss"]
            self._cmp(-1, "value", "objective = sum of the terms", torch.tensor(float(value), dtype=torch.float64),
                      torch.tensor(phi, dtype=torch.float64), 0.0, kind="terms")
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def check_score(self, score, kind, G=None, raise_on_failure=True):
        """``Engine.score(x, kind)`` (euclidean or cosine-similarity): the fp32 rounding of the match term with scale 1 of the
        G the scoring pass left (read afresh from the source; ``G``: the matched gradient of a multi-step engine, D)."""
        G = G if G is not None else [self.src.param("G", j).double() for j in range(len(self.P))]
        S, E = match_sums(G, self.g, kind)
        ref, bound = match_value(kind, S, E, 1.0)
        bound = bound + U * abs(ref) + 16 * D53 * (abs(ref) + 1.0)
        self._cmp(-1, kind, f"score ({kind})", torch.tensor(float(score), dtype=torch.float64), torch.tensor(ref, dtype=torch.float64),
                  bound, kind="score")
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings


class InterpreterSource:
    """Buffers of a float64 ``ProgramInterpreter.matching_gradient`` run; ``grad_x``: the full candidate gradient (priors and
    task term included, as the engine stores it in ``tangent_delta[0]``)."""

    def __init__(self, it, grad_x):
        self.it, self.V, self.grad_x = it, it.V, grad_x
        self.unwritten = set()

    def rounds_operands(self, i):
        return False

    def tensor(self, which, tid):
        it = self.it
        if which == "val":
            return it.a[tid]
        if which == "delta":
            return it.d_B.get(tid)
        if which == "tangent":
            return it.ta.get(tid)
        if tid == 0:
            return self.grad_x.reshape(it.a[0].shape)
        return it.d_T[tid] + it.inject.get(tid, 0)   # the engine adds the prior adjoints into the stored tangent delta

    def param(self, which, idx):
        return {"G": self.it.G, "v_operand": self.V, "W_operand": self.it.P}[which][idx]


class InterpreterStepSource:
    """Buffers of step k of a float64 ``program_interp.MultiStepInterpreter`` run, as the multi-step checker reads them."""

    def __init__(self, mi, k):
        self.it = mi.steps[k]
        self.has_tangent_G = k > 0
        self.unwritten = set()

    def rounds_operands(self, i):
        return False

    def tensor(self, which, tid):
        it = self.it
        if which == "tangent_delta":
            return it.gx if tid == 0 else it.d_T[tid]
        return InterpreterSource.tensor(self, which, tid)

    def param(self, which, idx):
        it = self.it
        return {"G": it.G, "v": it.U, "v_operand": it.U, "W_operand": it.P, "TG": getattr(it, "TG", None)}[which][idx]


class InterpreterGlue:
    """What the multi-step checker reads outside the steps, from a ``MultiStepInterpreter`` run: W_k / their operands (k = 0..K),
    D_k (k = 1..K), the whole candidate and its final gradient."""

    def __init__(self, mi, x, grad):
        self.x, self.grad, self.offsets, self.lr = x, grad, mi.offsets, mi.lr
        self.W, self.W_operand, self.D = mi.W, mi.W, {k: mi.D[k] for k in range(1, len(mi.D))}

    def shadowed(self, j):
        return False


class MultiStepChecker:
    """Layer-local check of every local step of a multi-step (FedAvg) evaluation, plus the glue between the steps.

    ``sources[k]`` is step k's buffer source: its forward / backward buffers (``val``, ``delta``, ``G`` = G_k) and those of its
    tangent sweeps (``tangent``, ``tangent_delta`` with the step's input gradient at tensor 0, ``v`` / ``v_operand`` = u_{k+1}, the
    direction step k used, ``TG`` = H_k u_{k+1} for k > 0).  ``glue`` provides ``W[k]`` / ``W_operand[k]`` (k = 0..K, lists in
    parameter order), ``D[k]`` (k = 1..K; missing entries are not checked), ``shadowed(j)`` (parameter j has a TF32 operand
    form), ``x`` (the whole candidate), ``grad`` (its final gradient), ``offsets`` (first image of each step's slice) and ``lr``
    (the step size as the source applied it: the engine's is the fp32 value).
    ``labels[k]``: step k's labels; ``objective``: as for ``SweepChecker`` (the priors act on the final assembly only)."""

    def __init__(self, prog, bn, g, labels, objective, sources, glue):
        self.prog, self.bn, self.g, self.labels = prog, bn, [t.detach().double() for t in g], labels
        self.obj, self.src, self.glue = objective, sources, glue
        self.K = len(sources)
        self.findings, self.ratios, self.off_grid = [], {}, set()

    def _step_objective(self):
        o = dict(self.obj)
        o.update(tv=None, norm=None, di=None, features=None, orthogonality=None, task_regularization=0.0)
        return o

    def _absorb(self, chk, step):
        for f in chk.findings:
            f.step = step if f.step is None else f.step
            self.findings.append(f)
        for key, r in chk.ratios.items():
            self.ratios[key] = max(self.ratios.get(key, 0.0), r)
        chk.findings, chk.ratios = [], {}

    def check(self, raise_on_failure=True):
        n = len(self.g)
        self.steps = []
        for k in range(self.K):
            W = [w.double() for w in self.glue.W[k]]
            chk = SweepChecker(self.prog, W, self.bn, self.g, self.labels[k], self._step_objective(), self.src[k])
            chk.forward()
            chk.backward()
            chk.tangent_forward()
            chk.tangent_backward()
            if k > 0:
                chk.tangent_G()
            self.off_grid.update({(k, i) for i in chk.off_grid})
            self._absorb(chk, k)
            self.steps.append(chk)
        self.glue_relations(n)
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def _last_step_checker(self):
        last = self.K - 1
        return SweepChecker(self.prog, [w.double() for w in self.glue.W[last]], self.bn, self.g, self.labels[last], self.obj,
                            self.src[last])

    def check_terms(self, terms, value=None, raise_on_failure=True):
        """The objective terms of a full multi-step evaluation: match from D_K, task loss and DeepInversion from the last local
        step's buffers, TV / norm on the whole candidate (see ``SweepChecker.check_terms``)."""
        chk = self._last_step_checker()
        chk.check_terms(terms, value, G=[d.double() for d in self.glue.D[self.K]], x=self.glue.x, raise_on_failure=False)
        self._absorb(chk, None)
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def check_score(self, score, kind, D, raise_on_failure=True):
        """``Engine.score`` of a multi-step engine: the match of ``D`` (``debug_step_param("D", ...)`` after the scoring pass)."""
        chk = self._last_step_checker()
        chk.check_score(score, kind, G=[d.double() for d in D], raise_on_failure=False)
        self._absorb(chk, None)
        if raise_on_failure and self.findings:
            raise SweepCheckError("\n".join(repr(f) for f in self.findings[:20]))
        return self.findings

    def _cmp(self, step, sweep, what, y, ref, bound):
        chk = self.steps[0]
        chk._cmp(-1, sweep, what, y.double(), ref, bound, kind="glue")
        self._absorb(chk, step)

    def glue_relations(self, n):
        lr, K, gl = self.glue.lr, self.K, self.glue
        G = [[self.src[k].param("G", j).double() for j in range(n)] for k in range(K)]
        for k in range(K):
            for j in range(n):
                # W_{k+1} = fl(W_k - lr G_k) (fp32 lr; one product, one sum); its TF32 operand form is rna(W_{k+1}) exactly
                Wk, Wn = gl.W[k][j].double(), gl.W[k + 1][j].double()
                step = lr * G[k][j]
                self._cmp(k, "W", f"W_{k + 1}[{j}] = W_{k} - lr G_{k}", Wn, Wk - step, 2 * U * (Wk.abs() + step.abs()))
                Wo = gl.W_operand[k + 1][j].double()
                self._cmp(k, "Wt", f"W_operand_{k + 1}[{j}] (TF32 shadow)", Wo, rna(Wn) if gl.shadowed(j) else Wn, 0.0)
                if k + 1 in gl.D and (k == 0 or k in gl.D):
                    Dk = gl.D[k][j].double() if k > 0 else torch.zeros_like(Wk)
                    Dn = gl.D[k + 1][j].double()
                    self._cmp(k, "D", f"D_{k + 1}[{j}] = D_{k} - lr G_{k}", Dn, Dk - step, 2 * U * (Dk.abs() + step.abs()))
        # the direction of the last step: make_v(D_K, g), the direction relation of the single-step check with G := D_K
        last = self.K - 1

        class _DirSource:
            def __init__(s, base):
                s.base = base

            def param(s, which, idx):
                return gl.D[K][idx] if which == "G" else s.base.param(which, idx)

        d = SweepChecker(self.prog, [w.double() for w in gl.W[0]], self.bn, self.g, self.labels[0], self.obj, _DirSource(self.src[last]))
        d.direction()
        for f in d.findings:
            f.step = last
        self.findings += d.findings
        for key, r in d.ratios.items():
            self.ratios[key] = max(self.ratios.get(key, 0.0), r)
        for k in range(K):
            u = [self.src[k].param("v", j).double() for j in range(n)]
            for j in range(n):   # the TF32 shadow of the direction step k used
                uo = self.src[k].param("v_operand", j).double()
                self._cmp(k, "Ut", f"v_operand[{j}] (TF32 shadow of u_{k + 1})", uo, rna(u[j]) if gl.shadowed(j) else u[j], 0.0)
            if k == 0:
                continue
            # u_k = fl(u_{k+1} - lr H_k u_{k+1}): the direction step k - 1 used
            un = [self.src[k - 1].param("v", j).double() for j in range(n)]
            for j in range(n):
                step = lr * self.src[k].param("TG", j).double()
                self._cmp(k, "U", f"u_{k}[{j}] = u_{k + 1} - lr TG_{k}", un[j], u[j] - step, 2 * U * (u[j].abs() + step.abs()))
        self._final_assembly()

    def _final_assembly(self):
        """gradx = sum_k -lr gradx_step_k scattered onto step k's slice (slices of wrapped steps accumulate) + the priors."""
        gl, lr = self.glue, self.glue.lr
        x = gl.x.double()
        ref, mag, cnt = torch.zeros_like(x), torch.zeros_like(x), torch.zeros_like(x)
        for k in range(self.K):
            gs = lr * self.src[k].tensor("tangent_delta", 0).double()
            o, b = gl.offsets[k], gs.shape[0]
            ref[o:o + b] -= gs
            mag[o:o + b] += gs.abs()
            cnt[o:o + b] += 1
        bound = (cnt + 2) * U2 * mag
        o = self.obj
        if o.get("tv") is not None or o.get("norm") is not None:
            from oracle.program_interp import image_prior
            _, gp = image_prior(x, o)
            ref = ref + gp
            tvs = o["tv"]["scale"] if o.get("tv") is not None else 0.0
            bound = bound + 64 * U * (gp.abs() + 4 * tvs / x.numel())
        if o.get("orthogonality"):
            _, _, og, eog = orthogonality_relation(x)
            ref = ref + og
            bound = bound + eog + 2 * U * (ref.abs() + og.abs())
        self._cmp(None, "GX", "candidate gradient (sum over the local steps + priors)", gl.grad.double(), ref, bound + U * ref.abs())
