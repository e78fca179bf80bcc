"""``OptimizationJointAttacker`` on the sm_90a engine: data and labels are optimised together ("deep leakage from
gradients"-style attacks; reference ``attacks/optimization_with_label_attack.py:38-230``, presets ``deepleakage.yaml``).

The label candidate is a second leaf ``[N, classes]``; the closure hands ``labels.softmax(-1)`` to the task loss as class
probabilities (:154), back-propagates the objective onto both leaves (:162), post-processes both gradients separately
(:164-186) and one optimiser steps both (:108).  On the engine one closure evaluation is one pass of the four sweeps with
soft targets in the cross-entropy (``bre_engine_load_soft_labels``); the gradient w.r.t. the probabilities falls out of the
tangent logits of that same pass (``bre_engine_label_gradient``: the matching term sees the probabilities only through
``dL/dq = -log_softmax(z)/N``) and is chained through the softmax here.  The loop is host-driven (two small leaves, any
torch-style optimiser incl. L-BFGS); the fused on-device step of the single-leaf attacker is not used.

Classification models (``deepleakage.yaml``) and causal language models (``tag.yaml``, SURVEY section 8 row a15, BASELINE
config 5: the candidate is the embedding sequence, the label leaf holds logits over the vocabulary for every position).
"""
import logging
import math
import time

import torch

from .. import dist as bdist
from ..config import cfg_get
from ..schedule import lr_table
from . import host, lbfgs
from .host_optim import OPTIMIZERS as _OPTIMIZERS
from .host_optim import LeafOptimizer as _LeafOptimizer
from .optimization_attack import OptimizationBasedAttacker

log = logging.getLogger(__name__)

class OptimizationJointAttacker(OptimizationBasedAttacker):
    """Optimises jointly for candidate data and labels on the engine."""

    _LOSSES = ("CrossEntropyLoss", "CausalLoss")   # CausalLoss: token models (tag.yaml), see _prepare_text

    # optimization_with_label_attack.py:43-51 -- the "recovered labels" are a template of label logits
    def _label_template(self, shared_data, metadata):
        n = shared_data[0]["metadata"]["num_data_points"]
        if metadata["task"] != "classification":
            raise NotImplementedError("joint optimisation of token labels (text models) is not implemented by the engine")
        return host.initialize_data(self.cfg.init, [n, metadata.classes], self.dm, self.ds, self.setup)

    # ---- text models (tag.yaml, BASELINE config 5) ----------------------------------------------------------------
    # The closure of this path on the engine (compiler.compile_transformer program, all four sweeps, soft token labels) is
    # verified on the GPU against the reference's TAG closure at miniature and full size, the attacker-level glue below
    # (prologue, loop, scoring, token recovery) against the reference trajectory (tests/test_tokens_gpu.py); its host pieces
    # are additionally tested on the CPU against the reference (tests/test_install_dropin.py, tests/test_host_loops_cpu.py).
    def _prepare_text(self, server_payload, shared_data):
        from collections import defaultdict

        stats = defaultdict(list)
        shared_data = [dict(d, gradients=list(d["gradients"])) for d in shared_data]
        metadata = server_payload[0]["metadata"]
        self.data_shape = list(metadata.shape)
        self.dm, self.ds = host.preprocessing_constants(metadata, self.setup)
        rec_models = host.construct_models(self.model_template, server_payload, shared_data, self.setup)
        shared_data = host.cast_shared_data(shared_data, self.setup["dtype"])
        self.embeddings, dim = host.prepare_for_text_data(rec_models, shared_data, cfg_get(self.cfg, "text_strategy", "run-embedding"))
        self.data_shape = [*self.data_shape, dim]                       # base_attack.py:113-114
        self._rec_models = rec_models
        n = shared_data[0]["metadata"]["num_data_points"]
        template = host.initialize_data(self.cfg.init, [n, self.data_shape[0], metadata.vocab_size], self.dm, self.ds, self.setup)
        if self.cfg.normalize_gradients:
            shared_data = host.normalize_gradients(shared_data)
        return rec_models, template, stats, shared_data

    def _get_text_engine(self, rec_models, shared_data):
        from .. import compiler
        from ..engine import Engine

        n = shared_data[0]["metadata"]["num_data_points"]
        T, d = self.data_shape
        prog = compiler.compile_transformer(rec_models[0], n, T)
        if self._engine is not None:
            self._engine.close()
        eng = Engine(None, (n * T, d, 1, 1), self.cfg, self.setup["device"], backend=self.backend, program=prog)
        eng.load_model(params=[p.detach() for p in rec_models[0].parameters()])
        tw = None
        if self.cfg.objective.type == "tag-euclidean":  # objectives.py:115-124
            L = len(shared_data[0]["gradients"])
            scheme = cfg_get(self.cfg.objective, "scale_scheme", "linear")
            if scheme == "linear":
                tw = torch.arange(L, 0, -1, dtype=torch.float32) / L
            elif scheme == "exp":
                tw = torch.arange(L, 0, -1, dtype=torch.float32).softmax(dim=0)
                tw = tw / tw[0]
            else:
                tw = torch.ones(L)
        eng.load_targets(shared_data[0]["gradients"], torch.zeros(n * T, dtype=torch.long), tensor_weights=tw)
        self._engine = eng
        return eng

    def _reconstruct_text(self, server_payload, shared_data, server_secrets, initial_data, dryrun):
        clock, t0 = self.last_timing, time.perf_counter()
        clock.clear()
        rec_models, labels, stats, shared_data = self._prepare_text(server_payload, shared_data)
        clock["prologue"], t0 = time.perf_counter() - t0, time.perf_counter()
        if len(rec_models) != 1 or self.regularizers:
            raise NotImplementedError("text models: one model query, no regularisers (the reference's TAG / DLG presets configure none)")
        engine = self._get_text_engine(rec_models, shared_data)
        clock["engine"], t0 = time.perf_counter() - t0, time.perf_counter()
        num_trials = self.cfg.restarts.num_trials
        rank, world = bdist.rank_and_world()
        scores = torch.full((num_trials,), float("inf"))
        candidate_solutions = [None] * num_trials
        shape = [shared_data[0]["metadata"]["num_data_points"], *self.data_shape]
        hard_labels = labels.argmax(dim=-1)                              # :67 (of the template, reference behaviour)
        for trial in range(num_trials):
            candidate = host.initialize_data(self.cfg.init, shape, self.dm, self.ds, self.setup)
            candidate_labels = host.initialize_data(self.cfg.init, list(labels.shape), self.dm, self.ds, self.setup)
            if initial_data is not None:
                candidate = initial_data.detach().clone().to(**self.setup)
            if trial % world != rank:
                continue
            data, _ = self._run_joint_trial(engine, candidate, candidate_labels, stats, trial, dryrun)
            candidate_solutions[trial] = data
            ts = time.perf_counter()
            q_hard = torch.nn.functional.one_hot(hard_labels, labels.shape[-1]).to(**self.setup)
            engine.load_soft_labels(q_hard.reshape(-1, labels.shape[-1]))
            scores[trial] = engine.score(data.reshape(-1, data.shape[-1], 1, 1), self.cfg.restarts.scoring)
            clock["trial_score"] = clock.get("trial_score", 0.0) + time.perf_counter() - ts
        clock["trials"], t0 = time.perf_counter() - t0, time.perf_counter()
        optimal_solution = self._select_optimal_reconstruction(candidate_solutions, scores, stats, shape)
        clock["select"], t0 = self.last_select_seconds, time.perf_counter()
        reconstructed = dict(data=optimal_solution, labels=hard_labels)
        reconstructed = host.postprocess_text_data(reconstructed, self.embeddings[0]["weight"].detach(), self.cfg.token_recovery)
        clock["token_recovery"] = time.perf_counter() - t0
        reconstructed["raw_embeddings"] = optimal_solution                # :80
        return reconstructed, stats

    def prepare_attack(self, server_payload, shared_data):
        if shared_data[0]["metadata"]["labels"] is not None:  # :56-60
            raise ValueError(
                "Joint optimization only makes sense if no labels are provided. Switch to attack.attack_type=optimization instead"
            )
        metadata = server_payload[0]["metadata"]
        # the base class would run a label-recovery strategy; the joint attacker replaces it by the template (:43-51)
        placeholder = shared_data[0]["metadata"]["num_data_points"]
        shared = [dict(d) for d in shared_data]
        shared[0] = dict(shared[0], metadata=dict(shared[0]["metadata"], labels=torch.zeros(placeholder, dtype=torch.long)))
        rec_models, _, stats, shared = super().prepare_attack(server_payload, shared)
        shared[0]["metadata"]["labels"] = None
        template = self._label_template(shared, metadata)
        return rec_models, template, stats, shared

    def reconstruct(self, server_payload, shared_data, server_secrets=None, initial_data=None, dryrun=False):
        if getattr(server_payload[0]["metadata"], "modality", "vision") == "text":
            if shared_data[0]["metadata"]["labels"] is not None:
                raise ValueError("Joint optimization only makes sense if no labels are provided. Switch to attack.attack_type=optimization instead")
            return self._reconstruct_text(server_payload, shared_data, server_secrets, initial_data, dryrun)
        from . import augment

        if augment.has_view_stages(self.cfg):   # the joint loop does not run the view pipeline: refuse rather than skip
            raise NotImplementedError("zoom / centerzoom / focus / antialias are not implemented for the joint attacker by the engine")
        rec_models, labels, stats, shared_data = self.prepare_attack(server_payload, shared_data)
        if any(True for _ in self.regularizers) and any(k in ("deep_inversion", "features") for k, _ in self.regularizers):
            raise NotImplementedError("feature / DeepInversion priors are not implemented for the joint attacker")
        engine = self._get_engine(rec_models, shared_data, torch.zeros(labels.shape[0], dtype=torch.long))
        num_trials = self.cfg.restarts.num_trials
        rank, world = bdist.rank_and_world()
        scores = torch.full((num_trials,), float("inf"))
        candidate_solutions = [None] * num_trials
        shape = [shared_data[0]["metadata"]["num_data_points"], *self.data_shape]
        hard_labels = labels.argmax(dim=-1)  # :67 -- of the template, not of the optimised labels (reference behaviour)
        try:
            for trial in range(num_trials):
                candidate = host.initialize_data(self.cfg.init, shape, self.dm, self.ds, self.setup)
                candidate_labels = host.initialize_data(self.cfg.init, list(labels.shape), self.dm, self.ds, self.setup)
                if initial_data is not None:
                    candidate = initial_data.detach().clone().to(**self.setup)
                if trial % world != rank:
                    continue
                data, _ = self._run_joint_trial(engine, candidate, candidate_labels, stats, trial, dryrun)
                candidate_solutions[trial] = data
                scores[trial] = self._score_joint(engine, data, hard_labels)
        except KeyboardInterrupt:
            print("Trial procedure manually interruped.")
        optimal_solution = self._select_optimal_reconstruction(candidate_solutions, scores, stats, shape)
        reconstructed_data = dict(data=optimal_solution, labels=hard_labels)
        if server_secrets is not None and "ClassAttack" in server_secrets:
            true_num_data = server_secrets["ClassAttack"]["true_num_data"]
            reconstructed_data["data"] = torch.zeros([true_num_data, *self.data_shape], **self.setup)
            reconstructed_data["data"][server_secrets["ClassAttack"]["target_indx"]] = optimal_solution
            reconstructed_data["labels"] = server_secrets["ClassAttack"]["all_labels"]
        return reconstructed_data, stats

    # ------------------------------------------------------------------------------------------------
    def _closure(self, engine, x, ell, iteration, lr):
        """optimization_with_label_attack.py:145-189 -> (objective, processed d/dx, processed d/dlabels, raw pair)."""
        q = ell.softmax(dim=-1)
        if ell.dim() == 3:   # token models: the engine works on rows = batch * seq_len
            engine.load_soft_labels(q.reshape(-1, q.shape[-1]))
            value, gx = engine.objective_and_gradient(x.reshape(-1, x.shape[-1], 1, 1))
            gx = gx.reshape(x.shape)
        else:
            engine.load_soft_labels(q)
            value, gx = engine.objective_and_gradient(x)
        gq = engine.label_gradient(tuple(ell.shape))
        gl = q * (gq - (q * gq).sum(dim=-1, keepdim=True))   # chain through the softmax (autograd does this at :162)
        raw = (gx, gl)
        opt = self.cfg.optim
        gx = lbfgs.postprocess_gradient(gx, opt, iteration, lr)
        gl = lbfgs.postprocess_gradient(gl, opt, iteration, lr)
        return float(value), gx, gl, raw

    def _run_joint_trial(self, engine, candidate, candidate_labels, stats, trial, dryrun=False, iterations=None):
        """optimization_with_label_attack.py:89-143.  Adam / AdamW / SGD trials run entirely on the device (both leaves stepped
        by the engine's fused kernels from one CUDA graph, ``bre_engine_begin_joint_trial``), and so do L-BFGS trials of
        classification models without augmentations or Langevin noise (``bre_engine_begin_lbfgs_trial``); token models with L-BFGS
        and engine stand-ins without those entry points are driven from the host."""
        opt = self.cfg.optim
        T = int(opt.max_iterations)
        table = lr_table(opt.step_size, cfg_get(opt, "step_size_decay"), cfg_get(opt, "warmup", 0), T)
        name = str(opt.optimizer).lower()
        if not getattr(self, "host_driven", False) and (
                (name in _OPTIMIZERS and hasattr(engine, "begin_joint_trial"))
                or (name == "l-bfgs" and candidate_labels.dim() == 2 and self._lbfgs_on_device(engine))):
            return self._run_joint_trial_device(engine, candidate, candidate_labels, stats, trial, table, dryrun, iterations)
        x = candidate.detach().clone().contiguous()
        ell = candidate_labels.detach().clone().contiguous()
        best, best_l, fmin = x.clone(), ell.clone(), float("inf")
        dm, ds = self.dm.to(x.device), self.ds.to(x.device)
        lo, hi = -dm / ds, (1 - dm) / ds
        if name == "l-bfgs":
            flat = torch.cat([x.view(-1), ell.view(-1)])   # torch's L-BFGS treats all leaves as one flat vector
            x, ell = flat[: x.numel()].view_as(x), flat[x.numel():].view_as(ell)
            optimizer = lbfgs.DeviceLBFGS(flat)
        elif name in _OPTIMIZERS:
            optimizer = _LeafOptimizer([x, ell], name)
        else:
            raise ValueError(f"Invalid optimizer {opt.optimizer} given.")
        total = 1 if dryrun else (T if iterations is None else iterations)
        history = []
        for it in range(total):
            lr = float(table[it])
            if name == "l-bfgs":
                def closure():
                    val, gx, gl, _ = self._closure(engine, x, ell, it, lr)
                    return val, torch.cat([gx.reshape(-1), gl.reshape(-1)])

                value = optimizer.step(closure, lr)
            else:
                value, gx, gl, _ = self._closure(engine, x, ell, it, lr)
                optimizer.step([gx, gl], lr)
            if cfg_get(opt, "boxed", False):
                torch.max(torch.min(x, hi, out=x), lo, out=x)
            if value < fmin:
                fmin = value
                best.copy_(x)
                best_l.copy_(ell)
            if not math.isfinite(value):
                log.info(f"Recovery loss is non-finite in iteration {it}. Cancelling reconstruction!")
                break
            history.append(value)
        stats[f"Trial_{trial}_Val"].extend(history)
        self._last_joint_state = (x.detach().clone(), ell.detach().clone())
        return best.detach(), best_l.detach()

    def _run_joint_trial_device(self, engine, candidate, candidate_labels, stats, trial, table, dryrun, iterations):
        x = candidate.detach().contiguous()
        if candidate_labels.dim() == 3:      # token models: the engine works on rows = batch * seq_len
            x = x.reshape(-1, x.shape[-1], 1, 1)
        clock, t0 = self.last_timing, time.perf_counter()
        if str(self.cfg.optim.optimizer).lower() == "l-bfgs":   # data and labels as one flat vector, as torch's L-BFGS sees them
            engine.begin_lbfgs_trial(x, table, label_logits=candidate_labels.detach().contiguous(), trial=trial)
        else:
            engine.begin_joint_trial(x, candidate_labels.detach().contiguous(), table, trial=trial)
        clock["trial_begin"] = clock.get("trial_begin", 0.0) + time.perf_counter() - t0
        t0 = time.perf_counter()
        T = int(self.cfg.optim.max_iterations)
        total = 1 if dryrun else (T if iterations is None else iterations)
        callback = int(cfg_get(self.cfg.optim, "callback", 0) or 0)
        done = 0
        while done < total:
            n = min(callback if callback > 0 else total, total - done) if done > 0 else 1
            engine.run(n)
            done += n
            st = engine.status()                      # one host sync per `callback` iterations
            if done == 1:
                clock["trial_first_iteration"] = clock.get("trial_first_iteration", 0.0) + time.perf_counter() - t0
            if st["stopped"]:
                log.info(f"Recovery loss is non-finite in iteration {st['recorded']}. Cancelling reconstruction!")
                break
        engine.sync()
        clock["trial_iterations"] = clock.get("trial_iterations", 0.0) + time.perf_counter() - t0
        t0 = time.perf_counter()
        stats[f"Trial_{trial}_Val"].extend(engine.history().tolist())
        best = engine.best().reshape(candidate.shape)
        best_l = engine.joint_labels(best=True)
        self._last_joint_state = (engine.candidate().reshape(candidate.shape), engine.joint_labels(best=False))
        clock["trial_readback"] = clock.get("trial_readback", 0.0) + time.perf_counter() - t0
        return best.detach(), best_l.detach()

    def _score_joint(self, engine, candidate, hard_labels):
        """optimization_with_label_attack.py:207-221: a fresh objective with the template's arg-max labels."""
        engine.load_soft_labels(None)
        engine.set_labels(hard_labels)
        return self._score_trial(engine, candidate)
