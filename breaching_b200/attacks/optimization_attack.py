"""``OptimizationBasedAttacker`` served by the sm_90a engine.

API-compatible with the reference class of the same name (``attacks/optimization_based_attack.py:24-218``):
``prepare_attack(model, loss_fn, cfg_attack, setup)`` builds it, ``reconstruct(server_payload, shared_data,
server_secrets, initial_data, dryrun)`` returns ``(dict(data=..., labels=...), stats)``.

What differs is *where* the trial runs: ``_run_trial`` hands the candidate to ``breaching_b200.engine.Engine``,
which executes all iterations on the GPU from a captured CUDA graph; the host only polls a status word every
``cfg.optim.callback`` iterations for the log line (the reference synchronises three times per iteration,
``:119,:131,:135``).  Independent trials are sharded round-robin over the ranks of an initialised
``torch.distributed`` process group and the winner is selected with one MIN all-reduce (``dist.py``).
"""
import copy
import logging
import time
from collections import defaultdict

import torch

from .. import dist as bdist
from ..config import cfg_get
from ..engine import OBJECTIVES, PEARLMUTTER, Engine, EngineError
from ..schedule import lr_table
from . import host

log = logging.getLogger(__name__)

_REGULARIZERS = ("total_variation", "orthogonality", "norm", "deep_inversion", "features")  # regularizers.py:233-239


def _loss_name(loss_fn):
    return getattr(loss_fn, "original_name", None) or type(loss_fn).__name__


class _EngineSum:
    """Several engines behind the two calls the host-driven loops use: objective and candidate gradient are summed over the
    (model, update) pairs (optimization_based_attack.py:157-160); only the first engine carries the image priors."""

    def __init__(self, engines):
        self.engines = engines

    def objective_and_gradient(self, x):
        total, grad = 0.0, None
        for eng in self.engines:
            val, g = eng.objective_and_gradient(x)
            total += float(val)
            grad = g if grad is None else grad.add_(g)
        return total, grad

    def score(self, candidate, scoring):
        return sum(eng.score(candidate, scoring) for eng in self.engines)


def _refuse_view_stages_off_device(cfg, n_models):
    """The host-driven loops (L-BFGS, several model queries) do not run the view pipeline; refuse shape-changing views there rather
    than skip them."""
    if str(cfg.optim.optimizer).lower() == "l-bfgs" or n_models > 1:
        raise NotImplementedError("zoom / centerzoom / focus / antialias are not implemented for L-BFGS or multi-query attacks by the engine")


class OptimizationBasedAttacker:
    """Implements the optimisation-based attacks of the reference on the engine."""

    _LOSSES = ("CrossEntropyLoss",)

    def __init__(self, model, loss_fn, cfg_attack, setup=dict(dtype=torch.float, device=torch.device("cpu"))):
        self.cfg = cfg_attack
        self.setup = dict(device=torch.device(setup["device"]), dtype=getattr(torch, cfg_attack.impl.dtype))
        self.backend = setup.get("backend")  # optional extension: "tc" (default, TF32 tensor cores) or "simt" (fp32)
        self.model_template = copy.deepcopy(model)
        self.loss_fn = copy.deepcopy(loss_fn)

        if cfg_attack.objective.type not in OBJECTIVES and cfg_attack.objective.type not in PEARLMUTTER:
            raise ValueError(f"Unknown objective type {self.cfg.objective.type} given.")  # reference :31
        self.regularizers = []
        reg = cfg_get(self.cfg, "regularization")
        if reg is not None:
            for key in reg.keys():
                if reg[key].scale > 0:
                    if key not in _REGULARIZERS:
                        raise KeyError(key)
                    self.regularizers.append((key, dict(reg[key])))
        self._aug_plans = {}   # candidate augmentations (attacks/augment.py), built per batch size on first use
        self.last_timing = {}  # seconds per phase of the last reconstruct() call
        self.last_select_seconds = 0.0
        if self.setup["dtype"] != torch.float32:
            raise NotImplementedError("the engine computes in fp32 (cfg.impl.dtype=float)")
        if cfg_get(self.cfg.impl, "mixed_precision", False):
            raise NotImplementedError("impl.mixed_precision is not implemented by the engine")
        if self.setup["device"].type != "cuda":
            raise EngineError("the engine needs setup['device'] to be a CUDA device (there is no CPU fallback)")
        if _loss_name(self.loss_fn) not in self._LOSSES:
            raise NotImplementedError(f"loss {_loss_name(self.loss_fn)} is not implemented by the engine ({', '.join(self._LOSSES)} only)")
        self._engine = None
        self._engine_key = None

    def __repr__(self):
        n = "\n"
        regs = (n + " " * 18).join(f"{k}: {v}" for k, v in self.regularizers)
        opt = (n + " " * 8).join(f"{key}: {val}" for key, val in self.cfg.optim.items())
        return f"""Attacker (of type {self.__class__.__name__}, H100 engine) with settings:
    Hyperparameter Template: {self.cfg.type}

    Objective: {self.cfg.objective.type} with scale={cfg_get(self.cfg.objective, 'scale', 1.0)} and task reg={cfg_get(self.cfg.objective, 'task_regularization', 0.0)}
    Regularizers: {regs}
    Augmentations:

    Optimization Setup:
        {opt}
        """

    # ------------------------------------------------------------------------------------------------
    def prepare_attack(self, server_payload, shared_data):
        """base_attack.py:43-74."""
        stats = defaultdict(list)
        shared_data = shared_data.copy()
        server_payload = server_payload.copy()
        metadata = server_payload[0]["metadata"]
        self.data_shape = metadata.shape
        self.dm, self.ds = host.preprocessing_constants(metadata, self.setup)
        if getattr(metadata, "modality", "vision") == "text":
            raise NotImplementedError("text modality is not implemented by the engine")
        rec_models = host.construct_models(self.model_template, server_payload, shared_data, self.setup)
        shared_data = host.cast_shared_data(shared_data, self.setup["dtype"])
        self._rec_models = rec_models
        if shared_data[0]["metadata"]["labels"] is None:
            labels = host.recover_labels(self.cfg.label_strategy, shared_data, self.setup, self.data_shape)
        else:
            labels = shared_data[0]["metadata"]["labels"].clone()
        if self.cfg.normalize_gradients:
            shared_data = host.normalize_gradients(shared_data)
        return rec_models, labels, stats, shared_data

    def _get_engine(self, rec_models, shared_data, labels, index=0, cfg=None, data_shape=None, primary=True, for_scoring=False):
        """Engine for model / payload ``index`` (``cfg`` overrides the attack config, used for the extra queries; ``data_shape``
        overrides the candidate's per-example shape and ``primary=False`` builds an additional engine next to the attacker's main
        one -- both used by the multi-scale attacker's stages).  The program is compiled at the shape the model sees: the view's
        (attacks/augment.py ``view_shape``).  ``for_scoring=True`` builds the scoring engine of a resizing view instead: compiled at
        the candidate's shape, and without a Langevin noise seed (it never steps, so it draws nothing from the global RNG)."""
        if len(rec_models) != 1 and cfg is None:
            raise NotImplementedError("use _get_engines for several model queries")
        cfg = self.cfg if cfg is None else cfg
        local = shared_data[index]["metadata"]["local_hyperparams"]
        model = rec_models[index]
        n = shared_data[index]["metadata"]["num_data_points"]
        # FedAvg (objectives.py:48-72): the layer program is compiled for one local step's batch.  task_regularization and
        # deep_inversion act on the last local step; the features prior is refused by Engine.set_local_steps (see its docstring)
        shape = (n if local is None else int(local["data_per_step"]), *(self.data_shape if data_shape is None else data_shape))
        if not for_scoring and local is None:
            from . import augment

            if augment.has_view_stages(cfg):
                _refuse_view_stages_off_device(cfg, len(rec_models))
            shape = augment.view_shape(cfg, shape)
        seed = int(torch.randint(0, 2 ** 31 - 1, (1,)).item()) if cfg_get(self.cfg.optim, "langevin_noise", 0.0) and not for_scoring else 0
        if self._engine is not None and index == 0 and primary:
            self._engine.close()
            for eng in getattr(self, "_score_engines", {}).values():
                eng.close()
            self._score_engines = {}
        # setup["backend"]: "tc" (TF32 tensor cores, default = torch's cuDNN-TF32 numerics) or "simt" (fp32, = allow_tf32 False)
        eng = Engine(model, shape, cfg, self.setup["device"], noise_seed=seed, backend=self.backend)
        eng.load_model()
        tw = None
        if self.cfg.objective.type == "tag-euclidean":  # objectives.py:115-124
            L = len(shared_data[index]["gradients"])
            scheme = cfg_get(self.cfg.objective, "scale_scheme", "linear")
            if scheme == "linear":
                tw = torch.arange(L, 0, -1, dtype=torch.float32) / L
            elif scheme == "exp":
                tw = torch.arange(L, 0, -1, dtype=torch.float32).softmax(dim=0)
                tw = tw / tw[0]
            else:
                tw = torch.ones(L)
        mean = self.dm.flatten() if self.dm.numel() > 1 else self.dm.flatten().expand(self.data_shape[0])
        std = self.ds.flatten() if self.ds.numel() > 1 else self.ds.flatten().expand(self.data_shape[0])
        step_labels = labels if local is None else local["labels"][0]
        eng.load_targets(shared_data[index]["gradients"], step_labels, mean=mean, std=std, tensor_weights=tw)
        if local is not None:
            eng.set_local_steps(n, int(local["steps"]), float(local["lr"]), [l for l in local["labels"][: int(local["steps"])]])
        if any(k == "features" for k, _ in self.regularizers):
            eng.load_feature_targets(host.measured_features(shared_data, labels)[0])
        if index == 0 and primary:
            self._engine = eng
        return eng

    def _get_engines(self, rec_models, shared_data, labels):
        """One engine per (model, update) pair of a multi-query attack (optimization_based_attack.py:157-160: the objective
        is summed over ``zip(rec_model, shared_data)``, the regularisers are added once)."""
        if any(d["metadata"]["local_hyperparams"] is not None for d in shared_data):
            raise NotImplementedError("multi-step local updates with several model queries are not implemented by the engine")
        if any(k in ("deep_inversion", "features") for k, _ in self.regularizers):
            raise NotImplementedError("DeepInversion / feature priors with several model queries are not implemented by the engine")
        no_priors = copy.deepcopy(self.cfg)
        reg = cfg_get(no_priors, "regularization")
        if reg is not None:
            for key in reg.keys():
                reg[key].scale = 0.0
        for eng in getattr(self, "_extra_engines", []):
            eng.close()
        first = self._get_engine(rec_models, shared_data, labels, 0, self.cfg)
        self._extra_engines = [self._get_engine(rec_models, shared_data, labels, i, no_priors) for i in range(1, len(rec_models))]
        return [first] + self._extra_engines

    def reconstruct(self, server_payload, shared_data, server_secrets=None, initial_data=None, dryrun=False):
        # wall-clock seconds per phase of the last call (host clock, no extra device syncs: asynchronous work lands in the phase
        # that first waits for it): prologue = prepare_attack, engine = compile + create + uploads, trials, select
        clock, t0 = self.last_timing, time.perf_counter()
        clock.clear()
        rec_models, labels, stats, shared_data = self.prepare_attack(server_payload, shared_data)
        clock["prologue"], t0 = time.perf_counter() - t0, time.perf_counter()
        multi = len(rec_models) > 1
        engine = _EngineSum(self._get_engines(rec_models, shared_data, labels)) if multi else self._get_engine(rec_models, shared_data, labels)
        self._score_context = (rec_models, shared_data, labels)
        clock["engine"], t0 = time.perf_counter() - t0, time.perf_counter()
        num_trials = self.cfg.restarts.num_trials
        rank, world = bdist.rank_and_world()
        scores = torch.full((num_trials,), float("inf"))
        candidate_solutions = [None] * num_trials
        shape = [shared_data[0]["metadata"]["num_data_points"], *self.data_shape]
        try:
            for trial in range(num_trials):
                # every rank draws every initialisation in reference order (base_attack.py:226-230), keeps its own
                candidate = host.initialize_data(self.cfg.init, shape, self.dm, self.ds, self.setup)
                if initial_data is not None:
                    candidate = initial_data.detach().clone().to(**self.setup)
                if trial % world != rank:
                    continue
                candidate_solutions[trial] = self._run_trial(engine, candidate, stats, trial, dryrun)
                scores[trial] = self._score_trial(engine, candidate_solutions[trial])
        except KeyboardInterrupt:
            print("Trial procedure manually interruped.")
        clock["trials"] = time.perf_counter() - t0
        optimal_solution = self._select_optimal_reconstruction(candidate_solutions, scores, stats, shape)
        clock["select"] = self.last_select_seconds
        reconstructed_data = dict(data=optimal_solution, labels=labels)
        if server_secrets is not None and "ClassAttack" in server_secrets:  # :82-87
            true_num_data = server_secrets["ClassAttack"]["true_num_data"]
            reconstructed_data["data"] = torch.zeros([true_num_data, *self.data_shape], **self.setup)
            reconstructed_data["data"][server_secrets["ClassAttack"]["target_indx"]] = optimal_solution
            reconstructed_data["labels"] = server_secrets["ClassAttack"]["all_labels"]
        return reconstructed_data, stats

    def _run_trial(self, engine, candidate, stats, trial, dryrun=False):
        """optimization_based_attack.py:90-143, iterations executed on the device."""
        opt = self.cfg.optim
        T = int(opt.max_iterations)
        table = lr_table(opt.step_size, cfg_get(opt, "step_size_decay"), cfg_get(opt, "warmup", 0), T)
        name = str(opt.optimizer).lower()
        if (name == "l-bfgs" and not self._lbfgs_on_device(engine)) or isinstance(engine, _EngineSum):
            # host-driven loops, every closure evaluation on the engine(s): L-BFGS (common.py:18) where the device loop does not
            # apply, and multi-query attacks, whose candidate gradient is a sum over engines and cannot use one engine's fused step
            from . import augment, lbfgs

            if augment.has_view_stages(self.cfg):
                _refuse_view_stages_off_device(self.cfg, 2)
            dm, ds = self.dm.to(candidate.device), self.ds.to(candidate.device)
            best, history = lbfgs.run_trial(engine, candidate, self.cfg, table, -dm / ds, (1 - dm) / ds, dryrun)
            stats[f"Trial_{trial}_Val"].extend(history)
            return best.detach()
        if name == "l-bfgs":   # one iteration = one optimizer.step, its inner loop inside the captured graph
            engine.begin_lbfgs_trial(candidate, table, trial=trial)
        else:
            if hasattr(engine, "set_augmentations"):
                plan = self._augmentation_plan(candidate)
                if plan is not None or getattr(engine, "_aug_active", False):   # (re-setting invalidates the captured graph: only when needed)
                    engine.set_augmentations(plan)
                    engine._aug_active = plan is not None
            engine.begin_trial(candidate, table, trial=trial)   # the global index: ranks sharing one noise seed still draw different fields
        callback = int(cfg_get(opt, "callback", 0) or 0)
        chunk = callback if callback > 0 else T
        total = 1 if dryrun else T
        done = 0
        current_wallclock = time.time()
        try:
            while done < total:
                n = min(chunk, total - done) if done > 0 else 1  # first log line after iteration 1, like the reference
                engine.run(n)
                done += n
                st = engine.status()  # one host sync per `callback` iterations
                if done == total or (callback > 0 and (done - 1) % callback == 0):
                    timestamp = time.time()
                    obj = engine.history(st["recorded"])[-1].item() if st["recorded"] > 0 else float("nan")
                    log.info(
                        f"| It: {done} | Rec. loss: {obj:2.4f} |  Task loss: {st['task_loss']:2.4f} | "
                        f"T: {timestamp - current_wallclock:4.2f}s"
                    )
                    current_wallclock = timestamp
                if st["stopped"]:
                    log.info(f"Recovery loss is non-finite in iteration {st['recorded']}. Cancelling reconstruction!")
                    break
        except KeyboardInterrupt:
            print(f"Recovery interrupted manually in iteration {done}!")
        engine.sync()
        stats[f"Trial_{trial}_Val"].extend(engine.history().tolist())
        return engine.best().detach()

    def _lbfgs_on_device(self, engine):
        """L-BFGS trials run on the device with one engine, no augmentations and no Langevin noise; multi-query attacks, augmented
        configs and Langevin noise keep the host loop of attacks/lbfgs.py."""
        return (hasattr(engine, "begin_lbfgs_trial") and not isinstance(engine, _EngineSum) and not cfg_get(self.cfg, "augmentations")
                and not float(cfg_get(self.cfg.optim, "langevin_noise", 0.0) or 0.0))

    def _augmentation_plan(self, candidate):
        """cfg.augmentations -> the engine's view pipeline (optimization_based_attack.py:42-48); colour constants are drawn once per
        attacker and batch size, like the reference module's ``shuffled`` flag."""
        from . import augment

        key = (candidate.shape[0], candidate.shape[1])
        if key not in self._aug_plans:
            self._aug_plans[key] = augment.build_plan(self.cfg, candidate.shape[0], candidate.shape[1], self.setup, spatial=tuple(candidate.shape[2:]))
        plan = self._aug_plans[key]
        if plan is not None and plan.stages and plan.candidate_shape != tuple(candidate.shape):
            plan = augment.with_spatial(plan, self.cfg, candidate.shape[2:])   # a multi-scale stage: same draws, its own geometry
        return plan

    def _score_trial(self, engine, candidate):
        """optimization_based_attack.py:191-204."""
        scoring = self.cfg.restarts.scoring
        if scoring in ("euclidean", "cosine-similarity"):
            return self._scoring_engine(engine, candidate).score(candidate, scoring)
        if scoring in ("TV", "total-variation"):
            from ..engine import total_variation

            return total_variation(candidate.contiguous(), scale=1.0)[0]
        raise ValueError(f"Scoring mechanism {scoring} not implemented.")

    def _scoring_engine(self, engine, candidate):
        """The score is taken on the un-augmented candidate at its own shape (:191-204).  When a view resizes, the trial's engine
        runs the model at the view's shape; the score then needs a program at the candidate's shape, built once per shape (a model
        that cannot take it raises UnsupportedModelError, as the reference's forward pass would fail)."""
        if isinstance(engine, _EngineSum):
            return engine
        t0 = engine.prog.tensors[0]
        if (t0.N, t0.C, t0.H, t0.W) == tuple(candidate.shape):
            return engine
        shape = tuple(candidate.shape)
        cache = self.__dict__.setdefault("_score_engines", {})
        if shape not in cache:
            rec_models, shared_data, labels = self._score_context
            cache[shape] = self._get_engine(rec_models, shared_data, labels, data_shape=shape[1:], primary=False, for_scoring=True)
        return cache[shape]

    def _select_optimal_reconstruction(self, candidate_solutions, scores, stats, shape):
        """optimization_based_attack.py:206-218 + the cross-rank MINLOC select (dist.py)."""
        t0 = time.perf_counter()
        optimal_val, optimal_index = bdist.select_best(scores)
        solution = bdist.fetch_solution(candidate_solutions, optimal_index, shape, self.setup)
        if solution.is_cuda:
            torch.cuda.synchronize(solution.device)
        self.last_select_seconds = time.perf_counter() - t0   # the one cross-rank exchange of a reconstruct() call
        stats["opt_value"] = optimal_val
        if optimal_val != float("inf") and optimal_val == optimal_val:
            log.info(f"Optimal candidate solution with rec. loss {optimal_val:2.4f} selected.")
            return solution
        log.info("No valid reconstruction could be found.")
        return torch.zeros_like(solution)
