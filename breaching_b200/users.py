"""User-side update production on the engine (SURVEY section 8 f-2): the step *before* the hot path.

Counterpart of ``UserSingleStep.compute_local_updates`` (``cases/users.py:107-188``): load the server's parameters
(and public buffers), run the model forward + backward on the user's batch, optionally clip per example
(``:158-165``, ``_clip_list_of_grad_`` ``:190-194``) and add differential-privacy noise (``:196-200``), and return the same
``(shared_data, true_user_data)`` dictionaries.  The forward / backward are sweeps F and B of the layer program on the GPU
(``bre_engine_param_gradients``); there is no eager fallback.
"""
import copy

import torch

from . import compiler as C
from .config import get_attack_config
from .engine import Engine, EngineError


class UserSingleStep:
    """A user computing one gradient of the mean loss over its batch (the reference class of the same name)."""

    def __init__(self, model, loss_fn, setup, num_data_points, provide_labels=True, provide_num_data_points=True,
                 provide_buffers=True, per_example_clipping=0.0, gradient_noise=0.0, noise_distribution="gaussian",
                 user_idx=0, backend=None):
        self.model = copy.deepcopy(model)
        self.loss_fn = loss_fn
        self.setup = dict(device=torch.device(setup["device"]), dtype=setup.get("dtype", torch.float))
        if self.setup["device"].type != "cuda":
            raise EngineError("the engine needs a CUDA device (there is no CPU fallback)")
        name = getattr(loss_fn, "original_name", None) or type(loss_fn).__name__
        if name != "CrossEntropyLoss":
            raise NotImplementedError(f"user-side updates on the engine: CrossEntropyLoss only (got {name})")
        self.num_data_points = int(num_data_points)
        self.provide_labels, self.provide_num_data_points, self.provide_buffers = provide_labels, provide_num_data_points, provide_buffers
        self.clip_value = float(per_example_clipping or 0.0)
        self.noise_scale, self.noise_distribution = float(gradient_noise or 0.0), noise_distribution
        self.user_idx = user_idx
        self.backend = backend
        self.counted_queries = 0
        self._engines = {}

    def _engine(self, batch, shape, train):
        key = (batch, tuple(shape), train)
        if key not in self._engines:
            cfg = get_attack_config("invertinggradients")   # only the layer program and sweeps F + B are used
            m = copy.deepcopy(self.model).to(self.setup["device"])
            m.train() if train else m.eval()
            if train:
                for module in m.modules():  # users.py:140-143
                    if hasattr(module, "momentum"):
                        module.momentum = None
            self._engines[key] = Engine(m, (batch, *shape), cfg, self.setup["device"], backend=self.backend)
        return self._engines[key]

    def compute_local_updates(self, server_payload, custom_data):
        """``custom_data``: ``dict(inputs=[B, ...], labels=[B])`` (the reference loads it from its dataloader)."""
        self.counted_queries += 1
        data = {k: v.to(self.setup["device"]) for k, v in custom_data.items()}
        key = "inputs" if "inputs" in data else "input_ids"
        x, y = data[key].to(torch.float32), data["labels"]
        B = y.shape[0]
        parameters, buffers = server_payload["parameters"], server_payload["buffers"]
        train = buffers is None
        with torch.no_grad():
            for p, src in zip(self.model.parameters(), parameters):
                p.copy_(src.to(p.device, p.dtype))
            if buffers is not None:
                for b, src in zip(self.model.buffers(), buffers):
                    b.copy_(src.to(b.device, b.dtype))

        def run(engine, xb, yb):
            engine.model.load_state_dict(self.model.state_dict())
            engine.load_model(params=[p.detach() for p in parameters])
            return engine.param_gradients(xb, yb)

        shared_buffers = None
        if self.clip_value > 0:   # per-example gradients, clipped, averaged (users.py:158-165)
            eng = self._engine(1, x.shape[1:], train)
            shared = None
            for i in range(B):
                g, _ = run(eng, x[i:i + 1], y[i:i + 1])
                norm = torch.stack([t.norm(2) for t in g]).norm(2)
                if norm > self.clip_value:
                    g = [t * (self.clip_value / (norm + 1e-6)) for t in g]
                shared = g if shared is None else [a + b for a, b in zip(shared, g)]
            shared = [t / B for t in shared]
        else:
            eng = self._engine(B, x.shape[1:], train)
            shared, _ = run(eng, x, y)
            if train:
                # per BN layer (engine order = order of the BN ops): batch mean / biased variance of this forward and the number
                # of samples per channel; momentum None -> cumulative average over one batch: running_mean = mean,
                # running_var = unbiased variance, num_batches_tracked = 1.  Shipped in model.buffers() order.
                stats, j = {}, 0
                measured = eng.bn_batch_stats()
                for op in eng.prog.ops:
                    if op.kind == C.OP_BNACT and op.has_bn:
                        t = eng.prog.tensors[op.tin]
                        n = t.N * t.H * t.W
                        mean, var = measured[j]
                        stats[id(eng._bn_modules[j])] = (mean, var * (n / max(n - 1, 1)))
                        j += 1
                shared_buffers = []
                for mod in eng.model.modules():
                    if isinstance(mod, torch.nn.BatchNorm2d):
                        mean, var = stats[id(mod)]
                        shared_buffers += [mean, var, torch.ones((), dtype=torch.long, device=mean.device)]
        if self.noise_scale > 0:  # users.py:196-200
            dist = (torch.distributions.normal.Normal if self.noise_distribution == "gaussian" else torch.distributions.laplace.Laplace)(
                torch.tensor(0.0, device=self.setup["device"]), torch.tensor(self.noise_scale, device=self.setup["device"]))
            shared = [t + dist.sample(t.shape) for t in shared]
        metadata = dict(num_data_points=self.num_data_points if self.provide_num_data_points else None,
                        labels=y.sort()[0] if self.provide_labels else None, local_hyperparams=None)
        shared_data = dict(gradients=shared, buffers=shared_buffers if (train and self.provide_buffers) else None, metadata=metadata)
        true_user_data = dict(data=data[key], labels=y, buffers=shared_buffers)
        return shared_data, true_user_data
