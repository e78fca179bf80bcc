"""Synthetic federated-learning cases for tests and benchmarks.

The reference's case machinery (``breaching/cases``) needs dataset downloads and hydra; what the
attack actually consumes is the pair ``server_payload`` / ``shared_data`` whose layout is fixed by
``cases/servers.py:138-147`` and ``cases/users.py:176-186`` (and shown literally in
``minimal_example.py:52-66``).  This module builds exactly those dictionaries from random-init models
and random user data, for the BASELINE.json configurations (SURVEY.md section 8d).
"""
from collections import OrderedDict

import torch


class DataConfig:
    """Stand-in for the hydra ``cfg.case.data`` node: attribute *and* item access (base_attack.py:51-62)."""

    def __init__(self, **kwargs):
        self.__dict__.update(kwargs)

    def __getitem__(self, key):
        return self.__dict__[key]

    def __contains__(self, key):
        return key in self.__dict__


IMAGENET = dict(  # config/case/data/ImageNet.yaml:1-22 (397-class subset used by the benchmark, SURVEY 8d)
    name="ImageNet", modality="vision", task="classification", classes=397, shape=(3, 224, 224),
    mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), normalize=True,
)
CIFAR10 = dict(  # config/case/data/CIFAR10.yaml:1-22
    name="CIFAR10", modality="vision", task="classification", classes=10, shape=(3, 32, 32),
    mean=(0.4914672374725342, 0.4822617471218109, 0.4467701315879822),
    std=(0.24703224003314972, 0.24348513782024384, 0.26158785820007324), normalize=True,
)


def convnet(width=64, num_classes=10, num_channels=3):
    """Architecture of the reference's ``ConvNet`` (cases/models/model_preparation.py:437-479):
    eight conv3x3(+bias)-BN-ReLU stages, MaxPool2d(3) after stages 5 and 7, then a linear head."""
    chans = [num_channels, width, 2 * width, 2 * width, 4 * width, 4 * width, 4 * width, 4 * width, 4 * width]
    layers = []
    for i in range(8):
        layers.append((f"conv{i}", torch.nn.Conv2d(chans[i], chans[i + 1], kernel_size=3, padding=1)))
        layers.append((f"bn{i}", torch.nn.BatchNorm2d(chans[i + 1])))
        layers.append((f"relu{i}", torch.nn.ReLU()))
        if i == 5:
            layers.append(("pool0", torch.nn.MaxPool2d(3)))
        if i == 7:
            layers.append(("pool1", torch.nn.MaxPool2d(3)))
    layers.append(("flatten", torch.nn.Flatten()))
    layers.append(("linear", torch.nn.Linear(36 * width, num_classes)))

    class ConvNet(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.model = torch.nn.Sequential(OrderedDict(layers))

        def forward(self, inputs):
            return self.model(inputs)

    return ConvNet()


def build_model(name, classes, seed=0):
    """Random-init model of the requested architecture (no checkpoints: there is no network)."""
    import torchvision

    torch.manual_seed(seed)
    if name == "convnet":
        model = convnet(width=64, num_classes=classes)
    elif name == "convnet-tiny":
        model = convnet(width=8, num_classes=classes)
    elif name == "linear":   # cases/models/model_preparation.py:236-238, :311-313 (input_dim from the CIFAR-10 shape)
        model = torch.nn.Sequential(torch.nn.Flatten(), torch.nn.Linear(3 * 32 * 32, classes))
    elif name in ("resnet18", "resnet34", "resnet50", "resnet101"):
        model = getattr(torchvision.models, name)(weights=None)
        model.fc = torch.nn.Linear(model.fc.in_features, classes)  # cases/models/model_preparation.py:172-177
    else:
        raise ValueError(name)
    return model


def randomize_bn(model, seed=1):
    """Give BN layers non-trivial affine parameters and running statistics so that parity tests
    exercise every term (random init has gamma=1, beta=0, mean=0, var=1)."""
    gen = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.copy_(1.0 + 0.2 * torch.randn(m.weight.shape, generator=gen))
                m.bias.copy_(0.1 * torch.randn(m.bias.shape, generator=gen))
                m.running_mean.copy_(0.1 * torch.randn(m.running_mean.shape, generator=gen))
                m.running_var.copy_(1.0 + 0.3 * torch.rand(m.running_var.shape, generator=gen))
    return model


def make_case(model_name="resnet18", data="imagenet", batch=1, seed=233, provide_labels=False,
              user_buffers=False, bn_random=False, image_size=None, classes=None, unique_labels=True, no_buffers=False):
    """Return ``(model, loss_fn, server_payload, shared_data, true_user_data)`` with CPU tensors.

    Single local step (``local_hyperparams=None``); honest server with public buffers (eval-mode BN) or,
    with ``user_buffers=True``, the see-through-gradients setting where the user computes its update in
    train mode with ``momentum=None`` and ships the buffers (cases/users.py:140-143,174).
    """
    base = dict(IMAGENET if data == "imagenet" else CIFAR10)
    if image_size is not None:
        base["shape"] = (3, image_size, image_size)
    if classes is not None:
        base["classes"] = classes
    meta = DataConfig(**base)
    model = build_model(model_name, meta.classes, seed=seed)
    if bn_random:
        randomize_bn(model, seed + 1)
    loss_fn = torch.nn.CrossEntropyLoss()

    gen = torch.Generator().manual_seed(seed + 7)
    x = torch.randn((batch, *meta.shape), generator=gen)
    if unique_labels and batch <= meta.classes:
        y = torch.randperm(meta.classes, generator=gen)[:batch].sort()[0]
    else:
        y = torch.randint(0, meta.classes, (batch,), generator=gen).sort()[0]

    params = [p for p in model.parameters()]
    if no_buffers:
        # neither the server nor the user publishes BN buffers: the user computes its update in train mode (batch statistics)
        # and the attacker has to do the same (base_attack.py:192-197)
        model.train()
        loss = loss_fn(model(x), y)
        grads = torch.autograd.grad(loss, params)
        shared_buffers, payload_buffers = None, None
    elif user_buffers:
        model.train()
        for m in model.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.momentum = None
                m.reset_running_stats()
        loss = loss_fn(model(x), y)
        grads = torch.autograd.grad(loss, params)
        model.eval()
        shared_buffers = [b.clone().detach() for b in model.buffers()]
        payload_buffers = None
    else:
        model.eval()
        loss = loss_fn(model(x), y)
        grads = torch.autograd.grad(loss, params)
        shared_buffers = None
        payload_buffers = [b for b in model.buffers()]

    server_payload = [dict(parameters=params, buffers=payload_buffers, metadata=meta)]
    shared_data = [
        dict(
            gradients=[g.detach().clone() for g in grads],
            buffers=shared_buffers,
            metadata=dict(num_data_points=batch, labels=y.clone() if provide_labels else None, local_hyperparams=None),
        )
    ]
    true_user_data = dict(data=x, labels=y)
    return model, loss_fn, server_payload, shared_data, true_user_data


def make_fedavg_case(model_name="resnet18", data="imagenet", num_data_points=4, steps=4, data_per_step=1, lr=1e-3, seed=233,
                     bn_random=False, image_size=None, classes=None, no_buffers=False):
    """Multi-step user (cases/users.py:336-413 ``UserMultiStep`` with ``local_updates.yaml``): ``steps`` SGD steps of size
    ``lr`` on consecutive slices of ``data_per_step`` images, eval-mode BN with the server's public buffers; the shared
    "gradient" is ``W_local - W_server`` and the local hyper-parameters (incl. the per-step labels) are shared.

    ``no_buffers=True``: the server publishes no BN buffers (``provide_public_buffers=False``), so the user trains in train mode,
    every local step normalising with its own batch statistics (cases/users.py:345-353), and the attacker has to do the same
    (base_attack.py:192-197); the payload then has ``buffers=None``, as in :func:`make_case`."""
    import copy

    base = dict(IMAGENET if data == "imagenet" else CIFAR10)
    if image_size is not None:
        base["shape"] = (3, image_size, image_size)
    if classes is not None:
        base["classes"] = classes
    meta = DataConfig(**base)
    model = build_model(model_name, meta.classes, seed=seed)
    if bn_random:
        randomize_bn(model, seed + 1)
    model.eval()
    loss_fn = torch.nn.CrossEntropyLoss()
    gen = torch.Generator().manual_seed(seed + 7)
    x = torch.randn((num_data_points, *meta.shape), generator=gen)
    y = torch.randperm(meta.classes, generator=gen)[:num_data_points]
    server_params = [p.detach().clone() for p in model.parameters()]
    local = copy.deepcopy(model).train(no_buffers)
    optimizer = torch.optim.SGD(local.parameters(), lr=lr)
    seen, label_list = 0, []
    for _ in range(steps):
        xs, ys = x[seen: seen + data_per_step], y[seen: seen + data_per_step]
        seen = (seen + data_per_step) % num_data_points
        label_list.append(ys.sort()[0])
        optimizer.zero_grad()
        loss_fn(local(xs), ys).backward()
        optimizer.step()
    shared_grads = [(pl - ps).clone().detach() for pl, ps in zip(local.parameters(), server_params)]
    payload_buffers = None if no_buffers else [b for b in model.buffers()]
    server_payload = [dict(parameters=[p for p in model.parameters()], buffers=payload_buffers, metadata=meta)]
    shared_data = [dict(gradients=shared_grads, buffers=None,
                        metadata=dict(num_data_points=num_data_points, labels=None,
                                      local_hyperparams=dict(lr=lr, steps=steps, data_per_step=data_per_step, labels=label_list)))]
    return model, loss_fn, server_payload, shared_data, dict(data=x, labels=y)


def make_multi_query_case(model_name="convnet-tiny", data="cifar", batch=1, seed=233, queries=2, bn_random=True, image_size=None,
                          classes=None):
    """Several model queries on the same user data (cases/servers.py ``num_queries``; the attack sums its objective over
    ``zip(rec_models, shared_data)``, optimization_based_attack.py:157-160): query 0 is ``make_case(seed)``, query k a
    model of the same architecture initialised with ``seed + 100 k``; the user answers each with the gradient on the same
    batch.  Returns ``(model_template, loss_fn, server_payload[list], shared_data[list], true_user_data)``."""
    model, loss_fn, payload, shared, true = make_case(model_name, data, batch=batch, seed=seed, bn_random=bn_random,
                                                      image_size=image_size, classes=classes)
    meta = payload[0]["metadata"]
    for k in range(1, queries):
        other = build_model(model_name, meta.classes, seed=seed + 100 * k)
        if bn_random:
            randomize_bn(other, seed + 100 * k + 1)
        other.eval()
        params = [p for p in other.parameters()]
        grads = torch.autograd.grad(loss_fn(other(true["data"]), true["labels"]), params)
        payload.append(dict(parameters=params, buffers=[b for b in other.buffers()], metadata=meta))
        shared.append(dict(gradients=[g.detach().clone() for g in grads], buffers=None,
                           metadata=dict(num_data_points=batch, labels=None, local_hyperparams=None)))
    return model, loss_fn, payload, shared, true


class TransformerLM(torch.nn.Module):
    """Architecture of the reference's ``TransformerModel`` (cases/models/language_models.py:150-205, BASELINE config 5:
    ntokens 50257, ninp 96, nhead 8, nhid 1536, nlayers 3, dropout 0, learnable positional embedding): token embedding
    (scaled by sqrt(ninp) at init), positional embedding added, ``nn.TransformerEncoder`` of post-norm ReLU layers
    (batch first, no mask), linear decoder.  Module names follow the reference so that ``parameters()`` has its order."""

    def __init__(self, ntokens=50257, ninp=96, nhead=8, nhid=1536, nlayers=3, max_positions=1024):
        super().__init__()
        import math

        self.pos_encoder = torch.nn.Module()
        self.pos_encoder.embedding = torch.nn.Embedding(max_positions, ninp)
        layer = torch.nn.TransformerEncoderLayer(ninp, nhead, nhid, 0.0, batch_first=True)
        self.transformer_encoder = torch.nn.TransformerEncoder(layer, nlayers, enable_nested_tensor=False)
        self.encoder = torch.nn.Embedding(ntokens, ninp)
        self.encoder.weight.data *= math.sqrt(ninp)
        self.decoder = torch.nn.Linear(ninp, ntokens)
        torch.nn.init.uniform_(self.encoder.weight, -0.1, 0.1)   # init_weights(), :177-181
        torch.nn.init.uniform_(self.decoder.weight, -0.1, 0.1)

    @property
    def pos_embedding(self):
        return self.pos_encoder.embedding

    @property
    def layers(self):
        return self.transformer_encoder.layers

    def attack_parameters(self):
        """Parameters in the order of the shared gradient after the attack has removed the token-embedding entry
        (base_attack.py:88-95)."""
        return [p for n, p in self.named_parameters() if n != "encoder.weight"]

    def forward(self, input_ids=None, inputs_embeds=None):
        inputs = self.encoder(input_ids) if inputs_embeds is None else inputs_embeds
        positions = torch.arange(inputs.shape[1], device=inputs.device)
        inputs = inputs + self.pos_encoder.embedding(positions[None, :])
        return self.decoder(self.transformer_encoder(inputs))


def causal_loss(outputs, labels):
    """``CausalLoss`` (cases/models/losses.py:7-26): next-token cross-entropy; ``labels`` are token ids [N, T] or class
    probabilities [N, T, vocab] (what the joint attacker passes)."""
    shift_logits = outputs[:, :-1, :].reshape(-1, outputs.shape[-1])
    if labels.dtype == torch.long:
        return torch.nn.functional.cross_entropy(shift_logits, labels[:, 1:].reshape(-1))
    return torch.nn.functional.cross_entropy(shift_logits, labels[:, 1:, :].reshape(-1, labels.shape[-1]))


class CausalLoss(torch.nn.Module):
    """Module form of :func:`causal_loss` (reference cases/models/losses.py:7-26)."""

    def forward(self, outputs, labels):
        return causal_loss(outputs, labels)


def make_text_case(batch=1, seq_len=8, seed=233, ntokens=50, ninp=16, nhead=4, nhid=24, nlayers=2):
    """BASELINE config 5 in miniature: a causal language model user (cases/data/datasets_text.py token batches, users.py
    single step) on ``TransformerLM``.  Returns ``(model, loss_fn, server_payload, shared_data, true_user_data)``; the shared
    gradient list includes the token-embedding entry (the attack removes it, base_attack.py:88-95)."""
    torch.manual_seed(seed)
    model = TransformerLM(ntokens, ninp, nhead, nhid, nlayers, max_positions=max(64, seq_len)).eval()
    gen = torch.Generator().manual_seed(seed + 7)
    with torch.no_grad():  # non-trivial LayerNorm parameters / biases
        for p in model.parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn(p.shape, generator=gen))
    tokens = torch.randint(0, ntokens, (batch, seq_len), generator=gen)
    loss_fn = CausalLoss()
    params = [p for p in model.parameters()]
    grads = torch.autograd.grad(loss_fn(model(tokens), tokens), params)
    meta = DataConfig(name="synthetic-text", modality="text", task="causal-lm", vocab_size=ntokens, shape=(seq_len,), classes=ntokens)
    server_payload = [dict(parameters=params, buffers=[], metadata=meta)]
    shared_data = [dict(gradients=[g.detach().clone() for g in grads], buffers=None,
                        metadata=dict(num_data_points=batch, labels=None, local_hyperparams=None))]
    return model, loss_fn, server_payload, shared_data, dict(data=tokens, labels=tokens)
