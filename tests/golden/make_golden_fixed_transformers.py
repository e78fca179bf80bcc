"""Generate ``fixed_transformers.pt``: the TAG joint attack (tag.yaml) of the UNMODIFIED reference on its fixed-position
``TransformerModel(positional_embedding="fixed")`` (language_models.py:150-205; the sinusoidal ``PositionalEmbedding`` buffer of
transformer3f, transformer1 and transformerS).

Run where the reference is importable (``BREACHING_REFERENCE_ROOT``, see oracle/refshim.py):
``python tests/golden/make_golden_fixed_transformers.py``

Each case builds ``synthetic.make_text_case(positional="fixed", ...)`` and loads its state dict -- parameters and the ``pe``
buffer -- into the reference's ``TransformerModel``, which then produces the user's gradient and runs the reference attacker
(``run_reference_joint`` of make_golden.py with that model): the TAG closure at the seeded x0 / label logits and a 6-iteration
trajectory.  The tests rebuild the same weights from the case arguments, so no GPU test imports the reference.
"""
import os
import sys
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
warnings.filterwarnings("ignore")

from breaching_b200 import synthetic  # noqa: E402
from oracle import refshim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))

# miniatures of the reference's fixed presets: transformer3f (3 layers, 8 heads of 12, nhid 1536) at T = 8, transformer1 (one head of
# 200, nhid 200) at T = 32 and transformerS (one head of 512, nhid 512) at T = 16, each with a small vocabulary
CASES = {
    "transformer3f": dict(batch=1, seq_len=8, seed=61, ntokens=40, ninp=96, nhead=8, nhid=1536, nlayers=3, positional="fixed"),
    "transformer1": dict(batch=1, seq_len=32, seed=62, ntokens=48, ninp=200, nhead=1, nhid=200, nlayers=1, positional="fixed"),
    "transformerS": dict(batch=1, seq_len=16, seed=63, ntokens=56, ninp=512, nhead=1, nhid=512, nlayers=1, positional="fixed"),
}
ITERS = 6


def reference_model_case(ref, case):
    """``make_text_case`` with its weights in the reference's ``TransformerModel``: the user's gradient from the reference model."""
    from breaching.cases.models.language_models import TransformerModel

    model, loss_fn, payload, shared, true = synthetic.make_text_case(**case)
    rm = TransformerModel(case["ntokens"], case["ninp"], case["nhead"], case["nhid"], case["nlayers"], dropout=0.0,
                          positional_embedding="fixed")
    rm.load_state_dict(model.state_dict())
    rm.eval()
    params = list(rm.parameters())
    grads = torch.autograd.grad(loss_fn(rm(true["data"]), true["labels"]), params)
    payload = [dict(parameters=params, buffers=[b for b in rm.buffers()], metadata=payload[0]["metadata"])]
    shared = [dict(gradients=[g.detach().clone() for g in grads], buffers=None,
                   metadata=dict(num_data_points=case["batch"], labels=None, local_hyperparams=None))]
    return rm, loss_fn, payload, shared, true


def run(ref, case):
    import make_golden
    from torch.nn.attention import SDPBackend, sdpa_kernel

    rm = reference_model_case(ref, case)
    make_golden.synthetic = types.SimpleNamespace(make_text_case=lambda **kw: rm)   # run_reference_joint attacks this case
    try:
        with sdpa_kernel(SDPBackend.MATH):
            fx = make_golden.run_reference_joint(ref, case, "tag", {}, ITERS)
    finally:
        make_golden.synthetic = synthetic
    fx["pe"] = rm[0].pos_encoder.pe[0, :case["seq_len"]].clone()
    fx["weight_checksum"] = float(sum(p.double().sum() for p in rm[0].parameters()))
    return fx


if __name__ == "__main__":
    ref = refshim.import_reference()
    torch.save({name: run(ref, case) for name, case in CASES.items()}, os.path.join(HERE, "fixed_transformers.pt"))
