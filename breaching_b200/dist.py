"""Multi-GPU restarts: independent trials shard one-per-rank, one MIN all-reduce selects the winner.

The reference runs its restarts sequentially in one process (``optimization_based_attack.py:70-74``; there is no
``torch.distributed`` call anywhere in it).  Trials only share read-only inputs, so the multi-GPU layout is one process
per GPU with trial ``k`` on rank ``k mod world`` and **no data-path collective**.  Selection
(``_select_optimal_reconstruction``, ``:206-218``: ``torch.min`` -> first index wins; non-finite -> +inf) becomes a
single all-reduce(MIN) over a packed 63-bit key ``(sortable_float32_bits(score) << 31) | trial_index`` followed by
one broadcast of the winning candidate from its owner.  Works with NCCL (GPU) and gloo (CPU tests).
"""
import struct

import torch
import torch.distributed as dist

_INF_BITS = 0x7F800000


def rank_and_world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def _sortable_bits(value):
    """Order-preserving map float32 -> uint32 (total order, -x < +x); NaN is treated as +inf (``:204``)."""
    if value != value:
        value = float("inf")
    bits = struct.unpack("<I", struct.pack("<f", value))[0]
    return (~bits) & 0xFFFFFFFF if bits & 0x80000000 else bits | 0x80000000


def _from_sortable(u):
    bits = u & 0x7FFFFFFF if u & 0x80000000 else (~u) & 0xFFFFFFFF
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def pack_key(score, index):
    return (_sortable_bits(float(score)) << 31) | (int(index) & 0x7FFFFFFF)


def unpack_key(key):
    return _from_sortable((key >> 31) & 0xFFFFFFFF), key & 0x7FFFFFFF


def _comm_device():
    backend = dist.get_backend()
    return torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")


def select_best(scores):
    """``scores[k]`` is finite only on the rank that ran trial ``k`` (``inf`` elsewhere).

    Returns ``(value, index)`` identical on every rank: the minimal score and the *first* trial attaining it.
    """
    local = min((pack_key(s, k) for k, s in enumerate(scores.tolist())), default=pack_key(float("inf"), 0))
    rank, world = rank_and_world()
    if world > 1:
        key = torch.tensor([local], dtype=torch.int64, device=_comm_device())
        dist.all_reduce(key, op=dist.ReduceOp.MIN)
        local = int(key.item())
    value, index = unpack_key(local)
    return value, index


def fetch_solution(candidate_solutions, index, shape, setup):
    """Return trial ``index``'s candidate on every rank (broadcast from the owning rank)."""
    rank, world = rank_and_world()
    owner = index % world
    if world == 1:
        sol = candidate_solutions[index]
        return sol if sol is not None else torch.zeros(shape, **setup)
    dev = _comm_device()
    if rank == owner and candidate_solutions[index] is not None:
        buf = candidate_solutions[index].detach().to(dev).contiguous()
    else:
        buf = torch.zeros(shape, dtype=setup["dtype"], device=dev)
    dist.broadcast(buf, src=owner)
    return buf.to(setup["device"])
