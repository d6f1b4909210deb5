"""Single-process arithmetic model of the reference's collectives (TEST INFRASTRUCTURE).

Every function takes the inputs of *all* W ranks (index 0 = rank 0) and returns what the
reference leaves in each rank's tensors.  Citations are into the reference checkout (facebookresearch/flashy).

Arithmetic contract restated from ``flashy/distrib.py``:

* ``average_tensors`` (:96-111): tensors that are neither floating point nor complex are
  skipped (:102); for the others SUM over ranks (:105-108) and afterwards a true division
  by the world size (:111).  Sum first, divide after.
* ``broadcast_tensors`` (:114-127): bit copy of rank ``src``'s float/complex tensors.
* ``average_metrics`` (:50-62): fp32 vector ``[v_1..v_k, 1] * count`` per rank, SUM, then
  ``v_i / last``.
* ``_check_number_of_params`` (:78-89): ``sum(len) != len * W`` on a rank => that rank raises.
* ``loader`` (:227-243): strided ``Subset`` shard for ``shuffle=False``, ``DistributedSampler``
  with its defaults for ``shuffle=True``.

Accumulation precision.  The reference accumulates in whatever ``torch.distributed`` does for
the dtype (gloo: ring in the native dtype; NCCL: tree/ring/NVLS), so the bits of an fp32 sum
depend on the backend.  The parity bar (SURVEY.md 8c, BASELINE.md 5) is therefore defined on
this model: fp32/fp64 summed in rank order in the native dtype; bf16/fp16 summed in fp32 and
rounded once -- ``bf16(fp32 path on the same bf16-valued inputs)``.
"""
from __future__ import annotations

import typing as tp

import torch

_WIDE = {
    torch.float32: torch.float32,
    torch.float64: torch.float64,
    torch.bfloat16: torch.float32,
    torch.float16: torch.float32,
    torch.complex64: torch.complex64,
    torch.complex128: torch.complex128,
}


def is_complex_or_float(t: torch.Tensor) -> bool:
    # flashy/distrib.py:92-93
    return torch.is_floating_point(t) or torch.is_complex(t)


def count_check(lengths: tp.Sequence[int]) -> tp.List[bool]:
    """flashy/distrib.py:78-89 -- per rank: does the rank raise?"""
    world = len(lengths)
    total = sum(int(n) for n in lengths)
    out = []
    for n in lengths:
        if world == 1 or n == 0:        # :81-82
            out.append(False)
        else:
            out.append(total != n * world)   # :86
    return out


def reduce_sum(columns: tp.Sequence[torch.Tensor]) -> torch.Tensor:
    """SUM over ranks of one tensor, rank order, in the wide dtype (not yet rounded)."""
    wide = _WIDE[columns[0].dtype]
    acc = columns[0].detach().to(wide).clone()
    for other in columns[1:]:
        acc += other.detach().to(wide)
    return acc


def average_one(columns: tp.Sequence[torch.Tensor]) -> torch.Tensor:
    """Mean over ranks of one tensor: (sum_r x_r) / W rounded once to the input dtype."""
    world = len(columns)
    acc = reduce_sum(columns)
    acc /= world                         # flashy/distrib.py:111, true division
    return acc.to(columns[0].dtype)


def average_tensors(per_rank: tp.Sequence[tp.Sequence[torch.Tensor]]) -> tp.List[tp.List[torch.Tensor]]:
    """flashy/distrib.py:96-111.  Returns the post-call tensors of every rank."""
    world = len(per_rank)
    if world == 1:                       # :100-101
        return [[t.clone() for t in per_rank[0]]]
    n = len(per_rank[0])
    out: tp.List[tp.List[torch.Tensor]] = [[] for _ in range(world)]
    for i in range(n):
        cols = [per_rank[r][i] for r in range(world)]
        if is_complex_or_float(cols[0]):
            mean = average_one(cols)
            for r in range(world):
                out[r].append(mean.clone())
        else:                            # :102 -- left untouched
            for r in range(world):
                out[r].append(cols[r].clone())
    return out


def all_reduce_sum(columns: tp.Sequence[torch.Tensor]) -> torch.Tensor:
    """flashy/distrib.py:45-47 with the default op (SUM); integer dtypes are exact."""
    if is_complex_or_float(columns[0]):
        return reduce_sum(columns).to(columns[0].dtype)
    acc = columns[0].clone()
    for other in columns[1:]:
        acc += other
    return acc


def broadcast_tensors(per_rank: tp.Sequence[tp.Sequence[torch.Tensor]], src: int = 0):
    """flashy/distrib.py:114-127."""
    world = len(per_rank)
    out = []
    for r in range(world):
        row = []
        for i, t in enumerate(per_rank[r]):
            if world > 1 and is_complex_or_float(t):
                row.append(per_rank[src][i].clone())
            else:
                row.append(t.clone())
        out.append(row)
    return out


def average_metrics(per_rank: tp.Sequence[tp.Dict[str, float]], counts: tp.Sequence[float]):
    """flashy/distrib.py:50-62 -- returns the dict every rank gets back."""
    world = len(per_rank)
    if world == 1:                       # :54-55 -- input returned unchanged
        return dict(per_rank[0])
    keys = list(per_rank[0].keys())
    acc = torch.zeros(len(keys) + 1, dtype=torch.float32)
    for metrics, count in zip(per_rank, counts):
        row = torch.tensor([metrics[k] for k in keys] + [1], dtype=torch.float32)
        row *= count                     # :59
        acc += row                       # :60
    averaged = (acc[:-1] / acc[-1]).tolist()   # :61
    return dict(zip(keys, averaged))


def loader_indices(n: int, rank: int, world: int, shuffle: bool) -> tp.List[int]:
    """Index list rank ``rank`` iterates for a dataset of length ``n`` (flashy/distrib.py:227-243)."""
    if world == 1:
        if shuffle:
            raise ValueError("single-process shuffle order is torch's global RNG; not modelled")
        return list(range(n))
    if not shuffle:
        return list(range(rank, n, world))       # :241
    # DistributedSampler defaults (:236): shuffle=True, seed=0, epoch=0, drop_last=False.
    g = torch.Generator()
    g.manual_seed(0)
    order = torch.randperm(n, generator=g).tolist()
    per = -(-n // world)
    total = per * world
    pad = total - len(order)
    if pad:
        reps = -(-pad // len(order))
        order += (order * reps)[:pad]
    return order[rank:total:world]
