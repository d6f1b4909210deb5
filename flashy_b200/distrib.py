"""Hopper-native (H100) drop-in for ``flashy.distrib`` (reference: ``flashy/distrib.py``).

Same names, signatures, in-place semantics and error behaviour as the reference module; the
body is new.  Where the reference issues one ``torch.distributed`` collective and one divide
per tensor plus two host-synchronising count checks per ``sync_model``
(``flashy/distrib.py:78-111``), this module packs each tensor list into a bucket and issues
ONE kernel of ``libflashy_b200.so`` that reads the peers' staging arenas directly over
NVLink and fuses the ``/ world_size``.  ``torch.distributed`` is used for bootstrap
(exchanging memory handles once) and by ``wrap`` (the DDP comparator); ``barrier``,
``broadcast_object`` and the count check ride the communicator's shared-memory fabric, so after
bootstrap this module does not touch NCCL/gloo.  There is no CPU / gloo fallback for tensor
data: CPU tensors in a distributed collective raise.

Environment knobs (none of them changes a public signature):
``FLASHY_B200_ARENA_MB`` (1024), ``FLASHY_B200_BUCKET_MB`` (128), ``FLASHY_B200_EAGER_BUCKET_MB`` (8),
``FLASHY_B200_ONE_SHOT_MAX`` (bytes, 262144), ``FLASHY_B200_SLICE_BYTES`` (8192),
``FLASHY_B200_WIRE=bf16`` (send fp32 gradients as bf16: opt-in, lossy, averaged gradients only),
``FLASHY_B200_CHECK=always|plan`` (count check every call, or only when a bucket plan is new),
``FLASHY_B200_OVERLAP=1`` / ``FLASHY_B200_OVERLAP_BUCKET_MB`` (8) / ``FLASHY_B200_OVERLAP_TAIL_KB`` (512) /
``FLASHY_B200_OVERLAP_BLOCKS`` (32): backward overlap for ``sync_model`` (see ``overlap``; an addition, off by default).
"""
from __future__ import annotations

import os
import pickle
import threading
import typing as tp
import weakref
from contextlib import contextmanager
from functools import wraps

import torch
from torch import distributed
from torch.nn.parallel.distributed import DistributedDataParallel
from torch.utils.data import DataLoader, Subset
from torch.utils.data.distributed import DistributedSampler

from . import _native as N
from . import context as _context
from .engine import Engine, _DTYPES, _ESIZE, _dense

__all__ = [
    "rank", "world_size", "init", "rank_zero_only", "is_rank_zero", "is_distributed", "all_reduce",
    "average_metrics", "wrap", "average_tensors", "broadcast_tensors", "broadcast_model",
    "sync_gradients", "eager_sync_gradients", "sync_model", "eager_sync_model", "loader",
    "broadcast_object", "barrier", "sync_buffers", "overlap",
]


# ------------------------------------------------------------------------------------------
# rank helpers (reference: re-exported from dora.distrib at flashy/distrib.py:21, and :24-42)
# ------------------------------------------------------------------------------------------

def rank() -> int:
    return _context.current().rank


def world_size() -> int:
    return _context.current().world


def init(backend: str = "nccl") -> None:
    """Same contract as ``dora.distrib.init``: no-op if already initialised or single process;
    otherwise ``env://`` rendezvous from RANK / WORLD_SIZE / LOCAL_RANK, one device per rank."""
    if distributed.is_initialized():
        return
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world == 1:
        return
    proc_rank = int(os.environ["RANK"])
    local = int(os.environ.get("LOCAL_RANK", proc_rank))
    if torch.cuda.is_available():
        torch.cuda.set_device(local)
    else:
        assert backend != "nccl", "the nccl backend needs CUDA"
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    distributed.init_process_group(backend=backend, init_method="env://", world_size=world, rank=proc_rank)


def rank_zero_only(fn: tp.Callable) -> tp.Callable:
    """Decorator: run ``fn`` on rank 0 only; other ranks get ``None`` (flashy/distrib.py:24-34)."""
    @wraps(fn)
    def guarded(*args: tp.Any, **kwargs: tp.Any) -> tp.Optional[tp.Any]:
        return fn(*args, **kwargs) if is_rank_zero() else None
    return guarded


def is_rank_zero() -> bool:
    return rank() == 0


def is_distributed() -> bool:
    return world_size() > 1


# ------------------------------------------------------------------------------------------
# internals
# ------------------------------------------------------------------------------------------

def _is_complex_or_float(tensor: torch.Tensor) -> bool:
    return torch.is_floating_point(tensor) or torch.is_complex(tensor)      # flashy/distrib.py:92-93


def _engine(ctx, tensors: tp.Sequence[torch.Tensor]) -> Engine:
    """The communicator of the calling rank, created (collectively) on first use."""
    eng = ctx.cached_engine()
    if eng is not None:
        return eng
    if not N.cuda_available():
        return ctx.engine_for(None, host_only=True)      # rendezvous fabric only; data calls will raise
    cuda = [t for t in tensors if t.is_cuda]
    return ctx.engine_for(cuda[0].device.index if cuda else torch.cuda.current_device())


def _flat(t: torch.Tensor, device: int) -> tp.Tuple[int, int, int]:
    """(fx dtype, address, numel in fx units) of a dense CUDA tensor on this rank's device."""
    if not t.is_cuda:
        raise RuntimeError(
            "flashy_b200 moves tensor data only with its CUDA kernels: a CPU tensor was passed to a "
            "distributed collective and there is no gloo/CPU fallback on this path.")
    if t.device.index != device:
        raise RuntimeError(f"tensor is on cuda:{t.device.index} but this rank's communicator is on cuda:{device}")
    if t.dtype not in _DTYPES:
        raise RuntimeError(f"dtype {t.dtype} is not supported by the flashy_b200 collectives")
    if not _dense(t):
        raise ValueError("Tensors must be contiguous")          # c10d raises the same for NCCL
    fx, mult = _DTYPES[t.dtype]
    return fx, t.data_ptr(), t.numel() * mult


# A dtype code that is the same integer in every process (hash(torch.dtype) is not).
_DT_CODE = {dt: i for i, dt in enumerate((
    torch.float32, torch.bfloat16, torch.float16, torch.float64, torch.int32, torch.int64,
    torch.complex64, torch.complex128, torch.uint8, torch.int8, torch.int16, torch.bool))}


def _list_key(tensors: tp.Sequence[torch.Tensor]) -> tp.Tuple[tp.Tuple[int, ...], tp.Tuple[int, ...]]:
    """(dtype codes, numels): what ranks must agree on, and what a bucket layout depends on."""
    return (tuple([_DT_CODE.get(t.dtype, -1) for t in tensors]), tuple([t.numel() for t in tensors]))


def _key_signature(key) -> int:
    return hash(key) & (2 ** 64 - 1)          # tuples of ints: independent of PYTHONHASHSEED


def _check_number_of_params(params: tp.Sequence[torch.Tensor], key=None) -> None:
    """Reference flashy/distrib.py:78-89, without its device all-reduce and ``.item()`` sync:
    the counts meet in host shared memory.  Raises on EVERY rank if any rank differs."""
    ctx = _context.current()
    if ctx.world == 1 or not params:
        return
    engine = _engine(ctx, params)
    sig = _key_signature(key if key is not None else _list_key(params))
    total, same = engine.host_exchange(ctx.local, len(params), sig)
    if total != len(params) * ctx.world:
        raise RuntimeError(f"Mismatch in number of params: ours is {len(params)}, "
                           "at least one worker has a different one.")
    if not same:
        raise RuntimeError("Mismatch in the shapes/dtypes of the tensors to synchronise: "
                           "at least one worker passed a different list.")


def _launch_streams(engine: Engine, payloads: tp.Sequence[tp.Any], launch: tp.Callable[[tp.Any], None]):
    """Run ``launch(stream)`` ordered after every hosted rank's current stream.  Returns an
    event the ranks must wait on, or None when everything already sits on one stream."""
    streams = [p["stream"] for p in payloads]
    handles = {s.cuda_stream for s in streams}
    if len(handles) == 1:
        launch(streams[0])
        return None
    side = engine.side_stream
    seen = set()
    for s in streams:
        if s.cuda_stream in seen:
            continue
        seen.add(s.cuda_stream)
        ev = torch.cuda.Event()
        ev.record(s)
        side.wait_event(ev)
    launch(side)
    done = torch.cuda.Event()
    done.record(side)
    return done


class _Bucket:
    """One launch: which tensors (index into the list, byte offset for cut tensors) it covers."""
    __slots__ = ("plan", "idx", "off", "plain", "in_arr", "out_arr")

    def __init__(self, plan, idx, off):
        self.plan, self.idx, self.off = plan, idx, off
        self.plain = not any(off)
        n = len(idx)
        self.in_arr = (N.C.c_void_p * n)()
        self.out_arr = (N.C.c_void_p * n)()


class _Layout:
    """Bucket plan of one ordered tensor list (cached by dtype/numel signature)."""
    __slots__ = ("kind", "buckets", "used", "last_in", "last_out", "fresh")

    def __init__(self, kind, buckets, used):
        self.kind, self.buckets, self.used = kind, buckets, used
        self.last_in = self.last_out = None
        self.fresh = True


def split_buckets(items: tp.Sequence[tp.Tuple[int, int]], cap: int, esize: int
                  ) -> tp.List[tp.Tuple[tp.List[int], tp.List[int], tp.List[int]]]:
    """Cut an ordered list of ``(tensor index, numel)`` into buckets of at most ``cap`` elements.

    Returns ``(indices, byte offsets, numels)`` per bucket.  Tensors are never reordered; a
    tensor larger than ``cap`` is cut into consecutive pieces (byte offset ``piece * cap * esize``
    into the tensor), each piece a bucket of its own.  Pure function: every rank computes the same
    split from the same list, which is what keeps the collective sequence identical everywhere."""
    out: tp.List[tp.Tuple[tp.List[int], tp.List[int], tp.List[int]]] = []
    idx: tp.List[int] = []
    off: tp.List[int] = []
    num: tp.List[int] = []
    fill = 0

    def flush():
        nonlocal idx, off, num, fill
        if idx:
            out.append((idx, off, num))
        idx, off, num, fill = [], [], [], 0

    for i, numel in items:
        if numel > cap:                            # one tensor larger than a bucket: cut it
            flush()
            done = 0
            while done < numel:
                n = min(cap, numel - done)
                out.append(([i], [done * esize], [n]))
                done += n
            continue
        if idx and fill + numel > cap:
            flush()
        idx.append(i)
        off.append(0)
        num.append(numel)
        fill += numel
    flush()
    return out


def _build_layout(engine: Engine, kind: str, tensors: tp.Sequence[torch.Tensor], op: int, lossy: bool = False) -> _Layout:
    """Validate the tensors, group them by fx dtype in first-appearance order (identical on
    every rank because the lists are), cut into buckets of at most ``bucket_cap`` wire bytes.
    ``lossy``: the caller is a gradient-averaging path, where ``FLASHY_B200_WIRE=bf16`` may apply."""
    groups: tp.Dict[int, tp.List[tp.Tuple[int, int]]] = {}
    used = []
    for i, t in enumerate(tensors):
        fx, _, numel = _flat(t, engine.device)
        if not numel:
            continue
        used.append(i)
        if kind == "bc":
            groups.setdefault(N.FX_U8, []).append((i, numel * _ESIZE[fx]))
        else:
            groups.setdefault(fx, []).append((i, numel))
    buckets = []
    for fx, items in groups.items():
        wire = N.FX_BF16 if (lossy and engine.wire_bf16 and fx == N.FX_F32 and kind == "ar" and op == N.FX_AVG) else fx
        cap = max(engine.bucket_cap // _ESIZE[wire], 64)
        cap -= cap % 64                            # keep cut pieces 128-byte aligned
        for idx, off, num in split_buckets(items, cap, _ESIZE[fx]):
            buckets.append(_Bucket(engine.get_plan(kind, tuple(num), fx, wire), idx, off))
    return _Layout(kind, buckets, used)


def _dense_or_raise(tensors: tp.Sequence[torch.Tensor], device: tp.Optional[int] = None) -> None:
    """Per-call re-validation of a list whose layout is cached (the cache key only covers dtypes
    and sizes): still CUDA, still on this rank's device, still dense."""
    for t in tensors:
        if not t.is_cuda or (device is not None and t.device.index != device):
            _flat(t, -1 if device is None else device)        # raises with the right message
        if not t.is_contiguous() and not _dense(t):
            raise ValueError("Tensors must be contiguous")


def _run_layout(ctx, engine: Engine, layout: _Layout, in_ptrs: tp.List[int],
                out_ptrs: tp.List[int], op: int, src: int = 0) -> None:
    """Launch every bucket of ``layout`` on the tensors' current addresses."""
    kind = layout.kind
    if ctx.n_local == 1:
        # production layout: straight into the C ABI on the current stream
        stream = torch.cuda.current_stream()
        refresh = in_ptrs != layout.last_in or out_ptrs != layout.last_out
        for b in layout.buckets:
            if refresh:
                if b.plain:
                    b.in_arr[:] = [in_ptrs[i] for i in b.idx]
                    b.out_arr[:] = [out_ptrs[i] for i in b.idx]
                else:
                    b.in_arr[:] = [in_ptrs[i] + o for i, o in zip(b.idx, b.off)]
                    b.out_arr[:] = [out_ptrs[i] + o for i, o in zip(b.idx, b.off)]
            if kind == "ar":
                engine.allreduce_raw(b.plan, op, b.in_arr, b.out_arr, stream)
            else:
                engine.broadcast_raw(b.plan, src, b.out_arr, stream)
        layout.last_in, layout.last_out = in_ptrs, out_ptrs
        return
    for b in layout.buckets:                       # hosted (virtual) ranks meet, then ONE launch
        payload = {"in": [in_ptrs[i] + o for i, o in zip(b.idx, b.off)],
                   "out": [out_ptrs[i] + o for i, o in zip(b.idx, b.off)],
                   "stream": torch.cuda.current_stream()}

        def lead(payloads, plan=b.plan):
            rows_in = [p["in"] for p in payloads]
            rows_out = [p["out"] for p in payloads]
            if kind == "ar":
                return _launch_streams(engine, payloads, lambda s: engine.allreduce(plan, op, rows_in, rows_out, s))
            return _launch_streams(engine, payloads, lambda s: engine.broadcast(plan, src, rows_out, s))

        done = ctx.rendezvous(payload, lead)
        if done is not None:
            torch.cuda.current_stream().wait_event(done)


def _layout_for(ctx, engine: Engine, kind: str, tensors: tp.Sequence[torch.Tensor], op: int, key,
                lossy: bool = False) -> _Layout:
    full = (kind, key, lossy and engine.wire_bf16 and op == N.FX_AVG)
    layout = engine.layouts.get(full)
    if layout is None or any(b.plan.handle is None for b in layout.buckets):
        for _ in range(2):       # an arena eviction while building invalidates earlier buckets: redo once
            layout = _build_layout(engine, kind, tensors, op, lossy)
            if all(b.plan.handle is not None for b in layout.buckets):
                break
        engine.layouts[full] = layout
    return layout


def _reduce(ctx, ins: tp.Sequence[torch.Tensor], outs: tp.Optional[tp.Sequence[torch.Tensor]], op: int,
            key=None, lossy: bool = False) -> None:
    """Bucketed all-reduce of ``ins`` (into ``outs`` if given, else in place)."""
    engine = _engine(ctx, ins)
    if engine.host_only:
        _flat(ins[0], -1)                          # raises: no CPU fallback
    key = key if key is not None else _list_key(ins)
    layout = _layout_for(ctx, engine, "ar", ins, op, key, lossy)
    _dense_or_raise(ins, engine.device)
    if outs is not None:
        if _list_key(outs) != key:
            raise RuntimeError("output tensors do not match the reduced tensors")
        _dense_or_raise(outs, engine.device)
    in_ptrs = [t.data_ptr() for t in ins]
    _run_layout(ctx, engine, layout, in_ptrs, in_ptrs if outs is None else [t.data_ptr() for t in outs], op)


# ------------------------------------------------------------------------------------------
# collectives of the reference surface
# ------------------------------------------------------------------------------------------

_OPS = {
    distributed.ReduceOp.SUM: N.FX_SUM, distributed.ReduceOp.AVG: N.FX_AVG,
    distributed.ReduceOp.MAX: N.FX_MAX, distributed.ReduceOp.MIN: N.FX_MIN,
    distributed.ReduceOp.PRODUCT: N.FX_PROD,
}


def all_reduce(tensor: torch.Tensor, op=distributed.ReduceOp.SUM):
    """In-place all-reduce, no-op when not distributed (flashy/distrib.py:45-47)."""
    ctx = _context.current()
    if ctx.world == 1:
        return None
    fx_op = _OPS.get(op)
    if fx_op is None:
        raise RuntimeError(f"reduce op {op} is not supported by flashy_b200")
    # Host rendezvous first (a few microseconds in shared memory): a rank that is late -- rank 0
    # writing a checkpoint, say -- is waited for on the host, not by GPUs spinning on flags, and
    # ranks that disagree on the tensor's size are refused instead of corrupting each other.
    key = _list_key([tensor])
    engine = _engine(ctx, [tensor])
    if not (engine.check_mode == "plan" and ("ar", key, False) in engine.layouts):
        _check_number_of_params([tensor], key)
    _reduce(ctx, [tensor], None, fx_op, key)
    return None


def average_metrics(metrics: tp.Dict[str, float], count=1.):
    """Weighted average of a metric dict over ranks (flashy/distrib.py:50-62)."""
    ctx = _context.current()
    if ctx.world == 1:
        return metrics
    keys, values = zip(*metrics.items())
    device = "cuda" if torch.cuda.is_available() else "cpu"
    tensor = torch.tensor(list(values) + [1], device=device, dtype=torch.float32)
    tensor *= count
    all_reduce(tensor)
    averaged = (tensor[:-1] / tensor[-1]).cpu().tolist()
    return dict(zip(keys, averaged))


def wrap(model):
    """DDP comparator, kept as in the reference (flashy/distrib.py:65-75)."""
    if is_distributed():
        return DistributedDataParallel(model, device_ids=[torch.cuda.current_device()],
                                       output_device=torch.cuda.current_device())
    return model


class _ListEntry:
    """Remembered validation of one tensor list: what a repeat call must still match."""
    __slots__ = ("numels", "dtypes", "key", "layout")

    def __init__(self, numels, dtypes, key, layout):
        self.numels, self.dtypes, self.key, self.layout = numels, dtypes, key, layout


def _average(ctx, todo: tp.List[torch.Tensor]) -> None:
    """Count check + bucketed in-place mean of an already filtered list.

    Repeat calls with a list of the same length, element counts and dtypes (the per-step
    ``sync_gradients`` / ``average_tensors`` pattern) skip the key building, the layout lookup and
    the density re-validation: three list passes instead of eight."""
    engine = _engine(ctx, todo)
    numels = [t.numel() for t in todo]
    slot = (len(todo), numels[0], numels[-1], engine.wire_bf16)
    ent = engine.fast_lists.get(slot)
    if ent is not None and ent.numels == numels and ent.dtypes == [t.dtype for t in todo] \
            and all(b.plan.handle is not None for b in ent.layout.buckets):
        key, layout, known = ent.key, ent.layout, True
    else:
        key = _list_key(todo)
        known = ("ar", key, engine.wire_bf16) in engine.layouts
        if engine.host_only or not all(t.is_cuda for t in todo):
            _check_number_of_params(todo, key)     # as in the reference, the count check comes first
            _dense_or_raise(todo)                  # raises: no CPU fallback
        layout = _layout_for(ctx, engine, "ar", todo, N.FX_AVG, key, lossy=True)
        engine.fast_lists[slot] = _ListEntry(numels, [t.dtype for t in todo], key, layout)
        if len(engine.fast_lists) > 64:
            engine.fast_lists.pop(next(iter(engine.fast_lists)))
    if not (known and engine.check_mode == "plan"):
        _check_number_of_params(todo, key)
    ptrs = [t.data_ptr() for t in todo]
    if ptrs != layout.last_in:
        _dense_or_raise(todo, engine.device)
    _run_layout(ctx, engine, layout, ptrs, ptrs, N.FX_AVG)


def average_tensors(tensors: tp.Iterable[torch.Tensor]) -> None:
    """In-place mean over ranks of every float/complex tensor (flashy/distrib.py:96-111);
    other dtypes are ignored.  One bucketed kernel instead of a collective per tensor."""
    ctx = _context.current()
    if ctx.world == 1:
        return
    todo = [t for t in tensors if t.dtype.is_floating_point or t.dtype.is_complex]
    if not todo:
        return
    _average(ctx, todo)


def broadcast_tensors(tensors: tp.Iterable[torch.Tensor], src: int = 0) -> None:
    """Bit copy of rank ``src``'s float/complex tensors to every rank (flashy/distrib.py:114-127)."""
    ctx = _context.current()
    if ctx.world == 1:
        return
    todo = [t for t in tensors if t.dtype.is_floating_point or t.dtype.is_complex]
    if not todo:
        return
    key = _list_key(todo)
    _check_number_of_params(todo, key)
    engine = _engine(ctx, todo)
    if engine.host_only:
        _flat(todo[0], -1)
    layout = _layout_for(ctx, engine, "bc", todo, N.FX_SUM, key)
    _dense_or_raise(todo, engine.device)
    ptrs = [t.data_ptr() for t in todo]
    _run_layout(ctx, engine, layout, ptrs, ptrs, N.FX_SUM, src)


def broadcast_model(model: torch.nn.Module, src: int = 0) -> None:
    """Parameters then buffers from ``src`` (flashy/distrib.py:130-133)."""
    broadcast_tensors(model.parameters(), src)
    broadcast_tensors(model.buffers(), src)


def sync_gradients(params: tp.Iterable[torch.Tensor]) -> None:
    """Average the existing ``.grad`` of ``params`` over ranks (flashy/distrib.py:136-150)."""
    grads = [p.grad for p in params if p.grad is not None]
    average_tensors(grads)


def _sync_buffers(model: torch.nn.Module, sync_buffers: bool, average_buffers: bool) -> None:
    if not sync_buffers:
        return
    if average_buffers:
        average_tensors(_model_entry(model).float_buffers)
    else:
        broadcast_tensors(_model_entry(model).float_buffers)


def sync_buffers(model: torch.nn.Module, average: bool = True) -> None:
    """Convenience alias (an ADDITION: the reference has no such function, only the
    ``sync_buffers=`` / ``average_buffers=`` arguments of ``sync_model``)."""
    _sync_buffers(model, True, average)


class _ModelLists:
    __slots__ = ("params", "buffers", "float_buffers", "age", "fast", "epoch", "overlap")

    def __init__(self, model):
        self.params = list(model.parameters())
        self.buffers = list(model.buffers())
        self.float_buffers = [b for b in self.buffers if b.dtype.is_floating_point or b.dtype.is_complex]
        self.age = 0
        self.epoch = _struct_epoch[0]
        self.overlap: tp.Optional["_Overlap"] = None    # hook-driven bucket launches (see overlap())
        self.fast: tp.Dict[tp.Any, tp.Any] = {}     # (tag, n) -> (key, layout) of a validated tensor list


_model_cache: "weakref.WeakKeyDictionary[torch.nn.Module, _ModelLists]" = weakref.WeakKeyDictionary()
_MODEL_REVALIDATE = 256

# Structural edits of ANY module (``model.fc = nn.Linear(...)``, ``register_parameter``,
# ``register_buffer``, ``add_module``, assigning ``None`` over a child) go through torch's global
# registration hooks: they bump this counter, and a cached parameter list taken at an older count
# is thrown away on its next use.  The reference walks the module tree on every call
# (flashy/distrib.py:205-210); this keeps that behaviour observable at O(1) per call.
_struct_epoch = [0]


def _bump_struct_epoch(*_args) -> None:
    _struct_epoch[0] += 1


torch.nn.modules.module.register_module_parameter_registration_hook(_bump_struct_epoch)
torch.nn.modules.module.register_module_module_registration_hook(_bump_struct_epoch)
torch.nn.modules.module.register_module_buffer_registration_hook(_bump_struct_epoch)


def _model_entry(model: torch.nn.Module) -> _ModelLists:
    """``list(model.parameters())`` / ``list(model.buffers())`` walk the whole module tree on
    every call (for ResNet-18 a cost of the order of the all-reduce itself), so
    the lists are cached per model.  The cache is dropped whenever any module's structure was
    edited since it was taken (``_struct_epoch``), and re-derived every 256 uses as a backstop for
    edits that bypass the registration API (``del model.fc``, writes to ``_parameters``)."""
    entry = _model_cache.get(model)
    if entry is None or entry.epoch != _struct_epoch[0] or entry.age >= _MODEL_REVALIDATE:
        fresh = _ModelLists(model)
        if entry is not None and len(fresh.params) == len(entry.params) and len(fresh.buffers) == len(entry.buffers) \
                and all(a is b for a, b in zip(fresh.params, entry.params)) \
                and all(a is b for a, b in zip(fresh.buffers, entry.buffers)):
            # some OTHER module was built or edited since: this model is unchanged, keep its layouts and hooks
            entry.epoch, entry.age = fresh.epoch, 0
        else:
            if entry is not None and entry.overlap is not None:
                entry.overlap.remove()             # hooks of the stale parameter list
            entry = fresh
            _model_cache[model] = entry
    entry.age += 1
    return entry


def _model_lists(model: torch.nn.Module) -> tp.Tuple[tp.List[torch.Tensor], tp.List[torch.Tensor]]:
    entry = _model_entry(model)
    return entry.params, entry.buffers


def _average_cached(ctx, entry: _ModelLists, tag: str, todo: tp.List[torch.Tensor]) -> None:
    """``average_tensors(todo)`` for a list derived from a cached model: the dtype/numel key and
    the bucket layout are remembered per (tag, length) and re-validated whenever an address moves."""
    if not todo:
        return
    engine = _engine(ctx, todo)
    slot = (tag, len(todo), engine.wire_bf16)
    cached = entry.fast.get(slot)
    ptrs = [t.data_ptr() for t in todo]
    if cached is not None and (ptrs == cached[1].last_in or _list_key(todo) == cached[0]) \
            and all(b.plan.handle is not None for b in cached[1].buckets):
        key, layout = cached
        fresh = False
    else:
        key = _list_key(todo)
        if engine.host_only or not all(t.is_cuda for t in todo):
            _check_number_of_params(todo, key)
            _dense_or_raise(todo)
        layout = _layout_for(ctx, engine, "ar", todo, N.FX_AVG, key, lossy=True)
        entry.fast[slot] = (key, layout)
        fresh = True
    if fresh or engine.check_mode != "plan":
        _check_number_of_params(todo, key)
    if ptrs != layout.last_in:
        _dense_or_raise(todo, engine.device)
    _run_layout(ctx, engine, layout, ptrs, ptrs, N.FX_AVG)


def sync_model(model: torch.nn.Module, sync_buffers: bool = True, average_buffers: bool = True) -> None:
    """Call after ``backward()``: averages gradients and (by default) float buffers over ranks
    (flashy/distrib.py:193-210).  Returns once the work is enqueued on the current stream.

    With the default arguments the gradients and the float buffers of one dtype travel in ONE
    bucket, i.e. one kernel launch for the whole model (the reference: one all-reduce and one
    divide per tensor, in two passes).  With backward overlap enabled for ``model`` (``overlap()`` or
    ``FLASHY_B200_OVERLAP=1``) most of that bucket is already on the wire when this is called."""
    ctx = _context.current()
    if ctx.world == 1:
        return
    entry = _model_entry(model)
    if ctx.n_local == 1 and (entry.overlap is not None or _overlap_wanted(model)):
        if _sync_model_overlapped(ctx, model, entry, sync_buffers, average_buffers):
            return
    grads = [p.grad for p in entry.params]
    for g in grads:
        if g is None:
            grads = [g for g in grads if g is not None]
            break
    if sync_buffers and average_buffers:
        _average_cached(ctx, entry, "grads+buffers", grads + entry.float_buffers)
    else:
        _average_cached(ctx, entry, "grads", grads)
        if sync_buffers:
            broadcast_tensors(entry.float_buffers)


# ------------------------------------------------------------------------------------------
# backward overlap for plain ``sync_model`` users (opt-in; an ADDITION to the reference surface)
# ------------------------------------------------------------------------------------------

_overlap_models: "weakref.WeakKeyDictionary[torch.nn.Module, int]" = weakref.WeakKeyDictionary()


def overlap(model: torch.nn.Module, enabled: bool = True, bucket_mb: tp.Optional[float] = None) -> None:
    """Opt ``model`` into (or out of) backward overlap for ``sync_model``.

    NOT part of the reference surface.  The reference offers overlap only through the
    ``eager_sync_model`` context manager (flashy/distrib.py:213-224); a solver written as
    ``loss.backward(); distrib.sync_model(model); optim.step()`` (examples/cifar/solver.py:50-52)
    exposes the whole exchange.  With overlap enabled, parameters get post-accumulate-grad hooks:
    gradients are grouped in buckets of ``bucket_mb`` MiB (``FLASHY_B200_OVERLAP_BUCKET_MB``, 8) in
    the order backward produces them, and a bucket is averaged IN PLACE on the communicator's side
    stream the moment its last gradient has been accumulated, while backward continues.
    ``sync_model`` then only sends the tail bucket (the first registered parameters' gradients, at most
    ``FLASHY_B200_OVERLAP_TAIL_KB`` = 512 KiB, plus the float buffers) and makes the current stream wait.
    The buckets sent during backward use ``FLASHY_B200_OVERLAP_BLOCKS`` (32) CTAs instead of one per SM, so
    that the compute kernels keep the other SMs.  The same ``sync_model`` call sites keep working;
    with several backward passes per ``sync_model`` (gradient accumulation) every pass re-averages,
    which gives the same mean by linearity.  Only the one-rank-per-process layout overlaps; the
    setting ``FLASHY_B200_OVERLAP=1`` enables it for every model passed to ``sync_model``."""
    if enabled:
        cap = bucket_mb if bucket_mb is not None else float(os.environ.get("FLASHY_B200_OVERLAP_BUCKET_MB", "8"))
        _overlap_models[model] = max(1, int(cap * (1 << 20)))
    else:
        _overlap_models.pop(model, None)
        entry = _model_cache.get(model)
        if entry is not None and entry.overlap is not None:
            entry.overlap.remove()
            entry.overlap = None


def _overlap_wanted(model: torch.nn.Module) -> bool:
    if model in _overlap_models:
        return True
    if os.environ.get("FLASHY_B200_OVERLAP", "0") == "1":
        overlap(model, True)
        return True
    return False


class _Overlap:
    """Hook-driven bucket launches of one model (one-rank-per-process layout)."""

    def __init__(self, ctx, engine: Engine, entry: "_ModelLists", cap: int):
        self.ctx, self.engine = ctx, engine
        self.params = [p for p in entry.params if p.requires_grad]
        # The tail bucket -- what sync_model itself has to send, i.e. the exposed part -- is the FIRST
        # registered parameters (their gradients arrive last anyway), at most `tail` bytes; everything else
        # is grouped in reverse registration order ~ the order backward yields gradients, `cap` bytes each.
        tail = int(float(os.environ.get("FLASHY_B200_OVERLAP_TAIL_KB", "512")) * 1024)
        n_tail, fill = 0, 0
        for p in self.params:
            size = p.numel() * p.element_size()
            if n_tail and fill + size > tail:
                break
            if p.dtype != self.params[0].dtype:
                break
            n_tail, fill = n_tail + 1, fill + size
        self.buckets: tp.List[tp.List[int]] = []
        fill, last_dtype = 0, None
        for i in range(len(self.params) - 1, n_tail - 1, -1):
            p = self.params[i]
            size = p.numel() * p.element_size()
            if self.buckets and p.dtype == last_dtype and fill + size <= cap:
                self.buckets[-1].append(i)
                fill += size
            else:
                self.buckets.append([i])
                fill, last_dtype = size, p.dtype
        self.buckets.append(list(range(n_tail - 1, -1, -1)))
        self.where = {}
        for k, idxs in enumerate(self.buckets):
            for i in idxs:
                self.where[i] = k
        self.n_hook = len(self.buckets) - 1            # the last (tail) bucket waits for sync_model
        self.left = [len(b) for b in self.buckets]
        self.next = 0                                  # next bucket to launch (strictly in order)
        self.layouts: tp.Dict[tp.Any, tp.Tuple[tp.Any, _Layout]] = {}
        self.pending = False                           # something is in flight on the side stream
        self.checked = False
        self.launched = 0                              # hook launches since the last sync_model
        self.blocks = int(os.environ.get("FLASHY_B200_OVERLAP_BLOCKS", "32"))
        self.handles = [p.register_post_accumulate_grad_hook(lambda _p, i=i: self._on_grad(i))
                        for i, p in enumerate(self.params)]

    def remove(self) -> None:
        for h in self.handles:
            h.remove()
        self.handles = []

    # -- called on the autograd thread ------------------------------------------------------
    def _on_grad(self, i: int) -> None:
        k = self.where[i]
        if k >= self.n_hook:
            return                                     # tail bucket: sent by sync_model
        self.left[k] -= 1
        while self.left[self.next] <= 0:               # strictly in bucket order: same sequence on every rank
            k = self.next
            self.left[k] += len(self.buckets[k])
            self.next = (k + 1) % self.n_hook
            self.launched += 1
            self._launch(("hook", k), [self.params[j].grad for j in self.buckets[k]])
            if self.next == 0:
                break                                  # every hook bucket of this backward pass is out

    def _launch(self, tag, tensors: tp.List[torch.Tensor]) -> None:
        """Average ``tensors`` in place on the side stream, ordered after the current stream."""
        engine, side = self.engine, self.engine.side_stream
        ptrs = [t.data_ptr() for t in tensors]
        cached = self.layouts.get(tag)
        if cached is None or (ptrs != cached[1].last_in and _list_key(tensors) != cached[0]) \
                or any(b.plan.handle is None for b in cached[1].buckets):
            key = _list_key(tensors)
            # buckets launched DURING backward run on a small grid (FLASHY_B200_OVERLAP_BLOCKS, 32): every CTA of
            # the fused kernel takes a whole SM's shared memory, and one per SM would lock backward out.  What
            # sync_model itself sends (tail, held-back buckets) is exposed anyway and uses the full grid.
            engine.plan_blocks = self.blocks if tag[0] == "hook" else 0
            try:
                for _ in range(2):                             # an arena eviction while building: redo once
                    layout = _build_layout(engine, "ar", tensors, N.FX_AVG, lossy=True)
                    if all(b.plan.handle is not None for b in layout.buckets):
                        break
            finally:
                engine.plan_blocks = 0
            self.layouts[tag] = cached = (key, layout)
        layout = cached[1]
        if ptrs != layout.last_in:
            _dense_or_raise(tensors, engine.device)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        side.wait_event(ev)
        with torch.cuda.stream(side):
            _run_layout(self.ctx, engine, layout, ptrs, ptrs, N.FX_AVG)
        self.pending = True

    # -- called from sync_model ---------------------------------------------------------------
    def finish(self, extra: tp.List[torch.Tensor]) -> None:
        """Send what the hooks did not (buckets the in-order rule held back, the tail bucket, the
        float buffers), then make the current stream wait for the side stream."""
        if self.n_hook:
            if self.next != 0:
                late = range(self.next, self.n_hook)   # held back by the in-order rule (a gradient is missing)
            elif self.launched == 0:
                late = range(0, self.n_hook)           # nothing went out during backward
            else:
                late = range(0)
            for k in late:
                got = [self.params[j].grad for j in self.buckets[k] if self.params[j].grad is not None]
                if got:
                    self._launch(("late", k, len(got)), got)
            self.next, self.launched = 0, 0
            self.left = [len(b) for b in self.buckets]
        tail = [self.params[j].grad for j in self.buckets[-1] if self.params[j].grad is not None] + extra
        if tail:
            self._launch(("tail", len(tail)), tail)
        if self.pending:
            self._join()
            self.pending = False

    def _join(self) -> None:
        """The current stream waits for everything launched on the side stream."""
        done = torch.cuda.Event()
        done.record(self.engine.side_stream)
        torch.cuda.current_stream().wait_event(done)


def _sync_model_overlapped(ctx, model, entry: "_ModelLists", sync_buffers: bool, average_buffers: bool) -> bool:
    """The overlap flavour of ``sync_model``; False if overlap cannot be used for this call."""
    grads = [p.grad for p in entry.params if p.grad is not None]
    if not grads:
        return False
    engine = _engine(ctx, grads)
    if engine.host_only:
        return False
    st = entry.overlap
    if st is None:
        # first call: install the hooks (they act from the next backward on) and sync the ordinary way
        entry.overlap = _Overlap(ctx, engine, entry, _overlap_models[model])
        return False
    extra = entry.float_buffers if (sync_buffers and average_buffers) else []
    if engine.check_mode != "plan" or not st.checked:
        # one host rendezvous per call, as the reference's count checks (flashy/distrib.py:205-208)
        total = len(grads) + len(extra)
        _check_number_of_params(grads + extra, (0x6F766C70, total, len(st.buckets)))   # ints only: str hashes differ per process
        st.checked = True
    st.finish(extra)
    engine.poll()                                  # a flag-wait timeout of an earlier launch surfaces here, not a step later
    if sync_buffers and not average_buffers:
        broadcast_tensors(entry.float_buffers)
    return True


# ------------------------------------------------------------------------------------------
# eager path: start reducing bucket k while backward is still producing bucket k+1
# ------------------------------------------------------------------------------------------

class _EagerBucket:
    def __init__(self, plan, n: int, n_local: int):
        self.plan = plan
        self.rows = [[0] * n for _ in range(n_local)]
        self.left = [n] * n_local
        self.events: tp.List[tp.Any] = [None] * n_local
        self.ready = 0
        self.launched = False
        self.done = None


class _EagerSession:
    """State shared by the hosted ranks of one ``eager_sync_gradients`` context."""

    def __init__(self, engine: Engine, n_local: int, specs):
        self.engine = engine
        self.n_local = n_local
        self.lock = threading.Lock()
        self.buckets = [_EagerBucket(plan, n, n_local) for plan, n in specs]
        self.next_launch = 0

    def arrive(self, local: int, k: int, j: int, ptr: int) -> None:
        """Called from the autograd thread: gradient j of bucket k of hosted rank ``local`` exists."""
        with self.lock:
            b = self.buckets[k]
            b.rows[local][j] = ptr
            b.left[local] -= 1
            if b.left[local] == 0:
                ev = torch.cuda.Event()
                ev.record(torch.cuda.current_stream())
                b.events[local] = ev
                b.ready += 1
            self._launch_ready()

    def _launch_ready(self) -> None:
        # strictly in bucket order, so every process issues the same collective sequence
        while self.next_launch < len(self.buckets):
            b = self.buckets[self.next_launch]
            if b.ready < self.n_local:
                return
            side = self.engine.side_stream
            for ev in b.events:
                side.wait_event(ev)
            self.engine.allreduce_begin(b.plan, N.FX_AVG, b.rows, side)
            b.done = torch.cuda.Event()
            b.done.record(side)
            b.launched = True
            self.next_launch += 1


@contextmanager
def eager_sync_gradients(params: tp.Iterable[torch.Tensor]):
    """Context manager: gradients are reduced as they become available during the (single)
    ``backward()`` run inside it (flashy/distrib.py:153-190).  Gradients are grouped into
    buckets in expected arrival order; a bucket's reduce-scatter/all-gather is launched on a
    side stream the moment its last gradient exists, and on exit the averaged values are
    written over ``param.grad`` (``torch.div(grad, W, out=param.grad)`` in the reference)."""
    ctx = _context.current()
    if ctx.world == 1:
        yield
        return
    params = [p for p in params if p.requires_grad]
    _check_number_of_params(params)
    if not params:
        yield
        return
    engine = _engine(ctx, params)
    cap = int(os.environ.get("FLASHY_B200_EAGER_BUCKET_MB", "8")) << 20

    # ---- bucket layout: reverse registration order ~ order in which backward yields grads.
    # Cached per parameter list (the entry keeps the parameters alive, so the ids stay unique).
    cache_key = ("eager", tuple(map(id, params)), cap, engine.wire_bf16)
    cached = engine.layouts.get(cache_key)
    if cached is None:
        layout: tp.List[tp.Tuple[int, tp.List[int]]] = []       # (fx dtype, [param index])
        fill = 0
        for i in range(len(params) - 1, -1, -1):
            p = params[i]
            if p.dtype not in _DTYPES or not p.is_cuda:
                _flat(p, engine.device)                          # raises with the right message
            fx, mult = _DTYPES[p.dtype]
            size = p.numel() * mult * _ESIZE[fx]
            if layout and layout[-1][0] == fx and fill + size <= cap:
                layout[-1][1].append(i)
                fill += size
            else:
                layout.append((fx, [i]))
                fill = size
        where = {}
        for k, (_, idxs) in enumerate(layout):
            for j, i in enumerate(idxs):
                where[i] = (k, j)
        cached = (layout, where, list(params))
        engine.layouts[cache_key] = cached
        stale = [k for k in engine.layouts if isinstance(k, tuple) and k and k[0] == "eager"]
        for k in stale[:-8]:                                     # the entries pin their parameters: keep a few
            del engine.layouts[k]
    layout, where, _keepalive = cached

    def make_session(_payloads):
        specs = []
        for fx, idxs in layout:
            numels = tuple(params[i].numel() * _DTYPES[params[i].dtype][1] for i in idxs)
            wire = N.FX_BF16 if (engine.wire_bf16 and fx == N.FX_F32) else fx
            algo = engine.sharded_algo(wire, sum(numels) * _ESIZE[wire])
            # tag = bucket index: two buckets of identical shape (e.g. the three 512x512x3x3 convolutions
            # of ResNet-18's layer4 with a small bucket cap) must not share one plan -- a plan has ONE
            # pair of staging regions and one call counter, and all begins precede all finishes.
            specs.append((engine.get_plan("ar", numels, fx, wire, algo, tag=("eager", len(specs))), len(idxs)))
        return _EagerSession(engine, ctx.n_local, specs)

    session: _EagerSession = ctx.rendezvous(None, make_session)
    local = ctx.local
    waiting = set(range(len(params)))
    fired: tp.Dict[int, torch.Tensor] = {}

    def _callback(i: int, grad: torch.Tensor):
        if i not in waiting:
            raise RuntimeError(f"We got a gradient twice for parameter {params[i]}.")
        data = grad.data
        if not _dense(data):
            data = data.contiguous()
        fired[i] = data                                         # keep the storage alive until exit
        waiting.remove(i)
        k, j = where[i]
        session.arrive(local, k, j, data.data_ptr())

    hooks = [p.register_hook(lambda g, i=i: _callback(i, g)) for i, p in enumerate(params)]
    try:
        yield
    finally:
        for hook in hooks:
            hook.remove()
        _check_number_of_params([params[i] for i in sorted(waiting)])   # same leftovers everywhere
        stream = torch.cuda.current_stream()
        for k, (fx, idxs) in enumerate(layout):
            bucket = session.buckets[k]
            complete = all(i in fired for i in idxs)
            if complete:
                def lead(payloads, bucket=bucket):
                    with session.lock:
                        session._launch_ready()
                    assert bucket.launched
                    outs = [p["out"] for p in payloads]
                    streams = {p["stream"].cuda_stream for p in payloads}
                    if len(streams) == 1:
                        payloads[0]["stream"].wait_event(bucket.done)
                        engine.allreduce_finish(bucket.plan, outs, payloads[0]["stream"])
                        return None
                    engine.allreduce_finish(bucket.plan, outs, engine.side_stream)
                    done = torch.cuda.Event()
                    done.record(engine.side_stream)
                    return done
                outs = []
                for i in idxs:
                    assert params[i].grad is not None
                    outs.append(_flat(params[i].grad.data, engine.device)[1])
                done = ctx.rendezvous({"out": outs, "stream": stream}, lead)
                if done is not None:
                    stream.wait_event(done)
            else:
                # Some gradients of this bucket never arrived (unused parameters): reduce the ones
                # that did with an ordinary fused launch.  The leftovers were checked to agree.
                got = [i for i in idxs if i in fired]

                def skip(_payloads, k=k):                        # keep the launch order identical
                    with session.lock:
                        if session.next_launch == k:
                            session.next_launch += 1
                ctx.rendezvous(None, skip)
                if got:
                    for i in got:
                        assert params[i].grad is not None
                    _reduce(ctx, [fired[i] for i in got], [params[i].grad.data for i in got], N.FX_AVG, lossy=True)
        fired.clear()
        engine.poll()                                  # device-side timeouts of the side-stream launches raise here


@contextmanager
def eager_sync_model(model: torch.nn.Module, sync_buffers: bool = True, average_buffers: bool = True):
    """``sync_model`` with the gradient part overlapped with backward (flashy/distrib.py:213-224)."""
    with eager_sync_gradients(model.parameters()):
        yield
    _sync_buffers(model, sync_buffers, average_buffers)


# ------------------------------------------------------------------------------------------
# data loading / objects / barrier  (stay Python: north_star)
# ------------------------------------------------------------------------------------------

def loader(dataset, *args, shuffle=False, klass=DataLoader, **kwargs):
    """Sharded dataloader (flashy/distrib.py:227-243): ``DistributedSampler`` when
    ``shuffle=True``, a strided ``Subset`` (no duplicated samples) otherwise."""
    ctx = _context.current()
    if ctx.world == 1:
        return klass(dataset, *args, shuffle=shuffle, **kwargs)
    if shuffle:
        sampler = DistributedSampler(dataset, num_replicas=ctx.world, rank=ctx.rank)
        return klass(dataset, *args, **kwargs, sampler=sampler)
    shard = Subset(dataset, list(range(ctx.rank, len(dataset), ctx.world)))
    return klass(shard, *args, shuffle=shuffle, **kwargs)


def broadcast_object(obj: tp.Any = None, src: int = 0, device=None):
    """Share a picklable object from rank ``src`` (flashy/distrib.py:246-269).  Every rank,
    the source included, returns the unpickled copy (as the reference effectively does).  The
    pickle travels through the communicator's shared-memory fabric, not ``torch.distributed``."""
    ctx = _context.current()
    if ctx.world == 1:
        return obj
    engine = ctx.cached_engine()
    if engine is None:
        engine = ctx.engine_for(torch.cuda.current_device() if N.cuda_available() else None,
                                host_only=not N.cuda_available())
    blob = pickle.dumps(obj) if ctx.rank == src else None
    return pickle.loads(engine.host_broadcast(ctx.local, src, blob))


def barrier() -> None:
    """All ranks wait for each other on the host (flashy/distrib.py:272-276)."""
    ctx = _context.current()
    if ctx.world == 1:
        return
    engine = ctx.engine_for(torch.cuda.current_device() if N.cuda_available() else None,
                            host_only=not N.cuda_available())
    engine.host_barrier(ctx.local)
