"""The reference's collective call sequence over ``torch.distributed`` (TEST INFRASTRUCTURE).

A behavioural restatement -- not a copy -- of the reference's ``flashy/distrib.py``: for each
public function of the hot path, the same collectives in the same order with the same
host synchronisation points, issued through whatever process group ``torch.distributed``
was initialised with (gloo on CPU here; NCCL on a GPU box).  It serves as

* the multi-process checker for the CUDA path (same seeded inputs on both sides), and
* the timed CPU baseline / ``bench.py --impl reference`` arm (gloo on the host cores).

It is pinned against the unmodified reference by ``tests/test_oracle.py`` through
``tests/golden/*.npz`` (see ``tests/golden/make_golden.py``).

The product (``flashy_b200``) never imports this module.
"""
from __future__ import annotations

import contextlib
import pickle
import typing as tp

import torch
import torch.distributed as dist
from torch.utils.data import DataLoader, Subset
from torch.utils.data.distributed import DistributedSampler


def _world() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def _rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def _reducible(t: torch.Tensor) -> bool:
    # reference flashy/distrib.py:92-93
    return t.is_floating_point() or t.is_complex()


class RefDistrib:
    """Reference semantics, one method per reference function (file:line in each docstring)."""

    # ---- rank helpers: flashy/distrib.py:21,37-42 -------------------------------------
    rank = staticmethod(_rank)
    world_size = staticmethod(_world)

    @staticmethod
    def is_rank_zero() -> bool:
        return _rank() == 0

    @staticmethod
    def is_distributed() -> bool:
        return _world() > 1

    # ---- flashy/distrib.py:45-47 -----------------------------------------------------
    @staticmethod
    def all_reduce(tensor: torch.Tensor, op=dist.ReduceOp.SUM):
        if _world() > 1:
            return dist.all_reduce(tensor, op)
        return None

    # ---- flashy/distrib.py:78-89 -----------------------------------------------------
    @classmethod
    def check_count(cls, tensors: tp.Sequence[torch.Tensor]) -> None:
        world = _world()
        if world == 1 or len(tensors) == 0:
            return
        n = len(tensors)
        probe = torch.full((1,), n, device=tensors[0].device, dtype=torch.long)
        cls.all_reduce(probe)
        if probe.item() != n * world:          # host sync, as in the reference
            raise RuntimeError(
                f"Mismatch in number of params: ours is {n}, at least one worker has a different one.")

    # ---- flashy/distrib.py:96-111 ----------------------------------------------------
    @classmethod
    def average_tensors(cls, tensors: tp.Iterable[torch.Tensor]) -> None:
        world = _world()
        if world == 1:
            return
        todo = [t for t in tensors if _reducible(t)]
        cls.check_count(todo)
        pending = [(t, dist.all_reduce(t.data, op=dist.ReduceOp.SUM, async_op=True)) for t in todo]
        for t, work in pending:
            work.wait()
            t.data /= world

    # ---- flashy/distrib.py:114-127 ---------------------------------------------------
    @classmethod
    def broadcast_tensors(cls, tensors: tp.Iterable[torch.Tensor], src: int = 0) -> None:
        if _world() == 1:
            return
        todo = [t for t in tensors if _reducible(t)]
        cls.check_count(todo)
        works = [dist.broadcast(t.data, src=src, async_op=True) for t in todo]
        for work in works:
            work.wait()

    # ---- flashy/distrib.py:130-133 ---------------------------------------------------
    @classmethod
    def broadcast_model(cls, model: torch.nn.Module, src: int = 0) -> None:
        cls.broadcast_tensors(model.parameters(), src)
        cls.broadcast_tensors(model.buffers(), src)

    # ---- flashy/distrib.py:136-150 ---------------------------------------------------
    @classmethod
    def sync_gradients(cls, params: tp.Iterable[torch.Tensor]) -> None:
        cls.average_tensors([p.grad for p in params if p.grad is not None])

    # ---- flashy/distrib.py:193-210 ---------------------------------------------------
    @classmethod
    def sync_model(cls, model, sync_buffers: bool = True, average_buffers: bool = True) -> None:
        cls.sync_gradients(model.parameters())
        cls._sync_buffers(model, sync_buffers, average_buffers)

    @classmethod
    def _sync_buffers(cls, model, sync_buffers: bool, average_buffers: bool) -> None:
        if not sync_buffers:
            return
        if average_buffers:
            cls.average_tensors(model.buffers())
        else:
            cls.broadcast_tensors(model.buffers())

    # ---- flashy/distrib.py:153-190 ---------------------------------------------------
    @classmethod
    @contextlib.contextmanager
    def eager_sync_gradients(cls, params: tp.Iterable[torch.Tensor]):
        world = _world()
        if world == 1:
            yield
            return
        watched = [p for p in params if p.requires_grad]
        cls.check_count(watched)
        outstanding = {id(p): p for p in watched}
        fired: tp.List[tp.Tuple[torch.Tensor, torch.Tensor, tp.Any]] = []

        def on_grad(param, grad):
            if id(param) not in outstanding:
                raise RuntimeError(f"We got a gradient twice for parameter {param}.")
            work = dist.all_reduce(grad.data, op=dist.ReduceOp.SUM, async_op=True)
            fired.append((param, grad.data, work))
            del outstanding[id(param)]

        handles = [p.register_hook(lambda g, p=p: on_grad(p, g)) for p in watched]
        try:
            yield
        finally:
            for h in handles:
                h.remove()
            cls.check_count(list(outstanding.values()))
            for param, grad, work in fired:
                work.wait()
                assert param.grad is not None
                torch.div(grad, world, out=param.grad)     # overwrite, :190

    # ---- flashy/distrib.py:213-224 ---------------------------------------------------
    @classmethod
    @contextlib.contextmanager
    def eager_sync_model(cls, model, sync_buffers: bool = True, average_buffers: bool = True):
        with cls.eager_sync_gradients(model.parameters()):
            yield
        cls._sync_buffers(model, sync_buffers, average_buffers)

    # ---- flashy/distrib.py:50-62 -----------------------------------------------------
    @classmethod
    def average_metrics(cls, metrics: tp.Dict[str, float], count: float = 1.0):
        if _world() == 1:
            return metrics
        names = list(metrics.keys())
        device = "cuda" if torch.cuda.is_available() else "cpu"
        packed = torch.tensor([metrics[k] for k in names] + [1], device=device, dtype=torch.float32)
        packed *= count
        cls.all_reduce(packed)
        means = (packed[:-1] / packed[-1]).cpu().tolist()
        return dict(zip(names, means))

    # ---- flashy/distrib.py:227-243 ---------------------------------------------------
    @staticmethod
    def loader(dataset, *args, shuffle: bool = False, klass=DataLoader, **kwargs):
        world = _world()
        if world == 1:
            return klass(dataset, *args, shuffle=shuffle, **kwargs)
        if shuffle:
            return klass(dataset, *args, **kwargs, sampler=DistributedSampler(dataset))
        shard = Subset(dataset, list(range(_rank(), len(dataset), world)))
        return klass(shard, *args, shuffle=shuffle, **kwargs)

    # ---- flashy/distrib.py:246-269 ---------------------------------------------------
    @staticmethod
    def broadcast_object(obj: tp.Any = None, src: int = 0, device=None):
        if _world() == 1:
            return obj
        if device is None:
            device = "cuda" if torch.cuda.is_available() else "cpu"
        size = torch.empty(1, device=device, dtype=torch.long)
        payload = None
        if _rank() == src:
            payload = bytearray(pickle.dumps(obj))
            size[0] = len(payload)
        dist.broadcast(size, src=src)
        if _rank() == src:
            buf = torch.frombuffer(payload, dtype=torch.uint8).to(device=device)
        else:
            buf = torch.empty(int(size[0].item()), device=device, dtype=torch.uint8)
        dist.broadcast(buf, src=src)
        # The reference compares the *function* `rank` with `src` (:267), which is always
        # unequal, so every rank -- the source included -- unpickles the payload.
        return pickle.loads(buf.cpu().numpy().tobytes())

    # ---- flashy/distrib.py:272-276 ---------------------------------------------------
    @staticmethod
    def barrier() -> None:
        if _world() > 1:
            dist.barrier()
