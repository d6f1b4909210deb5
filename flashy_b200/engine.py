"""Host engine between ``flashy_b200.distrib`` and the C ABI (``include/flashy_b200.h``).

Responsibilities: communicator bootstrap (``torch.distributed`` is used ONLY to move the
export blobs once), bucket planning and the plan cache, the host-side count check, and the
launch bookkeeping (streams, pointer rows).  No tensor arithmetic happens here: data only
moves inside the CUDA kernels of ``libflashy_b200.so``.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
import typing as tp

import torch

from . import _native as N

_DTYPES = {
    torch.float32: (N.FX_F32, 1), torch.bfloat16: (N.FX_BF16, 1), torch.float16: (N.FX_F16, 1),
    torch.float64: (N.FX_F64, 1), torch.int32: (N.FX_I32, 1), torch.int64: (N.FX_I64, 1),
    torch.complex64: (N.FX_F32, 2), torch.complex128: (N.FX_F64, 2),   # complex = pairs of reals
}
_ESIZE = {N.FX_F32: 4, N.FX_BF16: 2, N.FX_F16: 2, N.FX_F64: 8, N.FX_I32: 4, N.FX_I64: 8, N.FX_U8: 1}


def _env_int(name: str, default: int) -> int:
    v = os.environ.get(name)
    return int(v) if v else default


def _dense(t: torch.Tensor) -> bool:
    if t.is_contiguous():
        return True
    if t.dim() == 4 and t.is_contiguous(memory_format=torch.channels_last):
        return True
    if t.dim() == 5 and t.is_contiguous(memory_format=torch.channels_last_3d):
        return True
    return False


class Plan:
    __slots__ = ("handle", "info", "n", "key", "engine")

    def __init__(self, engine: "Engine", key, numels: tp.Sequence[int], dtype: int, wire: int, algo: int):
        arr = (C.c_int64 * len(numels))(*numels)
        handle = C.c_void_p()
        N.check(N.lib.fx_plan_create(engine.comm, engine.world, arr, len(numels), dtype, wire, algo, C.byref(handle)))
        self.handle = handle
        self.info = N.PlanInfo()
        N.check(N.lib.fx_plan_get_info(handle, C.byref(self.info)))
        self.n = len(numels)
        self.key = key
        self.engine = engine

    def destroy(self):
        if self.handle:
            N.lib.fx_plan_destroy(self.handle)
            self.handle = None


class Engine:
    """One communicator: hosts ``n_local`` consecutive ranks of the world on one device."""

    def __init__(self, n_local: int = 1, device: tp.Optional[int] = None,
                 proc_rank: int = 0, proc_world: int = 1, arena_mb: tp.Optional[int] = None,
                 host_only: bool = False):
        # Host-only communicators carry the rendezvous / count-check fabric but no device side:
        # any attempt to move tensor data through them fails loudly (no CPU fallback).
        self.host_only = host_only or not N.cuda_available()
        self.n_local = n_local
        self.proc_rank, self.proc_world = proc_rank, proc_world
        self.world = proc_world * n_local
        self.rank0 = proc_rank * n_local
        if self.world > N.FX_MAX_WORLD:
            raise RuntimeError(f"world size {self.world} exceeds the single-NVSwitch-domain limit {N.FX_MAX_WORLD}")
        if self.host_only:
            self.device = -1
        else:
            self.device = torch.cuda.current_device() if device is None else device
        arena = (arena_mb if arena_mb is not None else _env_int("FLASHY_B200_ARENA_MB", 1024)) << 20
        self.comm = C.c_void_p()
        self.multicast_error: tp.Optional[str] = None
        self._create(arena, N.FX_COMM_HOST_ONLY if self.host_only else N.FX_COMM_MEM_AUTO)
        if proc_world > 1:
            self._connect(arena)
        self.info = N.CommInfo()
        N.check(N.lib.fx_comm_get_info(self.comm, C.byref(self.info)))
        self.plans: tp.Dict[tp.Any, Plan] = {}
        self.lock = threading.RLock()
        self.bucket_cap = min(_env_int("FLASHY_B200_BUCKET_MB", 128) << 20, arena // 8)
        self.check_mode = os.environ.get("FLASHY_B200_CHECK", "always")
        self.wire_bf16 = os.environ.get("FLASHY_B200_WIRE", "") == "bf16"
        # hosted ranks average through fx_allreduce_hosted; 0 keeps the Python rendezvous (A/B runs and tests)
        self.hosted_launch = os.environ.get("FLASHY_B200_HOSTED_LAUNCH", "1") != "0"
        self.side_stream = None if self.host_only else torch.cuda.Stream(device=self.device)
        self.layouts: tp.Dict[tp.Any, tp.Any] = {}       # bucket layouts of tensor lists (distrib.py)
        self.fast_lists: tp.Dict[tp.Any, tp.Any] = {}    # validated repeat lists of average_tensors (distrib.py)
        self.plan_blocks = 0                             # > 0: grid cap for the plans created next (overlap buckets)
        self.multicast = bool(self.info.multicast)
        self.nvls_min = _env_int("FLASHY_B200_NVLS_MIN", 512 << 10)
        self.profile = False
        self.timings: tp.List[tp.Tuple[tp.Any, tp.Any, tp.Any]] = []

    # ------------------------------------------------------------------ bootstrap
    def _create(self, arena: int, flags: int) -> None:
        N.check(N.lib.fx_comm_create(self.world, self.rank0, self.n_local, self.device, arena, flags, C.byref(self.comm)))

    def _export(self) -> bytes:
        size = C.c_size_t()
        N.check(N.lib.fx_comm_export(self.comm, None, 0, C.byref(size)))
        buf = C.create_string_buffer(size.value)
        N.check(N.lib.fx_comm_export(self.comm, buf, size.value, C.byref(size)))
        return buf.raw

    def _connect(self, arena: int) -> None:
        import torch.distributed as dist
        kinds: tp.List[tp.Any] = [None] * self.proc_world
        me = N.CommInfo()
        N.check(N.lib.fx_comm_get_info(self.comm, C.byref(me)))
        dist.all_gather_object(kinds, int(me.mem_kind))
        if len(set(kinds)) != 1 and not self.host_only:   # some rank could not export VMM handles: all use cudaIpc
            N.lib.fx_comm_destroy(self.comm)
            self.comm = C.c_void_p()
            self._create(arena, N.FX_COMM_MEM_IPC)
        blobs: tp.List[tp.Any] = [None] * self.proc_world
        dist.all_gather_object(blobs, self._export())
        joined = b"".join(blobs)
        N.check(N.lib.fx_comm_connect(self.comm, joined, len(blobs[0]), self.proc_world))
        dist.barrier()
        # NVLS: bind every arena to one NVSwitch multicast object (collective; quietly stays on the
        # peer-to-peer kernels where the system cannot do it).
        if self.n_local == 1 and not self.host_only and os.environ.get("FLASHY_B200_NVLS", "1") != "0":
            rc = N.lib.fx_comm_enable_multicast(self.comm, joined, len(blobs[0]), self.proc_world)
            if rc != N.FX_OK:
                self.multicast_error = N.lib.fx_last_error().decode(errors="replace")
        dist.barrier()

    def close(self) -> None:
        """Tear the communicator down.  Peers may still be reading this rank's arena in their last
        kernel, so: finish our own work, wait until every process got here, only then unmap."""
        if self.comm and not self.host_only:
            try:
                torch.cuda.synchronize(self.device)
                if self.proc_world > 1 and self.n_local == 1:
                    N.lib.fx_host_barrier(self.comm, 0, 10.0)       # bounded: a dead peer must not hang exit
            except Exception:      # noqa: BLE001 - best effort at shutdown
                pass
        with self.lock:
            for plan in self.plans.values():
                plan.destroy()
            self.plans.clear()
            if self.comm:
                N.lib.fx_comm_destroy(self.comm)
                self.comm = C.c_void_p()

    # ------------------------------------------------------------------ host rendezvous
    def host_exchange(self, local: int, count: int, signature: int) -> tp.Tuple[int, bool]:
        total, equal = C.c_int64(), C.c_int()
        N.check(N.lib.fx_host_exchange(self.comm, local, count, signature & (2 ** 64 - 1),
                                       C.byref(total), C.byref(equal), 0.0))
        return total.value, bool(equal.value)

    def host_barrier(self, local: int) -> None:
        N.check(N.lib.fx_host_barrier(self.comm, local, 0.0))

    def host_broadcast(self, local: int, src: int, payload: tp.Optional[bytes]) -> bytes:
        """Bytes from rank ``src`` to every rank over the shared-memory fabric (size first)."""
        size = C.c_uint64(len(payload) if payload is not None else 0)
        N.check(N.lib.fx_host_broadcast(self.comm, local, src, C.byref(size), 8, 0.0))
        buf = C.create_string_buffer(payload, size.value) if payload is not None else C.create_string_buffer(size.value)
        N.check(N.lib.fx_host_broadcast(self.comm, local, src, buf, size.value, 0.0))
        return buf.raw[:size.value]

    # ------------------------------------------------------------------ planning
    def get_plan(self, kind: str, numels: tp.Tuple[int, ...], dtype: int, wire: int, algo: int = N.FX_ALGO_AUTO,
                 tag: tp.Any = None) -> Plan:
        """Cached plan of one bucket.  ``tag`` distinguishes plans of identical shape that must not
        share staging memory (several begin/finish buckets in flight at once).  ``self.plan_blocks``
        (set around the call by the overlap code) caps the grid of newly created plans."""
        if self.host_only:
            raise RuntimeError("flashy_b200: no CUDA device in this process; tensor collectives have no CPU fallback")
        if self.plan_blocks:
            tag = (tag, "blocks", self.plan_blocks)
        key = (kind, numels, dtype, wire, algo) if tag is None else (kind, numels, dtype, wire, algo, tag)
        with self.lock:
            plan = self.plans.get(key)
            if plan is not None:
                return plan
            N.check(N.lib.fx_comm_set_plan_blocks(self.comm, int(self.plan_blocks)))
            try:
                plan = Plan(self, key, numels, dtype, wire, algo)
            except N.NativeError as err:
                if err.code != N.FX_ERR_TOO_BIG or not self.plans:
                    raise
                # Arena exhausted: every rank reaches this point for the same plan (plans are
                # created in the same order everywhere), so dropping the cache is collective-safe.
                torch.cuda.synchronize(self.device)
                for old in self.plans.values():
                    old.destroy()
                self.plans.clear()
                self.layouts.clear()
                self.fast_lists.clear()
                plan = Plan(self, key, numels, dtype, wire, algo)
            self.plans[key] = plan
            return plan

    # ------------------------------------------------------------------ launches
    # `stream` arguments are torch.cuda.Stream objects.  With `self.profile` set, every
    # all-reduce launch is bracketed by CUDA events on its launch stream (bench.py reads
    # `self.timings` after a synchronize): (plan key, start event, end event).
    @staticmethod
    def _rows(rows: tp.Sequence[tp.Sequence[int]]):
        flat = [p for row in rows for p in row]
        return (C.c_void_p * len(flat))(*flat)

    def _timed(self, plan: Plan, stream, call) -> None:
        if not self.profile:
            call()
            return
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        self.timings.append((plan.key, e0, e1))

    def allreduce(self, plan: Plan, op: int, in_rows, out_rows, stream) -> None:
        ins, outs = self._rows(in_rows), self._rows(out_rows)
        self._timed(plan, stream, lambda: N.check(N.lib.fx_allreduce(plan.handle, op, ins, outs, stream.cuda_stream)))

    def allreduce_raw(self, plan: Plan, op: int, in_arr, out_arr, stream) -> None:
        """Fast path of the one-rank-per-process layout: prebuilt ctypes pointer arrays."""
        if self.profile:
            self._timed(plan, stream, lambda: N.check(N.lib.fx_allreduce(plan.handle, op, in_arr, out_arr, stream.cuda_stream)))
            return
        rc = N.lib.fx_allreduce(plan.handle, op, in_arr, out_arr, stream.cuda_stream)
        if rc:
            N.check(rc)

    def broadcast_raw(self, plan: Plan, src: int, arr, stream) -> None:
        rc = N.lib.fx_broadcast(plan.handle, src, arr, stream.cuda_stream)
        if rc:
            N.check(rc)

    def allreduce_begin(self, plan: Plan, op: int, in_rows, stream) -> None:
        ins = self._rows(in_rows)
        self._timed(plan, stream, lambda: N.check(N.lib.fx_allreduce_begin(plan.handle, op, ins, stream.cuda_stream)))

    def allreduce_finish(self, plan: Plan, out_rows, stream) -> None:
        N.check(N.lib.fx_allreduce_finish(plan.handle, self._rows(out_rows), stream.cuda_stream))

    def broadcast(self, plan: Plan, src: int, rows, stream) -> None:
        N.check(N.lib.fx_broadcast(plan.handle, src, self._rows(rows), stream.cuda_stream))

    def device_barrier(self, stream) -> None:
        N.check(N.lib.fx_barrier(self.comm, stream.cuda_stream))

    def sharded_algo(self, dtype: int, wire_bytes: int) -> int:
        """Algorithm for a begin/finish (eager) bucket: never one-shot."""
        if (self.multicast and dtype in (N.FX_F32, N.FX_BF16, N.FX_F16) and wire_bytes >= self.nvls_min
                and self.world >= _env_int("FLASHY_B200_NVLS_MIN_WORLD", 4)):
            return N.FX_ALGO_NVLS
        return N.FX_ALGO_TWO_SHOT

    def abort(self) -> None:
        """Poison the communicator world-wide: blocked host waits fail instead of hanging."""
        if self.comm:
            N.lib.fx_comm_abort(self.comm)

    def poll(self) -> None:
        N.check(N.lib.fx_comm_poll(self.comm))

    def native_launches(self) -> int:
        """Kernels launched by libflashy_b200.so through this communicator (counted in C)."""
        info = N.CommInfo()
        N.check(N.lib.fx_comm_get_info(self.comm, C.byref(info)))
        return int(info.launches)
