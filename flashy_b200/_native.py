"""ctypes binding of ``libflashy_b200.so`` (C ABI declared in ``include/flashy_b200.h``).

The library is built in-tree by ``__graft_entry__.build()`` / ``make -C flashy_b200/csrc``.
There is no Python or CPU fallback: if the shared object is missing, importing this module
raises, and every collective on the product path fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

LIB_PATH = Path(__file__).resolve().parent / "libflashy_b200.so"

FX_OK = 0
FX_ERR_INVALID, FX_ERR_CUDA, FX_ERR_UNSUPPORTED, FX_ERR_TOO_BIG = -1, -2, -3, -4
FX_ERR_MISMATCH, FX_ERR_TIMEOUT, FX_ERR_SYS, FX_ERR_STATE = -5, -6, -7, -8

FX_F32, FX_BF16, FX_F16, FX_F64, FX_I32, FX_I64, FX_U8 = range(7)
FX_SUM, FX_AVG, FX_MAX, FX_MIN, FX_PROD = range(5)
FX_ALGO_AUTO, FX_ALGO_ONE_SHOT, FX_ALGO_TWO_SHOT, FX_ALGO_NVLS = range(4)
FX_COMM_MEM_AUTO, FX_COMM_MEM_VMM, FX_COMM_MEM_IPC, FX_COMM_HOST_ONLY = 0, 1, 2, 4
FX_MAX_WORLD = 16

ALGO_NAMES = {FX_ALGO_ONE_SHOT: "one_shot", FX_ALGO_TWO_SHOT: "two_shot", FX_ALGO_NVLS: "nvls"}
KERNEL_NAMES = {1: "k_one_shot", 2: "k_two_shot", 3: "k_nvls", 4: "k_pipe<NVLS=false>", 5: "k_pipe<NVLS=true>",
                6: "k_fuse<NVLS=false>", 7: "k_fuse<NVLS=true>"}

# Every symbol include/flashy_b200.h declares (tests check the .so exports all of them).
EXPORTS = (
    "fx_last_error", "fx_abi_version", "fx_cuda_available",
    "fx_comm_create", "fx_comm_export", "fx_comm_connect", "fx_comm_enable_multicast",
    "fx_comm_get_info", "fx_comm_set_plan_blocks", "fx_comm_get_pointers", "fx_comm_trace_read", "fx_comm_poll", "fx_comm_abort", "fx_comm_destroy",
    "fx_host_exchange", "fx_host_barrier", "fx_host_broadcast",
    "fx_plan_create", "fx_plan_get_info", "fx_plan_offsets", "fx_plan_destroy",
    "fx_allreduce", "fx_allreduce_hosted", "fx_broadcast", "fx_allreduce_begin", "fx_allreduce_finish", "fx_barrier",
)


class CommInfo(C.Structure):
    _fields_ = [
        ("abi_version", C.c_int), ("world", C.c_int), ("rank0", C.c_int), ("n_local", C.c_int),
        ("device", C.c_int), ("mem_kind", C.c_int), ("connected", C.c_int), ("multicast", C.c_int),
        ("sm_count", C.c_int), ("max_blocks", C.c_int),
        ("arena_bytes", C.c_uint64), ("arena_used", C.c_uint64), ("launches", C.c_uint64),
    ]


class PlanInfo(C.Structure):
    _fields_ = [
        ("n_tensors", C.c_int), ("dtype", C.c_int), ("wire_dtype", C.c_int), ("world", C.c_int),
        ("algo", C.c_int), ("grid_x", C.c_int), ("block", C.c_int),
        ("total_elems", C.c_uint64), ("padded_elems", C.c_uint64), ("shard_elems", C.c_uint64),
        ("wire_bytes", C.c_uint64), ("region_offset", C.c_uint64 * 2), ("signature", C.c_uint64),
        ("kernel", C.c_int), ("chunks", C.c_int), ("chunk_bytes", C.c_uint64),
    ]


class NativeError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f"flashy_b200 native error {code}: {message}")
        self.code = code


def _load() -> C.CDLL:
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C flashy_b200/csrc`. flashy_b200 has no CPU / PyTorch fallback.")
    lib = C.CDLL(str(LIB_PATH), mode=getattr(os, "RTLD_NOW", 2))
    vp, i, u64, sz = C.c_void_p, C.c_int, C.c_uint64, C.c_size_t
    P = C.POINTER
    sigs = {
        "fx_last_error": (C.c_char_p, []),
        "fx_abi_version": (i, []),
        "fx_cuda_available": (i, []),
        "fx_comm_create": (i, [i, i, i, i, sz, C.c_uint, P(vp)]),
        "fx_comm_export": (i, [vp, vp, sz, P(sz)]),
        "fx_comm_connect": (i, [vp, vp, sz, i]),
        "fx_comm_enable_multicast": (i, [vp, vp, sz, i]),
        "fx_comm_get_info": (i, [vp, P(CommInfo)]),
        "fx_comm_set_plan_blocks": (i, [vp, i]),
        "fx_comm_get_pointers": (i, [vp, P(vp), P(vp), P(u64), P(u64)]),
        "fx_comm_trace_read": (i, [vp, P(u64), sz, P(sz)]),
        "fx_comm_poll": (i, [vp]),
        "fx_comm_abort": (i, [vp]),
        "fx_comm_destroy": (None, [vp]),
        "fx_host_exchange": (i, [vp, i, C.c_int64, u64, P(C.c_int64), P(i), C.c_double]),
        "fx_host_barrier": (i, [vp, i, C.c_double]),
        "fx_host_broadcast": (i, [vp, i, i, vp, sz, C.c_double]),
        "fx_plan_create": (i, [vp, i, P(C.c_int64), i, i, i, i, P(vp)]),
        "fx_plan_get_info": (i, [vp, P(PlanInfo)]),
        "fx_plan_offsets": (i, [vp, P(C.c_int64)]),
        "fx_plan_destroy": (None, [vp]),
        "fx_allreduce": (i, [vp, i, P(vp), P(vp), vp]),
        "fx_allreduce_hosted": (i, [vp, i, i, i, C.c_int64, u64, P(vp), P(vp), vp, vp, P(C.c_int64), P(i)]),
        "fx_broadcast": (i, [vp, i, P(vp), vp]),
        "fx_allreduce_begin": (i, [vp, i, P(vp), vp]),
        "fx_allreduce_finish": (i, [vp, P(vp), vp]),
        "fx_barrier": (i, [vp, vp]),
    }
    for name, (res, args) in sigs.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()
C = C  # re-exported for the pointer-array fast path


def check(rc: int) -> None:
    if rc != FX_OK:
        raise NativeError(rc, lib.fx_last_error().decode(errors="replace"))


def cuda_available() -> bool:
    return bool(lib.fx_cuda_available())
