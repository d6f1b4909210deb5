#!/usr/bin/env python
"""Raw NVLink / NVSwitch, multimem and local-copy primitive rates of the GPUs at hand (benchmark infrastructure).

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/nvls_probe.py [--quick]
    python benchmarks/nvls_probe.py --quick          # one GPU: the local copy and latency cases only

Times the building blocks of the bucketed all-reduce in isolation, over the communicator's own
arenas and multicast mapping (``fx_comm_get_pointers``): multimem.ld_reduce + multimem.st loops
for a grid of (CTAs, threads, unroll, access pattern), reduce-scatter-only / all-gather-only /
peer-to-peer variants, the same loop next to a concurrent local HBM copy role (register copies
or a cp.async.bulk ring driven by one thread), unloaded latencies and the cost of a cross-GPU
flag barrier.  Every number is CUDA-event time on the launching stream, max over ranks; bus
GB/s uses the all-reduce convention 2 (W-1)/W * N / t with N = W * shard bytes.
One JSON object per line on stdout (rank 0).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch                      # noqa: E402
import torch.distributed as dist  # noqa: E402


class ProbeArgs(C.Structure):
    _fields_ = [
        ("arena", C.c_void_p * 16), ("mc", C.c_void_p), ("rank", C.c_int), ("world", C.c_int),
        ("region", C.c_uint64), ("shard_vec", C.c_int64), ("flags_off", C.c_uint64),
        ("copy_src", C.c_void_p), ("copy_dst", C.c_void_p), ("copy_vec", C.c_int64),
        ("pattern", C.c_int), ("reduce_threads", C.c_int), ("out", C.c_void_p),
        ("iters", C.c_int), ("epoch0", C.c_uint32),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--mb", type=int, default=256, help="all-reduce payload N per rank (MiB)")
    ap.add_argument("--launches", type=int, default=5)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("gloo", init_method="env://")
    from flashy_b200 import _native as N
    from flashy_b200 import context as fctx
    probe = C.CDLL(str(ROOT / "benchmarks" / "libfx_probe.so"))
    assert probe.fxp_args_size() == C.sizeof(ProbeArgs), (probe.fxp_args_size(), C.sizeof(ProbeArgs))
    for name in ("fxp_mm", "fxp_mix", "fxp_mix_tma", "fxp_latency", "fxp_barrier"):
        getattr(probe, name).restype = C.c_int

    eng = fctx.current().engine_for(local)
    arenas = (C.c_void_p * 16)()
    mc, mc_bytes, pad = C.c_void_p(), C.c_uint64(), C.c_uint64()
    N.check(N.lib.fx_comm_get_pointers(eng.comm, arenas, C.byref(mc), C.byref(mc_bytes), C.byref(pad)))
    have_mc = bool(mc.value)
    nbytes = args.mb << 20
    region = 2 << 20
    flags_off = region + nbytes
    assert flags_off + 4096 <= int(eng.info.arena_bytes), "arena too small: raise FLASHY_B200_ARENA_MB"
    stream = torch.cuda.current_stream()
    probe.fxp_memset.argtypes = [C.c_void_p, C.c_int, C.c_size_t]
    probe.fxp_memcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]

    def memset(ptr, value, n):
        assert probe.fxp_memset(ptr, value, n) == 0

    def memcpy(dst, src, n):
        assert probe.fxp_memcpy(dst, src, n) == 0

    def emit(**kw):
        if rank == 0:
            print(json.dumps(kw), flush=True)

    # zero the data region and the probe flags of the own arena
    memset(arenas[rank] + region, 0, nbytes + 4096)
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()

    copy_src = torch.empty(2 * nbytes, dtype=torch.uint8, device=dev)
    copy_src.random_(0, 255)
    copy_dst = torch.zeros(2 * nbytes, dtype=torch.uint8, device=dev)
    out = torch.zeros(16, dtype=torch.int64, device=dev)

    def mkargs(**kw):
        a = ProbeArgs()
        for r in range(world):
            a.arena[r] = arenas[r]
        a.mc = mc.value
        a.rank, a.world = rank, world
        a.region = region
        a.shard_vec = nbytes // world // 16
        a.flags_off = flags_off
        a.copy_src, a.copy_dst = copy_src.data_ptr(), copy_dst.data_ptr()
        a.copy_vec = 2 * nbytes // 16
        a.out = out.data_ptr()
        a.iters = 100
        for k, v in kw.items():
            setattr(a, k, v)
        return a

    emit(kind="info", world=world, multicast=have_mc, mc_error=eng.multicast_error, payload_mb=args.mb,
         sm_count=int(eng.info.sm_count))
    sms = int(eng.info.sm_count)                                     # one CTA per SM (132 on an H100 SXM)

    # ------------------------------------------------------------------ sanity: results of one launch
    if have_mc:
        x = torch.full((nbytes // 4,), float(rank + 1), dtype=torch.float32, device=dev)
        memcpy(arenas[rank] + region, x.data_ptr(), nbytes)
        torch.cuda.synchronize()
        dist.barrier()
        a = mkargs(pattern=1)
        assert probe.fxp_mm(0, sms, 512, 4, C.byref(a), C.c_void_p(stream.cuda_stream)) == 0
        torch.cuda.synchronize()
        dist.barrier()
        memcpy(x.data_ptr(), arenas[rank] + region, nbytes)
        want = float(world * (world + 1) // 2)
        ok = bool((x == want).all())
        emit(kind="sanity", what="multimem all-reduce of rank+1", ok=ok, want=want, got=[float(x[0]), float(x[-1])])
        memset(arenas[rank] + region, 0, nbytes + 4096)
        torch.cuda.synchronize()
        dist.barrier()
    # TMA ring copy correctness
    a = mkargs(reduce_threads=0)
    rc = probe.fxp_mix_tma(sms, 32, 4, C.byref(a), C.c_void_p(stream.cuda_stream))
    torch.cuda.synchronize()
    emit(kind="sanity", what="cp.async.bulk ring copy", rc=rc, ok=bool(torch.equal(copy_src, copy_dst)))
    copy_dst.zero_()
    a = mkargs()
    rc = probe.fxp_mm(5, sms, 512, 8, C.byref(mkargs(pattern=1, shard_vec=2 * nbytes // 16, rank=0)), C.c_void_p(stream.cuda_stream))
    torch.cuda.synchronize()
    emit(kind="sanity", what="register copy", rc=rc, ok=bool(torch.equal(copy_src, copy_dst)))

    # ------------------------------------------------------------------ timed configurations
    records = []          # (descr dict, ms local)

    def timed(descr, fn):
        """fn() launches one kernel; returns False if the configuration cannot launch."""
        if fn() != 0:
            torch.cuda.synchronize()
            return
        N.check(N.lib.fx_barrier(eng.comm, C.c_void_p(stream.cuda_stream)))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.launches):
            fn()
        e1.record(stream)
        e1.synchronize()
        records.append((descr, e0.elapsed_time(e1) / args.launches))

    sptr = C.c_void_p(stream.cuda_stream)
    grids = [16, 32, 64, sms, 2 * sms] if not args.quick else [32, sms]
    threads_l = [64, 128, 256, 512, 1024] if not args.quick else [512]
    unrolls = [1, 2, 4, 8, 16] if not args.quick else [4, 8]
    mode_names = {0: "ld_reduce+mc_st", 1: "ld_reduce+local_st", 2: "mc_st", 3: "p2p_pull", 4: "ld_reduce+mc_st(swp)",
                  5: "local_copy", 6: "ld_reduce_bf16+mc_st"}
    modes = [0, 4, 1, 2, 6, 3] if have_mc else ([3] if world > 1 else [])
    for mode in modes:
        for pattern in (1, 0):
            for grid in grids:
                for threads in threads_l:
                    for u in unrolls:
                        if mode != 0 and (pattern == 0 or threads in (64, 1024) or u in (1, 16) or grid == 16):
                            continue        # the full grid only for the all-reduce core
                        if mode == 0 and pattern == 0 and (threads in (64, 1024) or u in (1, 16)):
                            continue
                        a = mkargs(pattern=pattern)
                        timed(dict(kind="mm", mode=mode_names[mode], grid=grid, threads=threads, unroll=u, pattern=pattern),
                              lambda: probe.fxp_mm(mode, grid, threads, u, C.byref(a), sptr))
    # local copy alone: register copy and TMA ring (2N bytes = the pack + unpack traffic of one call)
    for grid in (sms, 2 * sms):
        for threads in (128, 256, 512):
            a = mkargs(pattern=1, shard_vec=2 * nbytes // 16, rank=0)
            timed(dict(kind="copy", how="registers", grid=grid, threads=threads, unroll=8),
                  lambda: probe.fxp_mm(5, grid, threads, 8, C.byref(a), sptr))
    for grid in (sms, 2 * sms):
        a = mkargs(reduce_threads=0)
        timed(dict(kind="copy", how="tma_ring", grid=grid, threads=32), lambda: probe.fxp_mix_tma(grid, 32, 4, C.byref(a), sptr))
    if have_mc:
        # reduce role + copy role in one CTA
        for grid in (sms, 2 * sms):
            for tr, tc in ((64, 256), (128, 256), (256, 256), (384, 128), (512, 256), (512, 512), (768, 256)):
                for u in (1, 2, 4, 8):
                    a = mkargs(pattern=1, reduce_threads=tr)
                    timed(dict(kind="mix", how="registers", grid=grid, reduce_threads=tr, copy_threads=tc, unroll=u),
                          lambda: probe.fxp_mix(grid, tr + tc, u, 8, C.byref(a), sptr))
            for tr in (64, 128, 256, 512, 992):
                for u in (1, 2, 4, 8):
                    a = mkargs(pattern=1, reduce_threads=tr)
                    timed(dict(kind="mix", how="tma_ring", grid=grid, reduce_threads=tr, copy_threads=1, unroll=u),
                          lambda: probe.fxp_mix_tma(grid, tr + 32, u, C.byref(a), sptr))

    # ------------------------------------------------------------------ latencies and barriers
    lat = None
    if world > 1:
        a = mkargs(iters=64)
        N.check(N.lib.fx_barrier(eng.comm, sptr))
        probe.fxp_latency(C.byref(a), sptr)
        torch.cuda.synchronize()
        lat = out.cpu().tolist()
        dist.barrier()
        if have_mc:
            shard = nbytes // world
            ok = True
            for r in range(world):                     # rank r stored 64 tiles at ITS shard offset of every arena
                tiles = torch.empty(64 * 4096, dtype=torch.uint8, device=dev)
                memcpy(tiles.data_ptr(), arenas[rank] + region + r * shard + r * 64 * 4096, tiles.numel())
                ok = ok and bool((tiles.view(torch.int32) == 0x5a000000 + r).all())
            flag = torch.tensor([1.0 if ok else 0.0], dtype=torch.float64)
            dist.all_reduce(flag, op=dist.ReduceOp.MIN)
            emit(kind="sanity", what="cp.async.bulk store to the multicast address lands in every rank's arena", ok=bool(flag[0] == 1.0))
        bar = {}
        epochs = {0: 0, 1: 0, 2: 0}
        epochs[3] = 0
        for variant in ((0, 1, 2, 3) if have_mc else (0, 2, 3)):
            vals = []
            for rep in range(3):
                a = mkargs(iters=200, epoch0=epochs[variant])
                N.check(N.lib.fx_barrier(eng.comm, sptr))
                probe.fxp_barrier(variant, C.byref(a), sptr)
                torch.cuda.synchronize()
                epochs[variant] += 200
                vals.append(int(out[0]))
            bar[variant] = vals

    # ------------------------------------------------------------------ reduce over ranks, report
    t = torch.tensor([ms for _, ms in records], dtype=torch.float64)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    for (descr, _), ms in zip(records, t.tolist()):
        row = dict(descr, ms=ms)
        if descr["kind"] in ("mm", "mix"):
            row["bus_gbs"] = 2 * (world - 1) / world * nbytes / (ms * 1e-3) / 1e9
            row["us_per_mb"] = ms * 1e3 / (nbytes / 1e6)
        if descr["kind"] == "copy" or descr["kind"] == "mix":
            row["copy_gbs_rw"] = 2 * (2 * nbytes) / (ms * 1e-3) / 1e9
        emit(**row)
    if lat is not None:
        lt = torch.tensor(lat[:12], dtype=torch.float64)
        dist.all_reduce(lt, op=dist.ReduceOp.MAX)
        names = ["local_ld_ns", "peer_ld_ns", "multimem_ld_reduce_ns", "multimem_st_fence_ns", "peer_st_fence_ns",
                 "local_st_fence_ns", "fence_ns", "fence_gpu_ns", "local_st_fence_gpu_ns", "multimem_st_fence_gpu_ns",
                 "bulk_store_4k_to_multicast_wait_ns", "bulk_store_4k_local_wait_ns"]
        emit(kind="latency", **{n: v for n, v in zip(names, lt.tolist())})
        for variant, vals in bar.items():
            bt = torch.tensor(vals, dtype=torch.float64)
            dist.all_reduce(bt, op=dist.ReduceOp.MAX)
            emit(kind="barrier", variant={0: "W x st.release.sys + ld.acquire.sys", 1: "one multimem.red.release + ld.acquire.sys",
                                          2: "fence + W x st.relaxed.sys, relaxed poll + fence",
                                          3: "gpu-scope fence + W x st.relaxed.sys, relaxed poll + gpu-scope fence"}[variant],
                 ns_per_barrier=bt.tolist())
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
