#!/usr/bin/env python
"""Achieved NVLink GB/s of the gradient-bucket all-reduce, from the GPU's own link counters.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 benchmarks/nvlink_counters.py [--launches 200]

ncu cannot replay a kernel that spins on other processes' flags, so the multi-GPU kernel is measured from
outside: every rank reads the NVML NVLink data-throughput counters of its GPU (sum over links, TX and RX,
KiB granularity) before and after ``launches`` back-to-back ``sync_model`` calls on ResNet-sized gradient
lists, and the kernel time comes from CUDA events around every launch.  Reported per case: NVLink bytes per
launch and direction as counted by the hardware, next to the algorithmic figure of the algorithm in use
((1 + 1/W) N for the in-switch reduction, 2 (W-1)/W N peer to peer), and the resulting GB/s per direction
against the 450 GB/s per direction of NVLink 4 (H100 SXM data sheet).  One JSON line per case (rank 0 prints the
max over ranks of the time and the mean over ranks of the bytes).  Benchmark infrastructure only.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch                      # noqa: E402
import torch.distributed as dist  # noqa: E402


def read_counters(index: int):
    """(tx_bytes, rx_bytes, source) summed over the NVLinks of GPU `index`."""
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(index)
        tx_id = getattr(pynvml, "NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_TX", 138)
        rx_id = getattr(pynvml, "NVML_FI_DEV_NVLINK_THROUGHPUT_DATA_RX", 139)
        vals = pynvml.nvmlDeviceGetFieldValues(h, [(tx_id, 0xFFFFFFFF), (rx_id, 0xFFFFFFFF)])
        out = []
        for v in vals:
            if v.nvmlReturn != 0:
                raise RuntimeError(f"field {v.fieldId}: nvml return {v.nvmlReturn}")
            out.append(int(v.value.ullVal) * 1024)
        return out[0], out[1], "nvml field values (KiB, all links)"
    except Exception as err:      # noqa: BLE001 - fall back to the CLI
        why = f"{type(err).__name__}: {err}"
    try:
        text = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", str(index)], capture_output=True, text=True, timeout=20).stdout
        tx = sum(int(line.split(":")[1].split()[0]) for line in text.splitlines() if "Data Tx" in line)
        rx = sum(int(line.split(":")[1].split()[0]) for line in text.splitlines() if "Data Rx" in line)
        return tx * 1024, rx * 1024, f"nvidia-smi nvlink -gt d (pynvml failed: {why})"
    except Exception as err:      # noqa: BLE001
        return None, None, f"unavailable ({why}; {type(err).__name__}: {err})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    dist.init_process_group("gloo", init_method="env://")
    from flashy_b200 import _native as N
    from flashy_b200 import context as fctx
    from flashy_b200 import distrib
    import torchvision

    for name, dtype in (("resnet18", torch.bfloat16), ("resnet50", torch.float32)):
        model = (torchvision.models.resnet18(num_classes=10) if name == "resnet18" else torchvision.models.resnet50()).to(dev).to(dtype)
        for p in model.parameters():
            p.grad = torch.zeros_like(p)
        for _ in range(5):
            distrib.sync_model(model)
        torch.cuda.synchronize()
        eng = fctx.current().engine
        plan = max(eng.plans.values(), key=lambda pl: pl.info.wire_bytes)
        dist.barrier()
        tx0, rx0, source = read_counters(local)
        eng.profile, eng.timings = True, []
        for _ in range(args.launches):
            distrib.sync_model(model)
        torch.cuda.synchronize()
        eng.profile = False
        dist.barrier()
        tx1, rx1, _ = read_counters(local)
        per_launch = {}
        for key, e0, e1 in eng.timings:
            per_launch.setdefault(key, []).append(e0.elapsed_time(e1))
        eng.timings = []
        kernel_ms = sum(sum(v) for v in per_launch.values()) / args.launches         # all buckets of one call
        nbytes = int(plan.info.wire_bytes)
        stats = torch.tensor([kernel_ms, float(tx1 - tx0) if tx0 is not None else -1.0,
                              float(rx1 - rx0) if rx0 is not None else -1.0], dtype=torch.float64)
        mx = stats.clone()
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        dist.all_reduce(stats, op=dist.ReduceOp.SUM)
        if rank == 0:
            t = float(mx[0]) * 1e-3
            nvls = int(plan.info.kernel) in (3, 5, 7)
            alg = (1 + 1 / world) * nbytes if nvls else 2 * (world - 1) / world * nbytes
            row = {"case": f"{name}/{str(dtype).split('.')[-1]}", "world": world, "kernel": N.KERNEL_NAMES.get(int(plan.info.kernel)),
                   "bucket_bytes": nbytes, "launches": args.launches, "kernel_ms": float(mx[0]),
                   "bus_gbs": 2 * (world - 1) / world * nbytes / t / 1e9,
                   "algorithmic_bytes_per_direction": alg, "algorithmic_gbs_per_direction": alg / t / 1e9,
                   "counter_source": source}
            if float(stats[1]) >= 0:
                tx = float(stats[1]) / world / args.launches
                rx = float(stats[2]) / world / args.launches
                row.update(counted_tx_bytes_per_launch=tx, counted_rx_bytes_per_launch=rx,
                           counted_tx_gbs=tx / t / 1e9, counted_rx_gbs=rx / t / 1e9,
                           frac_of_450_nominal=max(tx, rx) / t / 1e9 / 450.0)
            print(json.dumps(row), flush=True)
        del model
    torch.cuda.synchronize()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
