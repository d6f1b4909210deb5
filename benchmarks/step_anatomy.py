#!/usr/bin/env python
"""Where the time of the flagship step goes: host work per thread against GPU busy time.

    python benchmarks/step_anatomy.py --out DIR [--steps 30] [--warmup 5]

Builds the workload of ``bench.py --gpus 1`` from its own ``Replica`` and ``make_model``: 8 virtual
ranks on one GPU (8 Python threads, one CUDA stream each), torchvision resnet18 in bf16, batch 64 per
rank, forward+backward replayed from a CUDA graph, then ``distrib.sync_model`` and ``optim.step()``.
It writes DIR/step_anatomy.json with:

* ``ms_per_step``: CUDA events on every rank's stream around the timed steps, max over ranks, as
  ``bench.py`` takes ``value``.
* ``host_us_per_step``: per thread, the host time spent inside ``graph.replay()``, ``sync_model`` and
  ``optim.step()`` (``time.perf_counter_ns`` around each call, in this script), and the sum over the
  threads.  The threads share one interpreter, so these sums are what the GIL has to serialise at most.
* ``gpu_busy``: a second, separate pass of the same steps under ``torch.profiler`` (CUDA activities
  only; tracing slows the host, so ``ms_per_step`` is never taken from it).  The union of all device
  activity intervals (kernels, copies, sets) over the window from the first activity's start to the
  last one's end, divided by that window.  The window starts at the first activity, not at the host's
  start signal, so the fraction is an upper bound by the few microseconds of the first launch.
* the card's name, ``power.limit`` and ``clocks.max.sm`` (nvidia-smi, read in the same run).

Benchmark infrastructure only; it needs a CUDA device and stops with a clear message without one.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

WORLD = 8
BATCH = 64


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for step_anatomy.json")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--tag", default="", help="free-form label stored in the JSON (e.g. the build compared)")
    return ap.parse_args()


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [c.strip() for c in out.split(",")[:3]]
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except (OSError, ValueError, subprocess.SubprocessError) as err:
        return {"error": f"nvidia-smi: {err}"}


def union_us(intervals) -> float:
    total, end = 0.0, None
    for s, e in sorted(intervals):
        if end is None or s > end:
            total += e - s
            end = e
        elif e > end:
            total += e - end
            end = e
    return total


def main():
    args = parse()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("step_anatomy.py measures the step on a GPU: no CUDA device is visible to this process")
    from bench import Replica
    from flashy_b200 import VirtualWorld, distrib

    ns = argparse.Namespace(model="resnet18", batch=BATCH, image=32, world=WORLD)
    torch.cuda.set_device(0)
    device = torch.device("cuda", 0)
    vw = VirtualWorld(WORLD, device=0)
    replicas = [Replica(r, ns, device, distrib, overlap=False) for r in range(WORLD)]
    for rep in replicas:
        rep.capture(None)
    torch.cuda.synchronize()

    def run(steps: int, clocked: bool):
        """Every rank runs `steps` steps; returns (max device ms over ranks, per-thread host ns)."""
        def body(rank, world):
            rep = replicas[rank]
            host = {"replay": 0, "sync_model": 0, "optim_step": 0}
            clock = time.perf_counter_ns
            with torch.cuda.stream(rep.stream):
                distrib.barrier()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(rep.stream)
                for _ in range(steps):
                    t0 = clock()
                    rep.graph.replay()
                    t1 = clock()
                    distrib.sync_model(rep.model)
                    t2 = clock()
                    rep.optim.step()
                    t3 = clock()
                    if clocked:
                        host["replay"] += t1 - t0
                        host["sync_model"] += t2 - t1
                        host["optim_step"] += t3 - t2
                e1.record(rep.stream)
                rep.stream.synchronize()
                return e0.elapsed_time(e1), host
        torch.cuda.synchronize()
        out = vw.run(body)
        torch.cuda.synchronize()
        return max(ms for ms, _ in out), [h for _, h in out]

    run(max(args.warmup, 3), False)
    ms, host = run(args.steps, True)
    ms_per_step = ms / args.steps
    per_thread = {k: [h[k] / 1e3 / args.steps for h in host] for k in ("replay", "sync_model", "optim_step")}
    summed = {k: sum(v) for k, v in per_thread.items()}

    from torch.profiler import ProfilerActivity, profile
    run(2, False)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        prof_ms, _ = run(args.steps, False)
    spans = [(e.time_range.start, e.time_range.end) for e in prof.events()
             if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range.end > e.time_range.start]
    busy = None
    if spans:
        lo, hi = min(s for s, _ in spans), max(e for _, e in spans)
        busy = {"fraction": union_us(spans) / (hi - lo), "window_us": hi - lo, "busy_us": union_us(spans),
                "activities": len(spans), "ms_per_step_under_profiler": prof_ms / args.steps}

    result = {
        "tag": args.tag,
        "hosted_launch_env": os.environ.get("FLASHY_B200_HOSTED_LAUNCH"),
        "workload": f"bench.py --gpus 1: {WORLD} virtual ranks, resnet18 bf16, batch {BATCH}, CUDA graphs, sync_model, SGD",
        "steps": args.steps, "warmup": max(args.warmup, 3),
        "ms_per_step": ms_per_step,
        "host_us_per_step": {"per_thread": per_thread, "sum_over_threads": summed,
                             "sum_all": sum(summed.values())},
        "sync_model_sum_over_ms_per_step": summed["sync_model"] / 1e3 / ms_per_step,
        "gpu_busy": busy,
        "card": card(),
    }
    out = Path(args.out)
    out.mkdir(parents=True, exist_ok=True)
    (out / "step_anatomy.json").write_text(json.dumps(result, indent=1) + "\n")
    print(json.dumps(result), flush=True)
    vw.close()


if __name__ == "__main__":
    main()
