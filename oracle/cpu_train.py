"""CPU baseline of the benchmark workload (TEST / BENCH INFRASTRUCTURE, never shipped).

Runs the reference's training step of ``examples/cifar`` (``examples/cifar/solver.py:46-53``
of the reference: forward, cross-entropy, backward, ``distrib.sync_model``, ``optim.step``,
``optim.zero_grad``) on the host cores: W processes over gloo, the gradient sync being the
reference's own call sequence as restated in ``oracle/refdistrib.py`` (one all-reduce and one
divide per tensor, two host-synchronising count checks).  Used by ``bench.py`` for the
``cpu_baseline`` object and for ``--impl reference``.

Placement (``benchmarks/cpu_baseline_variants.py`` compares the options on a given host): with
OpenMP's default ACTIVE wait policy the idle workers of W x (cores / W) threads spin on the very
cores gloo's transport threads need, which makes the baseline several times slower and unstable
from host to host.  A PASSIVE wait policy (``OMP_WAIT_POLICY=passive``, ``GOMP_SPINCOUNT=0``)
avoids that.  The default is therefore the fastest stable configuration found: every rank pinned to its own
disjoint core set (``os.sched_setaffinity``), one core of the set left to the transport, passive
waiting; the reported step time is the MEDIAN over the timed steps of the per-step max over ranks,
and the rendezvous is an explicit ``tcp://`` store so that a surrounding ``torch.distributed.run``
agent (``TORCHELASTIC_*`` variables) cannot redirect it.
"""
from __future__ import annotations

import json
import multiprocessing as mp
import os
import socket
import statistics
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

# Variables a torchrun / elastic agent exports to its workers.  Inherited by the spawned CPU ranks
# they would turn ``env://`` into a client of the agent's store (nobody serves it -> hang).
_LAUNCHER_VARS = ("RANK", "WORLD_SIZE", "LOCAL_RANK", "LOCAL_WORLD_SIZE", "GROUP_RANK", "GROUP_WORLD_SIZE",
                  "ROLE_RANK", "ROLE_WORLD_SIZE", "ROLE_NAME", "MASTER_ADDR", "MASTER_PORT",
                  "OMP_NUM_THREADS", "NCCL_ASYNC_ERROR_HANDLING")


def scrub_launcher_env(env=None) -> None:
    env = os.environ if env is None else env
    for key in list(env):
        if key in _LAUNCHER_VARS or key.startswith("TORCHELASTIC_") or key.startswith("TORCH_NCCL_"):
            del env[key]


def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def partition_cores(cores, world):
    """Disjoint, equally sized core sets (rank r gets cores[r*k:(r+1)*k]); [] when there are fewer
    cores than ranks (then nothing is pinned)."""
    cores = sorted(cores)
    k = len(cores) // world
    if k < 1:
        return [[] for _ in range(world)]
    return [cores[r * k:(r + 1) * k] for r in range(world)]


def _worker(rank: int, world: int, port: int, batch: int, steps: int, warmup: int, cores, queue, spare: int = 0,
            passive: bool = False):
    scrub_launcher_env()
    if cores:
        try:
            os.sched_setaffinity(0, cores)
        except OSError:
            pass
    # `spare` cores of the rank's set are left to gloo's own threads; `passive` makes idle OpenMP workers sleep
    # instead of spinning on the cores the transport needs
    threads = max(1, len(cores) - spare) if cores else 1
    os.environ["OMP_NUM_THREADS"] = str(threads)
    if passive:
        os.environ["OMP_WAIT_POLICY"] = "passive"
        os.environ["GOMP_SPINCOUNT"] = "0"
    if str(ROOT) not in sys.path:
        sys.path.insert(0, str(ROOT))
    import torch
    import torch.distributed as dist
    import torch.nn.functional as F
    import torchvision
    from oracle.refdistrib import RefDistrib

    torch.set_num_threads(threads)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    torch.manual_seed(1234)                                       # identical weights on every rank
    model = torchvision.models.resnet18(num_classes=10)
    optim = torch.optim.SGD(model.parameters(), lr=1e-4)
    g = torch.Generator().manual_seed(1234 + rank)                # per-rank data
    img = torch.randn(batch, 3, 32, 32, generator=g)
    label = torch.randint(0, 10, (batch,), generator=g)
    step_s, sync_s = [], []
    for step in range(warmup + steps):
        if step == warmup:
            dist.barrier()
        t0 = time.perf_counter()
        loss = F.cross_entropy(model(img), label)
        loss.backward()
        s0 = time.perf_counter()
        RefDistrib.sync_model(model)
        s1 = time.perf_counter()
        optim.step()
        optim.zero_grad()
        loss.item()
        if step >= warmup:
            step_s.append(time.perf_counter() - t0)
            sync_s.append(s1 - s0)
    stats = torch.tensor([step_s, sync_s], dtype=torch.float64)
    dist.all_reduce(stats, op=dist.ReduceOp.MAX)                  # per step: the slowest rank
    if rank == 0:
        queue.put({"step_s": stats[0].tolist(), "sync_s": stats[1].tolist()})
    dist.barrier()
    dist.destroy_process_group()


def run(world: int = 8, batch: int = 8, steps: int = 5, warmup: int = 1, cores: int | None = None,
        timeout_s: float = 780.0, pin: bool = True, spare: int = 1, passive: bool = True) -> dict:
    """Returns samples/s of the whole W-rank CPU job plus how it was obtained."""
    try:
        avail = sorted(os.sched_getaffinity(0))
    except AttributeError:
        avail = list(range(os.cpu_count() or 1))
    if cores:
        avail = avail[:cores]
    sets = partition_cores(avail, world)
    k = len(sets[0])
    if k <= 1:
        spare = 0                                 # a single core per rank: nothing to spare
    threads = max(1, k - spare)
    if not pin:                                   # same thread count, placement left to the OS scheduler
        sets = [[] for _ in range(world)]
        threads = max(1, k - spare)
    ctx = mp.get_context("spawn")
    queue = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, batch, steps, warmup, sets[r] if pin else list(avail), queue,
                                               (len(avail) - threads) if not pin else spare, passive))
             for r in range(world)]
    t0 = time.perf_counter()
    for p in procs:
        p.start()
    try:
        out = queue.get(timeout=timeout_s)
    except Exception:
        for p in procs:                       # exact PIDs we started
            if p.is_alive():
                p.kill()
        raise RuntimeError(f"CPU baseline did not finish within {timeout_s:.0f} s")
    for p in procs:
        p.join(60)
        if p.is_alive():
            p.kill()
        assert p.exitcode == 0, f"CPU baseline rank exited with {p.exitcode}"
    wall = time.perf_counter() - t0
    med = statistics.median(out["step_s"])
    sync_med = statistics.median(out["sync_s"])
    return {
        "value": world * batch / med,
        "unit": "samples/s",
        "cores": min(len(avail), max(k, 1) * world),
        "kind": "port",
        "sample": (f"median of {steps} timed steps (+{warmup} warm-up) of the ResNet-18/CIFAR step, world {world} gloo "
                   f"processes x batch {batch}, fp32 on CPU, {threads} OpenMP thread(s) per rank on {max(k, 1)} "
                   f"{'pinned' if pin and k else 'unpinned'} core(s), {'passive' if passive else 'active'} OpenMP waiting; "
                   f"sync_model (oracle/refdistrib.py) median "
                   f"{1e3 * sync_med:.0f} ms/step; step min/max {1e3 * min(out['step_s']):.0f}/{1e3 * max(out['step_s']):.0f} ms; "
                   f"{wall:.0f} s wall including process start-up"),
        "ms_per_step": 1e3 * med,
        "sync_ms_per_step": 1e3 * sync_med,
        "step_ms": [1e3 * s for s in out["step_s"]],
        "world": world, "batch_per_rank": batch, "steps": steps, "warmup": warmup,
    }


if __name__ == "__main__":
    print(json.dumps(run()))
