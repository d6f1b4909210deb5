"""More of the one-process-per-GPU layout (needs >= 2 GPUs): the cudaIpc memory path
(``FLASHY_B200_MEM=ipc``), ``FLASHY_B200_CHECK=plan``, ``distrib.wrap`` (the DDP comparator the reference
keeps, ``flashy/distrib.py:65-75``) and plan-cache eviction with real processes.
``python -m pytest tests/test_gpu_multiproc_extra.py -m gpu`` on a machine with 2 GPUs."""
import pytest
import torch
from torch import nn

from tests.harness import run_ranks

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _ipc_worker(rank, world):
    import os
    os.environ["FLASHY_B200_MEM"] = "ipc"                             # cudaMalloc + cudaIpc instead of VMM fd passing
    os.environ["FLASHY_B200_CHECK"] = "plan"                          # host count check only when a bucket plan is new
    from oracle import numeric
    from flashy_b200 import distrib, context, _native as N
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    numels = [5, 70001, 1 << 20, 33]
    for it in range(3):
        gens = [torch.Generator().manual_seed(77 + r + 5 * it) for r in range(world)]
        per_rank = [[torch.randn(n, generator=gens[r]) for n in numels] for r in range(world)]
        ts = [t.to(dev) for t in per_rank[rank]]
        distrib.average_tensors(ts)
        want = numeric.average_tensors(per_rank)[0]
        for t, w_ in zip(ts, want):
            assert torch.equal(t.cpu(), w_)                           # peer-to-peer kernels: rank-order sum, bit-exact
    eng = context.current().engine
    assert int(eng.info.mem_kind) == N.FX_COMM_MEM_IPC and not eng.multicast      # no multicast without VMM handles
    b = torch.full((1 << 18,), float(rank), device=dev)
    distrib.broadcast_tensors([b], src=world - 1)
    assert torch.equal(b.cpu(), torch.full((1 << 18,), float(world - 1)))
    distrib.barrier()
    torch.cuda.synchronize()
    context.reset_process_context()


def _wrap_and_eviction_worker(rank, world):
    import os
    os.environ["FLASHY_B200_ARENA_MB"] = "64"                         # small arena: the third big plan evicts the cache
    from flashy_b200 import distrib, context
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    # ---- arena eviction in the multi-process layout: every rank drops its plan cache at the same call
    for n in (3_000_000, 2_900_000, 2_800_000, 3_000_000, 2_700_000):  # 12 MB buckets, 2 regions each, 64 MB arena
        x = torch.full((n,), float(rank + 1), device=dev)
        distrib.all_reduce(x)
        assert torch.equal(x, torch.full_like(x, world * (world + 1) / 2))
    # ---- wrap: DistributedDataParallel over the process group that is already there (gloo in this harness)
    torch.manual_seed(5)
    model = nn.Linear(8, 4).to(dev)
    ddp = distrib.wrap(model)
    assert isinstance(ddp, nn.parallel.DistributedDataParallel)
    g = torch.Generator().manual_seed(100 + rank)
    ddp(torch.randn(16, 8, generator=g).to(dev)).square().mean().backward()
    grad = model.weight.grad.clone()
    lo, hi = grad.clone(), grad.clone()
    import torch.distributed as dist
    distrib.all_reduce(lo, dist.ReduceOp.MIN)
    distrib.all_reduce(hi, dist.ReduceOp.MAX)
    assert torch.equal(lo, hi)                                        # DDP averaged the gradients: identical everywhere
    distrib.barrier()
    torch.cuda.synchronize()
    del ddp
    context.reset_process_context()


def test_cuda_ipc_memory_path_and_plan_check_mode():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_ranks(2, "tests.test_gpu_multiproc_extra", "_ipc_worker", timeout=300)


def test_wrap_and_arena_eviction_with_real_processes():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_ranks(2, "tests.test_gpu_multiproc_extra", "_wrap_and_eviction_worker", timeout=300)
