"""The production layout: one process per GPU, peers mapped over NVLink (needs >= 2 GPUs).

Same golden vectors / oracle as tests/test_gpu_parity.py, but the ranks are real processes
whose arenas are exchanged through the C ABI bootstrap (VMM fd passing or cudaIpc); also the
hybrid layout (2 processes x 2 virtual ranks).  Skipped on a one-GPU box; run with
``python -m pytest tests/test_gpu_multiproc.py -m gpu`` on a machine with 2, 4 or 8 GPUs.
"""
import numpy as np
import pytest
import torch

from tests import golden_io as G
from tests.golden import cases
from tests.harness import run_ranks

pytestmark = pytest.mark.gpu
FP32_TOL = 1e-6


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _same(got, want, cols, nvls):
    """Bit-exact against the rank-order oracle on the peer-to-peer kernels; with NVLS the switch
    chooses the summation order, so fp32 is held to the 1e-6 bar and 16-bit floats to 1 ulp."""
    if not nvls or not got.dtype.is_floating_point:
        return torch.equal(got, want)
    if got.dtype == torch.bfloat16:
        return G.ulp_distance_bf16(got, want) <= 1
    if got.dtype == torch.float16:
        return bool(((got.float() - want.float()).abs() <= 1e-3 * want.float().abs() + 1e-7).all())
    return G.normalised_error(got, want, cols) <= FP32_TOL


def _worker(rank, world, nvls_env="1"):
    import os
    os.environ["FLASHY_B200_NVLS"] = nvls_env
    os.environ["FLASHY_B200_NVLS_MIN_WORLD"] = "2"        # exercise the multimem kernel at every world size
    from oracle import numeric
    from flashy_b200 import distrib, context
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    assert distrib.rank() == rank and distrib.world_size() == world
    distrib.barrier()
    warm = torch.ones(4, device=dev)
    distrib.all_reduce(warm)                              # creates the communicator
    nvls = context.current().engine.multicast
    if rank == 0:
        print(f"[world {world}] NVLS multicast: {nvls} ({context.current().engine.multicast_error})", flush=True)
    if nvls_env == "0":
        assert not nvls

    # ---- golden vectors of the unmodified reference
    if world in cases.WORLDS:
        for name, dtype in cases.AVG_DTYPES.items():
            per_rank = [cases.avg_inputs(r, name) for r in range(world)]
            model = numeric.average_tensors(per_rank)
            ts = [t.to(dev) for t in per_rank[rank]]
            distrib.average_tensors(ts)
            for i, t in enumerate(ts):
                t = t.cpu()
                if i == cases.INT_SLOT:
                    assert torch.equal(t, per_rank[rank][i])
                    continue
                assert _same(t, model[rank][i], [per_rank[q][i] for q in range(world)], nvls), (name, i)
                if name in ("fp32", "fp64", "c64"):
                    ref = G.golden_tensor(world, f"avg/{name}/out/{i}", dtype)
                    assert G.normalised_error(t, ref, [per_rank[q][i] for q in range(world)]) <= FP32_TOL
        for src in (0, world - 1):
            ts = [t.to(dev) for t in cases.avg_inputs(rank, "fp32")]
            distrib.broadcast_tensors(ts, src=src)
            for i, t in enumerate(ts):
                assert np.array_equal(G.get(world, f"bcast/src{src}/out/{i}", rank), cases.to_np(t))
        for variant in ("avg", "bcast", "eager"):
            model = cases.make_model().to(dev)
            grads, bufs = cases.model_local_state(rank)
            with torch.no_grad():
                for b, v in zip(model.buffers(), bufs):
                    b.copy_(v)
            if variant == "eager":
                loss = sum((p * g.to(dev)).sum() for p, g in zip(model.parameters(), grads))
                with distrib.eager_sync_model(model):
                    loss.backward()
            else:
                for p, g in zip(model.parameters(), grads):
                    p.grad = g.to(dev)
                distrib.sync_model(model, average_buffers=(variant == "avg"))
            local = [cases.model_local_state(r) for r in range(world)]
            for i, p in enumerate(model.parameters()):
                ref = G.golden_tensor(world, f"model/{variant}/grad/{i}", torch.float32)
                assert G.normalised_error(p.grad.cpu(), ref, [local[q][0][i] for q in range(world)]) <= FP32_TOL
        metrics, count = cases.metrics_inputs(rank)
        out = distrib.average_metrics(metrics, count)
        for v, w in zip(out.values(), G.get(world, "metrics/out")):
            assert abs(v - w) <= 1e-6 * max(1.0, abs(w))

    # ---- count mismatch raises everywhere, communicator stays usable
    x = torch.ones(3, device=dev)
    try:
        distrib.average_tensors([x, x.clone()] if rank == world - 1 else [x])
    except RuntimeError as err:
        assert "Mismatch in number of params" in str(err)
    else:
        raise AssertionError("Should have raised")

    # ---- ResNet-18 sized bucket, bf16 and fp32, repeated calls with changing data
    import torchvision
    numels = [p.numel() for p in torchvision.models.resnet18(num_classes=10).parameters()]
    for dtype in (torch.bfloat16, torch.float32):
        for it in range(2):
            gens = [torch.Generator().manual_seed(1000 + r + 31 * it) for r in range(world)]
            per_rank = [[(torch.randn(n, generator=gens[r]) * 1e-2).to(dtype) for n in numels] for r in range(world)]
            ts = [t.to(dev) for t in per_rank[rank]]
            distrib.average_tensors(ts)
            want = numeric.average_tensors(per_rank)[0]
            for j, (t, w_) in enumerate(zip(ts, want)):
                assert _same(t.cpu(), w_, [per_rank[q][j] for q in range(world)], nvls), (dtype, it, j)
    # ---- large single tensor (chunked) + integer sum
    big = torch.arange(40 << 20, device=dev, dtype=torch.float32) % 251 + rank
    distrib.all_reduce(big)
    expect = (torch.arange(40 << 20, device=dev, dtype=torch.float32) % 251) * world + sum(range(world))
    assert torch.equal(big, expect)
    cnt = torch.tensor([rank + 1, 7], device=dev)
    distrib.all_reduce(cnt)
    assert cnt.tolist() == [world * (world + 1) // 2, 7 * world]
    for _ in range(200):                                   # flag protocol soak: many tiny collectives
        s = torch.tensor([1.0], device=dev)
        distrib.all_reduce(s)
    assert s.item() == world
    distrib.barrier()
    torch.cuda.synchronize()
    context.reset_process_context()


def _hybrid_worker(rank, world):
    """2 processes x 2 virtual ranks: local and NVLink peers in the same launch."""
    from oracle import numeric
    from flashy_b200 import VirtualWorld, distrib
    torch.cuda.set_device(rank % torch.cuda.device_count())
    vw = VirtualWorld(2, device=torch.cuda.current_device(), arena_mb=128)
    total = vw.world
    assert total == 2 * world

    def body(vrank, w):
        assert w == total and distrib.rank() == vrank
        gens = [torch.Generator().manual_seed(500 + r) for r in range(w)]
        per_rank = [[torch.randn(n, generator=gens[r]) for n in (3, 70000, 2000000)] for r in range(w)]
        ts = [t.cuda() for t in per_rank[vrank]]
        distrib.average_tensors(ts)
        want = numeric.average_tensors(per_rank)[0]
        for t, w_ in zip(ts, want):
            assert torch.equal(t.cpu(), w_)
        b = torch.full((1000,), float(vrank), device="cuda")
        distrib.broadcast_tensors([b], src=w - 1)
        assert torch.equal(b.cpu(), torch.full((1000,), float(w - 1)))
        return True
    try:
        assert all(vw.run(body))
    finally:
        torch.cuda.synchronize()
        vw.close()


@pytest.mark.parametrize("nvls", ("0", "1"))
@pytest.mark.parametrize("world", (2, 4, 8))
def test_one_process_per_gpu(world, nvls):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    run_ranks(world, "tests.test_gpu_multiproc", "_worker", args=(nvls,), timeout=600)


def test_hybrid_two_processes_two_virtual_ranks():
    if _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    run_ranks(2, "tests.test_gpu_multiproc", "_hybrid_worker", timeout=300)
