"""Backward overlap for plain ``sync_model`` users (SURVEY.md 8(f) rank 1, second half; reference anchor
``flashy/distrib.py:193-224``), one process per GPU (needs >= 2 GPUs):
``python -m pytest tests/test_gpu_overlap.py -m gpu`` on a machine with 2 or more GPUs.

Every rank can rebuild every rank's seeded batch, so each process computes all per-rank gradients
locally and averages them with the oracle (``oracle/numeric.py``); the overlapped ``sync_model`` must
give the same gradients -- bit-exact on the peer-to-peer kernels (rank-order sum), <= 1e-6 normalised
with NVLS (the switch picks the order) and for gradient accumulation (the mean is re-taken per pass)."""
import pytest
import torch
from torch import nn

from tests import golden_io as G
from tests.harness import run_ranks

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


class Net(nn.Module):
    def __init__(self, width=256, depth=6):
        super().__init__()
        self.layers = nn.ModuleList([nn.Linear(width, width) for _ in range(depth)])
        self.norm = nn.BatchNorm1d(width)
        self.spare = nn.Linear(width, width)                       # only used when asked to

    def forward(self, x, use_spare=True):
        for layer in self.layers:
            x = torch.relu(layer(x))
        x = self.norm(x)
        if use_spare:
            x = self.spare(x)
        return x.square().mean()


def _batch(rank, step, width=256):
    g = torch.Generator().manual_seed(9000 + 17 * rank + step)
    return torch.randn(32, width, generator=g)


def _expected(world, dev, init_state, steps_per_sync, step0, use_spare=True):
    """Per-rank gradients of `steps_per_sync` accumulated backward passes, averaged by the oracle."""
    from oracle import numeric
    per_rank = []
    for r in range(world):
        m = Net().to(dev)
        m.load_state_dict(init_state)
        for k in range(steps_per_sync):
            m(_batch(r, step0 + k).to(dev), use_spare).backward()
        per_rank.append([None if p.grad is None else p.grad.detach().cpu() for p in m.parameters()])
    keep = [i for i, g in enumerate(per_rank[0]) if g is not None]
    mean = numeric.average_tensors([[row[i] for i in keep] for row in per_rank])[0]
    return keep, mean, [[row[i] for i in keep] for row in per_rank]


def _close(got, want, cols, exact):
    if exact:
        return torch.equal(got, want)
    return G.normalised_error(got, want, cols) <= 1e-6


def _worker(rank, world, nvls_env):
    import os
    os.environ["FLASHY_B200_NVLS"] = nvls_env
    os.environ["FLASHY_B200_NVLS_MIN_WORLD"] = "2"
    from flashy_b200 import distrib, context
    torch.cuda.set_device(rank % torch.cuda.device_count())
    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(4321)
    init = Net().state_dict()
    model = Net().to(dev)
    model.load_state_dict(init)
    distrib.overlap(model, True, bucket_mb=0.5)                     # 0.25 MB layers -> several hook buckets + a tail
    exact = nvls_env == "0"

    # ---- plain steps: the first sync_model installs the hooks, later ones find most buckets already sent
    for step in range(3):
        model.zero_grad(set_to_none=True)
        before = context.current().cached_engine().native_launches() if step else 0
        model(_batch(rank, step).to(dev)).backward()
        if step >= 1:
            during = context.current().engine.native_launches() - before
            assert during >= 2, f"no bucket left during backward (launches: {during})"
        distrib.sync_model(model)
        keep, mean, cols = _expected(world, dev, init, 1, step)
        params = list(model.parameters())
        for j, i in enumerate(keep):
            assert _close(params[i].grad.cpu(), mean[j], [c[j] for c in cols], exact), (step, i)

    # ---- gradient accumulation: two backward passes per sync_model (every pass re-averages: same mean)
    model.zero_grad(set_to_none=True)
    for k in range(2):
        model(_batch(rank, 10 + k).to(dev)).backward()
    distrib.sync_model(model)
    keep, mean, cols = _expected(world, dev, init, 2, 10)
    params = list(model.parameters())
    for j, i in enumerate(keep):
        # intermediate values (mean of pass 1 + local pass 2) are rounded where the oracle sums first: bound the
        # error by the magnitudes that were actually added, not by the (possibly cancelling) total
        got, scale = params[i].grad.cpu(), max(float(c[j].abs().max()) for c in cols)
        assert float((got - mean[j]).abs().max()) <= 8 * torch.finfo(torch.float32).eps * max(scale, 1e-30), i

    # ---- a module that gets no gradient in this step (the in-order rule holds its bucket back)
    model.zero_grad(set_to_none=True)
    model(_batch(rank, 20).to(dev), use_spare=False).backward()
    distrib.sync_model(model)
    keep, mean, cols = _expected(world, dev, init, 1, 20, use_spare=False)
    params = list(model.parameters())
    assert model.spare.weight.grad is None
    for j, i in enumerate(keep):
        assert _close(params[i].grad.cpu(), mean[j], [c[j] for c in cols], exact), i

    # ---- the whole step as one CUDA graph: forward, backward with hook launches, sync_model
    model.zero_grad(set_to_none=True)
    x = _batch(rank, 30).to(dev)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(2):
            model.zero_grad(set_to_none=True)
            model(x).backward()
            distrib.sync_model(model)
    side.synchronize()
    graph = torch.cuda.CUDAGraph()
    model.zero_grad(set_to_none=True)
    with torch.cuda.graph(graph, stream=side):
        model(x).backward()
        distrib.sync_model(model)
    for step in (31, 32):
        x.copy_(_batch(rank, step).to(dev))
        torch.cuda.synchronize()
        distrib.barrier()
        graph.replay()
        torch.cuda.synchronize()
        # BatchNorm statistics moved during warm-up and capture; gradients do not depend on running stats
        keep, mean, cols = _expected(world, dev, init, 1, step)
        params = list(model.parameters())
        for j, i in enumerate(keep):
            assert _close(params[i].grad.cpu(), mean[j], [c[j] for c in cols], exact), (step, i)

    # ---- switching it off restores the one-launch path
    distrib.overlap(model, False)
    model.zero_grad(set_to_none=True)
    model(_batch(rank, 40).to(dev)).backward()
    before = context.current().engine.native_launches()
    distrib.sync_model(model)
    assert context.current().engine.native_launches() - before == 1
    distrib.barrier()
    torch.cuda.synchronize()
    context.reset_process_context()


@pytest.mark.parametrize("nvls", ("0", "1"))
@pytest.mark.parametrize("world", (2, 4, 8))
def test_sync_model_backward_overlap(world, nvls):
    if _ngpu() < world:
        pytest.skip(f"needs {world} GPUs")
    run_ranks(world, "tests.test_gpu_overlap", "_worker", args=(nvls,), timeout=600)
