"""Hosted (virtual) ranks averaging through ``fx_allreduce_hosted``: one GIL-free native call per rank and
bucket, in which the ranks meet, run the count check and the last to arrive launches.

Covered: bit-exactness against oracle/numeric.py and against the Python rendezvous
(``FLASHY_B200_HOSTED_LAUNCH=0``) for ResNet-18 replicas, ranks on their own streams and on one shared
stream, W = 3 / 5 / 8, gradients replaced between calls, a model above the 128 MiB bucket cap, count and
signature mismatches, a rank that fails before arriving, the launch count, and ``engine.profile`` timings.
"""
import time

import pytest
import torch
from torch import nn

from oracle import numeric

pytestmark = pytest.mark.gpu

ARENA_MB = 256      # bucket cap = min(128 MiB, arena / 8): the 22.4 MB ResNet-18 bucket is ONE launch


def _resnet18():
    import torchvision
    torch.manual_seed(0)
    return torchvision.models.resnet18(num_classes=10).to(device="cuda", dtype=torch.bfloat16)


def _fill(model, rank: int, salt: int = 0):
    """Seeded gradients and float buffers, different on every rank."""
    g = torch.Generator().manual_seed(1000 * salt + rank)
    for p in model.parameters():
        p.grad = (torch.randn(p.shape, generator=g) * 1e-2).to(device="cuda", dtype=p.dtype)
    for b in model.buffers():
        if b.dtype.is_floating_point:
            b.copy_(torch.rand(b.shape, generator=g).to(b.dtype))


def _synced(model):
    return [p.grad for p in model.parameters()] + [b for b in model.buffers() if b.dtype.is_floating_point]


def _sync_resnets(vw, shared_stream: bool, calls: int = 1):
    """Every rank fills a ResNet-18 with its seeded values and calls sync_model; returns the inputs,
    the outputs and the launches per call."""
    from flashy_b200 import distrib
    models = [_resnet18() for _ in range(vw.n_local)]
    one = torch.cuda.Stream()

    def body(rank, world):
        model = models[rank]
        stream = one if shared_stream else torch.cuda.Stream()
        with torch.cuda.stream(stream):
            _fill(model, rank)
            stream.synchronize()
            inputs = [t.cpu() for t in _synced(model)]
            for _ in range(calls):
                distrib.sync_model(model)
            stream.synchronize()
            return inputs, [t.cpu() for t in _synced(model)]

    before = vw.engine.native_launches()
    out = vw.run(body)
    launches = vw.engine.native_launches() - before
    return models, [i for i, _ in out], [o for _, o in out], launches


def _layouts_used(model):
    from flashy_b200 import distrib
    return [layout for _key, layout in distrib._model_entry(model).fast.values()]


@pytest.mark.parametrize("world,shared", [(8, False), (8, True), (3, False), (5, True)])
def test_sync_model_resnet18_vs_oracle(world, shared):
    from flashy_b200 import VirtualWorld
    vw = VirtualWorld(world, device=0, arena_mb=ARENA_MB)
    try:
        models, ins, outs, launches = _sync_resnets(vw, shared)
        want = numeric.average_tensors(ins)[0]
        for r in range(world):
            assert len(outs[r]) == len(want)
            for got, w in zip(outs[r], want):
                assert torch.equal(got, w)
        assert launches == 1                                    # ONE launch for the whole model, all ranks
        for r, model in enumerate(models):                      # the hosted path ran, with this rank's rows
            assert any(r in layout.rows for layout in _layouts_used(model))
        if world == 8:
            big = [p.info for p in vw.engine.plans.values() if p.info.wire_bytes > (4 << 20)]
            assert big and all(int(i.kernel) == 6 for i in big)    # k_fuse<NVLS=false>
    finally:
        vw.close()


def test_hosted_and_python_rendezvous_give_the_same_bits(monkeypatch):
    from flashy_b200 import VirtualWorld
    results = {}
    for knob in ("1", "0"):
        monkeypatch.setenv("FLASHY_B200_HOSTED_LAUNCH", knob)
        vw = VirtualWorld(8, device=0, arena_mb=ARENA_MB)
        try:
            assert vw.engine.hosted_launch == (knob == "1")
            models, _ins, outs, launches = _sync_resnets(vw, shared_stream=False, calls=2)
            assert launches == 2
            rows = [bool(layout.rows) for model in models for layout in _layouts_used(model)]
            assert all(rows) if knob == "1" else not any(rows)
            results[knob] = outs
        finally:
            vw.close()
    for a, b in zip(results["1"], results["0"]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_replaced_gradients_refresh_the_rows():
    from flashy_b200 import VirtualWorld, distrib
    world = 8
    vw = VirtualWorld(world, device=0, arena_mb=ARENA_MB)
    models = [_resnet18() for _ in range(world)]
    try:
        def body(rank, w):
            model = models[rank]
            got = []
            keep = []
            for salt in range(3):
                keep.append([p.grad for p in model.parameters()])     # old tensors stay alive: new addresses
                _fill(model, rank, salt)
                torch.cuda.synchronize()
                ins = [t.cpu() for t in _synced(model)]
                distrib.sync_model(model)
                torch.cuda.synchronize()
                got.append((ins, [t.cpu() for t in _synced(model)]))
            return got

        out = vw.run(body)
        for salt in range(3):
            want = numeric.average_tensors([out[r][salt][0] for r in range(world)])[0]
            for r in range(world):
                for g, w_ in zip(out[r][salt][1], want):
                    assert torch.equal(g, w_)
    finally:
        vw.close()


def test_model_above_the_bucket_cap_launches_several_buckets():
    """3 x 4096 x 4096 fp32 weights = 192 MiB of gradients: two buckets under the 128 MiB cap.  Every value
    carries 8 significant bits, so the mean of (rank + 1) * x over 8 ranks is exactly 4.5 * x."""
    from flashy_b200 import VirtualWorld, distrib
    world = 8
    vw = VirtualWorld(world, device=0)
    base = torch.randn(3, 4096, 4096, generator=torch.Generator().manual_seed(5)).bfloat16().float().cuda()
    models = [nn.Sequential(*[nn.Linear(4096, 4096, bias=False) for _ in range(3)]).cuda() for _ in range(world)]
    try:
        def body(rank, w):
            model = models[rank]
            for i, p in enumerate(model.parameters()):
                p.grad = base[i] * float(rank + 1)
            distrib.sync_model(model)
            torch.cuda.synchronize()
            ok = all(torch.equal(p.grad, base[i] * 4.5) for i, p in enumerate(model.parameters()))
            layouts = _layouts_used(model)
            return ok, max(len(layout.buckets) for layout in layouts)

        before = vw.engine.native_launches()
        out = vw.run(body)
        launches = vw.engine.native_launches() - before
        assert all(ok for ok, _ in out)
        buckets = out[0][1]
        assert buckets >= 2 and launches == buckets
    finally:
        vw.close()


@pytest.mark.parametrize("case", ("count", "signature"))
def test_mismatch_raises_the_reference_message_on_every_rank_without_launching(case):
    from flashy_b200 import VirtualWorld, distrib
    world = 8
    vw = VirtualWorld(world, device=0, arena_mb=64)

    def make(rank):
        if rank == 5 and case == "count":
            return nn.Sequential(nn.Linear(8, 4), nn.Linear(4, 2)).cuda()
        if rank == 5:
            return nn.Linear(8, 5).cuda()                      # same number of tensors, other sizes
        return nn.Linear(8, 4).cuda()
    models = [make(r) for r in range(world)]
    good = [nn.Linear(8, 4).cuda() for _ in range(world)]
    try:
        def body(rank, w):
            for m in (models[rank], good[rank]):
                for p in m.parameters():
                    p.grad = torch.full_like(p, float(rank))
            msg = None
            try:
                distrib.sync_model(models[rank])
            except RuntimeError as err:
                msg = str(err)
            torch.cuda.synchronize()
            distrib.sync_model(good[rank])                     # the communicator is still healthy afterwards
            torch.cuda.synchronize()
            assert all(torch.equal(p.grad, torch.full_like(p, 3.5)) for p in good[rank].parameters())
            return msg

        before = vw.engine.native_launches()
        msgs = vw.run(body)
        assert vw.engine.native_launches() - before == 1      # the healthy call only
        start = "Mismatch in number of params" if case == "count" else "Mismatch in the shapes/dtypes"
        assert all(m is not None and m.startswith(start) for m in msgs), msgs
    finally:
        vw.close()


@pytest.mark.parametrize("check_mode", ("always", "plan"))
def test_rank_failing_before_arriving_makes_the_others_fail_fast(monkeypatch, check_mode):
    """The waiting ranks sit in the count check ("always") or in the wait for the launcher ("plan", warmed
    layout); VirtualWorld.run aborts the communicator and they return at once, with nothing launched."""
    from flashy_b200 import VirtualWorld, distrib
    monkeypatch.setenv("FLASHY_B200_HOST_TIMEOUT", "120")
    monkeypatch.setenv("FLASHY_B200_CHECK", check_mode)
    world = 8
    vw = VirtualWorld(world, device=0, arena_mb=64)
    models = [nn.Linear(64, 64).cuda() for _ in range(world)]
    try:
        def warm(rank, w):
            for p in models[rank].parameters():
                p.grad = torch.ones_like(p)
            distrib.sync_model(models[rank])
            torch.cuda.synchronize()
        vw.run(warm)
        before = vw.engine.native_launches()

        def body(rank, w):
            if rank == 3:
                time.sleep(0.5)                                # the others are already waiting
                raise ValueError("rank 3 failed before its sync_model")
            distrib.sync_model(models[rank])

        t0 = time.monotonic()
        with pytest.raises(ValueError, match="rank 3 failed"):
            vw.run(body)
        assert time.monotonic() - t0 < 30
        torch.cuda.synchronize()
        assert vw.engine.native_launches() == before
    finally:
        vw.close()


def test_launches_rise_by_one_per_call_and_profile_keeps_timings():
    from flashy_b200 import VirtualWorld, distrib
    world = 8
    vw = VirtualWorld(world, device=0, arena_mb=ARENA_MB)
    eng = vw.engine
    try:
        _models, _ins, _outs, launches = _sync_resnets(vw, shared_stream=False, calls=5)
        assert launches == 5
        models = [_resnet18() for _ in range(world)]

        def body(rank, w):
            _fill(models[rank], rank)
            distrib.sync_model(models[rank])
            torch.cuda.synchronize()
            distrib.barrier()
            eng.profile, eng.timings = True, []
            distrib.barrier()
            for _ in range(4):
                distrib.sync_model(models[rank])
            torch.cuda.synchronize()
            distrib.barrier()
            return True
        vw.run(body)
        eng.profile = False
        assert len(eng.timings) == 4
        assert all(e0.elapsed_time(e1) > 0 for _key, e0, e1 in eng.timings)
    finally:
        vw.close()
