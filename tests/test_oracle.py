"""Pin the oracle (oracle/numeric.py, oracle/refdistrib.py) to the unmodified reference.

Golden vectors: tests/golden/ref_w{2,4,8}.npz, produced by tests/golden/make_golden.py from
the reference's flashy/distrib.py over gloo.  Known answers: reference tests/test_distrib.py:29-46.
"""
import numpy as np
import pytest
import torch

from oracle import numeric
from tests import golden_io as G
from tests.golden import cases
from tests.harness import run_ranks

FP32_TOL = 1e-6      # BASELINE.json north_star: <= 1e-6 rel for fp32 (normalised by summand magnitude)


@pytest.mark.parametrize("world", cases.WORLDS)
def test_known_answers(world):
    cols = [torch.tensor([float(r) + 1]) for r in range(world)]
    mean = numeric.average_one(cols)
    assert mean.item() == sum(range(1, world + 1)) / world          # tests/test_distrib.py:29-31
    assert G.get(world, "known/avg")[0] == mean.item()
    out = numeric.broadcast_tensors([[c] for c in cols])
    assert all(row[0].item() == 1.0 for row in out)                 # tests/test_distrib.py:33-35
    assert G.get(world, "known/bcast")[0] == 1.0


@pytest.mark.parametrize("world", cases.WORLDS)
def test_count_check(world):
    lengths = [1] * world
    lengths[-1] = 2                                                 # tests/test_distrib.py:37-46
    assert all(numeric.count_check(lengths))
    assert not any(numeric.count_check([3] * world))
    for r in range(world):
        assert G.get(world, "mismatch/raised", r)[0] == 1
    assert numeric.count_check([5]) == [False]
    assert numeric.count_check([0] * world) == [False] * world


@pytest.mark.parametrize("world", cases.WORLDS)
@pytest.mark.parametrize("name", list(cases.AVG_DTYPES))
def test_average_tensors_vs_golden(world, name):
    dtype = cases.AVG_DTYPES[name]
    per_rank = [cases.avg_inputs(r, name) for r in range(world)]
    for r in range(world):
        for i, t in enumerate(per_rank[r]):
            G.check_input(world, f"avg/{name}/in/{i}", r, t)
    out = numeric.average_tensors(per_rank)
    for i in range(len(per_rank[0])):
        if i == cases.INT_SLOT:
            for r in range(world):     # int64 tensors are skipped by the reference (distrib.py:102)
                assert np.array_equal(G.get(world, f"avg/{name}/out/{i}", r), cases.to_np(per_rank[r][i]))
                assert torch.equal(out[r][i], per_rank[r][i])
            continue
        ref = G.golden_tensor(world, f"avg/{name}/out/{i}", dtype)
        cols = [per_rank[r][i] for r in range(world)]
        if name in ("fp32", "fp64", "c64"):
            assert G.normalised_error(out[0][i], ref, cols) <= FP32_TOL
        else:
            # gloo accumulates 16-bit floats in the 16-bit type: the reference's own result is
            # several 1e-3 from the exact mean (SURVEY.md 8c).  The model rounds once.
            exact = torch.stack([c.double() for c in cols]).mean(0)
            err_model = (out[0][i].double() - exact).abs().max()
            err_ref = (ref.double() - exact).abs().max()
            assert err_model <= err_ref + 1e-12
            scale = torch.stack([c.double().abs() for c in cols]).mean(0).clamp_min(1e-30)
            assert float(((out[0][i].double() - ref.double()).abs() / scale).max()) < 0.1


@pytest.mark.parametrize("world", cases.WORLDS)
def test_broadcast_vs_golden(world):
    per_rank = [cases.avg_inputs(r, "fp32") for r in range(world)]
    for src in (0, world - 1):
        out = numeric.broadcast_tensors(per_rank, src=src)
        for i in range(len(per_rank[0])):
            for r in (0, world - 1):
                assert np.array_equal(G.get(world, f"bcast/src{src}/out/{i}", r), cases.to_np(out[r][i]))


@pytest.mark.parametrize("world", cases.WORLDS)
def test_metrics_vs_golden(world):
    ins = [cases.metrics_inputs(r) for r in range(world)]
    got = numeric.average_metrics([m for m, _ in ins], [c for _, c in ins])
    assert list(got.keys()) == list(G.get(world, "metrics/keys"))
    ref = G.get(world, "metrics/out")
    for v, w in zip(got.values(), ref):
        assert abs(v - w) <= 1e-6 * max(1.0, abs(w))
    single = {"a": 1.0}
    assert numeric.average_metrics([single], [3.0]) == single


@pytest.mark.parametrize("world", cases.WORLDS)
def test_allreduce_and_loader_vs_golden(world):
    cols = [cases.allreduce_inputs(r) for r in range(world)]
    f = numeric.all_reduce_sum([c[0] for c in cols])
    ref = G.golden_tensor(world, "allreduce/out/0", torch.float32)
    assert G.normalised_error(f, ref, [c[0] for c in cols]) <= FP32_TOL * world
    i = numeric.all_reduce_sum([c[1] for c in cols])
    assert np.array_equal(G.get(world, "allreduce/out/1"), i.numpy())          # integers: exact
    for r in range(world):
        for shuffle in (False, True):
            want = G.get(world, f"loader/shuffle{int(shuffle)}", r).tolist()
            assert numeric.loader_indices(cases.LOADER_N, r, world, shuffle) == want   # bit-exact
        assert G.get(world, "rank", r).tolist() == [r, world, int(r == 0), 1]
        assert G.get(world, "rank_zero_only", r)[0] == (7 if r == 0 else -1)


# ---- oracle/refdistrib.py over gloo against the same golden file --------------------------

def _refdistrib_worker(rank, world):
    from oracle.refdistrib import RefDistrib as R
    for name, dtype in cases.AVG_DTYPES.items():
        ts = cases.avg_inputs(rank, name)
        R.average_tensors(ts)
        for i, t in enumerate(ts):
            assert np.array_equal(G.get(world, f"avg/{name}/out/{i}", rank), cases.to_np(t)), (name, i)
    for src in (0, world - 1):
        ts = cases.avg_inputs(rank, "fp32")
        R.broadcast_tensors(ts, src=src)
        for i, t in enumerate(ts):
            assert np.array_equal(G.get(world, f"bcast/src{src}/out/{i}", rank), cases.to_np(t))
    x = torch.tensor([1.0])
    try:
        R.broadcast_tensors([x, x.clone()] if rank == world - 1 else [x])
    except RuntimeError:
        pass
    else:
        raise AssertionError("count mismatch must raise on every rank")
    for variant in ("avg", "bcast", "eager"):
        model = cases.make_model()
        grads, bufs = cases.model_local_state(rank)
        with torch.no_grad():
            for b, v in zip(model.buffers(), bufs):
                b.copy_(v)
        if variant == "eager":
            loss = sum((p * g).sum() for p, g in zip(model.parameters(), grads))
            with R.eager_sync_model(model):
                loss.backward()
        else:
            for p, g in zip(model.parameters(), grads):
                p.grad = g.clone()
            R.sync_model(model, average_buffers=(variant == "avg"))
        for i, p in enumerate(model.parameters()):
            assert np.array_equal(G.get(world, f"model/{variant}/grad/{i}", rank), cases.to_np(p.grad))
        for i, b in enumerate(model.buffers()):
            assert np.array_equal(G.get(world, f"model/{variant}/buf/{i}", rank), cases.to_np(b))
    metrics, count = cases.metrics_inputs(rank)
    got = R.average_metrics(metrics, count)
    assert [got[k] for k in got] == G.get(world, "metrics/out").tolist()
    for i, t in enumerate(cases.allreduce_inputs(rank)):
        R.all_reduce(t)
        assert np.array_equal(G.get(world, f"allreduce/out/{i}", rank), cases.to_np(t))
    data = list(range(cases.LOADER_N))
    for shuffle in (False, True):
        seen = [int(v) for batch in R.loader(data, shuffle=shuffle, batch_size=4) for v in batch]
        assert seen == G.get(world, f"loader/shuffle{int(shuffle)}", rank).tolist()
    assert R.broadcast_object({"k": 1} if rank == 0 else None) == {"k": 1}
    R.barrier()


@pytest.mark.parametrize("world", (2, 8))
def test_refdistrib_matches_reference_bit_for_bit(world):
    """Same backend (gloo) + same call sequence => the restatement reproduces the golden bits."""
    run_ranks(world, "tests.test_oracle", "_refdistrib_worker")


def test_bench_reference_arm_line():
    """`bench.py --impl reference` (CPU, gloo, oracle/refdistrib.py) prints one well-formed JSON line."""
    import json
    import subprocess
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    out = subprocess.run([sys.executable, str(root / "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0",
                          "--world", "2", "--batch", "4"], capture_output=True, text=True, timeout=300, cwd=root)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["unit"] == "samples/s" and line["value"] > 0
    assert line["metric"] == "cifar_resnet18_train_samples_per_sec" and line["higher_is_better"] is True
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["cpu_baseline"]["kind"] == "port"
    assert line["cpu_baseline"]["cores"] >= 1 and "gloo" in line["cpu_baseline"]["sample"]
