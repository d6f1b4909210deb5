"""Generate tests/golden/ref_w{2,4,8}.npz by running the UNMODIFIED reference.

Needs a checkout of the reference (``$FLASHY_REFERENCE``, else ``/root/reference``, as for
``oracle/install_ref.py``); the tests only read the stored .npz files:

    FLASHY_REFERENCE=<checkout> python tests/golden/make_golden.py

The checkout's ``flashy/distrib.py`` is loaded as-is with ``importlib`` (the package's
``__init__`` cannot be imported: ``dora``/``colorlog`` are not installed);
the only stand-in is a three-function ``dora.distrib`` module (``rank``, ``world_size``,
``init``) placed in ``sys.modules`` before the import, exactly as SURVEY.md appendix A.1
describes.  Every value in the .npz files is therefore an output of the reference's own
code over ``torch.distributed`` gloo with W spawned processes.
"""
from __future__ import annotations

import hashlib
import importlib.util
import multiprocessing as mp
import os
import random
import sys
import types
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import cases  # noqa: E402

REFERENCE = Path(os.environ.get("FLASHY_REFERENCE") or "/root/reference") / "flashy" / "distrib.py"


def load_reference():
    stub = types.ModuleType("dora.distrib")
    stub.rank = lambda: dist.get_rank() if dist.is_initialized() else 0
    stub.world_size = lambda: dist.get_world_size() if dist.is_initialized() else 1

    def _init(backend="nccl"):
        raise NotImplementedError
    stub.init = _init
    pkg = types.ModuleType("dora")
    pkg.distrib = stub
    sys.modules.setdefault("dora", pkg)
    sys.modules["dora.distrib"] = stub
    spec = importlib.util.spec_from_file_location("reference_flashy_distrib", REFERENCE)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def run_rank(rank: int, world: int, port: int, out_path: str):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.set_num_threads(1)
    dist.init_process_group("gloo", init_method="env://")
    ref = load_reference()
    rec = {}

    # --- known answers of the reference's own tests/test_distrib.py:29-35 ------------------
    x = torch.tensor([float(rank) + 1])
    ref.average_tensors([x])
    rec["known/avg"] = cases.to_np(x)
    x = torch.tensor([float(rank) + 1])
    ref.broadcast_tensors([x])
    rec["known/bcast"] = cases.to_np(x)

    # --- tests/test_distrib.py:37-46: count mismatch must raise everywhere -------------------
    raised = 0
    try:
        y = torch.tensor([0.])
        if rank == world - 1:
            ref.broadcast_tensors([x, y])
        else:
            ref.broadcast_tensors([x])
    except RuntimeError:
        raised = 1
    rec["mismatch/raised"] = np.array([raised])

    # --- average_tensors / broadcast_tensors per dtype ---------------------------------------
    for name in cases.AVG_DTYPES:
        ts = cases.avg_inputs(rank, name)
        for i, t in enumerate(ts):
            rec[f"avg/{name}/in/{i}"] = cases.to_np(t)
        ref.average_tensors(ts)
        for i, t in enumerate(ts):
            rec[f"avg/{name}/out/{i}"] = cases.to_np(t)
    for src in (0, world - 1):
        ts = cases.avg_inputs(rank, "fp32")
        ref.broadcast_tensors(ts, src=src)
        for i, t in enumerate(ts):
            rec[f"bcast/src{src}/out/{i}"] = cases.to_np(t)

    # --- sync_model / eager_sync_model on the conv+BN model ------------------------------------
    for variant in ("avg", "bcast", "eager"):
        model = cases.make_model()
        grads, bufs = cases.model_local_state(rank)
        with torch.no_grad():
            model[1].running_mean.copy_(bufs[0])
            model[1].running_var.copy_(bufs[1])
            model[1].num_batches_tracked.copy_(bufs[2])
        if variant == "eager":
            loss = sum((p * g).sum() for p, g in zip(model.parameters(), grads))
            with ref.eager_sync_model(model):
                loss.backward()
        else:
            for p, g in zip(model.parameters(), grads):
                p.grad = g.clone()
            ref.sync_model(model, average_buffers=(variant == "avg"))
        for i, p in enumerate(model.parameters()):
            rec[f"model/{variant}/grad/{i}"] = cases.to_np(p.grad)
        for i, b in enumerate(model.buffers()):
            rec[f"model/{variant}/buf/{i}"] = cases.to_np(b)
    grads, bufs = cases.model_local_state(rank)
    for i, g in enumerate(grads):
        rec[f"model/in/grad/{i}"] = cases.to_np(g)
    for i, b in enumerate(bufs):
        rec[f"model/in/buf/{i}"] = cases.to_np(b)

    # --- average_metrics ---------------------------------------------------------------------
    metrics, count = cases.metrics_inputs(rank)
    got = ref.average_metrics(metrics, count)
    rec["metrics/keys"] = np.array(list(got.keys()))
    rec["metrics/out"] = np.array([got[k] for k in got], dtype=np.float64)

    # --- all_reduce ----------------------------------------------------------------------------
    for i, t in enumerate(cases.allreduce_inputs(rank)):
        rec[f"allreduce/in/{i}"] = cases.to_np(t)
        ref.all_reduce(t)
        rec[f"allreduce/out/{i}"] = cases.to_np(t)

    # --- loader shards ---------------------------------------------------------------------------
    data = list(range(cases.LOADER_N))
    for shuffle in (False, True):
        seen = [int(v) for batch in ref.loader(data, shuffle=shuffle, batch_size=4) for v in batch]
        rec[f"loader/shuffle{int(shuffle)}"] = np.array(seen, dtype=np.int64)

    # --- rank helpers --------------------------------------------------------------------------
    rec["rank"] = np.array([ref.rank(), ref.world_size(), int(ref.is_rank_zero()), int(ref.is_distributed())])
    rec["rank_zero_only"] = np.array([-1 if ref.rank_zero_only(lambda: 7)() is None else 7])

    obj = ref.broadcast_object({"k": [1, 2, 3]} if rank == 0 else None)
    assert obj == {"k": [1, 2, 3]}
    ref.barrier()

    gathered = [None] * world if rank == 0 else None
    dist.gather_object(rec, gathered, dst=0)
    if rank == 0:
        # Records that are bit-identical on every rank (all collective outputs) are stored once
        # under "all/"; records that differ (inputs, loader shards, skipped int64 tensors)
        # are stored per rank under "r{rank}/".
        flat = {}
        for k in gathered[0]:
            same = all(d[k].tobytes() == gathered[0][k].tobytes() for d in gathered)
            if "/in/" in k:
                # inputs are rebuilt from the seeds in cases.py; keep only a digest so that
                # a torch RNG change is detected instead of silently invalidating the file
                for r, d in enumerate(gathered):
                    flat[f"r{r}/{k}.sha"] = np.frombuffer(hashlib.sha256(d[k].tobytes()).digest(), dtype=np.uint8)
            elif same:
                flat[f"all/{k}"] = gathered[0][k]
            else:
                for r, d in enumerate(gathered):
                    flat[f"r{r}/{k}"] = d[k]
        np.savez_compressed(out_path, **flat)
    dist.barrier()
    dist.destroy_process_group()


def main():
    assert REFERENCE.exists(), f"{REFERENCE} not found: set FLASHY_REFERENCE to a checkout of the reference"
    ctx = mp.get_context("spawn")
    for world in cases.WORLDS:
        port = random.randrange(30000, 40000)
        out = str(HERE / f"ref_w{world}.npz")
        procs = [ctx.Process(target=run_rank, args=(r, world, port, out)) for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join()
            assert p.exitcode == 0, f"world {world}: a rank failed"
        print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()
