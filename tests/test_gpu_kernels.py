"""Every collective kernel at its geometry edges, against plain references (one H100, virtual ranks).

The C ABI is driven directly through ``Engine(n_local=W, device=0)`` from one thread, with one
pointer row per hosted rank, so each test chooses the kernel, the in / out addresses and the data:

* ``Carve`` places the tensors of every rank in one byte buffer filled with a per-rank sentinel,
  at every start residue mod 16 bytes, with >= 64-byte guard bands.  After every call every byte
  outside the tensors must still hold the sentinel, and an out-of-place call must leave its input
  bytes untouched.
* ``make_plan`` forces the kernel with the planner's environment knobs and asserts
  ``plan.info.kernel``; ``assert_geometry`` proves that the layout really has tensors that cross a
  slice, a shard and (pipelined kernels) a chunk boundary, and one shorter than 16 bytes.
* Every plan is called several times with fresh values (both staging halves, the epoch roll).

Expected values: SUM / AVG bit-exact against ``oracle.numeric`` (rank-order sum in the wide type,
true division, one rounding) and, independently, within ``ulp_T(ref) + W u_acc sum|x|`` of an
extended-precision numpy sum; MAX / MIN by value; PROD as a rank-order product in the accumulator
type rounded once; integers exact, int32 / int64 SUM wrapping in two's complement.  NaN and
signed-zero semantics of MAX / MIN are not defined by the reference and are not tested.
"""
import contextlib
import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import numeric

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 0xA0                    # rank r's buffers are filled with byte SENTINEL + r

F32, BF16, F16, F64 = torch.float32, torch.bfloat16, torch.float16, torch.float64
I32, I64, U8 = torch.int32, torch.int64, torch.uint8
_BITS = {F32: torch.int32, BF16: torch.int16, F16: torch.int16, F64: torch.int64, I32: I32, I64: I64, U8: U8}
_WIDE = {F32: F32, BF16: F32, F16: F32, F64: F64, I32: I32, I64: I64}
# (mantissa bits, smallest normal exponent) of the float types, for ulp_T
_FMT = {F32: (23, -126), BF16: (7, -126), F16: (10, -14), F64: (52, -1022)}


def N():
    from flashy_b200 import _native
    return _native


def abi_dtype(dt):
    n = N()
    return {F32: n.FX_F32, BF16: n.FX_BF16, F16: n.FX_F16, F64: n.FX_F64, I32: n.FX_I32, I64: n.FX_I64,
            U8: n.FX_U8}[dt]


# ------------------------------------------------------------------------------------ engines
_engines = {}


def engine(world):
    from flashy_b200.engine import Engine
    if world not in _engines:
        _engines[world] = Engine(n_local=world, device=0, arena_mb=64)
    return _engines[world]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    torch.cuda.synchronize()
    for eng in _engines.values():
        eng.close()
    _engines.clear()


@contextlib.contextmanager
def environ(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


# Kernel forcing.  The plan cache key does not include these knobs, so every configuration gets its
# own tag.  SLICE_BYTES is small so that a few tens of KiB already span several slices per shard.
BASE_ENV = {"FLASHY_B200_SLICE_BYTES": "1024"}
KERNEL_ENV = {
    "one_shot": {},
    "two_shot": {"FLASHY_B200_FUSE": "0", "FLASHY_B200_PIPE": "0"},
    "pipe": {"FLASHY_B200_FUSE": "0", "FLASHY_B200_PIPE": "2", "FLASHY_B200_CHUNK_BYTES": "256",
             "FLASHY_B200_MAX_CHUNKS": "8"},
    "fuse": {"FLASHY_B200_FUSE_CHUNK": "256"},
}
KERNEL_ID = {"one_shot": 1, "two_shot": 2, "pipe": 4, "fuse": 6}


def make_plan(eng, kernel, numels, dtype, wire=None, env=None, blocks=0, kind="ar"):
    """Plan of `numels` elements of ABI dtype `dtype`, forced onto `kernel` (asserted)."""
    n = N()
    algo = n.FX_ALGO_ONE_SHOT if kernel == "one_shot" else n.FX_ALGO_TWO_SHOT
    full = {**BASE_ENV, **KERNEL_ENV[kernel], **(env or {})}
    eng.plan_blocks = blocks
    try:
        with environ(full):
            plan = eng.get_plan(kind, tuple(int(x) for x in numels), dtype, dtype if wire is None else wire, algo,
                                tag=(kernel, tuple(sorted(full.items()))))
    finally:
        eng.plan_blocks = 0
    if kind == "ar":
        assert plan.info.kernel == KERNEL_ID[kernel], \
            f"planner chose {n.KERNEL_NAMES.get(plan.info.kernel)} instead of {kernel}"
    return plan


def plan_offsets(plan):
    arr = (C.c_int64 * plan.n)()
    N().check(N().lib.fx_plan_offsets(plan.handle, arr))
    return np.array(arr[:], dtype=np.int64)


def geometry(plan, numels, wsize):
    """Which boundaries of the plan's layout fall strictly inside a tensor."""
    info = plan.info
    off = plan_offsets(plan)
    n = np.asarray(numels, dtype=np.int64)
    live = n > 0
    slice_e = int(info.shard_elems) // info.grid_x
    x = np.arange(int(info.padded_elems) + 1, dtype=np.int64)

    def crosses(starts):
        cs = np.concatenate([[0], np.cumsum(starts)])            # cs[k] = boundaries in [0, k)
        inside = cs[off + n] - cs[off + 1]                        # boundaries in (off, off + n)
        return bool(np.any(live & (inside > 0)))

    out = {"slice": crosses((x % slice_e == 0)[:-1]),
           "shard": info.algo != N().FX_ALGO_ONE_SHOT and crosses((x % int(info.shard_elems) == 0)[:-1]),
           "small": bool(np.any(live & (n * wsize < 16)))}
    if info.chunks > 0:
        chunk_e = int(info.chunk_bytes) // wsize
        out["chunk"] = crosses((((x % slice_e) % chunk_e == 0) & (x % slice_e != 0))[:-1])
    return out


def assert_geometry(plan, numels, wsize, need=("slice", "shard", "chunk", "small")):
    geo = geometry(plan, numels, wsize)
    kernel = plan.info.kernel
    for what in need:
        if what == "shard" and plan.info.algo == N().FX_ALGO_ONE_SHOT:
            continue
        if what == "chunk" and kernel not in (4, 6):
            continue
        assert geo.get(what), f"layout has no tensor crossing / being a {what} boundary: {geo}, grid {plan.info.grid_x}, " \
                              f"shard {plan.info.shard_elems}, chunks {plan.info.chunks}"


# ------------------------------------------------------------------------------------ carving
class Carve:
    """Tensors of `numels` elements (`esize` bytes each) in one sentinel-filled byte buffer per rank.
    Tensor i starts at byte residue `residues[i] * esize` mod 16 and is followed by a guard band."""

    def __init__(self, world, numels, esize, residues, view_dtype):
        self.world, self.esize, self.dt = world, esize, view_dtype
        self.numels = [int(v) for v in numels]
        offs, cur = [], GUARD
        for cnt, res in zip(self.numels, residues):
            cur = (cur + 15) // 16 * 16 + res * esize
            offs.append(cur)
            cur += cnt * esize + GUARD
        self.nbytes = (cur + 15) // 16 * 16
        self.byte_off = offs
        self.pos = torch.cat([torch.arange(o // esize, o // esize + cnt) for o, cnt in zip(offs, self.numels)]
                             + [torch.zeros(0, dtype=torch.int64)])
        self.mask = torch.zeros(self.nbytes, dtype=torch.bool)
        self.mask[((self.pos * esize).unsqueeze(1) + torch.arange(esize)).reshape(-1)] = True
        self.dev = [torch.empty(self.nbytes, dtype=U8, device="cuda") for _ in range(world)]
        self.images = [None] * world

    def rows(self):
        return [[d.data_ptr() + o for o in self.byte_off] for d in self.dev]

    def blank(self, r):
        return torch.full((self.nbytes,), SENTINEL + r, dtype=U8)

    def load(self, r, flat):
        img = self.blank(r)
        img.view(self.dt)[self.pos] = flat.view(self.dt)
        self.dev[r].copy_(img)
        self.images[r] = img

    def reset(self, r):
        self.dev[r].fill_(SENTINEL + r)
        self.images[r] = None

    def where(self, byte):
        """Human-readable position of a buffer byte relative to the nearest tensor before it."""
        i = max([k for k, o in enumerate(self.byte_off) if o <= byte], default=-1)
        if i < 0:
            return f"byte {byte}, in the leading guard"
        end = self.byte_off[i] + self.numels[i] * self.esize
        return (f"byte {byte}: {byte - end} bytes past the end of tensor {i} "
                f"(numel {self.numels[i]}, start residue {self.byte_off[i] % 16})")

    def read(self, r, what=""):
        host = self.dev[r].cpu()
        bad = ((host != SENTINEL + r) & ~self.mask).nonzero()
        assert bad.numel() == 0, f"{what} rank {r}: guard band overwritten at {self.where(int(bad[0]))} " \
                                 f"({bad.numel()} bytes in all)"
        return host, host.view(self.dt)[self.pos].clone()

    def assert_unchanged(self, r, what=""):
        host = self.dev[r].cpu()
        bad = (host != self.images[r]).nonzero()
        assert bad.numel() == 0, f"{what} rank {r}: input buffer changed at {self.where(int(bad[0]))}"


def residues(n, esize, unit=1, salt=0):
    """Start residue (elements, multiples of `unit`) of each of `n` tensors: every residue mod 16 bytes."""
    choices = list(range(0, 16 // esize, unit))
    return [choices[(i * (1 + 2 * salt) + salt) % len(choices)] for i in range(n)]


def make_sizes(vec, target, seed, unit=1, big=True):
    """Bucket sizes: 0, 1, VEC-1, VEC, VEC+1, ..., one tensor of ~75% of `target` elements (longer than
    a shard: it crosses slice, shard and chunk boundaries), then a mix of small and medium tensors."""
    rng = np.random.default_rng(seed)
    sizes = [0, 1, max(vec - 1, 1), vec, vec + 1, 2 * vec - 1, 3, 2 * vec + 1]
    if big:
        sizes.append(int(target * 0.75) // vec * vec + 1)
    while sum(sizes) < target:
        if rng.random() < 0.5:
            sizes.append(int(rng.integers(1, 4 * vec + 2)))
        else:
            sizes.append(max(int(rng.integers(2, 200)) * vec + int(rng.integers(-1, 2)), 0))
    return [s * unit for s in sizes]


# ------------------------------------------------------------------------------------ references
def expect(cols, op):
    n = N()
    if op == n.FX_SUM:
        return numeric.all_reduce_sum(cols)
    if op == n.FX_AVG:
        return numeric.average_one(cols)
    if op in (n.FX_MAX, n.FX_MIN):
        st = torch.stack(cols)
        return st.amax(0) if op == n.FX_MAX else st.amin(0)
    acc = cols[0].to(_WIDE[cols[0].dtype]).clone()
    for c in cols[1:]:
        acc *= c.to(acc.dtype)
    return acc.to(cols[0].dtype)


def ulp(ref, dtype):
    mant, emin = _FMT[dtype]
    _, e = np.frexp(np.abs(ref).astype(np.float64))
    e = np.where(ref == 0, emin, np.maximum(e.astype(np.int64) - 1, emin))
    return np.ldexp(1.0, (e - mant).astype(np.int32))


def check_f64(got, cols, op, dtype, what):
    """|out - ref| <= ulp_T(ref) + W u_acc sum_r|x_r| (mean for AVG), ref in extended precision."""
    n = N()
    world = len(cols)
    x = np.stack([c.double().numpy().astype(np.longdouble) for c in cols])
    ref, mag = x.sum(0), np.abs(x).sum(0)
    if op == n.FX_AVG:
        ref, mag = ref / world, mag / world
    u = 2.0 ** -53 if dtype == F64 else 2.0 ** -24
    bound = ulp(ref, dtype) + world * u * mag
    err = np.abs(got.double().numpy().astype(np.longdouble) - ref)
    bad = np.nonzero(err > bound)[0]
    assert bad.size == 0, f"{what}: element {bad[0]} = {float(got[bad[0]])} is {float(err[bad[0]]):.3e} from " \
                          f"the float64 reference {float(ref[bad[0]])} (bound {float(bound[bad[0]]):.3e})"


def assert_same(got, want, numels, what, nan_equal=False):
    g, w = got.view(_BITS[got.dtype]), want.view(_BITS[want.dtype])
    diff = g != w
    if nan_equal:
        gn, wn = torch.isnan(got), torch.isnan(want)
        assert torch.equal(gn, wn), f"{what}: NaN positions differ"
        diff &= ~gn
    bad = diff.nonzero()
    if bad.numel():
        i = int(bad[0])
        t = int(np.searchsorted(np.cumsum(numels), i, side="right"))
        raise AssertionError(f"{what}: {bad.numel()} elements differ; first at bucket element {i} (tensor {t}, "
                             f"numel {numels[t]}): got {got[i].item()!r}, want {want[i].item()!r}")


def gen_values(dtype, count, op, seed, world):
    n = N()
    g = torch.Generator().manual_seed(seed)
    if dtype in (I32, I64):
        if op == n.FX_PROD:
            return [torch.randint(-4, 5, (count,), generator=g, dtype=dtype) for _ in range(world)]
        info = torch.iinfo(dtype)
        return [torch.randint(info.min, info.max, (count,), generator=g, dtype=dtype) for _ in range(world)]
    if op == n.FX_PROD:
        return [((torch.rand(count, generator=g, dtype=F64) + 0.5)
                 * (torch.randint(0, 2, (count,), generator=g) * 2 - 1)).to(dtype) for _ in range(world)]
    scale = torch.exp2(torch.randint(-6, 6, (count,), generator=g).to(F64))     # mixed magnitudes
    return [(torch.randn(count, generator=g, dtype=F64) * scale).to(dtype) for _ in range(world)]


# ------------------------------------------------------------------------------------ bucket
class Bucket:
    """One plan plus its in / out carvings; `unit` = 2 gives complex tensors as (re, im) pairs."""

    def __init__(self, world, kernel, sizes, dtype, wire=None, env=None, blocks=0, unit=1, salt=0, eng=None):
        self.eng = eng or engine(world)
        self.world, self.dtype, self.wire = world, dtype, wire
        self.numels = list(sizes)
        self.esize = torch.tensor([], dtype=dtype).element_size()
        self.wsize = torch.tensor([], dtype=wire or dtype).element_size()
        self.plan = make_plan(self.eng, kernel, self.numels, abi_dtype(dtype),
                              None if wire is None else abi_dtype(wire), env, blocks)
        k = len(self.numels)
        self.cin = Carve(world, self.numels, self.esize, residues(k, self.esize, unit, salt), dtype)
        self.cout = Carve(world, self.numels, self.esize, residues(k, self.esize, unit, salt + 1), dtype)
        self.total = sum(self.numels)

    def allreduce(self, op, cols, inplace, what):
        for r in range(self.world):
            self.cin.load(r, cols[r])
        out = self.cin if inplace else self.cout
        if not inplace:
            for r in range(self.world):
                out.reset(r)
        stream = torch.cuda.current_stream()
        self.eng.allreduce(self.plan, op, self.cin.rows(), out.rows(), stream)
        torch.cuda.synchronize()
        self.eng.poll()
        got = [out.read(r, what)[1] for r in range(self.world)]
        if not inplace:
            for r in range(self.world):
                self.cin.assert_unchanged(r, what)
        return got

    def run(self, ops, calls=4, seed=0, check64=True):
        """`calls` calls with fresh values, ops round-robin, alternating out-of-place / in-place."""
        for k in range(calls):
            op = ops[k % len(ops)]
            what = f"{N().KERNEL_NAMES[self.plan.info.kernel]} W={self.world} {self.dtype} op={op} call {k}"
            cols = gen_values(self.dtype, self.total, op, seed * 1000 + k, self.world)
            got = self.allreduce(op, cols, inplace=k % 2 == 1, what=what)
            if self.wire is not None:
                want = expect([c.to(self.wire) for c in cols], op).to(self.dtype)
            else:
                want = expect(cols, op)
            for r in range(self.world):
                assert_same(got[r], want, self.numels, f"{what} rank {r}")
            if check64 and self.wire is None and self.dtype in _FMT and op in (N().FX_SUM, N().FX_AVG):
                check_f64(got[0], cols, op, self.dtype, what)


def seed_of(*parts):
    return zlib.crc32(repr(parts).encode()) & 0xFFFF


def vec_of(dtype, wire=None):
    es = torch.tensor([], dtype=dtype).element_size()
    ws = torch.tensor([], dtype=wire or dtype).element_size()
    return 16 // min(es, ws)


# ------------------------------------------------------------------------------------ the matrix
@pytest.mark.parametrize("dtype", (F32, BF16, F16), ids=str)
@pytest.mark.parametrize("world", (2, 3, 5, 8, 16))
@pytest.mark.parametrize("kernel", ("fuse", "pipe", "two_shot", "one_shot"))
def test_sum_avg_matrix(kernel, world, dtype):
    n = N()
    vec = vec_of(dtype)
    target = max(3072, world * 768) * 4 // torch.tensor([], dtype=dtype).element_size()
    b = Bucket(world, kernel, make_sizes(vec, target, seed_of(kernel, world, dtype)), dtype)
    assert_geometry(b.plan, b.numels, b.wsize)
    b.run((n.FX_SUM, n.FX_AVG), calls=4, seed=seed_of(kernel, world, dtype))


# complex tensors travel as (re, im) pairs of their real type: complex64 as fp32 (so the fused kernel
# takes them), complex128 as fp64.  Their reference is the pair model: torch's complex / real-scalar
# division rounds through the reciprocal 1 / W, which is not a true division at odd W.
_WIDE_CASES = [(k, d) for d in ("f64", "i32", "i64", "c64", "c128") for k in ("two_shot", "one_shot")] + [("fuse", "c64")]
_WIDE_TYPES = {"f64": (F64, 1), "i32": (I32, 1), "i64": (I64, 1), "c64": (F32, 2), "c128": (F64, 2)}


@pytest.mark.parametrize("world", (3, 8))
@pytest.mark.parametrize("kernel,kind", _WIDE_CASES)
def test_wide_integer_and_complex_sums(kernel, kind, world):
    n = N()
    dtype, unit = _WIDE_TYPES[kind]
    esize = torch.tensor([], dtype=dtype).element_size()
    vec = 16 // esize
    sizes = make_sizes(max(vec // unit, 1), max(3072, world * 768) * 4 // esize // unit, seed_of(kernel, kind, world),
                       unit=unit)
    b = Bucket(world, kernel, sizes, dtype, unit=unit)
    need = ("slice", "shard", "chunk") + (("small",) if esize * unit < 16 else ())
    assert_geometry(b.plan, b.numels, b.wsize, need)
    ops = (n.FX_SUM,) if dtype in (I32, I64) else (n.FX_SUM, n.FX_AVG)
    b.run(ops, calls=4, seed=seed_of(kernel, kind, world))


@pytest.mark.parametrize("dtype", (F32, BF16, F16, F64, I32, I64), ids=str)
@pytest.mark.parametrize("world", (3, 8))
@pytest.mark.parametrize("kernel", ("two_shot", "one_shot"))
def test_max_min_prod(kernel, world, dtype):
    n = N()
    esize = torch.tensor([], dtype=dtype).element_size()
    b = Bucket(world, kernel, make_sizes(16 // esize, 3072 * 4 // esize, seed_of(kernel, world, dtype)), dtype)
    assert_geometry(b.plan, b.numels, b.wsize)
    b.run((n.FX_MAX, n.FX_MIN, n.FX_PROD), calls=3, seed=seed_of("mmp", kernel, world, dtype))


@pytest.mark.parametrize("world", (4, 7))
@pytest.mark.parametrize("kernel", ("two_shot", "one_shot", "pipe"))
def test_bf16_wire_avg(kernel, world):
    """fp32 tensors sent as bf16: fp32(bf16(sum_fp32 bf16(x_r) / W)).  k_fuse needs dtype == wire, so
    the planner must not pick it even with the fused kernel left enabled."""
    n = N()
    env = {"FLASHY_B200_FUSE": "1"}
    b = Bucket(world, kernel, make_sizes(vec_of(F32, BF16), 4096, seed_of("wire", kernel, world)), F32, wire=BF16,
               env=env)
    assert_geometry(b.plan, b.numels, b.wsize)
    b.run((n.FX_AVG, n.FX_SUM, n.FX_AVG), calls=3, seed=seed_of("wire", kernel, world))


# ------------------------------------------------------------------------------------ targeted cases
def _ring_remainder_env(kernel, world, sizes, dtype, env, blocks):
    """Knobs giving a chunk count that is not a multiple of the 3-buffer ring and a short last chunk.
    The slice does not depend on the chunk knobs, so it is read from a probe plan first; the chunk
    count each knob gives follows the planner (`fx_plan_create`), and the test asserts it."""
    probe = make_plan(engine(world), "two_shot", sizes, abi_dtype(dtype), env=env, blocks=blocks)
    es = torch.tensor([], dtype=dtype).element_size()
    align = 128 // es
    slice_e = int(probe.info.shard_elems) // probe.info.grid_x
    for k in range(1, slice_e // align):
        if kernel == "fuse":                   # FUSE_CHUNK = 128 k bytes
            chunk_e = k * align
            knobs = {"FLASHY_B200_FUSE_CHUNK": str(128 * k)}
        else:                                  # 128-byte chunk target, at most k + 1 chunks
            per = -(-slice_e // min(k + 1, slice_e // align))
            chunk_e = -(-per // align) * align
            knobs = {"FLASHY_B200_CHUNK_BYTES": "128", "FLASHY_B200_MAX_CHUNKS": str(k + 1)}
        chunks = -(-slice_e // chunk_e)
        if chunks >= 4 and chunks % 3 and slice_e % chunk_e:
            return knobs, chunks
    raise AssertionError(f"no chunk size gives a ring remainder for a slice of {slice_e} elements")


_EXTREMES = ["min_chunk", "ring_remainder", "one_cta", "full_grid"]


@pytest.mark.parametrize("case", _EXTREMES)
@pytest.mark.parametrize("kernel", ("fuse", "pipe"))
def test_fuse_pipe_geometry_extremes(kernel, case):
    n = N()
    world, dtype, blocks = {"min_chunk": (5, F32, 0), "ring_remainder": (3, BF16, 2),
                            "one_cta": (4, F32, 1), "full_grid": (8, BF16, 0)}[case]
    es = torch.tensor([], dtype=dtype).element_size()
    vec = 16 // es
    env = {"FLASHY_B200_SLICE_BYTES": {"min_chunk": "2048", "ring_remainder": "4096"}.get(case, "8192")}
    target = 24576 // es
    if case == "min_chunk":                      # 128-byte chunks: many per slice, each smaller than a reduce unit
        env.update({"FLASHY_B200_FUSE_CHUNK": "128"} if kernel == "fuse" else
                   {"FLASHY_B200_CHUNK_BYTES": "128", "FLASHY_B200_MAX_CHUNKS": "64"})
    elif case == "one_cta":                      # one CTA per rank walks thousands of chunks
        env.update({"FLASHY_B200_FUSE_CHUNK": "128"} if kernel == "fuse" else
                   {"FLASHY_B200_CHUNK_BYTES": "128", "FLASHY_B200_MAX_CHUNKS": "100000"})
        target = world * 2100 * 128 // es
    elif case == "full_grid":                    # 128-byte slices: the grid is as wide as the device allows
        env["FLASHY_B200_SLICE_BYTES"] = "128"
        target = 3 * 16 * 128 * world
    sizes = make_sizes(vec, target, seed_of(kernel, case))
    if case == "ring_remainder":
        extra, want_chunks = _ring_remainder_env(kernel, world, sizes, dtype, env, blocks)
        env.update(extra)
    b = Bucket(world, kernel, sizes, dtype, env=env, blocks=blocks)
    info = b.plan.info
    chunk_b = int(info.chunk_bytes)
    slice_b = int(info.shard_elems) // info.grid_x * es
    if case == "min_chunk":
        assert chunk_b == 128 and info.chunks >= 8, (chunk_b, info.chunks)
    elif case == "ring_remainder":
        assert info.chunks == want_chunks and info.chunks % 3 and slice_b % chunk_b, (info.chunks, slice_b, chunk_b)
    elif case == "one_cta":
        assert info.grid_x == 1 and info.chunks >= 2000, (info.grid_x, info.chunks)
    else:
        assert info.grid_x == b.eng.info.max_blocks, (info.grid_x, b.eng.info.max_blocks)
    need = ("slice", "shard", "chunk", "small") if info.grid_x > 1 else ("shard", "chunk", "small")
    assert_geometry(b.plan, b.numels, b.wsize, need)
    b.run((n.FX_AVG, n.FX_SUM, n.FX_AVG), calls=3, seed=seed_of(kernel, case))


@pytest.mark.parametrize("kernel", ("fuse", "pipe", "two_shot", "one_shot"))
def test_buckets_beyond_shared_memory_metadata(kernel):
    """~1500 tensors: more than FX_SMEM_TENSORS, so every kernel reads the bucket tables from global memory."""
    n = N()
    world = 3
    rng = np.random.default_rng(seed_of("many", kernel))
    sizes = [0, 1, 7, 8, 9] + [int(v) for v in rng.integers(0, 701, 1500)]
    b = Bucket(world, kernel, sizes, BF16)
    assert b.plan.n > 1024
    assert_geometry(b.plan, b.numels, b.wsize)
    b.run((n.FX_AVG, n.FX_SUM, n.FX_AVG), calls=3, seed=seed_of("many", kernel))


def _special_values(dtype, world):
    """Per-rank columns of the special-value groups and the rule each group must obey."""
    n_grp = 24
    info = torch.finfo(dtype)
    sub = info.tiny / 4                                       # a subnormal of the type, exact in it
    cols = []
    for r in range(world):
        nan = torch.full((n_grp,), float("nan") if r == 1 else 1.0)
        inf = torch.full((n_grp,), float("inf") if r == world - 1 else 2.0)
        pm = torch.full((n_grp,), float("inf") if r == 0 else (float("-inf") if r == 2 else 0.5))
        nz = torch.full((n_grp,), -0.0)
        dn = torch.full((n_grp,), sub, dtype=F64)
        big = torch.full((n_grp,), 60000.0 if dtype == F16 else 1.0)
        cols.append(torch.cat([t.to(F64) for t in (nan, inf, pm, nz, dn, big)]).to(dtype))
    return cols, n_grp


@pytest.mark.parametrize("kernel,dtype", [("fuse", d) for d in (F32, BF16, F16)]           # k_fuse: no fp64
                         + [("two_shot", d) for d in (F32, BF16, F16, F64)], ids=str)
def test_special_values(kernel, dtype):
    """NaN on one rank -> NaN; +inf on one rank -> +inf; +inf with -inf -> NaN; -0.0 everywhere stays
    -0.0; identical subnormals come back exactly; fp16 60000 on 8 ranks: AVG 60000, SUM +inf (fp32
    accumulation)."""
    n = N()
    world = 8
    cols, g = _special_values(dtype, world)
    sizes = [g - 1, 1, g, 2 * g - 3, 3, 2 * g]                # groups split over tensors of odd sizes
    b = Bucket(world, kernel, sizes, dtype)
    for k, op in enumerate((n.FX_SUM, n.FX_AVG, n.FX_SUM)):
        got = b.allreduce(op, cols, inplace=k == 1, what=f"special {kernel} {dtype} op={op}")
        want = expect(cols, op)
        for r in range(world):
            assert_same(got[r], want, b.numels, f"special {kernel} {dtype} op={op} rank {r}", nan_equal=True)
        res = got[0].double()
        grp = [res[i * g:(i + 1) * g] for i in range(6)]
        assert torch.isnan(grp[0]).all() and torch.isposinf(grp[1]).all() and torch.isnan(grp[2]).all()
        assert (grp[3] == 0).all() and torch.signbit(grp[3]).all()
        sub = torch.finfo(dtype).tiny / 4
        assert (grp[4] == (sub if op == n.FX_AVG else world * sub)).all()
        if dtype == F16:
            assert (grp[5] == 60000.0).all() if op == n.FX_AVG else torch.isposinf(grp[5]).all()


@pytest.mark.parametrize("world", (3, 4))
def test_begin_finish_two_buckets_in_flight(world):
    """The eager path (k_two_shot BEGIN + k_unpack): two buckets begun before either is finished,
    every float dtype plus complex pairs and the bf16 wire, fresh values on every round."""
    n = N()
    eng = engine(world)
    cases = [(F32, None, 1), (BF16, None, 1), (F16, None, 1), (F64, None, 1), (F32, None, 2), (F64, None, 2),
             (F32, BF16, 1)]
    stream = torch.cuda.current_stream()
    for dtype, wire, unit in cases:
        es = torch.tensor([], dtype=dtype).element_size()
        vec = max(vec_of(dtype, wire) // unit, 1)
        pair = [Bucket(world, "two_shot", make_sizes(vec, 6144 // es // unit, seed_of("bf", dtype, unit, j), unit=unit),
                       dtype, wire=wire, unit=unit, salt=j) for j in range(2)]
        for rnd in range(3):
            op = (n.FX_AVG, n.FX_SUM, n.FX_AVG)[rnd]
            cols = []
            for j, b in enumerate(pair):
                cols.append(gen_values(dtype, b.total, op, seed_of("bf", dtype, unit, j, rnd), world))
                for r in range(world):
                    b.cin.load(r, cols[j][r])
                    b.cout.reset(r)
                eng.allreduce_begin(b.plan, op, b.cin.rows(), stream)
            for b in pair:
                eng.allreduce_finish(b.plan, b.cout.rows(), stream)
            torch.cuda.synchronize()
            eng.poll()
            for j, b in enumerate(pair):
                what = f"begin/finish W={world} {dtype} wire={wire} unit={unit} bucket {j} round {rnd}"
                want = expect([c.to(wire) for c in cols[j]], op).to(dtype) if wire else expect(cols[j], op)
                for r in range(world):
                    got = b.cout.read(r, what)[1]
                    b.cin.assert_unchanged(r, what)
                    assert_same(got, want, b.numels, f"{what} rank {r}")


def _broadcast_bucket(world, seed, eng=None):
    rng = np.random.default_rng(seed)
    sizes = [0, 1, 15, 16, 17, 127, 128, 129] + [int(v) | 1 for v in rng.integers(1, 5000, 12)]
    eng = eng or engine(world)
    plan = make_plan(eng, "two_shot", sizes, N().FX_U8, kind="bc")
    carve = Carve(world, sizes, 1, [i % 16 for i in range(len(sizes))], U8)
    return eng, plan, carve, sizes


def _broadcast_once(eng, plan, carve, sizes, src, seed, what):
    world = eng.world
    g = torch.Generator().manual_seed(seed)
    total = sum(sizes)
    data = [torch.randint(0, 256, (total,), generator=g, dtype=torch.int64).to(U8) for _ in range(world)]
    for r in range(world):
        carve.load(r, data[r])
    eng.broadcast(plan, src, carve.rows(), torch.cuda.current_stream())
    torch.cuda.synchronize()
    eng.poll()
    for r in range(world):
        assert_same(carve.read(r, what)[1], data[src], sizes, f"{what} rank {r}")


@pytest.mark.parametrize("world", (3, 8))
def test_broadcast_every_src(world):
    """k_broadcast from every source: odd byte lengths, every start residue, guard bands."""
    eng, plan, carve, sizes = _broadcast_bucket(world, seed_of("bc", world))
    for src in range(world):
        _broadcast_once(eng, plan, carve, sizes, src, seed_of("bc", world, src), f"broadcast W={world} src={src}")


@pytest.mark.parametrize("world", (5, 8))
def test_interleaved_kernels_one_communicator(world):
    """fuse -> two-shot -> one-shot -> broadcast -> fuse ... on one communicator, fresh values each time."""
    n = N()
    target = 4096
    buckets = {k: Bucket(world, k, make_sizes(8, target, seed_of("il", k, world)), BF16, salt=i)
               for i, k in enumerate(("fuse", "two_shot", "one_shot"))}
    bc = _broadcast_bucket(world, seed_of("il-bc", world))
    for rnd in range(3):
        for k in ("fuse", "two_shot", "one_shot"):
            buckets[k].run((n.FX_AVG,), calls=1, seed=seed_of("il", k, world, rnd), check64=False)
        _broadcast_once(*bc, src=rnd % world, seed=seed_of("il-bc", rnd), what=f"interleaved broadcast round {rnd}")
    buckets["fuse"].run((n.FX_SUM, n.FX_AVG), calls=2, seed=seed_of("il-last", world))


def test_complex_order_ops_refused_then_sums_match():
    """distrib.all_reduce refuses MAX / MIN / PRODUCT on complex tensors on every rank (ValueError, the
    torch.distributed message); complex SUM and averages still match the oracle on that communicator."""
    from flashy_b200 import VirtualWorld, distrib
    from torch.distributed import ReduceOp
    world = 4
    g = torch.Generator().manual_seed(7)
    xs = [[torch.randn(n, dtype=dt, generator=g) for n, dt in ((1000, torch.complex64), (77, torch.complex128))]
          for _ in range(world)]
    vw = VirtualWorld(world, device=0, arena_mb=16)
    try:
        def body(rank, w):
            mine = [t.cuda() for t in xs[rank]]
            raised = []
            for op in (ReduceOp.MAX, ReduceOp.MIN, ReduceOp.PRODUCT):
                try:
                    distrib.all_reduce(mine[0], op)
                except ValueError as err:
                    raised.append(str(err))
            assert torch.equal(mine[0].cpu(), xs[rank][0])
            summed = [t.clone() for t in mine]
            for t in summed:
                distrib.all_reduce(t)
            distrib.average_tensors(mine)
            torch.cuda.synchronize()
            return raised, [t.cpu() for t in summed], [t.cpu() for t in mine]
        got = vw.run(body)
    finally:
        vw.close()
    avg = numeric.average_tensors(xs)
    for rank, (raised, summed, averaged) in enumerate(got):
        assert raised == [f"all_reduce does not support {op} on complex tensors"
                          for op in (ReduceOp.MAX, ReduceOp.MIN, ReduceOp.PRODUCT)]
        for i in range(2):
            assert torch.equal(summed[i], numeric.all_reduce_sum([x[i] for x in xs]))
            assert torch.equal(averaged[i], avg[rank][i])


class _DeviceWords:
    def __init__(self, ptr, words):
        self.__cuda_array_interface__ = {"shape": (words,), "typestr": "<i4", "data": (ptr, False), "version": 3}


def test_epoch_counters_wrap():
    """Every flag and epoch word of the signal pad set to 2^32 - 5, then every kernel and the barrier
    run across the 32-bit wrap, with fresh values and exact checks.  A short device timeout turns a
    wrap bug into the library's timeout error instead of a long spin."""
    from flashy_b200.engine import Engine
    n = N()
    world = 3
    with environ({"FLASHY_B200_DEVICE_TIMEOUT": "5"}):
        eng = Engine(n_local=world, device=0, arena_mb=16)
    try:
        arenas = (C.c_void_p * world)()
        mc, mc_bytes, pad_bytes = C.c_void_p(), C.c_uint64(), C.c_uint64()
        n.check(n.lib.fx_comm_get_pointers(eng.comm, arenas, C.byref(mc), C.byref(mc_bytes), C.byref(pad_bytes)))
        # FxPad: flags, flags_pack, flags_red [FX_MAX_BLOCKS][FX_MAX_WORLD], block_epoch, pipe_epoch [FX_MAX_BLOCKS]
        words = 3 * 512 * 16 + 2 * 512
        assert pad_bytes.value >= 4 * words
        pads = [torch.as_tensor(_DeviceWords(arenas[r], words), device="cuda") for r in range(world)]
        torch.cuda.synchronize()
        for p in pads:
            p.fill_(-5)                                              # 2^32 - 5
        torch.cuda.synchronize()

        env = {"FLASHY_B200_FUSE_CHUNK": "128"}
        pipe_env = {"FLASHY_B200_CHUNK_BYTES": "128", "FLASHY_B200_MAX_CHUNKS": "16"}
        sizes = make_sizes(4, 6144, seed_of("wrap"))
        fuse = Bucket(world, "fuse", sizes, F32, env=env, eng=eng)
        pipe = Bucket(world, "pipe", sizes, F32, env=pipe_env, eng=eng)
        two = Bucket(world, "two_shot", sizes, F32, salt=1, eng=eng)
        one = Bucket(world, "one_shot", sizes, F32, salt=2, eng=eng)
        assert fuse.plan.info.chunks >= 6 and pipe.plan.info.chunks >= 6
        bc = _broadcast_bucket(world, seed_of("wrap-bc"), eng=eng)
        stream = torch.cuda.current_stream()
        for rnd in range(4):
            for k, b in enumerate((fuse, pipe, two, one)):
                b.run((n.FX_AVG, n.FX_SUM), calls=2, seed=seed_of("wrap", rnd, k), check64=False)
            _broadcast_once(*bc, src=rnd % world, seed=seed_of("wrap-bc", rnd), what=f"wrap broadcast {rnd}")
            eng.device_barrier(stream)
        torch.cuda.synchronize()
        eng.poll()
        # the counters really went around: pipe_epoch / block_epoch of CTA 0 are small again
        pad = pads[0].cpu().numpy().view(np.uint32)
        assert pad[3 * 512 * 16] < 1000 and pad[3 * 512 * 16 + 512] < 1000, (pad[3 * 512 * 16], pad[3 * 512 * 16 + 512])
    finally:
        torch.cuda.synchronize()
        eng.close()
