// Micro-benchmarks of the raw NVLink / NVSwitch primitives the collective kernels are built
// from (BENCHMARK INFRASTRUCTURE, not on the product path): multimem.ld_reduce / multimem.st
// rates as a function of grid, block and unroll, the peer-to-peer pull rate, the same with
// concurrent local HBM copy traffic (register copies or a cp.async.bulk ring), unloaded
// latencies, and the cost of one cross-GPU flag barrier.  Driven by benchmarks/nvls_probe.py
// through ctypes; the arenas and the multicast alias come from fx_comm_get_pointers().
#include <cuda_runtime.h>
#include <stdint.h>

#define PROBE_MAX_WORLD 16

struct ProbeArgs {
    char* arena[PROBE_MAX_WORLD];
    char* mc;
    int rank, world;
    unsigned long long region;        // byte offset of the data region inside an arena
    long long shard_vec;              // 16-byte vectors per shard
    unsigned long long flags_off;     // byte offset of the probe's flag area inside an arena
    const char* copy_src;             // local (non-arena) buffers for the HBM copy roles
    char* copy_dst;
    long long copy_vec;               // 16-byte vectors the copy role moves per launch (per GPU)
    int pattern;                      // 0 grid-interleaved, 1 CTA-contiguous
    int reduce_threads;               // mixed kernels: threads of the reduce role
    unsigned long long* out;          // device buffer for latency results
    int iters;
    unsigned epoch0;                  // barrier probes: first epoch value of this launch
};

__device__ __forceinline__ uint4 ld16(const void* p) {
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st16(void* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint4 mm_ld_f32(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint4 mm_ld_bf16(const void* p) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void mm_st(void* p, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void mm_red_release(uint32_t* p, uint32_t v) {
    asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint4 add_f32(const uint4& a, const uint4& b) {
    uint4 r;
    r.x = __float_as_uint(__uint_as_float(a.x) + __uint_as_float(b.x));
    r.y = __float_as_uint(__uint_as_float(a.y) + __uint_as_float(b.y));
    r.z = __float_as_uint(__uint_as_float(a.z) + __uint_as_float(b.z));
    r.w = __float_as_uint(__uint_as_float(a.w) + __uint_as_float(b.w));
    return r;
}

// Range of vectors a thread group walks: v = v0 + k * nth (k < U), v0 += step, until limit.
struct Walk { long long v0, step, limit; };
__device__ __forceinline__ Walk make_walk(int pattern, long long nvec, int tid, int nth, int U, int b, int nb) {
    Walk w;
    if (pattern == 0) {
        w.v0 = (long long)b * nth * U + tid; w.step = (long long)nb * nth * U; w.limit = nvec;
    } else {
        const long long per = ((nvec + nb - 1) / nb + 7) / 8 * 8;      // 128-byte aligned slices
        const long long lo = (long long)b * per;
        w.limit = lo + per < nvec ? lo + per : nvec;
        w.v0 = lo + tid; w.step = (long long)nth * U;
    }
    return w;
}

// MODE 0: ld_reduce + multimem.st (all-reduce core)   1: ld_reduce + local st (reduce-scatter)
//      2: multimem.st only (all-gather)                 3: peer-to-peer pull of W copies + local st
//      4: as 0, software pipelined (next loads issued before the stores)
//      5: local copy (HBM)                              6: as 0 with bf16x2 adds
template <int U, int MODE>
__device__ __forceinline__ void mm_body(const ProbeArgs& a, int tid, int nth, int b, int nb) {
    const unsigned long long off = a.region + (unsigned long long)a.rank * a.shard_vec * 16ull;
    char* mcs = a.mc + off;
    char* loc = a.arena[a.rank] + off;
    Walk w = make_walk(a.pattern, a.shard_vec, tid, nth, U, b, nb);
    if (MODE == 4) {
        uint4 cur[U], nxt[U];
#pragma unroll
        for (int k = 0; k < U; ++k) { const long long v = w.v0 + (long long)k * nth; if (v < w.limit) cur[k] = mm_ld_f32(mcs + v * 16); }
        for (long long v0 = w.v0; v0 < w.limit; v0 += w.step) {
            const long long n0 = v0 + w.step;
#pragma unroll
            for (int k = 0; k < U; ++k) { const long long v = n0 + (long long)k * nth; if (v < w.limit) nxt[k] = mm_ld_f32(mcs + v * 16); }
#pragma unroll
            for (int k = 0; k < U; ++k) { const long long v = v0 + (long long)k * nth; if (v < w.limit) mm_st(mcs + v * 16, cur[k]); }
#pragma unroll
            for (int k = 0; k < U; ++k) cur[k] = nxt[k];
        }
        return;
    }
    for (long long v0 = w.v0; v0 < w.limit; v0 += w.step) {
        uint4 r[U];
        if (MODE == 3) {
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const long long v = v0 + (long long)k * nth;
                if (v < w.limit) {
                    uint4 raw[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) if (q < a.world) raw[q] = ld16(a.arena[q] + off + v * 16);
                    r[k] = raw[0];
#pragma unroll
                    for (int q = 1; q < 8; ++q) if (q < a.world) r[k] = add_f32(r[k], raw[q]);
                }
            }
        } else {
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const long long v = v0 + (long long)k * nth;
                if (v < w.limit) {
                    if (MODE == 0 || MODE == 1) r[k] = mm_ld_f32(mcs + v * 16);
                    else if (MODE == 6) r[k] = mm_ld_bf16(mcs + v * 16);
                    else if (MODE == 5) r[k] = ld16(a.copy_src + v * 16);
                    else r[k] = make_uint4(0, 0, 0, 0);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const long long v = v0 + (long long)k * nth;
            if (v < w.limit) {
                if (MODE == 0 || MODE == 2 || MODE == 6) mm_st(mcs + v * 16, r[k]);
                else if (MODE == 5) st16(a.copy_dst + v * 16, r[k]);
                else st16(loc + v * 16, r[k]);
            }
        }
    }
}

template <int U, int MODE>
__global__ void k_mm(const ProbeArgs a) {
    mm_body<U, MODE>(a, threadIdx.x, blockDim.x, blockIdx.x, gridDim.x);
}

// Register copy of the copy role: `copy_vec` vectors src -> dst, CTA-contiguous.
template <int UC>
__device__ __forceinline__ void copy_body(const ProbeArgs& a, int tid, int nth, int b, int nb) {
    Walk w = make_walk(1, a.copy_vec, tid, nth, UC, b, nb);
    for (long long v0 = w.v0; v0 < w.limit; v0 += w.step) {
        uint4 r[UC];
#pragma unroll
        for (int k = 0; k < UC; ++k) { const long long v = v0 + (long long)k * nth; if (v < w.limit) r[k] = ld16(a.copy_src + v * 16); }
#pragma unroll
        for (int k = 0; k < UC; ++k) { const long long v = v0 + (long long)k * nth; if (v < w.limit) st16(a.copy_dst + v * 16, r[k]); }
    }
}

// Reduce role (first reduce_threads threads) + register-copy role (the rest) in one CTA.
template <int U, int UC>
__global__ void k_mix(const ProbeArgs a) {
    const int tr = a.reduce_threads;
    if ((int)threadIdx.x < tr) mm_body<U, 0>(a, threadIdx.x, tr, blockIdx.x, gridDim.x);
    else copy_body<UC>(a, threadIdx.x - tr, blockDim.x - tr, blockIdx.x, gridDim.x);
}

// ---------------------------------------------------------------- cp.async.bulk (TMA) copy ring
#define TMA_STAGES 4
#define TMA_TILE 16384
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load(void* smem, const void* gptr, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(smem)), "l"(gptr), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store(void* gptr, const void* smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 :: "l"(gptr), "r"(smem_u32(smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// One thread moves bytes [lo, hi) of src to dst through a ring of shared-memory tiles.
__device__ __forceinline__ void tma_copy_range(const char* src, char* dst, long long lo, long long hi,
                                               char* ring, uint64_t* full) {
    const long long n = (hi - lo + TMA_TILE - 1) / TMA_TILE;
    auto tile_bytes = [&](long long i) -> uint32_t {
        const long long rest = hi - (lo + i * TMA_TILE);
        return (uint32_t)(rest < TMA_TILE ? rest : TMA_TILE);
    };
    auto load = [&](long long i) {
        const int s = (int)(i % TMA_STAGES);
        const uint32_t bytes = tile_bytes(i);
        mbar_expect_tx(&full[s], bytes);
        tma_load(ring + s * TMA_TILE, src + lo + i * TMA_TILE, bytes, &full[s]);
    };
    for (long long i = 0; i < TMA_STAGES - 1 && i < n; ++i) load(i);
    for (long long j = 0; j < n; ++j) {
        const int s = (int)(j % TMA_STAGES);
        mbar_wait(&full[s], (uint32_t)((j / TMA_STAGES) & 1));
        tma_store(dst + lo + j * TMA_TILE, ring + s * TMA_TILE, tile_bytes(j));
        tma_commit();
        const long long nl = j + TMA_STAGES - 1;
        if (nl < n) { tma_wait_read1(); load(nl); }
    }
    tma_wait_all();
}

// Reduce role (first reduce_threads threads, may be 0) + ONE thread driving a TMA copy ring.
template <int U>
__global__ void k_mix_tma(const ProbeArgs a) {
    extern __shared__ __align__(128) char dyn[];
    char* ring = dyn;
    uint64_t* full = reinterpret_cast<uint64_t*>(dyn + TMA_STAGES * TMA_TILE);
    if (threadIdx.x == 0) {
        for (int s = 0; s < TMA_STAGES; ++s) mbar_init(&full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int tr = a.reduce_threads;
    if ((int)threadIdx.x < tr) {
        mm_body<U, 0>(a, threadIdx.x, tr, blockIdx.x, gridDim.x);
    } else if ((int)threadIdx.x == tr) {
        const long long per = ((a.copy_vec + gridDim.x - 1) / gridDim.x + 7) / 8 * 8;
        const long long lo = (long long)blockIdx.x * per;
        const long long hi = lo + per < a.copy_vec ? lo + per : a.copy_vec;
        if (lo < hi) tma_copy_range(a.copy_src, a.copy_dst, lo * 16, hi * 16, ring, full);
    }
}

// ---------------------------------------------------------------- latency probes (one thread)
// out[0..]: ns per operation, averaged over `iters` dependent repetitions.
__global__ void k_latency(const ProbeArgs a) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const unsigned long long off = a.region + (unsigned long long)a.rank * a.shard_vec * 16ull;
    const int peer = (a.rank + 1) % a.world;
    unsigned acc = 0;
    // 0: local HBM/L2 load (dependent chain through the loaded value)
    unsigned long long t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) { uint4 v = ld16(a.arena[a.rank] + off + (size_t)(i * 4096 + (acc & 1)) * 16); acc += v.x; }
    unsigned long long t1 = gtimer();
    a.out[0] = (t1 - t0) / a.iters;
    // 1: peer load
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) { uint4 v = ld16(a.arena[peer] + off + (size_t)(i * 4096 + (acc & 1)) * 16); acc += v.x; }
    t1 = gtimer();
    a.out[1] = (t1 - t0) / a.iters;
    if (a.mc) {
        // 2: multimem.ld_reduce
        t0 = gtimer();
        for (int i = 0; i < a.iters; ++i) { uint4 v = mm_ld_f32(a.mc + off + (size_t)(i * 4096 + (acc & 1)) * 16); acc += v.x; }
        t1 = gtimer();
        a.out[2] = (t1 - t0) / a.iters;
        // 3: multimem.st + fence.acq_rel.sys (time until the multicast store is performed everywhere)
        t0 = gtimer();
        for (int i = 0; i < a.iters; ++i) { mm_st(a.mc + off + (size_t)i * 65536, make_uint4(0, 0, 0, 0)); fence_sys(); }
        t1 = gtimer();
        a.out[3] = (t1 - t0) / a.iters;
    }
    // 4: peer store + fence
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) { st16(a.arena[peer] + off + (size_t)i * 65536, make_uint4(0, 0, 0, 0)); fence_sys(); }
    t1 = gtimer();
    a.out[4] = (t1 - t0) / a.iters;
    // 5: local store + fence
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) { st16(a.arena[a.rank] + off + (size_t)i * 65536, make_uint4(0, 0, 0, 0)); fence_sys(); }
    t1 = gtimer();
    a.out[5] = (t1 - t0) / a.iters;
    // 6: fence alone
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) fence_sys();
    t1 = gtimer();
    a.out[6] = (t1 - t0) / a.iters;
    // 7: gpu-scope fence alone   8: local store + gpu fence   9: multimem.st + gpu fence
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) fence_gpu();
    t1 = gtimer();
    a.out[7] = (t1 - t0) / a.iters;
    t0 = gtimer();
    for (int i = 0; i < a.iters; ++i) { st16(a.arena[a.rank] + off + (size_t)i * 65536, make_uint4(0, 0, 0, 0)); fence_gpu(); }
    t1 = gtimer();
    a.out[8] = (t1 - t0) / a.iters;
    if (a.mc) {
        t0 = gtimer();
        for (int i = 0; i < a.iters; ++i) { mm_st(a.mc + off + (size_t)i * 65536, make_uint4(0, 0, 0, 0)); fence_gpu(); }
        t1 = gtimer();
        a.out[9] = (t1 - t0) / a.iters;
    }
    // 10: cp.async.bulk of a 4 KiB shared-memory tile to the MULTICAST address + wait_group 0 (completion of the
    //     bulk group instead of an SM-wide system fence); 11: the same to the own (unicast) arena
    {
        __shared__ __align__(128) unsigned char tile[4096];
        for (int i = 0; i < 4096; i += 4) *reinterpret_cast<uint32_t*>(tile + i) = 0x5a000000u + (uint32_t)a.rank;
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (a.mc) {
            t0 = gtimer();
            for (int i = 0; i < a.iters; ++i) {
                tma_store(a.mc + off + (size_t)(a.rank * a.iters + i) * 4096, tile, 4096);
                tma_commit();
                tma_wait_all();
            }
            t1 = gtimer();
            a.out[10] = (t1 - t0) / a.iters;
        }
        t0 = gtimer();
        for (int i = 0; i < a.iters; ++i) {
            tma_store(a.arena[a.rank] + off + (size_t)(a.world * a.iters + i) * 4096, tile, 4096);
            tma_commit();
            tma_wait_all();
        }
        t1 = gtimer();
        a.out[11] = (t1 - t0) / a.iters;
    }
    a.out[15] = acc;
}

// ---------------------------------------------------------------- barrier probes
// `iters` back-to-back cross-GPU barriers by one CTA per rank; out[0] = ns per barrier.
// VARIANT 0: W threads st.release.sys to each peer's flag slot + ld.acquire.sys poll (round-1 protocol)
// VARIANT 1: one multimem.red.release.add to a counter replicated on every rank; poll own copy
// VARIANT 2: W threads st.relaxed.sys after one fence; relaxed poll + fence after
template <int VARIANT>
__global__ void k_barrier_probe(const ProbeArgs a) {
    uint32_t* mine = reinterpret_cast<uint32_t*>(a.arena[a.rank] + a.flags_off);
    __shared__ unsigned long long t0s;
    if (threadIdx.x == 0) t0s = gtimer();
    for (int i = 0; i < a.iters; ++i) {
        const uint32_t epoch = a.epoch0 + i + 1;
        __syncthreads();
        if (VARIANT == 0) {
            if ((int)threadIdx.x < a.world) {
                const int q = threadIdx.x;
                st_release_sys(reinterpret_cast<uint32_t*>(a.arena[q] + a.flags_off) + a.rank, epoch);
                while ((int32_t)(ld_acquire_sys(mine + q) - epoch) < 0) {}
            }
        } else if (VARIANT == 1) {
            if (threadIdx.x == 0) {
                uint32_t* ctr = reinterpret_cast<uint32_t*>(a.mc + a.flags_off) + 64;      // one counter, every replica
                mm_red_release(ctr, 1u);
                const uint32_t want = epoch * (uint32_t)a.world;                           // epoch0 starts at 0 for this variant
                while ((int32_t)(ld_acquire_sys(mine + 64) - want) < 0) {}
            }
        } else if (VARIANT == 3) {
            if (threadIdx.x == 0) fence_gpu();
            __syncthreads();
            if ((int)threadIdx.x < a.world) {
                const int q = threadIdx.x;
                st_relaxed_sys(reinterpret_cast<uint32_t*>(a.arena[q] + a.flags_off) + 192 + a.rank, epoch);
                while ((int32_t)(ld_relaxed_sys(mine + 192 + q) - epoch) < 0) {}
                fence_gpu();
            }
        } else {
            if (threadIdx.x == 0) fence_sys();
            __syncthreads();
            if ((int)threadIdx.x < a.world) {
                const int q = threadIdx.x;
                st_relaxed_sys(reinterpret_cast<uint32_t*>(a.arena[q] + a.flags_off) + 128 + a.rank, epoch);
                while ((int32_t)(ld_relaxed_sys(mine + 128 + q) - epoch) < 0) {}
                fence_sys();
            }
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) a.out[0] = (gtimer() - t0s) / a.iters;
}

// ================================================================ C entry points
template <int MODE>
static int launch_mm(int grid, int threads, int unroll, const ProbeArgs& a, cudaStream_t s) {
    switch (unroll) {
        case 1: k_mm<1, MODE><<<grid, threads, 0, s>>>(a); break;
        case 2: k_mm<2, MODE><<<grid, threads, 0, s>>>(a); break;
        case 4: k_mm<4, MODE><<<grid, threads, 0, s>>>(a); break;
        case 8: k_mm<8, MODE><<<grid, threads, 0, s>>>(a); break;
        case 16: k_mm<16, MODE><<<grid, threads, 0, s>>>(a); break;
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" int fxp_mm(int mode, int grid, int threads, int unroll, const ProbeArgs* a, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (mode) {
        case 0: return launch_mm<0>(grid, threads, unroll, *a, s);
        case 1: return launch_mm<1>(grid, threads, unroll, *a, s);
        case 2: return launch_mm<2>(grid, threads, unroll, *a, s);
        case 3: return unroll > 4 ? -1 : launch_mm<3>(grid, threads, unroll, *a, s);
        case 4: return unroll > 8 ? -1 : launch_mm<4>(grid, threads, unroll, *a, s);
        case 5: return launch_mm<5>(grid, threads, unroll, *a, s);
        case 6: return launch_mm<6>(grid, threads, unroll, *a, s);
    }
    return -1;
}

extern "C" int fxp_mix(int grid, int threads, int unroll, int copy_unroll, const ProbeArgs* a, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (copy_unroll != 8) return -1;
    switch (unroll) {
        case 1: k_mix<1, 8><<<grid, threads, 0, s>>>(*a); break;
        case 2: k_mix<2, 8><<<grid, threads, 0, s>>>(*a); break;
        case 4: k_mix<4, 8><<<grid, threads, 0, s>>>(*a); break;
        case 8: k_mix<8, 8><<<grid, threads, 0, s>>>(*a); break;
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" int fxp_mix_tma(int grid, int threads, int unroll, const ProbeArgs* a, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    const int smem = TMA_STAGES * TMA_TILE + 64;
    static bool attr = false;
    if (!attr) {
        cudaFuncSetAttribute(k_mix_tma<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(k_mix_tma<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(k_mix_tma<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        cudaFuncSetAttribute(k_mix_tma<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        attr = true;
    }
    switch (unroll) {
        case 1: k_mix_tma<1><<<grid, threads, smem, s>>>(*a); break;
        case 2: k_mix_tma<2><<<grid, threads, smem, s>>>(*a); break;
        case 4: k_mix_tma<4><<<grid, threads, smem, s>>>(*a); break;
        case 8: k_mix_tma<8><<<grid, threads, smem, s>>>(*a); break;
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" int fxp_latency(const ProbeArgs* a, void* stream) {
    k_latency<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(*a);
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" int fxp_barrier(int variant, const ProbeArgs* a, void* stream) {
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    switch (variant) {
        case 0: k_barrier_probe<0><<<1, 64, 0, s>>>(*a); break;
        case 1: k_barrier_probe<1><<<1, 64, 0, s>>>(*a); break;
        case 2: k_barrier_probe<2><<<1, 64, 0, s>>>(*a); break;
        case 3: k_barrier_probe<3><<<1, 64, 0, s>>>(*a); break;
        default: return -1;
    }
    return cudaGetLastError() == cudaSuccess ? 0 : -2;
}

extern "C" int fxp_memset(void* p, int v, size_t n) { return cudaMemset(p, v, n) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess ? 0 : -2; }
extern "C" int fxp_memcpy(void* dst, const void* src, size_t n) {
    return cudaMemcpy(dst, src, n, cudaMemcpyDefault) == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess ? 0 : -2;
}
extern "C" int fxp_args_size(void) { return (int)sizeof(ProbeArgs); }
