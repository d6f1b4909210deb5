// k_fuse: the bucketed all-reduce as ONE kernel of five decoupled warp roles per CTA, with the
// bucket <-> tensor traffic staged through shared memory by the TMA engine (cp.async.bulk).
//
// Replaces, for float buckets averaged / summed in their own dtype, the per-tensor loop
//     all_reduce(t.data, SUM, async_op=True) ... handle.wait(); t.data /= world_size()
// of the reference (flashy/distrib.py:105-111) by a single launch.
//
// Layout (as in fx_kernels.cu): the bucket is W shards x gridDim.x slices; CTA b owns slice b of
// every shard and cuts it into `chunks` chunks of `chunk_elems` elements.  Chunk c of CTA b is
// W sub-ranges (one per shard) of <= FZ chunk bytes each.  Roles of a CTA:
//
//   pack    (1 warp)  tensors -> shared memory (cp.async.bulk, mbarrier) -> own arena, chunk by
//                     chunk, then "chunk c packed" to every peer's flags_pack[b][me]
//   poll    (1 warp)  reads flags_pack[b][*] / flags_red[b][*] of the own pad and publishes the
//                     minimum over ranks in shared memory (what every rank has packed / reduced)
//   reduce  (4 warps) units of 32 * U vectors of a chunk, round-robin over the warps: multimem.ld_reduce
//                     of the own shard's sub-range through the NVSwitch, / W, multimem.st to all arenas
//                     (or, without multicast: pull the W arenas in rank order, write the own one)
//   signal  (1 warp)  watches the reduce warps' progress in shared memory, fences ONCE at system
//                     scope and writes "chunks < n of shard me are reduced" to every peer
//   unpack  (1 warp)  arena (own after NVLS, peers' otherwise) -> shared memory -> output tensors
//
// Four reduce warps x U vectors per lane (U = 1 at 8 GPUs) keep 2 KiB of multimem requests in flight per
// SM: on an earlier target (B200) a few KiB per SM saturated the switch and much deeper queues only added
// queueing in front of the flags; benchmarks/nvls_probe.py measures both, not yet on H100.  The reduce warps
// never execute a system-scope fence (an order of magnitude dearer than a GPU-scope one on that target, more
// so while the SM streams multicast stores) and never wait
// for their own stores: the NVLink stream of a CTA only stalls when a peer is late.  Pieces whose tensor
// address is not 16-byte aligned and the (< 16 byte) tails of odd-sized tensors go through ordinary
// loads / stores of the same warp.
#include "fx_device.cuh"

namespace {

#define FZ_THREADS 256
#define FZ_WARP_POLL 0
#define FZ_WARP_SIG 1
#define FZ_WARP_PACK 2
#define FZ_WARP_UNPACK 3
#define FZ_WARP_RED0 4
#define FZ_RED_WARPS 4

// ---------------------------------------------------------------------------- shared-memory sync
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void st_release_cta(uint32_t* p, uint32_t v) {
    asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" :: "r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_cta(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// "chunks < n of my copy are packed": the packed data sits in THIS GPU's memory (written by bulk
// stores that have completed), and every reader -- the switch for multimem.ld_reduce, a peer's
// plain load -- is served by this GPU's L2, so ordering the flag behind the data at GPU scope is
// enough, and a GPU-scope fence was far cheaper than a system-scope one (benchmarks/nvls_probe.py, measured
// on an earlier target, B200; not yet on H100).
__device__ __forceinline__ void signal_packed(const FxLaunch& a, int lane, int world, int rank, int b, uint32_t value) {
    fence_gpu();
    if (lane < world) st_relaxed_sys(pipe_flag(a.arena[lane], FX_FLAG_PACK, b, rank), value);
}

// ---------------------------------------------------------------------------- TMA (cp.async.bulk)
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
// Wait until at most `n` of this thread's bulk groups are still reading shared memory / still in flight.
__device__ __forceinline__ void tma_wait_read(int n) {
    if (n <= 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    else if (n == 1) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
    else asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
}
__device__ __forceinline__ void tma_wait_done(int n) {
    if (n <= 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    else asm volatile("cp.async.bulk.wait_group 1;" ::: "memory");
}
// generic-proxy writes to shared memory -> visible to the async proxy (a following bulk store)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Debug trace of CTA 0 (FLASHY_B200_TRACE=1): globaltimer stamps, FZ_TR_CHUNKS chunks at most.
#define FZ_TR_CHUNKS 1024
#define FZ_TR_PACK 16                                  // [c][4]: loads issued, loads landed, stores complete(d), signalled
#define FZ_TR_UNPACK (FZ_TR_PACK + 4 * FZ_TR_CHUNKS)   // [c][4]: reduced seen, loads issued, loads landed, stores issued
#define FZ_TR_RED (FZ_TR_UNPACK + 4 * FZ_TR_CHUNKS)    // [c][4]: start wait, packed seen, stores issued, -
#define FZ_TR_SIG (FZ_TR_RED + 4 * FZ_TR_CHUNKS)       // [c][2]: detected, fence done
#define FZ_TR_POLLP (FZ_TR_SIG + 2 * FZ_TR_CHUNKS)     // [c]: "c+1 chunks packed everywhere" published
#define FZ_TR_POLLR (FZ_TR_POLLP + FZ_TR_CHUNKS)       // [c]: "c+1 chunks reduced everywhere" published
#define FZ_TR_CTA (FZ_TR_POLLR + FZ_TR_CHUNKS)         // [b][2]: kernel entry and exit of every CTA (hosted rank 0)
#define FZ_TR_WORDS (FZ_TR_CTA + 2 * FX_MAX_BLOCKS)

#define FZ_NB 3                             // staging buffers per copy role (chunks in flight)
struct FuseSync {
    uint64_t full_pack[FZ_NB], full_unp[FZ_NB];   // "the bulk loads of this buffer have landed"
    uint32_t packed;                       // chunks every rank has packed (this launch)
    uint32_t reduced;                      // chunks of every shard reduced and delivered
    uint32_t red_prog[FZ_RED_WARPS];       // units completed by each reduce warp
    uint32_t abort;                        // a peer never arrived: stop without touching the outputs
};

// Spin until *counter >= want (shared memory); false if the launch was aborted.
__device__ __forceinline__ bool wait_count(const uint32_t* counter, uint32_t want, const uint32_t* abort) {
    while (ld_acquire_cta(counter) < want) {
        if (*reinterpret_cast<const volatile uint32_t*>(abort)) return false;
        __nanosleep(20);
    }
    return true;
}

// The pieces of bucket range [lo, hi) (elements): for each tensor i intersecting it calls
// f(i, p0, p1) with the intersection [p0, p1).
template <typename F>
__device__ __forceinline__ void for_pieces(const Meta& m, long long lo, long long hi, F f) {
    if (lo >= m.off[m.n]) return;
    for (int i = find_tensor(m.off, m.n, lo); i < m.n && m.off[i] < hi; ++i) {
        const long long t0 = m.off[i], t1 = t0 + m.numel[i];
        const long long p0 = lo > t0 ? lo : t0, p1 = hi < t1 ? hi : t1;
        if (p1 > p0) f(i, p0, p1);
    }
}

// U: 16-byte vectors per lane a reduce warp keeps in flight (one unit = 32 * U vectors).
template <typename T, bool NVLS, int W, int U>
__global__ void __launch_bounds__(FZ_THREADS, 1) k_fuse(const FxLaunch a) {
    extern __shared__ __align__(128) unsigned char fz_dyn[];
    __shared__ MetaSmem meta_smem;
    __shared__ FuseSync sy;

    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = W > 0 ? W : a.world;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    FxPlanState* st = a.state + l;
    char* my = a.arena[rank];
    // the two owner-private words this launch depends on, fetched together
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const uint32_t base = ld_volatile_u32(&pad_of(my)->pipe_epoch[b]);
    const unsigned long long t_enter = (a.trace && l == 0 && threadIdx.x == 0) ? globaltimer_ns() : 0;
    if (a.trace && l == 0 && threadIdx.x == 0) a.trace[FZ_TR_CTA + 2 * b] = t_enter;
    const Meta m = load_meta(a, l, &meta_smem);                 // (contains a __syncthreads)
    if (a.trace && b == 0 && l == 0 && threadIdx.x == 0) { a.trace[0] = t_enter; a.trace[1] = globaltimer_ns(); a.trace[2] = (unsigned long long)a.chunks; }
    if (threadIdx.x == 0) {
        for (int i = 0; i < FZ_NB; ++i) { mbar_init(&sy.full_pack[i], 1); mbar_init(&sy.full_unp[i], 1); }
        sy.packed = 0; sy.reduced = 0; sy.abort = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (threadIdx.x < FZ_RED_WARPS) sy.red_prog[threadIdx.x] = 0;
    __syncthreads();

    const unsigned long long region = a.region[calls & 1];
    const long long slice = a.slice_elems, shard = a.shard_elems, csz = a.chunk_elems;
    const int chunks = a.chunks;
    const bool avg = a.op == FX_AVG;
    constexpr long long VEC = FX_VEC_BYTES / (long long)sizeof(T);
    const uint32_t cb = (uint32_t)(csz * sizeof(T));            // bytes of one full sub-range chunk
    unsigned char* pack_buf = fz_dyn;                                   // [FZ_NB][world * cb]
    unsigned char* unp_buf = fz_dyn + (size_t)FZ_NB * world * cb;       // [FZ_NB][world * cb]
    unsigned long long* trace = (a.trace && b == 0 && l == 0 && a.chunks <= FZ_TR_CHUNKS) ? a.trace : nullptr;

    if (warp == FZ_WARP_POLL) {
        // ------------------------------------------------------------ poll: peers' progress -> smem
        const int which = lane >> 4, q = lane & 15;
        const bool active = q < world;
        const uint32_t* flag = pipe_flag(my, which, b, active ? q : 0);
        uint32_t published = 0;
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        while (true) {
            uint32_t v = (uint32_t)chunks;
            if (active) {
                const int32_t d = (int32_t)(ld_acquire_sys(flag) - base);
                v = d < 0 ? 0u : ((uint32_t)d > (uint32_t)chunks ? (uint32_t)chunks : (uint32_t)d);
            }
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) { const uint32_t w = __shfl_xor_sync(0xffffffffu, v, o); v = w < v ? w : v; }
            if (q == 0 && v > published) {
                st_release_cta(which == FX_FLAG_PACK ? &sy.packed : &sy.reduced, v);
                if (trace) trace[(which == FX_FLAG_PACK ? FZ_TR_POLLP : FZ_TR_POLLR) + (v - 1)] = globaltimer_ns();
                published = v;
            }
            if (__all_sync(0xffffffffu, v >= (uint32_t)chunks)) break;
            if ((++spins & 0xff) == 0) {
                const unsigned long long now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                else if (now - t0 > a.timeout_ns) {               // a peer never arrived
                    if (lane == 0) {
                        *reinterpret_cast<volatile uint32_t*>(a.status) = (uint32_t)(-FX_ERR_TIMEOUT);
                        __threadfence_system();
                        *reinterpret_cast<volatile uint32_t*>(&sy.abort) = 1;
                    }
                    break;
                }
            }
        }
    } else if (warp == FZ_WARP_SIG) {
        // ------------------------------------------------------------ signal: reduced chunks -> peers
        constexpr uint32_t FZ_UNIT = 32 * U * FX_VEC_BYTES;
        const int upc = (int)((cb + FZ_UNIT - 1) / FZ_UNIT);
        int next = 0;
        while (next < chunks) {
            // lane w < FZ_RED_WARPS: how many chunks (counted from 0) are covered by warp w's finished units
            int covered = chunks;
            if (lane < FZ_RED_WARPS) {
                const long long done = ld_acquire_cta(&sy.red_prog[lane]);          // units finished by warp `lane`
                // warp w owns units w, w + R, ...: its first `done` units cover all units < done * R + w of its
                // residue class, i.e. every chunk c with (c + 1) * upc <= done * R + w ... conservatively:
                const long long upto = done * FZ_RED_WARPS + lane;                  // first unit of this warp NOT done
                covered = (int)(upto / upc);                                        // chunks entirely below it
                if (covered > chunks) covered = chunks;
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const int w = __shfl_xor_sync(0xffffffffu, covered, o); covered = w < covered ? w : covered; }
            if (covered <= next) {
                if (*reinterpret_cast<const volatile uint32_t*>(&sy.abort)) break;
                __nanosleep(40);
                continue;
            }
            if (trace && lane == 0) trace[FZ_TR_SIG + 2 * next] = globaltimer_ns();
            next = covered;
            // order the flag behind the reduce warps' stores (cumulative): they went to every peer's arena with
            // NVLS (system scope), to this GPU's own arena otherwise (GPU scope is enough, see signal_packed)
            // (holding the reduce warps' stores back for the moment of the fence was tried on B200: it made the kernel slower)
            if (NVLS) fence_sys(); else fence_gpu();
            if (trace && lane == 0) trace[FZ_TR_SIG + 2 * (next - 1) + 1] = globaltimer_ns();
            if (lane < world) st_relaxed_sys(pipe_flag(a.arena[lane], FX_FLAG_RED, b, rank), base + (uint32_t)next);
        }
    } else if (warp == FZ_WARP_PACK) {
        // ------------------------------------------------------------ pack: tensors -> smem -> arena
        // Greedy software pipeline over FZ_NB staging buffers: bulk loads run up to FZ_NB - 1 chunks
        // ahead of the bulk stores, and "chunk c is packed" goes out one chunk behind the stores
        // (wait_group 1), except for the first and the last chunk, which are drained at once.
        int L = 0, S = 0;                                          // chunks whose loads / stores are issued
        while (S < chunks) {
            if (L < chunks && L - S < FZ_NB - 1) {
                const int c = L;
                const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
                const int nb = c % FZ_NB;
                unsigned char* buf = pack_buf + (size_t)nb * world * cb;
                if (lane == 0) tma_wait_read(FZ_NB - 1 - (L - S));    // the stores of chunk c - FZ_NB left this buffer
                __syncwarp();
                // lane s enumerates sub-range s (the pieces of the W sub-ranges are independent): bulk loads
                // for every piece whose source is 16-byte aligned; odd pieces and tails are left to pass 2
                uint32_t tx = 0;
                bool generic = false;
                if (lane < world) {
                    const int s = lane;
                    const long long lo = s * shard + b * slice + c0, hi = lo + (c1 - c0);
                    unsigned char* sbase = buf + (size_t)s * cb;
                    for_pieces(m, lo, hi, [&](int i, long long p0, long long p1) {
                        const T* src = static_cast<const T*>(m.in[i]) + (p0 - m.off[i]);
                        T* dst = reinterpret_cast<T*>(sbase) + (p0 - lo);
                        const long long n = p1 - p0;
                        long long bulk = 0;
                        if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
                            bulk = n / VEC * VEC;
                            if (bulk) {
                                tma_load(dst, src, (uint32_t)(bulk * sizeof(T)), &sy.full_pack[nb]);
                                tx += (uint32_t)(bulk * sizeof(T));
                            }
                        }
                        if (bulk < n) generic = true;
                    });
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) tx += __shfl_xor_sync(0xffffffffu, tx, o);
                if (__any_sync(0xffffffffu, generic)) {
                    // pass 2 (rare): the whole warp copies what the bulk loads could not take
                    for (int s = 0; s < world; ++s) {
                        const long long lo = s * shard + b * slice + c0, hi = lo + (c1 - c0);
                        unsigned char* sbase = buf + (size_t)s * cb;
                        for_pieces(m, lo, hi, [&](int i, long long p0, long long p1) {
                            const T* src = static_cast<const T*>(m.in[i]) + (p0 - m.off[i]);
                            T* dst = reinterpret_cast<T*>(sbase) + (p0 - lo);
                            const long long n = p1 - p0;
                            const long long bulk = (reinterpret_cast<uintptr_t>(src) & 15) == 0 ? n / VEC * VEC : 0;
                            for (long long e = bulk + lane; e < n; e += 32) dst[e] = src[e];
                        });
                    }
                    fence_proxy_async_smem();
                }
                __syncwarp();
                if (lane == 0) mbar_expect_tx(&sy.full_pack[nb], tx);
                if (trace && lane == 0) trace[FZ_TR_PACK + 4 * c + 0] = globaltimer_ns();
                ++L;
                continue;
            }
            const int c = S;
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            const int nb = c % FZ_NB;
            unsigned char* buf = pack_buf + (size_t)nb * world * cb;
            mbar_wait(&sy.full_pack[nb], (uint32_t)((c / FZ_NB) & 1));
            if (trace && lane == 0) trace[FZ_TR_PACK + 4 * c + 1] = globaltimer_ns();
            if (lane == 0) {
                for (int s = 0; s < world; ++s) {
                    const long long lo = s * shard + b * slice + c0;
                    tma_store(my + region + (unsigned long long)lo * sizeof(T), buf + (size_t)s * cb, (uint32_t)((c1 - c0) * sizeof(T)));
                }
                tma_commit();
            }
            ++S;
            const bool drain = S == 1 || S == chunks;              // keep the first chunk's latency and the tail short
            if (lane == 0) tma_wait_done(drain ? 0 : 1);
            __syncwarp();
            const int ready = drain ? S : S - 1;                   // chunks whose stores have completed
            if (trace && lane == 0) trace[FZ_TR_PACK + 4 * c + 2] = globaltimer_ns();
            if (ready > 0) signal_packed(a, lane, world, rank, b, base + (uint32_t)ready);
            if (trace && lane == 0) trace[FZ_TR_PACK + 4 * c + 3] = globaltimer_ns();
        }
    } else if (warp == FZ_WARP_UNPACK) {
        // ------------------------------------------------------------ unpack: arena -> smem -> tensors
        // Same greedy pipeline: the bulk loads of a chunk start the moment every shard's part of it is
        // reduced (up to FZ_NB - 1 chunks ahead); otherwise the oldest landed chunk is stored.
        int L = 0, S = 0;
        bool alive = true;
        while (S < chunks && alive) {
            const bool can_load = L < chunks && L - S < FZ_NB - 1;
            const uint32_t seen = __shfl_sync(0xffffffffu, ld_acquire_cta(&sy.reduced), 0);
            if (can_load && (L == S || seen >= (uint32_t)L + 1)) {
                if (L == S && !wait_count(&sy.reduced, (uint32_t)L + 1, &sy.abort)) { alive = false; break; }
                const int c = L;
                const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
                const uint32_t bytes = (uint32_t)((c1 - c0) * sizeof(T));
                const int nb = c % FZ_NB;
                unsigned char* buf = unp_buf + (size_t)nb * world * cb;
                if (trace && lane == 0) trace[FZ_TR_UNPACK + 4 * c + 0] = globaltimer_ns();
                if (lane < world) tma_wait_read(FZ_NB - 1 - (L - S));  // lane s stored sub-range s of chunk c - FZ_NB from this buffer
                __syncwarp();
                if (lane == 0) {
                    mbar_expect_tx(&sy.full_unp[nb], bytes * (uint32_t)world);
                    for (int s = 0; s < world; ++s) {
                        const long long lo = s * shard + b * slice + c0;
                        const char* from = (NVLS ? my : a.arena[s]) + region + (unsigned long long)lo * sizeof(T);
                        tma_load(buf + (size_t)s * cb, from, bytes, &sy.full_unp[nb]);
                    }
                }
                __syncwarp();
                if (trace && lane == 0) trace[FZ_TR_UNPACK + 4 * c + 1] = globaltimer_ns();
                ++L;
                continue;
            }
            const int c = S;
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            const int nb = c % FZ_NB;
            const unsigned char* buf = unp_buf + (size_t)nb * world * cb;
            mbar_wait(&sy.full_unp[nb], (uint32_t)((c / FZ_NB) & 1));
            if (trace && lane == 0) trace[FZ_TR_UNPACK + 4 * c + 2] = globaltimer_ns();
            // lane s stores the pieces of sub-range s (one bulk group per lane and chunk)
            bool generic = false;
            if (lane < world) {
                const int s = lane;
                const long long lo = s * shard + b * slice + c0, hi = lo + (c1 - c0);
                const unsigned char* sbase = buf + (size_t)s * cb;
                for_pieces(m, lo, hi, [&](int i, long long p0, long long p1) {
                    T* dst = static_cast<T*>(m.out[i]) + (p0 - m.off[i]);
                    const T* src = reinterpret_cast<const T*>(sbase) + (p0 - lo);
                    const long long n = p1 - p0;
                    long long bulk = 0;
                    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
                        bulk = n / VEC * VEC;
                        if (bulk) tma_store(dst, src, (uint32_t)(bulk * sizeof(T)));
                    }
                    if (bulk < n) generic = true;
                });
                tma_commit();
            }
            if (__any_sync(0xffffffffu, generic)) {
                for (int s = 0; s < world; ++s) {
                    const long long lo = s * shard + b * slice + c0, hi = lo + (c1 - c0);
                    const unsigned char* sbase = buf + (size_t)s * cb;
                    for_pieces(m, lo, hi, [&](int i, long long p0, long long p1) {
                        T* dst = static_cast<T*>(m.out[i]) + (p0 - m.off[i]);
                        const T* src = reinterpret_cast<const T*>(sbase) + (p0 - lo);
                        const long long n = p1 - p0;
                        const long long bulk = (reinterpret_cast<uintptr_t>(dst) & 15) == 0 ? n / VEC * VEC : 0;
                        for (long long e = bulk + lane; e < n; e += 32) dst[e] = src[e];
                    });
                }
            }
            __syncwarp();
            if (trace && lane == 0) trace[FZ_TR_UNPACK + 4 * c + 3] = globaltimer_ns();
            ++S;
        }
        if (lane < world) tma_wait_done(0);
    } else {
        // ------------------------------------------------------------ reduce: 1 KiB units, round-robin over the warps
        // A chunk of one sub-range is cut into units of FZ_UNIT bytes (one unit = 2 vectors per lane); unit
        // u = c * upc + j goes to warp u % FZ_RED_WARPS, so the warps share a chunk's latency when chunks
        // are large (small worlds) and a chunk's latency is one batch of loads per warp.
        const int rw = warp - FZ_WARP_RED0;
        constexpr long long uvec = 32 * U;                          // vectors per unit
        constexpr uint32_t FZ_UNIT = 32 * U * FX_VEC_BYTES;         // bytes per unit
        const int upc = (int)((cb + FZ_UNIT - 1) / FZ_UNIT);       // units per chunk
        const long long units = (long long)chunks * upc;
        uint32_t mine = 0;
        for (long long u = rw; u < units; u += FZ_RED_WARPS) {
            const int c = (int)(u / upc), j = (int)(u % upc);
            if (trace && lane == 0 && j == 0) trace[FZ_TR_RED + 4 * c + 0] = globaltimer_ns();
            if (!wait_count(&sy.packed, (uint32_t)c + 1, &sy.abort)) break;
            if (trace && lane == 0 && j == 0) trace[FZ_TR_RED + 4 * c + 1] = globaltimer_ns();
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            const long long cvec = (c1 - c0) / VEC;                 // vectors of this chunk (the last one may be short)
            const long long v_lo = j * uvec, v_hi = (v_lo + uvec < cvec) ? v_lo + uvec : cvec;
            if (v_lo < v_hi) {
                const unsigned long long byte_off = region + (unsigned long long)(rank * shard + b * slice + c0) * sizeof(T)
                                                    + (unsigned long long)v_lo * FX_VEC_BYTES;
                const long long nvec = v_hi - v_lo;
                if (NVLS) {
                    char* mc = a.mc_arena + byte_off;
                    for (long long v0 = lane; v0 < nvec; v0 += 32 * U) {
                        uint4 r[U];
#pragma unroll
                        for (int k = 0; k < U; ++k) { const long long v = v0 + 32 * k; if (v < nvec) r[k] = Multimem<T>::ld_reduce(mc + v * FX_VEC_BYTES); }
#pragma unroll
                        for (int k = 0; k < U; ++k) { const long long v = v0 + 32 * k; if (v < nvec) multimem_st(mc + v * FX_VEC_BYTES, avg ? scale_vec<T>(r[k], world) : r[k]); }
                    }
                } else {
                    reduce_vectors<T, W, FX_SUM>(a, world, byte_off, nvec, avg, my, Lane{lane, 32});
                }
            }
            __syncwarp();
            if (trace && lane == 0 && j == upc - 1) trace[FZ_TR_RED + 4 * c + 2] = globaltimer_ns();
            if (lane == 0) st_release_cta(&sy.red_prog[rw], ++mine);
        }
    }
    __syncthreads();
    if (trace && threadIdx.x == 0) trace[3] = globaltimer_ns();
    if (a.trace && l == 0 && threadIdx.x == 0) a.trace[FZ_TR_CTA + 2 * b + 1] = globaltimer_ns();
    if (threadIdx.x == 0) {
        pad_of(my)->pipe_epoch[b] = base + (uint32_t)chunks;
        if (atomicAdd(&st->finished, 1u) == gridDim.x - 1) {
            st->finished = 0;
            *reinterpret_cast<volatile uint32_t*>(&st->calls) = calls + 1;
        }
    }
}

template <typename K>
int launch_fuse(K kernel, const fx_plan* plan, const FxLaunch& args, size_t smem, cudaStream_t stream) {
    static thread_local const void* configured[32];
    static thread_local int n_configured = 0;
    const void* fn = reinterpret_cast<const void*>(kernel);
    bool seen = false;
    for (int i = 0; i < n_configured; ++i) seen = seen || configured[i] == fn;
    if (!seen) {
        cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 192 << 10);
        if (e != cudaSuccess) return fx_fail(FX_ERR_CUDA, "cudaFuncSetAttribute(k_fuse): %s", cudaGetErrorString(e));
        if (n_configured < 32) configured[n_configured++] = fn;
    }
    dim3 grid(plan->grid_x, args.n_local), block(FZ_THREADS);
    void* params[] = {const_cast<FxLaunch*>(&args)};
    cudaError_t e = args.n_local > 1
        ? cudaLaunchCooperativeKernel(fn, grid, block, params, smem, stream)      // virtual ranks must be co-resident
        : cudaLaunchKernel(fn, grid, block, params, smem, stream);
    if (e != cudaSuccess) return fx_fail(FX_ERR_CUDA, "k_fuse launch failed: %s", cudaGetErrorString(e));
    return FX_OK;
}

template <typename T>
int launch_fuse_t(fx_plan* plan, const FxLaunch& a, size_t smem, cudaStream_t s) {
    if (plan->algo == FX_ALGO_NVLS) {
        switch (plan->fuse_unroll) {               // FLASHY_B200_FUSE_DEPTH: multimem vectors in flight per lane
            case 1: return launch_fuse(k_fuse<T, true, 0, 1>, plan, a, smem, s);
            case 4: return launch_fuse(k_fuse<T, true, 0, 4>, plan, a, smem, s);
            case 8: return launch_fuse(k_fuse<T, true, 0, 8>, plan, a, smem, s);
            default: return launch_fuse(k_fuse<T, true, 0, 2>, plan, a, smem, s);
        }
    }
    switch (a.world) {
        case 2: return launch_fuse(k_fuse<T, false, 2, 2>, plan, a, smem, s);
        case 4: return launch_fuse(k_fuse<T, false, 4, 2>, plan, a, smem, s);
        case 8: return launch_fuse(k_fuse<T, false, 8, 2>, plan, a, smem, s);
    }
    return launch_fuse(k_fuse<T, false, 0, 2>, plan, a, smem, s);
}

}  // namespace

size_t fx_fuse_smem_bytes(int world, long long chunk_bytes) { return 2ull * FZ_NB * world * chunk_bytes; }
size_t fx_fuse_trace_words(void) { return FZ_TR_WORDS; }

int fx_launch_fuse(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    if (plan->algo == FX_ALGO_NVLS && !a.mc_arena) return fx_fail(FX_ERR_STATE, "NVLS plan without a multicast mapping");
    const size_t smem = fx_fuse_smem_bytes(a.world, a.chunk_elems * (long long)plan->wsize);
    switch (plan->wire) {
        case FX_F32: return launch_fuse_t<float>(plan, a, smem, s);
        case FX_BF16: return launch_fuse_t<__nv_bfloat16>(plan, a, smem, s);
        case FX_F16: return launch_fuse_t<__half>(plan, a, smem, s);
    }
    return fx_fail(FX_ERR_UNSUPPORTED, "the fused kernel handles fp32 / bf16 / fp16 buckets only");
}
