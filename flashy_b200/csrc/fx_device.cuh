// Device-side building blocks shared by the collective kernels (fx_kernels.cu, fx_fuse.cu):
// 128-bit global accesses, system-scope flags, type traits, the per-CTA view of the bucket
// metadata and the converting copy / reduction loops.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "fx_internal.h"

namespace {

// ============================================================================ primitives
__device__ __forceinline__ uint4 ld16(const void* p) {
    uint4 v;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st16(void* p, const uint4& v) {
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ FxPad* pad_of(char* arena) { return reinterpret_cast<FxPad*>(arena); }

// All CTAs `b` of the W ranks meet here.  `target` is the new epoch value.  Returns false when a
// peer did not arrive within the time bound: the sticky status word is set and the caller must
// leave the kernel WITHOUT touching any output tensor (whatever sits in the peers' arenas is not
// the data of this collective; the host raises at its next call / poll).
__device__ __forceinline__ bool block_barrier(const FxLaunch& a, int rank, int world, int b,
                                              uint32_t target) {
    __shared__ int s_timed_out;
    if (threadIdx.x == 0) s_timed_out = 0;
    __syncthreads();
    if (threadIdx.x < world) {
        const int q = threadIdx.x;
        // release at system scope: the CTA's earlier writes (ordered before this thread by the
        // bar.sync above) are visible to whoever acquires the flag
        st_release_sys(&pad_of(a.arena[q])->flags[b][rank], target);
        const uint32_t* mine = &pad_of(a.arena[rank])->flags[b][q];
        unsigned long long t0 = 0;
        uint32_t spins = 0;
        // (polling relaxed + one fence.acq_rel.sys afterwards measured slower per barrier on B200)
        while ((int32_t)(ld_acquire_sys(mine) - target) < 0) {
            if ((++spins & 0x3ff) == 0) {
                const unsigned long long now = globaltimer_ns();
                if (t0 == 0) t0 = now;
                else if (now - t0 > a.timeout_ns) {        // peer never arrived: flag it, do not hang
                    *reinterpret_cast<volatile uint32_t*>(a.status) = (uint32_t)(-FX_ERR_TIMEOUT);
                    __threadfence_system();
                    s_timed_out = 1;
                    break;
                }
            }
        }
    }
    __syncthreads();
    return s_timed_out == 0;
}

// ============================================================================ type traits
template <typename T> struct Acc { using type = float; };
template <> struct Acc<double> { using type = double; };
template <> struct Acc<int32_t> { using type = int32_t; };
template <> struct Acc<int64_t> { using type = int64_t; };
template <> struct Acc<uint8_t> { using type = uint8_t; };

template <typename D, typename S> __device__ __forceinline__ D cvt(S x) { return static_cast<D>(x); }
template <> __device__ __forceinline__ float cvt<float, __nv_bfloat16>(__nv_bfloat16 x) { return __bfloat162float(x); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<__nv_bfloat16, float>(float x) { return __float2bfloat16_rn(x); }
template <> __device__ __forceinline__ float cvt<float, __half>(__half x) { return __half2float(x); }
template <> __device__ __forceinline__ __half cvt<__half, float>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<__nv_bfloat16, __nv_bfloat16>(__nv_bfloat16 x) { return x; }
template <> __device__ __forceinline__ __half cvt<__half, __half>(__half x) { return x; }

template <typename T> union Vec16 {
    uint4 u;
    T e[FX_VEC_BYTES / sizeof(T)];
    __device__ Vec16() {}
};

template <int OP, typename A> __device__ __forceinline__ A combine(A x, A y) {
    if (OP == FX_MAX) return x > y ? x : y;
    if (OP == FX_MIN) return x < y ? x : y;
    if (OP == FX_PROD) return x * y;
    return x + y;
}

// ============================================================================ bucket <-> tensors
// Per-CTA view of the bucket metadata.  Walking it from global memory costs a chain of
// dependent DRAM round trips per slice (binary search over the offsets, then the
// pointers), a large fixed latency per launch.  So each CTA first copies
// the tables into shared memory with one coalesced pass (buckets of up to FX_SMEM_TENSORS
// tensors; larger ones keep reading global memory).
#define FX_SMEM_TENSORS 1024
struct Meta {
    const long long* off;       // [n + 1]
    const long long* numel;     // [n]
    const void* const* in;      // [n] this hosted rank's input tensors
    void* const* out;           // [n] this hosted rank's output tensors
    int n;
};

struct MetaSmem {
    long long off[FX_SMEM_TENSORS + 1];
    long long numel[FX_SMEM_TENSORS];
    const void* in[FX_SMEM_TENSORS];
    void* out[FX_SMEM_TENSORS];
};

__device__ __forceinline__ Meta load_meta(const FxLaunch& a, int l, MetaSmem* sm) {
    Meta m;
    m.n = a.n;
    const long long* g_off = a.off;
    const long long* g_numel = a.off + a.n + 1;
    const void* const* g_in = a.in_ptrs + (long long)l * a.n;
    void* const* g_out = a.out_ptrs + (long long)l * a.n;
    if (a.n <= FX_SMEM_TENSORS) {
        for (int i = threadIdx.x; i <= a.n; i += (int)blockDim.x) sm->off[i] = g_off[i];
        for (int i = threadIdx.x; i < a.n; i += (int)blockDim.x) {
            sm->numel[i] = g_numel[i];
            sm->in[i] = g_in[i];
            sm->out[i] = g_out[i];
        }
        __syncthreads();
        m.off = sm->off; m.numel = sm->numel; m.in = sm->in; m.out = sm->out;
    } else {
        m.off = g_off; m.numel = g_numel; m.in = g_in; m.out = g_out;
    }
    return m;
}

// Largest i with off[i] <= x (off is sorted, n >= 1, off[0] == 0).
__device__ __forceinline__ int find_tensor(const long long* off, int n, long long x) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (off[mid] <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// Position of a thread inside the group of threads that works on one slice.
struct Lane {
    int tid, nth;
};
__device__ __forceinline__ Lane block_lane() { return Lane{(int)threadIdx.x, FX_THREADS}; }

// The W slices a CTA packs / gathers per phase are independent: they are handed to disjoint
// warp groups so that all W are in flight together (a serial loop over them pays W dependent
// memory round trips, which dominates small buckets).  Slice index s is served by the warps
// with warp % min(W, 16) == s; with W > 16 a group loops over s, s + 16, ...
__device__ __forceinline__ Lane slice_lane(int world, int* first, int* step) {
    constexpr int kWarps = FX_THREADS / 32;
    const int groups = world < kWarps ? world : kWarps;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = warp % groups;
    const int members = kWarps / groups + (g < kWarps % groups ? 1 : 0);
    *first = g;
    *step = groups;
    return Lane{(warp / groups) * 32 + lane, members * 32};
}

// Group-wide converting copy of `len` elements.  The vector path needs both ends 16-byte
// aligned (always true for the arena side; torch allocations make it true for the tensors in
// practice); otherwise the whole range goes element by element.
template <typename Src, typename Dst>
__device__ __forceinline__ void copy_convert(const Src* __restrict__ src, Dst* __restrict__ dst, long long len, Lane ln) {
    constexpr int kMin = sizeof(Src) < sizeof(Dst) ? sizeof(Src) : sizeof(Dst);
    constexpr int UE = FX_VEC_BYTES / kMin;                    // elements per unit
    constexpr int NL = UE * sizeof(Src) / FX_VEC_BYTES;        // 16-byte loads per unit
    constexpr int NS = UE * sizeof(Dst) / FX_VEC_BYTES;        // 16-byte stores per unit
    constexpr int U = NL >= 2 ? 4 : 8;                         // units in flight per thread
    const bool aligned = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    const long long nunit = aligned ? len / UE : 0;
    for (long long u0 = ln.tid; u0 < nunit; u0 += (long long)U * ln.nth) {
        Vec16<Src> in[U][NL];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const long long u = u0 + (long long)k * ln.nth;
            if (u < nunit) {
#pragma unroll
                for (int j = 0; j < NL; ++j)
                    in[k][j].u = ld16(reinterpret_cast<const uint4*>(src + u * UE) + j);
            }
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const long long u = u0 + (long long)k * ln.nth;
            if (u < nunit) {
                Vec16<Dst> out[NS];
#pragma unroll
                for (int e = 0; e < UE; ++e) {
                    constexpr int SPL = FX_VEC_BYTES / sizeof(Src), DPL = FX_VEC_BYTES / sizeof(Dst);
                    out[e / DPL].e[e % DPL] = cvt<Dst, Src>(in[k][e / SPL].e[e % SPL]);
                }
#pragma unroll
                for (int j = 0; j < NS; ++j)
                    st16(reinterpret_cast<uint4*>(dst + u * UE) + j, out[j].u);
            }
        }
    }
    for (long long e = nunit * UE + ln.tid; e < len; e += ln.nth)
        dst[e] = cvt<Dst, Src>(src[e]);
}

// Tensor index of bucket element e, walking forward from a known lower bound i.
__device__ __forceinline__ int walk_tensor(const Meta& m, int i, long long e) {
    while (i + 1 < m.n && m.off[i + 1] <= e) ++i;
    return i;
}

// Unit-by-unit move of bucket range [lo, hi) (a run of small tensors): every thread looks its
// unit's tensor up in the shared-memory table, so all loads of the run are in flight together
// instead of one short dependent copy per tensor.
template <typename T, typename S, bool PACK>
__device__ __forceinline__ void move_run(const Meta& m, T* stage, int i0, long long lo, long long hi, Lane ln) {
    constexpr int kMin = sizeof(S) < sizeof(T) ? sizeof(S) : sizeof(T);
    constexpr int UE = FX_VEC_BYTES / kMin;
    const long long nunit = (hi - lo + UE - 1) / UE;
    for (long long u = ln.tid; u < nunit; u += ln.nth) {
        const long long e = lo + u * UE;
        const int i = walk_tensor(m, i0, e);
        const long long t0 = m.off[i], t1 = t0 + m.numel[i];
        if (e >= t1) continue;                                 // alignment padding between tensors
        const int cnt = (t1 - e) < UE ? (int)(t1 - e) : UE;
        T* st = stage + e;
        if (PACK) {
            const S* src = static_cast<const S*>(m.in[i]) + (e - t0);
            if (cnt == UE && (reinterpret_cast<uintptr_t>(src) & 15) == 0) copy_convert<S, T>(src, st, UE, Lane{0, 1});
            else for (int k = 0; k < cnt; ++k) st[k] = cvt<T, S>(src[k]);
        } else {
            S* dst = static_cast<S*>(m.out[i]) + (e - t0);
            if (cnt == UE && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) copy_convert<T, S>(st, dst, UE, Lane{0, 1});
            else for (int k = 0; k < cnt; ++k) dst[k] = cvt<S, T>(st[k]);
        }
    }
}

// Move bucket range [lo, hi) between the tensors (type S) and the staging buffer (type T).
// PACK: tensors -> stage, else stage -> tensors.  Pieces of at least one unit per thread are
// streamed with the unrolled group-wide copy; runs of smaller pieces (BatchNorm vectors,
// biases) go through move_run.
template <typename T, typename S, bool PACK>
__device__ __forceinline__ void move_slice(const Meta& m, T* stage, long long lo, long long hi, Lane ln) {
    if (lo >= m.off[m.n]) return;                              // pure padding
    constexpr int kMin = sizeof(S) < sizeof(T) ? sizeof(S) : sizeof(T);
    constexpr int UE = FX_VEC_BYTES / kMin;
    const long long big = (long long)ln.nth * UE;
    const int i0 = find_tensor(m.off, m.n, lo);
    long long run_lo = -1, run_hi = 0;
    int run_i0 = 0;
    for (int i = i0; i < m.n && m.off[i] < hi; ++i) {
        const long long t0 = m.off[i], t1 = t0 + m.numel[i];
        const long long s0 = lo > t0 ? lo : t0, s1 = hi < t1 ? hi : t1;
        if (s1 <= s0) continue;
        if (s1 - s0 >= big) {
            if (run_lo >= 0) { move_run<T, S, PACK>(m, stage, run_i0, run_lo, run_hi, ln); run_lo = -1; }
            if (PACK) copy_convert<S, T>(static_cast<const S*>(m.in[i]) + (s0 - t0), stage + s0, s1 - s0, ln);
            else copy_convert<T, S>(stage + s0, static_cast<S*>(m.out[i]) + (s0 - t0), s1 - s0, ln);
        } else {
            if (run_lo < 0) { run_lo = s0; run_i0 = i; }
            run_hi = s1;
        }
    }
    if (run_lo >= 0) move_run<T, S, PACK>(m, stage, run_i0, run_lo, run_hi, ln);
}

// All W slices `b` of a CTA (slice b of every shard), spread over the warp groups.
template <typename T, typename S, bool PACK>
__device__ __forceinline__ void move_all_slices(const Meta& m, T* stage, long long shard, long long slice, int b, int world) {
    int first, step;
    const Lane ln = slice_lane(world, &first, &step);
    for (int s = first; s < world; s += step) {
        const long long lo = s * shard + b * slice;
        move_slice<T, S, PACK>(m, stage, lo, lo + slice, ln);
    }
}

// ============================================================================ reductions
template <typename T, int OP>
__device__ __forceinline__ void accumulate(typename Acc<T>::type* acc, const uint4& raw, bool first) {
    using A = typename Acc<T>::type;
    constexpr int VEC = FX_VEC_BYTES / sizeof(T);
    Vec16<T> v;
    v.u = raw;
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
        const A x = cvt<A, T>(v.e[e]);
        acc[e] = first ? x : combine<OP, A>(acc[e], x);
    }
}

template <typename T>
__device__ __forceinline__ uint4 finalize(typename Acc<T>::type* acc, bool avg, int world) {
    using A = typename Acc<T>::type;
    constexpr int VEC = FX_VEC_BYTES / sizeof(T);
    Vec16<T> v;
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
        A x = acc[e];
        if (avg) x = x / static_cast<A>(world);           // true division, flashy/distrib.py:111
        v.e[e] = cvt<T, A>(x);
    }
    return v.u;
}

// Reduce `nvec` 16-byte vectors starting at byte offset `byte_off` of every rank's arena, in
// rank order, and store the result at the same offset of `dst_arena`.  W > 0: compile-time
// world (all W loads of a vector in flight at once); W == 0: runtime world.
template <typename T, int W, int OP>
__device__ __forceinline__ void reduce_vectors(const FxLaunch& a, int world, unsigned long long byte_off,
                                               long long nvec, bool avg, char* dst_arena, Lane ln) {
    using A = typename Acc<T>::type;
    constexpr int VEC = FX_VEC_BYTES / sizeof(T);
    uint4* dst = reinterpret_cast<uint4*>(dst_arena + byte_off);
    if (W > 0) {
        constexpr int WW = W > 0 ? W : 1;
        constexpr int U = (16 / WW) < 1 ? 1 : ((16 / WW) > 4 ? 4 : (16 / WW));
        const uint4* base[WW];
#pragma unroll
        for (int q = 0; q < WW; ++q) base[q] = reinterpret_cast<const uint4*>(a.arena[q] + byte_off);
        for (long long v0 = ln.tid; v0 < nvec; v0 += (long long)U * ln.nth) {
            uint4 raw[U][WW];
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const long long v = v0 + (long long)k * ln.nth;
                if (v < nvec) {
#pragma unroll
                    for (int q = 0; q < WW; ++q) raw[k][q] = ld16(base[q] + v);
                }
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const long long v = v0 + (long long)k * ln.nth;
                if (v < nvec) {
                    A acc[VEC];
#pragma unroll
                    for (int q = 0; q < WW; ++q) accumulate<T, OP>(acc, raw[k][q], q == 0);
                    st16(dst + v, finalize<T>(acc, avg, world));
                }
            }
        }
    } else {
        constexpr int U = 4;
        for (long long v0 = ln.tid; v0 < nvec; v0 += (long long)U * ln.nth) {
            A acc[U][VEC];
            for (int q = 0; q < world; ++q) {
                const uint4* base = reinterpret_cast<const uint4*>(a.arena[q] + byte_off);
                uint4 raw[U];
#pragma unroll
                for (int k = 0; k < U; ++k) {
                    const long long v = v0 + (long long)k * ln.nth;
                    if (v < nvec) raw[k] = ld16(base + v);
                }
#pragma unroll
                for (int k = 0; k < U; ++k) {
                    const long long v = v0 + (long long)k * ln.nth;
                    if (v < nvec) accumulate<T, OP>(acc[k], raw[k], q == 0);
                }
            }
#pragma unroll
            for (int k = 0; k < U; ++k) {
                const long long v = v0 + (long long)k * ln.nth;
                if (v < nvec) st16(dst + v, finalize<T>(acc[k], avg, world));
            }
        }
    }
}

// One-shot tail: reduce bucket range [lo, hi) over all arenas and write the result straight
// into the output tensors (no second staging pass, no second barrier).  Unit by unit with a
// per-thread table lookup; the W loads of a unit are issued together.
template <typename T, typename S, int OP>
__device__ __forceinline__ void reduce_unpack_range(const FxLaunch& a, const Meta& m, int world, unsigned long long region,
                                                    long long lo, long long hi, bool avg) {
    using A = typename Acc<T>::type;
    constexpr int VEC = FX_VEC_BYTES / sizeof(T);
    if (lo >= m.off[m.n]) return;
    const int i0 = find_tensor(m.off, m.n, lo);
    const long long nvec = (hi - lo) / VEC;
    for (long long v = threadIdx.x; v < nvec; v += FX_THREADS) {
        const long long e = lo + v * VEC;
        const int i = walk_tensor(m, i0, e);
        const long long t0 = m.off[i], t1 = t0 + m.numel[i];
        if (e >= t1) continue;
        const int cnt = (t1 - e) < VEC ? (int)(t1 - e) : VEC;
        const unsigned long long byte_off = region + (unsigned long long)e * sizeof(T);
        A acc[VEC];
        if (world <= 8) {
            uint4 raw[8];
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q < world) raw[q] = ld16(a.arena[q] + byte_off);
#pragma unroll
            for (int q = 0; q < 8; ++q)
                if (q < world) accumulate<T, OP>(acc, raw[q], q == 0);
        } else {
            for (int q = 0; q < world; ++q) accumulate<T, OP>(acc, ld16(a.arena[q] + byte_off), q == 0);
        }
        S* dst = static_cast<S*>(m.out[i]) + (e - t0);
        __align__(16) S vals[VEC];
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
            A x = acc[k];
            if (avg) x = x / static_cast<A>(world);
            vals[k] = cvt<S, T>(cvt<T, A>(x));                 // round to the wire type first: same bits as two-shot
        }
        if (cnt == VEC && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            constexpr int NS = VEC * sizeof(S) / FX_VEC_BYTES;
            const uint4* packed = reinterpret_cast<const uint4*>(vals);
#pragma unroll
            for (int j = 0; j < NS; ++j) st16(reinterpret_cast<uint4*>(dst) + j, packed[j]);
        } else {
#pragma unroll
            for (int k = 0; k < VEC; ++k)
                if (k < cnt) dst[k] = vals[k];
        }
    }
}


// ---------------------------------------------------------------------------- NVLS
// multimem.ld_reduce: the NVSwitch reads the addressed 16 bytes from every GPU bound to the
// multicast object, adds them (fp32 accumulation) and returns the sum; multimem.st writes the
// 16 bytes into every GPU's copy.  Per GPU and direction this moves (1 + 1/W) N bytes instead
// of the 2 (W-1)/W N of the peer-to-peer two-shot.
template <typename T> struct Multimem;
template <> struct Multimem<float> {
    static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
        uint4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
        return v;
    }
};
template <> struct Multimem<__nv_bfloat16> {
    static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
        uint4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
        return v;
    }
};
template <> struct Multimem<__half> {
    static __device__ __forceinline__ uint4 ld_reduce(const void* p) {
        uint4 v;
        asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
        return v;
    }
};
__device__ __forceinline__ void multimem_st(void* p, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

template <typename T>
__device__ __forceinline__ uint4 scale_vec(const uint4& raw, int world) {
    using A = typename Acc<T>::type;
    constexpr int VEC = FX_VEC_BYTES / sizeof(T);
    Vec16<T> v;
    v.u = raw;
#pragma unroll
    for (int e = 0; e < VEC; ++e) v.e[e] = cvt<T, A>(cvt<A, T>(v.e[e]) / static_cast<A>(world));
    return v.u;
}

// In-switch reduction of `nvec` vectors at `mc` (multicast address of this rank's shard piece).
template <typename T>
__device__ __forceinline__ void nvls_vectors(char* mc, long long nvec, bool avg, int world, Lane ln) {
    constexpr int U = 4;
    for (long long v0 = ln.tid; v0 < nvec; v0 += (long long)U * ln.nth) {
        uint4 raw[U];
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const long long v = v0 + (long long)k * ln.nth;
            if (v < nvec) raw[k] = Multimem<T>::ld_reduce(mc + v * FX_VEC_BYTES);
        }
#pragma unroll
        for (int k = 0; k < U; ++k) {
            const long long v = v0 + (long long)k * ln.nth;
            if (v < nvec) multimem_st(mc + v * FX_VEC_BYTES, avg ? scale_vec<T>(raw[k], world) : raw[k]);
        }
    }
}


// ---------------------------------------------------------------------------- per-chunk flags
__device__ __forceinline__ void named_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

// Lane of a thread inside its role, and which slices its warp serves (see slice_lane).
__device__ __forceinline__ Lane role_slice_lane(int world, int role_warp, int role_warps, int* first, int* step) {
    const int groups = world < role_warps ? world : role_warps;
    const int g = role_warp % groups;
    const int members = role_warps / groups + (g < role_warps % groups ? 1 : 0);
    *first = g;
    *step = groups;
    return Lane{(role_warp / groups) * 32 + (int)(threadIdx.x & 31), members * 32};
}

enum { FX_FLAG_PACK = 0, FX_FLAG_RED = 1 };
__device__ __forceinline__ uint32_t* pipe_flag(char* arena, int which, int b, int q) {
    FxPad* pad = pad_of(arena);
    return which == FX_FLAG_PACK ? &pad->flags_pack[b][q] : &pad->flags_red[b][q];
}

__device__ __forceinline__ void signal_peers(const FxLaunch& a, int which, int q, int rank, int b, uint32_t value) {
    st_release_sys(pipe_flag(a.arena[q], which, b, rank), value);
}

// false: the peer never arrived (status word set); the caller must stop without writing outputs.
__device__ __forceinline__ bool wait_peer(const FxLaunch& a, int which, int q, int rank, int b, uint32_t value) {
    const uint32_t* mine = pipe_flag(a.arena[rank], which, b, q);
    unsigned long long t0 = 0;
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - value) < 0) {
        if ((++spins & 0x3ff) == 0) {
            const unsigned long long now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > a.timeout_ns) {
                *reinterpret_cast<volatile uint32_t*>(a.status) = (uint32_t)(-FX_ERR_TIMEOUT);
                __threadfence_system();
                return false;
            }
        }
    }
    return true;
}


}  // namespace
