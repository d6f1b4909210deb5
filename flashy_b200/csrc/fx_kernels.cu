// Collective kernels for sm_90a (H100): bucketed all-reduce (one-shot / two-shot over peer-mapped
// arenas), bucketed broadcast, local unpack and a device barrier.
//
// Replaces the per-tensor NCCL all-reduce + per-tensor divide loop of the reference
// (flashy/distrib.py:105-111, :122-127, :174-190).  The path is an elementwise reduction: it
// is bound by NVLink (W > 1 GPUs) or HBM (virtual ranks on one GPU), never by the tensor
// cores, so there is no wgmma here -- only 128-bit coalesced global/peer accesses, release /
// acquire flags at system scope, and fp32 accumulation in registers.
//
// Data flow of the two-shot kernel, for hosted rank r and CTA b (every CTA owns slice b of
// every shard, on every rank, so CTA b only ever needs to synchronise with the CTAs b of the
// other ranks):
//   pack      grads (any addresses) -> own arena, slice b of each of the W shards  [+ cast]
//   barrier   flags[b][r] <- epoch on every peer (st.release.sys), wait for all W flags
//   reduce    slice b of shard r: sum the W arenas in rank order (fp32), /W, store to own arena
//   barrier
//   gather    slice b of shard s from arena s, for all s -> output tensors      [+ cast]
// The staging region alternates between two halves on successive calls of a plan, which is
// what makes a third (end-of-kernel) barrier unnecessary.
#include "fx_device.cuh"

namespace {

// ============================================================================ kernels
__device__ __forceinline__ void finish_launch(FxPlanState* st, FxPad* pad, int b, uint32_t epoch, uint32_t calls) {
    __syncthreads();
    if (threadIdx.x == 0) {
        pad->block_epoch[b] = epoch;                            // (visible to the next launch: kernel boundary)
        if (atomicAdd(&st->finished, 1u) == gridDim.x - 1) {    // last CTA of this hosted rank
            st->finished = 0;
            *reinterpret_cast<volatile uint32_t*>(&st->calls) = calls + 1;
        }
    }
}

template <typename T, typename S, int W, int OP>
__global__ void __launch_bounds__(FX_THREADS, 1) k_two_shot(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = W > 0 ? W : a.world;
    FxPlanState* st = a.state + l;
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const unsigned long long region = a.region[calls & 1];
    char* my = a.arena[rank];
    T* stage = reinterpret_cast<T*>(my + region);
    uint32_t epoch = pad_of(my)->block_epoch[b];
    const long long slice = a.slice_elems, shard = a.shard_elems;
    const bool avg = a.op == FX_AVG;
    __shared__ MetaSmem meta_smem;
    const Meta m = load_meta(a, l, &meta_smem);

    move_all_slices<T, S, true>(m, stage, shard, slice, b, world);
    if (!block_barrier(a, rank, world, b, ++epoch)) return;

    {
        const long long lo = rank * shard + b * slice;
        reduce_vectors<T, W, OP>(a, world, region + (unsigned long long)lo * sizeof(T),
                                 slice / (FX_VEC_BYTES / (long long)sizeof(T)), avg, my, block_lane());
    }
    if (!block_barrier(a, rank, world, b, ++epoch)) return;

    {
        int first, step;
        const Lane ln = slice_lane(world, &first, &step);
        for (int j = first; j < world; j += step) {
            const int s = (rank + j) % world;                 // every group pulls from a different peer
            const long long lo = s * shard + b * slice;
            T* from = reinterpret_cast<T*>(a.arena[s] + region);
            if (a.mode == FX_MODE_FUSED) {
                move_slice<T, S, false>(m, from, lo, lo + slice, ln);
            } else if (s != rank) {
                copy_convert<T, T>(from + lo, stage + lo, slice, ln);
            }
        }
    }
    finish_launch(st, pad_of(my), b, epoch, calls);
}

template <typename T, typename S, int OP>
__global__ void __launch_bounds__(FX_THREADS, 1) k_one_shot(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = a.world;
    FxPlanState* st = a.state + l;
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const unsigned long long region = a.region[calls & 1];
    char* my = a.arena[rank];
    uint32_t epoch = pad_of(my)->block_epoch[b];
    const long long lo = b * a.slice_elems, hi = lo + a.slice_elems;
    __shared__ MetaSmem meta_smem;
    const Meta m = load_meta(a, l, &meta_smem);
    move_slice<T, S, true>(m, reinterpret_cast<T*>(my + region), lo, hi, block_lane());
    if (!block_barrier(a, rank, world, b, ++epoch)) return;
    reduce_unpack_range<T, S, OP>(a, m, world, region, lo, hi, a.op == FX_AVG);
    finish_launch(st, pad_of(my), b, epoch, calls);
}

// Bit copy from rank `src`: the source packs, everyone else pulls from the source's arena.
__global__ void __launch_bounds__(FX_THREADS, 1) k_broadcast(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = a.world;
    FxPlanState* st = a.state + l;
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const unsigned long long region = a.region[calls & 1];
    char* my = a.arena[rank];
    uint32_t epoch = pad_of(my)->block_epoch[b];
    const long long slice = a.slice_elems, shard = a.shard_elems;
    __shared__ MetaSmem meta_smem;
    const Meta m = load_meta(a, l, &meta_smem);
    if (rank == a.src) move_all_slices<uint8_t, uint8_t, true>(m, reinterpret_cast<uint8_t*>(my + region), shard, slice, b, world);
    if (!block_barrier(a, rank, world, b, ++epoch)) return;
    if (rank != a.src) {
        uint8_t* from = reinterpret_cast<uint8_t*>(a.arena[a.src] + region);
        int first, step;
        const Lane ln = slice_lane(world, &first, &step);
        for (int j = first; j < world; j += step) {
            const int s = (rank + j) % world;                 // spread the readers over the source's memory
            const long long lo = s * shard + b * slice;
            move_slice<uint8_t, uint8_t, false>(m, from, lo, lo + slice, ln);
        }
    }
    finish_launch(st, pad_of(my), b, epoch, calls);
}

// Second half of the eager path: local arena -> output tensors (flashy/distrib.py:187-190).
template <typename T, typename S>
__global__ void __launch_bounds__(FX_THREADS, 1) k_unpack(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const uint32_t calls = ld_volatile_u32(&a.state[l].calls);
    const unsigned long long region = a.region[(calls - 1) & 1];     // the region the matching BEGIN used
    T* stage = reinterpret_cast<T*>(a.arena[rank] + region);
    __shared__ MetaSmem meta_smem;
    const Meta m = load_meta(a, l, &meta_smem);
    move_all_slices<T, S, false>(m, stage, a.shard_elems, a.slice_elems, b, a.world);
}

template <typename T, typename S>
__global__ void __launch_bounds__(FX_THREADS, 1) k_nvls(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = a.world;
    FxPlanState* st = a.state + l;
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const unsigned long long region = a.region[calls & 1];
    char* my = a.arena[rank];
    T* stage = reinterpret_cast<T*>(my + region);
    uint32_t epoch = pad_of(my)->block_epoch[b];
    const long long slice = a.slice_elems, shard = a.shard_elems;
    const bool avg = a.op == FX_AVG;
    __shared__ MetaSmem meta_smem;
    const Meta m = load_meta(a, l, &meta_smem);

    move_all_slices<T, S, true>(m, stage, shard, slice, b, world);
    if (!block_barrier(a, rank, world, b, ++epoch)) return;
    {
        const long long lo = rank * shard + b * slice;
        nvls_vectors<T>(a.mc_arena + region + (unsigned long long)lo * sizeof(T),
                        slice / (FX_VEC_BYTES / (long long)sizeof(T)), avg, world, block_lane());
    }
    if (!block_barrier(a, rank, world, b, ++epoch)) return;
    if (a.mode == FX_MODE_FUSED) move_all_slices<T, S, false>(m, stage, shard, slice, b, world);
    finish_launch(st, pad_of(my), b, epoch, calls);
}

// ---------------------------------------------------------------------------- pipelined all-reduce
// The three phases of a sharded all-reduce (pack, reduce, gather/unpack) as three concurrent
// warp roles of one CTA, decoupled by per-chunk flags instead of CTA-wide barriers:
//   pack   warps  0-3 : tensors -> own arena, chunk c of slice b of every shard; then
//                       flagsP[b][me] <- base+c+1 on every peer                        (never waits)
//   reduce warps 4-11 : wait flagsP[b][*] >= base+c+1; reduce chunk c of slice b of shard `me`
//                       (multimem through the switch, or pull from the W arenas);
//                       flagsR[b][me] <- base+c+1 on every peer
//   gather warps 12-15: wait flagsR[b][*] >= base+c+1; chunk c of slice b of every shard ->
//                       output tensors (local arena after NVLS, peer arenas on the P2P path)
// so the NVLink phase of chunk c overlaps the HBM passes of chunks c+1 (pack) and c-1 (unpack),
// and a cross-GPU flag round trip is paid once at each end instead of once per phase.
#define FX_PACK_WARPS 4
#define FX_RED_WARPS 8
#define FX_UNP_WARPS 4

template <typename T, typename S, bool NVLS, int W, int OP>
__global__ void __launch_bounds__(FX_THREADS, 1) k_pipe(const FxLaunch a) {
    const int l = blockIdx.y, b = blockIdx.x;
    const int rank = a.rank0 + l;
    const int world = W > 0 ? W : a.world;
    FxPlanState* st = a.state + l;
    const uint32_t calls = ld_volatile_u32(&st->calls);
    const unsigned long long region = a.region[calls & 1];
    char* my = a.arena[rank];
    T* stage = reinterpret_cast<T*>(my + region);
    const uint32_t base = pad_of(my)->pipe_epoch[b];
    const long long slice = a.slice_elems, shard = a.shard_elems, csz = a.chunk_elems;
    const int chunks = a.chunks;
    const bool avg = a.op == FX_AVG;
    constexpr long long VEC = FX_VEC_BYTES / (long long)sizeof(T);
    __shared__ MetaSmem meta_smem;
    __shared__ int s_abort;                 // a peer never arrived: every role stops before its next store
    if (threadIdx.x == 0) s_abort = 0;
    const Meta m = load_meta(a, l, &meta_smem);

    const int warp = threadIdx.x >> 5;
    if (warp < FX_PACK_WARPS) {
        // ------------------------------------------------ pack role
        const int rt = threadIdx.x;                                   // thread index inside the role
        int first, step;
        const Lane ln = role_slice_lane(world, warp, FX_PACK_WARPS, &first, &step);
        for (int c = 0; c < chunks; ++c) {
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            for (int s = first; s < world; s += step) {
                const long long lo = s * shard + b * slice;
                move_slice<T, S, true>(m, stage, lo + c0, lo + c1, ln);
            }
            named_sync(1, FX_PACK_WARPS * 32);
            if (rt < world) signal_peers(a, FX_FLAG_PACK, rt, rank, b, base + c + 1);
        }
    } else if (warp < FX_PACK_WARPS + FX_RED_WARPS) {
        // ------------------------------------------------ reduce role
        const int rt = threadIdx.x - FX_PACK_WARPS * 32;
        const Lane ln{rt, FX_RED_WARPS * 32};
        for (int c = 0; c < chunks; ++c) {
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            if (rt < world && !wait_peer(a, FX_FLAG_PACK, rt, rank, b, base + c + 1)) *reinterpret_cast<volatile int*>(&s_abort) = 1;
            named_sync(2, FX_RED_WARPS * 32);
            if (*reinterpret_cast<volatile int*>(&s_abort)) break;
            const long long lo = rank * shard + b * slice + c0;
            const unsigned long long byte_off = region + (unsigned long long)lo * sizeof(T);
            if (NVLS) nvls_vectors<T>(a.mc_arena + byte_off, (c1 - c0) / VEC, avg, world, ln);
            else reduce_vectors<T, W, OP>(a, world, byte_off, (c1 - c0) / VEC, avg, my, ln);
            named_sync(2, FX_RED_WARPS * 32);
            if (rt < world) signal_peers(a, FX_FLAG_RED, rt, rank, b, base + c + 1);
        }
    } else {
        // ------------------------------------------------ gather / unpack role
        const int rw = warp - FX_PACK_WARPS - FX_RED_WARPS;
        const int rt = threadIdx.x - (FX_PACK_WARPS + FX_RED_WARPS) * 32;
        int first, step;
        const Lane ln = role_slice_lane(world, rw, FX_UNP_WARPS, &first, &step);
        for (int c = 0; c < chunks; ++c) {
            const long long c0 = c * csz, c1 = (c0 + csz < slice) ? c0 + csz : slice;
            if (rt < world && !wait_peer(a, FX_FLAG_RED, rt, rank, b, base + c + 1)) *reinterpret_cast<volatile int*>(&s_abort) = 1;
            named_sync(3, FX_UNP_WARPS * 32);
            if (*reinterpret_cast<volatile int*>(&s_abort)) break;
            for (int j = first; j < world; j += step) {
                const int s = (rank + j) % world;
                const long long lo = s * shard + b * slice;
                T* from = NVLS ? stage : reinterpret_cast<T*>(a.arena[s] + region);
                if (a.mode == FX_MODE_FUSED) move_slice<T, S, false>(m, from, lo + c0, lo + c1, ln);
                else if (!NVLS && s != rank) copy_convert<T, T>(from + lo + c0, stage + lo + c0, c1 - c0, ln);
            }
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        pad_of(my)->pipe_epoch[b] = base + chunks;
        if (atomicAdd(&st->finished, 1u) == gridDim.x - 1) {
            st->finished = 0;
            *reinterpret_cast<volatile uint32_t*>(&st->calls) = calls + 1;
        }
    }
}

__global__ void __launch_bounds__(FX_THREADS, 1) k_barrier(const FxLaunch a) {
    const int rank = a.rank0 + blockIdx.y;
    FxPad* pad = pad_of(a.arena[rank]);
    uint32_t epoch = pad->block_epoch[0];
    if (!block_barrier(a, rank, a.world, 0, ++epoch)) return;
    if (threadIdx.x == 0) pad->block_epoch[0] = epoch;
}

// ============================================================================ dispatch
template <typename K>
int launch(K kernel, const fx_plan* plan, int grid_x, const FxLaunch& args, cudaStream_t stream) {
    const fx_comm* c = plan ? plan->comm : nullptr;
    const int n_local = args.n_local;
    dim3 grid(grid_x, n_local), block(FX_THREADS);
    void* params[] = {const_cast<FxLaunch*>(&args)};
    cudaError_t e;
    if (n_local > 1) {
        // virtual ranks spin on each other's flags: all their CTAs must be co-resident
        e = cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kernel), grid, block, params, 0, stream);
    } else {
        e = cudaLaunchKernel(reinterpret_cast<const void*>(kernel), grid, block, params, 0, stream);
    }
    (void)c;
    if (e != cudaSuccess) return fx_fail(FX_ERR_CUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    return FX_OK;
}

template <typename T, typename S, int OP>
int launch_allreduce_w(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    if (plan->algo == FX_ALGO_ONE_SHOT) return launch(k_one_shot<T, S, OP>, plan, plan->grid_x, a, s);
    // (an NVLS plan asked for MAX / MIN / PROD lands here: same sharded layout, peer-to-peer kernel)
    if (OP == FX_SUM) {
        switch (a.world) {
            case 2: return launch(k_two_shot<T, S, 2, OP>, plan, plan->grid_x, a, s);
            case 4: return launch(k_two_shot<T, S, 4, OP>, plan, plan->grid_x, a, s);
            case 8: return launch(k_two_shot<T, S, 8, OP>, plan, plan->grid_x, a, s);
            default: break;
        }
    }
    return launch(k_two_shot<T, S, 0, OP>, plan, plan->grid_x, a, s);
}

template <typename T, typename S>
int launch_allreduce_op(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    switch (a.op) {
        case FX_SUM: case FX_AVG: return launch_allreduce_w<T, S, FX_SUM>(plan, a, s);
        case FX_MAX: return launch_allreduce_w<T, S, FX_MAX>(plan, a, s);
        case FX_MIN: return launch_allreduce_w<T, S, FX_MIN>(plan, a, s);
        case FX_PROD: return launch_allreduce_w<T, S, FX_PROD>(plan, a, s);
    }
    return fx_fail(FX_ERR_INVALID, "unknown reduce op %d", a.op);
}

}  // namespace

bool fx_kernel_supported(int dtype, int wire, int op, bool broadcast) {
    if (broadcast) return true;                       // bytes
    if (dtype == FX_U8 || wire == FX_U8) return false;
    if (dtype != wire && !(dtype == FX_F32 && wire == FX_BF16)) return false;
    if (op == FX_AVG && (dtype == FX_I32 || dtype == FX_I64)) return false;
    return op >= FX_SUM && op <= FX_PROD;
}

template <typename T, typename S>
int launch_pipe_p2p(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    switch (a.world) {
        case 2: return launch(k_pipe<T, S, false, 2, FX_SUM>, plan, plan->grid_x, a, s);
        case 4: return launch(k_pipe<T, S, false, 4, FX_SUM>, plan, plan->grid_x, a, s);
        case 8: return launch(k_pipe<T, S, false, 8, FX_SUM>, plan, plan->grid_x, a, s);
    }
    return launch(k_pipe<T, S, false, 0, FX_SUM>, plan, plan->grid_x, a, s);
}

int fx_launch_allreduce(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    const bool sum = a.op == FX_SUM || a.op == FX_AVG;
    if (a.chunks > 0 && sum && plan->algo != FX_ALGO_ONE_SHOT) {          // pipelined kernels
        const bool nvls = plan->algo == FX_ALGO_NVLS;
        if (nvls && !a.mc_arena) return fx_fail(FX_ERR_STATE, "NVLS plan without a multicast mapping");
        if (plan->dtype == FX_F32 && plan->wire == FX_BF16)
            return nvls ? launch(k_pipe<__nv_bfloat16, float, true, 0, FX_SUM>, plan, plan->grid_x, a, s)
                        : launch_pipe_p2p<__nv_bfloat16, float>(plan, a, s);
        switch (plan->wire) {
            case FX_F32: return nvls ? launch(k_pipe<float, float, true, 0, FX_SUM>, plan, plan->grid_x, a, s)
                                     : launch_pipe_p2p<float, float>(plan, a, s);
            case FX_BF16: return nvls ? launch(k_pipe<__nv_bfloat16, __nv_bfloat16, true, 0, FX_SUM>, plan, plan->grid_x, a, s)
                                      : launch_pipe_p2p<__nv_bfloat16, __nv_bfloat16>(plan, a, s);
            case FX_F16: return nvls ? launch(k_pipe<__half, __half, true, 0, FX_SUM>, plan, plan->grid_x, a, s)
                                     : launch_pipe_p2p<__half, __half>(plan, a, s);
            default: break;                                               // fp64 / ints: classic kernels
        }
    }
    if (plan->algo == FX_ALGO_NVLS && (a.op == FX_SUM || a.op == FX_AVG)) {
        if (!a.mc_arena) return fx_fail(FX_ERR_STATE, "NVLS plan without a multicast mapping");
        if (plan->dtype == FX_F32 && plan->wire == FX_BF16) return launch(k_nvls<__nv_bfloat16, float>, plan, plan->grid_x, a, s);
        switch (plan->wire) {
            case FX_F32: return launch(k_nvls<float, float>, plan, plan->grid_x, a, s);
            case FX_BF16: return launch(k_nvls<__nv_bfloat16, __nv_bfloat16>, plan, plan->grid_x, a, s);
            case FX_F16: return launch(k_nvls<__half, __half>, plan, plan->grid_x, a, s);
        }
        return fx_fail(FX_ERR_UNSUPPORTED, "NVLS supports fp32 / bf16 / fp16 sums only");
    }
    if (plan->dtype == FX_F32 && plan->wire == FX_BF16) return launch_allreduce_op<__nv_bfloat16, float>(plan, a, s);
    switch (plan->wire) {
        case FX_F32: return launch_allreduce_op<float, float>(plan, a, s);
        case FX_BF16: return launch_allreduce_op<__nv_bfloat16, __nv_bfloat16>(plan, a, s);
        case FX_F16: return launch_allreduce_op<__half, __half>(plan, a, s);
        case FX_F64: return launch_allreduce_op<double, double>(plan, a, s);
        case FX_I32: return launch_allreduce_op<int32_t, int32_t>(plan, a, s);
        case FX_I64: return launch_allreduce_op<int64_t, int64_t>(plan, a, s);
    }
    return fx_fail(FX_ERR_INVALID, "all-reduce: unsupported dtype %d", plan->wire);
}

int fx_launch_broadcast(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    return launch(k_broadcast, plan, plan->grid_x, a, s);
}

int fx_launch_unpack(fx_plan* plan, const FxLaunch& a, cudaStream_t s) {
    dim3 grid(plan->grid_x, a.n_local), block(FX_THREADS);
    if (plan->dtype == FX_F32 && plan->wire == FX_BF16) k_unpack<__nv_bfloat16, float><<<grid, block, 0, s>>>(a);
    else switch (plan->wire) {
        case FX_F32: k_unpack<float, float><<<grid, block, 0, s>>>(a); break;
        case FX_BF16: k_unpack<__nv_bfloat16, __nv_bfloat16><<<grid, block, 0, s>>>(a); break;
        case FX_F16: k_unpack<__half, __half><<<grid, block, 0, s>>>(a); break;
        case FX_F64: k_unpack<double, double><<<grid, block, 0, s>>>(a); break;
        case FX_I32: k_unpack<int32_t, int32_t><<<grid, block, 0, s>>>(a); break;
        case FX_I64: k_unpack<int64_t, int64_t><<<grid, block, 0, s>>>(a); break;
        default: return fx_fail(FX_ERR_INVALID, "unpack: unsupported dtype %d", plan->wire);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fx_fail(FX_ERR_CUDA, "unpack launch failed: %s", cudaGetErrorString(e));
    return FX_OK;
}

int fx_launch_barrier(fx_comm* comm, const FxLaunch& a, cudaStream_t s) {
    (void)comm;
    return launch(k_barrier, nullptr, 1, a, s);
}

int fx_max_coresident_blocks(int device, int n_local, int* sm_count) {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) return 0;
    if (sm_count) *sm_count = sms;
    // Every collective kernel is built for ONE CTA per SM (__launch_bounds__(.., 1); k_fuse takes the whole
    // shared memory of its SM), and the hosted ranks' CTAs must all be resident at once.
    int blocks = sms / (n_local > 0 ? n_local : 1);
    if (blocks > FX_MAX_BLOCKS) blocks = FX_MAX_BLOCKS;
    return blocks < 1 ? 1 : blocks;
}
