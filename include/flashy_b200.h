/*
 * flashy_b200.h -- C ABI of libflashy_b200.so, the native layer under flashy_b200/distrib.py.
 *
 * The reference (facebookresearch/flashy) has no FFI: its hot path is the Python module
 * flashy/distrib.py calling torch.distributed (c10d -> NCCL/gloo).  Each entry point below
 * names the reference call site(s) it replaces (paths relative to the reference checkout).
 *
 * Conventions
 *   - plain C, no torch / ATen types; device pointers are raw addresses in the caller's
 *     CUDA primary context; streams are cudaStream_t passed as void*.
 *   - every function returns FX_OK (0) or a negative fx_status; fx_last_error() gives the
 *     thread-local message for the last failure on the calling thread.
 *   - one fx_comm per process.  It hosts `n_local` consecutive ranks of the world on ONE
 *     device: n_local == 1 is the production layout (one process per GPU, the Dora/torchrun
 *     layout of the reference); n_local > 1 hosts several *virtual* ranks on the same GPU so
 *     that the multi-rank kernels can be run, profiled (ncu is single-process) and
 *     parity-tested on a one-GPU box.  The kernels are the same code in both layouts: a
 *     rank only ever sees a table of W arena base pointers, local or peer-mapped.
 *   - collectives on one comm must be issued in the same order by every rank (NCCL's rule,
 *     which the reference obeys: flashy/distrib.py:105 iterates tensors in a fixed order),
 *     and be stream-ordered on each rank (launch them on one stream, or chain with events).
 *   - thread safety: any thread may call; calls on one comm are serialised by an internal
 *     mutex (the eager-sync hooks run on the autograd engine thread, flashy/distrib.py:171-179).
 */
#ifndef FLASHY_B200_H
#define FLASHY_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FX_ABI_VERSION 2
#define FX_MAX_WORLD 16          /* single NVSwitch domain; >8 only reachable with virtual ranks */
#define FX_MAX_BLOCKS 512        /* upper bound of gridDim.x for any collective kernel */

typedef enum fx_status {
    FX_OK = 0,
    FX_ERR_INVALID = -1,         /* bad argument */
    FX_ERR_CUDA = -2,            /* a CUDA runtime/driver call failed (message has the detail) */
    FX_ERR_UNSUPPORTED = -3,     /* feature not available on this system (e.g. multicast) */
    FX_ERR_TOO_BIG = -4,         /* bucket does not fit the arena: split it */
    FX_ERR_MISMATCH = -5,        /* ranks disagree (count / layout signature) */
    FX_ERR_TIMEOUT = -6,         /* a peer did not arrive in time (host check or device flag wait) */
    FX_ERR_SYS = -7,             /* OS error (shm, socket) */
    FX_ERR_STATE = -8            /* call sequence error (e.g. not connected yet) */
} fx_status;

typedef enum fx_dtype {
    FX_F32 = 0, FX_BF16 = 1, FX_F16 = 2, FX_F64 = 3,
    FX_I32 = 4, FX_I64 = 5,
    FX_U8 = 6                    /* opaque bytes: broadcast only */
} fx_dtype;

typedef enum fx_op {
    FX_SUM = 0,                  /* torch.distributed.ReduceOp.SUM */
    FX_AVG = 1,                  /* SUM then true division by world (flashy/distrib.py:105-111) */
    FX_MAX = 2, FX_MIN = 3, FX_PROD = 4
} fx_op;

typedef enum fx_algo {
    FX_ALGO_AUTO = 0,
    FX_ALGO_ONE_SHOT = 1,        /* pack -> barrier -> every rank reduces all W copies */
    FX_ALGO_TWO_SHOT = 2,        /* pack -> barrier -> reduce-scatter -> barrier -> all-gather+unpack */
    FX_ALGO_NVLS = 3             /* multimem.ld_reduce / multimem.st through the NVSwitch (needs multicast) */
} fx_algo;

/* Which kernel a SUM / AVG all-reduce of a plan launches (fx_plan_info.kernel). */
typedef enum fx_kernel_id {
    FX_KERNEL_ONE_SHOT = 1,      /* k_one_shot  */
    FX_KERNEL_TWO_SHOT = 2,      /* k_two_shot  (three barrier-separated phases, register copies) */
    FX_KERNEL_NVLS = 3,          /* k_nvls      (same, multimem reduce phase) */
    FX_KERNEL_PIPE_P2P = 4,      /* k_pipe<.., NVLS=false>  (warp roles, register copies) */
    FX_KERNEL_PIPE_NVLS = 5,     /* k_pipe<.., NVLS=true> */
    FX_KERNEL_FUSE_P2P = 6,      /* k_fuse<.., NVLS=false>  (five decoupled roles, cp.async.bulk staging) */
    FX_KERNEL_FUSE_NVLS = 7      /* k_fuse<.., NVLS=true> */
} fx_kernel_id;

/* fx_comm_create flags */
#define FX_COMM_MEM_AUTO   0u    /* VMM (cuMemCreate, fd export) if the driver allows, else cudaMalloc + cudaIpc */
#define FX_COMM_MEM_VMM    1u
#define FX_COMM_MEM_IPC    2u
#define FX_COMM_MEM_MASK   3u
#define FX_COMM_HOST_ONLY  4u    /* no CUDA at all: rendezvous/count-check fabric only (CPU tests, planning) */

typedef struct fx_comm fx_comm;
typedef struct fx_plan fx_plan;

typedef struct fx_comm_info {
    int abi_version, world, rank0, n_local, device;
    int mem_kind;                /* FX_COMM_MEM_VMM / FX_COMM_MEM_IPC; 0 when host-only */
    int connected, multicast;    /* booleans */
    int sm_count, max_blocks;    /* device SM count; largest gridDim.x a launch may use */
    uint64_t arena_bytes;        /* staging bytes per rank (excluding the signal pad) */
    uint64_t arena_used;         /* bytes handed out to live plans */
    uint64_t launches;           /* kernels launched through this comm so far */
} fx_comm_info;

typedef struct fx_plan_info {
    int n_tensors, dtype, wire_dtype, world;
    int algo;                    /* algorithm AUTO resolves to for this bucket */
    int grid_x, block;           /* launch geometry (gridDim.y is n_local) */
    uint64_t total_elems;        /* sum of numel */
    uint64_t padded_elems;       /* bucket length incl. per-tensor 16-byte alignment and shard padding */
    uint64_t shard_elems;        /* padded_elems / world */
    uint64_t wire_bytes;         /* padded_elems * sizeof(wire dtype) = one staging copy */
    uint64_t region_offset[2];   /* the two (double-buffered) staging regions inside each arena */
    uint64_t signature;          /* hash of (n, dtype, numels): what ranks must agree on */
    int kernel;                  /* fx_kernel_id a SUM / AVG fx_allreduce of this plan launches */
    int chunks;                  /* chunks per slice of that kernel (0: not chunked) */
    uint64_t chunk_bytes;        /* bytes of one chunk of one shard's slice */
} fx_plan_info;

/* ------------------------------------------------------------------ errors / build info */

const char* fx_last_error(void);
int fx_abi_version(void);
/* 1 when a CUDA driver and at least one device are usable from this process, else 0. */
int fx_cuda_available(void);

/* ------------------------------------------------------------------ communicator
 * Replaces: the ProcessGroupNCCL communicator that dora.distrib.init -> torch.distributed
 * .init_process_group creates (flashy/distrib.py:21).  torch.distributed remains the
 * bootstrap channel only: the caller moves the export blobs between processes with it.
 */
int fx_comm_create(int world, int rank0, int n_local, int device, size_t arena_bytes,
                   unsigned flags, fx_comm** out);
/* Serialised description of this process's arenas, rendezvous socket and (for the process
 * hosting rank 0) the shared-memory check fabric.  Fixed size for a given build: query it
 * with blob == NULL. */
int fx_comm_export(fx_comm* comm, void* blob, size_t cap, size_t* len);
/* `blobs` = the export blobs of every process, in rank order (own blob included), each
 * `blob_len` bytes.  Maps every peer arena.  With n_local == world pass (NULL, 0, 0). */
int fx_comm_connect(fx_comm* comm, const void* blobs, size_t blob_len, int n_procs);
/* Bind all arenas to one NVSwitch multicast object (NVLS).  FX_ERR_UNSUPPORTED if the
 * device, driver or allocation kind cannot do it; the P2P algorithms keep working. */
int fx_comm_enable_multicast(fx_comm* comm, const void* blobs, size_t blob_len, int n_procs);
int fx_comm_get_info(fx_comm* comm, fx_comm_info* info);
/* Cap gridDim.x of the plans created AFTER this call (0 = back to the communicator's default, one CTA per
 * SM).  Every rank must make the same calls in the same order (the grid is part of the bucket layout).
 * Used for the buckets that are launched while backward is still running: a small grid leaves the other
 * SMs -- each CTA of the fused kernel takes a whole SM's shared memory -- to the compute kernels.
 * No reference counterpart (NCCL's channel count plays this role in the reference). */
int fx_comm_set_plan_blocks(fx_comm* comm, int max_blocks);
/* Diagnostics / benchmarks: the arena base of every rank as mapped in this process
 * (`arenas[world]`, staging starts `pad_bytes` in), and the NVSwitch multicast alias of the
 * arenas (`mc_base` NULL / `mc_bytes` 0 without NVLS).  No reference counterpart: this is
 * the window the micro-benchmarks under benchmarks/ use to time raw NVLink / multimem rates. */
int fx_comm_get_pointers(fx_comm* comm, void** arenas, void** mc_base, uint64_t* mc_bytes,
                         uint64_t* pad_bytes);
/* Diagnostics: with FLASHY_B200_TRACE=1 in the environment at fx_comm_create, CTA 0 of every fused
 * all-reduce launch (k_fuse) stamps %globaltimer at the hand-offs of its warp roles.  This copies the
 * stamps of the most recent launch out (`words` = 0 when tracing is off) and clears them;
 * benchmarks/trace_fuse.py turns them into a per-chunk timeline.  No reference counterpart. */
int fx_comm_trace_read(fx_comm* comm, uint64_t* out, size_t cap_words, size_t* words);
/* Asynchronous device-side error state (flag-wait timeout): FX_OK or the sticky error. */
int fx_comm_poll(fx_comm* comm);
/* Poison the communicator for every rank of the world: all blocked and future host-side
 * waits (fx_host_exchange / barrier / broadcast) fail with FX_ERR_STATE instead of waiting for
 * a rank that died.  The communicator cannot be used afterwards (like ncclCommAbort). */
int fx_comm_abort(fx_comm* comm);
void fx_comm_destroy(fx_comm* comm);

/* ------------------------------------------------------------------ host-side count check
 * Replaces: _check_number_of_params (flashy/distrib.py:78-89) -- an int64 all-reduce plus a
 * host-blocking .item(), twice per sync_model.  Here: every rank publishes (count,
 * signature) in a shared-memory slot and reads the others'; exact integers, no GPU work, no
 * stream sync.  `sum_out` receives the sum of counts over ranks (the reference's test is
 * sum != count * world); `sig_equal` is 0 if any rank published a different signature.
 * Every hosted rank (`local`) must call it once per collective, in the same order.
 * timeout_s <= 0 selects the default (FLASHY_B200_HOST_TIMEOUT, 600 s).
 */
int fx_host_exchange(fx_comm* comm, int local, int64_t count, uint64_t signature,
                     int64_t* sum_out, int* sig_equal, double timeout_s);
/* Host barrier over the same fabric.  Replaces torch.distributed.barrier (flashy/distrib.py:276). */
int fx_host_barrier(fx_comm* comm, int local, double timeout_s);
/* Copy `nbytes` of host memory from rank `src` to every rank through the shared-memory fabric
 * (chunked).  Every hosted rank calls it with the same `nbytes`.  Replaces the two
 * torch.distributed.broadcast calls of broadcast_object (flashy/distrib.py:258,265). */
int fx_host_broadcast(fx_comm* comm, int local, int src, void* buf, size_t nbytes, double timeout_s);

/* ------------------------------------------------------------------ plans (buckets)
 * A plan is the bucket layout for one ordered tensor list: tensor i of `numels[i]` elements
 * lives at a 16-byte aligned offset of one flat wire buffer, which is cut in `world` shards.
 * Replaces the per-tensor loop of average_tensors / broadcast_tensors
 * (flashy/distrib.py:104-111, 122-127): N collectives + N divides become one launch.
 * comm == NULL gives a dry plan (layout only; used by the CPU tests).
 */
int fx_plan_create(fx_comm* comm, int world, const int64_t* numels, int n, int dtype,
                   int wire_dtype, int algo, fx_plan** out);
int fx_plan_get_info(fx_plan* plan, fx_plan_info* info);
/* Element offset of each tensor in the bucket (n values). */
int fx_plan_offsets(fx_plan* plan, int64_t* offsets);
void fx_plan_destroy(fx_plan* plan);

/* One bucketed all-reduce for every hosted rank.
 *   in_ptrs / out_ptrs: n_local * n device pointers, row `l` = hosted rank `l`'s tensors
 *   (out == in for the in-place average of flashy/distrib.py:111; out != in gives
 *   torch.div(grad, W, out=param.grad) of the eager path, flashy/distrib.py:190).
 * Replaces: flashy/distrib.py:105-111 (average_tensors), :174-190 (eager hooks), :47
 * (all_reduce), :60 (average_metrics' reduction).
 */
int fx_allreduce(fx_plan* plan, int op, const void* const* in_ptrs, void* const* out_ptrs,
                 void* stream);
/* fx_allreduce for hosted (virtual) ranks, called once per bucket by EVERY hosted rank `local` of
 * the process, each from its own thread, with its own row of plan->n pointers and its own stream.
 * The ranks meet inside the library, so a caller that drops its interpreter lock for the call
 * (ctypes does) serialises nothing on the host:
 *   - the rank publishes its rows and records an event on `rank_stream`;
 *   - check != 0: the count check of fx_host_exchange (`count`, `signature`) across every process
 *     of the world.  If the counts' sum is not count * world or a signature differs, every rank
 *     gets FX_ERR_MISMATCH with `sum_out` / `sig_equal` filled in, and nothing is launched;
 *   - the last hosted rank to arrive launches exactly what fx_allreduce launches, on the ranks'
 *     stream if they all share one, else on `launch_stream` ordered after every rank's stream;
 *     every rank's stream then waits for the launch, and every rank returns the launcher's code.
 * The waits honour FLASHY_B200_HOST_TIMEOUT and fx_comm_abort.  Stream capture is refused with
 * FX_ERR_STATE (capture with fx_allreduce).  Replaces, for the one-GPU layout of several ranks,
 * the same reference call sites as fx_allreduce plus the count check of flashy/distrib.py:78-89. */
int fx_allreduce_hosted(fx_plan* plan, int local, int op, int check, int64_t count, uint64_t signature,
                        const void* const* in_row, void* const* out_row, void* rank_stream,
                        void* launch_stream, int64_t* sum_out, int* sig_equal);
/* Bit copy of rank `src`'s tensors into everybody's.  Replaces flashy/distrib.py:122-127. */
int fx_broadcast(fx_plan* plan, int src, void* const* ptrs, void* stream);
/* Split form used by the eager path: stage A packs and reduces the bucket into the arena as
 * soon as its gradients exist (flashy/distrib.py:174); stage B, at context exit, writes the
 * finished values into param.grad (flashy/distrib.py:187-190). */
int fx_allreduce_begin(fx_plan* plan, int op, const void* const* in_ptrs, void* stream);
int fx_allreduce_finish(fx_plan* plan, void* const* out_ptrs, void* stream);

/* Device-side barrier across all ranks on `stream` (one tiny kernel).  Replaces
 * torch.distributed.barrier for CUDA runs (flashy/distrib.py:276). */
int fx_barrier(fx_comm* comm, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* FLASHY_B200_H */
