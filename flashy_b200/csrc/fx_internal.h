// Internal declarations shared by the host runtime (fx_host.cu) and the kernels (fx_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <mutex>
#include <atomic>
#include <thread>

#include "../../include/flashy_b200.h"

#define FX_THREADS 512                 // threads per CTA of every collective kernel
#define FX_PAD_BYTES (128u << 10)      // signal pad at the head of each arena
#define FX_VEC_BYTES 16                // one 128-bit access
#define FX_SLICE_ALIGN 128             // slices start on 128-byte lines (no line shared by two CTAs)

// ---------------------------------------------------------------- arena signal pad (device)
// flags[b][q]  : written by rank q's CTA b (over NVLink or locally), polled by the owner's CTA b.
// block_epoch  : owner-private; last barrier value CTA b used (monotonic, wraps mod 2^32).
struct FxPad {
    uint32_t flags[FX_MAX_BLOCKS][FX_MAX_WORLD];        // CTA-wide barriers of the classic kernels
    uint32_t flags_pack[FX_MAX_BLOCKS][FX_MAX_WORLD];   // pipelined kernel: "chunk c is packed on rank q"
    uint32_t flags_red[FX_MAX_BLOCKS][FX_MAX_WORLD];    // pipelined kernel: "chunk c of shard q is reduced"
    uint32_t block_epoch[FX_MAX_BLOCKS];
    uint32_t pipe_epoch[FX_MAX_BLOCKS];                 // owner-private base value of the two arrays above
};
static_assert(sizeof(FxPad) <= FX_PAD_BYTES, "signal pad too small");

// Per (plan, hosted rank) device state: call counter (its parity selects the staging region)
// and the count of CTAs that finished the current launch.
struct FxPlanState {
    uint32_t calls;
    uint32_t finished;
};

enum FxMode : int {
    FX_MODE_FUSED = 0,     // all-gather phase writes straight into the output tensors
    FX_MODE_BEGIN = 1,     // all-gather phase lands in the local arena; fx_allreduce_finish unpacks
};

// Kernel argument block (passed by value; well under the 4 KB parameter limit).
struct FxLaunch {
    char* arena[FX_MAX_WORLD];        // arena base of every rank as mapped in THIS process
    char* mc_arena;                   // multicast (NVLS) alias of the arenas, or nullptr
    uint32_t* status;                 // host-mapped sticky error word
    unsigned long long timeout_ns;    // flag-wait bound
    int world, rank0, n_local;
    int n;                            // tensors in the bucket
    const long long* off;             // [n+1] element offset of each tensor; off[n] = end of data
    const void* const* in_ptrs;       // [n_local * n]
    void* const* out_ptrs;            // [n_local * n]
    FxPlanState* state;               // [n_local]
    unsigned long long region[2];     // byte offsets of the two staging regions inside an arena
    long long slice_elems;            // elements per (shard, CTA) slice
    long long shard_elems;            // slice_elems * gridDim.x
    int op;                           // fx_op
    int src;                          // broadcast source rank
    int mode;                         // FxMode
    int chunks;                       // > 0: pipelined kernel, chunks per slice
    long long chunk_elems;            // elements per chunk (multiple of 128 bytes)
    unsigned long long* trace;        // FLASHY_B200_TRACE=1: globaltimer stamps of CTA 0 (fx_fuse.cu), else nullptr
};

// ---------------------------------------------------------------- host objects
struct FxDriver;   // resolved driver entry points (fx_host.cu)

struct FxArena {
    char* base = nullptr;             // mapped address in this process
    size_t bytes = 0;                 // pad + staging, rounded to allocation granularity
    bool owned = false;               // allocated by this process
    unsigned long long vmm_handle = 0;  // CUmemGenericAllocationHandle
    int vmm_fd = -1;                  // exported POSIX fd (owner side)
    bool ipc_opened = false;
};

struct FxShmSlot {
    std::atomic<long long> seq;
    long long count;
    unsigned long long sig;
    long long pad[5];
};
#define FX_BCAST_CHUNK (256u << 10)
struct FxShm {                        // lives in POSIX shared memory (or the heap when single-process)
    FxShmSlot slot[2][FX_MAX_WORLD];
    std::atomic<int> attached;
    std::atomic<int> aborted;         // set by fx_comm_abort on any rank: every host wait fails
    // host broadcast channel: the source publishes chunk `bc_seq`, the W-1 readers acknowledge
    std::atomic<long long> bc_seq;
    std::atomic<int> bc_acks;
    long long bc_len;
    char bc_data[FX_BCAST_CHUNK];
};

struct fx_comm {
    int world = 0, rank0 = 0, n_local = 0, device = -1;
    unsigned flags = 0;
    int mem_kind = 0;
    bool host_only = false, connected = false, multicast = false;
    int sm_count = 0, max_blocks = 0;
    int plan_blocks = 0;              // fx_comm_set_plan_blocks: grid cap of the plans created next (0 = max_blocks)
    size_t arena_bytes = 0;           // staging bytes per rank
    size_t arena_total = 0;           // pad + staging (allocation size)
    size_t arena_used = 0;            // bump pointer inside the staging area
    size_t recycle_mark = 0;          // staging below this offset has been used by destroyed plans
    std::vector<std::pair<size_t, size_t>> free_regions;   // (offset, bytes) returned by destroyed plans
    FxArena arena[FX_MAX_WORLD];
    char* mc_base = nullptr;          // multicast mapping
    unsigned long long mc_handle = 0;
    int mc_fd = -1;
    size_t mc_bytes = 0;
    uint32_t* status_host = nullptr;  // pinned, mapped
    uint32_t* status_dev = nullptr;
    unsigned long long timeout_ns = 0;
    unsigned long long launches = 0;
    // host rendezvous fabric
    FxShm* shm = nullptr;
    bool shm_owner = false, shm_is_heap = false;
    char shm_name[64] = {0};
    long long host_seq[FX_MAX_WORLD] = {0};     // per hosted rank
    long long bcast_seq[FX_MAX_WORLD] = {0};    // per hosted rank: chunks seen on the broadcast channel
    // fd server (VMM export)
    char sock_name[64] = {0};
    int listen_fd = -1;
    std::thread server;
    std::atomic<bool> stop{false};
    std::mutex mu;
    void* last_stream = nullptr;      // stream of the most recent collective launch (see order_after_previous)
    bool have_last = false;
    cudaEvent_t order_event = nullptr;
    unsigned long long* trace_dev = nullptr;    // FLASHY_B200_TRACE=1: per-role time stamps of the fused kernel
    // fx_allreduce_hosted: the hosted ranks of this process meet here, and the last to arrive launches
    cudaEvent_t rank_event[FX_MAX_WORLD] = {nullptr};   // per hosted rank: its stream's state at arrival
    cudaEvent_t hosted_done = nullptr;                  // the launch stream after the launch
    void* hosted_stream[FX_MAX_WORLD] = {nullptr};      // per hosted rank: its stream of the current collective
    std::atomic<int> hosted_arrived{0};                 // hosted ranks arrived at the current collective
    std::atomic<long long> hosted_epoch{0};             // collectives launched (published by the launcher)
    int hosted_rc = FX_OK;                              // the launcher's return code, valid once the epoch moved
    bool hosted_join = false;                           // the ranks must wait on hosted_done
    char hosted_err[512] = {0};                         // the launcher's error message when hosted_rc != FX_OK
};

struct fx_plan {
    fx_comm* comm = nullptr;
    int world = 0, n = 0, dtype = 0, wire = 0, algo = 0;
    int grid_x = 1;
    std::vector<long long> numel, off;          // off has n+1 entries
    long long total = 0, padded = 0, shard = 0, slice = 0;
    int chunks = 0;                             // pipelined kernel: chunks per slice (0 = classic kernels)
    long long chunk = 0;
    int fuse_chunks = 0;                        // fused TMA kernel (fx_fuse.cu): chunks per slice (0 = not eligible)
    long long fuse_chunk = 0;                   // elements per chunk of one sub-range
    int fuse_unroll = 1;                        // NVLS: 16-byte multimem requests per lane in flight (1, 2, 4, 8)
    size_t esize = 0, wsize = 0, wire_bytes = 0;
    size_t region[2] = {0, 0};
    bool recycled = false;                      // region memory was used by an earlier plan
    unsigned long long signature = 0;
    // device side
    long long* d_off = nullptr;
    void** d_in = nullptr;
    void** d_out = nullptr;
    FxPlanState* d_state = nullptr;
    std::vector<const void*> h_in;
    std::vector<void*> h_out;
    std::vector<const void*> row_in;            // fx_allreduce_hosted: each hosted rank writes its row here
    std::vector<void*> row_out;
    bool in_valid = false, out_valid = false;
    bool begun = false;
    bool captured = false;                      // a launch of this plan was stream-captured (see upload_ptrs)
    std::vector<void*> capture_bufs;            // pinned pointer tables the captured copy nodes read
};

// ---------------------------------------------------------------- error plumbing
int fx_fail(int code, const char* fmt, ...);
#define FX_CUDA(expr)                                                                      \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess)                                                             \
            return fx_fail(FX_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,                    \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                    \
    } while (0)

size_t fx_dtype_size(int dtype);

// ---------------------------------------------------------------- kernel launchers (fx_kernels.cu)
int fx_launch_allreduce(fx_plan* plan, const FxLaunch& args, cudaStream_t stream);
int fx_launch_broadcast(fx_plan* plan, const FxLaunch& args, cudaStream_t stream);
int fx_launch_unpack(fx_plan* plan, const FxLaunch& args, cudaStream_t stream);
int fx_launch_barrier(fx_comm* comm, const FxLaunch& args, cudaStream_t stream);
// Fused five-role kernel with TMA staging (fx_fuse.cu): float SUM / AVG buckets sent in their own dtype.
int fx_launch_fuse(fx_plan* plan, const FxLaunch& args, cudaStream_t stream);
size_t fx_fuse_smem_bytes(int world, long long chunk_bytes);
size_t fx_fuse_trace_words(void);
// fx_kernel_id of the kernel an all-reduce of `op` on this plan launches (FUSED mode).
int fx_plan_kernel_id(const fx_plan* plan, int op);
// Largest gridDim.x such that gridDim.x * n_local CTAs of the widest kernel are co-resident.
int fx_max_coresident_blocks(int device, int n_local, int* sm_count);
bool fx_kernel_supported(int dtype, int wire, int op, bool broadcast);
