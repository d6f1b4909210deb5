// Host runtime of libflashy_b200.so: communicator bootstrap (symmetric arenas, peer mapping
// by VMM fd passing or cudaIpc, optional NVSwitch multicast), the shared-memory rendezvous
// that replaces the reference's host-synchronising count check, bucket planning, and the
// launch wrappers.  See include/flashy_b200.h for the contract of every entry point.
#include <cuda.h>
#include <cuda_runtime.h>

#include <errno.h>
#include <fcntl.h>
#include <poll.h>
#include <sched.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <sys/un.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <new>

#include "fx_internal.h"

// ============================================================================ errors
static thread_local char g_err[1024] = "";

int fx_fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

extern "C" const char* fx_last_error(void) { return g_err; }
extern "C" int fx_abi_version(void) { return FX_ABI_VERSION; }

extern "C" int fx_cuda_available(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n > 0;
}

size_t fx_dtype_size(int dtype) {
    switch (dtype) {
        case FX_F32: case FX_I32: return 4;
        case FX_BF16: case FX_F16: return 2;
        case FX_F64: case FX_I64: return 8;
        case FX_U8: return 1;
    }
    return 0;
}

static double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

static double env_double(const char* name, double dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atof(v) : dflt;
}
static long long env_ll(const char* name, long long dflt) {
    const char* v = getenv(name);
    return (v && *v) ? atoll(v) : dflt;
}

// ============================================================================ driver API (no link-time libcuda)
struct FxDriver {
    bool ok = false;
    CUresult (*MemCreate)(CUmemGenericAllocationHandle*, size_t, const CUmemAllocationProp*, unsigned long long);
    CUresult (*MemRelease)(CUmemGenericAllocationHandle);
    CUresult (*MemAddressReserve)(CUdeviceptr*, size_t, size_t, CUdeviceptr, unsigned long long);
    CUresult (*MemAddressFree)(CUdeviceptr, size_t);
    CUresult (*MemMap)(CUdeviceptr, size_t, size_t, CUmemGenericAllocationHandle, unsigned long long);
    CUresult (*MemUnmap)(CUdeviceptr, size_t);
    CUresult (*MemSetAccess)(CUdeviceptr, size_t, const CUmemAccessDesc*, size_t);
    CUresult (*MemExportToShareableHandle)(void*, CUmemGenericAllocationHandle, CUmemAllocationHandleType, unsigned long long);
    CUresult (*MemImportFromShareableHandle)(CUmemGenericAllocationHandle*, void*, CUmemAllocationHandleType);
    CUresult (*MemGetAllocationGranularity)(size_t*, const CUmemAllocationProp*, CUmemAllocationGranularity_flags);
    CUresult (*MulticastCreate)(CUmemGenericAllocationHandle*, const CUmulticastObjectProp*);
    CUresult (*MulticastAddDevice)(CUmemGenericAllocationHandle, CUdevice);
    CUresult (*MulticastBindMem)(CUmemGenericAllocationHandle, size_t, CUmemGenericAllocationHandle, size_t, size_t, unsigned long long);
    CUresult (*MulticastGetGranularity)(size_t*, const CUmulticastObjectProp*, CUmulticastGranularity_flags);
    CUresult (*DeviceGet)(CUdevice*, int);
    CUresult (*DeviceGetAttribute)(int*, CUdevice_attribute, CUdevice);
    CUresult (*GetErrorString)(CUresult, const char**);
};

static FxDriver& driver() {
    static FxDriver d;
    static std::once_flag once;
    std::call_once(once, [] {
        bool ok = true;
        auto get = [&](const char* name, void** fn) {
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint(name, fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !*fn) {
                cudaGetLastError();
                *fn = nullptr;
                ok = false;
            }
        };
        get("cuMemCreate", (void**)&d.MemCreate);
        get("cuMemRelease", (void**)&d.MemRelease);
        get("cuMemAddressReserve", (void**)&d.MemAddressReserve);
        get("cuMemAddressFree", (void**)&d.MemAddressFree);
        get("cuMemMap", (void**)&d.MemMap);
        get("cuMemUnmap", (void**)&d.MemUnmap);
        get("cuMemSetAccess", (void**)&d.MemSetAccess);
        get("cuMemExportToShareableHandle", (void**)&d.MemExportToShareableHandle);
        get("cuMemImportFromShareableHandle", (void**)&d.MemImportFromShareableHandle);
        get("cuMemGetAllocationGranularity", (void**)&d.MemGetAllocationGranularity);
        get("cuDeviceGet", (void**)&d.DeviceGet);
        get("cuDeviceGetAttribute", (void**)&d.DeviceGetAttribute);
        get("cuGetErrorString", (void**)&d.GetErrorString);
        bool core = ok;
        get("cuMulticastCreate", (void**)&d.MulticastCreate);
        get("cuMulticastAddDevice", (void**)&d.MulticastAddDevice);
        get("cuMulticastBindMem", (void**)&d.MulticastBindMem);
        get("cuMulticastGetGranularity", (void**)&d.MulticastGetGranularity);
        d.ok = core;
    });
    return d;
}

static const char* cu_err(CUresult r) {
    const char* s = nullptr;
    if (driver().GetErrorString && driver().GetErrorString(r, &s) == CUDA_SUCCESS && s) return s;
    return "unknown driver error";
}

#define FX_CU(expr)                                                                             \
    do {                                                                                        \
        CUresult _r = (expr);                                                                   \
        if (_r != CUDA_SUCCESS)                                                                 \
            return fx_fail(FX_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cu_err(_r), __FILE__, __LINE__); \
    } while (0)

// ============================================================================ export blob
#define FX_BLOB_MAGIC 0x46584232u   // "FXB2"
struct FxBlob {
    uint32_t magic;
    int32_t abi, world, rank0, n_local, device, mem_kind, pid;
    uint64_t arena_total;
    char sock[64];
    char shm[64];
    unsigned char uuid[16];
    cudaIpcMemHandle_t ipc[FX_MAX_WORLD];
    uint64_t host_id;                 // hash of (hostname, boot id): all ranks must share one host
    char hostname[64];
};

// Identity of the machine this process runs on.  The arenas are exchanged by fd passing over an
// abstract unix socket (or cudaIpc) and the count check lives in POSIX shared memory: both only
// exist inside one host.  FLASHY_B200_HOST_ID overrides the value (tests).
static uint64_t host_identity(char* name, size_t cap) {
    memset(name, 0, cap);
    if (gethostname(name, cap - 1) != 0) snprintf(name, cap, "unknown");
    const char* forced = getenv("FLASHY_B200_HOST_ID");
    if (forced && *forced) snprintf(name, cap, "%s", forced);
    unsigned long long h = 1469598103934665603ull;
    for (const char* p = name; *p; ++p) { h ^= (unsigned char)*p; h *= 1099511628211ull; }
    if (!(forced && *forced)) {
        char boot[64] = {0};
        FILE* f = fopen("/proc/sys/kernel/random/boot_id", "r");
        if (f) { if (!fgets(boot, sizeof(boot), f)) boot[0] = 0; fclose(f); }
        for (const char* p = boot; *p; ++p) { h ^= (unsigned char)*p; h *= 1099511628211ull; }
    }
    return h;
}

// ============================================================================ fd passing over an abstract unix socket
static int send_fd(int sock, int fd) {
    char dummy = 'F';
    iovec iov = {&dummy, 1};
    char ctrl[CMSG_SPACE(sizeof(int))];
    memset(ctrl, 0, sizeof(ctrl));
    msghdr msg = {};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    cmsghdr* c = CMSG_FIRSTHDR(&msg);
    c->cmsg_level = SOL_SOCKET;
    c->cmsg_type = SCM_RIGHTS;
    c->cmsg_len = CMSG_LEN(sizeof(int));
    memcpy(CMSG_DATA(c), &fd, sizeof(int));
    return sendmsg(sock, &msg, 0) == 1 ? 0 : -1;
}

static int recv_fd(int sock) {
    char dummy = 0;
    iovec iov = {&dummy, 1};
    char ctrl[CMSG_SPACE(sizeof(int))];
    memset(ctrl, 0, sizeof(ctrl));
    msghdr msg = {};
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    if (recvmsg(sock, &msg, 0) != 1) return -1;
    cmsghdr* c = CMSG_FIRSTHDR(&msg);
    if (!c || c->cmsg_level != SOL_SOCKET || c->cmsg_type != SCM_RIGHTS) return -1;
    int fd = -1;
    memcpy(&fd, CMSG_DATA(c), sizeof(int));
    return fd;
}

static socklen_t abstract_addr(sockaddr_un* addr, const char* name) {
    memset(addr, 0, sizeof(*addr));
    addr->sun_family = AF_UNIX;
    size_t n = strlen(name);
    memcpy(addr->sun_path + 1, name, n);            // leading NUL = abstract namespace
    return (socklen_t)(offsetof(sockaddr_un, sun_path) + 1 + n);
}

struct FdRequest { int32_t local; int32_t what; };  // what: 0 = arena handle, 1 = multicast handle

static void fd_server_loop(fx_comm* c) {
    while (!c->stop.load()) {
        pollfd p = {c->listen_fd, POLLIN, 0};
        int r = poll(&p, 1, 100);
        if (r <= 0) continue;
        int s = accept(c->listen_fd, nullptr, nullptr);
        if (s < 0) continue;
        FdRequest req;
        if (read(s, &req, sizeof(req)) == (ssize_t)sizeof(req)) {
            int fd = -1;
            if (req.what == 0 && req.local >= 0 && req.local < c->n_local) fd = c->arena[c->rank0 + req.local].vmm_fd;
            if (req.what == 1) fd = c->mc_fd;
            if (fd >= 0) send_fd(s, fd);
        }
        close(s);
    }
}

static int fetch_fd(const char* sock_name, int local, int what, double timeout_s) {
    const double t0 = now_s();
    while (true) {
        int s = socket(AF_UNIX, SOCK_STREAM, 0);
        if (s < 0) return -1;
        sockaddr_un addr;
        socklen_t len = abstract_addr(&addr, sock_name);
        if (connect(s, (sockaddr*)&addr, len) == 0) {
            FdRequest req = {local, what};
            int fd = -1;
            if (write(s, &req, sizeof(req)) == (ssize_t)sizeof(req)) fd = recv_fd(s);
            close(s);
            if (fd >= 0) return fd;
        } else {
            close(s);
        }
        if (now_s() - t0 > timeout_s) return -1;
        usleep(2000);
    }
}

// ============================================================================ arenas
static int arena_alloc_vmm(fx_comm* c, FxArena& a) {
    FxDriver& d = driver();
    if (!d.ok) return fx_fail(FX_ERR_UNSUPPORTED, "CUDA VMM driver entry points unavailable");
    CUmemAllocationProp prop = {};
    prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop.location.id = c->device;
    prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    size_t gran = 0;
    FX_CU(d.MemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (gran < (2u << 20)) gran = 2u << 20;
    a.bytes = (c->arena_total + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle h;
    FX_CU(d.MemCreate(&h, a.bytes, &prop, 0));
    CUdeviceptr va = 0;
    FX_CU(d.MemAddressReserve(&va, a.bytes, gran, 0, 0));
    FX_CU(d.MemMap(va, a.bytes, 0, h, 0));
    CUmemAccessDesc acc = {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = c->device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    FX_CU(d.MemSetAccess(va, a.bytes, &acc, 1));
    int fd = -1;
    if (c->n_local < c->world) {      // other processes will import it
        FX_CU(d.MemExportToShareableHandle(&fd, h, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    }
    a.base = reinterpret_cast<char*>(va);
    a.vmm_handle = h;
    a.vmm_fd = fd;
    a.owned = true;
    return FX_OK;
}

static int arena_alloc_plain(fx_comm* c, FxArena& a) {
    a.bytes = (c->arena_total + (2u << 20) - 1) / (2u << 20) * (2u << 20);
    void* p = nullptr;
    FX_CUDA(cudaMalloc(&p, a.bytes));
    a.base = static_cast<char*>(p);
    a.owned = true;
    return FX_OK;
}

static int arena_import_vmm(fx_comm* c, FxArena& a, int fd, size_t bytes) {
    FxDriver& d = driver();
    CUmemGenericAllocationHandle h;
    FX_CU(d.MemImportFromShareableHandle(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
    CUdeviceptr va = 0;
    FX_CU(d.MemAddressReserve(&va, bytes, 2u << 20, 0, 0));
    FX_CU(d.MemMap(va, bytes, 0, h, 0));
    CUmemAccessDesc acc = {};
    acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    acc.location.id = c->device;
    acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    FX_CU(d.MemSetAccess(va, bytes, &acc, 1));
    a.base = reinterpret_cast<char*>(va);
    a.bytes = bytes;
    a.vmm_handle = h;
    a.owned = false;
    return FX_OK;
}

static void arena_release(fx_comm* c, FxArena& a) {
    if (!a.base) return;
    if (c->mem_kind == FX_COMM_MEM_VMM) {
        FxDriver& d = driver();
        d.MemUnmap((CUdeviceptr)a.base, a.bytes);
        d.MemAddressFree((CUdeviceptr)a.base, a.bytes);
        if (a.vmm_handle) d.MemRelease(a.vmm_handle);
        if (a.vmm_fd >= 0) close(a.vmm_fd);
    } else if (a.owned) {
        cudaFree(a.base);
    } else if (a.ipc_opened) {
        cudaIpcCloseMemHandle(a.base);
    }
    a = FxArena();
}

// ============================================================================ communicator
extern "C" int fx_comm_create(int world, int rank0, int n_local, int device, size_t arena_bytes,
                              unsigned flags, fx_comm** out) {
    if (!out) return fx_fail(FX_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (world < 1 || world > FX_MAX_WORLD || n_local < 1 || rank0 < 0 || rank0 + n_local > world)
        return fx_fail(FX_ERR_INVALID, "bad geometry: world=%d rank0=%d n_local=%d (max world %d)", world, rank0, n_local, FX_MAX_WORLD);
    fx_comm* c = new (std::nothrow) fx_comm();
    if (!c) return fx_fail(FX_ERR_SYS, "out of memory");
    c->world = world; c->rank0 = rank0; c->n_local = n_local; c->device = device; c->flags = flags;
    c->host_only = (flags & FX_COMM_HOST_ONLY) != 0;
    c->timeout_ns = (unsigned long long)(env_double("FLASHY_B200_DEVICE_TIMEOUT", 120.0) * 1e9);
    srand((unsigned)(getpid() * 2654435761u) ^ (unsigned)time(nullptr));
    const unsigned nonce = (unsigned)rand();

    // ---- host rendezvous fabric: heap when this process hosts the whole world, else POSIX shm
    if (n_local == world) {
        c->shm = new (std::nothrow) FxShm();
        c->shm_is_heap = true;
        if (!c->shm) { delete c; return fx_fail(FX_ERR_SYS, "out of memory"); }
        memset((void*)c->shm, 0, sizeof(FxShm));
    } else if (rank0 == 0) {
        snprintf(c->shm_name, sizeof(c->shm_name), "/fxb200-%d-%08x", (int)getpid(), nonce);
        int fd = shm_open(c->shm_name, O_CREAT | O_EXCL | O_RDWR, 0600);
        if (fd < 0) { int e = errno; delete c; return fx_fail(FX_ERR_SYS, "shm_open(%s): %s", c->shm_name, strerror(e)); }
        if (ftruncate(fd, sizeof(FxShm)) != 0) { int e = errno; close(fd); shm_unlink(c->shm_name); delete c; return fx_fail(FX_ERR_SYS, "ftruncate: %s", strerror(e)); }
        void* p = mmap(nullptr, sizeof(FxShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        close(fd);
        if (p == MAP_FAILED) { shm_unlink(c->shm_name); delete c; return fx_fail(FX_ERR_SYS, "mmap shm failed"); }
        c->shm = static_cast<FxShm*>(p);      // zero-filled by ftruncate
        c->shm_owner = true;
    }

    if (c->host_only) {
        c->connected = (n_local == world);
        *out = c;
        return FX_OK;
    }

    // ---- device side
    int rc = FX_OK;
    do {
        cudaError_t e = cudaSetDevice(device);
        if (e != cudaSuccess) { rc = fx_fail(FX_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e)); break; }
        c->max_blocks = fx_max_coresident_blocks(device, n_local, &c->sm_count);
        long long cap = env_ll("FLASHY_B200_MAX_BLOCKS", 0);
        if (cap > 0 && cap < c->max_blocks) c->max_blocks = (int)cap;
        c->arena_bytes = (arena_bytes + 255) / 256 * 256;
        c->arena_total = FX_PAD_BYTES + c->arena_bytes;
        unsigned want = flags & FX_COMM_MEM_MASK;
        const char* env_mem = getenv("FLASHY_B200_MEM");
        if (want == FX_COMM_MEM_AUTO && env_mem) {
            if (!strcmp(env_mem, "ipc")) want = FX_COMM_MEM_IPC;
            else if (!strcmp(env_mem, "vmm")) want = FX_COMM_MEM_VMM;
        }
        c->mem_kind = (want == FX_COMM_MEM_IPC) ? FX_COMM_MEM_IPC : FX_COMM_MEM_VMM;
        for (int l = 0; l < n_local && rc == FX_OK; ++l) {
            FxArena& a = c->arena[rank0 + l];
            if (c->mem_kind == FX_COMM_MEM_VMM) {
                rc = arena_alloc_vmm(c, a);
                if (rc != FX_OK && want == FX_COMM_MEM_AUTO && l == 0) {   // driver refuses VMM export: fall back
                    c->mem_kind = FX_COMM_MEM_IPC;
                    rc = arena_alloc_plain(c, a);
                }
            } else {
                rc = arena_alloc_plain(c, a);
            }
            if (rc == FX_OK && cudaMemset(a.base, 0, FX_PAD_BYTES) != cudaSuccess)
                rc = fx_fail(FX_ERR_CUDA, "cudaMemset(pad) failed: %s", cudaGetErrorString(cudaGetLastError()));
        }
        if (rc != FX_OK) break;
        if (cudaHostAlloc((void**)&c->status_host, 64, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
            cudaHostGetDevicePointer((void**)&c->status_dev, c->status_host, 0) != cudaSuccess) {
            rc = fx_fail(FX_ERR_CUDA, "status word allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
            break;
        }
        *c->status_host = 0;
        if (env_ll("FLASHY_B200_TRACE", 0) != 0) {
            const size_t tb = fx_fuse_trace_words() * sizeof(unsigned long long);
            if (cudaMalloc((void**)&c->trace_dev, tb) != cudaSuccess || cudaMemset(c->trace_dev, 0, tb) != cudaSuccess) {
                rc = fx_fail(FX_ERR_CUDA, "trace buffer allocation failed: %s", cudaGetErrorString(cudaGetLastError()));
                break;
            }
        }
        if (cudaDeviceSynchronize() != cudaSuccess) { rc = fx_fail(FX_ERR_CUDA, "device sync failed"); break; }
        // ---- fd server for VMM handles
        if (c->mem_kind == FX_COMM_MEM_VMM && n_local < world) {
            snprintf(c->sock_name, sizeof(c->sock_name), "fxb200-%d-%08x", (int)getpid(), nonce);
            c->listen_fd = socket(AF_UNIX, SOCK_STREAM, 0);
            sockaddr_un addr;
            socklen_t len = abstract_addr(&addr, c->sock_name);
            if (c->listen_fd < 0 || bind(c->listen_fd, (sockaddr*)&addr, len) != 0 || listen(c->listen_fd, 64) != 0) {
                rc = fx_fail(FX_ERR_SYS, "unix socket setup failed: %s", strerror(errno));
                break;
            }
            c->server = std::thread(fd_server_loop, c);
        }
        c->connected = (n_local == world);
    } while (0);
    if (rc != FX_OK) {
        char keep[sizeof(g_err)];
        memcpy(keep, g_err, sizeof(keep));
        fx_comm_destroy(c);
        memcpy(g_err, keep, sizeof(keep));
        return rc;
    }
    *out = c;
    return FX_OK;
}

extern "C" int fx_comm_export(fx_comm* c, void* blob, size_t cap, size_t* len) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (len) *len = sizeof(FxBlob);
    if (!blob) return FX_OK;
    if (cap < sizeof(FxBlob)) return fx_fail(FX_ERR_INVALID, "blob buffer too small (%zu < %zu)", cap, sizeof(FxBlob));
    FxBlob b;
    memset(&b, 0, sizeof(b));
    b.magic = FX_BLOB_MAGIC; b.abi = FX_ABI_VERSION;
    b.world = c->world; b.rank0 = c->rank0; b.n_local = c->n_local; b.device = c->device;
    b.mem_kind = c->mem_kind; b.pid = (int)getpid();
    b.arena_total = c->host_only ? 0 : c->arena[c->rank0].bytes;
    memcpy(b.sock, c->sock_name, sizeof(b.sock));
    memcpy(b.shm, c->shm_name, sizeof(b.shm));
    b.host_id = host_identity(b.hostname, sizeof(b.hostname));
    if (!c->host_only) {
        cudaDeviceProp prop;
        FX_CUDA(cudaGetDeviceProperties(&prop, c->device));
        memcpy(b.uuid, &prop.uuid, 16);
        if (c->mem_kind == FX_COMM_MEM_IPC && c->n_local < c->world) {
            for (int l = 0; l < c->n_local; ++l)
                FX_CUDA(cudaIpcGetMemHandle(&b.ipc[l], c->arena[c->rank0 + l].base));
        }
    }
    memcpy(blob, &b, sizeof(b));
    return FX_OK;
}

extern "C" int fx_comm_connect(fx_comm* c, const void* blobs, size_t blob_len, int n_procs) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    std::lock_guard<std::mutex> lock(c->mu);
    if (c->connected) return FX_OK;
    if (!blobs || blob_len != sizeof(FxBlob) || n_procs < 1)
        return fx_fail(FX_ERR_INVALID, "connect: need %d-byte blobs of every process", (int)sizeof(FxBlob));
    const FxBlob* all = static_cast<const FxBlob*>(blobs);
    int covered = 0;
    for (int p = 0; p < n_procs; ++p) {
        const FxBlob& b = all[p];
        if (b.magic != FX_BLOB_MAGIC || b.abi != FX_ABI_VERSION) return fx_fail(FX_ERR_INVALID, "blob %d: bad magic/abi", p);
        if (b.world != c->world) return fx_fail(FX_ERR_MISMATCH, "blob %d: world %d != %d", p, b.world, c->world);
        if (b.rank0 != covered) return fx_fail(FX_ERR_INVALID, "blobs must be in rank order without gaps (got rank0=%d, expected %d)", b.rank0, covered);
        if (!c->host_only && b.mem_kind != c->mem_kind) return fx_fail(FX_ERR_MISMATCH, "blob %d: memory kind differs (%d vs %d)", p, b.mem_kind, c->mem_kind);
        covered += b.n_local;
    }
    if (covered != c->world) return fx_fail(FX_ERR_INVALID, "blobs cover %d ranks, world is %d", covered, c->world);
    // One NVSwitch domain = one host (SURVEY.md 8e): refuse a world that spans machines instead of failing
    // later in fd passing / shm_open with an unrelated message.
    for (int p = 1; p < n_procs; ++p) {
        if (all[p].host_id != all[0].host_id)
            return fx_fail(FX_ERR_UNSUPPORTED, "ranks span several hosts (rank %d is on '%.63s', rank %d on '%.63s'): flashy_b200 "
                           "moves data over NVLink inside ONE NVSwitch domain; run one job per node or use torch.distributed "
                           "(NCCL) for multi-node worlds", all[0].rank0, all[0].hostname, all[p].rank0, all[p].hostname);
    }
    // ---- rendezvous shm (created by the process hosting rank 0)
    if (!c->shm) {
        const char* name = all[0].shm;
        int fd = shm_open(name, O_RDWR, 0600);
        if (fd < 0) return fx_fail(FX_ERR_SYS, "shm_open(%s): %s", name, strerror(errno));
        void* p = mmap(nullptr, sizeof(FxShm), PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
        close(fd);
        if (p == MAP_FAILED) return fx_fail(FX_ERR_SYS, "mmap shm failed: %s", strerror(errno));
        c->shm = static_cast<FxShm*>(p);
        memcpy(c->shm_name, name, sizeof(c->shm_name));
    }
    if (!c->host_only) {
        FX_CUDA(cudaSetDevice(c->device));
        for (int p = 0; p < n_procs; ++p) {
            const FxBlob& b = all[p];
            if (b.rank0 == c->rank0) continue;               // ourselves
            for (int l = 0; l < b.n_local; ++l) {
                FxArena& a = c->arena[b.rank0 + l];
                if (c->mem_kind == FX_COMM_MEM_VMM) {
                    int fd = fetch_fd(b.sock, l, 0, 60.0);
                    if (fd < 0) return fx_fail(FX_ERR_SYS, "could not fetch the arena fd of rank %d from pid %d", b.rank0 + l, b.pid);
                    int rc = arena_import_vmm(c, a, fd, (size_t)b.arena_total);
                    close(fd);
                    if (rc != FX_OK) return rc;
                } else {
                    void* ptr = nullptr;
                    FX_CUDA(cudaIpcOpenMemHandle(&ptr, b.ipc[l], cudaIpcMemLazyEnablePeerAccess));
                    a.base = static_cast<char*>(ptr);
                    a.bytes = (size_t)b.arena_total;
                    a.ipc_opened = true;
                }
            }
        }
    }
    c->shm->attached.fetch_add(c->n_local);
    c->connected = true;
    return FX_OK;
}

// Collective agreement over the host fabric: every rank reports `ok`; returns true iff all did.
static bool all_agree(fx_comm* c, bool ok) {
    int64_t sum = 0;
    int eq = 0;
    if (fx_host_exchange(c, 0, ok ? 1 : 0, 0x4d43u, &sum, &eq, 120.0) != FX_OK) return false;
    return sum == c->world;
}

extern "C" int fx_comm_enable_multicast(fx_comm* c, const void* blobs, size_t blob_len, int n_procs) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (c->multicast) return FX_OK;
    if (c->host_only || !c->connected) return fx_fail(FX_ERR_STATE, "multicast needs a connected device communicator");
    if (c->n_local != 1 || c->world < 2)
        return fx_fail(FX_ERR_UNSUPPORTED, "NVLS multicast needs one rank per process and at least two GPUs");
    if (!blobs || blob_len != sizeof(FxBlob) || n_procs != c->world) return fx_fail(FX_ERR_INVALID, "multicast: need the export blobs of every process");
    const FxBlob* all = static_cast<const FxBlob*>(blobs);
    FxDriver& d = driver();
    FxArena& mine = c->arena[c->rank0];
    char why[256] = "";

    // ---- step 0: can everybody do it at all?
    bool ok = d.ok && d.MulticastCreate && d.MulticastAddDevice && d.MulticastBindMem && d.MulticastGetGranularity &&
              c->mem_kind == FX_COMM_MEM_VMM && mine.vmm_handle != 0;
    CUdevice dev = 0;
    if (ok) {
        int sup = 0;
        ok = d.DeviceGet(&dev, c->device) == CUDA_SUCCESS &&
             d.DeviceGetAttribute(&sup, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, dev) == CUDA_SUCCESS && sup == 1;
        if (!ok) snprintf(why, sizeof(why), "device reports no multicast support");
    } else {
        snprintf(why, sizeof(why), "driver lacks cuMulticast* or arenas are not VMM allocations");
    }
    if (!all_agree(c, ok)) return fx_fail(FX_ERR_UNSUPPORTED, "multicast unavailable on at least one rank (%s)", why);

    CUmulticastObjectProp prop = {};
    prop.numDevices = (unsigned)c->world;
    prop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    prop.flags = 0;
    size_t gran = 0;
    prop.size = mine.bytes;
    ok = d.MulticastGetGranularity(&gran, &prop, CU_MULTICAST_GRANULARITY_MINIMUM) == CUDA_SUCCESS && gran > 0;
    size_t mc_bytes = ok ? mine.bytes / gran * gran : 0;
    ok = ok && mc_bytes >= (size_t)FX_PAD_BYTES + (1u << 20);
    prop.size = mc_bytes;

    // ---- step 1: rank 0 creates the object and exports it
    CUmemGenericAllocationHandle mc = 0;
    if (ok && c->rank0 == 0) {
        CUresult r = d.MulticastCreate(&mc, &prop);
        int fd = -1;
        if (r == CUDA_SUCCESS) r = d.MemExportToShareableHandle(&fd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
        ok = r == CUDA_SUCCESS;
        if (ok) c->mc_fd = fd; else snprintf(why, sizeof(why), "cuMulticastCreate/export: %s", cu_err(r));
    }
    if (!all_agree(c, ok)) {
        if (mc) d.MemRelease(mc);
        return fx_fail(FX_ERR_UNSUPPORTED, "multicast object could not be created (%s)", why);
    }
    // ---- step 2: everyone else imports it; all add their device
    if (c->rank0 != 0) {
        int fd = fetch_fd(all[0].sock, 0, 1, 60.0);
        ok = fd >= 0;
        if (ok) {
            CUresult r = d.MemImportFromShareableHandle(&mc, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
            close(fd);
            ok = r == CUDA_SUCCESS;
            if (!ok) snprintf(why, sizeof(why), "import of the multicast handle: %s", cu_err(r));
        } else {
            snprintf(why, sizeof(why), "could not fetch the multicast fd from rank 0");
        }
    }
    if (ok) {
        CUresult r = d.MulticastAddDevice(mc, dev);
        ok = r == CUDA_SUCCESS;
        if (!ok) snprintf(why, sizeof(why), "cuMulticastAddDevice: %s", cu_err(r));
    }
    if (!all_agree(c, ok)) {
        if (mc) d.MemRelease(mc);
        return fx_fail(FX_ERR_UNSUPPORTED, "multicast join failed (%s)", why);
    }
    // ---- step 3: bind this rank's arena at offset 0 (every device binds its own memory there)
    {
        CUresult r = d.MulticastBindMem(mc, 0, mine.vmm_handle, 0, mc_bytes, 0);
        ok = r == CUDA_SUCCESS;
        if (!ok) snprintf(why, sizeof(why), "cuMulticastBindMem: %s", cu_err(r));
    }
    if (!all_agree(c, ok)) {
        d.MemRelease(mc);
        return fx_fail(FX_ERR_UNSUPPORTED, "multicast bind failed (%s)", why);
    }
    // ---- step 4: map the multicast address range
    CUdeviceptr va = 0;
    {
        CUresult r = d.MemAddressReserve(&va, mc_bytes, gran, 0, 0);
        if (r == CUDA_SUCCESS) r = d.MemMap(va, mc_bytes, 0, mc, 0);
        if (r == CUDA_SUCCESS) {
            CUmemAccessDesc acc = {};
            acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
            acc.location.id = c->device;
            acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
            r = d.MemSetAccess(va, mc_bytes, &acc, 1);
        }
        ok = r == CUDA_SUCCESS;
        if (!ok) snprintf(why, sizeof(why), "mapping the multicast range: %s", cu_err(r));
    }
    if (!all_agree(c, ok)) return fx_fail(FX_ERR_UNSUPPORTED, "multicast mapping failed (%s)", why);
    std::lock_guard<std::mutex> lock(c->mu);
    c->mc_handle = mc;
    c->mc_base = reinterpret_cast<char*>(va);
    c->mc_bytes = mc_bytes;
    c->multicast = true;
    return FX_OK;
}

extern "C" int fx_comm_get_info(fx_comm* c, fx_comm_info* info) {
    if (!c || !info) return fx_fail(FX_ERR_INVALID, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->abi_version = FX_ABI_VERSION;
    info->world = c->world; info->rank0 = c->rank0; info->n_local = c->n_local; info->device = c->device;
    info->mem_kind = c->host_only ? 0 : c->mem_kind;
    info->connected = c->connected; info->multicast = c->multicast;
    info->sm_count = c->sm_count; info->max_blocks = c->max_blocks;
    info->arena_bytes = c->arena_bytes; info->arena_used = c->arena_used; info->launches = c->launches;
    return FX_OK;
}

extern "C" int fx_comm_set_plan_blocks(fx_comm* c, int max_blocks) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (max_blocks < 0) return fx_fail(FX_ERR_INVALID, "max_blocks must be >= 0");
    std::lock_guard<std::mutex> lock(c->mu);
    c->plan_blocks = max_blocks;
    return FX_OK;
}

extern "C" int fx_comm_get_pointers(fx_comm* c, void** arenas, void** mc_base, uint64_t* mc_bytes, uint64_t* pad_bytes) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (c->host_only || !c->connected) return fx_fail(FX_ERR_STATE, "needs a connected device communicator");
    if (arenas) for (int r = 0; r < c->world; ++r) arenas[r] = c->arena[r].base;
    if (mc_base) *mc_base = c->mc_base;
    if (mc_bytes) *mc_bytes = c->multicast ? c->mc_bytes : 0;
    if (pad_bytes) *pad_bytes = FX_PAD_BYTES;
    return FX_OK;
}

extern "C" int fx_comm_trace_read(fx_comm* c, uint64_t* out, size_t cap_words, size_t* words) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    const size_t n = fx_fuse_trace_words();
    if (words) *words = c->trace_dev ? n : 0;
    if (!out || !c->trace_dev) return FX_OK;
    if (cap_words < n) return fx_fail(FX_ERR_INVALID, "trace buffer too small (%zu < %zu words)", cap_words, n);
    FX_CUDA(cudaSetDevice(c->device));
    FX_CUDA(cudaDeviceSynchronize());
    FX_CUDA(cudaMemcpy(out, c->trace_dev, n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    FX_CUDA(cudaMemset(c->trace_dev, 0, n * sizeof(uint64_t)));
    return FX_OK;
}

extern "C" int fx_comm_poll(fx_comm* c) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (c->host_only || !c->status_host) return FX_OK;
    uint32_t s = *reinterpret_cast<volatile uint32_t*>(c->status_host);
    if (s == 0) return FX_OK;
    return fx_fail(-(int)s, "device-side failure %d: a peer rank did not reach a collective within %.0f s "
                   "(ranks issued different collectives, or a rank died)", -(int)s, c->timeout_ns * 1e-9);
}

extern "C" int fx_comm_abort(fx_comm* c) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    if (c->shm) c->shm->aborted.store(1, std::memory_order_release);
    return FX_OK;
}

extern "C" void fx_comm_destroy(fx_comm* c) {
    if (!c) return;
    c->stop.store(true);
    if (c->server.joinable()) c->server.join();
    if (c->listen_fd >= 0) close(c->listen_fd);
    if (!c->host_only && c->device >= 0) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
        for (int r = 0; r < c->world; ++r) arena_release(c, c->arena[r]);
        if (c->status_host) cudaFreeHost(c->status_host);
        if (c->order_event) cudaEventDestroy(c->order_event);
        if (c->trace_dev) cudaFree(c->trace_dev);
        cudaGetLastError();
    }
    if (c->shm) {
        if (c->shm_is_heap) delete c->shm;
        else munmap((void*)c->shm, sizeof(FxShm));
    }
    if (c->shm_owner && c->shm_name[0]) shm_unlink(c->shm_name);
    delete c;
}

// ============================================================================ host rendezvous
static int host_wait_all(fx_comm* c, int parity, long long seq, double timeout_s, const char* what) {
    const double t0 = now_s();
    unsigned spins = 0;
    for (int q = 0; q < c->world; ++q) {
        while (c->shm->slot[parity][q].seq.load(std::memory_order_acquire) < seq) {
            if (++spins < 2000) continue;
            sched_yield();
            if ((spins & 0xff) == 0) {
                if (c->shm->aborted.load(std::memory_order_acquire))
                    return fx_fail(FX_ERR_STATE, "%s: the communicator was aborted by a rank that failed", what);
                if (now_s() - t0 > timeout_s)
                    return fx_fail(FX_ERR_TIMEOUT, "%s: rank %d did not arrive within %.0f s (collective #%lld)", what, q, timeout_s, seq);
                if (spins > 200000) usleep(50);
            }
        }
    }
    return FX_OK;
}

extern "C" int fx_host_exchange(fx_comm* c, int local, int64_t count, uint64_t signature,
                                int64_t* sum_out, int* sig_equal, double timeout_s) {
    if (!c || local < 0 || local >= c->n_local) return fx_fail(FX_ERR_INVALID, "bad comm/local index");
    if (!c->connected || !c->shm) return fx_fail(FX_ERR_STATE, "communicator is not connected yet");
    if (c->shm->aborted.load(std::memory_order_acquire)) return fx_fail(FX_ERR_STATE, "the communicator was aborted by a rank that failed");
    if (timeout_s <= 0) timeout_s = env_double("FLASHY_B200_HOST_TIMEOUT", 600.0);
    const int rank = c->rank0 + local;
    const long long seq = ++c->host_seq[local];
    const int parity = (int)(seq & 1);
    FxShmSlot& mine = c->shm->slot[parity][rank];
    mine.count = count;
    mine.sig = signature;
    mine.seq.store(seq, std::memory_order_release);
    int rc = host_wait_all(c, parity, seq, timeout_s, "host exchange");
    if (rc != FX_OK) return rc;
    long long sum = 0;
    int equal = 1;
    for (int q = 0; q < c->world; ++q) {
        sum += c->shm->slot[parity][q].count;
        if (c->shm->slot[parity][q].sig != signature) equal = 0;
    }
    if (sum_out) *sum_out = sum;
    if (sig_equal) *sig_equal = equal;
    return FX_OK;
}

extern "C" int fx_host_barrier(fx_comm* c, int local, double timeout_s) {
    return fx_host_exchange(c, local, 0, 0, nullptr, nullptr, timeout_s);
}

extern "C" int fx_host_broadcast(fx_comm* c, int local, int src, void* buf, size_t nbytes, double timeout_s) {
    if (!c || local < 0 || local >= c->n_local) return fx_fail(FX_ERR_INVALID, "bad comm/local index");
    if (!c->connected || !c->shm) return fx_fail(FX_ERR_STATE, "communicator is not connected yet");
    if (src < 0 || src >= c->world) return fx_fail(FX_ERR_INVALID, "broadcast source %d out of range", src);
    if (nbytes && !buf) return fx_fail(FX_ERR_INVALID, "buf is NULL");
    if (timeout_s <= 0) timeout_s = env_double("FLASHY_B200_HOST_TIMEOUT", 600.0);
    const int rank = c->rank0 + local;
    FxShm* sh = c->shm;
    char* p = static_cast<char*>(buf);
    const double t0 = now_s();
    auto spin = [&](auto done, const char* what) -> int {
        unsigned spins = 0;
        while (!done()) {
            if (++spins < 2000) continue;
            sched_yield();
            if ((spins & 0xff) == 0) {
                if (sh->aborted.load(std::memory_order_acquire))
                    return fx_fail(FX_ERR_STATE, "host broadcast: the communicator was aborted by a rank that failed");
                if (now_s() - t0 > timeout_s)
                    return fx_fail(FX_ERR_TIMEOUT, "host broadcast: %s timed out after %.0f s", what, timeout_s);
            }
        }
        return FX_OK;
    };
    const size_t rounds = nbytes ? (nbytes + FX_BCAST_CHUNK - 1) / FX_BCAST_CHUNK : 1;
    for (size_t r = 0; r < rounds; ++r) {
        const size_t lo = r * FX_BCAST_CHUNK;
        const size_t n = nbytes > lo ? std::min<size_t>(FX_BCAST_CHUNK, nbytes - lo) : 0;
        const long long seq = ++c->bcast_seq[local];
        int rc;
        if (rank == src) {
            // the previous chunk must have been consumed by all W-1 readers before it is overwritten
            if ((rc = spin([&] { return sh->bc_seq.load(std::memory_order_acquire) == seq - 1 &&
                                        (seq == 1 || sh->bc_acks.load(std::memory_order_acquire) == c->world - 1); },
                           "waiting for the readers")) != FX_OK) return rc;
            sh->bc_acks.store(0, std::memory_order_relaxed);
            if (n) memcpy(sh->bc_data, p + lo, n);
            sh->bc_len = (long long)n;
            sh->bc_seq.store(seq, std::memory_order_release);
        } else {
            if ((rc = spin([&] { return sh->bc_seq.load(std::memory_order_acquire) == seq; }, "waiting for the source")) != FX_OK) return rc;
            if ((size_t)sh->bc_len != n) return fx_fail(FX_ERR_MISMATCH, "host broadcast: ranks disagree on the size (%lld vs %zu)", sh->bc_len, n);
            if (n) memcpy(p + lo, sh->bc_data, n);
            sh->bc_acks.fetch_add(1, std::memory_order_acq_rel);
        }
    }
    return FX_OK;
}

// ============================================================================ plans
static unsigned long long fnv1a(unsigned long long h, const void* data, size_t n) {
    const unsigned char* p = static_cast<const unsigned char*>(data);
    for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

static size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

extern "C" int fx_plan_create(fx_comm* c, int world, const int64_t* numels, int n, int dtype,
                              int wire_dtype, int algo, fx_plan** out) {
    if (!out) return fx_fail(FX_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (c) world = c->world;
    if (world < 1 || world > FX_MAX_WORLD) return fx_fail(FX_ERR_INVALID, "bad world %d", world);
    if (n < 1 || !numels) return fx_fail(FX_ERR_INVALID, "a plan needs at least one tensor");
    const size_t esize = fx_dtype_size(dtype), wsize = fx_dtype_size(wire_dtype);
    if (!esize || !wsize) return fx_fail(FX_ERR_INVALID, "unknown dtype %d / %d", dtype, wire_dtype);
    if (dtype != wire_dtype && !(dtype == FX_F32 && wire_dtype == FX_BF16))
        return fx_fail(FX_ERR_UNSUPPORTED, "wire cast %d -> %d is not supported (only fp32 -> bf16)", dtype, wire_dtype);
    if (algo < FX_ALGO_AUTO || algo > FX_ALGO_NVLS) return fx_fail(FX_ERR_INVALID, "unknown algo %d", algo);
    if (algo == FX_ALGO_NVLS && !(c && c->multicast)) return fx_fail(FX_ERR_UNSUPPORTED, "NVLS needs an enabled multicast binding");

    fx_plan* p = new (std::nothrow) fx_plan();
    if (!p) return fx_fail(FX_ERR_SYS, "out of memory");
    p->comm = c; p->world = world; p->n = n; p->dtype = dtype; p->wire = wire_dtype;
    p->esize = esize; p->wsize = wsize;
    const long long align_e = FX_VEC_BYTES / (long long)std::min(esize, wsize);
    p->numel.assign(numels, numels + n);
    p->off.resize(n + 1);
    long long cur = 0;
    for (int i = 0; i < n; ++i) {
        if (numels[i] < 0) { delete p; return fx_fail(FX_ERR_INVALID, "negative numel for tensor %d", i); }
        p->off[i] = cur;
        p->total += numels[i];
        cur = (cur + numels[i] + align_e - 1) / align_e * align_e;
    }
    p->off[n] = cur;
    unsigned long long sig = 1469598103934665603ull;
    sig = fnv1a(sig, &n, sizeof(n));
    sig = fnv1a(sig, &dtype, sizeof(dtype));
    sig = fnv1a(sig, &wire_dtype, sizeof(wire_dtype));
    sig = fnv1a(sig, numels, sizeof(int64_t) * n);
    p->signature = sig;

    const size_t data_bytes = (size_t)cur * wsize;
    const size_t one_shot_max = (size_t)env_ll("FLASHY_B200_ONE_SHOT_MAX", 256 << 10);
    const size_t nvls_min = (size_t)env_ll("FLASHY_B200_NVLS_MIN", 512 << 10);
    // NVLS moves (1 + 1/W) N bytes per direction, the peer-to-peer two-shot 2 (W-1)/W N: at W = 2 the switch
    // moves 1.5 N against N.  The W = 4 default of FLASHY_B200_NVLS_MIN_WORLD and the size thresholds above
    // were tuned on an earlier target (B200, NVLink 5) and are not yet re-measured on H100.
    const bool nvls_ok = c && c->multicast && (wire_dtype == FX_F32 || wire_dtype == FX_BF16 || wire_dtype == FX_F16);
    const bool nvls_auto = nvls_ok && world >= (int)env_ll("FLASHY_B200_NVLS_MIN_WORLD", 4);
    if (algo == FX_ALGO_NVLS && !nvls_ok) { delete p; return fx_fail(FX_ERR_UNSUPPORTED, "NVLS handles fp32 / bf16 / fp16 buckets only"); }
    if (algo == FX_ALGO_AUTO) {
        if (dtype != FX_U8 && data_bytes <= one_shot_max) algo = FX_ALGO_ONE_SHOT;
        else if (nvls_auto && data_bytes >= nvls_min) algo = FX_ALGO_NVLS;
        else algo = FX_ALGO_TWO_SHOT;
    }
    if (dtype == FX_U8) algo = FX_ALGO_TWO_SHOT;            // broadcast uses the sharded layout
    p->algo = algo;
    const int shards = (algo == FX_ALGO_ONE_SHOT) ? 1 : world;
    const long long slice_align = FX_SLICE_ALIGN / (long long)wsize;
    const size_t slice_target = (size_t)env_ll("FLASHY_B200_SLICE_BYTES", 8 << 10);
    int max_blocks = c && !c->host_only ? c->max_blocks : 132;     // dry plans: one CTA per SM of an H100 SXM
    if (c && c->plan_blocks > 0 && c->plan_blocks < max_blocks) max_blocks = c->plan_blocks;
    const long long per_shard = std::max<long long>((cur + shards - 1) / shards, 1);
    long long grid = (long long)(((size_t)per_shard * wsize + slice_target - 1) / slice_target);
    grid = std::max<long long>(1, std::min<long long>(grid, max_blocks));
    p->grid_x = (int)grid;
    p->slice = ((per_shard + grid - 1) / grid + slice_align - 1) / slice_align * slice_align;
    p->shard = p->slice * grid;
    p->padded = p->shard * shards;
    p->wire_bytes = (size_t)p->padded * wsize;
    // Pipelined kernel (pack / reduce / gather as concurrent warp roles).  The per-tensor latency chains
    // of pack and unpack can hide behind the NVLink phase; when all ranks share one GPU the roles compete
    // for HBM instead.  The auto rule below (NVLS buckets of >= 8 tensors or >= 48 MiB, never with
    // virtual ranks) was tuned on an earlier target (B200) and is not yet re-measured on H100.
    // FLASHY_B200_PIPE: 0 never, 1 auto (default), 2 always.
    const long long pipe_mode = env_ll("FLASHY_B200_PIPE", 1);
    const bool pipe_able = algo != FX_ALGO_ONE_SHOT && dtype != FX_U8 &&
                           (wire_dtype == FX_F32 || wire_dtype == FX_BF16 || wire_dtype == FX_F16);
    // (on that target the roles starved each other on the peer-to-peer path, so auto mode pipelines NVLS buckets only)
    const bool pipe_auto = algo == FX_ALGO_NVLS && (n >= 8 || p->wire_bytes >= ((size_t)48 << 20)) && !(c && c->n_local > 1);
    if (pipe_able && (pipe_mode == 2 || (pipe_mode == 1 && pipe_auto))) {
        const long long chunk_target = env_ll("FLASHY_B200_CHUNK_BYTES", 4096) / (long long)wsize;
        long long chunks = std::max<long long>(1, std::min<long long>(env_ll("FLASHY_B200_MAX_CHUNKS", 8), p->slice / std::max<long long>(chunk_target, slice_align)));
        p->chunk = ((p->slice + chunks - 1) / chunks + slice_align - 1) / slice_align * slice_align;
        p->chunks = (int)((p->slice + p->chunk - 1) / p->chunk);
    }

    // Fused five-role kernel with TMA staging (fx_fuse.cu): float buckets reduced in their own dtype.
    // FLASHY_B200_FUSE: 0 never, 1 (default) whenever eligible.  One chunk = one reduce warp's batch.
    const bool fuse_able = algo != FX_ALGO_ONE_SHOT && dtype == wire_dtype &&
                           (wire_dtype == FX_F32 || wire_dtype == FX_BF16 || wire_dtype == FX_F16);
    if (fuse_able && env_ll("FLASHY_B200_FUSE", 1) != 0) {
        // one chunk = `world` sub-ranges of cbytes each; by default 32 KiB per chunk and CTA whatever the
        // world size (the staging buffers of the two copy roles then take 192 KiB of shared memory)
        long long cbytes = env_ll("FLASHY_B200_FUSE_CHUNK", (32 << 10) / world);
        cbytes = std::max<long long>(FX_SLICE_ALIGN, cbytes / FX_SLICE_ALIGN * FX_SLICE_ALIGN);
        while (cbytes > FX_SLICE_ALIGN && fx_fuse_smem_bytes(world, cbytes) > (size_t)(192 << 10)) cbytes -= FX_SLICE_ALIGN;
        if (fx_fuse_smem_bytes(world, cbytes) <= (size_t)(192 << 10)) {
            p->fuse_chunk = cbytes / (long long)wsize;
            // Multimem vectors in flight per lane.  A rank reduces N / W bytes, so the depth the links need shrinks
            // with the world.  The 1 / 2 / 4 defaults per world size were tuned on an earlier target (B200) and are
            // not yet re-measured on H100 (benchmarks/allreduce_sweep.py --variants compares them).
            const long long auto_depth = world >= 8 ? 1 : (world >= 4 ? 2 : 4);
            const long long depth = env_ll("FLASHY_B200_FUSE_DEPTH", auto_depth);
            p->fuse_unroll = (depth == 1 || depth == 2 || depth == 4 || depth == 8) ? (int)depth : (int)auto_depth;
            p->fuse_chunks = (int)((p->slice + p->fuse_chunk - 1) / p->fuse_chunk);
        }
    }

    if (c && !c->host_only) {
        std::lock_guard<std::mutex> lock(c->mu);
        const size_t need = round_up(p->wire_bytes, 256);
        bool got = false;
        for (size_t i = 0; i < c->free_regions.size(); ++i) {
            if (c->free_regions[i].second >= 2 * need) {
                p->region[0] = c->free_regions[i].first;
                p->region[1] = p->region[0] + need;
                c->free_regions[i].first += 2 * need;
                c->free_regions[i].second -= 2 * need;
                p->recycled = true;
                got = true;
                break;
            }
        }
        if (!got) {
            if (c->arena_used + 2 * need > c->arena_bytes) {
                const size_t wb = p->wire_bytes;
                delete p;
                return fx_fail(FX_ERR_TOO_BIG, "bucket of %zu wire bytes needs 2 x %zu arena bytes, %zu of %zu free",
                               wb, need, c->arena_bytes - c->arena_used, c->arena_bytes);
            }
            p->region[0] = c->arena_used;
            p->region[1] = c->arena_used + need;
            c->arena_used += 2 * need;
            if (p->region[0] < c->recycle_mark) p->recycled = true;   // memory an evicted plan used
        }
        p->region[0] += FX_PAD_BYTES;
        p->region[1] += FX_PAD_BYTES;
        if (p->algo == FX_ALGO_NVLS && p->region[1] + need > c->mc_bytes) p->algo = FX_ALGO_TWO_SHOT;   // outside the multicast window
        cudaError_t e = cudaSetDevice(c->device);
        std::vector<long long> table(p->off);
        table.insert(table.end(), p->numel.begin(), p->numel.end());
        const size_t nptr = (size_t)c->n_local * n;
        if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_off, table.size() * sizeof(long long));
        if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_in, nptr * sizeof(void*));
        if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_out, nptr * sizeof(void*));
        if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_state, c->n_local * sizeof(FxPlanState));
        if (e == cudaSuccess) e = cudaMemcpy(p->d_off, table.data(), table.size() * sizeof(long long), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemset(p->d_state, 0, c->n_local * sizeof(FxPlanState));
        if (e != cudaSuccess) {
            int rc = fx_fail(FX_ERR_CUDA, "plan device allocation failed: %s", cudaGetErrorString(e));
            cudaFree(p->d_off); cudaFree(p->d_in); cudaFree(p->d_out); cudaFree(p->d_state);
            delete p;
            return rc;
        }
        p->h_in.assign(nptr, nullptr);
        p->h_out.assign(nptr, nullptr);
    }
    *out = p;
    return FX_OK;
}

extern "C" int fx_plan_get_info(fx_plan* p, fx_plan_info* info) {
    if (!p || !info) return fx_fail(FX_ERR_INVALID, "NULL argument");
    memset(info, 0, sizeof(*info));
    info->n_tensors = p->n; info->dtype = p->dtype; info->wire_dtype = p->wire; info->world = p->world;
    info->algo = p->algo; info->grid_x = p->grid_x; info->block = FX_THREADS;
    info->total_elems = p->total; info->padded_elems = p->padded; info->shard_elems = p->shard;
    info->wire_bytes = p->wire_bytes;
    info->region_offset[0] = p->region[0]; info->region_offset[1] = p->region[1];
    info->signature = p->signature;
    info->kernel = fx_plan_kernel_id(p, FX_SUM);
    if (info->kernel == FX_KERNEL_FUSE_P2P || info->kernel == FX_KERNEL_FUSE_NVLS) {
        info->chunks = p->fuse_chunks; info->chunk_bytes = (uint64_t)p->fuse_chunk * p->wsize;
    } else if (info->kernel == FX_KERNEL_PIPE_P2P || info->kernel == FX_KERNEL_PIPE_NVLS) {
        info->chunks = p->chunks; info->chunk_bytes = (uint64_t)p->chunk * p->wsize;
    }
    return FX_OK;
}

extern "C" int fx_plan_offsets(fx_plan* p, int64_t* offsets) {
    if (!p || !offsets) return fx_fail(FX_ERR_INVALID, "NULL argument");
    for (int i = 0; i < p->n; ++i) offsets[i] = p->off[i];
    return FX_OK;
}

extern "C" void fx_plan_destroy(fx_plan* p) {
    if (!p) return;
    fx_comm* c = p->comm;
    if (c && !c->host_only) {
        std::lock_guard<std::mutex> lock(c->mu);
        cudaSetDevice(c->device);
        cudaFree(p->d_off); cudaFree(p->d_in); cudaFree(p->d_out); cudaFree(p->d_state);
        for (void* keep : p->capture_bufs) cudaFreeHost(keep);
        const size_t need = round_up(p->wire_bytes, 256);
        c->free_regions.push_back({p->region[0] - FX_PAD_BYTES, 2 * need});
        size_t freed = 0;
        for (auto& r : c->free_regions) freed += r.second;
        if (freed >= c->arena_used) {          // every plan is gone: restart the bump allocator
            c->recycle_mark = std::max(c->recycle_mark, c->arena_used);
            c->arena_used = 0;
            c->free_regions.clear();
        }
    }
    delete p;
}

// ============================================================================ launches
static void fill_launch(fx_comm* c, fx_plan* p, FxLaunch& a) {
    memset(&a, 0, sizeof(a));
    for (int r = 0; r < c->world; ++r) a.arena[r] = c->arena[r].base;
    a.mc_arena = c->mc_base;
    a.status = c->status_dev;
    a.timeout_ns = c->timeout_ns;
    a.trace = c->trace_dev;
    a.world = c->world; a.rank0 = c->rank0; a.n_local = c->n_local;
    if (p) {
        a.n = p->n; a.off = p->d_off;
        a.in_ptrs = (const void* const*)p->d_in; a.out_ptrs = (void* const*)p->d_out;
        a.state = p->d_state;
        a.region[0] = p->region[0]; a.region[1] = p->region[1];
        a.slice_elems = p->slice; a.shard_elems = p->shard;
        a.chunks = p->chunks; a.chunk_elems = p->chunk;
    }
}

// Upload a pointer table if it changed since the last launch.  The source must stay valid
// until the copy executes, so it goes through a small ring of pinned slots.
struct PinnedRing {
    static const int K = 8;
    void* slot[K] = {nullptr};
    size_t cap[K] = {0};
    cudaEvent_t ev[K] = {nullptr};
    int next = 0;
};

static std::mutex g_ring_mu;
static PinnedRing g_ring;

static int upload_ptrs(fx_plan* p, void** dst, std::vector<const void*>* shadow_c, std::vector<void*>* shadow_m,
                       const void* const* src, size_t nptr, bool* valid, cudaStream_t stream) {
    const size_t bytes = nptr * sizeof(void*);
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess) { cudaGetLastError(); cap = cudaStreamCaptureStatusNone; }
    if (cap != cudaStreamCaptureStatusNone) {
        // Inside a stream capture the copy becomes a graph node that re-reads its host source at every
        // replay: the source must live as long as the plan, not in the recycled ring.  A replayed graph
        // rewrites the device table behind the shadow's back, so a captured plan uploads on every call.
        void* keep = nullptr;
        cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;      // an allocation is "unsafe" under global capture
        FX_CUDA(cudaThreadExchangeStreamCaptureMode(&mode));
        const cudaError_t ae = cudaHostAlloc(&keep, round_up(bytes, 256), cudaHostAllocPortable);
        cudaThreadExchangeStreamCaptureMode(&mode);
        if (ae != cudaSuccess) return fx_fail(FX_ERR_CUDA, "pinned pointer table for a captured launch: %s", cudaGetErrorString(ae));
        p->capture_bufs.push_back(keep);
        memcpy(keep, src, bytes);
        FX_CUDA(cudaMemcpyAsync(dst, keep, bytes, cudaMemcpyHostToDevice, stream));
        p->captured = true;
        *valid = false;
        return FX_OK;
    }
    const void* const* cur = shadow_c ? shadow_c->data() : (const void* const*)shadow_m->data();
    if (*valid && !p->captured && memcmp(cur, src, bytes) == 0) return FX_OK;
    std::lock_guard<std::mutex> lock(g_ring_mu);
    const int k = g_ring.next;
    g_ring.next = (k + 1) % PinnedRing::K;
    if (!g_ring.ev[k]) FX_CUDA(cudaEventCreateWithFlags(&g_ring.ev[k], cudaEventDisableTiming));
    else FX_CUDA(cudaEventSynchronize(g_ring.ev[k]));
    if (g_ring.cap[k] < bytes) {
        if (g_ring.slot[k]) cudaFreeHost(g_ring.slot[k]);
        g_ring.slot[k] = nullptr; g_ring.cap[k] = 0;
        FX_CUDA(cudaHostAlloc(&g_ring.slot[k], round_up(bytes, 4096), cudaHostAllocPortable));
        g_ring.cap[k] = round_up(bytes, 4096);
    }
    memcpy(g_ring.slot[k], src, bytes);
    FX_CUDA(cudaMemcpyAsync(dst, g_ring.slot[k], bytes, cudaMemcpyHostToDevice, stream));
    FX_CUDA(cudaEventRecord(g_ring.ev[k], stream));
    if (shadow_c) memcpy(shadow_c->data(), src, bytes); else memcpy(shadow_m->data(), src, bytes);
    *valid = true;
    return FX_OK;
}

// All collective kernels of a communicator share one signal pad (flags, epochs), so two of them
// must never be in flight at once.  Launches on ONE stream are ordered by the stream; when the
// launch stream changes (eager buckets on the side stream, then a collective on the user's stream)
// the new stream is made to wait for everything the previous launch stream holds.  Inside a stream
// capture the caller orders the launches itself (fork / join of the side stream).
static int order_after_previous(fx_comm* c, cudaStream_t stream) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(stream, &cap) != cudaSuccess) { cudaGetLastError(); return FX_OK; }
    if (cap != cudaStreamCaptureStatusNone) return FX_OK;
    if (c->have_last && c->last_stream != (void*)stream) {
        cudaStream_t prev = static_cast<cudaStream_t>(c->last_stream);
        cudaStreamCaptureStatus pcap = cudaStreamCaptureStatusNone;
        if (cudaStreamIsCapturing(prev, &pcap) != cudaSuccess || pcap != cudaStreamCaptureStatusNone) {
            cudaGetLastError();
        } else {
            if (!c->order_event) FX_CUDA(cudaEventCreateWithFlags(&c->order_event, cudaEventDisableTiming));
            if (cudaEventRecord(c->order_event, prev) == cudaSuccess) FX_CUDA(cudaStreamWaitEvent(stream, c->order_event, 0));
            else cudaGetLastError();                       // the previous stream no longer exists
        }
    }
    c->last_stream = (void*)stream;
    c->have_last = true;
    return FX_OK;
}

static int pre_launch(fx_comm* c, fx_plan* p, cudaStream_t stream) {
    if (!c || c->host_only) return fx_fail(FX_ERR_STATE, "this communicator has no device side");
    if (!c->connected) return fx_fail(FX_ERR_STATE, "communicator is not connected yet");
    int rc = fx_comm_poll(c);
    if (rc != FX_OK) return rc;
    FX_CUDA(cudaSetDevice(c->device));
    if ((rc = order_after_previous(c, stream)) != FX_OK) return rc;
    if (p && p->recycled) {          // its arena region was used by a destroyed plan: fence the old readers
        FxLaunch a;
        fill_launch(c, nullptr, a);
        rc = fx_launch_barrier(c, a, stream);
        if (rc != FX_OK) return rc;
        c->launches++;
        p->recycled = false;
    }
    return FX_OK;
}

extern "C" int fx_allreduce(fx_plan* p, int op, const void* const* in_ptrs, void* const* out_ptrs, void* stream) {
    if (!p || !in_ptrs || !out_ptrs) return fx_fail(FX_ERR_INVALID, "NULL argument");
    fx_comm* c = p->comm;
    if (!c) return fx_fail(FX_ERR_STATE, "dry plan cannot be launched");
    if (!fx_kernel_supported(p->dtype, p->wire, op, false)) return fx_fail(FX_ERR_UNSUPPORTED, "all-reduce op %d on dtype %d is not supported", op, p->dtype);
    std::lock_guard<std::mutex> lock(c->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = pre_launch(c, p, s);
    if (rc != FX_OK) return rc;
    const size_t nptr = (size_t)c->n_local * p->n;
    if ((rc = upload_ptrs(p, p->d_in, &p->h_in, nullptr, in_ptrs, nptr, &p->in_valid, s)) != FX_OK) return rc;
    if ((rc = upload_ptrs(p, p->d_out, nullptr, &p->h_out, (const void* const*)out_ptrs, nptr, &p->out_valid, s)) != FX_OK) return rc;
    FxLaunch a;
    fill_launch(c, p, a);
    a.op = op; a.mode = FX_MODE_FUSED;
    const int kid = fx_plan_kernel_id(p, op);
    if (kid == FX_KERNEL_FUSE_P2P || kid == FX_KERNEL_FUSE_NVLS) {
        a.chunks = p->fuse_chunks; a.chunk_elems = p->fuse_chunk;
        rc = fx_launch_fuse(p, a, s);
    } else {
        rc = fx_launch_allreduce(p, a, s);
    }
    if (rc == FX_OK) c->launches++;
    return rc;
}

int fx_plan_kernel_id(const fx_plan* p, int op) {
    const bool sum = op == FX_SUM || op == FX_AVG;
    if (p->algo == FX_ALGO_ONE_SHOT) return FX_KERNEL_ONE_SHOT;
    const bool nvls = p->algo == FX_ALGO_NVLS && sum;
    if (sum && p->fuse_chunks > 0) return nvls ? FX_KERNEL_FUSE_NVLS : FX_KERNEL_FUSE_P2P;
    const bool pipe_ok = p->wire == FX_F32 || p->wire == FX_BF16 || p->wire == FX_F16;
    if (sum && p->chunks > 0 && pipe_ok) return nvls ? FX_KERNEL_PIPE_NVLS : FX_KERNEL_PIPE_P2P;
    return nvls ? FX_KERNEL_NVLS : FX_KERNEL_TWO_SHOT;
}

extern "C" int fx_allreduce_begin(fx_plan* p, int op, const void* const* in_ptrs, void* stream) {
    if (!p || !in_ptrs) return fx_fail(FX_ERR_INVALID, "NULL argument");
    fx_comm* c = p->comm;
    if (!c) return fx_fail(FX_ERR_STATE, "dry plan cannot be launched");
    if (p->algo == FX_ALGO_ONE_SHOT) return fx_fail(FX_ERR_INVALID, "begin/finish needs a sharded (TWO_SHOT / NVLS) plan");
    if (p->begun) return fx_fail(FX_ERR_STATE, "fx_allreduce_begin on a plan whose previous begin has no matching finish yet "
                                               "(a plan owns one pair of staging regions: use one plan per bucket in flight)");
    if (!fx_kernel_supported(p->dtype, p->wire, op, false)) return fx_fail(FX_ERR_UNSUPPORTED, "all-reduce op %d on dtype %d is not supported", op, p->dtype);
    std::lock_guard<std::mutex> lock(c->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = pre_launch(c, p, s);
    if (rc != FX_OK) return rc;
    const size_t nptr = (size_t)c->n_local * p->n;
    if ((rc = upload_ptrs(p, p->d_in, &p->h_in, nullptr, in_ptrs, nptr, &p->in_valid, s)) != FX_OK) return rc;
    FxLaunch a;
    fill_launch(c, p, a);
    a.op = op; a.mode = FX_MODE_BEGIN;
    rc = fx_launch_allreduce(p, a, s);
    if (rc == FX_OK) { c->launches++; p->begun = true; }
    return rc;
}

extern "C" int fx_allreduce_finish(fx_plan* p, void* const* out_ptrs, void* stream) {
    if (!p || !out_ptrs) return fx_fail(FX_ERR_INVALID, "NULL argument");
    fx_comm* c = p->comm;
    if (!c) return fx_fail(FX_ERR_STATE, "dry plan cannot be launched");
    if (!p->begun) return fx_fail(FX_ERR_STATE, "fx_allreduce_finish without a matching fx_allreduce_begin");
    std::lock_guard<std::mutex> lock(c->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    FX_CUDA(cudaSetDevice(c->device));
    const size_t nptr = (size_t)c->n_local * p->n;
    int rc;
    if ((rc = upload_ptrs(p, p->d_out, nullptr, &p->h_out, (const void* const*)out_ptrs, nptr, &p->out_valid, s)) != FX_OK) return rc;
    FxLaunch a;
    fill_launch(c, p, a);
    rc = fx_launch_unpack(p, a, s);
    if (rc == FX_OK) { c->launches++; p->begun = false; }
    return rc;
}

extern "C" int fx_broadcast(fx_plan* p, int src, void* const* ptrs, void* stream) {
    if (!p || !ptrs) return fx_fail(FX_ERR_INVALID, "NULL argument");
    fx_comm* c = p->comm;
    if (!c) return fx_fail(FX_ERR_STATE, "dry plan cannot be launched");
    if (p->dtype != FX_U8) return fx_fail(FX_ERR_INVALID, "broadcast plans are byte plans (dtype FX_U8)");
    if (src < 0 || src >= c->world) return fx_fail(FX_ERR_INVALID, "broadcast source %d out of range", src);
    std::lock_guard<std::mutex> lock(c->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = pre_launch(c, p, s);
    if (rc != FX_OK) return rc;
    const size_t nptr = (size_t)c->n_local * p->n;
    if ((rc = upload_ptrs(p, p->d_in, &p->h_in, nullptr, (const void* const*)ptrs, nptr, &p->in_valid, s)) != FX_OK) return rc;
    if ((rc = upload_ptrs(p, p->d_out, nullptr, &p->h_out, (const void* const*)ptrs, nptr, &p->out_valid, s)) != FX_OK) return rc;
    FxLaunch a;
    fill_launch(c, p, a);
    a.src = src;
    rc = fx_launch_broadcast(p, a, s);
    if (rc == FX_OK) c->launches++;
    return rc;
}

extern "C" int fx_barrier(fx_comm* c, void* stream) {
    if (!c) return fx_fail(FX_ERR_INVALID, "comm is NULL");
    std::lock_guard<std::mutex> lock(c->mu);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    int rc = pre_launch(c, nullptr, s);
    if (rc != FX_OK) return rc;
    FxLaunch a;
    fill_launch(c, nullptr, a);
    rc = fx_launch_barrier(c, a, s);
    if (rc == FX_OK) c->launches++;
    return rc;
}
