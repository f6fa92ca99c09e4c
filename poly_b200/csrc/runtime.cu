// runtime.cu -- the device runtime under the C ABI of libpolyb200.so (include/poly_b200.h): error and launch
// bookkeeping, one context per CUDA device and device selection, and the entry points that belong to no
// package (devices, memory, copies, IPC, synthetic reads).  The packages' entry points are the api_*.cu files.
// No compute happens on the host: when no sm_90 device is usable every compute entry point fails with
// PG_ERR_NO_DEVICE.
#include <algorithm>
#include <cctype>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "runtime.cuh"

namespace pg {

static thread_local char t_err[512] = "";
static thread_local const char *t_last_kernel = "";
static std::atomic<uint64_t> g_launches{0};
static DevCtx g_ctx[MAX_DEVICES];
static std::mutex g_init_mu;                 // context creation / default-device changes
static std::atomic<int> g_default_device{-1};  // process default (pg_init), -1: not chosen yet
static thread_local int t_bound_device = -1;   // pg_thread_device override for this thread
static thread_local DevCtx *t_ctx = nullptr;   // context the current entry point runs on

DevCtx *cur_ctx() { return t_ctx; }
void bind_thread_device(int device) { t_bound_device = device; }

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(t_err, sizeof t_err, fmt, ap);
    va_end(ap);
}
int cuda_fail(cudaError_t e, const char *what, const char *file, int line) {
    set_error("CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e), file, line, what);
    return PG_ERR_CUDA;
}
void note_launch(const char *name) {
    t_last_kernel = name;
    g_launches.fetch_add(1, std::memory_order_relaxed);
}
int sm_count() { return t_ctx && t_ctx->sms > 0 ? t_ctx->sms : 132; }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (device, kernel, size class): function
// attributes live in the device's context, so the cache is per device and lock-protected (several
// host threads may drive the same device through the *_dev entry points).
int func_smem(const void *fn, size_t bytes) {
    DevCtx *c = t_ctx;
    if (!c) { set_error("internal: no device context bound"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(c->fmu);
    size_t &cur = c->func_smem[fn];
    if (bytes > cur) {
        PG_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        cur = bytes;
    }
    return PG_OK;
}

int resident_blocks(const void *fn, int threads, size_t smem, uint64_t work, uint64_t *blocks) {
    { const int rc_ = func_smem(fn, smem); if (rc_ != PG_OK) return rc_; }
    int per_sm = 0;
    PG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem));
    *blocks = std::min<uint64_t>(work, (uint64_t)sm_count() * std::max(per_sm, 1));
    return PG_OK;
}

int host_row_starts(const uint64_t *d_offsets, uint64_t n_reads, cudaStream_t st, std::vector<uint64_t> &off) {
    off.resize(n_reads + 1);
    PG_CUDA(cudaMemcpyAsync(off.data(), d_offsets, (n_reads + 1) * 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// create (once) the context of `device`; g_init_mu held
static int ctx_create_locked(int device) {
    DevCtx &c = g_ctx[device];
    if (c.ready.load(std::memory_order_acquire)) return PG_OK;
    cudaDeviceProp prop;
    PG_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error("device %d is sm_%d%d; libpolyb200 is built for sm_90a only", device, prop.major, prop.minor);
        return PG_ERR_NO_DEVICE;
    }
    PG_CUDA(cudaSetDevice(device));
    for (Slot &sl : c.slots)
        if (!sl.stream) PG_CUDA(cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking));
    {   // Stream-ordered temporaries (cudaMallocAsync) are freed at the end of every call and most calls
        // synchronise: with the default release threshold of 0 the pool would hand its memory back to the
        // driver each time.  Keep up to 12 GiB cached (the 8 GiB pair tiles of the sparse distance path included) so that small calls do not pay a driver allocation.
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
            uint64_t keep = 12ull << 30, cur = 0;
            if (cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &cur) == cudaSuccess && cur < keep)
                cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
        cudaGetLastError();
    }
    c.device = device;
    c.sms = prop.multiProcessorCount;
    c.ready.store(true, std::memory_order_release);
    return PG_OK;
}

int device_count_checked(int *n) {
    cudaError_t e = cudaGetDeviceCount(n);
    if (e != cudaSuccess || *n == 0) {
        set_error("no CUDA device available (%s); libpolyb200 has no CPU fallback",
                  e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
        cudaGetLastError();
        return PG_ERR_NO_DEVICE;
    }
    if (*n > MAX_DEVICES) *n = MAX_DEVICES;
    return PG_OK;
}

// make `device` usable and current on the calling thread; t_ctx = its context
int use_device(int device) {
    int n = 0, rc = device_count_checked(&n);
    if (rc != PG_OK) return rc;
    if (device < 0 || device >= n) {
        set_error("device %d out of range (count %d)", device, n);
        return PG_ERR_ARG;
    }
    if (!g_ctx[device].ready.load(std::memory_order_acquire)) {
        std::lock_guard<std::mutex> lk(g_init_mu);
        if ((rc = ctx_create_locked(device)) != PG_OK) return rc;
    }
    PG_CUDA(cudaSetDevice(device));
    t_ctx = &g_ctx[device];
    return PG_OK;
}

// every entry point: the thread's bound device (pg_thread_device), else the process default
// (pg_init), else the current CUDA device / device 0
int ensure_device() {
    int device = t_bound_device;
    if (device < 0) device = g_default_device.load(std::memory_order_acquire);
    if (device < 0) {
        int n = 0, rc = device_count_checked(&n);
        if (rc != PG_OK) return rc;
        std::lock_guard<std::mutex> lk(g_init_mu);
        device = g_default_device.load();
        if (device < 0) {
            if (cudaGetDevice(&device) != cudaSuccess || device >= n) device = 0;
            if ((rc = ctx_create_locked(device)) != PG_OK) return rc;
            g_default_device.store(device, std::memory_order_release);
        }
    }
    return use_device(device);
}

uint64_t group_budget(uint64_t default_bytes) {
    if (const char *e = getenv("PG_GROUP_BYTES")) return std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    return default_bytes;
}

}  // namespace pg

using namespace pg;

extern "C" {

int pg_version(void) { return 100; }

int pg_init(int device) {
    if (device < 0) {
        g_default_device.store(-1);
        return ensure_device();
    }
    int rc = use_device(device);
    if (rc == PG_OK) g_default_device.store(device, std::memory_order_release);
    return rc;
}

int pg_thread_device(int device) {
    if (device < 0) { t_bound_device = -1; return PG_OK; }
    int rc = use_device(device);
    if (rc == PG_OK) t_bound_device = device;
    return rc;
}

int pg_shutdown(void) {
    std::lock_guard<std::mutex> lk(g_init_mu);
    for (int d = 0; d < MAX_DEVICES; ++d) {
        DevCtx &c = g_ctx[d];
        if (!c.ready.load()) continue;
        std::lock_guard<std::mutex> lk2(c.mu);
        cudaSetDevice(d);
        cudaDeviceSynchronize();
        for (Slot &sl : c.slots) sl.release();
        c.pool.stop();
        {
            std::lock_guard<std::mutex> lk3(c.fmu);
            c.func_smem.clear();
        }
        c.ready.store(false);
    }
    g_default_device.store(-1);
    t_ctx = nullptr;
    return PG_OK;
}

const char *pg_last_error(void) { return t_err; }
const char *pg_last_kernel(void) { return t_last_kernel; }
uint64_t pg_launch_count(void) { return g_launches.load(); }

int pg_device_count(int *count) {
    if (!count) return PG_ERR_ARG;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); n = 0; }
    *count = n;
    return PG_OK;
}
int pg_device_sm_count(int *sms) {
    if (!sms) return PG_ERR_ARG;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    *sms = t_ctx->sms;
    return PG_OK;
}

// Put the calling thread on the CPUs of the NUMA node `device` hangs off, and prefer that node for
// the pages it allocates from now on (pinned buffers included): PCIe traffic of 8 GPUs otherwise
// funnels through one socket's memory controllers / the inter-socket link.  Best effort: every
// failure (no sysfs, container without the syscall, single-node host) leaves the thread as it was.
int pg_numa_bind_thread(int device, int *node_out) {
    if (node_out) *node_out = -1;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) { cudaGetLastError(); set_error("device %d out of range", device); return PG_ERR_ARG; }
    char bus[64] = "";
    if (cudaDeviceGetPCIBusId(bus, (int)sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return PG_OK; }
    for (char *c = bus; *c; ++c) *c = (char)tolower((unsigned char)*c);
    char path[256];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    int node = -1;
    if (FILE *f = fopen(path, "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
    if (node < 0) return PG_OK;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    cpu_set_t want, cur, both;
    CPU_ZERO(&want);
    if (FILE *f = fopen(path, "r")) {
        int a, b;
        for (;;) {
            if (fscanf(f, "%d", &a) != 1) break;
            b = a;
            int ch = fgetc(f);
            if (ch == '-') { if (fscanf(f, "%d", &b) != 1) break; ch = fgetc(f); }
            for (int c = a; c <= b && c < CPU_SETSIZE; ++c) CPU_SET(c, &want);
            if (ch != ',') break;
        }
        fclose(f);
    }
    if (sched_getaffinity(0, sizeof cur, &cur) == 0) {
        CPU_AND(&both, &cur, &want);
        if (CPU_COUNT(&both) > 0) sched_setaffinity(0, sizeof both, &both);
    }
#ifdef SYS_set_mempolicy
    if (node < 1024) {
        unsigned long mask[16] = {0};
        mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
        (void)syscall(SYS_set_mempolicy, 1 /* MPOL_PREFERRED */, mask, (unsigned long)(sizeof mask * 8));
    }
#endif
    if (node_out) *node_out = node;
    return PG_OK;
}

int pg_host_alloc(void **ptr, size_t bytes) {
    if (!ptr) return PG_ERR_ARG;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    // portable: pinned for every device context of the process (the *_multi entry points)
    PG_CUDA(cudaHostAlloc(ptr, bytes ? bytes : 1, cudaHostAllocPortable));
    return PG_OK;
}
int pg_host_free(void *ptr) {
    if (ptr) PG_CUDA(cudaFreeHost(ptr));
    return PG_OK;
}
int pg_dev_alloc(void **dptr, size_t bytes) {
    if (!dptr) return PG_ERR_ARG;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    PG_CUDA(cudaMalloc(dptr, bytes ? bytes : 1));
    return PG_OK;
}
int pg_dev_free(void *dptr) {
    if (dptr) PG_CUDA(cudaFree(dptr));
    return PG_OK;
}
int pg_memcpy_h2d(void *dst, const void *src, size_t bytes, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    PG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream));
    return PG_OK;
}
int pg_memcpy_d2h(void *dst, const void *src, size_t bytes, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    PG_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    return PG_OK;
}
int pg_stream_sync(void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    PG_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return PG_OK;
}

int pg_ipc_export(void *dptr, uint8_t handle[PG_IPC_HANDLE_BYTES]) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    static_assert(sizeof(cudaIpcMemHandle_t) == PG_IPC_HANDLE_BYTES, "handle size");
    cudaIpcMemHandle_t h;
    PG_CUDA(cudaIpcGetMemHandle(&h, dptr));
    memcpy(handle, &h, sizeof h);
    return PG_OK;
}
int pg_ipc_import(const uint8_t handle[PG_IPC_HANDLE_BYTES], void **dptr) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    PG_CUDA(cudaIpcOpenMemHandle(dptr, h, cudaIpcMemLazyEnablePeerAccess));
    return PG_OK;
}
int pg_ipc_close(void *dptr) {
    if (dptr) PG_CUDA(cudaIpcCloseMemHandle(dptr));
    return PG_OK;
}

int pg_synth_reads_dev(uint8_t *d_bases, uint64_t first_read, uint64_t n_reads, uint32_t read_len,
                       uint64_t seed, int32_t kind, uint32_t family, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return launch_synth_reads(d_bases, first_read, n_reads, read_len, seed, kind, family, (cudaStream_t)stream);
}

}  // extern "C"
