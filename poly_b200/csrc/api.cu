// api.cu -- the C ABI of libpolyb200.so (include/poly_b200.h): argument checking,
// device selection, host<->device staging for the host-pointer entry points, and
// dispatch to the kernel launchers.  No compute happens on the host: when no sm_90
// device is usable every compute entry point fails with PG_ERR_NO_DEVICE.
#include <algorithm>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <cctype>
#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <string>
#include <vector>

#include "align_core.cuh"
#include "clone.cuh"
#include "common.cuh"

namespace pg {

static thread_local char t_err[512] = "";
static thread_local const char *t_last_kernel = "";
static std::atomic<uint64_t> g_launches{0};

// Grow-only buffer of the pipelined host path (under the context's mutex): device memory, or portable
// pinned host memory for staging pageable caller buffers.
template <bool Pinned>
struct GrowBuf {
    void *p = nullptr;
    size_t cap = 0;
    int reserve(size_t bytes) {
        if (bytes <= cap) return PG_OK;
        release();
        cudaError_t e = Pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocPortable) : cudaMalloc(&p, bytes);
        if (e != cudaSuccess) {
            p = nullptr;
            set_error("%s(%zu) failed: %s", Pinned ? "cudaHostAlloc" : "cudaMalloc", bytes, cudaGetErrorString(e));
            cudaGetLastError();
            return PG_ERR_NOMEM;
        }
        cap = bytes;
        return PG_OK;
    }
    void release() {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

// Fork-join helper threads for host-side copies between pageable caller memory and the pinned
// staging buffers: one memcpy thread moves ~10 GB/s, PCIe 5 x16 moves 55.
class CopyPool {
    std::vector<std::thread> workers_;
    std::mutex mu_;
    std::condition_variable cv_work_, cv_done_;
    const std::function<void(int)> *fn_ = nullptr;
    int parts_ = 0, next_ = 0, pending_ = 0;
    bool stop_ = false;

    void drain_parts(std::unique_lock<std::mutex> &lk) {
        while (fn_ && next_ < parts_) {
            const int i = next_++;
            const std::function<void(int)> *f = fn_;
            lk.unlock();
            (*f)(i);
            lk.lock();
            if (--pending_ == 0) cv_done_.notify_all();
        }
    }

public:
    CopyPool() = default;
    CopyPool(const CopyPool &) = delete;
    CopyPool &operator=(const CopyPool &) = delete;
    ~CopyPool() { stop(); }  // contexts are statics: joinable threads at exit would call std::terminate
    int threads() const { return (int)workers_.size() + 1; }
    void start(int helpers, int device) {
        if (!workers_.empty() || helpers <= 0) return;
        for (int t = 0; t < helpers; ++t)
            workers_.emplace_back([this, device] {
                pg_numa_bind_thread(device, nullptr);  // copies run next to the GPU's PCIe root
                std::unique_lock<std::mutex> lk(mu_);
                for (;;) {
                    cv_work_.wait(lk, [&] { return stop_ || (fn_ && next_ < parts_); });
                    if (stop_) return;
                    drain_parts(lk);
                }
            });
    }
    // f(0) .. f(parts-1), each exactly once, on the helpers and the calling thread; returns when all are done
    void run(int parts, const std::function<void(int)> &f) {
        if (parts <= 0) return;
        std::unique_lock<std::mutex> lk(mu_);
        fn_ = &f; parts_ = parts; next_ = 0; pending_ = parts;
        cv_work_.notify_all();
        drain_parts(lk);
        cv_done_.wait(lk, [&] { return pending_ == 0; });
        fn_ = nullptr;
    }
    void stop() {
        {
            std::lock_guard<std::mutex> lk(mu_);
            stop_ = true;
        }
        cv_work_.notify_all();
        for (std::thread &t : workers_) t.join();
        workers_.clear();
        stop_ = false;
    }
};

// One context per CUDA device of the process.  The library serves any number of devices from one
// process (pg_*_multi shard a batch over them; pg_thread_device binds a thread to one) as well as
// the one-process-per-GPU layout (pg_init(device) picks the process default).
constexpr int MAX_DEVICES = 32;
constexpr int N_SLOTS = 3;  // stream/buffer slots of the pipelined host path

// One stream/buffer slot of the pipelined host path and the chunk it has in flight.  Slot 0's stream
// also serves the one-shot host-pointer entry points.
struct Slot {
    cudaStream_t stream = nullptr;
    GrowBuf<false> in, out, aux, st;  // device: input bytes, rows, offsets + counts, statuses
    GrowBuf<true> pin_in, pin_out;    // pinned staging of pageable caller buffers
    uint64_t r0 = 0, nr = 0, dstride = 0;  // in flight: rows [r0, r0 + nr), dstride words per device row
    bool used = false;
    std::vector<int32_t> status;  // the chunk's statuses, copied back on the stream
    void release() {
        in.release(); out.release(); aux.release(); st.release();
        pin_in.release(); pin_out.release();
        if (stream) cudaStreamDestroy(stream);
        stream = nullptr;
    }
};

struct DevCtx {
    int device = -1;
    int sms = 0;
    std::atomic<bool> ready{false};
    Slot slots[N_SLOTS];
    CopyPool pool;
    std::mutex mu;   // serialises the host-pointer entry points on this device
    std::mutex fmu;  // guards func_smem
    std::unordered_map<const void *, size_t> func_smem;  // largest dynamic smem configured per kernel
};
static DevCtx g_ctx[MAX_DEVICES];
static std::mutex g_init_mu;                 // context creation / default-device changes
static std::atomic<int> g_default_device{-1};  // process default (pg_init), -1: not chosen yet
static thread_local int t_bound_device = -1;   // pg_thread_device override for this thread
static thread_local DevCtx *t_ctx = nullptr;   // context the current entry point runs on

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

static int device_count_checked(int *n) {
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
static int use_device(int device) {
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
static int ensure_device() {
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

static inline uint64_t kmers_of(uint64_t len, int k) { return len > (uint64_t)k ? len - (uint64_t)k : 0; }
// informative words of the sketch of a read of `len` bytes
static inline uint64_t sketch_words(uint64_t len, int k, int s) { return std::min<uint64_t>(kmers_of(len, k), (uint64_t)s); }

}  // namespace pg

// Staging for the one-shot host-pointer entry points: every step of such a call goes through a HostCall.
namespace pg {
namespace {
// `count` elements of T from `tmp`, at least 16 bytes
template <typename T>
int scratch_alloc(StreamScratch &tmp, T **p, uint64_t count) {
    const uint64_t bytes = count * sizeof(T);
    uint8_t *b = nullptr;
    cudaError_t e = tmp.alloc(&b, std::max<uint64_t>(bytes, 16));
    if (e != cudaSuccess) { set_error("cudaMallocAsync(%zu): %s", (size_t)bytes, cudaGetErrorString(e)); cudaGetLastError(); return PG_ERR_NOMEM; }
    *p = (T *)b;
    return PG_OK;
}

// Host ragged batches: item i is [offsets[i], offsets[i+1]) and offsets never decrease (a decrease would
// hand a kernel a length near 2^64).  *max_len = the longest item.
int check_ragged(const uint64_t *offsets, uint64_t n, uint64_t *max_len) {
    uint64_t m = 0;
    for (uint64_t i = 0; i < n; ++i) {
        if (offsets[i + 1] < offsets[i]) { set_error("offsets decrease at %llu", (unsigned long long)i); return PG_ERR_ARG; }
        m = std::max(m, offsets[i + 1] - offsets[i]);
    }
    *max_len = m;
    return PG_OK;
}

// a ragged batch on the device: item i is base[off[i] .. off[i+1]) with the caller's own offsets
template <typename T>
struct Ragged {
    const T *base;
    const uint64_t *off;
    uint64_t max_len;
};

// One call of a host-pointer entry point on the current device: holds the device's lock, runs on its
// first stream and owns the call's device temporaries.  The first error sticks: later steps do nothing
// and finish() returns it.  Unless finish() ran, the destructor waits for the stream, so that no copy
// into or out of the caller's memory is still running when the entry point returns.
class HostCall {
    std::lock_guard<std::mutex> lock_;
    StreamScratch tmp_;
    int rc_ = PG_OK;
    bool finished_ = false;
    void copy(void *dst, const void *src, uint64_t bytes, cudaMemcpyKind kind) {
        if (rc_ != PG_OK) return;
        cudaError_t e = cudaMemcpyAsync(dst, src, bytes, kind, st);
        if (e != cudaSuccess) rc_ = cuda_fail(e, "cudaMemcpyAsync", __FILE__, __LINE__);
    }

public:
    const cudaStream_t st;
    HostCall() : lock_(t_ctx->mu), tmp_(t_ctx->slots[0].stream), st(t_ctx->slots[0].stream) {}
    ~HostCall() {
        if (finished_) return;
        cudaStreamSynchronize(st);
        cudaGetLastError();
    }
    int error() const { return rc_; }
    // nullptr once an error has occurred
    template <typename T>
    T *alloc(uint64_t count, bool zero = false) {
        T *p = nullptr;
        if (rc_ != PG_OK || (rc_ = scratch_alloc(tmp_, &p, count)) != PG_OK) return nullptr;
        if (zero) {
            cudaError_t e = cudaMemsetAsync(p, 0, count * sizeof(T), st);
            if (e != cudaSuccess) { rc_ = cuda_fail(e, "cudaMemsetAsync", __FILE__, __LINE__); return nullptr; }
        }
        return p;
    }
    // h[0 .. count) on the device, in a buffer with room for `extra` more elements
    template <typename T>
    T *upload(const T *h, uint64_t count, uint64_t extra = 0) {
        T *d = alloc<T>(count + extra);
        if (count) copy(d, h, count * sizeof(T), cudaMemcpyHostToDevice);
        return rc_ == PG_OK ? d : nullptr;
    }
    // h[0 .. count) into the device buffer d
    template <typename T>
    void put(T *d, const T *h, uint64_t count) {
        if (count) copy(d, h, count * sizeof(T), cudaMemcpyHostToDevice);
    }
    template <typename T>
    void download(T *h, const T *d, uint64_t count) {
        if (h && count) copy(h, d, count * sizeof(T), cudaMemcpyDeviceToHost);
    }
    // check_ragged, then items [offsets[0], offsets[n]) and the n + 1 offsets to the device
    template <typename T>
    Ragged<T> ragged(const T *items, const uint64_t *offsets, uint64_t n) {
        Ragged<T> r{nullptr, nullptr, 0};
        if (rc_ != PG_OK || (rc_ = check_ragged(offsets, n, &r.max_len)) != PG_OK) return r;
        const uint64_t b0 = offsets[0];
        const T *d = upload(items + b0, offsets[n] - b0);
        r.off = upload(offsets, n + 1);
        if (rc_ == PG_OK) r.base = d - b0;  // the kernels index with the absolute offsets
        return r;
    }
    int sync() {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess && rc_ == PG_OK) rc_ = cuda_fail(e, "cudaStreamSynchronize", __FILE__, __LINE__);
        return rc_;
    }
    int finish() {
        finished_ = true;
        return sync();
    }
};

// Per-item statuses -> `status` (may be NULL) and the call's code: PG_ERR_PANIC if any item panics, else
// PG_ERR_UNSUPPORTED if any is unsupported, with that code's message
int fold_item_status(const std::vector<int32_t> &hst, int32_t *status, const char *panic_msg, const char *unsupported_msg) {
    int worst = PG_OK;
    for (size_t i = 0; i < hst.size(); ++i) {
        if (status) status[i] = hst[i];
        if (hst[i] == PG_ITEM_PANIC) worst = PG_ERR_PANIC;
        else if (hst[i] == PG_ITEM_UNSUPPORTED && worst == PG_OK) worst = PG_ERR_UNSUPPORTED;
    }
    if (worst == PG_ERR_PANIC) set_error("%s", panic_msg);
    if (worst == PG_ERR_UNSUPPORTED) set_error("%s", unsupported_msg);
    return worst;
}

// a device output list whose first entries come back to the caller's array
struct CappedList {
    void *host;
    const void *dev;
    size_t elem_bytes;
};

// Ends a call whose kernel stored its entry count at d_n: *n_out = that count, and the first min(count, cap)
// entries of every list come back.  More entries than cap is PG_ERR_ARG.
int finish_capped(HostCall &c, const unsigned long long *d_n, uint64_t cap, uint64_t *n_out, std::initializer_list<CappedList> lists,
                  const char *cap_name, const char *entries) {
    unsigned long long found = 0;
    c.download(&found, d_n, 1);
    int rc = c.sync();
    if (rc != PG_OK) return rc;
    *n_out = found;
    const uint64_t kept = std::min<uint64_t>(found, cap);
    for (const CappedList &l : lists) c.download((uint8_t *)l.host, (const uint8_t *)l.dev, kept * l.elem_bytes);
    if ((rc = c.finish()) != PG_OK) return rc;
    if (found > cap) { set_error("%s %llu < %llu %s", cap_name, (unsigned long long)cap, found, entries); return PG_ERR_ARG; }
    return PG_OK;
}

// Rows [rb, re) of a plan's matching counts and/or distances into host arrays that start at row rb, in row
// blocks of <= 64 Mi pairs per pass
int plan_rows_to_host(const DistancePlan &plan, uint64_t rb, uint64_t re, uint32_t *same, double *distance, cudaStream_t st) {
    const uint64_t n = plan.n, rows_per = std::max<uint64_t>(8, ((64ull << 20) / n) & ~7ull);
    for (uint64_t b = rb; b < re; b += rows_per) {
        const uint64_t e = std::min(re, b + rows_per), cells = (e - b) * n;
        StreamScratch tmp(st);
        uint32_t *d_same = nullptr;
        double *d_dist = nullptr;
        int rc;
        if (same && (rc = scratch_alloc(tmp, &d_same, cells))) return rc;
        if (distance && (rc = scratch_alloc(tmp, &d_dist, cells))) return rc;
        if ((rc = distance_plan_rows(plan, b, e, d_same, d_dist, st)) != PG_OK) return rc;
        if (same) PG_CUDA(cudaMemcpyAsync(same + (b - rb) * n, d_same, cells * 4, cudaMemcpyDeviceToHost, st));
        if (distance) PG_CUDA(cudaMemcpyAsync(distance + (b - rb) * n, d_dist, cells * 8, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
    }
    return PG_OK;
}
}  // namespace
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

// ---------------------------------------------------------------------------------
// mash.Sketch
// ---------------------------------------------------------------------------------
static int check_ks(int32_t k, int32_t s) {
    if (k < 0) { set_error("kmerSize %d < 0: the reference panics (slice bounds)", k); return PG_ERR_ARG; }
    if (s < 0) { set_error("sketchSize %d < 0: the reference panics (makeslice)", s); return PG_ERR_ARG; }
    return PG_OK;
}
static int check_dev_flags(uint32_t flags) {
    if (flags & PG_SKETCH_TAIL_KEEP) { set_error("PG_SKETCH_TAIL_KEEP applies to host buffers only"); return PG_ERR_ARG; }
    return PG_OK;
}
// the least row stride of a batch whose longest read has max_len bytes: its count, or s with PAD_ZERO
static uint64_t need_row_stride(uint64_t max_len, int32_t k, int32_t s, uint32_t flags) {
    return (flags & PG_SKETCH_PAD_ZERO) ? (uint64_t)s : sketch_words(max_len, k, s);
}
static int check_row_stride(uint64_t row_stride, uint64_t max_len, int32_t k, int32_t s, uint32_t flags) {
    const uint64_t need = need_row_stride(max_len, k, s, flags);
    if (row_stride < need) { set_error("row_stride %llu < %llu", (unsigned long long)row_stride, (unsigned long long)need); return PG_ERR_ARG; }
    return PG_OK;
}

int pg_mash_sketch_uniform_dev(const uint8_t *d_bases, uint64_t n_reads, uint32_t read_len,
                               int32_t k, int32_t s, uint32_t flags, uint32_t *d_out,
                               uint64_t row_stride, int32_t *d_status, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if ((rc = check_ks(k, s)) != PG_OK) return rc;
    if ((rc = check_dev_flags(flags)) != PG_OK) return rc;
    if (n_reads && (!d_bases || !d_out)) { set_error("null buffer"); return PG_ERR_ARG; }
    if ((rc = check_row_stride(row_stride, read_len, k, s, flags)) != PG_OK) return rc;
    return launch_sketch_uniform(d_bases, n_reads, read_len, k, s, flags, d_out, row_stride,
                                 d_status, (cudaStream_t)stream);
}

int pg_mash_sketch_batch_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_reads,
                             uint64_t max_read_len, int32_t k, int32_t s, uint32_t flags,
                             uint32_t *d_out, uint64_t row_stride, uint32_t *d_count,
                             int32_t *d_status, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if ((rc = check_ks(k, s)) != PG_OK) return rc;
    if ((rc = check_dev_flags(flags)) != PG_OK) return rc;
    if (n_reads && (!d_offsets || !d_out)) { set_error("null buffer"); return PG_ERR_ARG; }
    if ((rc = check_row_stride(row_stride, max_read_len, k, s, flags)) != PG_OK) return rc;
    return launch_sketch_ragged(d_bases, d_offsets, n_reads, max_read_len, k, s, flags, d_out,
                                row_stride, d_count, d_status, (cudaStream_t)stream);
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

// rows [row_offset, row_offset + n_local) of every destination buffer (compact rows of cnt words)
static int sketch_scatter_dev(const uint8_t *d_bases, uint64_t n_local, uint32_t read_len, int32_t k, int32_t s,
                              void *const *dst_ptrs, int32_t n_dst, int32_t self, uint64_t row_offset, cudaStream_t st) {
    int rc;
    if ((rc = check_ks(k, s)) != PG_OK) return rc;
    if (n_dst < 1 || n_dst > PG_MAX_PEERS || self < 0 || self >= n_dst || !dst_ptrs) {
        set_error("bad destination set (%d buffers, own index %d; at most %d)", n_dst, self, PG_MAX_PEERS);
        return PG_ERR_ARG;
    }
    const uint64_t cnt = sketch_words(read_len, k, s);
    SketchDst dst;
    dst.n = n_dst;
    for (int p = 0; p < n_dst; ++p) {
        if (!dst_ptrs[p]) { set_error("null gathered pointer for rank %d", p); return PG_ERR_ARG; }
        dst.ptr[p] = (uint32_t *)dst_ptrs[p] + row_offset * cnt;  // this rank's row block
    }
    return launch_sketch_uniform(d_bases, n_local, read_len, k, s, 0, dst.ptr[self], cnt, nullptr, st, &dst);
}

int pg_mash_sketch_uniform_gather_dev(const uint8_t *d_bases, uint64_t n_local, uint32_t read_len,
                                      int32_t k, int32_t s, void *const *gathered_ptrs,
                                      int32_t world, int32_t rank, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return sketch_scatter_dev(d_bases, n_local, read_len, k, s, gathered_ptrs, world, rank, (uint64_t)(rank < 0 ? 0 : rank) * n_local,
                              (cudaStream_t)stream);
}

int pg_mash_sketch_uniform_scatter_dev(const uint8_t *d_bases, uint64_t n_local, uint32_t read_len, int32_t k, int32_t s,
                                       void *const *dst_ptrs, int32_t n_dst, int32_t self, uint64_t row_offset, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return sketch_scatter_dev(d_bases, n_local, read_len, k, s, dst_ptrs, n_dst, self, row_offset, (cudaStream_t)stream);
}

// Pipelined host path shared by the uniform and ragged entry points: chunks of reads
// cycle through the N_SLOTS stream/buffer slots (H2D, kernel, D2H overlap across slots).
static bool is_pageable(const void *p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}

static int host_copy_helpers() {
    if (const char *e = getenv("PG_HOST_COPY_THREADS")) return std::max(0, atoi(e) - 1);
    cpu_set_t cur;
    int cores = (int)std::thread::hardware_concurrency();
    if (sched_getaffinity(0, sizeof cur, &cur) == 0) cores = std::min(cores, CPU_COUNT(&cur));
    return std::max(0, std::min(8, cores / 2) - 1);
}

namespace pg {
namespace {

// One host sketch call: reads [0, n) of a ragged batch (offsets) or of fixed-length reads (ulen bytes
// each, offsets == nullptr), the sketch of read i at out + i * row_stride
struct SketchCall {
    const uint8_t *bases;
    const uint64_t *offsets;
    uint32_t ulen;
    uint64_t n;
    int32_t k, s;
    uint32_t flags;
    uint32_t *out;
    uint64_t row_stride;
    uint32_t *count;
    int32_t *status;
};

// Every argument check of a host sketch call, made before anything is launched or written: k and s,
// the buffers, the offsets of the whole batch and the row stride its longest read needs.
static int sketch_check(const SketchCall &q) {
    int rc;
    if ((rc = check_ks(q.k, q.s)) != PG_OK || q.n == 0) return rc;
    if (!q.bases || !q.out) { set_error("null buffer"); return PG_ERR_ARG; }
    uint64_t max_len = q.ulen;
    if (q.offsets && (rc = check_ragged(q.offsets, q.n, &max_len)) != PG_OK) return rc;
    return check_row_stride(q.row_stride, max_len, q.k, q.s, q.flags);
}

// reads [r0, r1) of the batch, bytes [beg, end) of bases
struct Chunk {
    uint64_t r0, r1, beg, end, maxlen, minlen;
    bool uniform;  // all reads of one length below 2^32: the uniform kernel takes the chunk
};

// One pipelined host sketch call on the current device, over a batch sketch_check accepted; holds the
// device's lock.  Chunk i goes to slot i % N_SLOTS once the slot's previous chunk is drained.  Unless
// run() completes, the destructor waits for every slot's stream, so that no copy into or out of the
// caller's memory is still running when the entry point returns.
class SketchPipe {
    static constexpr uint64_t TARGET_OUT_BYTES = 128ull << 20;  // staged output bytes per chunk
    DevCtx &cx_;
    std::lock_guard<std::mutex> lock_;
    SketchCall q_;  // flags without PG_SKETCH_TAIL_KEEP
    // Pinned caller buffers (pg_host_alloc, cudaHostRegister) are DMA'd directly.  Pageable ones (a Go
    // []byte / []uint32) would be bounced by the driver at ~14 GB/s: they go through pinned staging
    // buffers instead, filled / emptied by a few host threads while the other slots' DMA runs; the
    // device then always produces compact rows and the zero tail of PG_SKETCH_PAD_ZERO rows is
    // written by the host threads, not shipped over PCIe.
    // PG_SKETCH_TAIL_KEEP: only the informative words of a row are written.  Ragged batches then always go through
    // the staging buffers, whose rows are copied out count[i] words at a time.
    const bool keep_tail_, stage_in_, stage_out_, want_status_;
    const uint64_t target_bytes_;  // input bytes per chunk
    bool any_panic_ = false, finished_ = false;

    // f(a, b) over min(threads, nrows) parts of rows [0, nrows), on the copy pool
    void par_rows(uint64_t nrows, const std::function<void(uint64_t, uint64_t)> &f) {
        const int parts = (int)std::min<uint64_t>((uint64_t)cx_.pool.threads(), std::max<uint64_t>(1, nrows));
        cx_.pool.run(parts, [&](int i) { f(nrows * (uint64_t)i / parts, nrows * (uint64_t)(i + 1) / parts); });
    }

    // the chunk that starts at read r0
    Chunk next_chunk(uint64_t r0) const {
        Chunk c{r0, r0, 0, 0, 0, ~0ull, false};
        if (q_.offsets) {
            const uint64_t *off = q_.offsets;
            c.beg = off[r0];
            while (c.r1 < q_.n && (c.r1 == r0 || off[c.r1 + 1] - c.beg <= target_bytes_)) {
                const uint64_t len = off[c.r1 + 1] - off[c.r1];
                c.maxlen = std::max(c.maxlen, len);
                c.minlen = std::min(c.minlen, len);
                ++c.r1;
                if (stage_out_ && (c.r1 - r0) * sketch_words(c.maxlen, q_.k, q_.s) * 4 >= TARGET_OUT_BYTES) break;
            }
            c.end = off[c.r1];
        } else {
            uint64_t per = std::max<uint64_t>(1, target_bytes_ / std::max<uint32_t>(q_.ulen, 1));
            const uint64_t row_bytes = sketch_words(q_.ulen, q_.k, q_.s) * 4;
            if (stage_out_ && row_bytes) per = std::min(per, std::max<uint64_t>(32, TARGET_OUT_BYTES / row_bytes));
            per = (per + 31) & ~31ull;  // keep chunk starts on K1 tile boundaries
            c.r1 = std::min(q_.n, r0 + per);
            c.beg = r0 * (uint64_t)q_.ulen;
            c.end = c.r1 * (uint64_t)q_.ulen;
            c.maxlen = c.minlen = q_.ulen;
        }
        c.uniform = c.maxlen == c.minlen && c.maxlen <= 0xffffffffull;
        return c;
    }

    // *src = the chunk's input bytes as the H2D copy reads them: pageable input is first copied into the
    // slot's pinned buffer, in 1 MiB granules over the copy pool
    int stage_in(Slot &sl, const Chunk &c, const uint8_t **src) {
        const uint8_t *h = q_.bases + c.beg;
        const uint64_t bytes = c.end - c.beg;
        *src = h;
        if (!stage_in_ || !bytes) return PG_OK;
        const int rc = sl.pin_in.reserve(bytes);
        if (rc != PG_OK) return rc;
        uint8_t *pin = (uint8_t *)sl.pin_in.p;
        par_rows((bytes + (1u << 20) - 1) >> 20, [&](uint64_t a, uint64_t b) {
            const uint64_t lo = a << 20, hi = std::min<uint64_t>(bytes, b << 20);
            if (hi > lo) memcpy(pin + lo, h + lo, hi - lo);
        });
        *src = pin;
        return PG_OK;
    }

    // the chunk's copies in, kernel and copies out on the slot's stream; the slot is drained
    int enqueue(Slot &sl, const Chunk &c) {
        const int32_t k = q_.k, s = q_.s;
        const uint64_t nr = c.r1 - c.r0, in_bytes = c.end - c.beg, cnt_max = sketch_words(c.maxlen, k, s);
        // staged output: compact device rows, the host threads pad; direct output: the device pads
        const bool compact = stage_out_ || keep_tail_;
        const uint32_t dev_flags = compact ? (q_.flags & ~PG_SKETCH_PAD_ZERO) : q_.flags;
        const uint64_t dev_stride = compact ? cnt_max : need_row_stride(c.maxlen, k, s, q_.flags);
        const cudaStream_t st = sl.stream;
        int rc;
        if ((rc = sl.in.reserve(in_bytes + 64)) != PG_OK) return rc;
        if ((rc = sl.out.reserve(std::max<uint64_t>(nr * dev_stride * 4, 16))) != PG_OK) return rc;
        uint8_t *d_in = (uint8_t *)sl.in.p;
        uint32_t *d_out = (uint32_t *)sl.out.p;
        int32_t *d_status = nullptr;
        uint32_t *d_count = nullptr;
        if (want_status_) {
            if ((rc = sl.st.reserve(nr * 4)) != PG_OK) return rc;
            d_status = (int32_t *)sl.st.p;
            PG_CUDA(cudaMemsetAsync(d_status, 0, nr * 4, st));
            sl.status.assign(nr, 0);
        }
        const uint8_t *h_src;
        if ((rc = stage_in(sl, c, &h_src)) != PG_OK) return rc;
        if (in_bytes) PG_CUDA(cudaMemcpyAsync(d_in, h_src, in_bytes, cudaMemcpyHostToDevice, st));
        if (c.uniform) {
            rc = launch_sketch_uniform(d_in, nr, (uint32_t)c.maxlen, k, s, dev_flags, d_out, dev_stride, d_status, st);
        } else {
            if ((rc = sl.aux.reserve((nr + 1) * 8 + nr * 4)) != PG_OK) return rc;
            uint64_t *d_off = (uint64_t *)sl.aux.p;
            d_count = (uint32_t *)(d_off + nr + 1);
            PG_CUDA(cudaMemcpyAsync(d_off, q_.offsets + c.r0, (nr + 1) * 8, cudaMemcpyHostToDevice, st));
            // kernels index bases with absolute offsets: shift the base pointer
            rc = launch_sketch_ragged(d_in - c.beg, d_off, nr, c.maxlen, k, s, dev_flags, d_out, dev_stride, d_count, d_status, st);
        }
        if (rc != PG_OK) return rc;
        uint32_t *out = q_.out + c.r0 * q_.row_stride;
        if (dev_stride) {
            if (stage_out_) {
                if ((rc = sl.pin_out.reserve(nr * dev_stride * 4)) != PG_OK) return rc;
                PG_CUDA(cudaMemcpyAsync(sl.pin_out.p, d_out, nr * dev_stride * 4, cudaMemcpyDeviceToHost, st));
            } else if (q_.row_stride == dev_stride) {
                PG_CUDA(cudaMemcpyAsync(out, d_out, nr * dev_stride * 4, cudaMemcpyDeviceToHost, st));
            } else {
                PG_CUDA(cudaMemcpy2DAsync(out, q_.row_stride * 4, d_out, dev_stride * 4, dev_stride * 4, nr, cudaMemcpyDeviceToHost, st));
            }
        }
        if (q_.count) {
            if (c.uniform) std::fill(q_.count + c.r0, q_.count + c.r1, (uint32_t)cnt_max);
            else PG_CUDA(cudaMemcpyAsync(q_.count + c.r0, d_count, nr * 4, cudaMemcpyDeviceToHost, st));
        }
        if (want_status_) PG_CUDA(cudaMemcpyAsync(sl.status.data(), d_status, nr * 4, cudaMemcpyDeviceToHost, st));
        sl.r0 = c.r0;
        sl.nr = nr;
        sl.dstride = dev_stride;
        sl.used = true;
        return PG_OK;
    }

    // waits for the slot's chunk, then unstages its rows (or zeroes their tails) and folds its statuses
    int drain(Slot &sl) {
        if (!sl.used) return PG_OK;
        PG_CUDA(cudaStreamSynchronize(sl.stream));
        const uint64_t rs = q_.row_stride, ds = sl.dstride;
        uint32_t *out = q_.out + sl.r0 * rs;
        if (stage_out_ && ds) {  // staged rows -> caller rows (+ zero tail up to the caller's stride)
            const uint32_t *src = (const uint32_t *)sl.pin_out.p;
            par_rows(sl.nr, [&](uint64_t a, uint64_t b) {
                if (ds == rs && !(keep_tail_ && q_.offsets)) {
                    memcpy(out + a * rs, src + a * ds, (b - a) * ds * 4);
                    return;
                }
                for (uint64_t i = a; i < b; ++i) {
                    if (keep_tail_) {  // exactly the informative words of this row
                        const uint64_t r = sl.r0 + i;
                        const uint64_t ci = q_.offsets ? sketch_words(q_.offsets[r + 1] - q_.offsets[r], q_.k, q_.s) : ds;
                        memcpy(out + i * rs, src + i * ds, ci * 4);
                        continue;
                    }
                    memcpy(out + i * rs, src + i * ds, ds * 4);
                    memset(out + i * rs + ds, 0, (rs - ds) * 4);
                }
            });
        } else if (rs > ds && !keep_tail_) {  // direct DMA wrote ds words per row: zero the rest of each row
            par_rows(sl.nr, [&](uint64_t a, uint64_t b) {
                for (uint64_t i = a; i < b; ++i) memset(out + i * rs + ds, 0, (rs - ds) * 4);
            });
        }
        if (want_status_) {
            for (uint64_t i = 0; i < sl.nr; ++i) {
                if (sl.status[i] != PG_ITEM_OK) any_panic_ = true;
                if (q_.status) q_.status[sl.r0 + i] = sl.status[i];
            }
        }
        sl.used = false;
        return PG_OK;
    }

public:
    explicit SketchPipe(const SketchCall &q)
        : cx_(*t_ctx), lock_(cx_.mu), q_(q), keep_tail_((q.flags & PG_SKETCH_TAIL_KEEP) != 0), stage_in_(is_pageable(q.bases)),
          stage_out_(is_pageable(q.out) || (keep_tail_ && q.offsets)), want_status_(q.status != nullptr || q.s <= 1),
          target_bytes_((stage_in_ || stage_out_) ? (32ull << 20) : (192ull << 20)) {
        q_.flags &= ~PG_SKETCH_TAIL_KEEP;
        if (stage_in_ || stage_out_) cx_.pool.start(host_copy_helpers(), cx_.device);
    }
    ~SketchPipe() {
        if (finished_) return;
        for (Slot &sl : cx_.slots) {
            cudaStreamSynchronize(sl.stream);
            sl.used = false;
        }
        cudaGetLastError();
    }
    int run() {
        int rc, slot = 0;
        for (uint64_t r0 = 0; r0 < q_.n; slot = (slot + 1) % N_SLOTS) {
            const Chunk c = next_chunk(r0);
            if ((rc = drain(cx_.slots[slot])) != PG_OK || (rc = enqueue(cx_.slots[slot], c)) != PG_OK) return rc;
            r0 = c.r1;
        }
        for (int i = 0; i < N_SLOTS; ++i)
            if ((rc = drain(cx_.slots[(slot + i) % N_SLOTS])) != PG_OK) return rc;  // oldest first
        finished_ = true;
        if (any_panic_) {
            set_error("at least one read hits an input on which mash.Sketch panics (sketchSize <= 1)");
            return PG_ERR_PANIC;
        }
        return PG_OK;
    }
};

static int sketch_host(const SketchCall &q) {
    int rc = ensure_device();
    if (rc != PG_OK || (rc = sketch_check(q)) != PG_OK || q.n == 0) return rc;
    return SketchPipe(q).run();
}

}  // namespace
}  // namespace pg

int pg_mash_sketch_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads, int32_t k,
                         int32_t s, uint32_t flags, uint32_t *out, uint64_t row_stride,
                         uint32_t *count, int32_t *status) {
    if (n_reads && !offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    return sketch_host({bases, offsets, 0, n_reads, k, s, flags, out, row_stride, count, status});
}

int pg_mash_sketch_uniform(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k,
                           int32_t s, uint32_t flags, uint32_t *out, uint64_t row_stride,
                           int32_t *status) {
    return sketch_host({bases, nullptr, read_len, n_reads, k, s, flags, out, row_stride, nullptr, status});
}

// ---------------------------------------------------------------------------------
// Single-process multi-GPU entry points (SURVEY.md 8b "multi-GPU variants taking a device
// count", 8e): one host thread per device, reads sharded in contiguous blocks, no data-path
// collective for Sketch; Sketch+Distance exchanges the finished sketches by peer stores issued
// from the sketch kernels themselves (in-process peer access, no IPC).
// ---------------------------------------------------------------------------------
namespace pg {
namespace {

struct WorkerResult {
    int rc = PG_OK;
    std::string msg;
};

// worst result of the workers, message copied to the caller's thread-local slot.  A reference panic
// (PG_ERR_PANIC: per-item statuses are still complete) ranks below real failures.
static int fold_results(const std::vector<WorkerResult> &res) {
    int worst = PG_OK;
    const std::string *msg = nullptr;
    for (const WorkerResult &r : res) {
        if (r.rc == PG_OK) continue;
        const bool soft = r.rc == PG_ERR_PANIC, worst_soft = worst == PG_ERR_PANIC || worst == PG_OK;
        if (worst == PG_OK || (!soft && worst_soft)) { worst = r.rc; msg = &r.msg; }
    }
    if (msg) set_error("%s", msg->c_str());
    return worst;
}

static int resolve_devices(const int32_t *devices, int32_t n_devices, std::vector<int> *out) {
    int n = 0, rc = device_count_checked(&n);
    if (rc != PG_OK) return rc;
    out->clear();
    if (!devices) {
        const int cnt = n_devices > 0 ? std::min<int>(n_devices, n) : n;
        for (int i = 0; i < cnt; ++i) out->push_back(i);
    } else {
        if (n_devices <= 0) { set_error("device list given with n_devices = %d", n_devices); return PG_ERR_ARG; }
        for (int i = 0; i < n_devices; ++i) {
            if (devices[i] < 0 || devices[i] >= n) { set_error("device %d out of range (count %d)", devices[i], n); return PG_ERR_ARG; }
            for (int j = 0; j < i; ++j)
                if (devices[j] == devices[i]) { set_error("device %d listed twice", devices[i]); return PG_ERR_ARG; }
            out->push_back(devices[i]);
        }
    }
    if (out->size() > (size_t)PG_MAX_PEERS) out->resize(PG_MAX_PEERS);
    return PG_OK;
}

// reusable barrier for the device threads of one call
class Rendezvous {
    std::mutex mu_;
    std::condition_variable cv_;
    int n_, waiting_ = 0;
    uint64_t gen_ = 0;
public:
    explicit Rendezvous(int n) : n_(n) {}
    void wait() {
        std::unique_lock<std::mutex> lk(mu_);
        const uint64_t g = gen_;
        if (++waiting_ == n_) { waiting_ = 0; ++gen_; cv_.notify_all(); }
        else cv_.wait(lk, [&] { return gen_ != g; });
    }
};

// P contiguous shards of n reads, cut on K1 tile boundaries (32 reads): shard r is [cut[r], cut[r + 1])
std::vector<uint64_t> uniform_cuts(uint64_t n, int P) {
    std::vector<uint64_t> cut(P + 1, n);
    cut[0] = 0;
    const uint64_t per = ((n + P - 1) / P + 31) & ~31ull;
    for (int r = 1; r < P; ++r) cut[r] = std::min(n, (uint64_t)r * per);
    return cut;
}

// The batch is checked once, here, before it is cut; each shard then runs the pipeline on its device's thread.
int sketch_multi(const SketchCall &q, const int32_t *devices, int32_t n_devices) {
    std::vector<int> dev;
    int rc;
    if ((rc = resolve_devices(devices, n_devices, &dev)) != PG_OK || (rc = sketch_check(q)) != PG_OK || q.n == 0) return rc;
    const int P = (int)dev.size();
    std::vector<uint64_t> cut = uniform_cuts(q.n, P);
    if (q.offsets) {  // ragged batches balance bytes instead
        const uint64_t b0 = q.offsets[0], total = q.offsets[q.n] - b0;
        for (int r = 1; r < P; ++r) {
            const uint64_t want = b0 + total / P * r;
            uint64_t i = std::lower_bound(q.offsets, q.offsets + q.n + 1, want) - q.offsets;
            i = std::min<uint64_t>((i + 31) & ~31ull, q.n);
            cut[r] = std::max(i, cut[r - 1]);
        }
    }
    std::vector<WorkerResult> res(P);
    std::vector<std::thread> th;
    for (int r = 0; r < P; ++r) {
        const uint64_t lo = cut[r], hi = cut[r + 1];
        if (hi <= lo) continue;
        SketchCall shard = q;
        shard.n = hi - lo;
        if (q.offsets) shard.offsets += lo;
        else shard.bases += lo * (uint64_t)q.ulen;
        shard.out += lo * q.row_stride;
        if (q.count) shard.count += lo;
        if (q.status) shard.status += lo;
        th.emplace_back([&res, &dev, r, shard] {
            t_bound_device = dev[r];  // this worker's entry points run on its device
            pg_numa_bind_thread(dev[r], nullptr);  // best effort: staging copies from the GPU's NUMA node
            int wrc = ensure_device();
            if (wrc == PG_OK) wrc = SketchPipe(shard).run();
            res[r].rc = wrc;
            if (wrc != PG_OK) res[r].msg = t_err;
        });
    }
    for (std::thread &t : th) t.join();
    return fold_results(res);
}

}  // namespace
}  // namespace pg

extern "C" int pg_mash_sketch_uniform_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k, int32_t s,
                                            uint32_t flags, uint32_t *out, uint64_t row_stride, int32_t *status,
                                            const int32_t *devices, int32_t n_devices) {
    return sketch_multi({bases, nullptr, read_len, n_reads, k, s, flags, out, row_stride, nullptr, status}, devices, n_devices);
}

extern "C" int pg_mash_sketch_batch_multi(const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads, int32_t k, int32_t s,
                                          uint32_t flags, uint32_t *out, uint64_t row_stride, uint32_t *count, int32_t *status,
                                          const int32_t *devices, int32_t n_devices) {
    if (n_reads && !offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    return sketch_multi({bases, offsets, 0, n_reads, k, s, flags, out, row_stride, count, status}, devices, n_devices);
}

// Sketch + all-pairs distance over several devices of this process (cfg3 / cfg4 pipeline, SURVEY 8e):
//   1. device r takes reads [lo_r, hi_r), copies them in and runs the sketch kernel, whose finished
//      tiles / rows are stored straight into the gathered buffer of EVERY device (peer access
//      enabled in-process): sketching and the all-gather are one kernel;
//   2. after a rendezvous every device holds all n sketches and computes row block r of the pair
//      matrix (receiver = row) with the same kernels as pg_mash_distance_block.
// Without peer access between two of the devices the exchange falls back to cudaMemcpyPeerAsync pulls.
extern "C" int pg_mash_sketch_distance_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k, int32_t s,
                                             const int32_t *devices, int32_t n_devices, uint32_t *sketches, uint32_t *same,
                                             double *distance) {
    int rc;
    if ((rc = check_ks(k, s)) != PG_OK) return rc;
    std::vector<int> dev;
    if ((rc = resolve_devices(devices, n_devices, &dev)) != PG_OK) return rc;
    if (n_reads == 0) return PG_OK;
    if (!bases) { set_error("null buffer"); return PG_ERR_ARG; }
    if (s <= 0) { set_error("distance over sketches of size %d: the reference panics", s); return PG_ERR_PANIC; }
    const uint64_t n = n_reads, L = read_len;
    const uint64_t cnt = sketch_words(L, k, s);
    const int P = (int)std::min<uint64_t>(dev.size(), (n + 31) / 32);
    dev.resize(P);
    const std::vector<uint64_t> cut = uniform_cuts(n, P);
    // peer access available between every pair?
    bool fused = true;
    for (int a = 0; a < P && fused; ++a)
        for (int b = 0; b < P && fused; ++b) {
            int can = 1;
            if (a != b && cudaDeviceCanAccessPeer(&can, dev[a], dev[b]) != cudaSuccess) can = 0;
            fused = fused && can;
        }
    cudaGetLastError();
    std::vector<void *> gathered(P, nullptr);  // [n][cnt] compact rows on every device
    std::vector<WorkerResult> res(P);
    std::atomic<bool> failed{false};
    Rendezvous meet(P);
    auto worker = [&](int r) {
        WorkerResult &my = res[r];
        auto fail = [&](int code) { my.rc = code; my.msg = t_err; failed.store(true); };
        auto step = [&](auto &&fn) { if (!failed.load()) { const int c = fn(); if (c != PG_OK) fail(c); } };
        t_bound_device = dev[r];
        pg_numa_bind_thread(dev[r], nullptr);
        const uint64_t lo = cut[r], hi = cut[r + 1], nl = hi - lo;
        uint8_t *d_reads = nullptr;
        uint32_t *d_full = nullptr;  // [n][s] full Go arrays (== gathered when cnt == s)
        cudaStream_t st = nullptr;
        step([&]() -> int {
            int c = ensure_device();
            if (c != PG_OK) return c;
            st = t_ctx->slots[0].stream;
            if (fused)
                for (int p = 0; p < P; ++p)
                    if (p != r) {
                        cudaError_t e = cudaDeviceEnablePeerAccess(dev[p], 0);
                        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return cuda_fail(e, "cudaDeviceEnablePeerAccess", __FILE__, __LINE__);
                        cudaGetLastError();
                    }
            PG_CUDA(cudaMalloc(&gathered[r], std::max<uint64_t>(n * cnt * 4, 16)));
            PG_CUDA(cudaMalloc(&d_reads, std::max<uint64_t>(nl * L, 16) + 64));
            return PG_OK;
        });
        meet.wait();  // every buffer exists, peer access is on
        step([&]() -> int {
            if (nl) PG_CUDA(cudaMemcpyAsync(d_reads, bases + lo * L, nl * L, cudaMemcpyHostToDevice, st));
            int c;
            if (fused) {
                c = sketch_scatter_dev(d_reads, nl, read_len, k, s, gathered.data(), P, r, lo, st);
            } else {
                void *own = gathered[r];
                c = sketch_scatter_dev(d_reads, nl, read_len, k, s, &own, 1, 0, lo, st);
            }
            if (c != PG_OK) return c;
            PG_CUDA(cudaStreamSynchronize(st));
            return PG_OK;
        });
        meet.wait();  // all sketches computed (fused: and stored everywhere)
        step([&]() -> int {
            if (!fused)  // pull the other devices' row blocks
                for (int p = 0; p < P; ++p)
                    if (p != r && cut[p + 1] > cut[p])
                        PG_CUDA(cudaMemcpyPeerAsync((uint32_t *)gathered[r] + cut[p] * cnt, dev[r], (uint32_t *)gathered[p] + cut[p] * cnt, dev[p],
                                                    (cut[p + 1] - cut[p]) * cnt * 4, st));
            if (cnt == (uint64_t)s) {
                d_full = (uint32_t *)gathered[r];
            } else {  // the zero tail of a fresh Mash is materialised after the exchange
                PG_CUDA(cudaMalloc(&d_full, n * (uint64_t)s * 4));
                PG_CUDA(cudaMemsetAsync(d_full, 0, n * (uint64_t)s * 4, st));
                if (cnt) PG_CUDA(cudaMemcpy2DAsync(d_full, (size_t)s * 4, gathered[r], cnt * 4, cnt * 4, n, cudaMemcpyDeviceToDevice, st));
            }
            if (sketches && nl) PG_CUDA(cudaMemcpyAsync(sketches + lo * (uint64_t)s, d_full + lo * (uint64_t)s, nl * (uint64_t)s * 4, cudaMemcpyDeviceToHost, st));
            if ((same || distance) && nl) {
                DistancePlan plan;
                int c = distance_plan_create(d_full, n, s, st, &plan);
                if (c == PG_OK) c = plan_rows_to_host(plan, lo, hi, same ? same + lo * n : nullptr, distance ? distance + lo * n : nullptr, st);
                distance_plan_destroy(plan, st);
                if (c != PG_OK) return c;
            }
            PG_CUDA(cudaStreamSynchronize(st));
            return PG_OK;
        });
        meet.wait();  // nobody reads a peer buffer any more
        if (t_ctx) {
            cudaSetDevice(dev[r]);
            if (d_full && d_full != gathered[r]) cudaFree(d_full);
            if (d_reads) cudaFree(d_reads);
            if (gathered[r]) cudaFree(gathered[r]);
            cudaGetLastError();
        }
    };
    std::vector<std::thread> th;
    for (int r = 0; r < P; ++r) th.emplace_back(worker, r);
    for (std::thread &t : th) t.join();
    return fold_results(res);
}

// ---------------------------------------------------------------------------------
// Similarity / Distance
// ---------------------------------------------------------------------------------
int pg_mash_similarity_pairs_dev(const uint32_t *d_sketches, const uint64_t *d_sk_offsets,
                                 uint64_t n_sketches, const uint32_t *d_pair_a,
                                 const uint32_t *d_pair_b, uint64_t n_pairs, int64_t *d_same,
                                 double *d_similarity, double *d_distance, int32_t *d_status,
                                 void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return launch_similarity_pairs(d_sketches, d_sk_offsets, n_sketches, d_pair_a, d_pair_b, n_pairs,
                                   d_same, d_similarity, d_distance, d_status, (cudaStream_t)stream);
}


int pg_mash_similarity_pairs(const uint32_t *sketches, const uint64_t *sk_offsets,
                             uint64_t n_sketches, const uint32_t *pair_a, const uint32_t *pair_b,
                             uint64_t n_pairs, int64_t *same, double *similarity, double *distance,
                             int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_pairs == 0) return PG_OK;
    if (!sk_offsets || !pair_a || !pair_b) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint32_t> sk = c.ragged(sketches, sk_offsets, n_sketches);
    const uint32_t *d_a = c.upload(pair_a, n_pairs), *d_b = c.upload(pair_b, n_pairs);
    int64_t *d_same = c.alloc<int64_t>(n_pairs);
    double *d_sim = c.alloc<double>(n_pairs), *d_dist = c.alloc<double>(n_pairs);
    int32_t *d_st = c.alloc<int32_t>(n_pairs, true);
    if ((rc = c.error()) || (rc = launch_similarity_pairs(sk.base, sk.off, n_sketches, d_a, d_b, n_pairs, d_same, d_sim, d_dist, d_st, c.st)))
        return rc;
    std::vector<int32_t> hst(n_pairs);
    c.download(same, d_same, n_pairs);
    c.download(similarity, d_sim, n_pairs);
    c.download(distance, d_dist, n_pairs);
    c.download(hst.data(), d_st, n_pairs);
    if ((rc = c.finish())) return rc;
    // the pair kernel reports no unsupported items
    return fold_item_status(hst, status, "at least one pair involves an empty sketch or an invalid index (reference panics)", nullptr);
}

int pg_mash_distance_block_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint64_t row_begin,
                               uint64_t row_end, uint32_t *d_same, double *d_distance, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (row_end > n || row_begin > row_end) { set_error("bad row range"); return PG_ERR_ARG; }
    return launch_distance_block(d_sketches, n, s, row_begin, row_end, d_same, d_distance, (cudaStream_t)stream);
}

int pg_mash_distance_block(const uint32_t *sketches, uint64_t n, int32_t s, uint64_t row_begin,
                           uint64_t row_end, uint32_t *same, double *distance) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (row_end > n || row_begin > row_end) { set_error("bad row range"); return PG_ERR_ARG; }
    if (row_end == row_begin || n == 0) return PG_OK;
    if (s <= 0) { set_error("distance over sketches of size %d: the reference panics", s); return PG_ERR_PANIC; }
    HostCall c;
    const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)s);
    if ((rc = c.error())) return rc;
    // one plan (sortedness + join index) for the whole call
    DistancePlan plan;
    rc = distance_plan_create(d_sk, n, s, c.st, &plan);
    if (rc == PG_OK) rc = plan_rows_to_host(plan, row_begin, row_end, same, distance, c.st);
    distance_plan_destroy(plan, c.st);
    return rc != PG_OK ? rc : c.finish();
}

int pg_mash_distance_sparse_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint64_t row_begin, uint64_t row_end, uint32_t flags,
                                uint32_t *d_pair_i, uint32_t *d_pair_j, uint32_t *d_pair_same, uint64_t pairs_cap, uint64_t *d_n_pairs,
                                void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (row_end > n || row_begin > row_end) { set_error("bad row range"); return PG_ERR_ARG; }
    if (!d_n_pairs || (pairs_cap && (!d_pair_i || !d_pair_j || !d_pair_same))) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_distance_sparse(d_sketches, n, s, row_begin, row_end, flags, d_pair_i, d_pair_j, d_pair_same, pairs_cap,
                                  (unsigned long long *)d_n_pairs, (cudaStream_t)stream);
}

int pg_mash_distance_sparse(const uint32_t *sketches, uint64_t n, int32_t s, uint64_t row_begin, uint64_t row_end, uint32_t flags,
                            uint32_t *pair_i, uint32_t *pair_j, uint32_t *pair_same, uint64_t pairs_cap, uint64_t *n_pairs) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_pairs) { set_error("null buffer"); return PG_ERR_ARG; }
    *n_pairs = 0;
    if (row_end > n || row_begin > row_end) { set_error("bad row range"); return PG_ERR_ARG; }
    if (row_end == row_begin || n == 0) return PG_OK;
    if (s <= 0) { set_error("distance over sketches of size %d: the reference panics", s); return PG_ERR_PANIC; }
    if (pairs_cap && (!pair_i || !pair_j || !pair_same)) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)s);
    uint32_t *d_i = c.alloc<uint32_t>(pairs_cap), *d_j = c.alloc<uint32_t>(pairs_cap), *d_c = c.alloc<uint32_t>(pairs_cap);
    unsigned long long *d_n = c.alloc<unsigned long long>(1);
    if ((rc = c.error()) || (rc = launch_distance_sparse(d_sk, n, s, row_begin, row_end, flags, d_i, d_j, d_c, pairs_cap, d_n, c.st)))
        return rc;
    return finish_capped(c, d_n, pairs_cap, n_pairs, {{pair_i, d_i, 4}, {pair_j, d_j, 4}, {pair_same, d_c, 4}}, "pairs_cap", "pairs");
}

// ---------------------------------------------------------------------------------
// Sketch index: top-k nearest references
// ---------------------------------------------------------------------------------
}  // extern "C"

struct pg_mash_index {
    int device;
    uint32_t *d_sk;        // the index's own copy of the n x s reference sketches
    DistancePlan plan;     // sortedness flags + join index over d_sk
};

static int index_create(const uint32_t *src, bool src_dev, uint64_t n, int32_t s, cudaStream_t st, pg_mash_index **out) {
    if (n && s <= 0) { set_error("index over sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    pg_mash_index *ix = new pg_mash_index{t_ctx->device, nullptr, DistancePlan()};
    const uint64_t words = n * (uint64_t)std::max(s, 0);
    int rc = PG_OK;
    cudaError_t e = cudaMallocAsync(&ix->d_sk, words ? words * 4 : 4, st);
    if (e != cudaSuccess) { cudaGetLastError(); ix->d_sk = nullptr; set_error("cudaMallocAsync(%llu) for the index failed", (unsigned long long)(words * 4)); rc = PG_ERR_NOMEM; }
    if (rc == PG_OK && words) {
        e = cudaMemcpyAsync(ix->d_sk, src, words * 4, src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) rc = cuda_fail(e, "index copy", __FILE__, __LINE__);
    }
    if (rc == PG_OK) rc = distance_plan_create(ix->d_sk, n, s, st, &ix->plan);
    if (rc == PG_OK) { e = cudaStreamSynchronize(st); if (e != cudaSuccess) rc = cuda_fail(e, "index build", __FILE__, __LINE__); }
    if (rc != PG_OK) {
        distance_plan_destroy(ix->plan, st);
        if (ix->d_sk) cudaFreeAsync(ix->d_sk, st);
        cudaStreamSynchronize(st);
        delete ix;
        return rc;
    }
    *out = ix;
    return PG_OK;
}

extern "C" {

int pg_mash_index_create(const uint32_t *sketches, uint64_t n, int32_t s, pg_mash_index **out) {
    if (!out) { set_error("null index pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n && s > 0 && !sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(t_ctx->mu);
    return index_create(sketches, false, n, s, t_ctx->slots[0].stream, out);
}

int pg_mash_index_create_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, void *stream, pg_mash_index **out) {
    if (!out) { set_error("null index pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n && s > 0 && !d_sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    return index_create(d_sketches, true, n, s, (cudaStream_t)stream, out);
}

int pg_mash_index_query_dev(const pg_mash_index *ix, const uint32_t *d_queries, uint64_t nq, int32_t sq, uint32_t top_k,
                            uint32_t min_same, uint32_t *d_hit_ref, uint32_t *d_hit_same, double *d_hit_distance,
                            uint32_t *d_n_hits, void *stream) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    return launch_index_query(ix->plan, d_queries, nq, sq, top_k, min_same, d_hit_ref, d_hit_same, d_hit_distance, d_n_hits,
                              (cudaStream_t)stream);
}

int pg_mash_index_query(const pg_mash_index *ix, const uint32_t *queries, uint64_t nq, int32_t sq, uint32_t top_k,
                        uint32_t min_same, uint32_t *hit_ref, uint32_t *hit_same, double *hit_distance, uint32_t *n_hits) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    if (top_k == 0 || top_k > PG_INDEX_MAX_TOP_K) { set_error("top_k %u outside [1, %u]", top_k, PG_INDEX_MAX_TOP_K); return PG_ERR_ARG; }
    if (nq == 0) return PG_OK;
    if (sq <= 0) { set_error("query sketches of size %d: the reference panics (Sketches[-1])", sq); return PG_ERR_PANIC; }
    if (!queries) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint64_t slots = nq * (uint64_t)top_k;
    const uint32_t *d_q = c.upload(queries, nq * (uint64_t)sq);
    uint32_t *d_ref = hit_ref ? c.alloc<uint32_t>(slots) : nullptr, *d_same = hit_same ? c.alloc<uint32_t>(slots) : nullptr;
    double *d_dist = hit_distance ? c.alloc<double>(slots) : nullptr;
    uint32_t *d_nh = n_hits ? c.alloc<uint32_t>(nq) : nullptr;
    if ((rc = c.error()) || (rc = launch_index_query(ix->plan, d_q, nq, sq, top_k, min_same, d_ref, d_same, d_dist, d_nh, c.st))) return rc;
    c.download(hit_ref, d_ref, slots);
    c.download(hit_same, d_same, slots);
    c.download(hit_distance, d_dist, slots);
    c.download(n_hits, d_nh, nq);
    return c.finish();
}

int pg_mash_index_free(pg_mash_index *ix) {
    if (!ix) return PG_OK;
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(t_ctx->mu);
    cudaStream_t st = t_ctx->slots[0].stream;
    distance_plan_destroy(ix->plan, st);
    if (ix->d_sk) cudaFreeAsync(ix->d_sk, st);
    delete ix;
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// ---------------------------------------------------------------------------------
// Smith-Waterman score
// ---------------------------------------------------------------------------------
static int align_score_dev(const AlignScoring &s, const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                           uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len, int32_t query_is_a, int64_t *d_score,
                           int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (s.has_null() || (n_queries && (!d_q_offsets || !d_score))) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_sw_score(d_queries, d_q_offsets, n_queries, max_query_len, d_templ, templ_len, query_is_a, s, d_score, d_err_code,
                           d_err_pos, (cudaStream_t)stream);
}

static int align_score_host(const AlignScoring &s, const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                            const uint8_t *templ, uint64_t templ_len, int32_t query_is_a, int64_t *score, int32_t *err_code,
                            int64_t *err_pos) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_queries == 0) return PG_OK;
    if (!q_offsets || !score || s.has_null()) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> q = c.ragged(queries, q_offsets, n_queries);
    const uint8_t *d_t = c.upload(templ, templ_len);
    int64_t *d_sc = c.alloc<int64_t>(n_queries), *d_ep = c.alloc<int64_t>(n_queries);
    int32_t *d_ec = c.alloc<int32_t>(n_queries);
    if ((rc = c.error()) || (rc = launch_sw_score(q.base, q.off, n_queries, q.max_len, d_t, templ_len, query_is_a, s, d_sc, d_ec, d_ep, c.st)))
        return rc;
    c.download(score, d_sc, n_queries);
    c.download(err_code, d_ec, n_queries);
    c.download(err_pos, d_ep, n_queries);
    return c.finish();
}

int pg_sw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return align_score_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 0}, d_queries, d_q_offsets, n_queries, max_query_len,
                           d_templ, templ_len, query_is_a, d_score, d_err_code, d_err_pos, stream);
}
int pg_nw_score_batch_dev(const uint8_t *d_queries, const uint64_t *d_q_offsets, uint64_t n_queries,
                          uint64_t max_query_len, const uint8_t *d_templ, uint64_t templ_len,
                          int32_t query_is_a, const int16_t *lut_a_host, const int16_t *lut_b_host,
                          const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return align_score_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 1}, d_queries, d_q_offsets, n_queries, max_query_len,
                           d_templ, templ_len, query_is_a, d_score, d_err_code, d_err_pos, stream);
}
int pg_sw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_score_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                            err_code, err_pos);
}
int pg_nw_score_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_score_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                            err_code, err_pos);
}

static int align_strings_host(const AlignScoring &s, const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                              const uint8_t *templ, uint64_t templ_len, int32_t query_is_a, int64_t *score, int32_t *err_code,
                              int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                              int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_queries == 0) return PG_OK;
    if (!q_offsets || !score || s.has_null() || !align_a || !align_b || !align_len || s.n_a <= 0 || s.n_b <= 0) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    HostCall c;
    const Ragged<uint8_t> q = c.ragged(queries, q_offsets, n_queries);
    const uint8_t *d_t = c.upload(templ, templ_len);
    int64_t *d_sc = c.alloc<int64_t>(n_queries), *d_ep = c.alloc<int64_t>(n_queries);
    int32_t *d_ec = c.alloc<int32_t>(n_queries);
    uint8_t *d_a = c.alloc<uint8_t>(n_queries * out_stride), *d_b = c.alloc<uint8_t>(n_queries * out_stride);
    uint32_t *d_len = c.alloc<uint32_t>(n_queries, true);
    int32_t *d_st = c.alloc<int32_t>(n_queries, true);
    if ((rc = c.error()) || (rc = launch_sw_align(q.base, q.off, n_queries, q.max_len, d_t, templ_len, query_is_a, s, d_sc, d_ec, d_ep, d_a,
                                                  d_b, out_stride, d_len, d_st, c.st)))
        return rc;
    c.download(score, d_sc, n_queries);
    c.download(err_code, d_ec, n_queries);
    c.download(err_pos, d_ep, n_queries);
    c.download(align_a, d_a, n_queries * out_stride);
    c.download(align_b, d_b, n_queries * out_stride);
    c.download(align_len, d_len, n_queries);
    c.download(status, d_st, n_queries);
    return c.finish();
}

int pg_sw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                      int32_t *status) {
    return align_strings_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                              err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}
int pg_nw_align_batch(const uint8_t *queries, const uint64_t *q_offsets, uint64_t n_queries,
                      const uint8_t *templ, uint64_t templ_len, int32_t query_is_a,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a,
                      int32_t n_b, int64_t gap, int64_t *score, int32_t *err_code, int64_t *err_pos,
                      uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len,
                      int32_t *status) {
    return align_strings_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, queries, q_offsets, n_queries, templ, templ_len, query_is_a, score,
                              err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}

// ---------------------------------------------------------------------------------
// Smith-Waterman / Needleman-Wunsch over pair lists
// ---------------------------------------------------------------------------------
// device bytes per pair of a host pair call: indices, outputs and the classify / list scratch
static constexpr uint64_t PAIR_BYTES = 4 + 4 + 8 + 4 + 8 + 1 + 4;
static constexpr uint64_t PAIR_GROUP_BYTES = 1ull << 30;

static int align_pairs_host(const AlignScoring &s, bool strings, const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a,
                            const uint8_t *seqs_b, const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a,
                            const uint32_t *pair_b, uint64_t n_pairs, int64_t *score, int32_t *err_code, int64_t *err_pos,
                            uint8_t *align_a, uint8_t *align_b, uint64_t out_stride, uint32_t *align_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_pairs == 0) return PG_OK;
    if (!offsets_a || !offsets_b || !pair_a || !pair_b || !score || s.has_null() ||
        (strings && (!align_a || !align_b || !align_len))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    // the whole call is checked before anything is uploaded or launched
    uint64_t set_max = 0;
    if ((rc = check_ragged(offsets_a, n_seqs_a, &set_max)) != PG_OK || (rc = check_ragged(offsets_b, n_seqs_b, &set_max)) != PG_OK) return rc;
    // the longest a and b the pairs reference: a long sequence no pair uses widens neither the score type nor any scratch
    uint64_t max_la = 0, max_lb = 0;
    for (uint64_t k = 0; k < n_pairs; ++k) {
        if (pair_a[k] >= n_seqs_a || pair_b[k] >= n_seqs_b) {
            set_error("pair %llu = (%u, %u) is out of range (%llu, %llu sequences)", (unsigned long long)k, pair_a[k], pair_b[k],
                      (unsigned long long)n_seqs_a, (unsigned long long)n_seqs_b);
            return PG_ERR_ARG;
        }
        max_la = std::max(max_la, offsets_a[pair_a[k] + 1] - offsets_a[pair_a[k]]);
        max_lb = std::max(max_lb, offsets_b[pair_b[k] + 1] - offsets_b[pair_b[k]]);
    }
    HostCall c;
    const Ragged<uint8_t> A = c.ragged(seqs_a, offsets_a, n_seqs_a);
    const bool same = seqs_a == seqs_b && offsets_a == offsets_b && n_seqs_a == n_seqs_b;
    const Ragged<uint8_t> B = same ? A : c.ragged(seqs_b, offsets_b, n_seqs_b);
    if ((rc = c.sync()) != PG_OK) return rc;  // the sets are resident: what is free now bounds a group
    size_t free_b = 0, total_b = 0;
    PG_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // half of the free memory (the rest for the long-pair rows and the aligned-string matrices), at most 1 GiB
    const uint64_t per_pair = PAIR_BYTES + (strings ? 2 * out_stride + 8 : 0);
    const uint64_t budget = std::min<uint64_t>(PAIR_GROUP_BYTES, free_b / 2);
    const uint64_t group = std::min<uint64_t>(n_pairs, std::max<uint64_t>(1, budget / per_pair));
    uint32_t *d_pa = c.alloc<uint32_t>(group), *d_pb = c.alloc<uint32_t>(group);
    int64_t *d_sc = c.alloc<int64_t>(group), *d_ep = c.alloc<int64_t>(group);
    int32_t *d_ec = c.alloc<int32_t>(group);
    uint8_t *d_oa = nullptr, *d_ob = nullptr;
    uint32_t *d_len = nullptr;
    int32_t *d_st = nullptr;
    if (strings) {
        d_oa = c.alloc<uint8_t>(group * out_stride);
        d_ob = c.alloc<uint8_t>(group * out_stride);
        d_len = c.alloc<uint32_t>(group);
        d_st = c.alloc<int32_t>(group);
    }
    for (uint64_t g0 = 0; g0 < n_pairs; g0 += group) {
        const uint64_t ng = std::min(group, n_pairs - g0);
        c.put(d_pa, pair_a + g0, ng);
        c.put(d_pb, pair_b + g0, ng);
        if ((rc = c.error()) || (rc = launch_sw_score_pairs(A.base, A.off, n_seqs_a, max_la, B.base, B.off, n_seqs_b, max_lb, d_pa, d_pb, ng,
                                                            s, d_sc, d_ec, d_ep, c.st)))
            return rc;
        if (strings) {  // matrices sized by this group's longest a and b
            uint64_t ga = 0, gb = 0;
            for (uint64_t k = g0; k < g0 + ng; ++k) {
                ga = std::max(ga, offsets_a[pair_a[k] + 1] - offsets_a[pair_a[k]]);
                gb = std::max(gb, offsets_b[pair_b[k] + 1] - offsets_b[pair_b[k]]);
            }
            if ((rc = launch_sw_align_long(A.base, A.off, ng, ga, B.base, gb, 1, s, d_sc, d_ec, d_oa, d_ob, out_stride, d_len, d_st, c.st,
                                           B.off, d_pa, d_pb)))
                return rc;
        }
        c.download(score + g0, d_sc, ng);
        if (err_code) c.download(err_code + g0, d_ec, ng);
        if (err_pos) c.download(err_pos + g0, d_ep, ng);
        if (strings) {
            c.download(align_a + g0 * out_stride, d_oa, ng * out_stride);
            c.download(align_b + g0 * out_stride, d_ob, ng * out_stride);
            c.download(align_len + g0, d_len, ng);
            if (status) c.download(status + g0, d_st, ng);
        }
    }
    return c.finish();
}

static int score_pairs_dev(const AlignScoring &s, const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a,
                           uint64_t max_len_a, const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b,
                           uint64_t max_len_b, const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, int64_t *d_score,
                           int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (s.has_null() || (n_pairs && (!d_offsets_a || !d_offsets_b || !d_pair_a || !d_pair_b || !d_score))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    return launch_sw_score_pairs(d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b, d_offsets_b, n_seqs_b, max_len_b, d_pair_a,
                                 d_pair_b, n_pairs, s, d_score, d_err_code, d_err_pos, (cudaStream_t)stream);
}

int pg_sw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, false, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, nullptr, nullptr, 0, nullptr, nullptr);
}
int pg_nw_score_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, false, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, nullptr, nullptr, 0, nullptr, nullptr);
}
int pg_sw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, const int16_t *lut_a_host,
                          const int16_t *lut_b_host, const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return score_pairs_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 0}, d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b,
                           d_offsets_b, n_seqs_b, max_len_b, d_pair_a, d_pair_b, n_pairs, d_score, d_err_code, d_err_pos, stream);
}
int pg_nw_score_pairs_dev(const uint8_t *d_seqs_a, const uint64_t *d_offsets_a, uint64_t n_seqs_a, uint64_t max_len_a,
                          const uint8_t *d_seqs_b, const uint64_t *d_offsets_b, uint64_t n_seqs_b, uint64_t max_len_b,
                          const uint32_t *d_pair_a, const uint32_t *d_pair_b, uint64_t n_pairs, const int16_t *lut_a_host,
                          const int16_t *lut_b_host, const int64_t *table_host, int32_t n_a, int32_t n_b, int64_t gap,
                          int64_t *d_score, int32_t *d_err_code, int64_t *d_err_pos, void *stream) {
    return score_pairs_dev({lut_a_host, lut_b_host, table_host, n_a, n_b, gap, 1}, d_seqs_a, d_offsets_a, n_seqs_a, max_len_a, d_seqs_b,
                           d_offsets_b, n_seqs_b, max_len_b, d_pair_a, d_pair_b, n_pairs, d_score, d_err_code, d_err_pos, stream);
}
int pg_sw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 0}, true, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}
int pg_nw_align_pairs(const uint8_t *seqs_a, const uint64_t *offsets_a, uint64_t n_seqs_a, const uint8_t *seqs_b,
                      const uint64_t *offsets_b, uint64_t n_seqs_b, const uint32_t *pair_a, const uint32_t *pair_b, uint64_t n_pairs,
                      const int16_t *lut_a, const int16_t *lut_b, const int64_t *table, int32_t n_a, int32_t n_b, int64_t gap,
                      int64_t *score, int32_t *err_code, int64_t *err_pos, uint8_t *align_a, uint8_t *align_b, uint64_t out_stride,
                      uint32_t *align_len, int32_t *status) {
    return align_pairs_host({lut_a, lut_b, table, n_a, n_b, gap, 1}, true, seqs_a, offsets_a, n_seqs_a, seqs_b, offsets_b, n_seqs_b,
                            pair_a, pair_b, n_pairs, score, err_code, err_pos, align_a, align_b, out_stride, align_len, status);
}

// ---------------------------------------------------------------------------------
// SantaLucia Tm
// ---------------------------------------------------------------------------------
int pg_tm_batch_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n, double cp,
                    double na, double mg, double *d_tm, double *d_dh, double *d_ds, int32_t *d_status,
                    void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return launch_tm(d_bases, d_offsets, n, cp, na, mg, d_tm, d_dh, d_ds, d_status, (cudaStream_t)stream);
}

int pg_tm_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, double cp, double na,
                double mg, double *tm, double *dh, double *ds, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    double *d_tm = c.alloc<double>(n, true), *d_dh = c.alloc<double>(n, true), *d_ds = c.alloc<double>(n, true);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_tm(b.base, b.off, n, cp, na, mg, d_tm, d_dh, d_ds, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(tm, d_tm, n);
    c.download(dh, d_dh, n);
    c.download(ds, d_ds, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one primer is empty: primers.SantaLucia panics (index out of range)",
                            "at least one primer holds a byte >= 0x80 (unsupported: strings.ToUpper would re-encode it)");
}

int pg_design_primers_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n,
                            double target_tm, uint32_t *fwd_len, uint32_t *rev_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets || !fwd_len || !rev_len) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    uint32_t *d_f = c.alloc<uint32_t>(n), *d_r = c.alloc<uint32_t>(n);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_design_primers(b.base, b.off, n, target_tm, d_f, d_r, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(fwd_len, d_f, n);
    c.download(rev_len, d_r, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one sequence is exhausted before the target Tm: pcr.DesignPrimers panics (slice bounds out of range)",
                            "at least one sequence holds a byte >= 0x80 (unsupported)");
}

int pg_pcr_minimal_primer_batch(const uint8_t *bases, const uint64_t *offsets, uint64_t n, double target_tm,
                                uint32_t *min_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets || !min_len) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> b = c.ragged(bases, offsets, n);
    uint32_t *d_m = c.alloc<uint32_t>(n);
    int32_t *d_st = c.alloc<int32_t>(n);
    if ((rc = c.error()) || (rc = launch_minimal_primer(b.base, b.off, n, target_tm, d_m, d_st, c.st))) return rc;
    std::vector<int32_t> hst(n);
    c.download(min_len, d_m, n);
    c.download(hst.data(), d_st, n);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one primer is shorter than 7 nt: pcr.SimulateSimple panics (slice bounds out of range)",
                            "at least one primer holds a byte >= 0x80 (unsupported)");
}

int pg_find_sites_batch(const uint8_t *seqs, const uint64_t *seq_offsets, uint64_t n_seq, const uint8_t *patterns,
                        const uint64_t *pat_offsets, uint32_t n_pat, uint32_t flags, uint32_t *hit_seq, uint64_t *hit_pos,
                        uint32_t *hit_pat, uint64_t hits_cap, uint64_t *n_hits) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_hits) { set_error("null buffer"); return PG_ERR_ARG; }
    *n_hits = 0;
    if (n_seq == 0 || n_pat == 0) return PG_OK;
    if (!seq_offsets || !pat_offsets || (hits_cap && (!hit_seq || !hit_pos || !hit_pat))) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> sq = c.ragged(seqs, seq_offsets, n_seq);
    uint64_t max_pat_len;
    if ((rc = c.error()) || (rc = check_ragged(pat_offsets, n_pat, &max_pat_len))) return rc;
    const uint64_t sbytes = seq_offsets[n_seq] - seq_offsets[0], p0 = pat_offsets[0], pbytes = pat_offsets[n_pat] - p0;
    std::vector<uint64_t> poff(n_pat + 1);
    for (uint32_t q = 0; q <= n_pat; ++q) poff[q] = pat_offsets[q] - p0;  // the kernel stages patterns from offset 0
    const uint8_t *d_p = c.upload(patterns + p0, pbytes);
    const uint64_t *d_poff = c.upload(poff.data(), n_pat + 1);
    uint32_t *d_hs = c.alloc<uint32_t>(hits_cap), *d_hq = c.alloc<uint32_t>(hits_cap);
    uint64_t *d_hp = c.alloc<uint64_t>(hits_cap);
    unsigned long long *d_n = c.alloc<unsigned long long>(1, true);
    if ((rc = c.error()) || (rc = launch_find_sites(sq.base, sq.off, n_seq, sbytes, d_p, d_poff, n_pat, pbytes, flags, d_hs, d_hp, d_hq, hits_cap,
                                                    d_n, c.st)))
        return rc;
    return finish_capped(c, d_n, hits_cap, n_hits, {{hit_seq, d_hs, 4}, {hit_pos, d_hp, 8}, {hit_pat, d_hq, 4}}, "hits_cap", "occurrences");
}

static int fastq_ingest_dev_impl(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                                 uint64_t *d_offsets, uint64_t *d_spans, uint64_t records_cap, uint64_t *n_records,
                                 uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_records || !total_bases || !err_code || !err_line || !d_offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_fastq_ingest(d_text, nbytes, d_bases, bases_cap, d_offsets, records_cap, n_records, total_bases, err_code,
                               err_line, (cudaStream_t)stream, d_spans);
}

static int fastq_ingest_host_impl(const uint8_t *text, uint64_t nbytes, uint8_t *bases, uint64_t bases_cap,
                                  uint64_t *offsets, uint64_t *spans, uint64_t records_cap, uint64_t *n_records,
                                  uint64_t *total_bases, int32_t *err_code, uint64_t *err_line) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_records || !total_bases || !err_code || !err_line || !offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint8_t *d_text = c.upload(text, nbytes, 16);
    uint8_t *d_bases = c.alloc<uint8_t>(bases_cap + 16);
    uint64_t *d_off = c.alloc<uint64_t>(records_cap + 1), *d_spans = spans ? c.alloc<uint64_t>((records_cap + 1) * 4) : nullptr;
    if ((rc = c.error()) || (rc = launch_fastq_ingest(d_text, nbytes, d_bases, bases_cap, d_off, records_cap, n_records, total_bases, err_code,
                                                      err_line, c.st, d_spans)))
        return rc;
    c.download(bases, d_bases, *total_bases);
    c.download(offsets, d_off, *n_records + 1);
    c.download(spans, d_spans, *n_records * 4);
    return c.finish();
}

int pg_fastq_ingest_dev(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                        uint64_t *d_offsets, uint64_t records_cap, uint64_t *n_records,
                        uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, void *stream) {
    return fastq_ingest_dev_impl(d_text, nbytes, d_bases, bases_cap, d_offsets, nullptr, records_cap, n_records, total_bases, err_code, err_line, stream);
}
int pg_fastq_ingest_records_dev(const uint8_t *d_text, uint64_t nbytes, uint8_t *d_bases, uint64_t bases_cap,
                                uint64_t *d_offsets, uint64_t *d_spans, uint64_t records_cap, uint64_t *n_records,
                                uint64_t *total_bases, int32_t *err_code, uint64_t *err_line, void *stream) {
    if (!d_spans) { set_error("null spans"); return PG_ERR_ARG; }
    return fastq_ingest_dev_impl(d_text, nbytes, d_bases, bases_cap, d_offsets, d_spans, records_cap, n_records, total_bases, err_code, err_line, stream);
}
int pg_fastq_ingest(const uint8_t *text, uint64_t nbytes, uint8_t *bases, uint64_t bases_cap,
                    uint64_t *offsets, uint64_t records_cap, uint64_t *n_records,
                    uint64_t *total_bases, int32_t *err_code, uint64_t *err_line) {
    return fastq_ingest_host_impl(text, nbytes, bases, bases_cap, offsets, nullptr, records_cap, n_records, total_bases, err_code, err_line);
}
int pg_fastq_ingest_records(const uint8_t *text, uint64_t nbytes, uint8_t *bases, uint64_t bases_cap,
                            uint64_t *offsets, uint64_t *spans, uint64_t records_cap, uint64_t *n_records,
                            uint64_t *total_bases, int32_t *err_code, uint64_t *err_line) {
    if (!spans) { set_error("null spans"); return PG_ERR_ARG; }
    return fastq_ingest_host_impl(text, nbytes, bases, bases_cap, offsets, spans, records_cap, n_records, total_bases, err_code, err_line);
}

int pg_fasta_ingest_dev(const uint8_t *d_text, uint64_t nbytes, uint32_t max_line_size, uint32_t flags,
                        uint8_t *d_bases, uint64_t bases_cap, uint64_t *d_offsets, uint8_t *d_names,
                        uint64_t names_cap, uint64_t *d_name_offsets, uint64_t records_cap, uint64_t *n_records,
                        uint64_t *total_bases, uint64_t *total_name_bytes, int32_t *err_code, uint64_t *err_line,
                        void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_records || !total_bases || !total_name_bytes || !err_code || !err_line || !d_offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_fasta_ingest(d_text, nbytes, max_line_size, flags, d_bases, bases_cap, d_offsets, d_names, names_cap, d_name_offsets,
                               records_cap, n_records, total_bases, total_name_bytes, err_code, err_line, (cudaStream_t)stream);
}

int pg_fasta_ingest(const uint8_t *text, uint64_t nbytes, uint32_t max_line_size, uint32_t flags, uint8_t *bases,
                    uint64_t bases_cap, uint64_t *offsets, uint8_t *names, uint64_t names_cap, uint64_t *name_offsets,
                    uint64_t records_cap, uint64_t *n_records, uint64_t *total_bases, uint64_t *total_name_bytes,
                    int32_t *err_code, uint64_t *err_line) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_records || !total_bases || !total_name_bytes || !err_code || !err_line || !offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    const bool want_names = names != nullptr || name_offsets != nullptr;
    if (want_names && (!names || !name_offsets)) { set_error("names and name_offsets must be given together"); return PG_ERR_ARG; }
    HostCall c;
    const uint8_t *d_text = c.upload(text, nbytes, 16);
    uint8_t *d_bases = c.alloc<uint8_t>(bases_cap + 16), *d_names = want_names ? c.alloc<uint8_t>(names_cap + 16) : nullptr;
    uint64_t *d_off = c.alloc<uint64_t>(records_cap + 1), *d_noff = want_names ? c.alloc<uint64_t>(records_cap + 1) : nullptr;
    if ((rc = c.error()) || (rc = launch_fasta_ingest(d_text, nbytes, max_line_size, flags, d_bases, bases_cap, d_off, d_names, names_cap, d_noff,
                                                      records_cap, n_records, total_bases, total_name_bytes, err_code, err_line, c.st)))
        return rc;
    c.download(bases, d_bases, *total_bases);
    c.download(offsets, d_off, *n_records + 1);
    c.download(names, d_names, *total_name_bytes);
    c.download(name_offsets, d_noff, *n_records + 1);
    return c.finish();
}

// ---------------------------------------------------------------------------------
static int seqhash_check(int32_t seq_type, uint32_t flags) {
    if (seq_type < PG_SEQHASH_DNA || seq_type > PG_SEQHASH_PROTEIN) {
        set_error("seq_type %d is not PG_SEQHASH_DNA, _RNA or _PROTEIN", seq_type);
        return PG_ERR_ARG;
    }
    if (flags & ~(PG_SEQHASH_CIRCULAR | PG_SEQHASH_DOUBLE_STRANDED)) {
        set_error("unknown seqhash flag bits 0x%x", flags);
        return PG_ERR_ARG;
    }
    return PG_OK;
}

int pg_seqhash_batch_dev(const uint8_t *d_seqs, const uint64_t *d_offsets, uint64_t n, int32_t seq_type, uint32_t flags,
                         uint8_t *d_digest, int32_t *d_err_code, uint64_t *d_err_pos, uint64_t max_len, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK || (rc = seqhash_check(seq_type, flags)) != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!d_offsets || !d_digest) { set_error("null offsets or digest"); return PG_ERR_ARG; }
    cudaStream_t st = (cudaStream_t)stream;
    uint64_t first = 0, last = 0;  // the scratch is sized by the total length
    PG_CUDA(cudaMemcpyAsync(&first, d_offsets, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaMemcpyAsync(&last, d_offsets + n, 8, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    if (last < first) { set_error("offsets[n] < offsets[0]"); return PG_ERR_ARG; }
    return launch_seqhash(d_seqs, d_offsets, n, max_len, last - first, seq_type, flags, d_digest, d_err_code, d_err_pos, st);
}

int pg_seqhash_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int32_t seq_type, uint32_t flags, uint8_t *digest,
                     int32_t *err_code, uint64_t *err_pos) {
    int rc = ensure_device();
    if (rc != PG_OK || (rc = seqhash_check(seq_type, flags)) != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    uint64_t max_len;  // the whole batch is checked before the first group is launched
    if ((rc = check_ragged(offsets, n, &max_len)) != PG_OK) return rc;
    if (!digest) { set_error("null digest"); return PG_ERR_ARG; }
    // Sequences go to the device in groups whose device memory stays within the budget (a single longer
    // sequence is a group of its own): input and canonical copy, one 32-byte chaining value per KiB and
    // per sequence, offsets, orientation, error and digest words per sequence.
    uint64_t budget = 2ull << 30;
    if (const char *e = getenv("PG_SEQHASH_GROUP_BYTES")) budget = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    auto cost = [&](uint64_t g, uint64_t e) {
        const uint64_t bytes = offsets[e] - offsets[g], cnt = e - g;
        return 2 * bytes + 64 + 32 * (bytes / 1024 + cnt) + 101 * cnt;
    };
    for (uint64_t g = 0; g < n;) {
        uint64_t e = g + 1;
        while (e < n && cost(g, e + 1) <= budget) ++e;
        const uint64_t cnt = e - g;
        HostCall c;
        const Ragged<uint8_t> in = c.ragged(seqs, offsets + g, cnt);
        uint8_t *d_dig = c.alloc<uint8_t>(cnt * 32);
        int32_t *d_err = c.alloc<int32_t>(cnt);
        uint64_t *d_pos = c.alloc<uint64_t>(cnt);
        if ((rc = c.error()) || (rc = launch_seqhash(in.base, in.off, cnt, in.max_len, offsets[e] - offsets[g], seq_type, flags, d_dig, d_err, d_pos,
                                                     c.st)))
            return rc;
        c.download(digest + 32 * g, d_dig, cnt * 32);
        c.download(err_code ? err_code + g : nullptr, d_err, cnt);
        c.download(err_pos ? err_pos + g : nullptr, d_pos, cnt);
        if ((rc = c.finish()) != PG_OK) return rc;
        g = e;
    }
    return PG_OK;
}

int pg_least_rotation_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, uint64_t *rotation) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    if (!rotation) { set_error("null rotation"); return PG_ERR_ARG; }
    HostCall c;
    const Ragged<uint8_t> in = c.ragged(seqs, offsets, n);
    uint64_t *d_rot = c.alloc<uint64_t>(n);
    if ((rc = c.error()) || (rc = launch_least_rotation(in.base, in.off, n, in.max_len, d_rot, c.st))) return rc;
    c.download(rotation, d_rot, n);
    return c.finish();
}

// ---- fold.Zuker (fold.cu) -----------------------------------------------------------------------------
int pg_fold_zuker_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, double temp, double *mfe, uint8_t *dot_bracket,
                        uint64_t *db_len, int32_t *status) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n == 0) return PG_OK;
    if (!offsets) { set_error("null offsets"); return PG_ERR_ARG; }
    uint64_t max_len;  // the whole batch is checked before the first group is launched
    if ((rc = check_ragged(offsets, n, &max_len)) != PG_OK) return rc;
    if (!mfe || !dot_bracket || !db_len) { set_error("null mfe, dot_bracket or db_len"); return PG_ERR_ARG; }
    // Items go to the device in groups whose scratch (V and W cells, branch lists) and input stay within the
    // budget; a single item over it is a group of its own.
    uint64_t budget = 8ull << 30;
    if (const char *e = getenv("PG_FOLD_GROUP_BYTES")) budget = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    const std::vector<uint8_t> tables = fold_tables(temp);
    std::vector<int32_t> hst(n);
    std::vector<uint64_t> scr;
    for (uint64_t g = 0; g < n;) {
        scr.assign(1, 0);
        uint64_t e = g;
        do {
            scr.push_back(scr.back() + fold_scratch_bytes(offsets[e + 1] - offsets[e]));
            ++e;
        } while (e < n && scr.back() + fold_scratch_bytes(offsets[e + 1] - offsets[e]) + 2 * (offsets[e + 1] - offsets[g]) + 64 * (e + 1 - g) <= budget);
        const uint64_t cnt = e - g, bytes = offsets[e] - offsets[g];
        HostCall c;
        const Ragged<uint8_t> in = c.ragged(seqs, offsets + g, cnt);
        uint8_t *d_tab = c.upload(tables.data(), tables.size());
        uint64_t *d_scr_off = c.upload(scr.data(), cnt);
        uint8_t *d_scratch = c.alloc<uint8_t>(std::max<uint64_t>(scr.back(), 8));
        double *d_mfe = c.alloc<double>(cnt);
        uint8_t *d_db = c.alloc<uint8_t>(bytes);
        uint64_t *d_len = c.alloc<uint64_t>(cnt);
        int32_t *d_st = c.alloc<int32_t>(cnt);
        if ((rc = c.error()) || (rc = launch_fold_zuker(in.base, in.off, cnt, d_tab, d_scratch, d_scr_off, d_mfe, d_db, d_len, d_st, c.st))) return rc;
        c.download(mfe + g, d_mfe, cnt);
        c.download(dot_bracket + (offsets[g] - offsets[0]), d_db, bytes);
        c.download(db_len + g, d_len, cnt);
        c.download(hst.data() + g, d_st, cnt);
        if ((rc = c.finish()) != PG_OK) return rc;
        g = e;
    }
    return fold_item_status(hst, status, "at least one sequence makes fold.Zuker panic (empty, 1 nt, or a traceback index out of range)",
                            "at least one sequence holds a byte >= 0x80 or is longer than PG_FOLD_MAX_LEN (unsupported)");
}

// ---- synthesis/fragment (fragment.cu) -------------------------------------------------------------------
static uint64_t fragment_budget() {
    uint64_t budget = 4ull << 30;
    if (const char *e = getenv("PG_FRAGMENT_GROUP_BYTES")) budget = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    return budget;
}

int pg_fragment_batch(const uint8_t *seqs, const uint64_t *offsets, uint64_t n, int64_t min_size, int64_t max_size, const uint8_t *exclude,
                      const uint64_t *exclude_offsets, uint64_t n_exclude, const uint8_t *include, const uint64_t *include_offsets,
                      uint64_t n_include, int32_t *status, double *efficiency, int64_t *err_min, int64_t *err_max, uint64_t *frag_offsets,
                      uint64_t *ends, uint64_t ends_cap, uint64_t *n_ends) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_ends || !frag_offsets) { set_error("null n_ends or frag_offsets"); return PG_ERR_ARG; }
    *n_ends = 0;
    frag_offsets[0] = 0;
    if (n == 0) return PG_OK;
    if (!offsets || !efficiency || !err_min || !err_max || (ends_cap && !ends) || (n_exclude && !exclude_offsets) || (n_include && !include_offsets)) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    uint64_t max_len, widest;  // the whole batch and both lists are checked before the first group is launched
    if ((rc = check_ragged(offsets, n, &max_len)) || (n_exclude && (rc = check_ragged(exclude_offsets, n_exclude, &widest))) ||
        (n_include && (rc = check_ragged(include_offsets, n_include, &widest))))
        return rc;
    if ((offsets[n] > offsets[0] && !seqs) || (n_exclude && exclude_offsets[n_exclude] > exclude_offsets[0] && !exclude) ||
        (n_include && include_offsets[n_include] > include_offsets[0] && !include)) {
        set_error("null seqs, exclude or include with non-empty entries");
        return PG_ERR_ARG;
    }
    const FragmentHost h = fragment_host(exclude, exclude_offsets, n_exclude, include, include_offsets, n_include);
    // Items go to the device in groups whose input and worst-case ends region stay within the budget; a single
    // item over it is a group of its own.  The per-warp scratch gets another budget's worth at most.
    const uint64_t budget = fragment_budget();
    auto item_bytes = [&](uint64_t i) { return (offsets[i + 1] - offsets[i]) + 8 * fragment_max_ends(offsets[i + 1] - offsets[i]) + 64; };
    std::vector<int32_t> hst(n);
    std::vector<uint64_t> region_off, cnt, out_off;
    uint64_t total = 0;
    for (uint64_t g = 0; g < n;) {
        uint64_t e = g, bytes = 0, group_max = 0;
        do {
            bytes += item_bytes(e);
            group_max = std::max(group_max, offsets[e + 1] - offsets[e]);
            ++e;
        } while (e < n && bytes + item_bytes(e) <= budget);
        const uint64_t m = e - g;
        region_off.assign(1, 0);
        for (uint64_t i = g; i < e; ++i) region_off.push_back(region_off.back() + fragment_max_ends(offsets[i + 1] - offsets[i]));
        HostCall c;
        const Ragged<uint8_t> in = c.ragged(seqs, offsets + g, m);
        FragmentArgs a{};
        a.seqs = in.base;
        a.off = in.off;
        a.n = m;
        a.min_size = min_size;
        a.max_size = max_size;
        a.fid = c.upload(h.fid.data(), h.fid.size());
        a.r_ex = c.upload(h.r_ex.data(), h.r_ex.size());
        a.ex_mask = c.upload(h.ex_mask.data(), 8);
        a.inc_mask = c.upload(h.inc_mask.data(), 8);
        a.ex_keys = c.upload(h.ex_keys.data(), h.ex_keys.size());
        a.n_ex_keys = h.ex_keys.size();
        a.ex_other = c.upload(h.ex_other.data(), h.ex_other.size());
        a.n_ex_other = h.ex_other.size();
        a.inc_other = c.upload(h.inc_other.data(), h.inc_other.size());
        a.n_inc_other = h.inc_other.size();
        a.has_include = n_include > 0;
        a.status = c.alloc<int32_t>(m);
        a.eff = c.alloc<double>(m);
        a.err_min = c.alloc<int64_t>(m);
        a.err_max = c.alloc<int64_t>(m);
        a.n_ends = c.alloc<uint64_t>(m);
        a.ends = c.alloc<uint64_t>(region_off.back());
        a.ends_off = c.upload(region_off.data(), m + 1);
        StreamScratch work(c.st);
        if ((rc = c.error()) || (rc = launch_fragment(a, group_max, budget, work, c.st))) return rc;
        cnt.resize(m);
        c.download(hst.data() + g, a.status, m);
        c.download(efficiency + g, a.eff, m);
        c.download(err_min + g, a.err_min, m);
        c.download(err_max + g, a.err_max, m);
        c.download(cnt.data(), a.n_ends, m);
        if ((rc = c.sync())) return rc;
        out_off.assign(1, 0);
        for (uint64_t i = 0; i < m; ++i) {
            out_off.push_back(out_off.back() + cnt[i]);
            frag_offsets[g + i + 1] = total + out_off.back();
        }
        if (total + out_off.back() <= ends_cap && out_off.back()) {
            const uint64_t *d_out_off = c.upload(out_off.data(), m + 1);
            uint64_t *d_out = c.alloc<uint64_t>(out_off.back());
            if ((rc = c.error()) || (rc = launch_fragment_compact(a.ends, a.ends_off, a.n_ends, d_out_off, m, d_out, c.st))) return rc;
            c.download(ends + total, d_out, out_off.back());
        }
        if ((rc = c.finish())) return rc;
        total += out_off.back();
        g = e;
    }
    *n_ends = total;
    if (total > ends_cap) {
        fold_item_status(hst, status, "", "");
        set_error("the batch has %llu fragment ends: ends_cap %llu", (unsigned long long)total, (unsigned long long)ends_cap);
        return PG_ERR_ARG;
    }
    return fold_item_status(hst, status, "at least one sequence is shorter than 4 bytes: fragment.Fragment panics (slice bounds out of range)",
                            "at least one sequence holds a byte >= 0x80 (unsupported)");
}

// SetEfficiency (next = 0) or NextOverhangs (next = 1) of every set, in groups of sets under the budget
static int overhang_sets(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets, int next,
                         uint8_t *cands, uint32_t *n_cands, double *efficiency) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_sets == 0) return PG_OK;
    if (!set_offsets || !efficiency || (next && (!cands || !n_cands))) { set_error("null buffer"); return PG_ERR_ARG; }
    uint64_t widest;
    if ((rc = check_ragged(set_offsets, n_sets, &widest))) return rc;
    const uint64_t n_ov = set_offsets[n_sets];
    if (n_ov && !overhang_offsets) { set_error("null overhang_offsets"); return PG_ERR_ARG; }
    if (n_ov && (rc = check_ragged(overhang_offsets, n_ov, &widest))) return rc;
    if (n_ov && overhang_offsets[n_ov] > overhang_offsets[0] && !overhangs) { set_error("null overhangs with non-empty entries"); return PG_ERR_ARG; }
    // the most keyed members of any set bounds the per-warp spill of its key list (every 4-byte member may be one)
    uint64_t max_keys = 0;
    for (uint64_t s = 0; s < n_sets; ++s) {
        uint64_t k = 0;
        for (uint64_t j = set_offsets[s]; j < set_offsets[s + 1]; ++j) k += overhang_offsets[j + 1] - overhang_offsets[j] == 4;
        max_keys = std::max(max_keys, k);
    }
    const FragmentHost h = fragment_host(nullptr, nullptr, 0, nullptr, nullptr, 0);
    const uint64_t budget = fragment_budget(), per_set = next ? 256 * (4 + 8) + 4 : 8;
    const uint64_t group = std::max<uint64_t>(1, budget / per_set);
    HostCall c;
    const uint64_t zero = 0;
    const Ragged<uint8_t> in = n_ov ? c.ragged(overhangs, overhang_offsets, n_ov) : Ragged<uint8_t>{nullptr, c.upload(&zero, 1), 0};
    SetArgs a{};
    a.fid = c.upload(h.fid.data(), h.fid.size());
    a.ov = in.base;
    a.ov_off = in.off;
    a.set_off = c.upload(set_offsets, n_sets + 1);
    a.next = next;
    const uint64_t m0 = std::min(group, n_sets);
    a.eff = c.alloc<double>(next ? 256 * m0 : m0);
    if (next) {
        a.cands = c.alloc<uint8_t>(1024 * m0);
        a.n_cands = c.alloc<uint32_t>(m0);
    }
    if ((rc = c.error())) return rc;
    for (uint64_t g = 0; g < n_sets; g += group) {
        a.first = g;
        a.n_sets = std::min(group, n_sets - g);
        StreamScratch work(c.st);
        if ((rc = launch_overhang_sets(a, max_keys, budget, work, c.st))) return rc;
        c.download(efficiency + (next ? 256 * g : g), a.eff, next ? 256 * a.n_sets : a.n_sets);
        if (next) {
            c.download(cands + 1024 * g, a.cands, 1024 * a.n_sets);
            c.download(n_cands + g, a.n_cands, a.n_sets);
        }
        if ((rc = c.sync())) return rc;
    }
    return c.finish();
}

int pg_fragment_set_efficiency_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     double *efficiency) {
    return overhang_sets(overhangs, overhang_offsets, set_offsets, n_sets, 0, nullptr, nullptr, efficiency);
}

int pg_fragment_next_overhangs_batch(const uint8_t *overhangs, const uint64_t *overhang_offsets, const uint64_t *set_offsets, uint64_t n_sets,
                                     uint8_t *cands, uint32_t *n_cands, double *efficiency) {
    return overhang_sets(overhangs, overhang_offsets, set_offsets, n_sets, 1, cands, n_cands, efficiency);
}

// ---- clone: CutWithEnzyme, CircularLigate, GoldenGate (clone.cu, clone_host.cpp) ---------------------
}  // extern "C"

namespace pg {
namespace {
// pg_clone_enzyme -> the kernels' form.  A site that is empty, longer than CLONE_MAX_SITE or holds a byte
// outside 0x01..0x7f is not a literal this library matches: PG_ERR_UNSUPPORTED.
int clone_enzyme(const pg_clone_enzyme &in, CloneEnzyme *out) {
    if (!in.forward_site || !in.reverse_site || (in.recognition_len && !in.recognition_site)) { set_error("null enzyme site"); return PG_ERR_ARG; }
    CloneEnzyme e{};
    for (int which = 0; which < 2; ++which) {
        const uint8_t *site = which ? in.reverse_site : in.forward_site;
        const uint32_t len = which ? in.reverse_len : in.forward_len;
        if (len == 0 || len > CLONE_MAX_SITE) { set_error("enzyme site of %u bytes: only literal sites of 1..%u bytes are supported", len, CLONE_MAX_SITE); return PG_ERR_UNSUPPORTED; }
        for (uint32_t j = 0; j < len; ++j) {
            if (site[j] == 0 || site[j] >= 0x80) { set_error("enzyme site byte 0x%02x is not supported", site[j]); return PG_ERR_UNSUPPORTED; }
            (which ? e.rsite : e.fsite)[j] = site[j];
        }
        (which ? e.rl : e.fl) = len;
    }
    e.recl = in.recognition_len;
    e.palindromic = 1;  // checks.IsPalindromic: RecognitionSite == transform.ReverseComplement(RecognitionSite)
    for (uint32_t j = 0; j < in.recognition_len; ++j)
        if (in.recognition_site[j] != complement(in.recognition_site[in.recognition_len - 1 - j])) e.palindromic = 0;
    e.skip = in.skip;
    e.ohl = in.overhang_length;
    *out = e;
    return PG_OK;
}

// The fragments of every reaction, on the host (for the enumeration) and in one device source buffer: the
// Sequence bytes at [0, seq_total), the overhang bytes after them.
struct LigationInput {
    const uint8_t *d_src;
    const uint8_t *seq, *oh;
    const uint64_t *seq_off, *oh_off;  // as pg_clone_digest_batch's outputs, from 0
    uint64_t seq_total;
    std::vector<uint64_t> reaction_frags;  // reaction r = fragments [reaction_frags[r], reaction_frags[r+1])
    std::vector<int32_t> status;           // per reaction: PG_ITEM_OK, or why it is not ligated
};

struct LigationOutput {
    uint64_t bytes_cap, constructs_cap;
    uint8_t *out, *kinds, *digests;
    uint64_t *construct_offsets, *counts, *need_bytes, *need_constructs;
    int32_t *status;
};

uint64_t clone_group_budget() {
    uint64_t budget = 1ull << 30;
    if (const char *e = getenv("PG_CLONE_GROUP_BYTES")) budget = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
    return budget;
}

// Enumerate every reaction on the host, materialise and seqhash its emits on the device in groups under a
// memory budget, keep the first emit of each seqhash per reaction, and copy back the kept survivors.
int ligate_reactions(HostCall &c, const LigationInput &in, const LigationOutput &o) {
    const uint64_t R = in.reaction_frags.size() - 1;
    LigationPlan plan;
    std::vector<uint64_t> reaction_emits(R + 1, 0);
    std::unordered_map<std::string, uint64_t> interned;
    for (uint64_t r = 0; r < R; ++r) {
        reaction_emits[r] = plan.emits.size();
        if (in.status[r] != PG_ITEM_OK) continue;
        std::vector<LigFragment> frags;
        for (uint64_t f = in.reaction_frags[r]; f < in.reaction_frags[r + 1]; ++f) {
            const uint64_t s0 = in.seq_off[f], s1 = in.seq_off[f + 1], o0 = in.oh_off[2 * f], o1 = in.oh_off[2 * f + 1], o2 = in.oh_off[2 * f + 2];
            if (s1 - s0 > UINT32_MAX || o2 - o0 > UINT32_MAX) { set_error("fragment %llu is longer than 4 GiB", (unsigned long long)f); return PG_ERR_ARG; }
            const uint64_t id = interned.emplace(std::string((const char *)in.seq + s0, s1 - s0), interned.size()).first->second;
            frags.push_back(LigFragment{id, std::string((const char *)in.oh + o0, o1 - o0), std::string((const char *)in.oh + o1, o2 - o1), s0,
                                        in.seq_total + o0, in.seq_total + o1, (uint32_t)(s1 - s0)});
        }
        enumerate_ligation(frags, o.bytes_cap, o.constructs_cap, plan);
    }
    reaction_emits[R] = plan.emits.size();
    *o.need_bytes = plan.bytes;
    *o.need_constructs = plan.n_emits;
    if (plan.over) {
        set_error("the ligations emit %llu constructs of %llu bytes in all: constructs_cap %llu, bytes_cap %llu", (unsigned long long)plan.n_emits,
                  (unsigned long long)plan.bytes, (unsigned long long)o.constructs_cap, (unsigned long long)o.bytes_cap);
        return PG_ERR_ARG;
    }
    for (uint64_t r = 0; r < 2 * R; ++r) o.counts[r] = 0;
    o.construct_offsets[0] = 0;
    const uint64_t budget = clone_group_budget(), n_emits = plan.emits.size();
    std::unordered_set<std::string> seen;  // existingSeqhashes of the current reaction
    uint64_t r = 0, n_out = 0, out_bytes = 0;
    for (uint64_t g = 0; g < n_emits;) {
        uint64_t e = g, bytes = 0;
        while (e < n_emits && (e == g || bytes + plan.emits[e].bytes <= budget)) bytes += plan.emits[e++].bytes;
        // group layout: closed clones first, then looping constructs, so that each kind is one ragged batch
        std::vector<uint64_t> at(e - g), off_c{0}, off_l;
        uint64_t max_c = 0, max_l = 0;
        for (uint64_t k = g; k < e; ++k)
            if (plan.emits[k].kind == 0) {
                at[k - g] = off_c.back();
                off_c.push_back(off_c.back() + plan.emits[k].bytes);
                max_c = std::max(max_c, plan.emits[k].bytes);
            }
        off_l.push_back(off_c.back());
        for (uint64_t k = g; k < e; ++k)
            if (plan.emits[k].kind == 1) {
                at[k - g] = off_l.back();
                off_l.push_back(off_l.back() + plan.emits[k].bytes);
                max_l = std::max(max_l, plan.emits[k].bytes);
            }
        std::vector<Piece> pieces(plan.pieces.begin() + plan.emits[g].piece_begin, plan.pieces.begin() + plan.emits[e - 1].piece_end);
        for (uint64_t k = g; k < e; ++k)
            for (uint64_t i = plan.emits[k].piece_begin; i < plan.emits[k].piece_end; ++i) pieces[i - plan.emits[g].piece_begin].dst += at[k - g];
        const uint64_t nc = off_c.size() - 1, nl = off_l.size() - 1, n = e - g;
        StreamScratch gs(c.st);
        uint8_t *d_buf = nullptr, *d_dig = nullptr;
        Piece *d_pieces = nullptr;
        uint64_t *d_offc = nullptr, *d_offl = nullptr, *d_pos = nullptr;
        int32_t *d_err = nullptr;
        int rc;
        if ((rc = scratch_alloc(gs, &d_buf, bytes)) || (rc = scratch_alloc(gs, &d_pieces, pieces.size())) || (rc = scratch_alloc(gs, &d_offc, nc + 1)) ||
            (rc = scratch_alloc(gs, &d_offl, nl + 1)) || (rc = scratch_alloc(gs, &d_dig, 32 * n)) || (rc = scratch_alloc(gs, &d_err, n)) ||
            (rc = scratch_alloc(gs, &d_pos, n)))
            return rc;
        c.put(d_pieces, pieces.data(), pieces.size());
        c.put(d_offc, off_c.data(), nc + 1);
        c.put(d_offl, off_l.data(), nl + 1);
        if ((rc = c.error()) || (rc = launch_clone_pieces(in.d_src, d_pieces, pieces.size(), d_buf, c.st))) return rc;
        // seqhash.Hash(construct, "DNA", true, true) for clones (clone.go:275), (.., false, true) for loops (:305)
        if (nc && (rc = launch_seqhash(d_buf, d_offc, nc, max_c, off_c[nc], PG_SEQHASH_DNA, PG_SEQHASH_CIRCULAR | PG_SEQHASH_DOUBLE_STRANDED, d_dig,
                                       d_err, d_pos, c.st)))
            return rc;
        if (nl && (rc = launch_seqhash(d_buf, d_offl, nl, max_l, off_l[nl] - off_l[0], PG_SEQHASH_DNA, PG_SEQHASH_DOUBLE_STRANDED, d_dig + 32 * nc,
                                       d_err + nc, d_pos + nc, c.st)))
            return rc;
        std::vector<uint8_t> dig(32 * n);
        std::vector<int32_t> err(n);
        c.download(dig.data(), d_dig, 32 * n);
        c.download(err.data(), d_err, n);
        if ((rc = c.sync())) return rc;
        // dedup in emit order; the survivors are compacted on the device and come back in one copy
        std::vector<Piece> keep;
        uint64_t kept_bytes = 0, ic = 0, il = 0;
        for (uint64_t k = g; k < e; ++k) {
            while (k >= reaction_emits[r + 1]) {
                ++r;
                seen.clear();
            }
            const Emit &em = plan.emits[k];
            const uint64_t slot = em.kind == 0 ? ic++ : nc + il++;
            std::string key = err[slot] ? std::string() : std::string(1, (char)(em.kind + 1)) + std::string((const char *)&dig[32 * slot], 32);
            if (!seen.insert(std::move(key)).second || !em.kept) continue;
            keep.push_back(Piece{at[k - g], kept_bytes, (uint32_t)em.bytes, 0});
            kept_bytes += em.bytes;
            o.counts[2 * r + em.kind] += 1;
            if (o.kinds) o.kinds[n_out] = em.kind;
            if (o.digests) memcpy(o.digests + 32 * n_out, &dig[32 * slot], 32);
            o.construct_offsets[n_out + 1] = o.construct_offsets[n_out] + em.bytes;
            ++n_out;
        }
        if (!keep.empty()) {
            uint8_t *d_keep = nullptr;
            Piece *d_kp = nullptr;
            if ((rc = scratch_alloc(gs, &d_keep, kept_bytes)) || (rc = scratch_alloc(gs, &d_kp, keep.size()))) return rc;
            c.put(d_kp, keep.data(), keep.size());
            if ((rc = c.error()) || (rc = launch_clone_pieces(d_buf, d_kp, keep.size(), d_keep, c.st))) return rc;
            c.download(o.out + out_bytes, d_keep, kept_bytes);
            if ((rc = c.sync())) return rc;
        }
        out_bytes += kept_bytes;
        g = e;
    }
    return PG_OK;
}

// reaction statuses -> `status` and the call's code, as fold_item_status
int ligation_status(const std::vector<int32_t> &st, int32_t *status) {
    return fold_item_status(st, status, "at least one reaction cuts a part where clone.CutWithEnzyme panics (slice bounds out of range)",
                            "at least one reaction has a part with a byte >= 0x80 (unsupported)");
}

// Before anything is uploaded: the item count fits in 64 bits, and no item can hold 2^32 matches of a site
// (the walks count them in 32 bits; a part read doubled has at most 2 L / site length of them).
int clone_batch_check(const uint64_t *part_offsets, uint64_t n_parts, const std::vector<CloneEnzyme> &enz) {
    if (n_parts > UINT64_MAX / enz.size()) { set_error("n_parts x n_enzymes overflows"); return PG_ERR_ARG; }
    uint64_t max_len;
    int rc = check_ragged(part_offsets, n_parts, &max_len);
    if (rc != PG_OK) return rc;
    for (const CloneEnzyme &e : enz) {
        const uint64_t site = e.palindromic ? e.fl : std::min(e.fl, e.rl);
        if (max_len > UINT64_MAX / 2 || 2 * max_len / site > UINT32_MAX) {
            set_error("a part of %llu bytes could hold 2^32 or more matches of a %u-byte site", (unsigned long long)max_len, site);
            return PG_ERR_ARG;
        }
    }
    return PG_OK;
}

bool ligation_output_ok(const LigationOutput &o) {
    if (!o.construct_offsets || !o.counts || !o.need_bytes || !o.need_constructs || (o.bytes_cap && !o.out)) {
        set_error("null buffer");
        return false;
    }
    return true;
}
}  // namespace
}  // namespace pg

extern "C" {

int pg_clone_digest_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                          const pg_clone_enzyme *enzymes, uint32_t n_enzymes, int32_t directional, uint32_t *frag_count, int32_t *status,
                          uint8_t *seq_bytes, uint64_t seq_cap, uint64_t *seq_offsets, uint8_t *oh_bytes, uint64_t oh_cap,
                          uint64_t *oh_offsets, uint64_t frag_cap, uint64_t *n_frags, uint64_t *n_seq_bytes, uint64_t *n_oh_bytes) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (!n_frags || !n_seq_bytes || !n_oh_bytes) { set_error("null buffer"); return PG_ERR_ARG; }
    *n_frags = *n_seq_bytes = *n_oh_bytes = 0;
    if (n_parts == 0 || n_enzymes == 0) return PG_OK;
    if (!part_offsets || !circular || !enzymes || !frag_count || !seq_offsets || !oh_offsets || (seq_cap && !seq_bytes) || (oh_cap && !oh_bytes)) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    std::vector<CloneEnzyme> enz(n_enzymes);
    for (uint32_t k = 0; k < n_enzymes; ++k)
        if ((rc = clone_enzyme(enzymes[k], &enz[k])) != PG_OK) return rc;
    if ((rc = clone_batch_check(part_offsets, n_parts, enz)) != PG_OK) return rc;
    const uint64_t n_items = n_parts * n_enzymes;
    HostCall c;
    const Ragged<uint8_t> in = c.ragged(parts, part_offsets, n_parts);
    const uint8_t *d_circ = c.upload(circular, n_parts);
    const CloneEnzyme *d_enz = c.upload(enz.data(), n_enzymes);
    if ((rc = c.error())) return rc;
    StreamScratch work(c.st);
    DigestPlan d;
    if ((rc = clone_digest_plan(in.base, in.off, d_circ, n_parts, d_enz, n_enzymes, directional != 0, work, c.st, &d))) return rc;
    std::vector<int32_t> hst(n_items);
    std::vector<uint64_t> cnt(n_items);
    c.download(hst.data(), d.status, n_items);
    c.download(cnt.data(), d.n_frag, n_items);
    if ((rc = c.sync())) return rc;
    for (uint64_t i = 0; i < n_items; ++i) frag_count[i] = (uint32_t)cnt[i];
    *n_frags = d.frags;
    *n_seq_bytes = d.seq_total;
    *n_oh_bytes = d.oh_total;
    if (d.frags > frag_cap || d.seq_total > seq_cap || d.oh_total > oh_cap) {
        fold_item_status(hst, status, "", "");
        set_error("the digest gives %llu fragments, %llu sequence bytes and %llu overhang bytes: frag_cap %llu, seq_cap %llu, oh_cap %llu",
                  (unsigned long long)d.frags, (unsigned long long)d.seq_total, (unsigned long long)d.oh_total, (unsigned long long)frag_cap,
                  (unsigned long long)seq_cap, (unsigned long long)oh_cap);
        return PG_ERR_ARG;
    }
    uint64_t *d_soff = c.alloc<uint64_t>(d.frags + 1), *d_ooff = c.alloc<uint64_t>(2 * d.frags + 1);
    uint8_t *d_seq = c.alloc<uint8_t>(d.seq_total), *d_oh = c.alloc<uint8_t>(d.oh_total);
    if ((rc = c.error()) || (rc = clone_digest_write(d, d_soff, d_seq, d_ooff, d_oh, work, c.st))) return rc;
    c.download(seq_offsets, d_soff, d.frags + 1);
    c.download(oh_offsets, d_ooff, 2 * d.frags + 1);
    c.download(seq_bytes, d_seq, d.seq_total);
    c.download(oh_bytes, d_oh, d.oh_total);
    if ((rc = c.finish())) return rc;
    return fold_item_status(hst, status, "at least one item panics in clone.CutWithEnzyme (slice bounds out of range)",
                            "at least one part holds a byte >= 0x80 (unsupported)");
}

int pg_clone_golden_gate_batch(const uint8_t *parts, const uint64_t *part_offsets, const uint8_t *circular, uint64_t n_parts,
                               const uint64_t *reaction_offsets, uint64_t n_reactions, const pg_clone_enzyme *enzyme, uint64_t bytes_cap,
                               uint64_t constructs_cap, uint8_t *out, uint64_t *construct_offsets, uint8_t *kinds, uint8_t *digests,
                               uint64_t *counts, int32_t *status, uint64_t *need_bytes, uint64_t *need_constructs) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    const LigationOutput o{bytes_cap, constructs_cap, out, kinds, digests, construct_offsets, counts, need_bytes, need_constructs, status};
    if (!ligation_output_ok(o) || !reaction_offsets || !enzyme || (n_parts && (!part_offsets || !circular))) {
        set_error("null buffer");
        return PG_ERR_ARG;
    }
    *need_bytes = *need_constructs = 0;
    uint64_t widest;
    if ((rc = check_ragged(reaction_offsets, n_reactions, &widest))) return rc;
    if (reaction_offsets[0] != 0 || reaction_offsets[n_reactions] != n_parts) { set_error("reaction_offsets must run from 0 to n_parts"); return PG_ERR_ARG; }
    CloneEnzyme enz;
    if ((rc = clone_enzyme(*enzyme, &enz))) return rc;
    if (n_parts && (rc = clone_batch_check(part_offsets, n_parts, {enz}))) return rc;
    HostCall c;
    LigationInput in;
    in.status.assign(n_reactions, PG_ITEM_OK);
    in.reaction_frags.assign(n_reactions + 1, 0);
    std::vector<uint8_t> seq, oh;
    std::vector<uint64_t> soff{0}, ooff{0};
    StreamScratch work(c.st);
    uint8_t *d_src = nullptr;
    if (n_parts) {
        const Ragged<uint8_t> p = c.ragged(parts, part_offsets, n_parts);
        const uint8_t *d_circ = c.upload(circular, n_parts);
        const CloneEnzyme *d_enz = c.upload(&enz, 1);
        DigestPlan d;
        if ((rc = c.error()) || (rc = clone_digest_plan(p.base, p.off, d_circ, n_parts, d_enz, 1, 1, work, c.st, &d))) return rc;
        // the fragments stay on the device as the ligation's source: Sequence bytes, then overhang bytes
        uint64_t *d_soff = c.alloc<uint64_t>(d.frags + 1), *d_ooff = c.alloc<uint64_t>(2 * d.frags + 1);
        d_src = c.alloc<uint8_t>(d.seq_total + d.oh_total);
        if ((rc = c.error()) || (rc = clone_digest_write(d, d_soff, d_src, d_ooff, d_src + d.seq_total, work, c.st))) return rc;
        std::vector<int32_t> pst(n_parts);
        std::vector<uint64_t> cnt(n_parts);
        seq.resize(d.seq_total);
        oh.resize(d.oh_total);
        soff.resize(d.frags + 1);
        ooff.resize(2 * d.frags + 1);
        c.download(pst.data(), d.status, n_parts);
        c.download(cnt.data(), d.n_frag, n_parts);
        c.download(soff.data(), d_soff, d.frags + 1);
        c.download(ooff.data(), d_ooff, 2 * d.frags + 1);
        c.download(seq.data(), d_src, d.seq_total);
        c.download(oh.data(), d_src + d.seq_total, d.oh_total);
        if ((rc = c.sync())) return rc;
        for (uint64_t r = 0; r < n_reactions; ++r) {
            uint64_t nf = 0;
            for (uint64_t q = reaction_offsets[r]; q < reaction_offsets[r + 1]; ++q) {
                nf += cnt[q];
                if (pst[q] != PG_ITEM_OK && in.status[r] == PG_ITEM_OK) in.status[r] = pst[q];  // GoldenGate stops at the first
            }
            in.reaction_frags[r + 1] = in.reaction_frags[r] + nf;
        }
        in.seq_total = d.seq_total;
    } else {
        in.seq_total = 0;
    }
    in.d_src = d_src;
    in.seq = seq.data();
    in.oh = oh.data();
    in.seq_off = soff.data();
    in.oh_off = ooff.data();
    if ((rc = ligate_reactions(c, in, o))) return rc;
    if ((rc = c.finish())) return rc;
    return ligation_status(in.status, status);
}

int pg_clone_circular_ligate_batch(const uint8_t *seq_bytes, const uint64_t *seq_offsets, const uint8_t *oh_bytes, const uint64_t *oh_offsets,
                                   uint64_t n_frags, const uint64_t *reaction_offsets, uint64_t n_reactions, uint64_t bytes_cap,
                                   uint64_t constructs_cap, uint8_t *out, uint64_t *construct_offsets, uint8_t *kinds, uint8_t *digests,
                                   uint64_t *counts, uint64_t *need_bytes, uint64_t *need_constructs) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    const LigationOutput o{bytes_cap, constructs_cap, out, kinds, digests, construct_offsets, counts, need_bytes, need_constructs, nullptr};
    if (!ligation_output_ok(o) || !reaction_offsets || !seq_offsets || !oh_offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    *need_bytes = *need_constructs = 0;
    uint64_t widest;
    if ((rc = check_ragged(reaction_offsets, n_reactions, &widest)) || (rc = check_ragged(seq_offsets, n_frags, &widest)) ||
        (rc = check_ragged(oh_offsets, 2 * n_frags, &widest)))
        return rc;
    if (reaction_offsets[0] != 0 || reaction_offsets[n_reactions] != n_frags) { set_error("reaction_offsets must run from 0 to n_frags"); return PG_ERR_ARG; }
    // offsets from 0, as the digest writes them
    const uint64_t s0 = seq_offsets[0], o0 = oh_offsets[0], S = seq_offsets[n_frags] - s0, O = oh_offsets[2 * n_frags] - o0;
    std::vector<uint64_t> soff(n_frags + 1), ooff(2 * n_frags + 1);
    for (uint64_t f = 0; f <= n_frags; ++f) soff[f] = seq_offsets[f] - s0;
    for (uint64_t f = 0; f <= 2 * n_frags; ++f) ooff[f] = oh_offsets[f] - o0;
    // seqhash.Hash upper-cases with strings.ToUpper, which maps some non-ASCII letters into the alphabet
    // (U+017F -> S, U+212A -> K): a byte >= 0x80 is not hashed here, so such fragments are refused
    for (uint64_t i = 0; i < S; ++i)
        if (seq_bytes[s0 + i] >= 0x80) { set_error("fragment sequence byte %llu is >= 0x80 (unsupported)", (unsigned long long)(s0 + i)); return PG_ERR_UNSUPPORTED; }
    for (uint64_t i = 0; i < O; ++i)
        if (oh_bytes[o0 + i] >= 0x80) { set_error("overhang byte %llu is >= 0x80 (unsupported)", (unsigned long long)(o0 + i)); return PG_ERR_UNSUPPORTED; }
    HostCall c;
    uint8_t *d_src = c.alloc<uint8_t>(S + O);
    if (d_src) {
        c.put(d_src, seq_bytes + s0, S);
        c.put(d_src + S, oh_bytes + o0, O);
    }
    if ((rc = c.error())) return rc;
    LigationInput in{d_src, seq_bytes + s0, oh_bytes + o0, soff.data(), ooff.data(), S,
                     std::vector<uint64_t>(reaction_offsets, reaction_offsets + n_reactions + 1), std::vector<int32_t>(n_reactions, PG_ITEM_OK)};
    if ((rc = ligate_reactions(c, in, o))) return rc;
    return c.finish();
}

// ---------------------------------------------------------------------------------
int pg_synth_reads_dev(uint8_t *d_bases, uint64_t first_read, uint64_t n_reads, uint32_t read_len,
                       uint64_t seed, int32_t kind, uint32_t family, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    return launch_synth_reads(d_bases, first_read, n_reads, read_len, seed, kind, family, (cudaStream_t)stream);
}

}  // extern "C"
