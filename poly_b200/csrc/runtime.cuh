// runtime.cuh -- what the entry files of the C ABI (api_*.cu) share (internal): the per-device contexts
// and device selection, the staging of the one-shot host-pointer entry points, and the rule that cuts a
// batch into groups under a device-memory budget.  runtime.cu holds the runtime itself.
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <initializer_list>
#include <mutex>
#include <thread>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace pg {

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

// the context the calling thread's entry point runs on (ensure_device, use_device), nullptr before the first
DevCtx *cur_ctx();
// binds the calling thread's later entry points to `device` as pg_thread_device does, without touching the device yet
void bind_thread_device(int device);
int device_count_checked(int *n);
int use_device(int device);
int ensure_device();

// Staging for the one-shot host-pointer entry points: every step of such a call goes through a HostCall.

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
inline int check_ragged(const uint64_t *offsets, uint64_t n, uint64_t *max_len) {
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
    HostCall() : lock_(cur_ctx()->mu), tmp_(cur_ctx()->slots[0].stream), st(cur_ctx()->slots[0].stream) {}
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
inline int fold_item_status(const std::vector<int32_t> &hst, int32_t *status, const char *panic_msg, const char *unsupported_msg) {
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
inline int finish_capped(HostCall &c, const unsigned long long *d_n, uint64_t cap, uint64_t *n_out, std::initializer_list<CappedList> lists,
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

// Batched entry points send their items to the device in groups under a byte budget: the default of the
// entry point, or PG_GROUP_BYTES when that is set.
uint64_t group_budget(uint64_t default_bytes);

// The end of the group that starts at item g of n: the largest e > g with cost(g) + ... + cost(e - 1) <= budget,
// or g + 1 when item g alone is over the budget.
template <typename Cost>
uint64_t group_end(uint64_t g, uint64_t n, uint64_t budget, Cost cost) {
    uint64_t e = g + 1, sum = cost(g);
    for (; e < n; ++e) {
        const uint64_t c = cost(e);
        if (sum + c > budget) break;
        sum += c;
    }
    return e;
}

}  // namespace pg
