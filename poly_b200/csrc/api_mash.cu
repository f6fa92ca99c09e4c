// api_mash.cu -- the C ABI of poly's mash: Sketch on device and host buffers (the pipelined host path),
// the single-process multi-GPU entry points, Similarity / Distance, the groups and the representatives of a
// sketch set, the sketch index and the screen.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <functional>
#include <sched.h>
#include <shared_mutex>
#include <string>
#include <thread>
#include <vector>

#include "runtime.cuh"

struct pg_mash_index {
    int device;
    uint32_t *d_sk;        // the index's own copy of the n x s reference sketches
    pg::DistancePlan plan;  // sortedness flags + join index over d_sk
    mutable std::shared_mutex rw;  // queries hold it shared while they read the plan and enqueue, an add exclusively
};

struct pg_mash_dereplicator {
    int device;
    int32_t s;
    uint32_t min_same, flags;
    pg_mash_index *ix;  // the kept representatives, in id order; callers borrow it for queries
    uint32_t *d_ids;    // ix's reference p is sketch d_ids[p] (ascending), ix->plan.n entries
    uint64_t n;         // sketches added so far: the next batch's first id
    mutable std::mutex mu;  // serialises adds, and reps against them
};

struct pg_mash_clusterer {
    int device;
    int32_t s;
    uint32_t min_same;
    pg_mash_index *ix;      // every sketch added, in id order; callers borrow it for queries
    uint32_t *d_label;      // label[i] = the smallest id of sketch i's group, ix->plan.n entries
    uint64_t n, n_groups;   // sketches added so far (the next batch's first id) and their groups
    mutable std::mutex mu;  // serialises adds, and label reads against them
};

struct pg_mash_screen {
    int device;
    int32_t k;
    pg::ScreenIndex ix;            // the sorted reference keys, their distinct values and the pool counts
    mutable std::shared_mutex rw;  // results hold it shared while they enqueue, an add or a reset exclusively
};

struct pg_mash_sketcher {
    int device;
    pg::SketcherState st;
    cudaEvent_t read;       // recorded behind every rows_dev: an add waits for it before it frees the old state
    mutable std::mutex mu;  // serialises adds, and rows against them
};

namespace pg {
namespace {

static inline uint64_t kmers_of(uint64_t len, int k) { return len > (uint64_t)k ? len - (uint64_t)k : 0; }
// informative words of the sketch of a read of `len` bytes
static inline uint64_t sketch_words(uint64_t len, int k, int s) { return std::min<uint64_t>(kmers_of(len, k), (uint64_t)s); }

// Rows [rb, re) of the n x s sketches' matching counts and/or distances into host arrays that start at row rb, in
// row blocks of <= 64 Mi pairs, each copied out and waited for before the next
int rows_to_host(const uint32_t *d_sk, uint64_t n, int s, uint64_t rb, uint64_t re, uint32_t *same, double *distance, cudaStream_t st) {
    const uint64_t rows_per = std::max<uint64_t>(8, ((64ull << 20) / n) & ~7ull);
    return distance_plan_tiles(d_sk, n, s, rb, re, rows_per, same != nullptr, distance != nullptr, st,
                               [&](const uint32_t *d_same, const double *d_dist, uint64_t b, uint64_t e) {
        const uint64_t cells = (e - b) * n;
        if (same) PG_CUDA(cudaMemcpyAsync(same + (b - rb) * n, d_same, cells * 4, cudaMemcpyDeviceToHost, st));
        if (distance) PG_CUDA(cudaMemcpyAsync(distance + (b - rb) * n, d_dist, cells * 8, cudaMemcpyDeviceToHost, st));
        PG_CUDA(cudaStreamSynchronize(st));
        return PG_OK;
    });
}

static int check_rows(uint64_t n, uint64_t row_begin, uint64_t row_end) {
    if (row_end > n || row_begin > row_end) { set_error("bad row range"); return PG_ERR_ARG; }
    return PG_OK;
}
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
        : cx_(*cur_ctx()), lock_(cx_.mu), q_(q), keep_tail_((q.flags & PG_SKETCH_TAIL_KEEP) != 0), stage_in_(is_pageable(q.bases)),
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
            bind_thread_device(dev[r]);  // this worker's entry points run on its device
            pg_numa_bind_thread(dev[r], nullptr);  // best effort: staging copies from the GPU's NUMA node
            int wrc = ensure_device();
            if (wrc == PG_OK) wrc = SketchPipe(shard).run();
            res[r].rc = wrc;
            if (wrc != PG_OK) res[r].msg = pg_last_error();
        });
    }
    for (std::thread &t : th) t.join();
    return fold_results(res);
}

static int index_create(const uint32_t *src, bool src_dev, uint64_t n, int32_t s, cudaStream_t st, pg_mash_index **out) {
    if (n && s <= 0) { set_error("index over sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    pg_mash_index *ix = new pg_mash_index{cur_ctx()->device, nullptr, DistancePlan()};
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

// Appends m rows of size s from src (checked by the caller, who holds ix->rw exclusively): a new copy of the n + m
// rows and the plan grown over it; the index takes both only once they are complete, so on an error it keeps
// what it held.
static int index_add(pg_mash_index *ix, const uint32_t *src, bool src_dev, uint64_t m, int32_t s, cudaStream_t st) {
    const uint64_t n = ix->plan.n, old_words = n * (uint64_t)s, words = old_words + m * (uint64_t)s;
    uint32_t *d_sk = nullptr;
    cudaError_t e = cudaMallocAsync(&d_sk, words * 4, st);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("cudaMallocAsync(%llu) for the index failed", (unsigned long long)(words * 4)); return PG_ERR_NOMEM; }
    if (old_words) e = cudaMemcpyAsync(d_sk, ix->d_sk, old_words * 4, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_sk + old_words, src, (words - old_words) * 4, src_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st);
    int rc = e == cudaSuccess ? PG_OK : cuda_fail(e, "index copy", __FILE__, __LINE__);
    DistancePlan plan;
    if (rc == PG_OK) rc = distance_plan_grow(ix->plan, d_sk, m, s, st, &plan);
    if (rc == PG_OK) { e = cudaStreamSynchronize(st); if (e != cudaSuccess) rc = cuda_fail(e, "index add", __FILE__, __LINE__); }
    if (rc != PG_OK) {
        distance_plan_destroy(plan, st);
        cudaFreeAsync(d_sk, st);
        cudaStreamSynchronize(st);
        return rc;
    }
    distance_plan_destroy(ix->plan, st);
    if (ix->d_sk) cudaFreeAsync(ix->d_sk, st);
    ix->d_sk = d_sk;
    ix->plan = plan;
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// The argument rules of pg_mash_index_add after the null index and m == 0, in their order
static int index_add_check(const pg_mash_index *ix, const void *sketches, uint64_t m, int32_t s) {
    if (s <= 0) { set_error("index over sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    if (ix->plan.n && s != ix->plan.s) { set_error("sketches of size %d added to an index of size %d", s, ix->plan.s); return PG_ERR_ARG; }
    if (m > 0xffffffffull - ix->plan.n) { set_error("%llu + %llu references exceed 2^32 - 1", (unsigned long long)ix->plan.n, (unsigned long long)m); return PG_ERR_ARG; }
    if (!sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    return PG_OK;
}

// The argument rules of pg_mash_dereplicator_add after the null dereplicator and m == 0, in their order
static int derep_add_check(const pg_mash_dereplicator *d, const void *sketches, uint64_t m, int32_t s, const void *rep) {
    if (s <= 0) { set_error("sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    if (s != d->s) { set_error("sketches of size %d added to a dereplication of size %d", s, d->s); return PG_ERR_ARG; }
    if (m > 0xffffffffull - d->n) { set_error("%llu + %llu sketches exceed 2^32 - 1", (unsigned long long)d->n, (unsigned long long)m); return PG_ERR_ARG; }
    if (!sketches || !rep) { set_error("null buffer"); return PG_ERR_ARG; }
    return PG_OK;
}

// One batch of m rows on the device (checked by the caller, who holds d->mu and d->ix->rw exclusively): the batch's
// global assignments into d_rep (and, when rep is not NULL, copied to the host with the count's one sync), then
// the new representatives appended to the representative index and to the ids.  The dereplicator takes the grown
// index, ids and n only once everything has succeeded, so on an error it keeps what it held.
static int derep_add(pg_mash_dereplicator *d, const uint32_t *d_b, uint64_t m, uint32_t *d_rep, uint32_t *rep, uint64_t *n_new,
                     cudaStream_t st) {
    const uint64_t R = d->ix->plan.n, s = (uint64_t)d->s;
    const uint32_t base = (uint32_t)d->n;
    StreamScratch tmp(st);
    unsigned long long *d_cnt = nullptr;
    PG_CUDA(tmp.alloc(&d_cnt, 1));
    int rc = launch_mash_derep_add(d->ix->plan, d->d_ids, d_b, m, d->s, d->min_same, d->flags, base, d_rep, d_cnt, st);
    if (rc != PG_OK) return rc;
    unsigned long long cnt = 0;
    PG_CUDA(cudaMemcpyAsync(&cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
    if (rep) PG_CUDA(cudaMemcpyAsync(rep, d_rep, m * 4, cudaMemcpyDeviceToHost, st));
    PG_CUDA(cudaStreamSynchronize(st));
    if (cnt) {
        uint32_t *d_rows = nullptr, *d_ids = nullptr;
        if (tmp.alloc(&d_rows, cnt * s) != cudaSuccess || cudaMallocAsync(&d_ids, (R + cnt) * 4, st) != cudaSuccess) {
            cudaGetLastError();
            set_error("cudaMallocAsync for %llu new representatives failed", cnt);
            return PG_ERR_NOMEM;
        }
        cudaError_t e = R ? cudaMemcpyAsync(d_ids, d->d_ids, R * 4, cudaMemcpyDeviceToDevice, st) : cudaSuccess;
        rc = e == cudaSuccess ? launch_derep_gather(d_b, m, d->s, base, d_rep, cnt, d_rows, d_ids + R, st) : cuda_fail(e, "ids copy", __FILE__, __LINE__);
        if (rc == PG_OK) rc = index_add(d->ix, d_rows, true, cnt, d->s, st);  // synchronises; takes the rows only on success
        if (rc != PG_OK) {
            cudaFreeAsync(d_ids, st);
            cudaStreamSynchronize(st);
            return rc;
        }
        if (d->d_ids) cudaFreeAsync(d->d_ids, st);
        d->d_ids = d_ids;
    }
    d->n += m;
    *n_new = cnt;
    return PG_OK;
}

// The argument rules of pg_mash_clusterer_add after the null clusterer and m == 0, in their order
static int cluster_add_check(const pg_mash_clusterer *c, const void *sketches, uint64_t m, int32_t s) {
    if (s <= 0) { set_error("sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    if (s != c->s) { set_error("sketches of size %d added to a clustering of size %d", s, c->s); return PG_ERR_ARG; }
    if (m > 0xffffffffull - c->n) { set_error("%llu + %llu sketches exceed 2^32 - 1", (unsigned long long)c->n, (unsigned long long)m); return PG_ERR_ARG; }
    if (!sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    return PG_OK;
}

// One batch of m rows on the device (checked by the caller, who holds c->mu and c->ix->rw exclusively): the labels
// of all n + m sketches into a new array, the batch's slice of them into d_out or out (either may be NULL), the
// counts into cnt (links, groups, merged), then the batch appended to the index.  The clusterer takes the new
// labels, n and the group count only once everything has succeeded, so on an error it keeps what it held.
static int cluster_add(pg_mash_clusterer *c, const uint32_t *d_b, uint64_t m, uint32_t *d_out, uint32_t *out, unsigned long long cnt[3],
                       cudaStream_t st) {
    const uint64_t n = c->n;
    StreamScratch tmp(st), keep(st);  // keep: the new labels, released unless the add succeeds
    unsigned long long *d_cnt = nullptr;
    uint32_t *d_label = nullptr;
    PG_CUDA(tmp.alloc(&d_cnt, 3));
    if (keep.alloc(&d_label, n + m) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync(%llu) for the labels failed", (unsigned long long)((n + m) * 4));
        return PG_ERR_NOMEM;
    }
    int rc = launch_mash_cluster_add(c->ix->plan, c->d_label, d_b, m, c->s, c->min_same, d_label, d_cnt, st);
    if (rc != PG_OK) return rc;
    PG_CUDA(cudaMemcpyAsync(cnt, d_cnt, 24, cudaMemcpyDeviceToHost, st));
    if (out) PG_CUDA(cudaMemcpyAsync(out, d_label + n, m * 4, cudaMemcpyDeviceToHost, st));
    if (d_out) PG_CUDA(cudaMemcpyAsync(d_out, d_label + n, m * 4, cudaMemcpyDeviceToDevice, st));
    PG_CUDA(cudaStreamSynchronize(st));
    if ((rc = index_add(c->ix, d_b, true, m, c->s, st)) != PG_OK) return rc;  // synchronises; takes the rows only on success
    keep.ptr.clear();
    if (c->d_label) cudaFreeAsync(c->d_label, st);
    c->d_label = d_label;
    c->n = n + m;
    c->n_groups = cnt[1];
    return PG_OK;
}

// The k-mer mode rules that follow the k < 0 rule of the grouped sketch, the sketcher and the screen: a known flag, and a
// strand to choose (k >= 1) in canonical mode
static int kmer_flags_check(int32_t k, uint32_t flags) {
    if (flags & ~(uint32_t)PG_KMER_CANONICAL) { set_error("unknown k-mer flags 0x%x", flags & ~(uint32_t)PG_KMER_CANONICAL); return PG_ERR_ARG; }
    if ((flags & PG_KMER_CANONICAL) && k == 0) { set_error("canonical k-mers of size 0: no strand to choose"); return PG_ERR_ARG; }
    return PG_OK;
}

// The argument rules of pg_mash_screen_create after the null out pointer, in their order
static int screen_create_check(const void *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags) {
    if (k < 0) { set_error("k-mer size %d < 0", k); return PG_ERR_ARG; }
    if (int rc = kmer_flags_check(k, flags)) return rc;
    if (n && s <= 0) { set_error("screen over sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    if (n > 0xffffffffull) { set_error("%llu references exceed 2^32 - 1", (unsigned long long)n); return PG_ERR_ARG; }
    if (n_samples == 0) { set_error("a screen of 0 samples"); return PG_ERR_ARG; }
    if (n && !sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    return PG_OK;
}

static pg_mash_screen *screen_new(int32_t k, uint32_t flags, ScreenIndex ix) {
    ix.canon = (flags & PG_KMER_CANONICAL) != 0;
    return new pg_mash_screen{cur_ctx()->device, k, ix};
}

static int screen_create_host(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags, pg_mash_screen **out) {
    if (!out) { set_error("null screen pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = screen_create_check(sketches, n, s, k, n_samples, flags);
    if (rc != PG_OK || (rc = ensure_device()) != PG_OK) return rc;
    ScreenIndex ix;
    {
        HostCall c;
        const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)std::max(s, 0));
        if ((rc = c.error()) || (rc = screen_build(d_sk, n, s, n_samples, c.st, &ix))) return rc;
        if ((rc = c.finish()) != PG_OK) {
            screen_free(ix, c.st);
            return rc;
        }
    }
    *out = screen_new(k, flags, ix);
    return PG_OK;
}

static int screen_create_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags, void *stream,
                             pg_mash_screen **out) {
    if (!out) { set_error("null screen pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = screen_create_check(d_sketches, n, s, k, n_samples, flags);
    if (rc != PG_OK || (rc = ensure_device()) != PG_OK) return rc;
    ScreenIndex ix;
    if ((rc = screen_build(d_sketches, n, s, n_samples, (cudaStream_t)stream, &ix)) != PG_OK) return rc;
    *out = screen_new(k, flags, ix);
    return PG_OK;
}

// A host add; ids == null: every read is sample 0.  The ids are checked against the screen's samples before any
// copy or launch.
static int screen_add_host(pg_mash_screen *sc, const uint8_t *bases, const uint64_t *offsets, const uint32_t *ids, uint64_t n_reads) {
    if (!sc) { set_error("null screen"); return PG_ERR_ARG; }
    if (n_reads == 0) return PG_OK;
    if (!bases || !offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    const uint32_t samples = sc->ix.samples;  // fixed at creation
    if (ids)
        for (uint64_t i = 0; i < n_reads; ++i)
            if (ids[i] >= samples) {
                set_error("read %llu has sample id %u, the screen has %u samples", (unsigned long long)i, ids[i], samples);
                return PG_ERR_ARG;
            }
    int rc = use_device(sc->device);
    if (rc != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> lk(sc->rw);
    HostCall c;
    const Ragged<uint8_t> r = c.ragged(bases, offsets, n_reads);
    const uint32_t *d_ids = ids ? c.upload(ids, n_reads) : nullptr;
    if ((rc = c.error()) || (rc = screen_add(sc->ix, sc->k, r.base, r.off, d_ids, n_reads, c.st))) return rc;
    return c.finish();
}

// add_dev and add_samples_dev; ids == null: every read is sample 0
static int screen_add_dev(pg_mash_screen *sc, const uint8_t *d_bases, const uint64_t *d_offsets, const uint32_t *d_ids, uint64_t n_reads,
                          void *stream) {
    if (!sc) { set_error("null screen"); return PG_ERR_ARG; }
    if (n_reads == 0) return PG_OK;
    if (!d_bases || !d_offsets) { set_error("null buffer"); return PG_ERR_ARG; }
    int rc = use_device(sc->device);
    if (rc != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> lk(sc->rw);
    return screen_add(sc->ix, sc->k, d_bases, d_offsets, d_ids, n_reads, (cudaStream_t)stream);
}

// results and winners: the same rules, locking and copies around a different tally, over rows [first, first + count)
using ScreenTally = int (*)(const ScreenIndex &, uint32_t, uint32_t, uint32_t *, double *, uint64_t *, cudaStream_t);

static int screen_rows_check(const pg_mash_screen *sc, uint32_t first, uint32_t count) {
    if (!sc) { set_error("null screen"); return PG_ERR_ARG; }
    if ((uint64_t)first + count > sc->ix.samples) {
        set_error("rows [%u, %llu) of a screen of %u samples", first, (unsigned long long)first + count, sc->ix.samples);
        return PG_ERR_ARG;
    }
    return PG_OK;
}

static int screen_tally_host(const pg_mash_screen *sc, ScreenTally tally, uint32_t first, uint32_t count, uint32_t *shared, double *containment,
                             uint64_t *multiplicity) {
    int rc = screen_rows_check(sc, first, count);
    if (rc != PG_OK || (rc = use_device(sc->device)) != PG_OK) return rc;
    std::shared_lock<std::shared_mutex> lk(sc->rw);
    const uint64_t m = sc->ix.n * count;
    if (m == 0 || (!shared && !containment && !multiplicity)) return PG_OK;
    HostCall c;
    uint32_t *d_sh = shared ? c.alloc<uint32_t>(m) : nullptr;
    double *d_c = containment ? c.alloc<double>(m) : nullptr;
    uint64_t *d_m = multiplicity ? c.alloc<uint64_t>(m) : nullptr;
    if ((rc = c.error()) || (rc = tally(sc->ix, first, count, d_sh, d_c, d_m, c.st))) return rc;
    c.download(shared, d_sh, m);
    c.download(containment, d_c, m);
    c.download(multiplicity, d_m, m);
    return c.finish();
}

static int screen_tally_dev(const pg_mash_screen *sc, ScreenTally tally, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_containment,
                            uint64_t *d_multiplicity, void *stream) {
    int rc = screen_rows_check(sc, first, count);
    if (rc != PG_OK || (rc = use_device(sc->device)) != PG_OK) return rc;
    std::shared_lock<std::shared_mutex> lk(sc->rw);
    return tally(sc->ix, first, count, d_shared, d_containment, d_multiplicity, (cudaStream_t)stream);
}

// The argument rules of pg_mash_sketch_groups and its _dev form that need no buffer, in their order
static int sketch_groups_check(uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t flags, uint64_t row_stride, const void *out,
                               const void *count) {
    if (n_groups && (!out || !count)) { set_error("null out or count"); return PG_ERR_ARG; }
    if (k < 0) { set_error("kmerSize %d < 0: the reference panics (slice bounds)", k); return PG_ERR_ARG; }
    if (int rc = kmer_flags_check(k, flags)) return rc;
    if (s < 1) { set_error("sketchSize %d < 1: a grouped sketch holds at least one value", s); return PG_ERR_ARG; }
    if (min_copies < 1) { set_error("min_copies 0: every value occurs at least once"); return PG_ERR_ARG; }
    if (row_stride < (uint64_t)s) { set_error("row_stride %llu < sketchSize %d", (unsigned long long)row_stride, s); return PG_ERR_ARG; }
    return PG_OK;
}

// The argument rules of pg_mash_sketcher_add and its _dev form that need no buffer content, in their order; *work:
// whether the add has records to count
static int sketcher_add_check(const pg_mash_sketcher *sk, const void *bases, const uint64_t *offsets, uint64_t n_records, const void *group_offsets,
                              uint64_t first, uint64_t nb, bool host, bool *work) {
    *work = false;
    if (!sk) { set_error("null sketcher"); return PG_ERR_ARG; }
    if (n_records == 0 && nb == 0) return PG_OK;
    if (first > sk->st.G || nb > sk->st.G - first) {
        set_error("groups [%llu, %llu + %llu) of a sketcher of %llu groups", (unsigned long long)first, (unsigned long long)first,
                  (unsigned long long)nb, (unsigned long long)sk->st.G);
        return PG_ERR_ARG;
    }
    if (n_records == 0) return PG_OK;
    // bases may be null in the host add when the records hold no byte
    if (!offsets || !group_offsets || (!bases && (!host || offsets[n_records] != offsets[0]))) { set_error("null buffer"); return PG_ERR_ARG; }
    *work = true;
    return PG_OK;
}

// The argument rules of pg_mash_sketcher_rows and its _dev form, in their order
static int sketcher_rows_check(const pg_mash_sketcher *sk, uint64_t first, uint64_t count, const void *out, uint64_t row_stride, const void *n_values) {
    if (!sk) { set_error("null sketcher"); return PG_ERR_ARG; }
    if (first > sk->st.G || count > sk->st.G - first) {
        set_error("rows [%llu, %llu + %llu) of a sketcher of %llu groups", (unsigned long long)first, (unsigned long long)first,
                  (unsigned long long)count, (unsigned long long)sk->st.G);
        return PG_ERR_ARG;
    }
    if (row_stride < (uint64_t)sk->st.s) { set_error("row_stride %llu < sketchSize %d", (unsigned long long)row_stride, sk->st.s); return PG_ERR_ARG; }
    if (count && (!out || !n_values)) { set_error("null out or n_values"); return PG_ERR_ARG; }
    return PG_OK;
}

// The argument rules of pg_mash_dist(_within) and their _dev forms that need no buffer content, in their order.
// need_len: a p-value is computed.
static int dist_check(uint64_t nq, uint64_t nr, int32_t s, int32_t k, uint64_t row_stride, const void *q_rows, const void *q_count, const void *r_rows,
                      const void *r_count, bool need_len, const void *q_length, const void *r_length) {
    if (nq > 0xffffffffull || nr > 0xffffffffull) {
        set_error("%llu queries x %llu references: each side holds at most 2^32 - 1 rows", (unsigned long long)nq, (unsigned long long)nr);
        return PG_ERR_ARG;
    }
    if (k < 1) { set_error("kmerSize %d < 1", k); return PG_ERR_ARG; }
    if (s < 1) { set_error("sketchSize %d < 1", s); return PG_ERR_ARG; }
    if (row_stride < (uint64_t)s) { set_error("row_stride %llu < sketchSize %d", (unsigned long long)row_stride, s); return PG_ERR_ARG; }
    if ((nq && (!q_rows || !q_count)) || (nr && (!r_rows || !r_count))) { set_error("null rows or count"); return PG_ERR_ARG; }
    if (need_len && ((nq && !q_length) || (nr && !r_length))) { set_error("null lengths: the p-value needs them"); return PG_ERR_ARG; }
    return PG_OK;
}

// the rules of the filtered form that follow dist_check, in their order
static int dist_within_check(uint64_t nq, uint64_t nr, double max_distance, double max_p_value, uint32_t flags, const void *pair_q, const void *pair_r,
                             const void *n_pairs) {
    if (std::isnan(max_distance) || std::isnan(max_p_value)) { set_error("NaN limit"); return PG_ERR_ARG; }
    if (flags & ~PG_PAIRS_UPPER) { set_error("unknown flag bits 0x%x", flags & ~PG_PAIRS_UPPER); return PG_ERR_ARG; }
    if ((flags & PG_PAIRS_UPPER) && nq != nr) {
        set_error("PG_PAIRS_UPPER needs one set: %llu queries, %llu references", (unsigned long long)nq, (unsigned long long)nr);
        return PG_ERR_ARG;
    }
    if (!pair_q || !pair_r || !n_pairs) { set_error("null pair_q, pair_r or n_pairs"); return PG_ERR_ARG; }
    return PG_OK;
}

// The host forms' checks of the rows themselves: counts <= s, strictly ascending rows, lengths >= 1
static int dist_rows_check(const uint32_t *rows, const uint32_t *count, uint64_t n, int32_t s, uint64_t row_stride, const uint64_t *len, const char *side) {
    for (uint64_t i = 0; i < n; ++i) {
        if (count[i] > (uint32_t)s) {
            set_error("%s row %llu holds %u values > sketchSize %d", side, (unsigned long long)i, count[i], s);
            return PG_ERR_ARG;
        }
        const uint32_t *row = rows + i * row_stride;
        for (uint32_t w = 1; w < count[i]; ++w)
            if (row[w] <= row[w - 1]) {
                set_error("%s row %llu is not strictly ascending at word %u", side, (unsigned long long)i, w);
                return PG_ERR_ARG;
            }
    }
    if (len)
        for (uint64_t i = 0; i < n; ++i)
            if (len[i] == 0) { set_error("%s length %llu is 0", side, (unsigned long long)i); return PG_ERR_ARG; }
    return PG_OK;
}

static DistArgs dist_args(const uint32_t *q_rows, const uint32_t *q_count, uint64_t nq, const uint32_t *r_rows, const uint32_t *r_count, uint64_t nr,
                          uint64_t row_stride, int32_t s, int32_t k, const uint64_t *q_len, const uint64_t *r_len) {
    DistArgs g{};
    g.q_rows = q_rows; g.q_count = q_count; g.r_rows = r_rows; g.r_count = r_count;
    g.nq = nq; g.nr = nr; g.stride = row_stride; g.s = s; g.k = k; g.q_len = q_len; g.r_len = r_len;
    return g;
}

// device bytes of the dense host form's outputs per block; the queries are cut into blocks that fit
constexpr uint64_t DIST_BLOCK_BYTES = 1ull << 30;

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

// ---------------------------------------------------------------------------------
// mash.Sketch
// ---------------------------------------------------------------------------------
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

int pg_mash_sketch_groups_flags(const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets,
                                uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t flags, uint32_t *out, uint64_t row_stride,
                                uint32_t *count) {
    int rc = sketch_groups_check(n_groups, k, s, min_copies, flags, row_stride, out, count);
    if (rc != PG_OK || n_groups == 0) return rc;
    if (!group_offsets || !offsets || (!bases && offsets[n_records] != offsets[0])) { set_error("null buffer"); return PG_ERR_ARG; }
    uint64_t longest = 0;  // the groups partition the records: ragged offsets over the records, from 0 to n_records
    if ((rc = check_ragged(group_offsets, n_groups, &longest)) != PG_OK) return rc;
    if (group_offsets[0] != 0 || group_offsets[n_groups] != n_records) {
        set_error("group offsets run from %llu to %llu, not over the %llu records", (unsigned long long)group_offsets[0],
                  (unsigned long long)group_offsets[n_groups], (unsigned long long)n_records);
        return PG_ERR_ARG;
    }
    if ((rc = check_ragged(offsets, n_records, &longest)) != PG_OK || (rc = ensure_device()) != PG_OK) return rc;
    HostCall c;
    const Ragged<uint8_t> r = c.ragged(bases, offsets, n_records);
    const uint64_t *d_goff = c.upload(group_offsets, n_groups + 1);
    uint32_t *d_out = c.alloc<uint32_t>(n_groups * row_stride);
    uint32_t *d_count = c.alloc<uint32_t>(n_groups);
    const bool canon = (flags & PG_KMER_CANONICAL) != 0;
    if ((rc = c.error()) || (rc = sketch_groups(r.base, r.off, n_records, d_goff, n_groups, k, s, min_copies, canon, d_out, row_stride, d_count, c.st)))
        return rc;
    c.download(out, d_out, n_groups * row_stride);
    c.download(count, d_count, n_groups);
    return c.finish();
}

int pg_mash_sketch_groups(const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets, uint64_t n_groups,
                          int32_t k, int32_t s, uint32_t min_copies, uint32_t *out, uint64_t row_stride, uint32_t *count) {
    return pg_mash_sketch_groups_flags(bases, offsets, n_records, group_offsets, n_groups, k, s, min_copies, 0, out, row_stride, count);
}

int pg_mash_sketch_groups_flags_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records, const uint64_t *d_group_offsets,
                                    uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t flags, uint32_t *d_out,
                                    uint64_t row_stride, uint32_t *d_count, void *stream) {
    int rc = sketch_groups_check(n_groups, k, s, min_copies, flags, row_stride, d_out, d_count);
    if (rc != PG_OK || n_groups == 0) return rc;
    if (!d_group_offsets || !d_offsets || (n_records && !d_bases)) { set_error("null buffer"); return PG_ERR_ARG; }
    if ((rc = ensure_device()) != PG_OK) return rc;
    return sketch_groups(d_bases, d_offsets, n_records, d_group_offsets, n_groups, k, s, min_copies, (flags & PG_KMER_CANONICAL) != 0, d_out,
                         row_stride, d_count, (cudaStream_t)stream);
}

int pg_mash_sketch_groups_dev(const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records, const uint64_t *d_group_offsets,
                              uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint32_t *d_out, uint64_t row_stride,
                              uint32_t *d_count, void *stream) {
    return pg_mash_sketch_groups_flags_dev(d_bases, d_offsets, n_records, d_group_offsets, n_groups, k, s, min_copies, 0, d_out, row_stride,
                                           d_count, stream);
}

int pg_mash_sketcher_create(uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint64_t max_values, pg_mash_sketcher **out) {
    return pg_mash_sketcher_create_flags(n_groups, k, s, min_copies, max_values, 0, out);
}

int pg_mash_sketcher_create_flags(uint64_t n_groups, int32_t k, int32_t s, uint32_t min_copies, uint64_t max_values, uint32_t flags,
                                  pg_mash_sketcher **out) {
    if (!out) { set_error("null sketcher pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    if (n_groups == 0 || n_groups > 0xffffffffull) { set_error("a sketcher of %llu groups: need 1 .. 2^32 - 1", (unsigned long long)n_groups); return PG_ERR_ARG; }
    if (k < 0) { set_error("kmerSize %d < 0: the reference panics (slice bounds)", k); return PG_ERR_ARG; }
    if (int rc = kmer_flags_check(k, flags)) return rc;
    if (s < 1) { set_error("sketchSize %d < 1: a grouped sketch holds at least one value", s); return PG_ERR_ARG; }
    if (min_copies < 1) { set_error("min_copies 0: every value occurs at least once"); return PG_ERR_ARG; }
    if (max_values < (uint64_t)s) { set_error("max_values %llu < sketchSize %d", (unsigned long long)max_values, s); return PG_ERR_ARG; }
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    pg_mash_sketcher *sk = nullptr;
    try {
        sk = new pg_mash_sketcher();
        sk->st.seg.reserve(n_groups + 1);
        sk->st.cap.reserve(n_groups);
    } catch (const std::bad_alloc &) {
        delete sk;
        set_error("host memory for %llu groups", (unsigned long long)n_groups);
        return PG_ERR_NOMEM;
    }
    sk->device = cur_ctx()->device;
    sk->st.G = n_groups;
    sk->st.B = max_values;
    sk->st.k = k;
    sk->st.s = s;
    sk->st.m = min_copies;
    sk->st.canon = (flags & PG_KMER_CANONICAL) != 0;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    cudaStream_t st = cur_ctx()->slots[0].stream;
    cudaError_t e = cudaEventCreateWithFlags(&sk->read, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        delete sk;
        return cuda_fail(e, "cudaEventCreate", __FILE__, __LINE__);
    }
    if ((rc = sketcher_init(sk->st, st)) != PG_OK) {
        cudaEventDestroy(sk->read);
        delete sk;
        return rc;
    }
    *out = sk;
    return PG_OK;
}

int pg_mash_sketcher_add(pg_mash_sketcher *sk, const uint8_t *bases, const uint64_t *offsets, uint64_t n_records, const uint64_t *group_offsets,
                         uint64_t first_group, uint64_t n_batch_groups) {
    bool work = false;
    int rc = sketcher_add_check(sk, bases, offsets, n_records, group_offsets, first_group, n_batch_groups, true, &work);
    if (rc != PG_OK || !work) return rc;
    uint64_t longest = 0;  // the batch's groups partition its records
    if ((rc = check_ragged(group_offsets, n_batch_groups, &longest)) != PG_OK) return rc;
    if (group_offsets[0] != 0 || group_offsets[n_batch_groups] != n_records) {
        set_error("group offsets run from %llu to %llu, not over the %llu records", (unsigned long long)group_offsets[0],
                  (unsigned long long)group_offsets[n_batch_groups], (unsigned long long)n_records);
        return PG_ERR_ARG;
    }
    if ((rc = check_ragged(offsets, n_records, &longest)) != PG_OK || (rc = use_device(sk->device)) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(sk->mu);
    HostCall c;
    const Ragged<uint8_t> r = c.ragged(bases, offsets, n_records);
    const uint64_t *d_goff = c.upload(group_offsets, n_batch_groups + 1);
    if ((rc = c.error())) return rc;
    PG_CUDA(cudaStreamWaitEvent(c.st, sk->read, 0));
    if ((rc = sketcher_add(sk->st, r.base, r.off, n_records, d_goff, first_group, n_batch_groups, c.st))) return rc;
    return c.finish();
}

int pg_mash_sketcher_add_dev(pg_mash_sketcher *sk, const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_records,
                             const uint64_t *d_group_offsets, uint64_t first_group, uint64_t n_batch_groups, void *stream) {
    bool work = false;
    int rc = sketcher_add_check(sk, d_bases, d_offsets, n_records, d_group_offsets, first_group, n_batch_groups, false, &work);
    if (rc != PG_OK || !work || (rc = use_device(sk->device)) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(sk->mu);
    PG_CUDA(cudaStreamWaitEvent((cudaStream_t)stream, sk->read, 0));
    return sketcher_add(sk->st, d_bases, d_offsets, n_records, d_group_offsets, first_group, n_batch_groups, (cudaStream_t)stream);
}

int pg_mash_sketcher_rows(const pg_mash_sketcher *sk, uint64_t first, uint64_t count, uint32_t *out, uint64_t row_stride, uint32_t *n_values,
                          uint8_t *complete, uint64_t *held) {
    int rc = sketcher_rows_check(sk, first, count, out, row_stride, n_values);
    if (rc != PG_OK || count == 0 || (rc = use_device(sk->device)) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(sk->mu);
    HostCall c;
    uint32_t *d_out = c.alloc<uint32_t>(count * row_stride), *d_n = c.alloc<uint32_t>(count);
    uint8_t *d_c = complete ? c.alloc<uint8_t>(count) : nullptr;
    uint64_t *d_h = held ? c.alloc<uint64_t>(count) : nullptr;
    if ((rc = c.error()) || (rc = sketcher_rows(sk->st, first, count, d_out, row_stride, d_n, d_c, d_h, c.st))) return rc;
    c.download(out, d_out, count * row_stride);
    c.download(n_values, d_n, count);
    c.download(complete, d_c, count);
    c.download(held, d_h, count);
    return c.finish();
}

int pg_mash_sketcher_rows_dev(const pg_mash_sketcher *sk, uint64_t first, uint64_t count, uint32_t *d_out, uint64_t row_stride, uint32_t *d_n_values,
                              uint8_t *d_complete, uint64_t *d_held, void *stream) {
    int rc = sketcher_rows_check(sk, first, count, d_out, row_stride, d_n_values);
    if (rc != PG_OK || count == 0 || (rc = use_device(sk->device)) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(sk->mu);
    if ((rc = sketcher_rows(sk->st, first, count, d_out, row_stride, d_n_values, d_complete, d_held, (cudaStream_t)stream)) != PG_OK) return rc;
    PG_CUDA(cudaEventRecord(sk->read, (cudaStream_t)stream));
    return PG_OK;
}

int pg_mash_sketcher_free(pg_mash_sketcher *sk) {
    if (!sk) return PG_OK;
    int rc = use_device(sk->device);
    if (rc != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    cudaStream_t st = cur_ctx()->slots[0].stream;
    cudaStreamWaitEvent(st, sk->read, 0);
    sketcher_free(sk->st, st);
    cudaEventDestroy(sk->read);
    delete sk;
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
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
int pg_mash_sketch_uniform_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k, int32_t s,
                                            uint32_t flags, uint32_t *out, uint64_t row_stride, int32_t *status,
                                            const int32_t *devices, int32_t n_devices) {
    return sketch_multi({bases, nullptr, read_len, n_reads, k, s, flags, out, row_stride, nullptr, status}, devices, n_devices);
}

int pg_mash_sketch_batch_multi(const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads, int32_t k, int32_t s,
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
int pg_mash_sketch_distance_multi(const uint8_t *bases, uint64_t n_reads, uint32_t read_len, int32_t k, int32_t s,
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
        auto fail = [&](int code) { my.rc = code; my.msg = pg_last_error(); failed.store(true); };
        auto step = [&](auto &&fn) { if (!failed.load()) { const int c = fn(); if (c != PG_OK) fail(c); } };
        bind_thread_device(dev[r]);
        pg_numa_bind_thread(dev[r], nullptr);
        const uint64_t lo = cut[r], hi = cut[r + 1], nl = hi - lo;
        uint8_t *d_reads = nullptr;
        uint32_t *d_full = nullptr;  // [n][s] full Go arrays (== gathered when cnt == s)
        cudaStream_t st = nullptr;
        step([&]() -> int {
            int c = ensure_device();
            if (c != PG_OK) return c;
            st = cur_ctx()->slots[0].stream;
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
                const int c = rows_to_host(d_full, n, s, lo, hi, same ? same + lo * n : nullptr, distance ? distance + lo * n : nullptr, st);
                if (c != PG_OK) return c;
            }
            PG_CUDA(cudaStreamSynchronize(st));
            return PG_OK;
        });
        meet.wait();  // nobody reads a peer buffer any more
        if (cur_ctx()) {
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
    if (rc != PG_OK || (rc = check_rows(n, row_begin, row_end)) != PG_OK) return rc;
    return launch_distance_block(d_sketches, n, s, row_begin, row_end, d_same, d_distance, (cudaStream_t)stream);
}

int pg_mash_distance_block(const uint32_t *sketches, uint64_t n, int32_t s, uint64_t row_begin,
                           uint64_t row_end, uint32_t *same, double *distance) {
    int rc = ensure_device();
    if (rc != PG_OK || (rc = check_rows(n, row_begin, row_end)) != PG_OK) return rc;
    if (row_end == row_begin || n == 0) return PG_OK;
    if (s <= 0) { set_error("distance over sketches of size %d: the reference panics", s); return PG_ERR_PANIC; }
    HostCall c;
    const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)s);
    if ((rc = c.error()) || (rc = rows_to_host(d_sk, n, s, row_begin, row_end, same, distance, c.st))) return rc;
    return c.finish();
}

int pg_mash_distance_sparse_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint64_t row_begin, uint64_t row_end, uint32_t flags,
                                uint32_t *d_pair_i, uint32_t *d_pair_j, uint32_t *d_pair_same, uint64_t pairs_cap, uint64_t *d_n_pairs,
                                void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK || (rc = check_rows(n, row_begin, row_end)) != PG_OK) return rc;
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
    if ((rc = check_rows(n, row_begin, row_end)) != PG_OK) return rc;
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
// Single-linkage groups of a sketch set
// ---------------------------------------------------------------------------------
int pg_mash_cluster_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t *d_label,
                        uint64_t *d_n_groups, uint64_t *d_n_links, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n && s > 0 && (!d_sketches || !d_label)) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_mash_cluster(d_sketches, n, s, min_same, d_label, (unsigned long long *)d_n_groups, (unsigned long long *)d_n_links,
                               (cudaStream_t)stream);
}

int pg_mash_cluster(const uint32_t *sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t *label, uint64_t *n_groups,
                    uint64_t *n_links) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_groups) *n_groups = 0;
    if (n_links) *n_links = 0;
    if ((rc = mash_cluster_check(n, s, min_same)) != PG_OK || n == 0) return rc;
    if (!sketches || !label) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)s);
    uint32_t *d_label = c.alloc<uint32_t>(n);
    unsigned long long *d_cnt = c.alloc<unsigned long long>(2);
    if ((rc = c.error()) || (rc = launch_mash_cluster(d_sk, n, s, min_same, d_label, d_cnt, d_cnt + 1, c.st))) return rc;
    c.download(label, d_label, n);
    c.download((unsigned long long *)n_groups, d_cnt, 1);
    c.download((unsigned long long *)n_links, d_cnt + 1, 1);
    return c.finish();
}

// ---------------------------------------------------------------------------------
// Greedy representatives of a sketch set
// ---------------------------------------------------------------------------------
int pg_mash_dereplicate_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t flags, uint32_t *d_rep,
                            uint64_t *d_n_reps, void *stream) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n && s > 0 && (!d_sketches || !d_rep)) { set_error("null buffer"); return PG_ERR_ARG; }
    return launch_mash_derep(d_sketches, n, s, min_same, flags, d_rep, (unsigned long long *)d_n_reps, (cudaStream_t)stream);
}

int pg_mash_dereplicate(const uint32_t *sketches, uint64_t n, int32_t s, uint32_t min_same, uint32_t flags, uint32_t *rep,
                        uint64_t *n_reps) {
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n_reps) *n_reps = 0;
    if ((rc = mash_derep_check(n, s, min_same, flags)) != PG_OK || n == 0) return rc;
    if (!sketches || !rep) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint32_t *d_sk = c.upload(sketches, n * (uint64_t)s);
    uint32_t *d_rep = c.alloc<uint32_t>(n);
    unsigned long long *d_cnt = c.alloc<unsigned long long>(1);
    if ((rc = c.error()) || (rc = launch_mash_derep(d_sk, n, s, min_same, flags, d_rep, d_cnt, c.st))) return rc;
    c.download(rep, d_rep, n);
    c.download((unsigned long long *)n_reps, d_cnt, 1);
    return c.finish();
}

// ---------------------------------------------------------------------------------
// Sketch index: top-k nearest references
// ---------------------------------------------------------------------------------
int pg_mash_index_create(const uint32_t *sketches, uint64_t n, int32_t s, pg_mash_index **out) {
    if (!out) { set_error("null index pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = ensure_device();
    if (rc != PG_OK) return rc;
    if (n && s > 0 && !sketches) { set_error("null buffer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    return index_create(sketches, false, n, s, cur_ctx()->slots[0].stream, out);
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
    std::shared_lock<std::shared_mutex> lk(ix->rw);
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
    std::shared_lock<std::shared_mutex> lk(ix->rw);
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

// ---------------------------------------------------------------------------------
// Sketch index: every reference within a matching-count cut
// ---------------------------------------------------------------------------------
int pg_mash_index_query_within_dev(const pg_mash_index *ix, const uint32_t *d_queries, uint64_t nq, int32_t sq, uint32_t min_same,
                                   uint64_t *d_hit_offsets, uint32_t *d_hit_ref, uint32_t *d_hit_same, double *d_hit_distance,
                                   uint64_t hits_cap, uint64_t *d_n_hits, void *stream) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    std::shared_lock<std::shared_mutex> lk(ix->rw);
    return launch_index_within(ix->plan, d_queries, nq, sq, min_same, d_hit_offsets, d_hit_ref, d_hit_same, d_hit_distance, hits_cap,
                               d_n_hits, (cudaStream_t)stream);
}

int pg_mash_index_query_within(const pg_mash_index *ix, const uint32_t *queries, uint64_t nq, int32_t sq, uint32_t min_same,
                               uint64_t *hit_offsets, uint32_t *hit_ref, uint32_t *hit_same, double *hit_distance, uint64_t hits_cap,
                               uint64_t *n_hits) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    if (n_hits) *n_hits = 0;
    std::shared_lock<std::shared_mutex> lk(ix->rw);
    if (min_same == 0) { set_error("min_same 0 would list all %llu x %llu pairs", (unsigned long long)nq, (unsigned long long)ix->plan.n); return PG_ERR_ARG; }
    if (nq == 0) {
        if (hit_offsets) hit_offsets[0] = 0;
        return PG_OK;
    }
    if (sq <= 0) { set_error("query sketches of size %d: the reference panics (Sketches[-1])", sq); return PG_ERR_PANIC; }
    if (!hit_offsets || !queries) { set_error("null buffer"); return PG_ERR_ARG; }
    HostCall c;
    const uint32_t *d_q = c.upload(queries, nq * (uint64_t)sq);
    uint64_t *d_off = c.alloc<uint64_t>(nq + 1);
    uint32_t *d_ref = hit_ref ? c.alloc<uint32_t>(hits_cap) : nullptr, *d_same = hit_same ? c.alloc<uint32_t>(hits_cap) : nullptr;
    double *d_dist = hit_distance ? c.alloc<double>(hits_cap) : nullptr;
    unsigned long long *d_n = c.alloc<unsigned long long>(1);
    if ((rc = c.error()) ||
        (rc = launch_index_within(ix->plan, d_q, nq, sq, min_same, d_off, d_ref, d_same, d_dist, hits_cap, (uint64_t *)d_n, c.st)))
        return rc;
    c.download(hit_offsets, d_off, nq + 1);
    uint64_t total = 0;
    const bool counting = !hit_ref && !hit_same && !hit_distance;  // no list to overflow
    return finish_capped(c, d_n, counting ? ~0ull : hits_cap, n_hits ? n_hits : &total,
                         {{hit_ref, d_ref, 4}, {hit_same, d_same, 4}, {hit_distance, d_dist, 8}}, "hits_cap", "hits");
}

// ---------------------------------------------------------------------------------
// Sketch index: growing it
// ---------------------------------------------------------------------------------
int pg_mash_index_add(pg_mash_index *ix, const uint32_t *sketches, uint64_t m, int32_t s) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    if (m == 0) return PG_OK;
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> lk(ix->rw);
    if ((rc = index_add_check(ix, sketches, m, s)) != PG_OK) return rc;
    HostCall c;
    const uint32_t *d_b = c.upload(sketches, m * (uint64_t)s);
    if ((rc = c.error()) || (rc = index_add(ix, d_b, true, m, s, c.st))) return rc;
    return c.finish();
}

int pg_mash_index_add_dev(pg_mash_index *ix, const uint32_t *d_sketches, uint64_t m, int32_t s, void *stream) {
    if (!ix) { set_error("null index"); return PG_ERR_ARG; }
    if (m == 0) return PG_OK;
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> lk(ix->rw);
    if ((rc = index_add_check(ix, d_sketches, m, s)) != PG_OK) return rc;
    return index_add(ix, d_sketches, true, m, s, (cudaStream_t)stream);
}

int pg_mash_index_free(pg_mash_index *ix) {
    if (!ix) return PG_OK;
    int rc = use_device(ix->device);
    if (rc != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    cudaStream_t st = cur_ctx()->slots[0].stream;
    distance_plan_destroy(ix->plan, st);
    if (ix->d_sk) cudaFreeAsync(ix->d_sk, st);
    delete ix;
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// ---------------------------------------------------------------------------------
// Growing a dereplication
// ---------------------------------------------------------------------------------
int pg_mash_dereplicator_create(int32_t s, uint32_t min_same, uint32_t flags, pg_mash_dereplicator **out) {
    if (!out) { set_error("null dereplicator pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = mash_derep_check(1, s, min_same, flags);  // the rules dereplicate applies to a non-empty set
    if (rc != PG_OK || (rc = ensure_device()) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    pg_mash_index *ix = nullptr;
    if ((rc = index_create(nullptr, false, 0, s, cur_ctx()->slots[0].stream, &ix)) != PG_OK) return rc;
    *out = new pg_mash_dereplicator{ix->device, s, min_same, flags, ix, nullptr, 0};
    return PG_OK;
}

int pg_mash_dereplicator_add(pg_mash_dereplicator *d, const uint32_t *sketches, uint64_t m, int32_t s, uint32_t *rep, uint64_t *first,
                             uint64_t *n_new_reps) {
    if (!d) { set_error("null dereplicator"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(d->mu);
    if (first) *first = d->n;
    if (n_new_reps) *n_new_reps = 0;
    if (m == 0) return PG_OK;
    int rc = derep_add_check(d, sketches, m, s, rep);
    if (rc != PG_OK || (rc = use_device(d->device)) != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> wl(d->ix->rw);  // before the device lock, as the index's own add takes them
    HostCall c;
    const uint32_t *d_b = c.upload(sketches, m * (uint64_t)s);
    uint32_t *d_rep = c.alloc<uint32_t>(m);
    uint64_t n_new = 0;
    if ((rc = c.error()) || (rc = derep_add(d, d_b, m, d_rep, rep, &n_new, c.st)) || (rc = c.finish())) return rc;
    if (n_new_reps) *n_new_reps = n_new;
    return PG_OK;
}

int pg_mash_dereplicator_add_dev(pg_mash_dereplicator *d, const uint32_t *d_sketches, uint64_t m, int32_t s, uint32_t *d_rep,
                                 uint64_t *first, uint64_t *n_new_reps, void *stream) {
    if (!d) { set_error("null dereplicator"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(d->mu);
    if (first) *first = d->n;
    if (n_new_reps) *n_new_reps = 0;
    if (m == 0) return PG_OK;
    int rc = derep_add_check(d, d_sketches, m, s, d_rep);
    if (rc != PG_OK || (rc = use_device(d->device)) != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> wl(d->ix->rw);
    uint64_t n_new = 0;
    if ((rc = derep_add(d, d_sketches, m, d_rep, nullptr, &n_new, (cudaStream_t)stream)) != PG_OK) return rc;
    if (n_new_reps) *n_new_reps = n_new;
    return PG_OK;
}

int pg_mash_dereplicator_reps(const pg_mash_dereplicator *d, uint32_t *ids, uint64_t cap, uint64_t *n_reps) {
    if (!d) { set_error("null dereplicator"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(d->mu);
    const uint64_t R = d->ix->plan.n;
    if (n_reps) *n_reps = R;
    if (cap && !ids) { set_error("null buffer"); return PG_ERR_ARG; }
    if (const uint64_t k = std::min(cap, R)) {
        int rc = use_device(d->device);
        if (rc != PG_OK) return rc;
        HostCall c;
        c.download(ids, d->d_ids, k);
        if ((rc = c.finish()) != PG_OK) return rc;
    }
    if (R > cap) { set_error("%llu representatives exceed cap %llu", (unsigned long long)R, (unsigned long long)cap); return PG_ERR_ARG; }
    return PG_OK;
}

const pg_mash_index *pg_mash_dereplicator_index(const pg_mash_dereplicator *d) { return d ? d->ix : nullptr; }

int pg_mash_dereplicator_free(pg_mash_dereplicator *d) {
    if (!d) return PG_OK;
    int rc = use_device(d->device);
    if (rc != PG_OK) return rc;
    if (d->d_ids) {
        std::lock_guard<std::mutex> lk(cur_ctx()->mu);
        cudaStream_t st = cur_ctx()->slots[0].stream;
        cudaFreeAsync(d->d_ids, st);
        cudaStreamSynchronize(st);
    }
    rc = pg_mash_index_free(d->ix);
    delete d;
    return rc;
}

// ---------------------------------------------------------------------------------
// Growing a clustering
// ---------------------------------------------------------------------------------
int pg_mash_clusterer_create(int32_t s, uint32_t min_same, pg_mash_clusterer **out) {
    if (!out) { set_error("null clusterer pointer"); return PG_ERR_ARG; }
    *out = nullptr;
    int rc = mash_cluster_check(1, s, min_same);  // the rules cluster applies to a non-empty set
    if (rc != PG_OK || (rc = ensure_device()) != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    pg_mash_index *ix = nullptr;
    if ((rc = index_create(nullptr, false, 0, s, cur_ctx()->slots[0].stream, &ix)) != PG_OK) return rc;
    *out = new pg_mash_clusterer{ix->device, s, min_same, ix, nullptr, 0, 0};
    return PG_OK;
}

// The per-add outputs before any work: what an empty batch or an error reports
static void cluster_add_outputs(const pg_mash_clusterer *c, uint64_t *first, uint64_t *n_groups, uint64_t *n_links, uint64_t *n_merged) {
    if (first) *first = c->n;
    if (n_groups) *n_groups = c->n_groups;
    if (n_links) *n_links = 0;
    if (n_merged) *n_merged = 0;
}

int pg_mash_clusterer_add(pg_mash_clusterer *c, const uint32_t *sketches, uint64_t m, int32_t s, uint32_t *label, uint64_t *first,
                          uint64_t *n_groups, uint64_t *n_links, uint64_t *n_merged) {
    if (!c) { set_error("null clusterer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(c->mu);
    cluster_add_outputs(c, first, n_groups, n_links, n_merged);
    if (m == 0) return PG_OK;
    int rc = cluster_add_check(c, sketches, m, s);
    if (rc != PG_OK || (rc = use_device(c->device)) != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> wl(c->ix->rw);  // before the device lock, as the index's own add takes them
    HostCall hc;
    const uint32_t *d_b = hc.upload(sketches, m * (uint64_t)s);
    unsigned long long cnt[3] = {};
    if ((rc = hc.error()) || (rc = cluster_add(c, d_b, m, nullptr, label, cnt, hc.st)) || (rc = hc.finish())) return rc;
    if (n_links) *n_links = cnt[0];
    if (n_groups) *n_groups = cnt[1];
    if (n_merged) *n_merged = cnt[2];
    return PG_OK;
}

int pg_mash_clusterer_add_dev(pg_mash_clusterer *c, const uint32_t *d_sketches, uint64_t m, int32_t s, uint32_t *d_label, uint64_t *first,
                              uint64_t *n_groups, uint64_t *n_links, uint64_t *n_merged, void *stream) {
    if (!c) { set_error("null clusterer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(c->mu);
    cluster_add_outputs(c, first, n_groups, n_links, n_merged);
    if (m == 0) return PG_OK;
    int rc = cluster_add_check(c, d_sketches, m, s);
    if (rc != PG_OK || (rc = use_device(c->device)) != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> wl(c->ix->rw);
    unsigned long long cnt[3] = {};
    if ((rc = cluster_add(c, d_sketches, m, d_label, nullptr, cnt, (cudaStream_t)stream)) != PG_OK) return rc;
    if (n_links) *n_links = cnt[0];
    if (n_groups) *n_groups = cnt[1];
    if (n_merged) *n_merged = cnt[2];
    return PG_OK;
}

static int cluster_labels_check(const pg_mash_clusterer *c, uint64_t begin, uint64_t end, const void *label) {
    if (begin > end || end > c->n) {
        set_error("labels [%llu, %llu) outside the %llu sketches added", (unsigned long long)begin, (unsigned long long)end, (unsigned long long)c->n);
        return PG_ERR_ARG;
    }
    if (end > begin && !label) { set_error("null buffer"); return PG_ERR_ARG; }
    return PG_OK;
}

int pg_mash_clusterer_labels(const pg_mash_clusterer *c, uint64_t begin, uint64_t end, uint32_t *label) {
    if (!c) { set_error("null clusterer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(c->mu);
    int rc = cluster_labels_check(c, begin, end, label);
    if (rc != PG_OK || end == begin || (rc = use_device(c->device)) != PG_OK) return rc;
    HostCall hc;
    hc.download(label, c->d_label + begin, end - begin);
    return hc.finish();
}

int pg_mash_clusterer_labels_dev(const pg_mash_clusterer *c, uint64_t begin, uint64_t end, uint32_t *d_label, void *stream) {
    if (!c) { set_error("null clusterer"); return PG_ERR_ARG; }
    std::lock_guard<std::mutex> lk(c->mu);
    int rc = cluster_labels_check(c, begin, end, d_label);
    if (rc != PG_OK || end == begin || (rc = use_device(c->device)) != PG_OK) return rc;
    PG_CUDA(cudaMemcpyAsync(d_label, c->d_label + begin, (end - begin) * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return PG_OK;
}

const pg_mash_index *pg_mash_clusterer_index(const pg_mash_clusterer *c) { return c ? c->ix : nullptr; }

int pg_mash_clusterer_free(pg_mash_clusterer *c) {
    if (!c) return PG_OK;
    int rc = use_device(c->device);
    if (rc != PG_OK) return rc;
    if (c->d_label) {
        std::lock_guard<std::mutex> lk(cur_ctx()->mu);
        cudaStream_t st = cur_ctx()->slots[0].stream;
        cudaFreeAsync(c->d_label, st);
        cudaStreamSynchronize(st);
    }
    rc = pg_mash_index_free(c->ix);
    delete c;
    return rc;
}

// ---------------------------------------------------------------------------------
// Screen: which references a pool of reads contains
// ---------------------------------------------------------------------------------
int pg_mash_screen_create(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, pg_mash_screen **out) {
    return screen_create_host(sketches, n, s, k, 1, 0, out);
}

int pg_mash_screen_create_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, void *stream, pg_mash_screen **out) {
    return screen_create_dev(d_sketches, n, s, k, 1, 0, stream, out);
}

int pg_mash_screen_create_samples(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, pg_mash_screen **out) {
    return screen_create_host(sketches, n, s, k, n_samples, 0, out);
}

int pg_mash_screen_create_flags(const uint32_t *sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags, pg_mash_screen **out) {
    return screen_create_host(sketches, n, s, k, n_samples, flags, out);
}

int pg_mash_screen_create_flags_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, uint32_t flags, void *stream,
                                    pg_mash_screen **out) {
    return screen_create_dev(d_sketches, n, s, k, n_samples, flags, stream, out);
}

int pg_mash_screen_create_samples_dev(const uint32_t *d_sketches, uint64_t n, int32_t s, int32_t k, uint32_t n_samples, void *stream,
                                      pg_mash_screen **out) {
    return screen_create_dev(d_sketches, n, s, k, n_samples, 0, stream, out);
}

int pg_mash_screen_add(pg_mash_screen *sc, const uint8_t *bases, const uint64_t *offsets, uint64_t n_reads) {
    return screen_add_host(sc, bases, offsets, nullptr, n_reads);
}

int pg_mash_screen_add_dev(pg_mash_screen *sc, const uint8_t *d_bases, const uint64_t *d_offsets, uint64_t n_reads, void *stream) {
    return screen_add_dev(sc, d_bases, d_offsets, nullptr, n_reads, stream);
}

int pg_mash_screen_add_samples(pg_mash_screen *sc, const uint8_t *bases, const uint64_t *offsets, const uint32_t *sample_ids, uint64_t n_reads) {
    if (sc && n_reads && !sample_ids) { set_error("null sample ids"); return PG_ERR_ARG; }
    return screen_add_host(sc, bases, offsets, sample_ids, n_reads);
}

int pg_mash_screen_add_samples_dev(pg_mash_screen *sc, const uint8_t *d_bases, const uint64_t *d_offsets, const uint32_t *d_sample_ids,
                                   uint64_t n_reads, void *stream) {
    if (sc && n_reads && !d_sample_ids) { set_error("null sample ids"); return PG_ERR_ARG; }
    return screen_add_dev(sc, d_bases, d_offsets, d_sample_ids, n_reads, stream);
}

int pg_mash_screen_reset(pg_mash_screen *sc) {
    if (!sc) { set_error("null screen"); return PG_ERR_ARG; }
    int rc = use_device(sc->device);
    if (rc != PG_OK) return rc;
    std::unique_lock<std::shared_mutex> lk(sc->rw);
    HostCall c;
    if ((rc = screen_reset(sc->ix, c.st)) != PG_OK) return rc;
    return c.finish();
}

int pg_mash_screen_results(const pg_mash_screen *sc, uint32_t *shared, double *containment, uint64_t *multiplicity) {
    return screen_tally_host(sc, screen_results, 0, 1, shared, containment, multiplicity);
}

int pg_mash_screen_results_dev(const pg_mash_screen *sc, uint32_t *d_shared, double *d_containment, uint64_t *d_multiplicity, void *stream) {
    return screen_tally_dev(sc, screen_results, 0, 1, d_shared, d_containment, d_multiplicity, stream);
}

int pg_mash_screen_winners(const pg_mash_screen *sc, uint32_t *shared, double *containment, uint64_t *multiplicity) {
    return screen_tally_host(sc, screen_winners, 0, 1, shared, containment, multiplicity);
}

int pg_mash_screen_winners_dev(const pg_mash_screen *sc, uint32_t *d_shared, double *d_containment, uint64_t *d_multiplicity, void *stream) {
    return screen_tally_dev(sc, screen_winners, 0, 1, d_shared, d_containment, d_multiplicity, stream);
}

int pg_mash_screen_results_samples(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *shared, double *containment,
                                   uint64_t *multiplicity) {
    return screen_tally_host(sc, screen_results, first, count, shared, containment, multiplicity);
}

int pg_mash_screen_results_samples_dev(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_containment,
                                       uint64_t *d_multiplicity, void *stream) {
    return screen_tally_dev(sc, screen_results, first, count, d_shared, d_containment, d_multiplicity, stream);
}

int pg_mash_screen_winners_samples(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *shared, double *containment,
                                   uint64_t *multiplicity) {
    return screen_tally_host(sc, screen_winners, first, count, shared, containment, multiplicity);
}

int pg_mash_screen_winners_samples_dev(const pg_mash_screen *sc, uint32_t first, uint32_t count, uint32_t *d_shared, double *d_containment,
                                       uint64_t *d_multiplicity, void *stream) {
    return screen_tally_dev(sc, screen_winners, first, count, d_shared, d_containment, d_multiplicity, stream);
}

int pg_mash_screen_free(pg_mash_screen *sc) {
    if (!sc) return PG_OK;
    int rc = use_device(sc->device);
    if (rc != PG_OK) return rc;
    std::lock_guard<std::mutex> lk(cur_ctx()->mu);
    cudaStream_t st = cur_ctx()->slots[0].stream;
    screen_free(sc->ix, st);
    delete sc;
    PG_CUDA(cudaStreamSynchronize(st));
    return PG_OK;
}

// ---------------------------------------------------------------------------------
// Mash distance between grouped sketches
// ---------------------------------------------------------------------------------
int pg_mash_dist_dev(const uint32_t *d_q_rows, const uint32_t *d_q_count, uint64_t nq, const uint32_t *d_r_rows, const uint32_t *d_r_count, uint64_t nr,
                     uint64_t row_stride, int32_t s, int32_t k, const uint64_t *d_q_length, const uint64_t *d_r_length, uint32_t *d_common,
                     uint32_t *d_denom, double *d_distance, double *d_p_value, void *stream) {
    int rc = dist_check(nq, nr, s, k, row_stride, d_q_rows, d_q_count, d_r_rows, d_r_count, d_p_value != nullptr, d_q_length, d_r_length);
    if (rc != PG_OK || nq == 0 || nr == 0 || !(d_common || d_denom || d_distance || d_p_value)) return rc;
    if ((rc = ensure_device()) != PG_OK) return rc;
    DistArgs g = dist_args(d_q_rows, d_q_count, nq, d_r_rows, d_r_count, nr, row_stride, s, k, d_q_length, d_r_length);
    g.common = d_common; g.denom = d_denom; g.distance = d_distance; g.p_value = d_p_value;
    return launch_mash_dist(g, false, (cudaStream_t)stream);
}

int pg_mash_dist(const uint32_t *q_rows, const uint32_t *q_count, uint64_t nq, const uint32_t *r_rows, const uint32_t *r_count, uint64_t nr,
                 uint64_t row_stride, int32_t s, int32_t k, const uint64_t *q_length, const uint64_t *r_length, uint32_t *common, uint32_t *denom,
                 double *distance, double *p_value) {
    const bool need_len = p_value != nullptr;
    int rc = dist_check(nq, nr, s, k, row_stride, q_rows, q_count, r_rows, r_count, need_len, q_length, r_length);
    if (rc != PG_OK || (rc = dist_rows_check(q_rows, q_count, nq, s, row_stride, need_len ? q_length : nullptr, "query")) != PG_OK ||
        (rc = dist_rows_check(r_rows, r_count, nr, s, row_stride, need_len ? r_length : nullptr, "reference")) != PG_OK)
        return rc;
    const uint64_t per_pair = (common ? 4 : 0) + (denom ? 4 : 0) + (distance ? 8 : 0) + (p_value ? 8 : 0);
    if (nq == 0 || nr == 0 || per_pair == 0) return PG_OK;
    if ((rc = ensure_device()) != PG_OK) return rc;
    const uint64_t rows_per = std::max<uint64_t>(1, std::min<uint64_t>(nq, DIST_BLOCK_BYTES / (nr * per_pair)));
    HostCall c;
    const uint32_t *d_r = c.upload(r_rows, nr * row_stride), *d_rc = c.upload(r_count, nr);
    const uint64_t *d_rl = need_len ? c.upload(r_length, nr) : nullptr;
    uint32_t *d_q = c.alloc<uint32_t>(rows_per * row_stride), *d_qc = c.alloc<uint32_t>(rows_per);
    uint64_t *d_ql = need_len ? c.alloc<uint64_t>(rows_per) : nullptr;
    uint32_t *d_common = common ? c.alloc<uint32_t>(rows_per * nr) : nullptr, *d_denom = denom ? c.alloc<uint32_t>(rows_per * nr) : nullptr;
    double *d_dist = distance ? c.alloc<double>(rows_per * nr) : nullptr, *d_p = p_value ? c.alloc<double>(rows_per * nr) : nullptr;
    if ((rc = c.error()) != PG_OK) return rc;
    for (uint64_t b = 0; b < nq; b += rows_per) {
        const uint64_t m = std::min(rows_per, nq - b);
        c.put(d_q, q_rows + b * row_stride, m * row_stride);
        c.put(d_qc, q_count + b, m);
        if (need_len) c.put(d_ql, q_length + b, m);
        DistArgs g = dist_args(d_q, d_qc, m, d_r, d_rc, nr, row_stride, s, k, d_ql, d_rl);
        g.q0 = b; g.common = d_common; g.denom = d_denom; g.distance = d_dist; g.p_value = d_p;
        if ((rc = c.error()) != PG_OK || (rc = launch_mash_dist(g, false, c.st)) != PG_OK) return rc;
        if (common) c.download(common + b * nr, d_common, m * nr);
        if (denom) c.download(denom + b * nr, d_denom, m * nr);
        if (distance) c.download(distance + b * nr, d_dist, m * nr);
        if (p_value) c.download(p_value + b * nr, d_p, m * nr);
    }
    return c.finish();
}

int pg_mash_dist_within_dev(const uint32_t *d_q_rows, const uint32_t *d_q_count, uint64_t nq, const uint32_t *d_r_rows, const uint32_t *d_r_count,
                            uint64_t nr, uint64_t row_stride, int32_t s, int32_t k, const uint64_t *d_q_length, const uint64_t *d_r_length,
                            double max_distance, double max_p_value, uint32_t flags, uint32_t *d_pair_q, uint32_t *d_pair_r, uint32_t *d_common,
                            uint32_t *d_denom, double *d_distance, double *d_p_value, uint64_t pairs_cap, uint64_t *d_n_pairs, void *stream) {
    const bool need_len = d_p_value != nullptr || max_p_value < 1.0;
    int rc = dist_check(nq, nr, s, k, row_stride, d_q_rows, d_q_count, d_r_rows, d_r_count, need_len, d_q_length, d_r_length);
    if (rc != PG_OK || (rc = dist_within_check(nq, nr, max_distance, max_p_value, flags, d_pair_q, d_pair_r, d_n_pairs)) != PG_OK ||
        (rc = ensure_device()) != PG_OK)
        return rc;
    PG_CUDA(cudaMemsetAsync(d_n_pairs, 0, sizeof(uint64_t), (cudaStream_t)stream));
    DistArgs g = dist_args(d_q_rows, d_q_count, nq, d_r_rows, d_r_count, nr, row_stride, s, k, d_q_length, d_r_length);
    g.max_distance = max_distance; g.max_p_value = max_p_value; g.upper = (flags & PG_PAIRS_UPPER) != 0;
    g.pair_q = d_pair_q; g.pair_r = d_pair_r; g.common = d_common; g.denom = d_denom; g.distance = d_distance; g.p_value = d_p_value;
    g.cap = pairs_cap; g.n_pairs = (unsigned long long *)d_n_pairs;
    return launch_mash_dist(g, true, (cudaStream_t)stream);
}

int pg_mash_dist_within(const uint32_t *q_rows, const uint32_t *q_count, uint64_t nq, const uint32_t *r_rows, const uint32_t *r_count, uint64_t nr,
                        uint64_t row_stride, int32_t s, int32_t k, const uint64_t *q_length, const uint64_t *r_length, double max_distance,
                        double max_p_value, uint32_t flags, uint32_t *pair_q, uint32_t *pair_r, uint32_t *common, uint32_t *denom, double *distance,
                        double *p_value, uint64_t pairs_cap, uint64_t *n_pairs) {
    const bool need_len = p_value != nullptr || max_p_value < 1.0;
    int rc = dist_check(nq, nr, s, k, row_stride, q_rows, q_count, r_rows, r_count, need_len, q_length, r_length);
    if (rc != PG_OK || (rc = dist_within_check(nq, nr, max_distance, max_p_value, flags, pair_q, pair_r, n_pairs)) != PG_OK ||
        (rc = dist_rows_check(q_rows, q_count, nq, s, row_stride, need_len ? q_length : nullptr, "query")) != PG_OK ||
        (rc = dist_rows_check(r_rows, r_count, nr, s, row_stride, need_len ? r_length : nullptr, "reference")) != PG_OK)
        return rc;
    *n_pairs = 0;
    if (nq == 0 || nr == 0) return PG_OK;
    if ((rc = ensure_device()) != PG_OK) return rc;
    HostCall c;
    const uint32_t *d_q = c.upload(q_rows, nq * row_stride), *d_qc = c.upload(q_count, nq);
    const uint32_t *d_r = c.upload(r_rows, nr * row_stride), *d_rc = c.upload(r_count, nr);
    const uint64_t *d_ql = need_len ? c.upload(q_length, nq) : nullptr, *d_rl = need_len ? c.upload(r_length, nr) : nullptr;
    uint32_t *d_pq = c.alloc<uint32_t>(pairs_cap), *d_pr = c.alloc<uint32_t>(pairs_cap);
    uint32_t *d_c = common ? c.alloc<uint32_t>(pairs_cap) : nullptr, *d_d = denom ? c.alloc<uint32_t>(pairs_cap) : nullptr;
    double *d_dist = distance ? c.alloc<double>(pairs_cap) : nullptr, *d_p = p_value ? c.alloc<double>(pairs_cap) : nullptr;
    unsigned long long *d_n = c.alloc<unsigned long long>(1, true);
    if ((rc = c.error()) != PG_OK) return rc;
    DistArgs g = dist_args(d_q, d_qc, nq, d_r, d_rc, nr, row_stride, s, k, d_ql, d_rl);
    g.max_distance = max_distance; g.max_p_value = max_p_value; g.upper = (flags & PG_PAIRS_UPPER) != 0;
    g.pair_q = d_pq; g.pair_r = d_pr; g.common = d_c; g.denom = d_d; g.distance = d_dist; g.p_value = d_p;
    g.cap = pairs_cap; g.n_pairs = d_n;
    if ((rc = launch_mash_dist(g, true, c.st)) != PG_OK) return rc;
    return finish_capped(c, d_n, pairs_cap, n_pairs,
                         {{pair_q, d_pq, 4}, {pair_r, d_pr, 4}, {common, d_c, 4}, {denom, d_d, 4}, {distance, d_dist, 8}, {p_value, d_p, 8}},
                         "pairs_cap", "pairs");
}

}  // extern "C"
