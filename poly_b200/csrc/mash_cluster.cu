// mash_cluster.cu -- single-linkage groups of a sketch set at a matching-count threshold.
//
// Sketches i < j are linked iff same(i, j) >= min_same, same(i, j) being what
// sketches[i].Similarity(sketches[j]) counts with the LOWER index as the receiver (the entry the dense
// pass of distance.cu writes at row i, column j).  Groups are the connected components of that graph and
// label[i] is the smallest index of i's group.
//
// The dense row-block tiles of distance.cu are scanned on the device as they are produced and every
// qualifying entry is merged into a union-find forest over parent[n]; no pair list exists anywhere.
//
// cluster_link_kernel<Upper> : qualifying entries of one tile of counts -> lock-free unions + the link count.  Tile
//                              row t is sketch row0 + t and column j is sketch col0 + j; Upper keeps only the
//                              entries whose column sketch is above the row sketch.
// cluster_flatten_kernel     : label[i] = root(i) and the number of roots, after the last tile (a growing clustering
//                              also counts the earlier roots that stopped being roots)
//
// A growing clustering (launch_mash_cluster_add) runs the same kernels over a forest of n + m sketches that starts
// as the n earlier labels followed by the batch's own ids: the batch's links to the earlier sketches come from a
// query of the index over them (launch_index_cluster, Upper off: every entry of the batch row's counts is one
// cross pair), the links inside the batch from the dense pass over the batch alone (Upper on, ids offset by n).
// The earlier labels are a flattened forest (every label is a root no larger than its sketch), so the union rule
// below applies unchanged.
//
// The union rule: a root is only ever re-parented, by atomicCAS, to a SMALLER root.  parent[x] <= x then holds
// for every x at every moment, so the root of a finished component is its smallest member whatever order the
// atomics landed in: the labels are a function of the input alone (not of tile size, grid or timing).
#include <algorithm>

#include "common.cuh"

namespace pg {

namespace {

// Loads of parent[] while other CTAs are linking go to L2 (volatile): a root seen through a stale L1 line
// would fail its CAS, be read as a root again and never make progress.
__device__ __forceinline__ uint32_t parent_of(const uint32_t *parent, uint32_t x) {
    return *reinterpret_cast<const volatile uint32_t *>(parent + x);
}

// Root of x with path halving.  x's new parent is one of its ancestors, and ancestors stay ancestors (links
// only re-parent roots), so the plain store races only with stores of other valid ancestors.  A node that is
// already a child of its root is not written, so a settled forest is found read-only.
__device__ __forceinline__ uint32_t find_root(uint32_t *parent, uint32_t x) {
    for (;;) {
        const uint32_t p = parent_of(parent, x);
        if (p == x) return x;
        const uint32_t g = parent_of(parent, p);
        if (g == p) return p;
        parent[x] = g;
        x = g;
    }
}

__device__ __forceinline__ void unite(uint32_t *parent, uint32_t a, uint32_t b) {
    for (;;) {
        a = find_root(parent, a);
        b = find_root(parent, b);
        if (a == b) return;  // members of one family meet here: ~R^2 links, ~R CAS
        const uint32_t lo = min(a, b), hi = max(a, b);
        const uint32_t seen = atomicCAS(parent + hi, hi, lo);
        if (seen == hi) return;
        a = seen;  // hi was linked elsewhere meanwhile: go on from its new parent
        b = lo;
    }
}

// One warp covers 128 consecutive words of the (rows x n) tile per step, as compact_pairs_kernel does.
template <bool Upper>
__global__ void __launch_bounds__(256)
cluster_link_kernel(const uint32_t *__restrict__ tile, uint64_t rows, uint64_t n, uint64_t row0, uint64_t col0, uint32_t min_same,
                    uint32_t *parent, unsigned long long *__restrict__ n_links) {
    const uint64_t total = rows * n;
    const uint32_t lane = threadIdx.x & 31u;
    const bool vec = (n & 3) == 0;  // rows are 16-byte aligned
    uint32_t links = 0;
    // the loop bound is warp-uniform: the warp reduction behind the loop needs every lane
    for (uint64_t w0 = ((uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u)) * 4; w0 < total; w0 += (uint64_t)gridDim.x * blockDim.x * 4) {
        const uint64_t e0 = w0 + lane * 4;
        uint32_t v[4];
        load_count_quad(tile, e0, total, vec, v);
        // most of a tile is zeros: nothing below this line runs for them (min_same >= 1)
        if (max(max(v[0], v[1]), max(v[2], v[3])) < min_same) continue;
        uint64_t i = row0 + e0 / n, j = e0 % n;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            if (v[t] >= min_same && (!Upper || col0 + j > i)) {
                ++links;
                unite(parent, (uint32_t)i, (uint32_t)(col0 + j));
            }
            if (++j == n) { j = 0; ++i; }
        }
    }
    links = __reduce_add_sync(0xffffffffu, links);
    if (lane == 0 && links) atomicAdd(n_links, (unsigned long long)links);
}

__global__ void __launch_bounds__(256)
cluster_init_kernel(uint32_t *__restrict__ parent, uint64_t n) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) parent[i] = (uint32_t)i;
}

// label[i] = root(i) for the n entries and the number of roots into *n_groups; with n_merged, also the number of
// the first n_old sketches that were roots of `old` (old[i] == i) and are no longer roots
__global__ void __launch_bounds__(256)
cluster_flatten_kernel(const uint32_t *__restrict__ parent, uint64_t n, uint32_t *__restrict__ label,
                       unsigned long long *__restrict__ n_groups, const uint32_t *__restrict__ old, uint64_t n_old,
                       unsigned long long *__restrict__ n_merged) {
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t roots = 0, merged = 0;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + (threadIdx.x & ~31u); i0 < n; i0 += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = i0 + lane;
        if (i >= n) continue;
        uint32_t r = (uint32_t)i;
        for (uint32_t p = parent[r]; p != r; p = parent[r]) r = p;
        label[i] = r;
        roots += r == (uint32_t)i;
        merged += i < n_old && r != (uint32_t)i && old[i] == (uint32_t)i;
    }
    roots = __reduce_add_sync(0xffffffffu, roots);
    if (lane == 0 && roots) atomicAdd(n_groups, (unsigned long long)roots);
    if (n_merged) {  // uniform over the grid
        merged = __reduce_add_sync(0xffffffffu, merged);
        if (lane == 0 && merged) atomicAdd(n_merged, (unsigned long long)merged);
    }
}

// The links inside one set of n sketches whose rows are sketches base .. base + n - 1: its dense tiles, upper
// triangle, united into parent
int cluster_tiles(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t base, uint32_t *d_parent,
                  unsigned long long *d_n_links, cudaStream_t st) {
    return distance_plan_tiles(d_sk, n, s, 0, n, distance_tile_rows(n, n), true, false, st,
                               [&](const uint32_t *tile, const double *, uint64_t rb, uint64_t re) {
        return launch_cluster_link(tile, re - rb, n, base + rb, base, true, min_same, d_parent, d_n_links, st);
    });
}

}  // namespace

int launch_cluster_link(const uint32_t *d_counts, uint64_t rows, uint64_t n, uint64_t row0, uint64_t col0, bool upper, uint32_t min_same,
                        uint32_t *d_parent, unsigned long long *d_n_links, cudaStream_t st) {
    const uint64_t quads = (rows * n + 3) / 4;
    const unsigned grid = (unsigned)std::min<uint64_t>((quads + 255) / 256, (uint64_t)sm_count() * 16);
    if (upper) {
        cluster_link_kernel<true><<<grid, 256, 0, st>>>(d_counts, rows, n, row0, col0, min_same, d_parent, d_n_links);
        PG_LAUNCH_CHECK("cluster_link_kernel");
    } else {
        cluster_link_kernel<false><<<grid, 256, 0, st>>>(d_counts, rows, n, row0, col0, min_same, d_parent, d_n_links);
        PG_LAUNCH_CHECK("cluster_link_kernel<false>");
    }
    return PG_OK;
}

int mash_cluster_check(uint64_t n, int s, uint32_t min_same) {
    if (n > 0xffffffffull) { set_error("too many sketches for 32-bit labels"); return PG_ERR_ARG; }
    if (n == 0) return PG_OK;
    if (s <= 0) { set_error("cluster over sketches of size %d: the reference panics (Sketches[-1])", s); return PG_ERR_PANIC; }
    if (min_same == 0 || min_same > (uint32_t)s) {
        set_error("min_same %u outside [1, %d]: 0 links every pair, more than the sketch size links none", min_same, s);
        return PG_ERR_ARG;
    }
    return PG_OK;
}

int launch_mash_cluster(const uint32_t *d_sk, uint64_t n, int s, uint32_t min_same, uint32_t *d_label,
                        unsigned long long *d_n_groups, unsigned long long *d_n_links, cudaStream_t st) {
    if (d_n_groups) PG_CUDA(cudaMemsetAsync(d_n_groups, 0, 8, st));
    if (d_n_links) PG_CUDA(cudaMemsetAsync(d_n_links, 0, 8, st));
    int rc = mash_cluster_check(n, s, min_same);
    if (rc != PG_OK || n == 0) return rc;
    StreamScratch tmp(st);  // parent[n], then the two counters: freed on every way out
    uint32_t *d_parent = nullptr;
    const uint64_t parent_words = (n + 1) & ~1ull;
    cudaError_t e = tmp.alloc(&d_parent, parent_words + 4);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("cudaMallocAsync(%llu) for the cluster forest failed", (unsigned long long)((parent_words + 4) * 4)); return PG_ERR_NOMEM; }
    unsigned long long *d_cnt = reinterpret_cast<unsigned long long *>(d_parent + parent_words);  // [0] links, [1] groups
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, 16, st));
    const unsigned row_blocks = (unsigned)std::min<uint64_t>((n + 255) / 256, (uint64_t)sm_count() * 16);
    cluster_init_kernel<<<row_blocks, 256, 0, st>>>(d_parent, n);
    PG_LAUNCH_CHECK("cluster_init_kernel");

    rc = cluster_tiles(d_sk, n, s, min_same, 0, d_parent, d_cnt, st);
    if (rc != PG_OK) return rc;
    cluster_flatten_kernel<<<row_blocks, 256, 0, st>>>(d_parent, n, d_label, d_cnt + 1, nullptr, 0, nullptr);
    PG_LAUNCH_CHECK("cluster_flatten_kernel");
    if (d_n_links) PG_CUDA(cudaMemcpyAsync(d_n_links, d_cnt, 8, cudaMemcpyDeviceToDevice, st));
    if (d_n_groups) PG_CUDA(cudaMemcpyAsync(d_n_groups, d_cnt + 1, 8, cudaMemcpyDeviceToDevice, st));
    return PG_OK;
}

int launch_mash_cluster_add(const DistancePlan &plan, const uint32_t *d_old, const uint32_t *d_b, uint64_t m, int s, uint32_t min_same,
                            uint32_t *d_label, unsigned long long *d_cnt, cudaStream_t st) {
    const uint64_t n = plan.n, total = n + m;
    PG_CUDA(cudaMemsetAsync(d_cnt, 0, 24, st));
    StreamScratch tmp(st);
    uint32_t *d_parent = nullptr;
    if (tmp.alloc(&d_parent, total) != cudaSuccess) {
        cudaGetLastError();
        set_error("cudaMallocAsync(%llu) for the cluster forest failed", (unsigned long long)(total * 4));
        return PG_ERR_NOMEM;
    }
    // the forest: every sketch its own root, then the earlier labels over the first n (each a root <= its sketch)
    const unsigned row_blocks = (unsigned)std::min<uint64_t>((total + 255) / 256, (uint64_t)sm_count() * 16);
    cluster_init_kernel<<<row_blocks, 256, 0, st>>>(d_parent, total);
    PG_LAUNCH_CHECK("cluster_init_kernel");
    if (n) PG_CUDA(cudaMemcpyAsync(d_parent, d_old, n * 4, cudaMemcpyDeviceToDevice, st));
    int rc = launch_index_cluster(plan, d_b, m, s, min_same, n, d_parent, d_cnt, st);
    if (rc == PG_OK) rc = cluster_tiles(d_b, m, s, min_same, (uint32_t)n, d_parent, d_cnt, st);
    if (rc != PG_OK) return rc;
    cluster_flatten_kernel<<<row_blocks, 256, 0, st>>>(d_parent, total, d_label, d_cnt + 1, d_old, n, d_cnt + 2);
    PG_LAUNCH_CHECK("cluster_flatten_kernel");
    return PG_OK;
}

}  // namespace pg
