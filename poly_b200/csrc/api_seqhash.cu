// api_seqhash.cu -- the C ABI of poly's seqhash: Seqhash v1 digests and the least rotation.
#include "runtime.cuh"

namespace pg {
namespace {

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

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

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
    // A sequence's device memory: input and canonical copy, one 32-byte chaining value per KiB and per
    // sequence, offsets, orientation, error and digest words.  Over a group this bound is never below the
    // group's 2 B + 64 + 32 (B / 1024 + cnt) + 101 cnt bytes.
    const uint64_t budget = group_budget(2ull << 30);
    auto cost = [&](uint64_t i) {
        const uint64_t len = offsets[i + 1] - offsets[i];
        return 2 * len + 32 * (len / 1024 + 2) + 165;
    };
    for (uint64_t g = 0; g < n;) {
        const uint64_t e = group_end(g, n, budget, cost), cnt = e - g;
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

}  // extern "C"
