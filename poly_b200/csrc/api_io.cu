// api_io.cu -- the C ABI of poly's io: FASTQ and FASTA parsing.
#include "runtime.cuh"

namespace pg {
namespace {

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

}  // namespace
}  // namespace pg

using namespace pg;

extern "C" {

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

}  // extern "C"
