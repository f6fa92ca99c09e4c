"""GPU tier: the pipelined host sketch path (pg_mash_sketch_uniform / pg_mash_sketch_batch and their
_multi forms).

Every combination of batch layout, pinned or pageable input and output, flags and row stride must give
the rows, counts and statuses the device-pointer entry point gives on the same reads, and a sample of rows
is checked against the oracle.  A chunk holds 32 MiB of input when either side is staged through pinned
buffers and 192 MiB when both caller buffers are pinned, so the 256 MiB batches here run 8 chunks and
2 chunks: every mode cycles through the three stream slots, and the staged modes reuse each of them.  The
ragged batch holds 96 MiB of equal-length reads, so whole 32 MiB chunks of it take the uniform kernel.

A host sketch call rejected for its arguments writes nothing: a decreasing offset, or a read too long for
row_stride, in the second chunk of a batch fails before the first chunk is launched."""
import numpy as np
import pytest
import torch

from poly_b200 import _lib, mash

pytestmark = pytest.mark.gpu

K, S = 21, 24  # reads of >= K + S bases take the select regime (bottom-S of their k-mers)
MiB = 1 << 20
SENTINEL = 0xDEADBEEF
READ_LEN = 1000


def _acgt(rng, n):
    return np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, n, dtype=np.uint8)]


def _offsets(lens):
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    return off


class Batch:
    def __init__(self, bases, offsets):
        self.offsets = offsets  # None: fixed-length reads of READ_LEN bases
        self.n = len(offsets) - 1 if offsets is not None else len(bases) // READ_LEN
        self.pageable = bases
        self.pinned = torch.empty(len(bases), dtype=torch.uint8, pin_memory=True).numpy()
        self.pinned[:] = bases
        self.dev = torch.from_numpy(bases).cuda()
        self.dev_off = torch.from_numpy(offsets.view(np.int64)).cuda() if offsets is not None else None
        self.max_len = int(np.diff(offsets).max()) if offsets is not None else READ_LEN
        self.out_pinned = torch.empty(self.n * (S + 3), dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
        self.refs = {}

    def read(self, i):
        if self.offsets is None:
            return self.pageable[i * READ_LEN:(i + 1) * READ_LEN]
        return self.pageable[int(self.offsets[i]):int(self.offsets[i + 1])]

    def reference(self, flags, stride):
        """rows, counts and statuses of the device-pointer entry point, which stages nothing"""
        key = (flags, stride)
        if key not in self.refs:
            L = _lib.lib()
            out = torch.full((self.n * stride,), -1, dtype=torch.int32, device="cuda")  # dirty rows
            count = torch.zeros(self.n, dtype=torch.int32, device="cuda")
            status = torch.zeros(self.n, dtype=torch.int32, device="cuda")
            if self.offsets is None:
                rc = L.pg_mash_sketch_uniform_dev(self.dev.data_ptr(), self.n, READ_LEN, K, S, flags, out.data_ptr(), stride,
                                                  status.data_ptr(), None)
                count.fill_(min(READ_LEN - K, S))
            else:
                rc = L.pg_mash_sketch_batch_dev(self.dev.data_ptr(), self.dev_off.data_ptr(), self.n, self.max_len, K, S, flags,
                                                out.data_ptr(), stride, count.data_ptr(), status.data_ptr(), None)
            assert rc == 0, _lib.last_error()
            torch.cuda.synchronize()
            self.refs[key] = (out.cpu().numpy().view(np.uint32).reshape(self.n, stride), count.cpu().numpy().view(np.uint32),
                              status.cpu().numpy())
        return self.refs[key]

    def host(self, pinned_in, pinned_out, flags, stride):
        src = self.pinned if pinned_in else self.pageable
        out = self.out_pinned[: self.n * stride].reshape(self.n, stride) if pinned_out else np.empty((self.n, stride), np.uint32)
        out[:] = SENTINEL
        count = np.full(self.n, SENTINEL, np.uint32)
        status = np.full(self.n, -1, np.int32)
        L = _lib.lib()
        if self.offsets is None:
            rc = L.pg_mash_sketch_uniform(src.ctypes.data, self.n, READ_LEN, K, S, flags, out.ctypes.data, stride, status.ctypes.data)
            count[:] = min(READ_LEN - K, S)
        else:
            rc = L.pg_mash_sketch_batch(src.ctypes.data, self.offsets.ctypes.data, self.n, K, S, flags, out.ctypes.data, stride,
                                        count.ctypes.data, status.ctypes.data)
        assert rc == 0, _lib.last_error()
        return out, count, status


@pytest.fixture(scope="module")
def batches(gpu):
    rng = np.random.default_rng(11)

    def mixed(nbytes):  # 200-1600 bases, every 7th read shorter than K + S (a sketch of fewer than S words)
        lens = rng.integers(200, 1600, nbytes // 700)
        lens[::7] = rng.integers(0, K + S, len(lens[::7]))
        return lens[np.cumsum(lens) <= nbytes]

    lens = np.concatenate([mixed(96 * MiB), np.full(96 * MiB // READ_LEN, READ_LEN), mixed(64 * MiB)])
    off = _offsets(lens)
    assert 192 * MiB < off[-1] <= 256 * MiB
    return {"uniform": Batch(_acgt(rng, 256 * MiB), None), "ragged": Batch(_acgt(rng, int(off[-1])), off)}


FLAGS = {"none": 0, "pad_zero": _lib.PG_SKETCH_PAD_ZERO, "tail_keep": _lib.PG_SKETCH_TAIL_KEEP}


@pytest.mark.parametrize("extra", [0, 3])
@pytest.mark.parametrize("flags", sorted(FLAGS))
@pytest.mark.parametrize("pinned_out", [False, True])
@pytest.mark.parametrize("pinned_in", [False, True])
@pytest.mark.parametrize("layout", ["uniform", "ragged"])
def test_host_rows_equal_device_rows(batches, layout, pinned_in, pinned_out, flags, extra):
    b = batches[layout]
    stride = S + extra  # the batch's need: its longest reads have S words
    keep = flags == "tail_keep"
    want, want_count, want_status = b.reference(0 if keep else FLAGS[flags], stride)
    out, count, status = b.host(pinned_in, pinned_out, FLAGS[flags], stride)
    assert np.array_equal(count, want_count)
    assert np.array_equal(status, want_status) and not status.any()
    tail = np.arange(stride)[None, :] >= count[:, None]
    if keep:  # nothing beyond a row's count words is written
        want = np.where(tail, np.uint32(SENTINEL), want)
    else:
        assert not out[tail].any()
    assert np.array_equal(out, want)


@pytest.mark.parametrize("layout", ["uniform", "ragged"])
def test_sample_rows_match_oracle(batches, oracle, layout):
    b = batches[layout]
    rng = np.random.default_rng(4)
    idx = np.unique(np.concatenate([[0, b.n - 1], rng.choice(b.n, 96, replace=False)]))
    out, count, _ = b.host(False, False, _lib.PG_SKETCH_PAD_ZERO, S)
    bases, offsets = mash.flatten([b.read(i) for i in idx])
    rc, want = oracle.sketch_batch(bases, offsets, K, S, variant=1)
    assert rc == 0
    assert np.array_equal(out[idx], want)
    assert np.array_equal(count[idx], [min(max(len(b.read(i)) - K, 0), S) for i in idx])


@pytest.mark.parametrize("multi", [False, True])
@pytest.mark.parametrize("fault", ["offsets", "row_stride"])
def test_bad_batch_fails_before_the_first_chunk(gpu, fault, multi):
    """A pageable ragged batch of 80 MiB runs in 32 MiB chunks; the fault sits 40 MiB in."""
    rng = np.random.default_rng(3)
    read_len = 30  # K + 9 bases: sketches of 9 words
    n = 80 * MiB // read_len
    j = n // 2
    lens = np.full(n, read_len)
    if fault == "row_stride":
        lens[j] = 100  # the batch's only sketch of S words
    off = _offsets(lens)
    bases = _acgt(rng, int(off[-1]))
    if fault == "offsets":
        off[j + 1] = off[j] - 1
    stride = read_len - K
    out = np.full((n, stride), SENTINEL, np.uint32)
    count = np.full(n, SENTINEL, np.uint32)
    status = np.full(n, -1, np.int32)
    L = gpu.lib()
    before = L.pg_launch_count()
    args = (bases.ctypes.data, off.ctypes.data, n, K, S, 0, out.ctypes.data, stride, count.ctypes.data, status.ctypes.data)
    rc = L.pg_mash_sketch_batch_multi(*args, None, 0) if multi else L.pg_mash_sketch_batch(*args)
    assert rc == _lib.PG_ERR_ARG
    assert L.pg_launch_count() == before
    assert (out == SENTINEL).all() and (count == SENTINEL).all() and (status == -1).all()
    assert (f"offsets decrease at {j}" if fault == "offsets" else f"row_stride {stride} < {S}") in _lib.last_error()
