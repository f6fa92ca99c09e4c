// Package polyb200 is the cgo binding of libpolyb200.so (include/poly_b200.h): the thin
// shim the mash / align / primers drop-in packages call.  NOT COMPILED IN THIS REPOSITORY'S
// CI: the build image has no Go toolchain (DESIGN.md); the same C ABI is exercised by the
// C++ and Python host mirrors.  Build with:
//
//	CGO_CFLAGS="-I${POLYB200}/include" CGO_LDFLAGS="-L${POLYB200}/poly_b200/lib -lpolyb200" go build ./...
package polyb200

/*
#include <stdlib.h>
#include "poly_b200.h"
*/
import "C"

import (
	"errors"
	"fmt"
	"runtime"
	"unsafe"
)

// ErrPanic is returned where the pure-Go reference would panic (index out of range).
var ErrPanic = errors.New("poly: reference panics on this input (index out of range)")

// ErrCloneUnsupported is returned by the clone wrappers for PG_ERR_UNSUPPORTED: a part or fragment with a
// byte >= 0x80 (strings.ToUpper would re-encode it), or an enzyme site that is not a plain literal.
var ErrCloneUnsupported = errors.New("clone: unsupported input (non-literal enzyme site or non-ASCII byte)")

// cloneCheck is check with PG_ERR_UNSUPPORTED mapped to ErrCloneUnsupported.
func cloneCheck(rc C.int) error {
	if rc == C.PG_ERR_UNSUPPORTED {
		return ErrCloneUnsupported
	}
	return check(rc)
}

// locked runs one C ABI call with the goroutine pinned to its OS thread, so that pg_last_error()
// (a thread-local string) is read on the thread that produced it.
func locked(call func() C.int) error {
	runtime.LockOSThread()
	defer runtime.UnlockOSThread()
	return check(call())
}

func check(rc C.int) error {
	switch rc {
	case C.PG_OK:
		return nil
	case C.PG_ERR_PANIC:
		return ErrPanic
	default:
		return fmt.Errorf("libpolyb200 error %d: %s", int(rc), C.GoString(C.pg_last_error()))
	}
}

// Flatten copies []string into the bytes+offsets layout of the C ABI.  The copy is what
// makes the call legal under the cgo pointer rules (no Go pointer to Go pointers crosses;
// nothing is retained by C after return).
func Flatten(seqs []string) ([]byte, []uint64) {
	total := 0
	for _, s := range seqs {
		total += len(s)
	}
	bases := make([]byte, 0, total+1)
	offsets := make([]uint64, len(seqs)+1)
	for i, s := range seqs {
		bases = append(bases, s...)
		offsets[i+1] = uint64(len(bases))
	}
	if len(bases) == 0 {
		bases = bases[:1] // keep &bases[0] valid
	}
	return bases, offsets
}

// SketchBatch wraps pg_mash_sketch_batch: compact rows of rowStride words, count[i] informative words.
func SketchBatch(bases []byte, offsets []uint64, k, s int, rowStride int) (out []uint32, count []uint32, status []int32, err error) {
	n := len(offsets) - 1
	out = make([]uint32, n*rowStride+1)
	count = make([]uint32, n+1)
	status = make([]int32, n+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_mash_sketch_batch((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
		C.int32_t(k), C.int32_t(s), 0, (*C.uint32_t)(unsafe.Pointer(&out[0])), C.uint64_t(rowStride),
		(*C.uint32_t)(unsafe.Pointer(&count[0])), (*C.int32_t)(unsafe.Pointer(&status[0])))
	return out, count, status, check(rc)
}

// SketchGroups wraps pg_mash_sketch_groups: group g is records [groupOffsets[g], groupOffsets[g+1]) of the ragged
// batch (bases, offsets); row g of out (s words) holds the smallest count[g] distinct window hashes of the group seen at
// least minCopies times, ascending, then zeros.
func SketchGroups(bases []byte, offsets []uint64, groupOffsets []uint64, k, s int, minCopies uint32) (out []uint32, count []uint32, err error) {
	return SketchGroupsFlags(bases, offsets, groupOffsets, k, s, minCopies, 0)
}

// KmerCanonical is PG_KMER_CANONICAL: windows 0 .. L-k of each record, each hashing the smaller of itself and its
// reverse complement.
const KmerCanonical = uint32(C.PG_KMER_CANONICAL)

// SketchGroupsFlags wraps pg_mash_sketch_groups_flags: SketchGroups with flags (0 or KmerCanonical).
func SketchGroupsFlags(bases []byte, offsets []uint64, groupOffsets []uint64, k, s int, minCopies, flags uint32) (out []uint32, count []uint32, err error) {
	n, g := len(offsets)-1, len(groupOffsets)-1
	out = make([]uint32, g*s+1)
	count = make([]uint32, g+1)
	err = locked(func() C.int {
		return C.pg_mash_sketch_groups_flags((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
			(*C.uint64_t)(unsafe.Pointer(&groupOffsets[0])), C.uint64_t(g), C.int32_t(k), C.int32_t(s), C.uint32_t(minCopies), C.uint32_t(flags),
			(*C.uint32_t)(unsafe.Pointer(&out[0])), C.uint64_t(s), (*C.uint32_t)(unsafe.Pointer(&count[0])))
	})
	return out[:g*s], count[:g], err
}

// Sketcher wraps a pg_mash_sketcher: nGroups grouped sketches grown in place, batch by batch, on the device of the
// calling thread.  Close must not run while another call on it is in flight.
type Sketcher struct {
	h    *C.pg_mash_sketcher
	n, s int
}

// NewSketcher wraps pg_mash_sketcher_create (maxValues: the most distinct values a group keeps between adds).
func NewSketcher(nGroups uint64, k, s int, minCopies uint32, maxValues uint64) (*Sketcher, error) {
	return NewSketcherFlags(nGroups, k, s, minCopies, maxValues, 0)
}

// NewSketcherFlags wraps pg_mash_sketcher_create_flags: NewSketcher with flags (0 or KmerCanonical).
func NewSketcherFlags(nGroups uint64, k, s int, minCopies uint32, maxValues uint64, flags uint32) (*Sketcher, error) {
	var h *C.pg_mash_sketcher
	if err := locked(func() C.int {
		return C.pg_mash_sketcher_create_flags(C.uint64_t(nGroups), C.int32_t(k), C.int32_t(s), C.uint32_t(minCopies), C.uint64_t(maxValues),
			C.uint32_t(flags), &h)
	}); err != nil {
		return nil, err
	}
	return &Sketcher{h: h, n: int(nGroups), s: s}, nil
}

// Add wraps pg_mash_sketcher_add: records [groupOffsets[i], groupOffsets[i+1]) of the ragged batch (bases, offsets) go
// to group firstGroup + i.
func (sk *Sketcher) Add(bases []byte, offsets []uint64, groupOffsets []uint64, firstGroup uint64) error {
	n, g := len(offsets)-1, len(groupOffsets)-1
	if n <= 0 {
		return nil
	}
	var b *C.uint8_t
	if len(bases) > 0 {
		b = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	return locked(func() C.int {
		return C.pg_mash_sketcher_add(sk.h, b, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
			(*C.uint64_t)(unsafe.Pointer(&groupOffsets[0])), C.uint64_t(firstGroup), C.uint64_t(g))
	})
}

// Rows wraps pg_mash_sketcher_rows over every group: s words per group, the values each row holds, whether it is
// complete, and the values each group keeps.
func (sk *Sketcher) Rows() (out []uint32, count []uint32, complete []bool, held []uint64, err error) {
	out, count, c, held := make([]uint32, sk.n*sk.s+1), make([]uint32, sk.n+1), make([]uint8, sk.n+1), make([]uint64, sk.n+1)
	err = locked(func() C.int {
		return C.pg_mash_sketcher_rows(sk.h, 0, C.uint64_t(sk.n), (*C.uint32_t)(unsafe.Pointer(&out[0])), C.uint64_t(sk.s),
			(*C.uint32_t)(unsafe.Pointer(&count[0])), (*C.uint8_t)(unsafe.Pointer(&c[0])), (*C.uint64_t)(unsafe.Pointer(&held[0])))
	})
	complete = make([]bool, sk.n)
	for i := range complete {
		complete[i] = c[i] != 0
	}
	return out[:sk.n*sk.s], count[:sk.n], complete, held[:sk.n], err
}

// Close wraps pg_mash_sketcher_free.
func (sk *Sketcher) Close() error {
	if sk.h == nil {
		return nil
	}
	h := sk.h
	sk.h = nil
	return locked(func() C.int { return C.pg_mash_sketcher_free(h) })
}

func devicePtr(devices []int32) (*C.int32_t, C.int32_t) {
	if len(devices) == 0 {
		return nil, 0 // all visible GPUs
	}
	return (*C.int32_t)(unsafe.Pointer(&devices[0])), C.int32_t(len(devices))
}

// SketchBatchMulti wraps pg_mash_sketch_batch_multi: the batch is cut into contiguous shards, one per
// GPU of this process (devices == nil: every visible GPU), each driven by its own host thread inside the
// library.  Same results as SketchBatch.
func SketchBatchMulti(bases []byte, offsets []uint64, k, s int, rowStride int, devices []int32) (out []uint32, count []uint32, status []int32, err error) {
	n := len(offsets) - 1
	out = make([]uint32, n*rowStride+1)
	count = make([]uint32, n+1)
	status = make([]int32, n+1)
	dp, dn := devicePtr(devices)
	err = locked(func() C.int {
		return C.pg_mash_sketch_batch_multi((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
			C.int32_t(k), C.int32_t(s), 0, (*C.uint32_t)(unsafe.Pointer(&out[0])), C.uint64_t(rowStride),
			(*C.uint32_t)(unsafe.Pointer(&count[0])), (*C.int32_t)(unsafe.Pointer(&status[0])), dp, dn)
	})
	return out, count, status, err
}

// SketchInto wraps pg_mash_sketch_batch_multi with PG_SKETCH_TAIL_KEEP: sketches is the caller's n x s slab (the
// Sketches arrays of n Mash values back to back); row i receives its min(len_i-k, s) words and nothing else is
// written -- a fresh make([]uint32, n*s) therefore ends up as n full, zero-tailed Sketches arrays without a
// per-read allocation or copy on the Go side, and a reused slab keeps its tails as (*Mash).Sketch does.
func SketchInto(bases []byte, offsets []uint64, k, s int, sketches []uint32, devices []int32) (count []uint32, status []int32, err error) {
	n := len(offsets) - 1
	if len(sketches) < n*s {
		return nil, nil, fmt.Errorf("polyb200: sketches holds %d words, need %d", len(sketches), n*s)
	}
	count = make([]uint32, n+1)
	status = make([]int32, n+1)
	if n == 0 {
		return count[:n], status[:n], nil
	}
	if len(bases) == 0 {
		bases = make([]byte, 1)
	}
	if len(sketches) == 0 { // s == 0: the call still reports the reads on which the reference panics
		sketches = make([]uint32, 1)
	}
	dp, dn := devicePtr(devices)
	err = locked(func() C.int {
		return C.pg_mash_sketch_batch_multi((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
			C.int32_t(k), C.int32_t(s), C.PG_SKETCH_TAIL_KEEP, (*C.uint32_t)(unsafe.Pointer(&sketches[0])), C.uint64_t(s),
			(*C.uint32_t)(unsafe.Pointer(&count[0])), (*C.int32_t)(unsafe.Pointer(&status[0])), dp, dn)
	})
	return count[:n], status[:n], err
}

// SketchDistanceMulti wraps pg_mash_sketch_distance_multi for fixed-length reads stored back to back:
// sketches (n x s full arrays), matching counts and distances (n x n), computed on all listed GPUs with
// the all-gather of the sketches fused into the sketch kernels.
func SketchDistanceMulti(bases []byte, n, readLen, k, s int, devices []int32) (sketches []uint32, same []uint32, dist []float64, err error) {
	sketches = make([]uint32, n*s+1)
	same = make([]uint32, n*n+1)
	dist = make([]float64, n*n+1)
	dp, dn := devicePtr(devices)
	err = locked(func() C.int {
		return C.pg_mash_sketch_distance_multi((*C.uint8_t)(unsafe.Pointer(&bases[0])), C.uint64_t(n), C.uint32_t(readLen), C.int32_t(k), C.int32_t(s),
			dp, dn, (*C.uint32_t)(unsafe.Pointer(&sketches[0])), (*C.uint32_t)(unsafe.Pointer(&same[0])), (*C.double)(unsafe.Pointer(&dist[0])))
	})
	return sketches[:n*s], same[:n*n], dist[:n*n], err
}

// SimilarityPairs wraps pg_mash_similarity_pairs.
func SimilarityPairs(sketches []uint32, skOffsets []uint64, pairA, pairB []uint32) (same []int64, sim, dist []float64, err error) {
	np := len(pairA)
	same, sim, dist = make([]int64, np+1), make([]float64, np+1), make([]float64, np+1)
	status := make([]int32, np+1)
	if len(sketches) == 0 {
		sketches = make([]uint32, 1)
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_mash_similarity_pairs((*C.uint32_t)(unsafe.Pointer(&sketches[0])), (*C.uint64_t)(unsafe.Pointer(&skOffsets[0])),
		C.uint64_t(len(skOffsets)-1), (*C.uint32_t)(unsafe.Pointer(&pairA[0])), (*C.uint32_t)(unsafe.Pointer(&pairB[0])), C.uint64_t(np),
		(*C.int64_t)(unsafe.Pointer(&same[0])), (*C.double)(unsafe.Pointer(&sim[0])), (*C.double)(unsafe.Pointer(&dist[0])),
		(*C.int32_t)(unsafe.Pointer(&status[0])))
	return same[:np], sim[:np], dist[:np], check(rc)
}

// DistanceBlock wraps pg_mash_distance_block (rows [rowBegin,rowEnd) x all n columns).
func DistanceBlock(sketches []uint32, n, s int, rowBegin, rowEnd int) (same []uint32, dist []float64, err error) {
	rows := rowEnd - rowBegin
	same, dist = make([]uint32, rows*n+1), make([]float64, rows*n+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_mash_distance_block((*C.uint32_t)(unsafe.Pointer(&sketches[0])), C.uint64_t(n), C.int32_t(s), C.uint64_t(rowBegin),
		C.uint64_t(rowEnd), (*C.uint32_t)(unsafe.Pointer(&same[0])), (*C.double)(unsafe.Pointer(&dist[0])))
	return same[:rows*n], dist[:rows*n], check(rc)
}

// DistanceSparse wraps pg_mash_distance_sparse: the pairs (i, j) of rows [rowBegin,rowEnd) x all n columns that share
// at least one hash, with their matching counts; every pair not listed has Similarity 0 / Distance 1
// (mash.go:134,139).  upper: only j > i.  The order of the triples is unspecified.
func DistanceSparse(sketches []uint32, n, s int, rowBegin, rowEnd int, upper bool) (pi, pj, same []uint32, err error) {
	capPairs := 4*(rowEnd-rowBegin) + 1024
	flags := C.uint32_t(0)
	if upper {
		flags = C.PG_PAIRS_UPPER
	}
	for {
		pi, pj, same = make([]uint32, capPairs), make([]uint32, capPairs), make([]uint32, capPairs)
		var cnt C.uint64_t
		var rc C.int
		err = locked(func() C.int {
			rc = C.pg_mash_distance_sparse((*C.uint32_t)(unsafe.Pointer(&sketches[0])), C.uint64_t(n), C.int32_t(s), C.uint64_t(rowBegin),
				C.uint64_t(rowEnd), flags, (*C.uint32_t)(unsafe.Pointer(&pi[0])), (*C.uint32_t)(unsafe.Pointer(&pj[0])),
				(*C.uint32_t)(unsafe.Pointer(&same[0])), C.uint64_t(capPairs), &cnt)
			return rc
		})
		if rc == C.PG_ERR_ARG && int(cnt) > capPairs { // the buffers were too small: the call reports the size it needs
			capPairs = int(cnt)
			continue
		}
		if err != nil {
			return nil, nil, nil, err
		}
		k := int(cnt)
		return pi[:k], pj[:k], same[:k], nil
	}
}

// DistResult holds pg_mash_dist's nq x nr outputs, row-major with the query as the row.
type DistResult struct {
	Common, Denom    []uint32
	Distance, PValue []float64
}

func u32p(a []uint32) *C.uint32_t {
	if len(a) == 0 {
		return nil
	}
	return (*C.uint32_t)(unsafe.Pointer(&a[0]))
}

func u64p(a []uint64) *C.uint64_t {
	if len(a) == 0 {
		return nil
	}
	return (*C.uint64_t)(unsafe.Pointer(&a[0]))
}

func f64p(a []float64) *C.double {
	if len(a) == 0 {
		return nil
	}
	return (*C.double)(unsafe.Pointer(&a[0]))
}

// Dist wraps pg_mash_dist: nq query rows against nr reference rows, each row s words (row stride s) holding count[i]
// ascending values.  qLen and rLen (nil: no p-value) are the bases behind each sketch.
func Dist(q, qCount []uint32, r, rCount []uint32, s, k int, qLen, rLen []uint64) (res DistResult, err error) {
	nq, nr := len(qCount), len(rCount)
	res = DistResult{make([]uint32, nq*nr), make([]uint32, nq*nr), make([]float64, nq*nr), nil}
	if qLen != nil {
		res.PValue = make([]float64, nq*nr)
	}
	err = locked(func() C.int {
		return C.pg_mash_dist(u32p(q), u32p(qCount), C.uint64_t(nq), u32p(r), u32p(rCount), C.uint64_t(nr), C.uint64_t(s), C.int32_t(s), C.int32_t(k),
			u64p(qLen), u64p(rLen), u32p(res.Common), u32p(res.Denom), f64p(res.Distance), f64p(res.PValue))
	})
	return res, err
}

// DistPairs holds pg_mash_dist_within's list, in the call's (unspecified) order.
type DistPairs struct {
	Q, R, Common, Denom []uint32
	Distance, PValue    []float64
}

// DistWithin wraps pg_mash_dist_within: the pairs of Dist with distance <= maxDistance and p-value <= maxPValue;
// upper keeps r > q only (nq == nr).  qLen and rLen may be nil when maxPValue >= 1 (no p-value then).
func DistWithin(q, qCount []uint32, r, rCount []uint32, s, k int, qLen, rLen []uint64, maxDistance, maxPValue float64, upper bool) (DistPairs, error) {
	nq, nr := len(qCount), len(rCount)
	flags := C.uint32_t(0)
	if upper {
		flags = C.PG_PAIRS_UPPER
	}
	capPairs := 4*nq + 1024
	for {
		p := DistPairs{make([]uint32, capPairs), make([]uint32, capPairs), make([]uint32, capPairs), make([]uint32, capPairs),
			make([]float64, capPairs), nil}
		if qLen != nil {
			p.PValue = make([]float64, capPairs)
		}
		var cnt C.uint64_t
		var rc C.int
		err := locked(func() C.int {
			rc = C.pg_mash_dist_within(u32p(q), u32p(qCount), C.uint64_t(nq), u32p(r), u32p(rCount), C.uint64_t(nr), C.uint64_t(s), C.int32_t(s),
				C.int32_t(k), u64p(qLen), u64p(rLen), C.double(maxDistance), C.double(maxPValue), flags, u32p(p.Q), u32p(p.R), u32p(p.Common),
				u32p(p.Denom), f64p(p.Distance), f64p(p.PValue), C.uint64_t(capPairs), &cnt)
			return rc
		})
		if rc == C.PG_ERR_ARG && int(cnt) > capPairs { // the buffers were too small: the call reports the size it needs
			capPairs = int(cnt)
			continue
		}
		if err != nil {
			return DistPairs{}, err
		}
		n := int(cnt)
		p.Q, p.R, p.Common, p.Denom, p.Distance = p.Q[:n], p.R[:n], p.Common[:n], p.Denom[:n], p.Distance[:n]
		if p.PValue != nil {
			p.PValue = p.PValue[:n]
		}
		return p, nil
	}
}

// Cluster wraps pg_mash_cluster: single-linkage groups of n sketches of size s, sketches i < j being linked when
// sketches[i].Similarity(sketches[j]) counts at least minSame matching hashes (the lower index is the receiver).
// label[i] is the smallest index of i's group; nGroups counts the groups and nLinks the linked pairs.
func Cluster(sketches []uint32, n, s, minSame int) (label []uint32, nGroups, nLinks uint64, err error) {
	label = make([]uint32, n+1)
	var sk *C.uint32_t
	if len(sketches) > 0 {
		sk = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	var groups, links C.uint64_t
	err = locked(func() C.int {
		return C.pg_mash_cluster(sk, C.uint64_t(n), C.int32_t(s), C.uint32_t(minSame), (*C.uint32_t)(unsafe.Pointer(&label[0])), &groups, &links)
	})
	if err != nil {
		return nil, 0, 0, err
	}
	return label[:n], uint64(groups), uint64(links), nil
}

// Dereplicate wraps pg_mash_dereplicate: greedy representatives of n sketches of size s, linked as in Cluster.
// In index order, i is a representative iff no representative r < i is linked to i; rep[i] = i for one, else the
// smallest linked representative, or with nearest the one with the largest count (ties to the smaller index).
func Dereplicate(sketches []uint32, n, s, minSame int, nearest bool) (rep []uint32, nReps uint64, err error) {
	rep = make([]uint32, n+1)
	var sk *C.uint32_t
	if len(sketches) > 0 {
		sk = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	flags := C.uint32_t(0)
	if nearest {
		flags = C.PG_DEREP_NEAREST
	}
	var reps C.uint64_t
	err = locked(func() C.int {
		return C.pg_mash_dereplicate(sk, C.uint64_t(n), C.int32_t(s), C.uint32_t(minSame), flags, (*C.uint32_t)(unsafe.Pointer(&rep[0])), &reps)
	})
	if err != nil {
		return nil, 0, err
	}
	return rep[:n], uint64(reps), nil
}

// SWScoreBatch wraps pg_sw_score_batch.
func SWScoreBatch(queries []byte, qOffsets []uint64, template string, queryIsA bool, lutA, lutB *[256]int16, table []int64,
	nA, nB int, gap int64) (score []int64, errCode []int32, errPos []int64, err error) {
	n := len(qOffsets) - 1
	score, errCode, errPos = make([]int64, n+1), make([]int32, n+1), make([]int64, n+1)
	t := []byte(template)
	if len(t) == 0 {
		t = make([]byte, 1)
	}
	qa := C.int32_t(0)
	if queryIsA {
		qa = 1
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_sw_score_batch((*C.uint8_t)(unsafe.Pointer(&queries[0])), (*C.uint64_t)(unsafe.Pointer(&qOffsets[0])), C.uint64_t(n),
		(*C.uint8_t)(unsafe.Pointer(&t[0])), C.uint64_t(len(template)), qa, (*C.int16_t)(unsafe.Pointer(&lutA[0])),
		(*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])), C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
		(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])))
	return score[:n], errCode[:n], errPos[:n], check(rc)
}

// NWScoreBatch wraps pg_nw_score_batch (same arguments as SWScoreBatch).
func NWScoreBatch(queries []byte, qOffsets []uint64, template string, queryIsA bool, lutA, lutB *[256]int16, table []int64,
	nA, nB int, gap int64) (score []int64, errCode []int32, errPos []int64, err error) {
	n := len(qOffsets) - 1
	score, errCode, errPos = make([]int64, n+1), make([]int32, n+1), make([]int64, n+1)
	t := []byte(template)
	if len(t) == 0 {
		t = make([]byte, 1)
	}
	qa := C.int32_t(0)
	if queryIsA {
		qa = 1
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_nw_score_batch((*C.uint8_t)(unsafe.Pointer(&queries[0])), (*C.uint64_t)(unsafe.Pointer(&qOffsets[0])), C.uint64_t(n),
		(*C.uint8_t)(unsafe.Pointer(&t[0])), C.uint64_t(len(template)), qa, (*C.int16_t)(unsafe.Pointer(&lutA[0])),
		(*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])), C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
		(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])))
	return score[:n], errCode[:n], errPos[:n], check(rc)
}

// NWAlignBatch wraps pg_nw_align_batch (same contract as SWAlignBatch).
func NWAlignBatch(queries []byte, qOffsets []uint64, template string, queryIsA bool, lutA, lutB *[256]int16, table []int64,
	nA, nB int, gap int64, stride int) ([]int64, []int32, []int64, []string, []string, error) {
	return alignBatch(true, queries, qOffsets, template, queryIsA, lutA, lutB, table, nA, nB, gap, stride)
}

// SWAlignBatch wraps pg_sw_align_batch: scores plus the two aligned strings per query.  Rows that
// do not fit `stride` bytes are retried with the reported length.
func SWAlignBatch(queries []byte, qOffsets []uint64, template string, queryIsA bool, lutA, lutB *[256]int16, table []int64,
	nA, nB int, gap int64, stride int) ([]int64, []int32, []int64, []string, []string, error) {
	return alignBatch(false, queries, qOffsets, template, queryIsA, lutA, lutB, table, nA, nB, gap, stride)
}

func alignBatch(global bool, queries []byte, qOffsets []uint64, template string, queryIsA bool, lutA, lutB *[256]int16, table []int64,
	nA, nB int, gap int64, stride int) (score []int64, errCode []int32, errPos []int64, alignA, alignB []string, err error) {
	n := len(qOffsets) - 1
	t := []byte(template)
	if len(t) == 0 {
		t = make([]byte, 1)
	}
	qa := C.int32_t(0)
	if queryIsA {
		qa = 1
	}
	for {
		score, errCode, errPos = make([]int64, n+1), make([]int32, n+1), make([]int64, n+1)
		oa, ob := make([]byte, n*stride+1), make([]byte, n*stride+1)
		ln, st := make([]uint32, n+1), make([]int32, n+1)
		var rc C.int
		if global {
			rc = C.pg_nw_align_batch((*C.uint8_t)(unsafe.Pointer(&queries[0])), (*C.uint64_t)(unsafe.Pointer(&qOffsets[0])), C.uint64_t(n),
				(*C.uint8_t)(unsafe.Pointer(&t[0])), C.uint64_t(len(template)), qa, (*C.int16_t)(unsafe.Pointer(&lutA[0])),
				(*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])), C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
				(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])),
				(*C.uint8_t)(unsafe.Pointer(&oa[0])), (*C.uint8_t)(unsafe.Pointer(&ob[0])), C.uint64_t(stride),
				(*C.uint32_t)(unsafe.Pointer(&ln[0])), (*C.int32_t)(unsafe.Pointer(&st[0])))
		} else {
			rc = C.pg_sw_align_batch((*C.uint8_t)(unsafe.Pointer(&queries[0])), (*C.uint64_t)(unsafe.Pointer(&qOffsets[0])), C.uint64_t(n),
				(*C.uint8_t)(unsafe.Pointer(&t[0])), C.uint64_t(len(template)), qa, (*C.int16_t)(unsafe.Pointer(&lutA[0])),
				(*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])), C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
				(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])),
				(*C.uint8_t)(unsafe.Pointer(&oa[0])), (*C.uint8_t)(unsafe.Pointer(&ob[0])), C.uint64_t(stride),
				(*C.uint32_t)(unsafe.Pointer(&ln[0])), (*C.int32_t)(unsafe.Pointer(&st[0])))
		}
		if e := check(rc); e != nil {
			return nil, nil, nil, nil, nil, e
		}
		grow := 0
		for i := 0; i < n; i++ {
			if st[i] == 2 && int(ln[i]) > grow {
				grow = int(ln[i])
			}
		}
		if grow > 0 {
			stride = grow + 8
			continue
		}
		alignA, alignB = make([]string, n), make([]string, n)
		for i := 0; i < n; i++ {
			alignA[i] = string(oa[i*stride : i*stride+int(ln[i])])
			alignB[i] = string(ob[i*stride : i*stride+int(ln[i])])
		}
		return score[:n], errCode[:n], errPos[:n], alignA, alignB, nil
	}
}

// ScorePairs wraps pg_sw_score_pairs (global = false) / pg_nw_score_pairs (global = true): pair p scores
// A[pairA[p]] against B[pairB[p]] of the two flattened sets.
func ScorePairs(global bool, aBases []byte, aOff []uint64, bBases []byte, bOff []uint64, pairA, pairB []uint32,
	lutA, lutB *[256]int16, table []int64, nA, nB int, gap int64) (score []int64, errCode []int32, errPos []int64, err error) {
	n := len(pairA)
	score, errCode, errPos = make([]int64, n+1), make([]int32, n+1), make([]int64, n+1)
	pa, pb := append(pairA[:n:n], 0), append(pairB[:n:n], 0) // copies with room for &pa[0] when n == 0
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	var rc C.int
	if global {
		rc = C.pg_nw_score_pairs((*C.uint8_t)(unsafe.Pointer(&aBases[0])), (*C.uint64_t)(unsafe.Pointer(&aOff[0])), C.uint64_t(len(aOff)-1),
			(*C.uint8_t)(unsafe.Pointer(&bBases[0])), (*C.uint64_t)(unsafe.Pointer(&bOff[0])), C.uint64_t(len(bOff)-1),
			(*C.uint32_t)(unsafe.Pointer(&pa[0])), (*C.uint32_t)(unsafe.Pointer(&pb[0])), C.uint64_t(n),
			(*C.int16_t)(unsafe.Pointer(&lutA[0])), (*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])),
			C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
			(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])))
	} else {
		rc = C.pg_sw_score_pairs((*C.uint8_t)(unsafe.Pointer(&aBases[0])), (*C.uint64_t)(unsafe.Pointer(&aOff[0])), C.uint64_t(len(aOff)-1),
			(*C.uint8_t)(unsafe.Pointer(&bBases[0])), (*C.uint64_t)(unsafe.Pointer(&bOff[0])), C.uint64_t(len(bOff)-1),
			(*C.uint32_t)(unsafe.Pointer(&pa[0])), (*C.uint32_t)(unsafe.Pointer(&pb[0])), C.uint64_t(n),
			(*C.int16_t)(unsafe.Pointer(&lutA[0])), (*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])),
			C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
			(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])))
	}
	return score[:n], errCode[:n], errPos[:n], check(rc)
}

// AlignPairs wraps pg_sw_align_pairs / pg_nw_align_pairs: ScorePairs plus the two aligned strings of
// every pair.  Rows are len(a) + len(b) bytes wide, which no alignment exceeds.
func AlignPairs(global bool, aBases []byte, aOff []uint64, bBases []byte, bOff []uint64, pairA, pairB []uint32,
	lutA, lutB *[256]int16, table []int64, nA, nB int, gap int64) (score []int64, errCode []int32, errPos []int64, alignA, alignB []string, err error) {
	n := len(pairA)
	stride := 1
	for p := 0; p < n; p++ {
		if int(pairA[p]) < len(aOff)-1 && int(pairB[p]) < len(bOff)-1 {
			if w := int(aOff[pairA[p]+1]-aOff[pairA[p]]) + int(bOff[pairB[p]+1]-bOff[pairB[p]]); w > stride {
				stride = w
			}
		}
	}
	score, errCode, errPos = make([]int64, n+1), make([]int32, n+1), make([]int64, n+1)
	oa, ob := make([]byte, n*stride+1), make([]byte, n*stride+1)
	ln, st := make([]uint32, n+1), make([]int32, n+1)
	pa, pb := append(pairA[:n:n], 0), append(pairB[:n:n], 0)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	var rc C.int
	if global {
		rc = C.pg_nw_align_pairs((*C.uint8_t)(unsafe.Pointer(&aBases[0])), (*C.uint64_t)(unsafe.Pointer(&aOff[0])), C.uint64_t(len(aOff)-1),
			(*C.uint8_t)(unsafe.Pointer(&bBases[0])), (*C.uint64_t)(unsafe.Pointer(&bOff[0])), C.uint64_t(len(bOff)-1),
			(*C.uint32_t)(unsafe.Pointer(&pa[0])), (*C.uint32_t)(unsafe.Pointer(&pb[0])), C.uint64_t(n),
			(*C.int16_t)(unsafe.Pointer(&lutA[0])), (*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])),
			C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
			(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])),
			(*C.uint8_t)(unsafe.Pointer(&oa[0])), (*C.uint8_t)(unsafe.Pointer(&ob[0])), C.uint64_t(stride),
			(*C.uint32_t)(unsafe.Pointer(&ln[0])), (*C.int32_t)(unsafe.Pointer(&st[0])))
	} else {
		rc = C.pg_sw_align_pairs((*C.uint8_t)(unsafe.Pointer(&aBases[0])), (*C.uint64_t)(unsafe.Pointer(&aOff[0])), C.uint64_t(len(aOff)-1),
			(*C.uint8_t)(unsafe.Pointer(&bBases[0])), (*C.uint64_t)(unsafe.Pointer(&bOff[0])), C.uint64_t(len(bOff)-1),
			(*C.uint32_t)(unsafe.Pointer(&pa[0])), (*C.uint32_t)(unsafe.Pointer(&pb[0])), C.uint64_t(n),
			(*C.int16_t)(unsafe.Pointer(&lutA[0])), (*C.int16_t)(unsafe.Pointer(&lutB[0])), (*C.int64_t)(unsafe.Pointer(&table[0])),
			C.int32_t(nA), C.int32_t(nB), C.int64_t(gap),
			(*C.int64_t)(unsafe.Pointer(&score[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.int64_t)(unsafe.Pointer(&errPos[0])),
			(*C.uint8_t)(unsafe.Pointer(&oa[0])), (*C.uint8_t)(unsafe.Pointer(&ob[0])), C.uint64_t(stride),
			(*C.uint32_t)(unsafe.Pointer(&ln[0])), (*C.int32_t)(unsafe.Pointer(&st[0])))
	}
	if e := check(rc); e != nil {
		return nil, nil, nil, nil, nil, e
	}
	alignA, alignB = make([]string, n), make([]string, n)
	for p := 0; p < n; p++ {
		alignA[p] = string(oa[p*stride : p*stride+int(ln[p])])
		alignB[p] = string(ob[p*stride : p*stride+int(ln[p])])
	}
	return score[:n], errCode[:n], errPos[:n], alignA, alignB, nil
}

// TmBatch wraps pg_tm_batch.
func TmBatch(bases []byte, offsets []uint64, cp, na, mg float64) (tm, dH, dS []float64, status []int32, err error) {
	n := len(offsets) - 1
	tm, dH, dS, status = make([]float64, n+1), make([]float64, n+1), make([]float64, n+1), make([]int32, n+1)
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_tm_batch((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
		C.double(cp), C.double(na), C.double(mg), (*C.double)(unsafe.Pointer(&tm[0])), (*C.double)(unsafe.Pointer(&dH[0])),
		(*C.double)(unsafe.Pointer(&dS[0])), (*C.int32_t)(unsafe.Pointer(&status[0])))
	return tm[:n], dH[:n], dS[:n], status[:n], check(rc)
}

// FastaIngest parses a whole FASTA text on the GPU (pg_fasta_ingest): dense sequence bytes +
// offsets and dense name bytes + offsets for the records fasta.Parse would return, and the
// error it would stop with (errCode 0 = nil; errLine = the line number its message prints).
func FastaIngest(text []byte, maxLineSize int, bufioAlias bool) (seq []byte, seqOff []uint64, names []byte, nameOff []uint64, errCode int, errLine uint64, err error) {
	if len(text) == 0 {
		return nil, []uint64{0}, nil, []uint64{0}, 0, 0, nil
	}
	lines := 1
	for _, c := range text {
		if c == '\n' {
			lines++
		}
	}
	seq, names = make([]byte, len(text)), make([]byte, len(text))
	seqOff, nameOff = make([]uint64, lines+1), make([]uint64, lines+1)
	var n, tot, ntot C.uint64_t
	var ec C.int32_t
	var el C.uint64_t
	flags := C.uint32_t(0)
	if bufioAlias {
		flags = C.PG_FASTA_BUFIO_ALIAS
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_fasta_ingest((*C.uint8_t)(unsafe.Pointer(&text[0])), C.uint64_t(len(text)), C.uint32_t(maxLineSize), flags,
		(*C.uint8_t)(unsafe.Pointer(&seq[0])), C.uint64_t(len(seq)), (*C.uint64_t)(unsafe.Pointer(&seqOff[0])),
		(*C.uint8_t)(unsafe.Pointer(&names[0])), C.uint64_t(len(names)), (*C.uint64_t)(unsafe.Pointer(&nameOff[0])),
		C.uint64_t(lines), &n, &tot, &ntot, &ec, &el)
	if err = check(rc); err != nil {
		return nil, nil, nil, nil, 0, 0, err
	}
	return seq[:tot], seqOff[:n+1], names[:ntot], nameOff[:n+1], int(ec), uint64(el), nil
}

// DesignPrimersBatch wraps pg_design_primers_batch: per sequence the lengths of the forward and
// reverse primers of pcr.DesignPrimersWithOverhangs (status 1: the reference slices out of range).
func DesignPrimersBatch(bases []byte, offsets []uint64, targetTm float64) (fwdLen, revLen []uint32, status []int32, err error) {
	n := len(offsets) - 1
	fwdLen, revLen, status = make([]uint32, n+1), make([]uint32, n+1), make([]int32, n+1)
	base := (*C.uint8_t)(nil)
	if len(bases) > 0 {
		base = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_design_primers_batch(base, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n), C.double(targetTm),
		(*C.uint32_t)(unsafe.Pointer(&fwdLen[0])), (*C.uint32_t)(unsafe.Pointer(&revLen[0])), (*C.int32_t)(unsafe.Pointer(&status[0])))
	return fwdLen[:n], revLen[:n], status[:n], check(rc)
}

// MinimalPrimerBatch wraps pg_pcr_minimal_primer_batch (the loop of pcr.go:93-100 for every primer).
func MinimalPrimerBatch(bases []byte, offsets []uint64, targetTm float64) (minLen []uint32, status []int32, err error) {
	n := len(offsets) - 1
	minLen, status = make([]uint32, n+1), make([]int32, n+1)
	base := (*C.uint8_t)(nil)
	if len(bases) > 0 {
		base = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	runtime.LockOSThread()
	defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
	rc := C.pg_pcr_minimal_primer_batch(base, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n), C.double(targetTm),
		(*C.uint32_t)(unsafe.Pointer(&minLen[0])), (*C.int32_t)(unsafe.Pointer(&status[0])))
	return minLen[:n], status[:n], check(rc)
}

// Site is one exact occurrence of a pattern in a sequence.
type Site struct {
	Seq     int
	Pos     int
	Pattern int
}

// FindSites wraps pg_find_sites_batch: every (overlapping) occurrence of every pattern in every
// sequence, what suffixarray.Lookup(pattern, -1) returns per sequence.  Order is unspecified.
func FindSites(seqs []byte, seqOff []uint64, patterns []byte, patOff []uint64) ([]Site, error) {
	nSeq, nPat := len(seqOff)-1, len(patOff)-1
	if nSeq <= 0 || nPat <= 0 || len(seqs) == 0 || len(patterns) == 0 {
		return nil, nil
	}
	capHits := 1024
	for {
		hs, hp, hq := make([]uint32, capHits), make([]uint64, capHits), make([]uint32, capHits)
		var n C.uint64_t
		runtime.LockOSThread()
		defer runtime.UnlockOSThread() // pg_last_error() is thread-local: read it on the calling thread
		rc := C.pg_find_sites_batch((*C.uint8_t)(unsafe.Pointer(&seqs[0])), (*C.uint64_t)(unsafe.Pointer(&seqOff[0])), C.uint64_t(nSeq),
			(*C.uint8_t)(unsafe.Pointer(&patterns[0])), (*C.uint64_t)(unsafe.Pointer(&patOff[0])), C.uint32_t(nPat), 0,
			(*C.uint32_t)(unsafe.Pointer(&hs[0])), (*C.uint64_t)(unsafe.Pointer(&hp[0])), (*C.uint32_t)(unsafe.Pointer(&hq[0])),
			C.uint64_t(capHits), &n)
		if rc == C.PG_ERR_ARG && int(n) > capHits {
			capHits = int(n)
			continue
		}
		if err := check(rc); err != nil {
			return nil, err
		}
		sites := make([]Site, int(n))
		for i := range sites {
			sites[i] = Site{Seq: int(hs[i]), Pos: int(hp[i]), Pattern: int(hq[i])}
		}
		return sites, nil
	}
}

// FastqIngestRecords wraps pg_fastq_ingest_records: dense sequences + offsets, and per record the
// spans {identifier line begin, length, quality line begin, length} into text.
func FastqIngestRecords(text []byte) (bases []byte, offsets []uint64, spans []uint64, errCode int32, errLine uint64, err error) {
	newlines := 0
	for _, c := range text {
		if c == '\n' {
			newlines++
		}
	}
	capRec := newlines/4 + 1
	bases = make([]byte, len(text)+1)
	offsets = make([]uint64, capRec+1)
	spans = make([]uint64, 4*(capRec+1))
	var n, total C.uint64_t
	var code C.int32_t
	var line C.uint64_t
	var tp *C.uint8_t
	if len(text) > 0 {
		tp = (*C.uint8_t)(unsafe.Pointer(&text[0]))
	}
	err = locked(func() C.int {
		return C.pg_fastq_ingest_records(tp, C.uint64_t(len(text)), (*C.uint8_t)(unsafe.Pointer(&bases[0])), C.uint64_t(len(bases)),
			(*C.uint64_t)(unsafe.Pointer(&offsets[0])), (*C.uint64_t)(unsafe.Pointer(&spans[0])), C.uint64_t(capRec), &n, &total, &code, &line)
	})
	return bases[:total], offsets[:n+1], spans[:4*n], int32(code), uint64(line), err
}

// Index wraps a pg_mash_index: a reference sketch set copied to the device of the calling thread
// (pg_thread_device / pg_init) and indexed there once.  Any number of goroutines may call Query at once; Add
// waits for the queries in flight and they wait for it.  Close must not run while a Query is in flight.
type Index struct {
	h *C.pg_mash_index
}

// MaxTopK is the largest k Query accepts (PG_INDEX_MAX_TOP_K).
const MaxTopK = int(C.PG_INDEX_MAX_TOP_K)

// NewIndex wraps pg_mash_index_create over n sketches of s words each (full arrays, zero tails included).
func NewIndex(sketches []uint32, n, s int) (*Index, error) {
	var h *C.pg_mash_index
	var p *C.uint32_t
	if len(sketches) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	if err := locked(func() C.int { return C.pg_mash_index_create(p, C.uint64_t(n), C.int32_t(s), &h) }); err != nil {
		return nil, err
	}
	return &Index{h: h}, nil
}

// Add wraps pg_mash_index_add: n more sketches of s words each (full arrays, zero tails included) become
// references len .. len + n - 1, merged into the index on the device.
func (ix *Index) Add(sketches []uint32, n, s int) error {
	var p *C.uint32_t
	if len(sketches) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	return locked(func() C.int { return C.pg_mash_index_add(ix.h, p, C.uint64_t(n), C.int32_t(s)) })
}

// Query wraps pg_mash_index_query: for each of nq query sketches of sq words, up to k references with
// same >= minSame, ordered by same descending and then reference index ascending.  Row q of ref / same /
// dist holds nHits[q] entries.
func (ix *Index) Query(queries []uint32, nq, sq, k, minSame int) (ref, same []uint32, dist []float64, nHits []uint32, err error) {
	slots := nq * k
	ref, same, dist, nHits = make([]uint32, slots+1), make([]uint32, slots+1), make([]float64, slots+1), make([]uint32, nq+1)
	var p *C.uint32_t
	if len(queries) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&queries[0]))
	}
	err = locked(func() C.int {
		return C.pg_mash_index_query(ix.h, p, C.uint64_t(nq), C.int32_t(sq), C.uint32_t(k), C.uint32_t(minSame),
			(*C.uint32_t)(unsafe.Pointer(&ref[0])), (*C.uint32_t)(unsafe.Pointer(&same[0])), (*C.double)(unsafe.Pointer(&dist[0])),
			(*C.uint32_t)(unsafe.Pointer(&nHits[0])))
	})
	return ref[:slots], same[:slots], dist[:slots], nHits[:nq], err
}

// QueryWithin wraps pg_mash_index_query_within: for each of nq query sketches of sq words, every reference with
// same >= minSame (>= 1), in reference order.  Query q's hits are entries offsets[q] .. offsets[q+1] of ref / same /
// dist.  A counting call sizes the lists, a second call fills them.
func (ix *Index) QueryWithin(queries []uint32, nq, sq, minSame int) (offsets []uint64, ref, same []uint32, dist []float64, err error) {
	offsets = make([]uint64, nq+1)
	var p *C.uint32_t
	if len(queries) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&queries[0]))
	}
	var total C.uint64_t
	err = locked(func() C.int {
		return C.pg_mash_index_query_within(ix.h, p, C.uint64_t(nq), C.int32_t(sq), C.uint32_t(minSame),
			(*C.uint64_t)(unsafe.Pointer(&offsets[0])), nil, nil, nil, 0, &total)
	})
	if err != nil {
		return nil, nil, nil, nil, err
	}
	m := int(total)
	ref, same, dist = make([]uint32, m+1), make([]uint32, m+1), make([]float64, m+1)
	err = locked(func() C.int {
		return C.pg_mash_index_query_within(ix.h, p, C.uint64_t(nq), C.int32_t(sq), C.uint32_t(minSame),
			(*C.uint64_t)(unsafe.Pointer(&offsets[0])), (*C.uint32_t)(unsafe.Pointer(&ref[0])), (*C.uint32_t)(unsafe.Pointer(&same[0])),
			(*C.double)(unsafe.Pointer(&dist[0])), C.uint64_t(m), &total)
	})
	return offsets, ref[:m], same[:m], dist[:m], err
}

// Close wraps pg_mash_index_free.
func (ix *Index) Close() error {
	if ix.h == nil {
		return nil
	}
	h := ix.h
	ix.h = nil
	return locked(func() C.int { return C.pg_mash_index_free(h) })
}

// Dereplicator wraps a pg_mash_dereplicator: a dereplication that grows batch by batch on the device of the
// calling thread.  Adds from several goroutines are serialised by the library.  Close must not run while an Add
// is in flight.
type Dereplicator struct {
	h *C.pg_mash_dereplicator
}

// NewDereplicator wraps pg_mash_dereplicator_create for sketches of s words at same >= minSame.
func NewDereplicator(s, minSame int, nearest bool) (*Dereplicator, error) {
	flags := C.uint32_t(0)
	if nearest {
		flags = C.PG_DEREP_NEAREST
	}
	var h *C.pg_mash_dereplicator
	if err := locked(func() C.int { return C.pg_mash_dereplicator_create(C.int32_t(s), C.uint32_t(minSame), flags, &h) }); err != nil {
		return nil, err
	}
	return &Dereplicator{h: h}, nil
}

// Add wraps pg_mash_dereplicator_add: n sketches of s words each (full arrays, zero tails included) become sketches
// first .. first + n - 1; rep[i] is the id of row i's representative (first + i for a new one).
func (d *Dereplicator) Add(sketches []uint32, n, s int) (rep []uint32, first, nNew uint64, err error) {
	rep = make([]uint32, n+1)
	var p *C.uint32_t
	if len(sketches) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	var f, nn C.uint64_t
	err = locked(func() C.int {
		return C.pg_mash_dereplicator_add(d.h, p, C.uint64_t(n), C.int32_t(s), (*C.uint32_t)(unsafe.Pointer(&rep[0])), &f, &nn)
	})
	return rep[:n], uint64(f), uint64(nn), err
}

// Reps wraps pg_mash_dereplicator_reps: the ids of the representatives kept so far, ascending.
func (d *Dereplicator) Reps() ([]uint32, error) {
	var n C.uint64_t
	ids := make([]uint32, 1)
	for {
		capIDs := len(ids) - 1
		err := locked(func() C.int { return C.pg_mash_dereplicator_reps(d.h, (*C.uint32_t)(unsafe.Pointer(&ids[0])), C.uint64_t(capIDs), &n) })
		if err == nil {
			return ids[:n], nil
		}
		if int(n) <= capIDs {
			return nil, err
		}
		ids = make([]uint32, int(n)+1) // an add kept more since the last call
	}
}

// Close wraps pg_mash_dereplicator_free.
func (d *Dereplicator) Close() error {
	if d.h == nil {
		return nil
	}
	h := d.h
	d.h = nil
	return locked(func() C.int { return C.pg_mash_dereplicator_free(h) })
}

// Clusterer wraps a pg_mash_clusterer: a single-linkage clustering that grows batch by batch on the device of the
// calling thread.  Adds from several goroutines are serialised by the library.  Close must not run while an Add
// is in flight.
type Clusterer struct {
	h *C.pg_mash_clusterer
}

// NewClusterer wraps pg_mash_clusterer_create for sketches of s words at same >= minSame.
func NewClusterer(s, minSame int) (*Clusterer, error) {
	var h *C.pg_mash_clusterer
	if err := locked(func() C.int { return C.pg_mash_clusterer_create(C.int32_t(s), C.uint32_t(minSame), &h) }); err != nil {
		return nil, err
	}
	return &Clusterer{h: h}, nil
}

// Add wraps pg_mash_clusterer_add: n sketches of s words each (full arrays, zero tails included) become sketches
// first .. first + n - 1; label[i] is row i's label after the add, nGroups every group, nLinks the links this add
// found and nMerged the earlier groups it absorbed into another.
func (c *Clusterer) Add(sketches []uint32, n, s int) (label []uint32, first, nGroups, nLinks, nMerged uint64, err error) {
	label = make([]uint32, n+1)
	var p *C.uint32_t
	if len(sketches) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	var f, g, l, m C.uint64_t
	err = locked(func() C.int {
		return C.pg_mash_clusterer_add(c.h, p, C.uint64_t(n), C.int32_t(s), (*C.uint32_t)(unsafe.Pointer(&label[0])), &f, &g, &l, &m)
	})
	return label[:n], uint64(f), uint64(g), uint64(l), uint64(m), err
}

// Labels wraps pg_mash_clusterer_labels: the current labels of sketches [begin, end).
func (c *Clusterer) Labels(begin, end int) ([]uint32, error) {
	size := 0
	if end > begin {
		size = end - begin
	}
	out := make([]uint32, size+1)
	err := locked(func() C.int {
		return C.pg_mash_clusterer_labels(c.h, C.uint64_t(begin), C.uint64_t(end), (*C.uint32_t)(unsafe.Pointer(&out[0])))
	})
	if err != nil {
		return nil, err
	}
	return out[:size], nil
}

// Close wraps pg_mash_clusterer_free.
func (c *Clusterer) Close() error {
	if c.h == nil {
		return nil
	}
	h := c.h
	c.h = nil
	return locked(func() C.int { return C.pg_mash_clusterer_free(h) })
}

// Screen wraps a pg_mash_screen: a reference sketch set and one pool of reads per sample on the device of the
// calling thread.  Close must not run while another call on it is in flight.
type Screen struct {
	h       *C.pg_mash_screen
	n       int
	samples int
}

// NewScreen wraps pg_mash_screen_create for n references of s words each (full arrays, zero tails included) and
// k-mer size k.
func NewScreen(sketches []uint32, n, s, k int) (*Screen, error) { return NewScreenSamples(sketches, n, s, k, 1) }

// NewScreenSamples wraps pg_mash_screen_create_samples: NewScreen with one pool for each of `samples` samples.
func NewScreenSamples(sketches []uint32, n, s, k, samples int) (*Screen, error) {
	return NewScreenFlags(sketches, n, s, k, samples, 0)
}

// NewScreenFlags wraps pg_mash_screen_create_flags: NewScreenSamples with flags (0 or KmerCanonical).
func NewScreenFlags(sketches []uint32, n, s, k, samples int, flags uint32) (*Screen, error) {
	var h *C.pg_mash_screen
	var p *C.uint32_t
	if len(sketches) > 0 {
		p = (*C.uint32_t)(unsafe.Pointer(&sketches[0]))
	}
	if samples < 0 || uint64(samples) > 0xffffffff {
		return nil, errors.New("polyb200: sample count does not fit 32 bits")
	}
	if err := locked(func() C.int {
		return C.pg_mash_screen_create_flags(p, C.uint64_t(n), C.int32_t(s), C.int32_t(k), C.uint32_t(samples), C.uint32_t(flags), &h)
	}); err != nil {
		return nil, err
	}
	return &Screen{h: h, n: n, samples: samples}, nil
}

// Add wraps pg_mash_screen_add: every window of the reads is counted into the pool.
func (sc *Screen) Add(reads []string) error {
	if len(reads) == 0 {
		return nil
	}
	bases, offsets := Flatten(reads)
	return locked(func() C.int {
		return C.pg_mash_screen_add(sc.h, (*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(len(reads)))
	})
}

// AddSamples wraps pg_mash_screen_add_samples: every window of reads[i] is counted into the pool of sample ids[i].
func (sc *Screen) AddSamples(reads []string, ids []uint32) error {
	if len(ids) != len(reads) {
		return errors.New("polyb200: one sample id per read")
	}
	if len(reads) == 0 {
		return nil
	}
	bases, offsets := Flatten(reads)
	return locked(func() C.int {
		return C.pg_mash_screen_add_samples(sc.h, (*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])),
			(*C.uint32_t)(unsafe.Pointer(&ids[0])), C.uint64_t(len(reads)))
	})
}

// Reset wraps pg_mash_screen_reset: the pool of every sample is emptied.
func (sc *Screen) Reset() error { return locked(func() C.int { return C.pg_mash_screen_reset(sc.h) }) }

// Results wraps pg_mash_screen_results: per reference, the shared hash count, the containment and the median
// multiplicity of the pool so far.
func (sc *Screen) Results() (shared []uint32, containment []float64, multiplicity []uint64, err error) {
	shared, containment, multiplicity = make([]uint32, sc.n+1), make([]float64, sc.n+1), make([]uint64, sc.n+1)
	err = locked(func() C.int {
		return C.pg_mash_screen_results(sc.h, (*C.uint32_t)(unsafe.Pointer(&shared[0])), (*C.double)(unsafe.Pointer(&containment[0])),
			(*C.uint64_t)(unsafe.Pointer(&multiplicity[0])))
	})
	return shared[:sc.n], containment[:sc.n], multiplicity[:sc.n], err
}

// Winners wraps pg_mash_screen_winners: the three arrays of Results after Mash Screen's winner-take-all, each pool
// hash given to the reference that holds it with the largest first-pass shared count (ties to the smallest index).
func (sc *Screen) Winners() (shared []uint32, containment []float64, multiplicity []uint64, err error) {
	shared, containment, multiplicity = make([]uint32, sc.n+1), make([]float64, sc.n+1), make([]uint64, sc.n+1)
	err = locked(func() C.int {
		return C.pg_mash_screen_winners(sc.h, (*C.uint32_t)(unsafe.Pointer(&shared[0])), (*C.double)(unsafe.Pointer(&containment[0])),
			(*C.uint64_t)(unsafe.Pointer(&multiplicity[0])))
	})
	return shared[:sc.n], containment[:sc.n], multiplicity[:sc.n], err
}

// ResultsSamples wraps pg_mash_screen_results_samples: the arrays of Results for samples [first, first+count),
// row-major (element (q-first)*n + r).
func (sc *Screen) ResultsSamples(first, count int) (shared []uint32, containment []float64, multiplicity []uint64, err error) {
	return sc.table(true, first, count)
}

// WinnersSamples wraps pg_mash_screen_winners_samples: the arrays of Winners for samples [first, first+count), each
// sample voting alone, row-major as ResultsSamples.
func (sc *Screen) WinnersSamples(first, count int) (shared []uint32, containment []float64, multiplicity []uint64, err error) {
	return sc.table(false, first, count)
}

func (sc *Screen) table(results bool, first, count int) (shared []uint32, containment []float64, multiplicity []uint64, err error) {
	if first < 0 || count < 0 || first+count > sc.samples {
		return nil, nil, nil, errors.New("polyb200: sample rows out of range")
	}
	m := sc.n * count
	shared, containment, multiplicity = make([]uint32, m+1), make([]float64, m+1), make([]uint64, m+1)
	err = locked(func() C.int {
		sh, c, mu := (*C.uint32_t)(unsafe.Pointer(&shared[0])), (*C.double)(unsafe.Pointer(&containment[0])), (*C.uint64_t)(unsafe.Pointer(&multiplicity[0]))
		if results {
			return C.pg_mash_screen_results_samples(sc.h, C.uint32_t(first), C.uint32_t(count), sh, c, mu)
		}
		return C.pg_mash_screen_winners_samples(sc.h, C.uint32_t(first), C.uint32_t(count), sh, c, mu)
	})
	return shared[:m], containment[:m], multiplicity[:m], err
}

// Close wraps pg_mash_screen_free.
func (sc *Screen) Close() error {
	if sc.h == nil {
		return nil
	}
	h := sc.h
	sc.h = nil
	return locked(func() C.int { return C.pg_mash_screen_free(h) })
}

// SeqhashBatch wraps pg_seqhash_batch: digest[32*i:32*i+32], errCode[i] and errPos[i] for each of the
// sequences bases[offsets[i]:offsets[i+1]], all of one seqType (0 DNA, 1 RNA, 2 PROTEIN) and flags
// (1 circular | 2 double-stranded).
func SeqhashBatch(bases []byte, offsets []uint64, seqType int32, flags uint32) (digest []byte, errCode []int32, errPos []uint64, err error) {
	n := len(offsets) - 1
	digest, errCode, errPos = make([]byte, 32*n+32), make([]int32, n+1), make([]uint64, n+1)
	var p *C.uint8_t
	if len(bases) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	err = locked(func() C.int {
		return C.pg_seqhash_batch(p, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n), C.int32_t(seqType), C.uint32_t(flags),
			(*C.uint8_t)(unsafe.Pointer(&digest[0])), (*C.int32_t)(unsafe.Pointer(&errCode[0])), (*C.uint64_t)(unsafe.Pointer(&errPos[0])))
	})
	return digest[:32*n], errCode[:n], errPos[:n], err
}

// LeastRotationBatch wraps pg_least_rotation_batch: the smallest start of the least rotation of each sequence.
func LeastRotationBatch(bases []byte, offsets []uint64) ([]uint64, error) {
	n := len(offsets) - 1
	rot := make([]uint64, n+1)
	var p *C.uint8_t
	if len(bases) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	err := locked(func() C.int {
		return C.pg_least_rotation_batch(p, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n), (*C.uint64_t)(unsafe.Pointer(&rot[0])))
	})
	return rot[:n], err
}

// FoldZukerBatch wraps pg_fold_zuker_batch: per sequence the minimum free energy, the dot-bracket and the
// item status (PG_ITEM_*).  PG_ERR_PANIC / PG_ERR_UNSUPPORTED are per-item outcomes here, not call errors.
func FoldZukerBatch(bases []byte, offsets []uint64, temp float64) (mfe []float64, dotBracket []string, status []int32, err error) {
	n := len(offsets) - 1
	mfe, status = make([]float64, n+1), make([]int32, n+1)
	dbLen := make([]uint64, n+1)
	db := make([]byte, len(bases)+1)
	var p *C.uint8_t
	if len(bases) > 0 {
		p = (*C.uint8_t)(unsafe.Pointer(&bases[0]))
	}
	err = locked(func() C.int {
		rc := C.pg_fold_zuker_batch(p, (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n), C.double(temp),
			(*C.double)(unsafe.Pointer(&mfe[0])), (*C.uint8_t)(unsafe.Pointer(&db[0])), (*C.uint64_t)(unsafe.Pointer(&dbLen[0])),
			(*C.int32_t)(unsafe.Pointer(&status[0])))
		if rc == C.PG_ERR_PANIC || rc == C.PG_ERR_UNSUPPORTED {
			return C.PG_OK
		}
		return rc
	})
	dotBracket = make([]string, n)
	for i := 0; i < n; i++ {
		b := offsets[i] - offsets[0]
		dotBracket[i] = string(db[b : b+dbLen[i]])
	}
	return mfe[:n], dotBracket, status[:n], err
}

// FragmentBatch wraps pg_fragment_batch: per sequence the item status (PG_ITEM_*), the efficiency, the failing
// step's min and max and the fragment ends (fragment j of item i is [start, ends[i][j]) with start 0 for j = 0,
// else ends[i][j-1] - 4).  An empty include list is Fragment.  PG_ERR_PANIC / PG_ERR_UNSUPPORTED are per-item
// outcomes here, not call errors.
func FragmentBatch(seqs []string, minSize, maxSize int, exclude, include []string) (status []int32, eff []float64, errMin, errMax []int64,
	ends [][]uint64, err error) {
	n := len(seqs)
	bases, offsets := Flatten(seqs)
	ex, exOff := Flatten(exclude)
	inc, incOff := Flatten(include)
	status, eff = make([]int32, n+1), make([]float64, n+1)
	errMin, errMax = make([]int64, n+1), make([]int64, n+1)
	fragOff := make([]uint64, n+1)
	flat := make([]uint64, len(bases)/8+2*n+1)
	var total C.uint64_t
	for attempt := 0; attempt < 2; attempt++ {
		err = locked(func() C.int {
			rc := C.pg_fragment_batch((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])), C.uint64_t(n),
				C.int64_t(minSize), C.int64_t(maxSize), (*C.uint8_t)(unsafe.Pointer(&ex[0])), (*C.uint64_t)(unsafe.Pointer(&exOff[0])),
				C.uint64_t(len(exclude)), (*C.uint8_t)(unsafe.Pointer(&inc[0])), (*C.uint64_t)(unsafe.Pointer(&incOff[0])), C.uint64_t(len(include)),
				(*C.int32_t)(unsafe.Pointer(&status[0])), (*C.double)(unsafe.Pointer(&eff[0])), (*C.int64_t)(unsafe.Pointer(&errMin[0])),
				(*C.int64_t)(unsafe.Pointer(&errMax[0])), (*C.uint64_t)(unsafe.Pointer(&fragOff[0])), (*C.uint64_t)(unsafe.Pointer(&flat[0])),
				C.uint64_t(len(flat)), &total)
			if rc == C.PG_ERR_PANIC || rc == C.PG_ERR_UNSUPPORTED {
				return C.PG_OK
			}
			if rc == C.PG_ERR_ARG && uint64(total) > uint64(len(flat)) {
				return C.PG_OK // too small a guess: once more with the exact count
			}
			return rc
		})
		if err != nil || uint64(total) <= uint64(len(flat)) {
			break
		}
		flat = make([]uint64, uint64(total))
	}
	if err != nil {
		return nil, nil, nil, nil, nil, err
	}
	ends = make([][]uint64, n)
	for i := 0; i < n; i++ {
		ends[i] = flat[fragOff[i]:fragOff[i+1]]
	}
	return status[:n], eff[:n], errMin[:n], errMax[:n], ends, nil
}

// fragmentSets flattens a list of overhang sets for the set entry points.
func fragmentSets(sets [][]string) ([]byte, []uint64, []uint64) {
	var all []string
	setOff := make([]uint64, len(sets)+1)
	for i, s := range sets {
		all = append(all, s...)
		setOff[i+1] = uint64(len(all))
	}
	b, off := Flatten(all)
	return b, off, setOff
}

// FragmentSetEfficiencyBatch wraps pg_fragment_set_efficiency_batch: SetEfficiency of every set.
func FragmentSetEfficiencyBatch(sets [][]string) ([]float64, error) {
	n := len(sets)
	b, off, setOff := fragmentSets(sets)
	eff := make([]float64, n+1)
	err := locked(func() C.int {
		return C.pg_fragment_set_efficiency_batch((*C.uint8_t)(unsafe.Pointer(&b[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])),
			(*C.uint64_t)(unsafe.Pointer(&setOff[0])), C.uint64_t(n), (*C.double)(unsafe.Pointer(&eff[0])))
	})
	return eff[:n], err
}

// FragmentNextOverhangsBatch wraps pg_fragment_next_overhangs_batch: NextOverhangs of every set.
func FragmentNextOverhangsBatch(sets [][]string) (cands [][]string, effs [][]float64, err error) {
	n := len(sets)
	b, off, setOff := fragmentSets(sets)
	raw := make([]byte, 1024*n+1)
	nc := make([]uint32, n+1)
	eff := make([]float64, 256*n+1)
	err = locked(func() C.int {
		return C.pg_fragment_next_overhangs_batch((*C.uint8_t)(unsafe.Pointer(&b[0])), (*C.uint64_t)(unsafe.Pointer(&off[0])),
			(*C.uint64_t)(unsafe.Pointer(&setOff[0])), C.uint64_t(n), (*C.uint8_t)(unsafe.Pointer(&raw[0])), (*C.uint32_t)(unsafe.Pointer(&nc[0])),
			(*C.double)(unsafe.Pointer(&eff[0])))
	})
	if err != nil {
		return nil, nil, err
	}
	cands, effs = make([][]string, n), make([][]float64, n)
	for i := 0; i < n; i++ {
		for j := 0; j < int(nc[i]); j++ {
			cands[i] = append(cands[i], string(raw[1024*i+4*j:1024*i+4*j+4]))
		}
		effs[i] = eff[256*i : 256*i+int(nc[i])]
	}
	return cands, effs, nil
}

// CloneEnzyme is an enzyme for the clone entry points: the two sites are literals (clone.go:77-84).
type CloneEnzyme struct {
	ForwardSite, ReverseSite, RecognitionSite string
	Skip, OverheadLength                      int
}

// cEnzymes copies enzymes into C memory (the struct holds pointers, which may not point into Go memory);
// free releases it.
func cEnzymes(enzymes []CloneEnzyme) (p *C.pg_clone_enzyme, free func()) {
	n := len(enzymes)
	arr := (*[1 << 20]C.pg_clone_enzyme)(C.malloc(C.size_t(n+1) * C.size_t(unsafe.Sizeof(C.pg_clone_enzyme{}))))[: n+1 : n+1]
	var strs []unsafe.Pointer
	cstr := func(s string) *C.uint8_t {
		b := C.CBytes([]byte(s + "\x00"))
		strs = append(strs, b)
		return (*C.uint8_t)(b)
	}
	for i, e := range enzymes {
		arr[i] = C.pg_clone_enzyme{forward_site: cstr(e.ForwardSite), forward_len: C.uint32_t(len(e.ForwardSite)),
			reverse_site: cstr(e.ReverseSite), reverse_len: C.uint32_t(len(e.ReverseSite)),
			recognition_site: cstr(e.RecognitionSite), recognition_len: C.uint32_t(len(e.RecognitionSite)),
			skip: C.int32_t(e.Skip), overhang_length: C.int32_t(e.OverheadLength)}
	}
	return &arr[0], func() {
		for _, s := range strs {
			C.free(s)
		}
		C.free(unsafe.Pointer(&arr[0]))
	}
}

// CloneFragments is pg_clone_digest_batch's output: fragment f is Seq[SeqOff[f]:SeqOff[f+1]] with overhangs
// OH[OHOff[2f]:OHOff[2f+1]] and OH[OHOff[2f+1]:OHOff[2f+2]]; Count[i] fragments for item i.
type CloneFragments struct {
	Count         []uint32
	Status        []int32
	Seq, OH       []byte
	SeqOff, OHOff []uint64
}

// CloneDigest wraps pg_clone_digest_batch: CutWithEnzyme of every part x enzyme (item = part*len(enzymes)+enzyme).
// ErrPanic when an item panics in the reference; the other items' fragments are still returned.
func CloneDigest(bases []byte, offsets []uint64, circular []bool, enzymes []CloneEnzyme, directional bool) (*CloneFragments, error) {
	n := len(offsets) - 1
	circ := make([]uint8, n+1)
	for i, c := range circular {
		if c {
			circ[i] = 1
		}
	}
	enz, free := cEnzymes(enzymes)
	defer free()
	dir := C.int32_t(0)
	if directional {
		dir = 1
	}
	items := n*len(enzymes) + 1
	out := &CloneFragments{Count: make([]uint32, items), Status: make([]int32, items)}
	var caps, need [3]C.uint64_t
	for {
		out.Seq, out.OH = make([]byte, caps[1]+1), make([]byte, caps[2]+1)
		out.SeqOff, out.OHOff = make([]uint64, caps[0]+1), make([]uint64, 2*caps[0]+1)
		rc := C.int(0)
		_ = locked(func() C.int {
			rc = C.pg_clone_digest_batch((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])),
				(*C.uint8_t)(unsafe.Pointer(&circ[0])), C.uint64_t(n), enz, C.uint32_t(len(enzymes)), dir,
				(*C.uint32_t)(unsafe.Pointer(&out.Count[0])), (*C.int32_t)(unsafe.Pointer(&out.Status[0])),
				(*C.uint8_t)(unsafe.Pointer(&out.Seq[0])), caps[1], (*C.uint64_t)(unsafe.Pointer(&out.SeqOff[0])),
				(*C.uint8_t)(unsafe.Pointer(&out.OH[0])), caps[2], (*C.uint64_t)(unsafe.Pointer(&out.OHOff[0])), caps[0],
				&need[0], &need[1], &need[2])
			return rc
		})
		if rc == C.PG_ERR_ARG && (need[0] > caps[0] || need[1] > caps[1] || need[2] > caps[2]) {
			caps = need
			continue
		}
		out.Count, out.Status = out.Count[:items-1], out.Status[:items-1]
		return out, cloneCheck(rc)
	}
}

// CloneConstructs is the output of the ligation entry points: construct k is Bytes[Off[k]:Off[k+1]],
// Kind[k] 0 a clone or 1 a looping construct; Counts[2r], Counts[2r+1] per reaction; Status[r] per reaction.
type CloneConstructs struct {
	Bytes  []byte
	Off    []uint64
	Kind   []uint8
	Counts []uint64
	Status []int32
}

// cloneLigation runs one ligation entry point with buffers grown to the reported need.
func cloneLigation(nReactions int, call func(bcap, ccap C.uint64_t, o *CloneConstructs, nb, nc *C.uint64_t) C.int) (*CloneConstructs, error) {
	bcap, ccap := C.uint64_t(1<<20), C.uint64_t(1<<12)
	for {
		o := &CloneConstructs{Bytes: make([]byte, bcap+1), Off: make([]uint64, ccap+1), Kind: make([]uint8, ccap+1),
			Counts: make([]uint64, 2*nReactions+2), Status: make([]int32, nReactions+1)}
		var nb, nc C.uint64_t
		rc := C.int(0)
		_ = locked(func() C.int { rc = call(bcap, ccap, o, &nb, &nc); return rc })
		if rc == C.PG_ERR_ARG && (nb > bcap || nc > ccap) {
			if nb > bcap {
				bcap = nb
			}
			if nc > ccap {
				ccap = nc
			}
			continue
		}
		return o, cloneCheck(rc)
	}
}

// CloneGoldenGate wraps pg_clone_golden_gate_batch: reaction r is parts [reactionOffsets[r], reactionOffsets[r+1]).
func CloneGoldenGate(bases []byte, offsets []uint64, circular []bool, reactionOffsets []uint64, enzyme CloneEnzyme) (*CloneConstructs, error) {
	n, R := len(offsets)-1, len(reactionOffsets)-1
	circ := make([]uint8, n+1)
	for i, c := range circular {
		if c {
			circ[i] = 1
		}
	}
	enz, free := cEnzymes([]CloneEnzyme{enzyme})
	defer free()
	return cloneLigation(R, func(bcap, ccap C.uint64_t, o *CloneConstructs, nb, nc *C.uint64_t) C.int {
		return C.pg_clone_golden_gate_batch((*C.uint8_t)(unsafe.Pointer(&bases[0])), (*C.uint64_t)(unsafe.Pointer(&offsets[0])),
			(*C.uint8_t)(unsafe.Pointer(&circ[0])), C.uint64_t(n), (*C.uint64_t)(unsafe.Pointer(&reactionOffsets[0])), C.uint64_t(R), enz,
			bcap, ccap, (*C.uint8_t)(unsafe.Pointer(&o.Bytes[0])), (*C.uint64_t)(unsafe.Pointer(&o.Off[0])), (*C.uint8_t)(unsafe.Pointer(&o.Kind[0])),
			nil, (*C.uint64_t)(unsafe.Pointer(&o.Counts[0])), (*C.int32_t)(unsafe.Pointer(&o.Status[0])), nb, nc)
	})
}

// CloneCircularLigate wraps pg_clone_circular_ligate_batch on fragments in CloneFragments' layout.
func CloneCircularLigate(seq []byte, seqOff []uint64, oh []byte, ohOff []uint64, reactionOffsets []uint64) (*CloneConstructs, error) {
	nf, R := len(seqOff)-1, len(reactionOffsets)-1
	return cloneLigation(R, func(bcap, ccap C.uint64_t, o *CloneConstructs, nb, nc *C.uint64_t) C.int {
		return C.pg_clone_circular_ligate_batch((*C.uint8_t)(unsafe.Pointer(&seq[0])), (*C.uint64_t)(unsafe.Pointer(&seqOff[0])),
			(*C.uint8_t)(unsafe.Pointer(&oh[0])), (*C.uint64_t)(unsafe.Pointer(&ohOff[0])), C.uint64_t(nf),
			(*C.uint64_t)(unsafe.Pointer(&reactionOffsets[0])), C.uint64_t(R), bcap, ccap, (*C.uint8_t)(unsafe.Pointer(&o.Bytes[0])),
			(*C.uint64_t)(unsafe.Pointer(&o.Off[0])), (*C.uint8_t)(unsafe.Pointer(&o.Kind[0])), nil, (*C.uint64_t)(unsafe.Pointer(&o.Counts[0])), nb, nc)
	})
}
