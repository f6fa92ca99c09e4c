// Package mash is the drop-in for github.com/bebop/poly/search/mash backed by libpolyb200.so:
// same exported names and semantics (search/mash/mash.go:52-140 of the reference), plus
// batched entry points.  NOT COMPILED HERE (no Go toolchain in the build image).
package mash

import (
	"errors"
	"fmt"
	"math"
	"sort"
	"sync"

	"github.com/bebop/poly/internal/polyb200"
)

// Mash is a collection of hashes of kmers from a given sequence (mash.go:52-56).
type Mash struct {
	KmerSize   int
	SketchSize int
	Sketches   []uint32
}

// New initializes a new mash sketch (mash.go:59-65).
func New(kmerSize int, sketchSize int) *Mash {
	return &Mash{KmerSize: kmerSize, SketchSize: sketchSize, Sketches: make([]uint32, sketchSize)}
}

// Sketch generates a mash sketch of the sequence (mash.go:68-104), on the GPU.
func (mash *Mash) Sketch(sequence string) {
	n := len(sequence) - mash.KmerSize
	if n <= 0 {
		return // the reference's loop body never runs (mash.go:73)
	}
	cnt := n
	if cnt > mash.SketchSize {
		cnt = mash.SketchSize
	}
	bases, offsets := polyb200.Flatten([]string{sequence})
	stride := cnt
	if stride < 1 {
		stride = 1
	}
	out, _, _, err := polyb200.SketchBatch(bases, offsets, mash.KmerSize, mash.SketchSize, stride)
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]") // mash.go:96-98 with sketchSize in {0,1}
	} else if err != nil {
		panic(err)
	}
	copy(mash.Sketches[:cnt], out[:cnt]) // n < s: the tail keeps its previous contents (mash.go:81-84)
}

func (mash *Mash) pair(other *Mash) (float64, float64) {
	sk := append(append([]uint32{}, mash.Sketches[:mash.SketchSize]...), other.Sketches[:other.SketchSize]...)
	off := []uint64{0, uint64(mash.SketchSize), uint64(mash.SketchSize + other.SketchSize)}
	_, sim, dist, err := polyb200.SimilarityPairs(sk, off, []uint32{0}, []uint32{1})
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]")
	} else if err != nil {
		panic(err)
	}
	return sim[0], dist[0]
}

// Similarity returns the Jaccard similarity between two sketches (mash.go:107-135).
func (mash *Mash) Similarity(other *Mash) float64 { s, _ := mash.pair(other); return s }

// Distance returns the Jaccard distance between two sketches (mash.go:138-140).
func (mash *Mash) Distance(other *Mash) float64 { _, d := mash.pair(other); return d }

// SketchBatch is New(kmerSize, sketchSize) + Sketch(seq) for every sequence: one call, sharded over every
// GPU of the box (reads are independent, mash.go:68-104; no collective is involved).
func SketchBatch(sequences []string, kmerSize, sketchSize int) []*Mash {
	if sketchSize < 0 {
		panic("runtime error: makeslice: len out of range") // mash.New would
	}
	bases, offsets := polyb200.Flatten(sequences)
	// one zeroed slab for all Sketches arrays (the runtime hands out zeroed memory, as New's make does per read);
	// the library writes the informative words of every row in place and leaves the zero tails alone
	slab := make([]uint32, len(sequences)*sketchSize)
	_, status, err := polyb200.SketchInto(bases, offsets, kmerSize, sketchSize, slab, nil)
	if err != nil && !errors.Is(err, polyb200.ErrPanic) {
		panic(err)
	}
	res := make([]*Mash, len(sequences))
	for i := range sequences {
		if status[i] != 0 {
			panic("runtime error: index out of range [-1]")
		}
		res[i] = &Mash{KmerSize: kmerSize, SketchSize: sketchSize,
			Sketches: slab[i*sketchSize : (i+1)*sketchSize : (i+1)*sketchSize]}
	}
	return res
}

// SketchGroups returns one sketch per group of sequences: a draft assembly's contigs (`mash sketch genome.fa`) or a
// sample's reads (`mash sketch -r -m minCopies`).  Each holds the smallest sketchSize distinct window hashes of its
// group seen at least minCopies times, ascending, then a zero tail when fewer qualify.  Windows never cross a
// sequence.  The sketches compare with Similarity and Distance like those of Sketch.
func SketchGroups(groups [][]string, kmerSize, sketchSize, minCopies int) ([]*Mash, error) {
	return sketchGroups(groups, kmerSize, sketchSize, minCopies, 0)
}

// SketchGroupsCanonical is SketchGroups over canonical k-mers, as Mash hashes them: the windows 0 .. L-k of each
// sequence, each the smaller of itself and its reverse complement, so contigs of either orientation and reads of either
// strand count as one (kmerSize >= 1).
func SketchGroupsCanonical(groups [][]string, kmerSize, sketchSize, minCopies int) ([]*Mash, error) {
	return sketchGroups(groups, kmerSize, sketchSize, minCopies, polyb200.KmerCanonical)
}

func sketchGroups(groups [][]string, kmerSize, sketchSize, minCopies int, flags uint32) ([]*Mash, error) {
	if minCopies < 1 || minCopies > math.MaxUint32 {
		return nil, fmt.Errorf("mash: minCopies %d out of range", minCopies)
	}
	var seqs []string
	goff := make([]uint64, 1, len(groups)+1)
	for _, g := range groups {
		seqs = append(seqs, g...)
		goff = append(goff, uint64(len(seqs)))
	}
	bases, offsets := polyb200.Flatten(seqs)
	out, _, err := polyb200.SketchGroupsFlags(bases, offsets, goff, kmerSize, sketchSize, uint32(minCopies), flags)
	if err != nil {
		return nil, err
	}
	res := make([]*Mash, len(groups))
	for g := range groups {
		res[g] = &Mash{KmerSize: kmerSize, SketchSize: sketchSize, Sketches: out[g*sketchSize : (g+1)*sketchSize : (g+1)*sketchSize]}
	}
	return res, nil
}

// DistResult is Dist's answer for every (query, reference) pair, row-major with the query as the row:
// index q*len(refs) + r.
type DistResult = polyb200.DistResult

// DistPairs is DistWithin's answer, sorted by (query, reference).
type DistPairs = polyb200.DistPairs

// distRows lays a sketch set out as the C ABI's rows.  A *Mash holds no count, so a sketch's count is the length of the
// strictly ascending prefix of Sketches; a sketch whose words are all zero is empty.  This reads the sketches of
// SketchGroups and Sketcher exactly (their rows are ascending with a zero tail); a real hash of 0 can only open a row,
// and is counted there when the row goes on.
func distRows(set []*Mash, s int) (rows, count []uint32, err error) {
	rows, count = make([]uint32, len(set)*s), make([]uint32, len(set))
	for i, m := range set {
		if m.SketchSize != s || len(m.Sketches) < s {
			return nil, nil, fmt.Errorf("mash: sketch %d has SketchSize %d, want %d", i, m.SketchSize, s)
		}
		copy(rows[i*s:(i+1)*s], m.Sketches[:s])
		n := 0
		if s > 0 && (m.Sketches[0] != 0 || (s > 1 && m.Sketches[1] != 0)) {
			n = 1
			for n < s && m.Sketches[n] > m.Sketches[n-1] {
				n++
			}
		}
		count[i] = uint32(n)
	}
	return rows, count, nil
}

func distInputs(queries, refs []*Mash) (s, k int, err error) {
	switch {
	case len(queries) > 0:
		s, k = queries[0].SketchSize, queries[0].KmerSize
	case len(refs) > 0:
		s, k = refs[0].SketchSize, refs[0].KmerSize
	default:
		return 1, 1, nil
	}
	for _, m := range append(append([]*Mash{}, queries...), refs...) {
		if m.KmerSize != k {
			return 0, 0, fmt.Errorf("mash: sketches of kmerSize %d and %d", k, m.KmerSize)
		}
	}
	return s, k, nil
}

// Dist is `mash dist` over grouped sketches: for every query and reference, Mash's shared count among the bottom
// SketchSize values of the pair's union (Denom = min(SketchSize, union size)), the distance -ln(2J/(1+J))/k with
// J = Common/Denom, and the p-value from the genome lengths (bases behind each sketch; nil lengths: no p-value).
// Unlike Distance, a sketch with fewer than SketchSize values compares as the set it is.  All sketches share one
// SketchSize and KmerSize.  A sketch's count is the length of the strictly ascending prefix of its Sketches, and a
// sketch of all zeros is empty: what SketchGroups and Sketcher return.
func Dist(queries, refs []*Mash, qLen, rLen []uint64) (DistResult, error) {
	s, k, err := distInputs(queries, refs)
	if err != nil {
		return DistResult{}, err
	}
	q, qc, err := distRows(queries, s)
	if err != nil {
		return DistResult{}, err
	}
	r, rc, err := distRows(refs, s)
	if err != nil {
		return DistResult{}, err
	}
	return polyb200.Dist(q, qc, r, rc, s, k, qLen, rLen)
}

// DistWithin is `mash dist -d maxDistance -v maxPValue` (upper: `mash triangle`, a set against itself, reference >
// query only): the pairs of Dist within both limits, sorted by (query, reference).  Counts are read as in Dist.
func DistWithin(queries, refs []*Mash, qLen, rLen []uint64, maxDistance, maxPValue float64, upper bool) (DistPairs, error) {
	s, k, err := distInputs(queries, refs)
	if err != nil {
		return DistPairs{}, err
	}
	q, qc, err := distRows(queries, s)
	if err != nil {
		return DistPairs{}, err
	}
	r, rc, err := distRows(refs, s)
	if err != nil {
		return DistPairs{}, err
	}
	p, err := polyb200.DistWithin(q, qc, r, rc, s, k, qLen, rLen, maxDistance, maxPValue, upper)
	if err != nil {
		return DistPairs{}, err
	}
	order := make([]int, len(p.Q))
	for i := range order {
		order[i] = i
	}
	sort.Slice(order, func(a, b int) bool {
		x, y := order[a], order[b]
		return p.Q[x] < p.Q[y] || (p.Q[x] == p.Q[y] && p.R[x] < p.R[y])
	})
	out := DistPairs{}
	for _, i := range order {
		out.Q, out.R = append(out.Q, p.Q[i]), append(out.R, p.R[i])
		out.Common, out.Denom, out.Distance = append(out.Common, p.Common[i]), append(out.Denom, p.Denom[i]), append(out.Distance, p.Distance[i])
		if p.PValue != nil {
			out.PValue = append(out.PValue, p.PValue[i])
		}
	}
	return out, nil
}

// Sketcher grows SketchGroups in place: nGroups sketches fed batch by batch, for read sets larger than the GPU or a
// host can stage.  Per group it keeps a cap (2^32 at first, never growing) and every value below it with its count
// saturated at minCopies; after an add the cap is the smallest of the old cap, the sketchSize-th value seen minCopies
// times plus one, and the (maxValues+1)-th distinct value.  A sketch is complete when it holds sketchSize values or
// its cap is still 2^32: a complete sketch equals SketchGroups over every sequence added to the group, whatever the
// split, and every sketch is a prefix of that one.  With minCopies 1 every sketch is complete.  Call Close when done.
type Sketcher struct {
	sk           *polyb200.Sketcher
	k, s, groups int
}

// NewSketcher prepares nGroups sketches; maxValues <= 0 means 64 * sketchSize.
func NewSketcher(nGroups, kmerSize, sketchSize, minCopies, maxValues int) (*Sketcher, error) {
	return newSketcher(nGroups, kmerSize, sketchSize, minCopies, maxValues, 0)
}

// NewSketcherCanonical is NewSketcher over canonical k-mers (see SketchGroupsCanonical, whose sketches its complete
// sketches equal).
func NewSketcherCanonical(nGroups, kmerSize, sketchSize, minCopies, maxValues int) (*Sketcher, error) {
	return newSketcher(nGroups, kmerSize, sketchSize, minCopies, maxValues, polyb200.KmerCanonical)
}

func newSketcher(nGroups, kmerSize, sketchSize, minCopies, maxValues int, flags uint32) (*Sketcher, error) {
	if nGroups < 0 || minCopies < 1 || minCopies > math.MaxUint32 {
		return nil, fmt.Errorf("mash: nGroups %d or minCopies %d out of range", nGroups, minCopies)
	}
	if maxValues <= 0 {
		maxValues = 64 * sketchSize
	}
	sk, err := polyb200.NewSketcherFlags(uint64(nGroups), kmerSize, sketchSize, uint32(minCopies), uint64(maxValues), flags)
	if err != nil {
		return nil, err
	}
	return &Sketcher{sk: sk, k: kmerSize, s: sketchSize, groups: nGroups}, nil
}

// Add counts the sequences of groups[i] into group firstGroup + i.
func (s *Sketcher) Add(groups [][]string, firstGroup int) error {
	if firstGroup < 0 {
		return fmt.Errorf("mash: firstGroup %d out of range", firstGroup)
	}
	var seqs []string
	goff := make([]uint64, 1, len(groups)+1)
	for _, g := range groups {
		seqs = append(seqs, g...)
		goff = append(goff, uint64(len(seqs)))
	}
	if len(seqs) == 0 {
		return nil
	}
	bases, offsets := polyb200.Flatten(seqs)
	return s.sk.Add(bases, offsets, goff, uint64(firstGroup))
}

// Sketches returns one sketch per group so far, and whether each is complete.
func (s *Sketcher) Sketches() ([]*Mash, []bool, error) {
	out, _, complete, _, err := s.sk.Rows()
	if err != nil {
		return nil, nil, err
	}
	res := make([]*Mash, s.groups)
	for g := range res {
		res[g] = &Mash{KmerSize: s.k, SketchSize: s.s, Sketches: out[g*s.s : (g+1)*s.s : (g+1)*s.s]}
	}
	return res, complete, nil
}

// Close releases the sketcher's device memory.
func (s *Sketcher) Close() error { return s.sk.Close() }

// DistanceMatrix returns D[i][j] = sketches[i].Distance(sketches[j]) for sketches of one common SketchSize.
func DistanceMatrix(sketches []*Mash) [][]float64 {
	n := len(sketches)
	if n == 0 {
		return nil
	}
	s := sketches[0].SketchSize
	flat := make([]uint32, 0, n*s)
	for _, m := range sketches {
		flat = append(flat, m.Sketches[:s]...)
	}
	_, dist, err := polyb200.DistanceBlock(flat, n, s, 0, n)
	if err != nil {
		panic(err)
	}
	res := make([][]float64, n)
	for i := range res {
		res[i] = dist[i*n : (i+1)*n]
	}
	return res
}

// RelatedPair is one pair of sketches that share at least one hash.
type RelatedPair struct {
	I, J     int     // indices into the sketch list, I < J
	Same     int     // matching hashes as the walk of Similarity counts them (mash.go:121-132)
	Distance float64 // sketches[I].Distance(sketches[J]) == 1 - Same/SketchSize (mash.go:134,139)
}

// RelatedPairs returns every pair i < j of ascending (select-regime) or zero-padded sketches of one common SketchSize
// whose Distance is below 1, i.e. the non-trivial entries of DistanceMatrix, without materialising the n x n matrix
// (for n = 100k sketches: 334 MB instead of 40 GB).  Pairs that are not returned have Distance 1.
func RelatedPairs(sketches []*Mash) []RelatedPair {
	n := len(sketches)
	if n == 0 {
		return nil
	}
	s := sketches[0].SketchSize
	flat := make([]uint32, 0, n*s)
	for _, m := range sketches {
		flat = append(flat, m.Sketches[:s]...)
	}
	pi, pj, same, err := polyb200.DistanceSparse(flat, n, s, 0, n, true)
	if err != nil {
		panic(err)
	}
	out := make([]RelatedPair, len(pi))
	for t := range pi {
		out[t] = RelatedPair{I: int(pi[t]), J: int(pj[t]), Same: int(same[t]), Distance: 1 - float64(same[t])/float64(s)}
	}
	return out
}

// Cluster groups sketches of one common SketchSize by single linkage: sketches i < j are linked when
// sketches[i].Distance(sketches[j]) <= maxDistance (the lower index is the receiver), and the groups are the connected
// components.  labels[i] is the smallest index in i's group, so labels[i] == i marks one representative per group.
// The threshold is turned into a matching count by evaluating Distance's own expression 1 - same/SketchSize
// (mash.go:134,139), so a maxDistance that sits exactly on a pair's Distance includes the pair.  A maxDistance that
// every pair satisfies (>= 1) is an error; one that none can satisfy labels every sketch with itself.
func Cluster(sketches []*Mash, maxDistance float64) ([]int, error) {
	n := len(sketches)
	if n == 0 {
		return nil, nil
	}
	s := sketches[0].SketchSize
	minSame := 0
	for minSame <= s && !(1-float64(minSame)/float64(s) <= maxDistance) {
		minSame++
	}
	if minSame == 0 && s > 0 {
		return nil, fmt.Errorf("mash: maxDistance %v links every pair", maxDistance)
	}
	labels := make([]int, n)
	if minSame > s && s > 0 {
		for i := range labels {
			labels[i] = i
		}
		return labels, nil
	}
	flat := make([]uint32, 0, n*s)
	for _, m := range sketches {
		if m.SketchSize != s {
			return nil, errors.New("mash: Cluster needs one common SketchSize")
		}
		flat = append(flat, m.Sketches[:s]...)
	}
	label, _, _, err := polyb200.Cluster(flat, n, s, minSame)
	if err != nil {
		return nil, err
	}
	for i, l := range label {
		labels[i] = int(l)
	}
	return labels, nil
}

// Dereplicate picks representatives of sketches of one common SketchSize, in index order: sketch i is a
// representative iff no representative r < i has sketches[r].Distance(sketches[i]) <= maxDistance.  It returns
// rep, with rep[i] == i for a representative; any other sketch gets the first representative within the cut, or
// with nearest the one at the smallest Distance (the earlier one on a tie).  That is the result of
//
//	for i := range sketches {
//		for _, r := range reps { if sketches[r].Distance(sketches[i]) <= maxDistance { rep[i] = r; continue outer } }
//		reps = append(reps, i); rep[i] = i
//	}
//
// computed in one GPU pass.  Permute sketches first to give some of them priority.  The threshold becomes a matching
// count as in Cluster; a maxDistance that every pair satisfies (>= 1) is an error, one that none can satisfy makes
// every sketch its own representative.
func Dereplicate(sketches []*Mash, maxDistance float64, nearest bool) ([]int, error) {
	n := len(sketches)
	if n == 0 {
		return nil, nil
	}
	s := sketches[0].SketchSize
	minSame := 0
	for minSame <= s && !(1-float64(minSame)/float64(s) <= maxDistance) {
		minSame++
	}
	if minSame == 0 && s > 0 {
		return nil, fmt.Errorf("mash: maxDistance %v links every pair", maxDistance)
	}
	reps := make([]int, n)
	if minSame > s && s > 0 {
		for i := range reps {
			reps[i] = i
		}
		return reps, nil
	}
	flat := make([]uint32, 0, n*s)
	for _, m := range sketches {
		if m.SketchSize != s {
			return nil, errors.New("mash: Dereplicate needs one common SketchSize")
		}
		flat = append(flat, m.Sketches[:s]...)
	}
	rep, _, err := polyb200.Dereplicate(flat, n, s, minSame, nearest)
	if err != nil {
		return nil, err
	}
	for i, r := range rep {
		reps[i] = int(r)
	}
	return reps, nil
}

// Dereplicator is a dereplication that grows: each Add assigns a batch of sketches against the representatives kept
// so far, on the GPU, without dereplicating the earlier sketches again.  Sketches are numbered in the order they are
// added, and after any sequence of adds the concatenated results equal Dereplicate of the concatenated batches.
// Safe for concurrent use; call Close when done.
type Dereplicator struct {
	d *polyb200.Dereplicator
	s int
}

// NewDereplicator prepares a dereplication of sketches of SketchSize s at Distance <= maxDistance, with the
// assignment of Dereplicate.  A maxDistance that every pair satisfies, or none can, is an error.
func NewDereplicator(s int, maxDistance float64, nearest bool) (*Dereplicator, error) {
	if s <= 0 {
		panic("runtime error: index out of range [-1]") // Similarity on a sketch of size 0 would
	}
	minSame := 0
	for minSame <= s && !(1-float64(minSame)/float64(s) <= maxDistance) {
		minSame++
	}
	if minSame == 0 || minSame > s {
		return nil, fmt.Errorf("mash: maxDistance %v links every pair or none", maxDistance)
	}
	d, err := polyb200.NewDereplicator(s, minSame, nearest)
	if err != nil {
		return nil, err
	}
	return &Dereplicator{d: d, s: s}, nil
}

// Add assigns a batch of sketches of the dereplicator's SketchSize.  rep[i] is the position, among every sketch
// added so far, of the representative of sketches[i]; it is first + i when sketches[i] is a new representative.
func (d *Dereplicator) Add(sketches []*Mash) (rep []int, first int, err error) {
	flat := make([]uint32, 0, len(sketches)*d.s)
	for _, m := range sketches {
		if m.SketchSize != d.s {
			return nil, 0, errors.New("mash: Dereplicator needs one common SketchSize")
		}
		flat = append(flat, m.Sketches[:d.s]...)
	}
	r, f, _, err := d.d.Add(flat, len(sketches), d.s)
	if err != nil {
		return nil, 0, err
	}
	rep = make([]int, len(r))
	for i, x := range r {
		rep[i] = int(x)
	}
	return rep, int(f), nil
}

// Reps returns the positions of the representatives kept so far, ascending.
func (d *Dereplicator) Reps() ([]int, error) {
	ids, err := d.d.Reps()
	if err != nil {
		return nil, err
	}
	out := make([]int, len(ids))
	for i, x := range ids {
		out[i] = int(x)
	}
	return out, nil
}

// Close releases the dereplicator's device memory.
func (d *Dereplicator) Close() error { return d.d.Close() }

// Clusterer is a clustering that grows: each Add merges a batch of sketches into the single-linkage groups of the
// sketches added so far, on the GPU, without clustering the earlier sketches again.  Sketches are numbered in the
// order they are added, and after every add Labels equals Cluster of the concatenated batches.  Earlier labels
// change when a batch joins two earlier groups (Merged > 0).  Safe for concurrent use; call Close when done.
type Clusterer struct {
	c  *polyb200.Clusterer
	s  int
	mu sync.Mutex
	n  int
}

// ClusterBatch is the result of one Add.
type ClusterBatch struct {
	Labels []int // the label of each batch sketch after the add; batch[i] is sketch First + i
	First  int
	Groups int   // every group after the add
	Links  int   // the links this add found
	Merged int   // earlier groups absorbed into another by this add; 0 means no earlier label changed
}

// NewClusterer prepares a clustering of sketches of SketchSize s at Distance <= maxDistance, with the links of
// Cluster.  A maxDistance that every pair satisfies, or none can, is an error.
func NewClusterer(s int, maxDistance float64) (*Clusterer, error) {
	if s <= 0 {
		panic("runtime error: index out of range [-1]") // Similarity on a sketch of size 0 would
	}
	minSame := 0
	for minSame <= s && !(1-float64(minSame)/float64(s) <= maxDistance) {
		minSame++
	}
	if minSame == 0 || minSame > s {
		return nil, fmt.Errorf("mash: maxDistance %v links every pair or none", maxDistance)
	}
	c, err := polyb200.NewClusterer(s, minSame)
	if err != nil {
		return nil, err
	}
	return &Clusterer{c: c, s: s}, nil
}

// Add merges a batch of sketches of the clusterer's SketchSize.
func (c *Clusterer) Add(sketches []*Mash) (ClusterBatch, error) {
	flat := make([]uint32, 0, len(sketches)*c.s)
	for _, m := range sketches {
		if m.SketchSize != c.s {
			return ClusterBatch{}, errors.New("mash: Clusterer needs one common SketchSize")
		}
		flat = append(flat, m.Sketches[:c.s]...)
	}
	label, first, groups, links, merged, err := c.c.Add(flat, len(sketches), c.s)
	if err != nil {
		return ClusterBatch{}, err
	}
	out := ClusterBatch{Labels: make([]int, len(label)), First: int(first), Groups: int(groups), Links: int(links), Merged: int(merged)}
	for i, x := range label {
		out.Labels[i] = int(x)
	}
	c.mu.Lock()
	if end := out.First + len(label); end > c.n {
		c.n = end
	}
	c.mu.Unlock()
	return out, nil
}

// N returns the number of sketches added through Add so far.
func (c *Clusterer) N() int {
	c.mu.Lock()
	defer c.mu.Unlock()
	return c.n
}

// Labels returns the current labels of sketches [begin, end).
func (c *Clusterer) Labels(begin, end int) ([]int, error) {
	ids, err := c.c.Labels(begin, end)
	if err != nil {
		return nil, err
	}
	out := make([]int, len(ids))
	for i, x := range ids {
		out[i] = int(x)
	}
	return out, nil
}

// Close releases the clusterer's device memory.
func (c *Clusterer) Close() error { return c.c.Close() }

// Screen is Mash Screen (Ondov et al. 2019) on the GPU: which of a set of reference sketches a pool of reads
// contains.  Add counts every window a Sketch would hash of every read (forward strand, raw bytes; canonical k-mers for
// NewScreenCanonical) into the pool;
// Results gives, per reference, Shared = the sum over hashes v of min(c_ref(v), c_pool(v)), Containment = Shared /
// SketchSize and Multiplicity = the lower median pool count of the shared hashes; Winners gives them after Mash
// Screen's winner-take-all.  Any split of the pool into Adds gives the same Results and Winners, and Reset empties
// the pool.  Identity is Containment^(1/kmerSize), computed on the host.  A screen made by NewScreenSamples holds one
// pool per sample of a multiplexed run: AddSamples tags each read with its sample, and ResultsSamples and
// WinnersSamples answer, for each sample, what a screen fed only that sample's reads would answer.  Add counts into
// sample 0, and Results and Winners answer for it.
// Call Close when done.
type Screen struct {
	sc *polyb200.Screen
	k  int
}

// ScreenResult is the answer for one reference.
type ScreenResult struct {
	Shared       int
	Containment  float64
	Multiplicity uint64
	Identity     float64
}

// NewScreen prepares a screen against refs, which must share one SketchSize, for k-mers of kmerSize (the size they
// were sketched with; it is not checked, as Similarity does not check it).
func NewScreen(refs []*Mash, kmerSize int) (*Screen, error) { return NewScreenSamples(refs, kmerSize, 1) }

// NewScreenSamples is NewScreen with one pool for each of `samples` samples (samples >= 1).
func NewScreenSamples(refs []*Mash, kmerSize int, samples int) (*Screen, error) {
	return newScreen(refs, kmerSize, samples, 0)
}

// NewScreenCanonical is NewScreenSamples counting canonical k-mers, for refs sketched the same way (SketchGroupsCanonical;
// the mode, like kmerSize, is not checked), so reads of both strands count.
func NewScreenCanonical(refs []*Mash, kmerSize int, samples int) (*Screen, error) {
	return newScreen(refs, kmerSize, samples, polyb200.KmerCanonical)
}

func newScreen(refs []*Mash, kmerSize int, samples int, flags uint32) (*Screen, error) {
	s := 0
	if len(refs) > 0 {
		s = refs[0].SketchSize
	}
	flat := make([]uint32, 0, len(refs)*s)
	for _, m := range refs {
		if m.SketchSize != s {
			return nil, errors.New("mash: Screen needs one common SketchSize")
		}
		flat = append(flat, m.Sketches[:s]...)
	}
	if len(refs) > 0 && s <= 0 {
		panic("runtime error: index out of range [-1]") // Similarity on a sketch of size 0 would
	}
	sc, err := polyb200.NewScreenFlags(flat, len(refs), s, kmerSize, samples, flags)
	if err != nil {
		return nil, err
	}
	return &Screen{sc: sc, k: kmerSize}, nil
}

// Add counts the windows of reads into the pool.
func (s *Screen) Add(reads []string) error { return s.sc.Add(reads) }

// AddSamples counts the windows of reads[i] into the pool of sample samples[i].
func (s *Screen) AddSamples(reads []string, samples []int) error {
	ids := make([]uint32, len(samples))
	for i, q := range samples {
		if q < 0 || uint64(q) > 0xffffffff {
			return errors.New("mash: sample id does not fit 32 bits")
		}
		ids[i] = uint32(q)
	}
	return s.sc.AddSamples(reads, ids)
}

// Reset empties the pool of every sample.
func (s *Screen) Reset() error { return s.sc.Reset() }

// Results returns one ScreenResult per reference, in the order given to NewScreen.
func (s *Screen) Results() ([]ScreenResult, error) {
	return s.resultsOf(s.sc.Results())
}

// Winners returns one ScreenResult per reference after Mash Screen's winner-take-all (mash screen -w): each pool
// hash is given to the reference that holds it with the largest Shared of Results, a tie to the smallest index, and
// every field is recomputed over the hashes a reference won.  Sibling strains of the one a pool came from then stop
// reporting the hashes it explains better.
func (s *Screen) Winners() ([]ScreenResult, error) {
	return s.resultsOf(s.sc.Winners())
}

// ResultsSamples returns, for each sample q in [first, first+count), one ScreenResult per reference.
func (s *Screen) ResultsSamples(first, count int) ([][]ScreenResult, error) {
	return s.rowsOf(count)(s.sc.ResultsSamples(first, count))
}

// WinnersSamples returns Winners for each sample q in [first, first+count); every sample votes alone.
func (s *Screen) WinnersSamples(first, count int) ([][]ScreenResult, error) {
	return s.rowsOf(count)(s.sc.WinnersSamples(first, count))
}

func (s *Screen) rowsOf(count int) func([]uint32, []float64, []uint64, error) ([][]ScreenResult, error) {
	return func(shared []uint32, cont []float64, mult []uint64, err error) ([][]ScreenResult, error) {
		flat, err := s.resultsOf(shared, cont, mult, err)
		if err != nil {
			return nil, err
		}
		out := make([][]ScreenResult, count)
		if count > 0 {
			n := len(flat) / count
			for q := range out {
				out[q] = flat[q*n : (q+1)*n]
			}
		}
		return out, nil
	}
}

func (s *Screen) resultsOf(shared []uint32, cont []float64, mult []uint64, err error) ([]ScreenResult, error) {
	if err != nil {
		return nil, err
	}
	out := make([]ScreenResult, len(shared))
	for i := range out {
		out[i] = ScreenResult{Shared: int(shared[i]), Containment: cont[i], Multiplicity: mult[i], Identity: math.Pow(cont[i], 1/float64(s.k))}
	}
	return out, nil
}

// Close releases the screen's device memory.
func (s *Screen) Close() error { return s.sc.Close() }

// Neighbor is one reference of a Nearest result.
type Neighbor struct {
	Index    int     // position in the reference list given to NewIndex
	Same     int     // matching hashes as query.Similarity(reference) counts them (mash.go:121-132)
	Distance float64 // query.Distance(reference) (mash.go:134,139)
}

// Index holds a reference sketch set on the GPU for repeated nearest-neighbour queries (the sketches are
// copied; the references may be changed or dropped afterwards).  Safe for concurrent use; call Close when done.
type Index struct {
	ix *polyb200.Index
	mu sync.Mutex // guards n and s, which Add changes
	n  int
	s  int
}

// NewIndex copies references of one common SketchSize to the GPU and indexes them.
func NewIndex(references []*Mash) (*Index, error) {
	s := 0
	if len(references) > 0 {
		s = references[0].SketchSize
	}
	flat := make([]uint32, 0, len(references)*s)
	for _, m := range references {
		if m.SketchSize != s {
			return nil, errors.New("mash: every reference of an index must have the same SketchSize")
		}
		flat = append(flat, m.Sketches[:s]...)
	}
	ix, err := polyb200.NewIndex(flat, len(references), s)
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]") // Similarity on a sketch of size 0 would
	} else if err != nil {
		return nil, err
	}
	return &Index{ix: ix, n: len(references), s: s}, nil
}

// Add appends references of the index's SketchSize (any one SketchSize when the index holds none yet) on the
// GPU: they take the next positions, and later queries answer as an index built over the whole list would.
func (ix *Index) Add(references []*Mash) error {
	if len(references) == 0 {
		return nil
	}
	s := references[0].SketchSize
	flat := make([]uint32, 0, len(references)*s)
	for _, m := range references {
		if m.SketchSize != s {
			return errors.New("mash: every reference of an index must have the same SketchSize")
		}
		flat = append(flat, m.Sketches[:s]...)
	}
	ix.mu.Lock()
	defer ix.mu.Unlock()
	if ix.n > 0 && s != ix.s {
		return errors.New("mash: every reference of an index must have the same SketchSize")
	}
	err := ix.ix.Add(flat, len(references), s)
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]") // Similarity on a sketch of size 0 would
	} else if err != nil {
		return err
	}
	ix.n += len(references)
	ix.s = s
	return nil
}

// Nearest returns, for each query (all of one SketchSize), the k references with the largest matching counts
// (query.Similarity(reference), the query as receiver) that share at least one hash, ordered by count
// descending and then by reference position.  1 <= k <= 1024.
func (ix *Index) Nearest(queries []*Mash, k int) [][]Neighbor {
	sq := 0
	if len(queries) > 0 {
		sq = queries[0].SketchSize
	}
	flat := make([]uint32, 0, len(queries)*sq)
	for _, m := range queries {
		if m.SketchSize != sq {
			panic("mash: every query of a batch must have the same SketchSize")
		}
		flat = append(flat, m.Sketches[:sq]...)
	}
	ref, same, dist, nHits, err := ix.ix.Query(flat, len(queries), sq, k, 1)
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]")
	} else if err != nil {
		panic(err)
	}
	res := make([][]Neighbor, len(queries))
	for q := range res {
		res[q] = make([]Neighbor, nHits[q])
		for t := range res[q] {
			res[q][t] = Neighbor{Index: int(ref[q*k+t]), Same: int(same[q*k+t]), Distance: dist[q*k+t]}
		}
	}
	return res
}

// Within returns, for each query (all of one SketchSize), every reference with query.Distance(reference) <=
// maxDistance, however many there are, ordered by reference position.  The threshold becomes a matching count
// as in Cluster, over min(query SketchSize, reference SketchSize); a maxDistance that every pair satisfies (>= 1)
// is an error.
func (ix *Index) Within(queries []*Mash, maxDistance float64) ([][]Neighbor, error) {
	sq := 0
	if len(queries) > 0 {
		sq = queries[0].SketchSize
	}
	ix.mu.Lock()
	den := sq
	if ix.s < den {
		den = ix.s
	}
	ix.mu.Unlock()
	minSame := 0
	for minSame <= den && !(1-float64(minSame)/float64(den) <= maxDistance) {
		minSame++
	}
	if minSame == 0 && den > 0 {
		return nil, fmt.Errorf("mash: maxDistance %v lists every pair", maxDistance)
	}
	flat := make([]uint32, 0, len(queries)*sq)
	for _, m := range queries {
		if m.SketchSize != sq {
			return nil, errors.New("mash: every query of a batch must have the same SketchSize")
		}
		flat = append(flat, m.Sketches[:sq]...)
	}
	off, ref, same, dist, err := ix.ix.QueryWithin(flat, len(queries), sq, minSame)
	if errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: index out of range [-1]")
	} else if err != nil {
		return nil, err
	}
	res := make([][]Neighbor, len(queries))
	for q := range res {
		res[q] = make([]Neighbor, 0, off[q+1]-off[q])
		for h := off[q]; h < off[q+1]; h++ {
			res[q] = append(res[q], Neighbor{Index: int(ref[h]), Same: int(same[h]), Distance: dist[h]})
		}
	}
	return res, nil
}

// Close releases the index's device memory.
func (ix *Index) Close() error { return ix.ix.Close() }
