// Package pcr is the H100-backed drop-in for bebop/poly's primers/pcr (primers/pcr/pcr.go): same
// exported functions and results.  The Tm searches (DesignPrimers*: pcr.go:44-60; the minimal-primer
// loop of SimulateSimple: pcr.go:93-100) and the binding-site search the reference does with a suffix
// array (pcr.go:87,110-115) run on the GPU through libpolyb200.so; the fragment assembly
// (pcr.go:117-166,181-195) is the same bookkeeping as in the reference.
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image); see INTEGRATION.md.
package pcr

import (
	"errors"
	"sort"
	"strings"

	"github.com/bebop/poly/internal/polyb200"
	"github.com/bebop/poly/transform"
)

// shortest binding part the Tm loop of SimulateSimple starts from (reference: pcr.go:35; the 15 of
// pcr.go:38, designedMinimalPrimerLength, only concerns DesignPrimers and lives in the kernel)
const minimalPrimerLength = 7

// DesignPrimersWithOverhangs: reference pcr.go:44-60.  The two Tm searches run on the GPU; the
// strings are cut from the upper-cased sequence with the lengths that come back.
func DesignPrimersWithOverhangs(sequence, forwardOverhang, reverseOverhang string, targetTm float64) (string, string) {
	template := strings.ToUpper(sequence)
	flat, bounds := polyb200.Flatten([]string{template})
	fwdLen, revLen, status, err := polyb200.DesignPrimersBatch(flat, bounds, targetTm)
	if (len(status) > 0 && status[0] == 1) || errors.Is(err, polyb200.ErrPanic) {
		panic("runtime error: slice bounds out of range") // the reference slices past the end of the sequence
	}
	if err != nil {
		panic(err)
	}
	head := template[:fwdLen[0]]
	tail := transform.ReverseComplement(template[len(template)-int(revLen[0]):])
	return forwardOverhang + head, transform.ReverseComplement(reverseOverhang) + tail
}

// DesignPrimers: reference pcr.go:62-66 (no overhangs).
func DesignPrimers(sequence string, targetTm float64) (string, string) {
	return DesignPrimersWithOverhangs(sequence, "", "", targetTm)
}

// binding sites of one template: position -> primers bound there (in primer-list order), plus the
// ascending positions
type siteIndex struct {
	primersAt map[int][]int
	positions []int
}

func newSiteIndex() *siteIndex { return &siteIndex{primersAt: map[int][]int{}} }

func (ix *siteIndex) add(pos, primer int) {
	if _, seen := ix.primersAt[pos]; !seen {
		ix.positions = append(ix.positions, pos)
	}
	ix.primersAt[pos] = append(ix.primersAt[pos], primer)
}

// SimulateSimple: reference pcr.go:73-169.  Like the reference it upper-cases primerList in place.
func SimulateSimple(sequences []string, targetTm float64, circular bool, primerList []string) []string {
	for i := range primerList {
		primerList[i] = strings.ToUpper(primerList[i])
	}
	if len(sequences) == 0 {
		return nil
	}
	templates := make([]string, len(sequences))
	for i, s := range sequences {
		templates[i] = strings.ToUpper(s)
	}

	// GPU pass 1: the minimal binding part of every primer (pcr.go:93-103).  A primer whose minimal
	// part is the whole primer is ignored, exactly as the reference does.
	minimal := make([]string, len(primerList))
	var patterns []string
	var patternPrimer []int
	var patternIsReverse []bool
	if len(primerList) > 0 {
		flat, bounds := polyb200.Flatten(primerList)
		minLen, status, err := polyb200.MinimalPrimerBatch(flat, bounds, targetTm)
		for _, st := range status {
			if st == 1 {
				panic("runtime error: slice bounds out of range") // primer shorter than 7 nt
			}
		}
		if err != nil {
			panic(err)
		}
		for p, primer := range primerList {
			part := primer[len(primer)-int(minLen[p]):]
			if part == primer {
				continue
			}
			minimal[p] = part
			patterns = append(patterns, part, transform.ReverseComplement(part))
			patternPrimer = append(patternPrimer, p, p)
			patternIsReverse = append(patternIsReverse, false, true)
		}
	}

	// GPU pass 2: every occurrence of every pattern in every template (the suffix-array lookups of
	// pcr.go:110,113), then ordered the way the reference fills its maps: by primer, forward first.
	var hits []polyb200.Site
	if len(patterns) > 0 {
		tFlat, tBounds := polyb200.Flatten(templates)
		pFlat, pBounds := polyb200.Flatten(patterns)
		var err error
		if hits, err = polyb200.FindSites(tFlat, tBounds, pFlat, pBounds); err != nil {
			panic(err)
		}
		sort.Slice(hits, func(a, b int) bool {
			x, y := hits[a], hits[b]
			if x.Seq != y.Seq {
				return x.Seq < y.Seq
			}
			if x.Pattern != y.Pattern {
				return x.Pattern < y.Pattern
			}
			return x.Pos < y.Pos
		})
	}

	var fragments []string
	cursor := 0
	for t, template := range templates {
		fwd, rev := newSiteIndex(), newSiteIndex()
		for ; cursor < len(hits) && hits[cursor].Seq == t; cursor++ {
			h := hits[cursor]
			if patternIsReverse[h.Pattern] {
				rev.add(h.Pos, patternPrimer[h.Pattern])
			} else {
				fwd.add(h.Pos, patternPrimer[h.Pattern])
			}
		}
		sort.Ints(fwd.positions)
		sort.Ints(rev.positions)
		// amplicons of one (forward site, reverse site) pair: every forward primer x every reverse primer
		emit := func(text string, from, to, fwdPos, revPos int) {
			for _, fp := range fwd.primersAt[fwdPos] {
				overhang := primerList[fp][:len(primerList[fp])-len(minimal[fp])]
				for _, rp := range rev.primersAt[revPos] {
					fragments = append(fragments, overhang+text[from:to]+transform.ReverseComplement(primerList[rp]))
				}
			}
		}
		for i, f := range fwd.positions {
			firstAfter := sort.SearchInts(rev.positions, f+1) // reverse sites strictly right of f
			if i+1 < len(fwd.positions) {
				// not the last forward site: only the first reverse site before the next forward site
				if firstAfter < len(rev.positions) && rev.positions[firstAfter] < fwd.positions[i+1] {
					r := rev.positions[firstAfter]
					emit(template, f, r, f, r)
				}
				continue
			}
			for _, r := range rev.positions[firstAfter:] { // last forward site: every reverse site to its right
				emit(template, f, r, f, r)
			}
			if circular && firstAfter == len(rev.positions) {
				// nothing to the right: on a circular template look across the origin
				rotated := template[f:] + template[:f]
				for _, r := range rev.positions[:sort.SearchInts(rev.positions, fwd.positions[0])] {
					emit(rotated, 0, len(template)-f+r, f, r)
				}
			}
		}
	}
	return fragments
}

// Simulate: reference pcr.go:171-186 -- SimulateSimple twice, the second time with the products
// added to the primers; a different number of products means concatemerization.
func Simulate(sequences []string, targetTm float64, circular bool, primerList []string) ([]string, error) {
	for _, primer := range primerList {
		if len(primer) < minimalPrimerLength {
			return nil, errors.New("Primers are too short.")
		}
	}
	first := SimulateSimple(sequences, targetTm, circular, primerList)
	second := SimulateSimple(sequences, targetTm, circular, append(primerList, first...))
	if len(first) != len(second) {
		return first, errors.New("Concatemerization detected in PCR.")
	}
	return first, nil
}
