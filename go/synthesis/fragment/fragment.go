// Package fragment is the drop-in for github.com/bebop/poly/synthesis/fragment backed by libpolyb200.so: same
// exported names and results (synthesis/fragment/fragment.go of the reference), plus FragmentBatch,
// FragmentWithOverhangsBatch, SetEfficiencyBatch and NextOverhangsBatch, which run many genes or sets in one GPU
// call.  The overhang choice runs in the library's CUDA kernel.  A sequence with a byte >= 0x80 returns
// ErrUnsupported; where the reference panics (fewer than 4 bytes) so does the mirror.  NOT COMPILED HERE (no Go
// toolchain in the build image).
package fragment

import (
	"errors"
	"fmt"
	"strings"

	"github.com/bebop/poly/internal/polyb200"
)

// ErrUnsupported is returned for a sequence with a byte >= 0x80 (strings.ToUpper would re-encode it).
var ErrUnsupported = errors.New("fragment: unsupported sequence (a byte >= 0x80)")

// Result is what Fragment returns for one sequence.
type Result struct {
	Fragments  []string
	Efficiency float64
	Err        error
}

// FragmentWithOverhangsBatch runs FragmentWithOverhangs on every sequence in one GPU call; the exclude and
// include lists are shared by the batch.  Where the reference panics, it panics as well, after the whole
// batch has run.
func FragmentWithOverhangsBatch(sequences []string, minFragmentSize int, maxFragmentSize int, excludeOverhangs []string,
	includeOverhangs []string) ([]Result, error) {
	out := make([]Result, len(sequences))
	if len(sequences) == 0 {
		return out, nil
	}
	status, eff, errMin, errMax, ends, err := polyb200.FragmentBatch(sequences, minFragmentSize, maxFragmentSize, excludeOverhangs, includeOverhangs)
	if err != nil {
		return nil, err
	}
	panicked := false
	for i, s := range sequences {
		switch status[i] {
		case 0:
			up := strings.ToUpper(s)
			frags := make([]string, len(ends[i]))
			for j, e := range ends[i] {
				start := uint64(0)
				if j > 0 {
					start = ends[i][j-1] - 4
				}
				frags[j] = up[start:e]
			}
			out[i] = Result{Fragments: frags, Efficiency: eff[i]}
		case 5:
			out[i] = Result{Fragments: []string{}, Err: fmt.Errorf("minFragmentSize (%d) larger than maxFragmentSize (%d)", errMin[i], errMax[i])}
		case 6:
			out[i] = Result{Fragments: []string{}, Err: fmt.Errorf("minFragmentSize must be equal to or greater than 12 . Got size of %d", errMin[i])}
		case 7:
			out[i] = Result{Fragments: []string{}, Err: errors.New("bestOverhangPosition failed by equaling zero")}
		case 1:
			panicked = true
		default:
			out[i] = Result{Err: ErrUnsupported}
		}
	}
	if panicked {
		panic("runtime error: slice bounds out of range")
	}
	return out, nil
}

// FragmentBatch runs Fragment on every sequence in one GPU call.
func FragmentBatch(sequences []string, minFragmentSize int, maxFragmentSize int, excludeOverhangs []string) ([]Result, error) {
	return FragmentWithOverhangsBatch(sequences, minFragmentSize, maxFragmentSize, excludeOverhangs, nil)
}

// Fragment fragments a sequence into fragments between the min and max size, choosing fragment ends for
// optimal assembly efficiency (fragment.go:191-194).
func Fragment(sequence string, minFragmentSize int, maxFragmentSize int, excludeOverhangs []string) ([]string, float64, error) {
	r, err := FragmentBatch([]string{sequence}, minFragmentSize, maxFragmentSize, excludeOverhangs)
	if err != nil {
		return []string{}, 0, err
	}
	return r[0].Fragments, r[0].Efficiency, r[0].Err
}

// FragmentWithOverhangs fragments a sequence with only a certain overhang set (fragment.go:199-202).
func FragmentWithOverhangs(sequence string, minFragmentSize int, maxFragmentSize int, excludeOverhangs []string,
	includeOverhangs []string) ([]string, float64, error) {
	r, err := FragmentWithOverhangsBatch([]string{sequence}, minFragmentSize, maxFragmentSize, excludeOverhangs, includeOverhangs)
	if err != nil {
		return []string{}, 0, err
	}
	return r[0].Fragments, r[0].Efficiency, r[0].Err
}

// SetEfficiencyBatch gets SetEfficiency of every set in one GPU call.
func SetEfficiencyBatch(sets [][]string) ([]float64, error) {
	return polyb200.FragmentSetEfficiencyBatch(sets)
}

// SetEfficiency gets the estimated fidelity rate of a given set of GoldenGate overhangs (fragment.go:24-38).
// It panics if the library call fails, as the reference has no error to return.
func SetEfficiency(overhangs []string) float64 {
	eff, err := SetEfficiencyBatch([][]string{overhangs})
	if err != nil {
		panic(err)
	}
	return eff[0]
}

// NextOverhangsBatch gets NextOverhangs of every set in one GPU call.
func NextOverhangsBatch(sets [][]string) ([][]string, [][]float64, error) {
	return polyb200.FragmentNextOverhangsBatch(sets)
}

// NextOverhangs gets a list of possible next overhangs to use for an overhang list, along with their
// efficiencies (fragment.go:43-79).  It panics if the library call fails.
func NextOverhangs(currentOverhangs []string) ([]string, []float64) {
	cands, effs, err := NextOverhangsBatch([][]string{currentOverhangs})
	if err != nil {
		panic(err)
	}
	return cands[0], effs[0]
}

// NextOverhang gets next most efficient overhang to use for a given set of overhangs (fragment.go:85-98).
func NextOverhang(currentOverhangs []string) string {
	overhangsToTest, efficiencies := NextOverhangs(currentOverhangs)
	var newOverhang string
	maxEfficiency := float64(0)
	for i, overhang := range overhangsToTest {
		if efficiencies[i] > maxEfficiency {
			maxEfficiency = efficiencies[i]
			newOverhang = overhang
		}
	}
	return newOverhang
}
