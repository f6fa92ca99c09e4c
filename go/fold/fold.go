// Package fold is the drop-in for github.com/bebop/poly/fold backed by libpolyb200.so: same exported names
// and results (fold/fold.go and fold/seqfold.go of the reference), plus ZukerBatch, which folds many
// sequences in one GPU call.  The fold runs in the library's CUDA kernel.  A sequence with a byte >= 0x80 or
// longer than MaxLen nt returns ErrUnsupported.  NOT COMPILED HERE (no Go toolchain in the build image).
package fold

import (
	"errors"
	"fmt"
	"math"
	"strings"

	"github.com/bebop/poly/internal/polyb200"
)

// MaxLen is the longest sequence the library folds (PG_FOLD_MAX_LEN).
const MaxLen = 1024

// ErrUnsupported is returned for a sequence with a byte >= 0x80 (strings.ToUpper would re-encode it) or
// longer than MaxLen nt.
var ErrUnsupported = errors.New("fold: unsupported sequence (a byte >= 0x80, or longer than 1024 nt)")

// ErrInternal is returned where one of the reference's internal errors fired.
var ErrInternal = errors.New("fold: an internal error of the reference fired on this sequence")

// Result holds the resulting structure of a folded sequence (seqfold.go:195-197).
type Result struct {
	valid      bool
	mfe        float64
	dotBracket string
}

// DotBracket returns the dot-bracket notation of the structure (seqfold.go:205-230).
func (r Result) DotBracket() string {
	if !r.valid {
		return ""
	}
	return r.dotBracket
}

// MinimumFreeEnergy returns the delta G of the structure (seqfold.go:236-247).
func (r Result) MinimumFreeEnergy() float64 {
	if !r.valid {
		return math.Inf(1)
	}
	return r.mfe
}

// ZukerBatch folds every sequence at temp degrees Celsius in one GPU call: results[i] and errs[i] are what
// Zuker(seqs[i], temp) returns.  Where the reference panics (an empty or 1-nt sequence, a traceback index
// out of range), ZukerBatch panics as well, after the whole batch has been folded.
func ZukerBatch(seqs []string, temp float64) (results []Result, errs []error, err error) {
	results, errs = make([]Result, len(seqs)), make([]error, len(seqs))
	if len(seqs) == 0 {
		return results, errs, nil
	}
	bases, offsets := polyb200.Flatten(seqs)
	mfe, db, status, err := polyb200.FoldZukerBatch(bases, offsets, temp)
	if err != nil {
		return nil, nil, err
	}
	panicked := false
	for i := range seqs {
		switch status[i] {
		case 0:
			results[i] = Result{valid: true, mfe: mfe[i], dotBracket: db[i]}
		case 3:
			errs[i] = fmt.Errorf("error creating folding context: the sequence %s is not RNA or DNA", strings.ToUpper(seqs[i]))
		case 1:
			panicked = true
		case 2:
			errs[i] = ErrUnsupported
		default:
			errs[i] = ErrInternal
		}
	}
	if panicked {
		panic("runtime error: index out of range")
	}
	return results, errs, nil
}

// Zuker folds seq at temp degrees Celsius and returns its minimum free energy structure (fold.go:56-67).
func Zuker(seq string, temp float64) (Result, error) {
	results, errs, err := ZukerBatch([]string{seq}, temp)
	if err != nil {
		return Result{}, err
	}
	return results[0], errs[0]
}
