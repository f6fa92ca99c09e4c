// Package align: drop-in for github.com/bebop/poly/search/align.SmithWaterman
// (search/align/align.go:171-232: score, aligned strings, error) and for the score of
// NeedlemanWunsch (align.go:100-134,166), backed by libpolyb200.so.  NOT COMPILED HERE.
// SmithWaterman / NeedlemanWunsch need the shorter string to have <= 64 symbols; longer pairs keep the
// pure-Go path.  The *Pair* functions take lists of pairs of strings of any length.
package align

import (
	"fmt"

	"github.com/bebop/poly/alphabet"
	"github.com/bebop/poly/internal/polyb200"
	"github.com/bebop/poly/search/align/matrix"
)

// Scoring mirrors align.Scoring (align.go:73-76).
type Scoring struct {
	SubstitutionMatrix *matrix.SubstitutionMatrix
	GapPenalty         int
}

// NewScoring mirrors align.NewScoring (align.go:79-87).
func NewScoring(substitutionMatrix *matrix.SubstitutionMatrix, gapPenalty int) (Scoring, error) {
	if substitutionMatrix == nil {
		substitutionMatrix = matrix.Default
	}
	return Scoring{SubstitutionMatrix: substitutionMatrix, GapPenalty: gapPenalty}, nil
}

// flatten turns the interface-keyed alphabets into byte LUTs + a dense table (host side, once per call).
func flatten(m *matrix.SubstitutionMatrix) (lutA, lutB [256]int16, table []int64, nA, nB int) {
	symA, symB := m.FirstAlphabet.Symbols(), m.SecondAlphabet.Symbols()
	nA, nB = len(symA), len(symB)
	for b := 0; b < 256; b++ {
		lutA[b], lutB[b] = -1, -1
		if c, err := m.FirstAlphabet.Encode(string(byte(b))); err == nil {
			lutA[b] = int16(c)
		}
		if c, err := m.SecondAlphabet.Encode(string(byte(b))); err == nil {
			lutB[b] = int16(c)
		}
	}
	table = make([]int64, nA*nB)
	for i := 0; i < nA; i++ {
		for j := 0; j < nB; j++ {
			v, _ := m.Score(symA[i], symB[j])
			table[i*nB+j] = int64(v)
		}
	}
	return
}

// SmithWatermanScores scores SmithWaterman(query, template, scoring) for every query in one GPU pass.
func SmithWatermanScores(queries []string, template string, scoring Scoring) ([]int, []error) {
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	bases, offsets := polyb200.Flatten(queries)
	score, ec, ep, err := polyb200.SWScoreBatch(bases, offsets, template, true, &lutA, &lutB, table, nA, nB, int64(scoring.GapPenalty))
	if err != nil {
		panic(err)
	}
	scores, errs := make([]int, len(queries)), make([]error, len(queries))
	for i := range queries {
		scores[i] = int(score[i])
		if ec[i] == 1 {
			_, errs[i] = scoring.SubstitutionMatrix.FirstAlphabet.Encode(string(queries[i][ep[i]]))
		} else if ec[i] == 2 {
			_, errs[i] = scoring.SubstitutionMatrix.SecondAlphabet.Encode(string(template[ep[i]]))
		}
	}
	return scores, errs
}

// SmithWatermanScore is the score (and error) of align.SmithWaterman(stringA, stringB, scoring).
func SmithWatermanScore(stringA, stringB string, scoring Scoring) (int, error) {
	s, e := SmithWatermanScores([]string{stringA}, stringB, scoring)
	if e[0] != nil {
		return 0, e[0]
	}
	return s[0], nil
}

// SmithWaterman keeps the reference signature (align.go:171): score, aligned strings, error.
// The shorter of the two strings must have <= 64 symbols (it rides in registers on the GPU);
// longer pairs should keep using the pure-Go implementation.
func SmithWaterman(stringA string, stringB string, scoring Scoring) (int, string, string, error) {
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	queryIsA := len(stringA) <= 64
	q, t := stringA, stringB
	if !queryIsA {
		q, t = stringB, stringA
	}
	bases, offsets := polyb200.Flatten([]string{q})
	score, ec, ep, alignA, alignB, err := polyb200.SWAlignBatch(bases, offsets, t, queryIsA, &lutA, &lutB, table, nA, nB,
		int64(scoring.GapPenalty), 2*len(q)+64)
	if err != nil {
		panic(err)
	}
	if ec[0] == 1 {
		_, e := scoring.SubstitutionMatrix.FirstAlphabet.Encode(string(stringA[ep[0]]))
		return 0, "", "", e
	} else if ec[0] == 2 {
		_, e := scoring.SubstitutionMatrix.SecondAlphabet.Encode(string(stringB[ep[0]]))
		return 0, "", "", e
	}
	return int(score[0]), alignA[0], alignB[0], nil
}

// NeedlemanWunsch keeps the reference signature (align.go:100): score, aligned strings, error.
func NeedlemanWunsch(stringA string, stringB string, scoring Scoring) (int, string, string, error) {
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	queryIsA := len(stringA) <= 64
	q, t := stringA, stringB
	if !queryIsA {
		q, t = stringB, stringA
	}
	bases, offsets := polyb200.Flatten([]string{q})
	score, ec, ep, alignA, alignB, err := polyb200.NWAlignBatch(bases, offsets, t, queryIsA, &lutA, &lutB, table, nA, nB,
		int64(scoring.GapPenalty), len(q)+len(t)+8)
	if err != nil {
		panic(err)
	}
	if ec[0] == 1 {
		_, e := scoring.SubstitutionMatrix.FirstAlphabet.Encode(string(stringA[ep[0]]))
		return 0, "", "", e
	} else if ec[0] == 2 {
		_, e := scoring.SubstitutionMatrix.SecondAlphabet.Encode(string(stringB[ep[0]]))
		return 0, "", "", e
	}
	return int(score[0]), alignA[0], alignB[0], nil
}

// NeedlemanWunschScore is the score of align.NeedlemanWunsch(stringA, stringB, scoring).
func NeedlemanWunschScore(stringA, stringB string, scoring Scoring) (int, error) {
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	bases, offsets := polyb200.Flatten([]string{stringA})
	score, ec, ep, err := polyb200.NWScoreBatch(bases, offsets, stringB, true, &lutA, &lutB, table, nA, nB, int64(scoring.GapPenalty))
	if err != nil {
		panic(err)
	}
	if ec[0] == 1 {
		_, e := scoring.SubstitutionMatrix.FirstAlphabet.Encode(string(stringA[ep[0]]))
		return 0, e
	} else if ec[0] == 2 {
		_, e := scoring.SubstitutionMatrix.SecondAlphabet.Encode(string(stringB[ep[0]]))
		return 0, e
	}
	return int(score[0]), nil
}

// pairIndices checks every pair against the two sets -- out of range panics, as indexing as[i] / bs[j]
// in the caller's loop would -- and converts the indices for the C ABI.
func pairIndices(as, bs []string, pairA, pairB []int) ([]uint32, []uint32) {
	if len(pairA) != len(pairB) {
		panic(fmt.Sprintf("align: %d pairA indices but %d pairB indices", len(pairA), len(pairB)))
	}
	pa, pb := make([]uint32, len(pairA)), make([]uint32, len(pairB))
	for p := range pairA {
		_, _ = as[pairA[p]], bs[pairB[p]]
		pa[p], pb[p] = uint32(pairA[p]), uint32(pairB[p])
	}
	return pa, pb
}

// pairError rebuilds the reference's *alphabet.Error of a pair from its error code and position.
func pairError(scoring Scoring, ec int32, ep int64, a, b string) error {
	var e error
	if ec == 1 {
		_, e = scoring.SubstitutionMatrix.FirstAlphabet.Encode(string(a[ep]))
	} else if ec == 2 {
		_, e = scoring.SubstitutionMatrix.SecondAlphabet.Encode(string(b[ep]))
	}
	return e
}

func pairScores(global bool, as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []error) {
	pa, pb := pairIndices(as, bs, pairA, pairB)
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	aBases, aOff := polyb200.Flatten(as)
	bBases, bOff := polyb200.Flatten(bs)
	score, ec, ep, err := polyb200.ScorePairs(global, aBases, aOff, bBases, bOff, pa, pb, &lutA, &lutB, table, nA, nB, int64(scoring.GapPenalty))
	if err != nil {
		panic(err)
	}
	scores, errs := make([]int, len(pa)), make([]error, len(pa))
	for p := range pa {
		scores[p] = int(score[p])
		errs[p] = pairError(scoring, ec[p], ep[p], as[pairA[p]], bs[pairB[p]])
	}
	return scores, errs
}

// SmithWatermanPairScores scores SmithWaterman(as[pairA[p]], bs[pairB[p]], scoring) for every pair p in one
// GPU pass, with each pair's error as SmithWaterman returns it.  A string may have any length.
func SmithWatermanPairScores(as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []error) {
	return pairScores(false, as, bs, pairA, pairB, scoring)
}

// NeedlemanWunschPairScores scores NeedlemanWunsch(as[pairA[p]], bs[pairB[p]], scoring) for every pair p.
func NeedlemanWunschPairScores(as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []error) {
	return pairScores(true, as, bs, pairA, pairB, scoring)
}

func pairAligns(global bool, as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []string, []string, []error) {
	pa, pb := pairIndices(as, bs, pairA, pairB)
	lutA, lutB, table, nA, nB := flatten(scoring.SubstitutionMatrix)
	aBases, aOff := polyb200.Flatten(as)
	bBases, bOff := polyb200.Flatten(bs)
	score, ec, ep, alignA, alignB, err := polyb200.AlignPairs(global, aBases, aOff, bBases, bOff, pa, pb, &lutA, &lutB, table, nA, nB,
		int64(scoring.GapPenalty))
	if err != nil {
		panic(err)
	}
	scores, errs := make([]int, len(pa)), make([]error, len(pa))
	for p := range pa {
		if errs[p] = pairError(scoring, ec[p], ep[p], as[pairA[p]], bs[pairB[p]]); errs[p] != nil {
			alignA[p], alignB[p] = "", "" // (0, "", "", err), as the reference returns
			continue
		}
		scores[p] = int(score[p])
	}
	return scores, alignA, alignB, errs
}

// SmithWatermanPairAligns is SmithWaterman(as[pairA[p]], bs[pairB[p]], scoring) for every pair p: scores,
// aligned strings and errors, in one call.
func SmithWatermanPairAligns(as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []string, []string, []error) {
	return pairAligns(false, as, bs, pairA, pairB, scoring)
}

// NeedlemanWunschPairAligns is NeedlemanWunsch(as[pairA[p]], bs[pairB[p]], scoring) for every pair p.
func NeedlemanWunschPairAligns(as, bs []string, pairA, pairB []int, scoring Scoring) ([]int, []string, []string, []error) {
	return pairAligns(true, as, bs, pairA, pairB, scoring)
}

var _ = alphabet.DNA
var _ = fmt.Sprintf
