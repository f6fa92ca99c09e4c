// Package seqhash is the drop-in for github.com/bebop/poly/seqhash backed by libpolyb200.so: same
// exported names and results (seqhash/seqhash.go:64-223 of the reference), plus HashBatch, which hashes
// many sequences of one type and shape in one GPU call.  NOT COMPILED HERE (no Go toolchain in the
// build image).
package seqhash

import (
	"encoding/hex"
	"errors"
	"fmt"

	"github.com/bebop/poly/internal/polyb200"
)

// SequenceType is the type of sequence a Seqhash describes (seqhash.go:62).
type SequenceType string

const (
	DNA     SequenceType = "DNA"
	RNA     SequenceType = "RNA"
	PROTEIN SequenceType = "PROTEIN"
)

// ErrUnsupported is returned for a sequence in which a byte >= 0x80 comes before any letter outside the
// alphabet: strings.ToUpper would re-encode it, and the library does not guess at the result.
var ErrUnsupported = errors.New("seqhash: non-ASCII byte (unsupported)")

// Result is one sequence's Seqhash or error.
type Result struct {
	Seqhash string
	Err     error
}

// HashBatch is Hash of every sequence, in one call to the GPU.
func HashBatch(sequences []string, sequenceType SequenceType, circular bool, doubleStranded bool) ([]Result, error) {
	out := make([]Result, len(sequences))
	var t int32
	switch sequenceType {
	case DNA:
		t = 0
	case RNA:
		t = 1
	case PROTEIN:
		t = 2
	default:
		for i := range out {
			out[i].Err = errors.New("Only sequenceTypes of DNA, RNA, or PROTEIN allowed. Got sequenceType: " + string(sequenceType))
		}
		return out, nil
	}
	if len(sequences) == 0 {
		return out, nil
	}
	offsets := make([]uint64, len(sequences)+1)
	total := 0
	for i, s := range sequences {
		total += len(s)
		offsets[i+1] = uint64(total)
	}
	bases := make([]byte, 0, total)
	for _, s := range sequences {
		bases = append(bases, s...)
	}
	var flags uint32
	if circular {
		flags |= 1
	}
	if doubleStranded {
		flags |= 2
	}
	digest, code, pos, err := polyb200.SeqhashBatch(bases, offsets, t, flags)
	if err != nil {
		return nil, err
	}
	meta := string(sequenceType[0])
	if circular {
		meta += "C"
	} else {
		meta += "L"
	}
	if doubleStranded {
		meta += "D"
	} else {
		meta += "S"
	}
	for i := range sequences {
		switch code[i] {
		case 0:
			out[i].Seqhash = "v1_" + meta + "_" + hex.EncodeToString(digest[32*i:32*i+32])
		case 1:
			c := sequences[i][pos[i]]
			if c >= 'a' && c <= 'z' {
				c -= 'a' - 'A'
			}
			if t == 2 {
				out[i].Err = errors.New("Only letters ACDEFGHIKLMNPQRSTVWYUO*BXZ are allowed for Proteins. Got letter: " + string(c))
			} else {
				out[i].Err = errors.New("Only letters ATUGCYRSWKMBDHVNZ are allowed for DNA/RNA. Got letter: " + string(c))
			}
		case 2:
			out[i].Err = errors.New("Proteins cannot be double stranded")
		default:
			out[i].Err = fmt.Errorf("%w at byte %d", ErrUnsupported, pos[i])
		}
	}
	return out, nil
}

// Hash is a function to create Seqhashes, a specific kind of identifier (seqhash.go:141-223).
func Hash(sequence string, sequenceType SequenceType, circular bool, doubleStranded bool) (string, error) {
	res, err := HashBatch([]string{sequence}, sequenceType, circular, doubleStranded)
	if err != nil {
		return "", err
	}
	return res[0].Seqhash, res[0].Err
}

// RotateSequence rotates circular sequences to deterministic point (seqhash.go:127-138).
func RotateSequence(sequence string) string {
	rot, err := polyb200.LeastRotationBatch([]byte(sequence), []uint64{0, uint64(len(sequence))})
	if err != nil {
		panic(err)
	}
	r := rot[0]
	return sequence[r:] + sequence[:r]
}
