// Package fasta is the H100-backed drop-in for bebop/poly's io/fasta parser entry points
// (io/fasta/fasta.go:66-77,89-99): same exported names and results, the parsing itself runs on
// the GPU through libpolyb200.so (pg_fasta_ingest).  The writer half of the reference package
// (Build / Write) and the channel-based ParseConcurrent are untouched pure Go and stay as they are.
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image); see INTEGRATION.md.
package fasta

import (
	"errors"
	"fmt"
	"io"

	"github.com/bebop/poly/internal/polyb200"
)

// Fasta: one record, the header line without '>' and the concatenated sequence lines (reference: fasta.go:66-69).
type Fasta struct {
	Name     string `json:"name"`
	Sequence string `json:"sequence"`
}

// BufioAlias selects bit-for-bit reference behaviour (true, the default): the reference uses the
// slice returned by bufio.Reader.ReadSlice after a Peek, so a line that ends exactly at the end of
// a full reader buffer is seen with bytes from one buffer further on.  Set it to false to take
// every line as written.
var BufioAlias = true

var errBufferFull = errors.New("bufio: buffer full")

// Parse reads r to the end and returns what the reference's Parse returns for the same bytes (fasta.go:72-77).
func Parse(r io.Reader) ([]Fasta, error) {
	const maxLineSize = 2 * 32 * 1024
	return parseAll(r, maxLineSize)
}

// ParseAllSize is NewParser(r, maxLineSize).ParseAll() of the reference in one call.
func ParseAllSize(r io.Reader, maxLineSize int) ([]Fasta, error) { return parseAll(r, maxLineSize) }

func parseAll(r io.Reader, maxLineSize int) ([]Fasta, error) {
	text, err := io.ReadAll(r)
	if err != nil {
		return nil, err
	}
	seq, seqOff, names, nameOff, code, line, err := polyb200.FastaIngest(text, maxLineSize, BufioAlias)
	if err != nil {
		return nil, err
	}
	fastas := make([]Fasta, len(seqOff)-1)
	for i := range fastas {
		fastas[i] = Fasta{Name: string(names[nameOff[i]:nameOff[i+1]]), Sequence: string(seq[seqOff[i]:seqOff[i+1]])}
	}
	switch code {
	case 1:
		return fastas, fmt.Errorf("did not find fasta start '>', got to line %d", line)
	case 2: // the reference's message also quotes the name of the empty record; it is not carried across the ABI
		return fastas, fmt.Errorf("empty fasta sequence, got to line %d", line)
	case 3:
		return fastas, fmt.Errorf("line %d too large for buffer, use larger maxLineSize: %w", line, errBufferFull)
	case 4:
		return fastas, errBufferFull
	}
	return fastas, nil
}
