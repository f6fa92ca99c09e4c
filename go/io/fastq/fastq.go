// Package fastq is the H100-backed drop-in for the record parser of bebop/poly's io/fastq
// (io/fastq/fastq.go:46-99,117-214): Parse returns the same []Fastq and the same error for the same
// bytes.  The line index, the reference's per-record checks (in its order) and the dense copy of the
// sequences run on the GPU (pg_fastq_ingest_records); Identifier, Optionals and Quality are cut out of
// the caller's text with the line spans the kernel reports.
// NOT COMPILED IN THIS REPOSITORY (no Go toolchain in the build image); see INTEGRATION.md.
package fastq

import (
	"errors"
	"fmt"
	"io"
	"strings"

	"github.com/bebop/poly/internal/polyb200"
)

// Fastq: reference fastq.go:46-51.
type Fastq struct {
	Identifier string            `json:"identifier"`
	Optionals  map[string]string `json:"optionals"`
	Sequence   string            `json:"sequence"`
	Quality    string            `json:"quality"`
}

// Parse: reference fastq.go:54-59 (NewParser(r, 64 KiB).ParseAll()).
func Parse(r io.Reader) ([]Fastq, error) {
	text, err := io.ReadAll(r)
	if err != nil {
		return nil, err
	}
	bases, offsets, spans, code, line, err := polyb200.FastqIngestRecords(text)
	if err != nil {
		return nil, err
	}
	records := make([]Fastq, len(offsets)-1)
	for i := range records {
		idLine := string(text[spans[4*i] : spans[4*i]+spans[4*i+1]])
		tokens := strings.Split(idLine, " ") // fastq.go:157
		optionals := make(map[string]string)
		for _, datum := range tokens[1:] { // every datum holds '=': the kernel reported a panic otherwise
			kv := strings.Split(datum, "=")
			optionals[kv[0]] = kv[1]
		}
		records[i] = Fastq{
			Identifier: tokens[0][1:],
			Optionals:  optionals,
			Sequence:   string(bases[offsets[i]:offsets[i+1]]),
			Quality:    string(text[spans[4*i+2] : spans[4*i+2]+spans[4*i+3]]),
		}
	}
	return records, parseError(code, line, records)
}

// the reference's error values (fastq.go:124-133,180,198,204) for the codes of pg_fastq_ingest
func parseError(code int32, line uint64, parsed []Fastq) error {
	switch code {
	case 0:
		return nil
	case 1:
		return fmt.Errorf("line %d failed: unexepcted EOF encountered", line)
	case 2:
		return fmt.Errorf("empty fastq sequence for %q,  got to line %d: %w", "", line, error(nil))
	case 3:
		return fmt.Errorf("empty quality sequence for %q,  got to line %d: %w", "", line, error(nil))
	case 4:
		return fmt.Errorf("did not find fastq start '@', got to line %d: %w", line, error(nil))
	case 5:
		panic("runtime error: index out of range") // empty identifier line or an optional without '=' (fastq.go:155,163)
	case 6:
		return fmt.Errorf("line %d too large for buffer, use larger maxLineSize: %w", line, errors.New("bufio: buffer full"))
	}
	return fmt.Errorf("fastq: unknown error code %d at line %d", code, line)
}
