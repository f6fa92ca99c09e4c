// Package clone is the drop-in for github.com/bebop/poly/clone backed by libpolyb200.so: same exported
// names and results (clone/clone.go of the reference), plus CutWithEnzymeBatch and GoldenGateBatch, which
// run many digests or reactions in one GPU call.  The digest runs in CUDA kernels; the ligation recursion
// runs once, in the library's host code, and every construct it closes is built and seqhashed on the
// device.  Enzyme patterns must be literals (the GPU does not implement Go's regexp language): Enzyme
// keeps them as strings.  NOT COMPILED HERE (no Go toolchain in the build image).
package clone

import (
	"errors"
	"math"
	"strings"

	"github.com/bebop/poly/internal/polyb200"
)

// Part is a circular or linear DNA sequence (clone.go:56-59).
type Part struct {
	Sequence string
	Circular bool
}

// Fragment is a linear sequence with sticky ends (clone.go:70-74).
type Fragment struct {
	Sequence        string
	ForwardOverhang string
	ReverseOverhang string
}

// Enzyme is a restriction enzyme (clone.go:77-84); RegexpFor and RegexpRev are literal patterns.
type Enzyme struct {
	Name            string
	RegexpFor       string
	RegexpRev       string
	Skip            int
	OverheadLength  int
	RecognitionSite string
}

// ErrUnsupported is returned for a non-literal pattern, a Skip or OverheadLength outside int32, or a part or
// fragment with a byte >= 0x80 (strings.ToUpper would re-encode it).  It is the error the library wrappers return for PG_ERR_UNSUPPORTED.
var ErrUnsupported = polyb200.ErrCloneUnsupported

func (e Enzyme) lib() (polyb200.CloneEnzyme, error) {
	for _, p := range []string{e.RegexpFor, e.RegexpRev} {
		if p == "" || len(p) > 32 || strings.ContainsAny(p, "\\.+*?()|[]{}^$\x00") || strings.IndexFunc(p, func(r rune) bool { return r >= 0x80 }) >= 0 {
			return polyb200.CloneEnzyme{}, ErrUnsupported
		}
	}
	// pg_clone_enzyme holds Skip and OverheadLength as int32: a wider value would wrap
	for _, v := range []int{e.Skip, e.OverheadLength} {
		if v < math.MinInt32 || v > math.MaxInt32 {
			return polyb200.CloneEnzyme{}, ErrUnsupported
		}
	}
	return polyb200.CloneEnzyme{ForwardSite: e.RegexpFor, ReverseSite: e.RegexpRev, RecognitionSite: e.RecognitionSite, Skip: e.Skip,
		OverheadLength: e.OverheadLength}, nil
}

// EnzymeManager holds enzymes by name (clone.go:88-107).
type EnzymeManager struct {
	enzymeMap map[string]Enzyme
}

// NewEnzymeManager creates a new EnzymeManager given some enzymes.
func NewEnzymeManager(enzymes []Enzyme) EnzymeManager {
	m := make(map[string]Enzyme)
	for _, e := range enzymes {
		m[e.Name] = e
	}
	return EnzymeManager{enzymeMap: m}
}

// GetEnzymeByName gets the enzyme by its name (clone.go:130-135).
func (enzymeManager EnzymeManager) GetEnzymeByName(name string) (Enzyme, error) {
	if enzyme, ok := enzymeManager.enzymeMap[name]; ok {
		return enzyme, nil
	}
	return Enzyme{}, errors.New("Enzyme " + name + " not found")
}

// CutWithEnzymeByName cuts a part with the enzyme of that name (clone.go:116-127).
func (enzymeManager EnzymeManager) CutWithEnzymeByName(part Part, directional bool, name string) ([]Fragment, error) {
	enzyme, err := enzymeManager.GetEnzymeByName(name)
	if err != nil {
		return []Fragment{}, err
	}
	return CutWithEnzyme(part, directional, enzyme), nil
}

// CutWithEnzymeBatch is CutWithEnzyme of every part x enzyme in one call: out[p][e].  A panic of the
// reference on any item panics here too; ErrUnsupported is returned for unsupported input.
func CutWithEnzymeBatch(parts []Part, directional bool, enzymes []Enzyme) ([][][]Fragment, error) {
	lib := make([]polyb200.CloneEnzyme, len(enzymes))
	for i, e := range enzymes {
		var err error
		if lib[i], err = e.lib(); err != nil {
			return nil, err
		}
	}
	seqs := make([]string, len(parts))
	circ := make([]bool, len(parts))
	for i, p := range parts {
		seqs[i], circ[i] = p.Sequence, p.Circular
	}
	out := make([][][]Fragment, len(parts))
	if len(parts) == 0 || len(enzymes) == 0 {
		return out, nil
	}
	bases, offsets := polyb200.Flatten(seqs)
	r, err := polyb200.CloneDigest(bases, offsets, circ, lib, directional)
	if err == polyb200.ErrPanic {
		panic("runtime error: slice bounds out of range")
	}
	if err != nil {
		return nil, err
	}
	f := 0
	for p := range parts {
		out[p] = make([][]Fragment, len(enzymes))
		for e := range enzymes {
			i := p*len(enzymes) + e
			for k := uint32(0); k < r.Count[i]; k++ {
				out[p][e] = append(out[p][e], Fragment{string(r.Seq[r.SeqOff[f]:r.SeqOff[f+1]]), string(r.OH[r.OHOff[2*f]:r.OHOff[2*f+1]]),
					string(r.OH[r.OHOff[2*f+1]:r.OHOff[2*f+2]])})
				f++
			}
		}
	}
	return out, nil
}

// CutWithEnzyme cuts a part with an enzyme (clone.go:138-268).
func CutWithEnzyme(part Part, directional bool, enzyme Enzyme) []Fragment {
	out, err := CutWithEnzymeBatch([]Part{part}, directional, []Enzyme{enzyme})
	if err != nil {
		panic(err)
	}
	return out[0][0]
}

// Constructs is one reaction's result: closed clones and looping constructs, in the reference's order.
type Constructs struct {
	Clones, Loops []string
}

func split(r *polyb200.CloneConstructs, nReactions int) []Constructs {
	out := make([]Constructs, nReactions)
	k := 0
	for i := 0; i < nReactions; i++ {
		for j := uint64(0); j < r.Counts[2*i]+r.Counts[2*i+1]; j++ {
			s := string(r.Bytes[r.Off[k]:r.Off[k+1]])
			if r.Kind[k] == 0 {
				out[i].Clones = append(out[i].Clones, s)
			} else {
				out[i].Loops = append(out[i].Loops, s)
			}
			k++
		}
	}
	return out
}

// GoldenGateBatch is GoldenGate of every reaction in one call.
func GoldenGateBatch(reactions [][]Part, cuttingEnzyme Enzyme) ([]Constructs, error) {
	enz, err := cuttingEnzyme.lib()
	if err != nil {
		return nil, err
	}
	var seqs []string
	var circ []bool
	roff := []uint64{0}
	for _, r := range reactions {
		for _, p := range r {
			seqs, circ = append(seqs, p.Sequence), append(circ, p.Circular)
		}
		roff = append(roff, uint64(len(seqs)))
	}
	bases, offsets := polyb200.Flatten(seqs)
	r, err := polyb200.CloneGoldenGate(bases, offsets, circ, roff, enz)
	if err == polyb200.ErrPanic {
		panic("runtime error: slice bounds out of range")
	}
	if err != nil {
		return nil, err
	}
	return split(r, len(reactions)), nil
}

// GoldenGate simulates a GoldenGate cloning reaction (clone.go:342-355).
func GoldenGate(sequences []Part, cuttingEnzyme Enzyme) (openConstructs []string, infiniteLoops []string) {
	out, err := GoldenGateBatch([][]Part{sequences}, cuttingEnzyme)
	if err != nil {
		panic(err)
	}
	return out[0].Clones, out[0].Loops
}

// CircularLigate simulates ligation of all possible fragment combinations into circular plasmids (clone.go:326-338).
func CircularLigate(fragments []Fragment) ([]string, []string) {
	var seqs, ohs []string
	for _, f := range fragments {
		seqs = append(seqs, f.Sequence)
		ohs = append(ohs, f.ForwardOverhang, f.ReverseOverhang)
	}
	sb, so := polyb200.Flatten(seqs)
	ob, oo := polyb200.Flatten(ohs)
	r, err := polyb200.CloneCircularLigate(sb, so, ob, oo, []uint64{0, uint64(len(fragments))})
	if err != nil {
		panic(err)
	}
	out := split(r, 1)
	return out[0].Clones, out[0].Loops
}

// GetBaseRestrictionEnzymes returns the common Golden Gate enzymes (clone.go:358-364).
func GetBaseRestrictionEnzymes() []Enzyme {
	return []Enzyme{
		{"BsaI", "GGTCTC", "GAGACC", 1, 4, "GGTCTC"},
		{"BbsI", "GAAGAC", "GTCTTC", 2, 4, "GAAGAC"},
		{"BtgZI", "GCGATG", "CATCGC", 10, 4, "GCGATG"},
	}
}
