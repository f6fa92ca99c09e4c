"""Regenerates tests/golden/seqhash_goldens.json and tests/golden/seqhash/puc19.txt.

Run with the `blake3` package importable and POLY_REFERENCE set to a bebop/poly checkout (for data/puc19.gbk):
    POLY_REFERENCE=/path/to/poly python tests/golden/make_seqhash_goldens.py
The BLAKE3 digests come from the `blake3` package, an implementation independent of
oracle/seqhash_oracle.c and of the CUDA kernels; the Seqhashes of the random sequences are a short
restatement of seqhash.Hash (seqhash.go:141-223) on top of it.  Tests read only the JSON.
"""
import json
import os
import random
import re

import blake3

HERE = os.path.dirname(os.path.abspath(__file__))

# seqhash_test.go:36-64, example_test.go:19,30
PINS = [
    ["TTAGCCCAT", "DNA", True, True, "v1_DCD_a376845b679740014f3eb501429b45e592ecc32a6ba8ba922cbe99217f6e9287"],
    ["TTAGCCCAT", "DNA", True, False, "v1_DCS_ef79b6e62394e22a176942dfc6a5e62eeef7b5281ffcb2686ecde208ec836ba4"],
    ["TTAGCCCAT", "DNA", False, True, "v1_DLD_c2c9fc44df72035082a152e94b04492182331bc3be2f62729d203e072211bdbf"],
    ["TTAGCCCAT", "DNA", False, False, "v1_DLS_063ea37d1154351639f9a48546bdae62fd8a3c18f3d3d3061060c9a55352d967"],
    ["TTAGCCCAT", "RNA", False, False, "v1_RLS_063ea37d1154351639f9a48546bdae62fd8a3c18f3d3d3061060c9a55352d967"],
    ["MGC*", "PROTEIN", False, False, "v1_PLS_922ec11f5227ce77a42f07f565a7a1a479772b5cf3f1f6e93afc5ecbc0fd5955"],
    ["ATGC", "DNA", False, True, "v1_DLD_f4028f93e08c5c23cbb8daa189b0a9802b378f1a1c919dcbcf1608a615f46350"],
]
# seqhash_test.go:14-33: each call must fail; the message is the reference's
ERRORS = [
    ["ATGGGCTAA", "TNA", True, True, "Only sequenceTypes of DNA, RNA, or PROTEIN allowed. Got sequenceType: TNA"],
    ["XTGGCCTAA", "DNA", True, True, "Only letters ATUGCYRSWKMBDHVNZ are allowed for DNA/RNA. Got letter: X"],
    ["MGCJ*", "PROTEIN", False, False, "Only letters ACDEFGHIKLMNPQRSTVWYUO*BXZ are allowed for Proteins. Got letter: J"],
    ["MGCS*", "PROTEIN", False, True, "Proteins cannot be double stranded"],
]
BLAKE3_LENGTHS = [0, 1, 63, 64, 65, 1023, 1024, 1025, 2048, 2049, 3072, 3073, 4096, 4097, 5120, 5121, 6144, 6145, 7168, 7169,
                  8192, 8193, 16384, 31744, 102400, (1 << 20) - 1, 1 << 20, (1 << 20) + 1]

COMP = dict(zip(b"ABCDGHKMNRSTVWYabcdghkmnrstvwy", b"TVGHCDMKNYSABWRtvghcdmknysabwr"))  # transform.go:78-109
NUCLEIC, PROTEIN = "ATUGCYRSWKMBDHVNZ", "ACDEFGHIKLMNPQRSTVWYUO*BXZ"


def least_rotation(s: bytes) -> bytes:  # the lexicographically least rotation (its bytes do not depend on which start)
    return min((s[i:] + s[:i] for i in range(len(s))), default=b"")


def seqhash(seq: str, t: str, circular: bool, ds: bool):
    s = seq.upper()
    if t == "RNA":
        s = s.replace("U", "T")
    alpha = PROTEIN if t == "PROTEIN" else NUCLEIC
    for ch in s:
        if ch not in alpha:
            return None
    if t == "PROTEIN" and ds:
        return None
    b = s.encode()
    rc = bytes(COMP.get(c, 0) for c in reversed(b))
    if circular and ds:
        det = min(least_rotation(b), least_rotation(rc))
    elif circular:
        det = least_rotation(b)
    elif ds:
        det = min(b, rc)
    else:
        det = b
    return "v1_" + t[0] + ("C" if circular else "L") + ("D" if ds else "S") + "_" + blake3.blake3(det).hexdigest()


def random_cases(rng: random.Random):
    out = []
    for t in ("DNA", "RNA", "PROTEIN"):
        for circular in (False, True):
            for ds in (False, True):
                if t == "PROTEIN" and ds:
                    continue
                for _ in range(40):
                    if t == "PROTEIN":
                        letters = PROTEIN + PROTEIN.lower()
                    elif rng.random() < 0.3:
                        letters = "ACGTUZNacgtuz"  # U/Z complement to NUL; lowercase folds
                    else:
                        letters = "ACGT" if rng.random() < 0.5 else "AC"
                    n = rng.choice([0, 1, 2, 3, rng.randint(4, 40), rng.randint(40, 1100), rng.randint(1000, 3100)])
                    seq = "".join(rng.choice(letters) for _ in range(n))
                    out.append([seq, t, circular, ds, seqhash(seq, t, circular, ds)])
    return out


def puc19() -> str:
    text = open(os.path.join(os.environ["POLY_REFERENCE"], "data", "puc19.gbk")).read()
    origin = text[text.index("\nORIGIN") + 1:]
    origin = origin[origin.index("\n") + 1: origin.index("//")]
    return re.sub("[^a-zA-Z]+", "", origin)  # genbank.go:125,633


def main():
    for seq, t, c, d, want in PINS:
        assert seqhash(seq, t, c, d) == want, (seq, t, c, d)
    vectors = [[n, blake3.blake3(bytes(i % 251 for i in range(n))).hexdigest()] for n in BLAKE3_LENGTHS]
    p = puc19()
    assert len(p) == 2686
    with open(os.path.join(HERE, "seqhash", "puc19.txt"), "w") as f:
        f.write(p + "\n")
    goldens = {
        "pins": PINS,
        "errors": ERRORS,
        "blake3_input": "byte i = i mod 251",
        "blake3": vectors,
        "random": random_cases(random.Random(20261015)),
        "puc19_circular_double_stranded": seqhash(p, "DNA", True, True),
    }
    with open(os.path.join(HERE, "seqhash_goldens.json"), "w") as f:
        json.dump(goldens, f, indent=0)
        f.write("\n")


if __name__ == "__main__":
    main()
