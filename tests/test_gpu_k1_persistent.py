"""K1's persistent CTAs: batches with more 32-read tiles than resident CTAs, so each CTA hashes
several tiles through both input stages, compared bit-exact with the CPU oracle."""
import numpy as np
import pytest

from poly_b200 import mash, synth

pytestmark = pytest.mark.gpu

# K1 keeps 8 one-warp CTAs per SM at L = 150 (2 x 4816 B input stages + a 16,512 B output tile);
# 132 SMs x 8 = 1056 CTAs on an H100 SXM.  3 x 1056 + 37 tiles is neither fewer than nor a multiple
# of that, and the 19 rows after the last whole tile take the generic kernel.
TILES = 3 * 132 * 8 + 37


@pytest.mark.parametrize("k", [21, 31])
def test_uniform_more_tiles_than_resident_ctas(gpu, oracle, k):
    L, s = 150, 1000
    n = 32 * TILES + 19
    reads = synth.independent_reads(n, L, first_read=11)
    got = mash.sketch_uniform(reads, n, L, k, s)
    rc, want = oracle.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    assert np.array_equal(got, want[:, : L - k])
