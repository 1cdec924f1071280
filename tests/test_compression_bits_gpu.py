"""One MARGINALIZE at every tiling the compression stage dispatches on (the benchmark's batch of 8 config-B filters; c a
multiple of 64, a partial 64-block, an odd number of 32-tiles; one and sixteen split-K chunks; m <= n; SIMT and FP64
tensor-core members in one batch; fp64) leaves exactly the bits of tests/golden/compression_bits.npz, filter by filter and
as one device batch.  The rank decision of a long fp32 window looks at pivots that are rounding noise, so the Gram products,
their split-K sum and T'', R'', r'' must not move by one bit (DESIGN.md 4.5)."""
from pathlib import Path

import numpy as np
import pytest

from tests.golden import make_compression_bits as mcb

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).parent / "golden" / "compression_bits.npz"


@pytest.fixture(scope="module")
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.mark.parametrize("batched", [False, True])
@pytest.mark.parametrize("case", list(mcb.CASES))
def test_marginalize_bits_match_the_golden_vectors(golden, case, batched):
    for i, out in enumerate(mcb.run(case, batched)):
        for name, a in out.items():
            ref = golden[mcb.key(case, i, name)]
            assert a.dtype == ref.dtype and a.shape == ref.shape, (case, i, name, a.dtype, ref.dtype, a.shape, ref.shape)
            assert np.array_equal(a, ref), (case, i, name, float(np.max(np.abs(a.astype(np.float64) - ref))))
        n = out["delta_x"].size
        assert (out["m_rank"][0] <= n) == (case == "m_le_n"), (case, out["m_rank"], n)
