"""The packed PCG-II tiles in both widths of their non-constant values.

k_link_pcg2 keeps the non-constant values of a candidate as 16-bit halves, two per word, when every non-constant
vocabulary has at most 65536 values, and as 32-bit words otherwise; DBL_NO_ID16 forces the 32-bit words on a model
that would get the 16-bit ones.  For an odd and an even number of non-constant attributes, both widths must draw
what the oracle draws and give every record's categorical the oracle's total, bit for bit, under the same kernel name.
"""
import numpy as np
import pytest

from helpers import assert_same_mass, oracle_setup, product_setup, random_state
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu


def _model(n_const, n_str):
    from dblink_b200 import synth

    C = synth.SynthAttr
    attrs = [C(f"c{i}", "constant", v, 0.5) for i, v in enumerate((5, 9, 31, 50)[:n_const])]
    attrs += [C(f"s{i}", "levenshtein", 40 + 10 * i) for i in range(n_str)]
    return synth.generate(13, 900, attrs, dup=0.3, distortion=0.15, missing=0.05, n_files=2)


@pytest.mark.parametrize("width", ["16", "32"])
@pytest.mark.parametrize("shape", [(2, 3), (4, 6)])
def test_packed_tiles_against_oracle(oracle, monkeypatch, shape, width):
    n_const, n_str = shape
    if width == "32":
        monkeypatch.setenv("DBL_NO_ID16", "1")
    g = _model(n_const, n_str)
    A = n_const + n_str
    eng, rc, x, file = product_setup(g, 17, 1, (A - 1,))
    eng.set_link_mass_capture(True)
    assert eng.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS={n_str},HC=32,PK=1>"
    assert eng.link_tile_format("PCG-II")["id16"] == (width == "16")
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 17, 1, (A - 1,))
    np.testing.assert_array_equal(x, ox)
    for it in range(3):
        eng.sweep("PCG-II", 1)
        assert st.sweep(oracle.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit sweep {it}")
    # a random state: candidates whose values are not the records' own
    Vs = [ix.num_values for ix in rc.indexes]
    rng = np.random.default_rng(3)
    y, link, z = random_state(rng, x, x.shape[0] // 2, Vs)
    theta = rng.uniform(0.01, 0.3, (A, int(file.max()) + 1))
    eng.upload_state(x, file, z, link, y, theta, iteration=7)
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 7)
    for it in range(2):
        eng.sweep("PCG-II", 1)
        assert st.sweep(oracle.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit random state sweep {it}")
    eng.close()
