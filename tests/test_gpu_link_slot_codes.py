"""The packed PCG-II tiles with slot codes in place of the non-constant value ids.

When every non-constant attribute's values colour (AttributeIndex.slot_codes), k_link_pcg2 stores each candidate's
slot codes in its packed tiles and probes every record's table at code & 31, with no per-record hash multipliers;
DBL_NO_SC forces the value ids and the multipliers on such a model.  Both, in both widths of the tile values and with
missing values, must draw what the oracle draws and give every record's categorical the oracle's total, bit for bit,
under the same kernel name.
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
    return synth.generate(29, 900, attrs, dup=0.3, distortion=0.15, missing=0.08, n_files=2)


@pytest.mark.parametrize("codes", ["sc", "no-sc"])
@pytest.mark.parametrize("width", ["16", "32"])
@pytest.mark.parametrize("shape", [(2, 3), (4, 6)])
def test_slot_code_tiles_against_oracle(oracle, monkeypatch, shape, width, codes):
    n_const, n_str = shape
    if width == "32":
        monkeypatch.setenv("DBL_NO_ID16", "1")
    if codes == "no-sc":
        monkeypatch.setenv("DBL_NO_SC", "1")
    g = _model(n_const, n_str)
    A = n_const + n_str
    eng, rc, x, file = product_setup(g, 23, 1, (A - 1,))
    assert all(ix.slot_codes is not None for ix in rc.indexes if not ix.is_constant)
    assert (x < 0).any(axis=0)[n_const:].all()  # records with a missing value in every non-constant attribute
    eng.set_link_mass_capture(True)
    assert eng.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS={n_str},HC=32,PK=1>"
    fmt = eng.link_tile_format("PCG-II")
    assert (fmt["slot_codes"], fmt["id16"]) == (codes == "sc", width == "16")
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 23, 1, (A - 1,))
    np.testing.assert_array_equal(x, ox)
    for it in range(3):
        eng.sweep("PCG-II", 1)
        assert st.sweep(oracle.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit {codes} sweep {it}")
    # a random state: candidates whose values are not the records' own
    Vs = [ix.num_values for ix in rc.indexes]
    rng = np.random.default_rng(5)
    y, link, z = random_state(rng, x, x.shape[0] // 2, Vs)
    theta = rng.uniform(0.01, 0.3, (A, int(file.max()) + 1))
    eng.upload_state(x, file, z, link, y, theta, iteration=7)
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 7)
    for it in range(2):
        eng.sweep("PCG-II", 1)
        assert st.sweep(oracle.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit {codes} random state sweep {it}")
    eng.close()
