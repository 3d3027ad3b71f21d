"""k_link_pcg2 with four records per warp (Pcg2Format::quad), against the oracle and against the two-record shape.

The quad shape scores each candidate for the four records of a warp, whose keys sit in two paired key tables, and
keeps each record's pass-1 chunk totals in shared memory.  A model gets it with the paired tables, at most 6
non-constant attributes and enough records to give every persistent CTA QUAD_ITEMS_PER_CTA work items of 32 records:
here the benchmark's attributes (4 constant, 6 Levenshtein) and 72 000 records in 64 blocks, which clears that bar
on a 132-SM H100.  DBL_NO_QUAD runs the same chain on the two-record shape.  Each sweep must equal the oracle's state
and give every record's categorical the oracle's total, bit for bit, and the two shapes must give the same links
and totals, bit for bit.

Inside a block, the records are ordered by cost class, and every record with a missing non-constant value sorts
behind every record without one (k_rec_class), so they fill the block's last positions.  The model is checked to
reach: blocks whose record count leaves 1, 2 and 3 records in the last warp, and blocks whose run of records with a
missing value starts at each of the four positions of a warp and is at least four records long (a missing value at
every position, beside records without one in the same warp).
"""
import numpy as np
import pytest

from helpers import assert_same_mass, oracle_setup, product_setup, synth_problem

pytestmark = pytest.mark.gpu

R = 72_000
SEED, LEVELS, SPLIT = 29, 6, (0, 1, 2, 3)
SWEEPS = 3
QUAD = {"id16": True, "slot_codes": True, "paired": True, "records_per_warp": 4}
PAIR = dict(QUAD, records_per_warp=2)


@pytest.fixture(scope="module")
def problem():
    from dblink_b200 import synth

    return synth_problem(seed=11, R=R, attrs=synth.config_attrs(4), dup=0.1, distortion=0.05, missing=0.01,
                         n_files=2)


def _chain(g, monkeypatch, no_quad):
    """SWEEPS PCG-II sweeps -> (format, [(state before the sweep, state after, link masses)] per sweep, x)"""
    with monkeypatch.context() as mp:
        if no_quad:
            mp.setenv("DBL_NO_QUAD", "1")
        eng, rc, x, file = product_setup(g, SEED, LEVELS, SPLIT)
        eng.set_link_mass_capture(True)
        fmt = eng.link_tile_format("PCG-II")
        out = []
        for _ in range(SWEEPS):
            before = eng.download_state()
            eng.sweep("PCG-II", 1)
            out.append((before, eng.download_state(), eng.link_mass()))
        eng.close()
    return fmt, out, x


def _block_counts(x, str_cols, d):
    """per block: (records, records with a missing non-constant value), in the state d"""
    blk = d["block"][d["link"]]
    miss = (x[:, str_cols] < 0).any(axis=1)
    return np.bincount(blk), np.bincount(blk, weights=miss).astype(np.int64)


def test_quad_shape_against_oracle_and_two_record_shape(oracle, problem, monkeypatch):
    g = problem
    fmt4, quad, x = _chain(g, monkeypatch, no_quad=False)
    fmt2, pair, _ = _chain(g, monkeypatch, no_quad=True)
    assert fmt4 == QUAD
    assert fmt2 == PAIR

    str_cols = [a for a, at in enumerate(g["attributes"]) if not at.is_constant]
    n, m = _block_counts(x, str_cols, quad[0][0])
    assert {1, 2, 3} <= set((n[n > 0] % 4).tolist()), "blocks whose last warp holds 1, 2 and 3 records"
    starts = set(((n - m)[m >= 4] % 4).tolist())
    assert starts == {0, 1, 2, 3}, f"runs of records with a missing value start at warp positions {starts}"

    m_, st, tree, ox, ofile = oracle_setup(oracle, g, SEED, LEVELS, SPLIT)
    for it, ((_, d4, mass4), (_, d2, mass2)) in enumerate(zip(quad, pair)):
        assert st.sweep(oracle.PCG_II) == 0
        for k in ("theta", "link", "y", "z", "block"):
            np.testing.assert_array_equal(d4[k], getattr(st, k), err_msg=f"quad sweep {it}: {k}")
            np.testing.assert_array_equal(d2[k], d4[k], err_msg=f"two-record shape sweep {it}: {k}")
        assert_same_mass(mass4, st.last_link_mass(), f"quad sweep {it} against the oracle")
        assert_same_mass(mass2, mass4, f"two-record shape against quad, sweep {it}")


def test_small_state_keeps_two_records_per_warp():
    """the same model with too few records for four per warp keeps the two-record shape"""
    from dblink_b200 import synth

    g = synth_problem(seed=11, R=4000, attrs=synth.config_attrs(4), missing=0.01, n_files=2)
    eng, rc, x, file = product_setup(g, SEED, 2, SPLIT[:2])
    assert eng.link_tile_format("PCG-II") == PAIR
    eng.close()
