"""The paired key tables of the PCG-II link kernel.

With 16-bit slot codes in the packed tiles, the two records of a k_link_pcg2 warp share one key word per slot and
non-constant attribute (record 0's code in the low half, record 1's in the high half; an empty half holds slot ^ 1),
so one load probes both records.  Cases that only the pairing has: a warp whose second record is absent (a block with
an odd number of records), records missing every non-constant value (both halves of their tables empty), and codes of
2^15 and more (the high bit of a half).  Each must draw what the oracle draws and give every record's categorical the
oracle's total, bit for bit, under the same kernel name; DBL_NO_ID16 runs the same model on the unpaired 32-bit tiles.
"""
import numpy as np
import pytest

from helpers import assert_same_mass, random_state
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu

BIG_V = 40_000  # vocabulary of the first two non-constant attributes: codes up to ~40 000, i.e. beyond 2^15
SMALL_V = 400
CONST_V = (5, 9, 31, 50)


def _grouped_tables(V):
    """A non-constant attribute whose values come in groups of four mutually similar values: CSR rows (the diagonal
    included, columns ascending) and value probabilities."""
    start = (np.arange(V) // 4) * 4
    size = np.minimum(start + 4, V) - start
    rowptr = np.r_[0, np.cumsum(size)].astype(np.int32)
    col = np.concatenate([np.arange(s, s + n) for s, n in zip(start, size)]).astype(np.int32)
    row = np.repeat(np.arange(V), size)
    expsim = np.where(col == row, np.exp(10.0), 2.0 + (col + row) % 5)
    w = 1.0 / (1.0 + np.arange(V) % 97)
    return w / w.sum(), rowptr, col, expsim


def _model(O, n_const, n_str):
    """Both sides' indexes from the same tables: (product indexes, oracle indexes, V per attribute)."""
    import dblink_b200 as D

    p_idx, o_idx, Vs = [], [], []
    for V in CONST_V[:n_const]:
        probs = np.full(V, 1.0 / V)
        p_idx.append(D.AttributeIndex.from_tables(probs, constant=True, expected_max_cluster_size=10))
        o_idx.append(O.Index.from_tables(probs, np.zeros(V + 1, np.int32), [], [], True, 10))
        Vs.append(V)
    for q in range(n_str):
        V = BIG_V if q < 2 else SMALL_V
        probs, rowptr, col, expsim = _grouped_tables(V)
        p_idx.append(D.AttributeIndex.from_tables(probs, rowptr, col, expsim, constant=False,
                                                  expected_max_cluster_size=10))
        o_idx.append(O.Index.from_tables(probs, rowptr, col, expsim, False, 10))
        Vs.append(V)
    return p_idx, o_idx, Vs


def _records(rng, p_idx, Vs, n_const, R, n_ent):
    """Records of n_ent entities: distorted values move within their group of similar values, 5 % are missing, and
    20 records miss every non-constant value.  Half the entities take their large-vocabulary values among the codes
    >= 2^15."""
    A = len(Vs)
    ent = np.empty((n_ent, A), np.int64)
    for a, V in enumerate(Vs):
        ent[:, a] = rng.integers(0, V, n_ent)
        if V == BIG_V:
            high = np.flatnonzero(p_idx[a].slot_codes >= 1 << 15)
            pick = rng.random(n_ent) < 0.5
            ent[pick, a] = rng.choice(high, int(pick.sum()))
    ent_of = np.concatenate([np.arange(n_ent), rng.integers(0, n_ent, R - n_ent)])
    rng.shuffle(ent_of)
    x = ent[ent_of].copy()
    for a, V in enumerate(Vs):
        dist = rng.random(R) < 0.15
        if a < n_const:
            x[dist, a] = rng.integers(0, V, int(dist.sum()))
        else:
            start = (x[dist, a] // 4) * 4
            x[dist, a] = np.minimum(start + rng.integers(0, 4, int(dist.sum())), V - 1)
        x[rng.random(R) < 0.05, a] = -1
    x[rng.choice(R, 20, replace=False), n_const:] = -1
    return np.ascontiguousarray(x, np.int32), rng.integers(0, 2, R).astype(np.int32)


@pytest.mark.parametrize("width", ["16", "32"])
@pytest.mark.parametrize("shape", [(2, 3), (4, 6)])
def test_paired_key_tables_against_oracle(oracle, monkeypatch, shape, width):
    import dblink_b200 as D

    O = oracle
    if width == "32":
        monkeypatch.setenv("DBL_NO_ID16", "1")  # the same model on the unpaired 32-bit tiles
    n_const, n_str = shape
    A = n_const + n_str
    seed, R = 31, 1001  # one block of an odd number of records: the last warp has one record
    rng = np.random.default_rng(11)
    p_idx, o_idx, Vs = _model(O, n_const, n_str)
    x, file = _records(rng, p_idx, Vs, n_const, R, 700)
    F = 2
    alpha, beta = [10.0] * A, [1000.0] * A

    # what makes the engine take 16-bit slot codes: codes for every non-constant attribute, all below 2^16
    codes = [ix.slot_codes for ix in p_idx[n_const:]]
    assert all(c is not None for c in codes)
    assert max(int(c.max()) for c in codes) < 1 << 16
    for q in range(2):  # records and codes in the upper half of the 16-bit range
        obs = x[:, n_const + q][x[:, n_const + q] >= 0]
        assert int(codes[q].max()) >= 1 << 15 and (codes[q][obs] >= 1 << 15).sum() > 100
    assert ((x[:, n_const:] < 0).all(axis=1)).sum() >= 20

    eng = D.GibbsEngine(p_idx, alpha, beta, None, seed, F)
    eng.init_state(x, file)
    part = D.KDTreePartitioner(0, []).fit(eng.download_state()["y"])
    eng.set_partitioner(part)
    assert eng.num_partitions == 1 and R % 2 == 1
    eng.set_link_mass_capture(True)
    assert eng.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS={n_str},HC=32,PK=1>"
    assert eng.link_tile_format("PCG-II")["paired"] == (width == "16")  # the 32-bit tiles keep unpaired tables

    m0 = O.Model(o_idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    m = O.Model(o_idx, alpha, beta, O.KDTree.fit(s0.y, 0, []), seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0)
    for it in range(3):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit sweep {it}")
    # a random state: entities spread over every code of the large vocabularies
    y, link, z = random_state(rng, x, 701, Vs)
    assert (codes[0][y[:, n_const]] >= 1 << 15).sum() > 100
    theta = rng.uniform(0.01, 0.3, (A, F))
    eng.upload_state(x, file, z, link, y, theta, iteration=7)
    st = O.State.from_arrays(m, x, file, z, link, y, theta, 7)
    for it in range(2):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{shape} {width}-bit random state sweep {it}")
    eng.close()
