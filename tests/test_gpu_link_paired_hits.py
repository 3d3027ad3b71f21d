"""The hit tests of the PCG-II link kernel's paired key tables, over the whole 16-bit code range.

In the paired k_link_pcg2 instantiations (16-bit slot codes, two records per warp) one key word holds both records'
codes of a slot, and record 0 hits where the low half of key ^ {code, code} is zero, record 1 where the high half is,
each tested by one 3-input lop3 (pcg2_half_hit).  Cases: every code from 0 to 65535 in one vocabulary (the top bit of
either half set or not, each of the eight top-three-bit patterns among the records' values); rows that fill 24 of the
32 slots, so that most probes of a step hit in both records; a warp where one record has a table for an attribute and
the other has not (records missing exactly one non-constant value, each at a random attribute, or no second record at
the end of an odd block); records missing values, scored through the 1/n(y) gather.  Each must draw what the oracle
draws and give every record's categorical the oracle's total, bit for bit, and on the first sweep from a random state
match the literal conditionals.
"""
import numpy as np
import pytest

from helpers import assert_literal_mass, assert_same_mass, literal_link_mass, random_state
from test_gpu_link_paired_keys import BIG_V, _grouped_tables
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu

FULL_V = 1 << 16  # slot codes 0..65535, every one of them
WIDE_V, WIDE_G = 960, 24  # groups of 24 mutually similar values: every row fills 24 of the 32 slots
SMALL_V = 400
CONST_V = (5, 9, 31, 50)
R = 1001          # one block, odd: the last warp has one record
N_ONE = 120       # records missing exactly one non-constant value, at a random attribute
N_ALL = 20        # records missing every non-constant value


def _group_tables(V, g):
    """Values in groups of g mutually similar values (as _grouped_tables, any group size)"""
    start = (np.arange(V) // g) * g
    size = np.minimum(start + g, V) - start
    rowptr = np.r_[0, np.cumsum(size)].astype(np.int32)
    col = np.concatenate([np.arange(s, s + n) for s, n in zip(start, size)]).astype(np.int32)
    row = np.repeat(np.arange(V), size)
    expsim = np.where(col == row, np.exp(10.0), 1.5 + (col + row) % 7)
    w = 1.0 / (1.0 + np.arange(V) % 89)
    return w / w.sum(), rowptr, col, expsim


# non-constant attributes in kernel order: (vocabulary, group size)
STR_ATTRS = [(FULL_V, 4), (WIDE_V, WIDE_G), (BIG_V, 4), (SMALL_V, 4), (SMALL_V, 4), (SMALL_V, 4), (SMALL_V, 4),
             (SMALL_V, 4)]


def _model(O, n_const, n_str):
    import dblink_b200 as D

    p_idx, o_idx, Vs, groups = [], [], [], []
    for V in CONST_V[:n_const]:
        probs = np.full(V, 1.0 / V)
        p_idx.append(D.AttributeIndex.from_tables(probs, constant=True, expected_max_cluster_size=10))
        o_idx.append(O.Index.from_tables(probs, np.zeros(V + 1, np.int32), [], [], True, 10))
        Vs.append(V)
        groups.append(1)
    for V, g in STR_ATTRS[:n_str]:
        probs, rowptr, col, expsim = _grouped_tables(V) if g == 4 else _group_tables(V, g)
        p_idx.append(D.AttributeIndex.from_tables(probs, rowptr, col, expsim, constant=False,
                                                  expected_max_cluster_size=10))
        o_idx.append(O.Index.from_tables(probs, rowptr, col, expsim, False, 10))
        Vs.append(V)
        groups.append(g)
    return p_idx, o_idx, Vs, groups


def _records(rng, p_idx, Vs, groups, n_const, n_ent):
    """Records of n_ent entities.  In the FULL_V attribute the entities' values are spread evenly over the eight
    patterns of the code's top three bits; distorted values move within their group; 5 % of the values are missing,
    N_ONE records miss exactly one non-constant value and N_ALL miss all of them."""
    A = len(Vs)
    ent = np.empty((n_ent, A), np.int64)
    for a, V in enumerate(Vs):
        ent[:, a] = rng.integers(0, V, n_ent)
        if V == FULL_V:
            top = p_idx[a].slot_codes >> 13
            ent[:, a] = [rng.choice(np.flatnonzero(top == t)) for t in np.arange(n_ent) % 8]
    ent_of = np.concatenate([np.arange(n_ent), rng.integers(0, n_ent, R - n_ent)])
    rng.shuffle(ent_of)
    x = ent[ent_of].copy()
    for a, V in enumerate(Vs):
        dist = rng.random(R) < 0.15
        if a < n_const:
            x[dist, a] = rng.integers(0, V, int(dist.sum()))
        else:
            g = groups[a]
            x[dist, a] = np.minimum((x[dist, a] // g) * g + rng.integers(0, g, int(dist.sum())), V - 1)
        x[rng.random(R) < 0.05, a] = -1
    rows = rng.permutation(R)
    x[rows[:N_ALL], n_const:] = -1
    one = rows[N_ALL:N_ALL + N_ONE]
    x[one, n_const + rng.integers(0, A - n_const, N_ONE)] = -1
    return np.ascontiguousarray(x, np.int32), rng.integers(0, 2, R).astype(np.int32)


@pytest.mark.parametrize("shape", [(4, 6), (1, 8), (2, 3)], ids=lambda s: f"nc{s[0]}-ns{s[1]}")
def test_paired_hits_against_oracle(oracle, shape):
    import dblink_b200 as D

    O = oracle
    n_const, n_str = shape
    A = n_const + n_str
    seed = 53
    rng = np.random.default_rng(17)
    p_idx, o_idx, Vs, groups = _model(O, n_const, n_str)
    x, file = _records(rng, p_idx, Vs, groups, n_const, 700)
    F = 2
    alpha, beta = [10.0] * A, [1000.0] * A

    # the model is what the case says it is: 16-bit slot codes in 32-slot tables
    strs = range(n_const, A)
    codes = [p_idx[a].slot_codes for a in strs]
    assert all(c is not None for c in codes) and max(int(c.max()) for c in codes) < 1 << 16
    assert all(p_idx[a].hash_slots == 32 for a in strs)
    # every code of the full vocabulary, and all eight top-three-bit patterns among the records' values
    assert np.array_equal(np.sort(codes[0]), np.arange(FULL_V))
    obs = x[:, n_const][x[:, n_const] >= 0]
    assert set(np.unique(codes[0][obs] >> 13)) == set(range(8))
    if n_str >= 3:
        obs = x[:, n_const + 2][x[:, n_const + 2] >= 0]
        assert (codes[2][obs] >= 1 << 15).sum() > 100
    # every row of the wide-group attribute (its group of values) fills 24 distinct slots
    if n_str >= 2:
        slots = codes[1].reshape(-1, WIDE_G) & 31
        assert all(len(set(row)) == WIDE_G for row in slots.tolist())
    # missing values: whole records, exactly one attribute, and the rest
    miss = x[:, n_const:] < 0
    assert miss.all(axis=1).sum() >= N_ALL and (miss.sum(axis=1) == 1).sum() >= N_ONE // 2
    assert R % 2 == 1

    eng = D.GibbsEngine(p_idx, alpha, beta, None, seed, F)
    eng.init_state(x, file)
    eng.set_partitioner(D.KDTreePartitioner(0, []).fit(eng.download_state()["y"]))
    assert eng.num_partitions == 1
    eng.set_link_mass_capture(True)
    assert eng.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS={n_str},HC=32,PK=1>"
    assert eng.link_tile_format("PCG-II") == {"id16": True, "slot_codes": True, "paired": True,
                                              "records_per_warp": 2}

    m0 = O.Model(o_idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    m = O.Model(o_idx, alpha, beta, O.KDTree.fit(s0.y, 0, []), seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0)
    what = f"nc{n_const}-ns{n_str}"
    for it in range(3):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{what} sweep {it}")

    # a random state: entities spread over every code of the vocabularies
    y, link, z = random_state(rng, x, 701, Vs)
    assert set(np.unique(codes[0][y[:, n_const]] >> 13)) == set(range(8))
    theta = rng.uniform(0.01, 0.3, (A, F))
    eng.upload_state(x, file, z, link, y, theta, iteration=7)
    st = O.State.from_arrays(m, x, file, z, link, y, theta, 7)
    for it in range(2):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        mass = eng.link_mass()
        assert_same_mass(mass, st.last_link_mass(), f"{what} random state sweep {it}")
        if it == 0:
            ref = literal_link_mass(O, m, x, file, y, z, link, st.theta, "PCG-II")
            assert_literal_mass(mass, ref, f"{what} random state sweep 0")
    eng.close()
