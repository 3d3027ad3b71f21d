"""Every packed k_link_pcg2 shape in every tile format, against the oracle.

dbl_link_inst.cu compiles k_link_pcg2<A, NS, 32, PK=1, ID16, SC> for 1-4 byte-packed constants and every NS, and the
shape changes the code: one record per warp from NS = 9 (unpaired tables, 1/n(y) read through p.attrs), the quad-group
boundaries of the tile (the packed constant word moves to a second LDS.128 group at NS = 7, 8 with 16-bit ids; the
group count changes at NS = 4, 8, 12 with 32-bit ids; an odd NS leaves the high half of the last id word empty), the
byte of the top constant in the packed word (byte 3 only at NC = 4).  One synthetic model per (NC constants, NS
non-constant attributes) reaches each of them: the constant at kernel position NC - 1 observes all 255 of its values
(0xFE in the top packed byte), the attributes are interleaved so that kernel order differs from attribute order, and
records miss every string value, every constant value or exactly one string value.  One block of an odd number of
records: the last warp has one record, and the block spans several 128-entity tiles.

Each case first asserts the kernel and the tile format it gets (GibbsEngine.link_tile_format), before the engine has a
state and after, then after every sweep
from the initial state and from a random one: the state equals the oracle's and every record's link mass equals the
oracle's, bit for bit; on the first sweep from the random state the masses also match the literal GU conditionals.
The four high-code cases give the last non-constant attribute a 40 000-value vocabulary, so that codes >= 2^15 (the
top bit of a 16-bit half) sit in the last id word: its low half at NS = 7, its high half at NS = 8.
"""
import numpy as np
import pytest

from helpers import (assert_literal_mass, assert_same_mass, encode, literal_link_mass, oracle_indexes,
                     random_state)
from test_gpu_link_paired_keys import BIG_V, _grouped_tables
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu

R = 601          # one block, odd: the last warp of a two-record shape has one record
SMALL_CONST = (5, 9, 31)  # the vocabularies of the other constants, by kernel position
N_MISSING = 37   # missing values forced per attribute: >= 6 % of R
N_ALL = 12       # records missing every string value; as many missing every constant value
N_ONE = 30       # records missing exactly one string value

# id -> (environment, packed constants, 16-bit ids, slot codes)
FORMATS = {
    "sc16": ({}, True, True, True),
    "sc32": ({"DBL_NO_ID16": "1"}, True, False, True),
    "id16": ({"DBL_NO_SC": "1"}, True, True, False),
    "id32": ({"DBL_NO_SC": "1", "DBL_NO_ID16": "1"}, True, False, False),
    "unpacked": ({"DBL_NO_PACK": "1"}, False, False, False),
}


def _ns_range(nc):
    return range(1, min(16 - nc, 12) + 1)


CASES = ([(nc, ns, "sc16", False) for nc in (1, 2, 3, 4) for ns in _ns_range(nc)] +
         [(nc, ns, f, False) for f in ("sc32", "id16", "id32", "unpacked") for nc in (1, 4) for ns in _ns_range(nc)] +
         [(nc, ns, "sc16", True) for nc in (1, 4) for ns in (7, 8)])


def _case_id(case):
    nc, ns, fmt, high = case
    return f"nc{nc}-ns{ns}-{fmt}" + ("-high" if high else "")


def expected_format(ns, fmt):
    """The tile format k_link_pcg2 reads, restated from the kernel's rules: two records per warp in the 32-slot
    shapes with at most 8 non-constant attributes; their key tables paired when the tiles hold 16-bit slot codes."""
    _, _, id16, sc = FORMATS[fmt]
    rpw = 2 if ns <= 8 else 1
    return {"id16": id16, "slot_codes": sc, "paired": id16 and sc and rpw == 2, "records_per_warp": rpw}


def _model(O, n_const, n_str, high=False, seed=0):
    """A model of n_const constant and n_str non-constant attributes, interleaved, with one block of R records.
    -> (product indexes, oracle indexes, x, file, F, attribute index of kernel position k)"""
    import dblink_b200 as D
    from dblink_b200 import synth

    names = [("c", i) for i in range(n_const)] + [("s", i) for i in range(n_str)]
    names = names[::2] + names[1::2]  # attribute order; kernel order = constants, then the rest, each in this order
    kpos = [a for a, (k, _) in enumerate(names) if k == "c"] + [a for a, (k, _) in enumerate(names) if k == "s"]
    C = synth.SynthAttr
    attrs = []
    for a, (kind, i) in enumerate(names):
        if kind == "c":
            k = kpos.index(a)
            attrs.append(C(f"c{i}", "constant", 255 if k == n_const - 1 else SMALL_CONST[k], 0.5))
        else:
            attrs.append(C(f"s{i}", "levenshtein", 40 + 10 * i))
    g = synth.generate(seed + 100 * n_const + n_str, R, attrs, dup=0.3, distortion=0.15, missing=0.0, n_files=2)
    vals = g["values"]
    top = kpos[n_const - 1]
    for r in range(255):  # every value of the 255-value constant observed: its top id 254 = 0xFE occurs
        vals[r][top] = f"{r:03d}"
    rng = np.random.default_rng(seed + 7)
    consts, strs = kpos[:n_const], kpos[n_const:]
    for a in range(len(attrs)):
        for r in rng.choice(np.arange(255 if a == top else 0, R), N_MISSING, replace=False):
            vals[r][a] = None
    rest = rng.permutation(np.arange(255, R))
    for r in rest[:N_ALL]:
        for a in strs:
            vals[r][a] = None
    for r in rest[N_ALL:2 * N_ALL]:
        for a in consts:
            vals[r][a] = None
    full = [r for r in rest[2 * N_ALL:] if all(vals[r][a] is not None for a in strs)]
    for r in full[:N_ONE]:
        vals[r][strs[rng.integers(0, n_str)]] = None

    rc = D.RecordsCache.build(vals, g["files"], g["attributes"], 10)
    x, file = rc.transform_records(vals, g["files"])
    p_idx = list(rc.indexes)
    o_idx = oracle_indexes(O, g)
    ox, ofile, F = encode(o_idx, g)
    np.testing.assert_array_equal(x, ox)
    np.testing.assert_array_equal(file, ofile)
    assert p_idx[top].num_values == 255 and (x[:, top] == 254).any()
    if high:
        # the last non-constant attribute in kernel order: 40 000 values in groups of four similar ones; half the
        # entities take values whose codes are >= 2^15
        a = strs[-1]
        probs, rowptr, col, expsim = _grouped_tables(BIG_V)
        p_idx[a] = D.AttributeIndex.from_tables(probs, rowptr, col, expsim, constant=False,
                                                expected_max_cluster_size=10)
        o_idx[a] = O.Index.from_tables(probs, rowptr, col, expsim, False, 10)
        hi = np.flatnonzero(p_idx[a].slot_codes >= 1 << 15)
        ent = np.asarray(g["ent_ids"])
        n_ent = int(ent.max()) + 1
        ev = np.where(rng.random(n_ent) < 0.5, rng.choice(hi, n_ent), rng.integers(0, BIG_V, n_ent))
        v = ev[ent]
        dist = rng.random(R) < 0.15
        v[dist] = np.minimum((v[dist] // 4) * 4 + rng.integers(0, 4, int(dist.sum())), BIG_V - 1)
        x[:, a] = np.where(x[:, a] < 0, -1, v)
    return p_idx, o_idx, np.ascontiguousarray(x, np.int32), file, F, kpos


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_link_shape_against_oracle(oracle, monkeypatch, case):
    import dblink_b200 as D

    O = oracle
    n_const, n_str, fmt, high = case
    env, pk, _, _ = FORMATS[fmt]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    A = n_const + n_str
    p_idx, o_idx, x, file, F, kpos = _model(O, n_const, n_str, high)
    strs = kpos[n_const:]
    # the model is what the case says it is
    assert (x < 0).mean(axis=0).min() >= 0.05
    assert (x[:, strs] < 0).all(axis=1).sum() >= 10
    assert (x[:, kpos[:n_const]] < 0).all(axis=1).sum() >= 10
    assert ((x[:, strs] < 0).sum(axis=1) == 1).sum() >= 10
    codes = [p_idx[a].slot_codes for a in strs]
    assert all(p_idx[a].hash_slots == 32 for a in strs)
    assert all(c is not None for c in codes) and max(int(c.max()) for c in codes) < 1 << 16
    if high:
        obs = x[:, strs[-1]][x[:, strs[-1]] >= 0]
        assert (codes[-1][obs] >= 1 << 15).sum() >= 100

    alpha = [10.0] * A
    beta = [1000.0] * A
    seed = 41
    eng = D.GibbsEngine(p_idx, alpha, beta, None, seed, F)
    # the kernel and its tile format follow from the model alone: already decided before the first state
    kernel = f"k_link_pcg2<A={A},NS={n_str},HC=32,PK={int(pk)}>"
    assert eng.link_kernel("PCG-II") == kernel
    assert eng.link_tile_format("PCG-II") == expected_format(n_str, fmt)
    eng.init_state(x, file)
    eng.set_partitioner(D.KDTreePartitioner(0, []).fit(eng.download_state()["y"]))
    assert eng.num_partitions == 1
    eng.set_link_mass_capture(True)
    # routing first: the case tests what it says it tests
    assert eng.link_kernel("PCG-II") == kernel
    assert eng.link_tile_format("PCG-II") == expected_format(n_str, fmt)

    m0 = O.Model(o_idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    m = O.Model(o_idx, alpha, beta, O.KDTree.fit(s0.y, 0, []), seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0)
    what = _case_id(case)
    for it in range(3):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{what} sweep {it}")

    rng = np.random.default_rng(9)
    Vs = [ix.num_values for ix in p_idx]
    y, link, z = random_state(rng, x, R // 2, Vs)
    if high:
        assert (codes[-1][y[:, strs[-1]]] >= 1 << 15).sum() >= 100
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
