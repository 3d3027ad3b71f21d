"""Every link-kernel variant against the oracle, with the total mass of every record's categorical checked.

One table of models, each built to reach one family of kernels: k_link_pcg2 with run-time hash tables of 64, 128
and 256 slots (HC=0), both silent fall-backs of PCG-II to k_link_generic (tables over the 100 KB limit; rows that
do not hash into 256 slots), the packed-constant boundary (255 / 256 values), A = 32, and crafted states that drive
k_link_pruned through its re-walk path (> PRUNED_SCAP survivors), its single-survivor shortcut and k_link_heavy.
Each row first asserts the hash-table sizes and the kernel every (sampler, link mode) gets, so that a routing
change fails loudly instead of quietly testing something else.

Then, for every sampler and link modes 0 / 1 / 2, after every sweep: the state equals the oracle's bit for bit, the
per-record totals (dbl_link_mass) equal the oracle's bit for bit and each other across the three modes, and they
match the literal GU conditionals summed over the block (helpers.literal_link_mass) to LITERAL_MASS_REL.  A draw
only moves when its uniform falls into the interval a wrong weight shifts; the total of every record sees every
candidate's weight on every sweep.
"""
import numpy as np
import pytest

from helpers import (assert_literal_mass, assert_same_mass, literal_link_mass, oracle_setup, product_setup,
                     random_state, threshold_problem)
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu

SAMPLERS = ["PCG-II", "PCG-I", "Gibbs", "Gibbs-Sequential"]
MODES = (0, 1, 2)
PRUNED_SCAP = 48           # k_link_pruned keeps this many survivors for its second pass (dbl_link.cuh)
HEAVY_MIN_CANDIDATES = 256  # blocks beyond this size hand records without a must-match attribute to k_link_heavy


def _attrs():
    from dblink_b200 import synth

    return synth.SynthAttr


def _forced_constant(vocab):
    """s0 (60 strings, threshold 7) + c0: a constant over `vocab` values, every one of them observed (records 0 ..
    vocab-1 carry values 0 .. vocab-1), so the index has exactly `vocab` values and the top id vocab-1 occurs"""
    C = _attrs()
    g = threshold_problem(60, 7.0, extra=[C("c0", "constant", vocab)], n_files=2)
    for i in range(vocab):
        g["values"][i][1] = f"{i:03d}"
    return g


def _a32():
    """16 constant and 16 string attributes, interleaved: every lane of a warp holds an attribute, bit 31 of zmask"""
    C = _attrs()
    from dblink_b200 import synth

    attrs = []
    for i in range(16):
        attrs += [C(f"c{i}", "constant", 3 + i % 5, 0.5), C(f"s{i}", "levenshtein", 16 + 2 * i)]
    return synth.generate(7, 900, attrs, dup=0.3, distortion=0.15, missing=0.05, n_files=2)


def _pruned_model():
    C = _attrs()
    from dblink_b200 import synth

    return synth.generate(7, 900, [C("c0", "constant", 3, 0.5), C("s0", "levenshtein", 60)], dup=0.3,
                          distortion=0.15, missing=0.05, n_files=2)


def _c(n):
    C = _attrs()
    return [C(f"c{i}", "constant", v, 0.5) for i, v in enumerate((100, 12, 31, 50)[:n])]


OTHERS = ("k_link_pruned", "k_link_match")  # PCG-I / Gibbs / Gibbs-Sequential in link modes 0 and 2
# name -> (recipe, k-d levels, hash slots per attribute, PCG-II kernel in modes 0 and 2, other samplers in modes 0 / 2,
#          environment)
ROWS = {
    "hash64": (lambda: threshold_problem(60, 3.0, extra=[_attrs()("c0", "constant", 5), _attrs()("c1", "constant", 9)],
                                         n_files=2),
               1, [64, 0, 0], "k_link_pcg2<A=3,NS=1,HC=0,PK=0>", OTHERS, {}),
    # s1's own 32-slot tables are re-hashed to the model's 128 slots
    "hash128": (lambda: threshold_problem(120, 3.0, extra=[_attrs()("s1", "levenshtein", 80)], n_files=2),
                1, [128, 32], "k_link_pcg2<A=2,NS=2,HC=0,PK=0>", OTHERS, {}),
    "hash256": (lambda: threshold_problem(400, 3.0, n_files=2), 1, [256], "k_link_pcg2<A=1,NS=1,HC=0,PK=0>", OTHERS, {}),
    # configs[4]-like 4 constants + 6 strings, one with 128-slot rows: the tables exceed 100 KB -> generic
    "over_smem": (lambda: threshold_problem(1200, 4.0, R=3000, n_files=2,
                                            extra=_c(4) + [_attrs()(f"s{i}", "levenshtein", 300) for i in range(1, 6)]),
                  1, [128, 0, 0, 0, 0, 32, 32, 32, 32, 32], "k_link_generic", OTHERS, {}),
    # a 147-entry row does not hash into 256 slots -> generic
    "no_hash": (lambda: threshold_problem(1200, 3.5, R=3000, n_files=2), 1, [0], "k_link_generic", OTHERS, {}),
    "const255": (lambda: _forced_constant(255), 1, [32, 0], "k_link_pcg2<A=2,NS=1,HC=32,PK=1>", OTHERS, {}),
    "const255_nopack": (lambda: _forced_constant(255), 1, [32, 0], "k_link_pcg2<A=2,NS=1,HC=32,PK=0>", OTHERS,
                        {"DBL_NO_PACK": "1"}),
    "const256": (lambda: _forced_constant(256), 1, [32, 0], "k_link_pcg2<A=2,NS=1,HC=32,PK=0>", OTHERS, {}),
    "a32": (_a32, 1, [0, 32] * 16, "k_link_generic", OTHERS, {}),
    "pruned": (_pruned_model, 0, [0, 32], "k_link_pcg2<A=2,NS=1,HC=32,PK=1>", OTHERS, {}),
    "pruned_bsearch": (_pruned_model, 0, [0, 32], "k_link_pcg2<A=2,NS=1,HC=32,PK=1>", OTHERS,
                       {"DBL_INV_DENSE_MAX": "0"}),
}


def expected_kernel(row, sampler, mode):
    _, _, _, pcg2, other, _ = ROWS[row]
    if mode == 1:
        return "k_link_generic"
    if sampler == "PCG-II":
        return pcg2
    return other[0] if mode == 0 else other[1]


def survivors(x, z, y, link, block):
    """per record: (must-match attributes, candidates of its block that agree on all of them, block size)"""
    R = x.shape[0]
    out = np.zeros((R, 3), np.int64)
    for r in range(R):
        mm = (x[r] >= 0) & (z[r] == 0)
        cand = np.flatnonzero(block == block[link[r]])
        ok = (y[cand][:, mm] == x[r, mm]).all(axis=1)
        out[r] = (mm.sum(), ok.sum(), len(cand))
    return out


def crafted_pruned_state(rng, x, E, Vs):
    """A valid state (z = 0 and x observed => x == y[link]) in one block of E entities with three kinds of records:
    (a) must match only on the 3-value constant c0 (shared by ~E/3 > PRUNED_SCAP entities), distorted on the string s0
    so that their weights differ; (b) one record that must match on a string value exactly one entity has; (c) every
    observed attribute distorted (no must-match attribute: the whole block is scored, by k_link_heavy when
    E > HEAVY_MIN_CANDIDATES)."""
    R = x.shape[0]
    c0, s0 = 0, 1
    link = rng.integers(0, E, R).astype(np.int32)
    y = np.stack([rng.integers(0, Vs[a], E) for a in range(2)], axis=1).astype(np.int32)
    z = np.ones((R, 2), np.uint8)
    z[x < 0] = (rng.random((R, 2)) < 0.1)[x < 0]
    both = np.flatnonzero((x[:, c0] >= 0) & (x[:, s0] >= 0))
    single = int(both[0])
    v = x[single, s0]
    e1 = link[single]
    # only `single` constrains s0: every other entity gets another string value
    y[:, s0] = np.where(y[:, s0] == v, (v + 1) % Vs[s0], y[:, s0])
    y[e1, s0] = v
    z[single, s0] = 0
    taken = {int(e1)}
    for r in both[1:]:
        if rng.random() < 0.6 and int(link[r]) not in taken:  # kind (a); the rest stay kind (c)
            y[link[r], c0] = x[r, c0]
            z[r, c0] = 0
    # a later record of kind (a) on the same entity may have overwritten the c0 value: such records are distorted
    for r in range(R):
        for a in range(2):
            if z[r, a] == 0 and x[r, a] >= 0 and x[r, a] != y[link[r], a]:
                z[r, a] = 1
    # x observed and different from the entity's value => distorted
    assert not ((z == 0) & (x >= 0) & (x != y[link])).any()
    return y, link, z


def _run_chain(oracle, engines, st, sampler, n, row, what):
    m = st.model
    for it in range(n):
        y, z, link = st.y, st.z, st.link
        for eng in engines:
            eng.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        omass = st.last_link_mass()
        masses = []
        for mode, eng in zip(MODES, engines):
            assert_same_state(eng, st)
            masses.append(eng.link_mass())
            assert_same_mass(masses[-1], omass, f"{row} {sampler} {what} sweep {it} mode {mode} vs oracle")
        for mode, ms in zip(MODES[1:], masses[1:]):
            assert_same_mass(ms, masses[0], f"{row} {sampler} {what} sweep {it} mode {mode} vs mode 0")
        ref = literal_link_mass(oracle, m, st.x, st.file, y, z, link, st.theta, sampler)
        assert_literal_mass(masses[0], ref, f"{row} {sampler} {what} sweep {it}")


@pytest.mark.parametrize("sampler", SAMPLERS)
@pytest.mark.parametrize("row", list(ROWS))
def test_link_kernel_against_oracle_and_literal_mass(oracle, monkeypatch, row, sampler):
    recipe, levels, slots, _, _, env = ROWS[row]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = recipe()
    attr_ids = (0,) if levels else ()
    engines = []
    for mode in MODES:
        eng, rc, x, file = product_setup(g, 31, levels, attr_ids)
        eng.set_link_mode(mode)
        eng.set_link_mass_capture(True)
        engines.append(eng)
    # routing first: the row tests what it says it tests
    assert [ix.hash_slots for ix in rc.indexes] == slots
    for mode, eng in zip(MODES, engines):
        for s in SAMPLERS:
            assert eng.link_kernel(s) == expected_kernel(row, s, mode), (row, s, mode)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 31, levels, attr_ids)
    np.testing.assert_array_equal(x, ox)
    _run_chain(oracle, engines, st, sampler, 4, row, "init")

    Vs = [ix.num_values for ix in rc.indexes]
    F = int(file.max()) + 1
    assert F >= 2
    rng = np.random.default_rng(5)
    starts = []
    if row.startswith("pruned"):
        for E in (HEAVY_MIN_CANDIDATES, HEAVY_MIN_CANDIDATES + 1):
            y, link, z = crafted_pruned_state(rng, x, E, Vs)
            cnt = survivors(x, z, y, link, np.zeros(E, np.int32))
            nmm, ns, nb = cnt[:, 0], cnt[:, 1], cnt[:, 2]
            # the branches of k_link_pruned the state is built for
            assert ((nmm > 0) & (ns > PRUNED_SCAP)).any()  # pass 2 walks the postings again
            assert ((nmm > 0) & (ns == 1)).any()           # single-survivor shortcut
            if E > HEAVY_MIN_CANDIDATES:
                assert ((nmm == 0) & (nb > HEAVY_MIN_CANDIDATES)).any()  # k_link_heavy
            else:
                assert ((nmm == 0) & (nb == HEAVY_MIN_CANDIDATES)).any()  # the whole block, still in k_link_pruned
            starts.append((y, link, z))
    else:
        for E in (x.shape[0], x.shape[0] // 3):
            starts.append(random_state(rng, x, E, Vs))
    for trial, (y, link, z) in enumerate(starts):
        theta = rng.uniform(0.01, 0.3, (len(Vs), F))
        for eng in engines:
            eng.upload_state(x, file, z, link, y, theta, iteration=5 * trial)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 5 * trial)
        _run_chain(oracle, engines, st, sampler, 2, row, f"state {trial}")
    for eng in engines:
        eng.close()


def test_link_mass_capture_calls(oracle):
    """capture is off by default, dbl_link_mass needs a sweep with it on, several sweeps in one call (a replayed CUDA
    graph) leave the last sweep's totals, and turning it off stops it"""
    import dblink_b200 as D

    from helpers import synth_problem

    g = synth_problem(seed=5, R=400, n_files=2)
    eng, rc, x, file = product_setup(g, 3, 1, (2,))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 3, 1, (2,))
    eng.sweep("PCG-II", 1)
    st.sweep(oracle.PCG_II)
    with pytest.raises(D.DblinkError):
        eng.link_mass()  # off by default
    eng.set_link_mass_capture(True)
    with pytest.raises(D.DblinkError):
        eng.link_mass()  # no sweep with the capture on yet
    for n in (1, 4):
        eng.sweep("PCG-I", n)  # 4 sweeps in one call replay a captured graph
        st.sweep(oracle.PCG_I, n)
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"{n} sweeps")
    eng.set_link_mass_capture(False)
    eng.sweep("PCG-II", 3)
    st.sweep(oracle.PCG_II, 3)
    assert_same_state(eng, st)
    with pytest.raises(D.DblinkError):
        eng.link_mass()
    eng.close()
