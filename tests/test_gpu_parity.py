"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Bar: bit-exact links / entity values / distortion flags / block ids / theta / integer summaries;
log-likelihood (a floating-point diagnostic reduced in a different order) to 1e-9 relative.
"""
import numpy as np
import pytest

from helpers import assert_same_mass, oracle_setup, product_setup, random_state, synth_problem

pytestmark = pytest.mark.gpu

SAMPLERS = ["PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential"]


def assert_same_state(eng, st, check_ll=True):
    d = eng.download_state()
    np.testing.assert_array_equal(d["theta"], st.theta)
    np.testing.assert_array_equal(d["link"], st.link)
    np.testing.assert_array_equal(d["y"], st.y)
    np.testing.assert_array_equal(d["z"], st.z)
    np.testing.assert_array_equal(d["block"], st.block)
    ps, os_ = eng.summary(), st.summary()
    assert ps["iteration"] == os_["iteration"]
    assert ps["num_isolates"] == os_["num_isolates"]
    np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"])
    np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"])
    if check_ll:
        assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9)


@pytest.mark.parametrize("levels,attr_ids", [(0, ()), (2, (2, 3))])
def test_initial_state(oracle, levels, attr_ids):
    g = synth_problem(seed=3, R=700)
    eng, rc, x, file = product_setup(g, 1234, levels, attr_ids)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 1234, levels, attr_ids)
    np.testing.assert_array_equal(x, ox)
    assert eng.num_partitions == tree.n_leaves
    assert_same_state(eng, st)


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("sampler", SAMPLERS)
@pytest.mark.parametrize("levels,attr_ids", [(0, ()), (2, (2, 3))])
def test_chain_from_init(oracle, sampler, levels, attr_ids, mode):
    """mode 0 = default kernels (TMA-staged PCG-II, index-pruned PCG-I), 1 = generic fallback, 2 = dense TMA kernels for
    every sampler: identical draws"""
    g = synth_problem(seed=5, R=900, n_files=2)
    eng, rc, x, file = product_setup(g, 99, levels, attr_ids)
    eng.set_link_mode(mode)
    eng.set_link_mass_capture(True)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, levels, attr_ids)
    for it in range(6):
        eng.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same_state(eng, st)
        # the total mass of every record's categorical, not just the one draw taken from it
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"sweep {it}")
    # several sweeps in one call == the same sweeps one by one
    eng.sweep(sampler, 3)
    st.sweep(oracle.SAMPLERS[sampler], 3)
    assert_same_state(eng, st)
    assert_same_mass(eng.link_mass(), st.last_link_mass(), "3 sweeps in one call")


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_random_states(oracle, sampler):
    """single sweeps from random valid states: exercises clusters of many records, isolated entities,
    distorted/non-distorted mixtures, several files and blocks"""
    g = synth_problem(seed=11, R=500, n_files=3, missing=0.08, distortion=0.2)
    eng, rc, x, file = product_setup(g, 7, 3, (3, 2, 0))
    eng.set_link_mass_capture(True)
    m, st0, tree, ox, ofile = oracle_setup(oracle, g, 7, 3, (3, 2, 0))
    Vs = [ix.num_values for ix in rc.indexes]
    rng = np.random.default_rng(2024)
    for trial, E in enumerate([500, 60, 1200]):
        y, link, z = random_state(rng, x, E, Vs)
        theta = rng.uniform(0.005, 0.3, (len(Vs), 3))
        eng.upload_state(x, file, z, link, y, theta, iteration=10 * trial)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10 * trial)
        assert_same_state(eng, st)
        for it in range(2):
            eng.sweep(sampler, 1)
            assert st.sweep(oracle.SAMPLERS[sampler]) == 0
            assert_same_state(eng, st)
            assert_same_mass(eng.link_mass(), st.last_link_mass(), f"trial {trial} sweep {it}")


@pytest.mark.parametrize("sampler", ["PCG-I", "Gibbs", "Gibbs-Sequential"])
def test_records_without_a_must_match_attribute(oracle, sampler):
    """every observed attribute of a record distorted: nothing prunes its candidates, the whole block is scored.  In
    blocks beyond 256 entities the pruned kernel hands such records to k_link_heavy (a CTA per record); same draws"""
    g = synth_problem(seed=21, R=1500, n_files=2, missing=0.05, distortion=0.2)
    eng, rc, x, file = product_setup(g, 5)
    m, st0, tree, ox, ofile = oracle_setup(oracle, g, 5)
    Vs = [ix.num_values for ix in rc.indexes]
    rng = np.random.default_rng(77)
    for trial, E in enumerate([1500, 700]):
        y, link, z = random_state(rng, x, E, Vs)
        heavy = rng.choice(x.shape[0], 120, replace=False)
        z[heavy] = 1
        theta = rng.uniform(0.01, 0.3, (len(Vs), 2))
        eng.upload_state(x, file, z, link, y, theta, iteration=3 * trial)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 3 * trial)
        for mode in (0, 2):  # pruned + heavy kernels / dense kernel
            eng.upload_state(x, file, z, link, y, theta, iteration=3 * trial)
            eng.set_link_mode(mode)
            eng.sweep(sampler, 1)
            if mode == 0:
                assert st.sweep(oracle.SAMPLERS[sampler], 1) == 0
            assert_same_state(eng, st)
        eng.set_link_mode(0)
        eng.sweep(sampler, 2)
        assert st.sweep(oracle.SAMPLERS[sampler], 2) == 0
        assert_same_state(eng, st)


@pytest.mark.parametrize("pop", [150, 450, 1000])
def test_population_sizes(oracle, pop):
    """populationSize below / above the number of records (State.scala:221-250, 296-301)"""
    g = synth_problem(seed=21, R=450)
    eng, rc, x, file = product_setup(g, 5, 1, (2,), pop=pop)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 5, 1, (2,), pop=pop)
    assert eng.num_entities == pop
    assert_same_state(eng, st)
    for sampler in ("PCG-I", "PCG-II"):
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        assert_same_state(eng, st)


def test_large_cluster_beyond_cached_powers(oracle):
    """cluster sizes above expectedMaxClusterSize take the uncached base-distribution path
    (AttributeIndex.scala:197-205)"""
    g = synth_problem(seed=31, R=300, dup=0.0)
    eng, rc, x, file = product_setup(g, 17, 0, (), kmax=2)
    m, st0, tree, ox, ofile = oracle_setup(oracle, g, 17, 0, (), kmax=2)
    Vs = [ix.num_values for ix in rc.indexes]
    rng = np.random.default_rng(5)
    y, link, z = random_state(rng, x, 12, Vs)  # 300 records on 12 entities
    theta = np.full((len(Vs), 1), 0.05)
    for sampler in SAMPLERS:
        eng.upload_state(x, file, z, link, y, theta, 0)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
        eng.sweep(sampler, 1)
        st.sweep(oracle.SAMPLERS[sampler], 1)
        assert_same_state(eng, st)


def test_tiny_and_degenerate_inputs(oracle):
    from dblink_b200 import synth

    attrs = [synth.SynthAttr("s0", "levenshtein", 40, 1.0)]
    g = synth.generate(3, 1, attrs, dup=0.0, distortion=0.0, missing=0.0)
    eng, rc, x, file = product_setup(g, 1)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 1)
    for sampler in SAMPLERS:
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        assert_same_state(eng, st)
    # records with every attribute missing
    g = synth_problem(seed=8, R=64, missing=0.0)
    for r in range(0, 64, 5):
        g["values"][r] = [None] * len(g["values"][r])
    eng, rc, x, file = product_setup(g, 2, 1, (0,))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 2, 1, (0,))
    for sampler in SAMPLERS:
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        assert_same_state(eng, st)


def test_phase_times_add_up():
    """dbl_phase_ms: CUDA-event time of the eagerly enqueued sweeps by phase; the phases tile the sweep"""
    g = synth_problem(seed=4, R=2000)
    eng, rc, x, file = product_setup(g, 3, 2, (0, 1))
    eng.set_graph_mode(1)
    eng.sweep("PCG-II", 2)
    eng.phase_ms()
    eng.sweep("PCG-II", 5)
    ph, n = eng.phase_ms()
    assert n == 5
    assert ph["link"] > 0 and ph["values_distortions_summary"] > 0 and ph["relayout"] > 0
    assert ph["exchange"] < 0.05  # one rank: nothing to exchange
    assert sum(ph.values()) * n <= eng.last_sweep_ms() * 1.02
    assert sum(ph.values()) * n >= eng.last_sweep_ms() * 0.5
    assert eng.phase_ms()[1] == 0  # the call resets the accumulators


def test_error_conventions():
    import dblink_b200 as D

    g = synth_problem(seed=2, R=50)
    eng, rc, x, file = product_setup(g, 1)
    with pytest.raises(ValueError):
        eng.sweep(7, 1)
    bad = x.copy()
    bad[0, 0] = 10_000
    with pytest.raises(ValueError):
        eng.init_state(bad, file)
    eng2 = D.GibbsEngine(rc.indexes, [1.0] * 4, [1.0] * 4, None, 1, 1)
    with pytest.raises(D.DblinkError):
        eng2.sweep("PCG-I", 1)  # no state yet


def test_block_size_many_tiles(oracle):
    """one block spanning several 128-entity tiles and several draw chunks"""
    from dblink_b200 import synth

    attrs = [synth.SynthAttr("c0", "constant", 6, 0.5), synth.SynthAttr("s0", "levenshtein", 200, 1.0)]
    g = synth.generate(9, 2600, attrs, dup=0.2, distortion=0.1, missing=0.02)
    eng, rc, x, file = product_setup(g, 77)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 77)
    for sampler in ("PCG-II", "PCG-I"):
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        assert_same_state(eng, st)


def test_attribute_index_gpu_build_equals_host(monkeypatch):
    """the tiled bit-parallel Levenshtein kernel, the normalisation and the base-pmf kernels (csrc/dbl_index_gpu.cu)
    build the tables the host loops build, bit for bit"""
    import dblink_b200 as D
    from dblink_b200 import synth

    rng = np.random.default_rng(3)
    strings, _ = synth._string_vocab(rng, 1600)
    strings += ["", "A", "AB", "BB", "John Smith", "Jane Smith", "Zo\u00eb", "Zoe", "Jos\u00e9", "Jose", "x" * 64,
                "x" * 63 + "y", "ab" * 32, "ba" * 32, "a" * 33 + "b" * 31]
    vw = {s: float(1 + (i * 7919) % 13) for i, s in enumerate(dict.fromkeys(strings))}
    for thr in (7.0, 5.0, 0.0):
        monkeypatch.setenv("DBL_INDEX_GPU", "0")
        host = D.AttributeIndex.build(vw, "levenshtein", thr, 10.0).tables()
        monkeypatch.setenv("DBL_INDEX_GPU", "1")
        dev = D.AttributeIndex.build(vw, "levenshtein", thr, 10.0).tables()
        for k in ("phi", "norm", "rowptr", "col", "expsim"):
            np.testing.assert_array_equal(host[k], dev[k])
        if thr == 0.0:
            assert len(host["col"]) > 0.5 * len(vw) ** 2  # no truncation: nearly all pairs are "similar"
    # the chain that follows only sees the tables: a sweep with GPU-built and host-built indexes is the same sweep
    from helpers import synth_problem

    g = synth_problem(seed=2, R=300)
    states = []
    for flag in ("0", "1"):
        monkeypatch.setenv("DBL_INDEX_GPU", flag)
        rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
        x, file = rc.transform_records(g["values"], g["files"])
        eng = D.GibbsEngine(rc.indexes, [a.alpha for a in g["attributes"]], [a.beta for a in g["attributes"]], None, 5,
                            len(rc.file_ids))
        eng.init_state(x, file)
        eng.sweep("PCG-II", 3)
        states.append(eng.download_state())
        eng.close()
    for k in ("link", "y", "z", "theta"):
        np.testing.assert_array_equal(states[0][k], states[1][k])
    # a string longer than 64 bytes: the device path declines, the host loop builds the index
    vw2 = dict(list(vw.items())[:50])
    vw2["q" * 80] = 2.0
    monkeypatch.setenv("DBL_INDEX_GPU", "1")
    assert D.AttributeIndex.build(vw2, "levenshtein", 7.0, 10.0).num_values == 51


@pytest.mark.parametrize("n_const,n_str", [(1, 0), (0, 1), (3, 0), (0, 6), (7, 5), (8, 8), (14, 3)])
def test_model_shapes(oracle, n_const, n_str):
    """different (A, NS) instantiations of the unrolled PCG-II kernel, and A > 16 which takes the generic kernel"""
    from dblink_b200 import synth

    attrs = [synth.SynthAttr(f"c{i}", "constant", 5 + 3 * i, 0.5) for i in range(n_const)]
    attrs += [synth.SynthAttr(f"s{i}", "levenshtein", 60 + 10 * i, 1.0) for i in range(n_str)]
    # interleave so that kernel order (constants first) differs from attribute order
    attrs = attrs[::2] + attrs[1::2]
    g = synth.generate(40 + n_const, 400, attrs, dup=0.3, distortion=0.15, missing=0.05, n_files=2)
    levels = 1 if len(attrs) > 1 else 0
    eng, rc, x, file = product_setup(g, 3, levels, (len(attrs) - 1,) if levels else ())
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 3, levels, (len(attrs) - 1,) if levels else ())
    for sampler in ("PCG-II", "PCG-I", "Gibbs"):
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        assert_same_state(eng, st)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_sweep_block_by_block(oracle, sampler):
    """dbl_block_sweep_begin / dbl_update_block / dbl_block_sweep_end (the reference's per-partition task,
    GU:156-211): any block order gives the oracle's sweep; a block update only touches rows of that block."""
    g = synth_problem(seed=17, R=1100, n_files=2)
    eng, rc, x, file = product_setup(g, 7, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 7, 2, (2, 3))
    P = eng.num_partitions
    assert P == 4
    rng = np.random.default_rng(0)
    for it in range(4):
        eng.sweep_by_block(sampler, order=rng.permutation(P))
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same_state(eng, st)
    # one block at a time: rows outside the block keep their values
    from dblink_b200 import _lib
    from dblink_b200.engine import SAMPLERS as S, _check
    L = _lib.load()
    before = eng.download_state()
    _check(L.dbl_block_sweep_begin(eng._h, S[sampler]), "begin", eng._h)
    assert L.dbl_sweep(eng._h, S[sampler], 1) != 0           # no whole-sweep call inside an open block sweep
    _check(L.dbl_update_block(eng._h, 2), "update", eng._h)
    assert L.dbl_update_block(eng._h, 2) != 0                 # each block once
    assert L.dbl_update_block(eng._h, P) != 0
    assert L.dbl_block_sweep_end(eng._h) != 0                 # not every block was updated
    mid = eng.download_state()
    ent_in = before["block"] == 2
    rec_in = ent_in[before["link"]]
    np.testing.assert_array_equal(mid["y"][~ent_in], before["y"][~ent_in])
    np.testing.assert_array_equal(mid["link"][~rec_in], before["link"][~rec_in])
    np.testing.assert_array_equal(mid["z"][~rec_in], before["z"][~rec_in])
    assert ent_in[mid["link"][rec_in]].all()                   # links stay inside the block
    for b in (3, 0, 1):
        _check(L.dbl_update_block(eng._h, b), "update", eng._h)
    _check(L.dbl_block_sweep_end(eng._h), "end", eng._h)
    assert st.sweep(oracle.SAMPLERS[sampler]) == 0
    assert_same_state(eng, st)


def test_pruned_link_update_without_dense_pointers(oracle, monkeypatch):
    """PCG-I with the (block, attribute, value) pointer table disabled: posting lists found by binary search inside
    the (block, attribute) segments; same draws."""
    monkeypatch.setenv("DBL_INV_DENSE_MAX", "0")
    g = synth_problem(seed=21, R=1000, n_files=2)
    eng, rc, x, file = product_setup(g, 5, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 5, 2, (2, 3))
    for it in range(4):
        eng.sweep("PCG-I", 1)
        assert st.sweep(oracle.SAMPLERS["PCG-I"]) == 0
        assert_same_state(eng, st)


def test_pcg2_unpacked_constants_on_a_packable_model(oracle, monkeypatch):
    """k_link_pcg2 reads the constant attributes of a candidate as one byte-packed word when there are 1..4 of them
    with vocabularies <= 255; DBL_NO_PACK forces the per-attribute kernels on the same model: same draws."""
    monkeypatch.setenv("DBL_NO_PACK", "1")
    g = synth_problem(seed=23, R=900, n_files=2)
    eng, rc, x, file = product_setup(g, 11, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 11, 2, (2, 3))
    for it in range(4):
        eng.sweep("PCG-II", 1)
        assert st.sweep(oracle.SAMPLERS["PCG-II"]) == 0
        assert_same_state(eng, st)
