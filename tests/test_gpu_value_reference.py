"""GPU: the tables behind the entity-value draws, and sweeps over clusters large enough that the draws rescale.

The device-built base pmfs (k_base_pmfs, k_sim_norms: the default for V >= 2048) equal the host-built ones and the
oracle's bit for bit, including the rows whose weights underflow; sweeps from states holding the crafted clusters of
tests/test_value_reference.py equal the oracle's, through both k_values instantiations and a batch of two chains.
"""
import numpy as np
import pytest

from test_gpu_parity import SAMPLERS, assert_same_state
from test_value_reference import crafted_specs, crafted_state

pytestmark = pytest.mark.gpu

TABLES = ("phi", "norm", "invnorm", "pk", "cdf", "logphi", "lognorm", "rowptr", "col", "expsim")


def vocabulary(V):
    from dblink_b200 import synth

    strings, _ = synth._string_vocab(np.random.default_rng(V), V + 64)
    strings = list(dict.fromkeys(strings))[:V]
    assert len(strings) == V
    return {s: float(1 + (i * 7919) % 13) for i, s in enumerate(strings)}


@pytest.mark.parametrize("similarity", ["levenshtein", "jaro-winkler", "constant"])
def test_index_tables_device_host_and_oracle(oracle, monkeypatch, similarity):
    """DBL_INDEX_GPU=1 against =0 (and unset at V = 2048) against the oracle's index (Levenshtein and constant), every
    table bit for bit, for vocabulary sizes around the warp and block widths and kmax up to 300 (rows that underflow)"""
    import dblink_b200 as D

    for V in (1, 31, 32, 33, 127, 128, 129, 2047, 2048):
        vw = vocabulary(V)
        for kmax in ((0, 1, 10, 300) if V < 2048 else (300,)):
            got = {}
            for flag in (("0", "1") if V < 2048 else ("0", None)):
                if flag is None:
                    monkeypatch.delenv("DBL_INDEX_GPU", raising=False)
                else:
                    monkeypatch.setenv("DBL_INDEX_GPU", flag)
                got[flag] = D.AttributeIndex.build(vw, similarity, 7.0, 10.0, kmax).tables()
            host, dev = got.values()
            what = f"{similarity} V={V} kmax={kmax}"
            for k in TABLES:
                np.testing.assert_array_equal(host[k], dev[k], err_msg=f"{what} {k}")
            assert np.isfinite(host["pk"]).all(), what
            if similarity != "jaro-winkler":
                ix = oracle.Index.build(vw, similarity == "constant", 7.0, 10.0, kmax)
                for k in ("phi", "norm", "invnorm", "pk", "cdf", "rowptr", "col", "expsim"):
                    np.testing.assert_array_equal(host[k], getattr(ix, k), err_msg=f"{what} {k} (oracle)")


def crafted_setup(oracle, pad=0, sizes=None, seeds=(99,)):
    """engine + oracle models of the crafted attributes and a state holding every crafted cluster; pad isolated
    entities whose constant value (t) puts them in a block of their own"""
    import dblink_b200 as D

    specs, picks = crafted_specs(oracle)
    kw = {} if sizes is None else {"sizes": sizes}
    x, file, z, link, y, theta, info = crafted_state(picks, **kw)
    if pad:
        yp = np.zeros((pad, y.shape[1]), np.int32)
        yp[:, 3] = 4
        y = np.concatenate([y, yp])
    F = theta.shape[1]
    A = len(specs)
    oix = [oracle.Index.build(vw, const, 7.0, 10.0, kmax) for vw, const, kmax in specs]
    dix = [D.AttributeIndex.build(vw, "constant" if const else "levenshtein", 7.0, 10.0, kmax)
           for vw, const, kmax in specs]
    tree = oracle.KDTree.fit(y, 1, [3])
    part = D.KDTreePartitioner(1, [3]).fit(y)
    models = [oracle.Model(oix, [1.0] * A, [4.0] * A, tree, s, F) for s in seeds]
    return dix, part, models, (x, file, z, link, y, theta), info


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_crafted_clusters_sweep_like_the_oracle(oracle, sampler):
    """two sweeps from a state of 81 crafted clusters (1 to 300 records) in two blocks: k_values<8>"""
    import dblink_b200 as D

    dix, part, (m,), st_arrays, info = crafted_setup(oracle)
    x, file, z, link, y, theta = st_arrays
    eng = D.GibbsEngine(dix, m.alpha, m.beta, None, m.seed, m.F)
    eng.set_partitioner(part)
    eng.upload_state(x, file, z, link, y, theta, 0)
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    assert len(set(st.block.tolist())) == 2
    assert_same_state(eng, st)
    for _ in range(2):
        eng.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same_state(eng, st)
    eng.close()


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_crafted_clusters_among_isolated_entities(oracle, sampler):
    """the largest crafted clusters with 300 000 isolated entities: E * A beyond sm_count * 8192, so k_values<2>"""
    import dblink_b200 as D

    dix, part, (m,), st_arrays, info = crafted_setup(oracle, pad=300_000, sizes=[2, 55, 91, 300])
    x, file, z, link, y, theta = st_arrays
    eng = D.GibbsEngine(dix, m.alpha, m.beta, None, m.seed, m.F)
    eng.set_partitioner(part)
    eng.upload_state(x, file, z, link, y, theta, 0)
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    blk = st.block  # the clusters' entities come first; the isolated ones fill a block of their own
    assert not set(blk[:len(info)].tolist()) & set(blk[len(info):].tolist())
    eng.sweep(sampler, 1)
    assert st.sweep(oracle.SAMPLERS[sampler]) == 0
    assert_same_state(eng, st)
    eng.close()


def test_crafted_clusters_in_a_batch_of_two_chains(oracle):
    """K = 2 chains from the same crafted state: chain k equals the oracle run with seed s_k"""
    import dblink_b200 as D

    seeds = (99, 1099)
    dix, part, models, st_arrays, info = crafted_setup(oracle, sizes=[1, 11, 55, 140], seeds=seeds)
    x, file, z, link, y, theta = st_arrays
    eng = D.GibbsEngine(dix, models[0].alpha, models[0].beta, None, seeds[0], models[0].F)
    eng.set_partitioner(part)
    state = {"z": z, "link": link, "y": y, "theta": theta}
    eng.upload_chains(x, file, [state, state], list(seeds))
    for sampler in ("PCG-I", "Gibbs"):
        eng.sweep(sampler, 1)
        got = eng.download_chains()
        for k, m in enumerate(models):
            st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
            assert st.sweep(oracle.SAMPLERS[sampler]) == 0
            for key in ("link", "y", "z", "theta", "block"):
                np.testing.assert_array_equal(got[k][key], getattr(st, key), err_msg=f"{sampler} chain {k} {key}")
        eng.upload_chains(x, file, [state, state], list(seeds))
    eng.close()
