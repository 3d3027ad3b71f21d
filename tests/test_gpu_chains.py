"""Batched chains: K chains of one model in one context (dbl_chains_*).

The invariant: chain k of a batch is bit-equal to a one-chain engine created with seed s_k and given the same
partition function (the tree fitted on chain 0's initial entity values) -- links, entity values, distortions, theta,
block ids, the integer summaries and every record's link mass; the log-likelihood (a floating-point sum in another
order) to 1e-9.  One chain k >= 1 is also checked against the CPU oracle run with seed s_k and that tree, which pins
the key and id mapping independently of the product.
"""
import math
import os

import numpy as np
import pytest

from helpers import assert_same_mass, encode, oracle_indexes, synth_problem

pytestmark = pytest.mark.gpu


def _model(g):
    import dblink_b200 as D

    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    x, file = rc.transform_records(g["values"], g["files"])
    alpha = [a.alpha for a in g["attributes"]]
    beta = [a.beta for a in g["attributes"]]
    return rc, x, file, alpha, beta


def chains_setup(g, seeds, levels, attr_ids, pop=0, singles=True):
    """-> (batch engine, [one-chain engine per seed], partitioner, records cache, x, file)"""
    import dblink_b200 as D

    rc, x, file, alpha, beta = _model(g)
    F = len(rc.file_ids)
    batch = D.GibbsEngine(rc.indexes, alpha, beta, None, seeds[0], F)
    batch.init_chains(x, file, pop, seeds)
    part = D.KDTreePartitioner(levels, list(attr_ids)).fit(batch.download_chains()[0]["y"])
    batch.set_partitioner(part)
    ones = []
    for s in (seeds if singles else ()):
        e = D.GibbsEngine(rc.indexes, alpha, beta, None, s, F)
        e.init_state(x, file, pop)
        e.set_partitioner(part)
        ones.append(e)
    return batch, ones, part, rc, x, file


def assert_chains_equal(batch, ones, chains=None, mass=False):
    ds = batch.download_chains()
    chains = range(len(ones)) if chains is None else chains
    for k, e in zip(chains, ones):
        d = e.download_state()
        for key in ("z", "link", "y", "theta", "block"):
            np.testing.assert_array_equal(ds[k][key], d[key], err_msg=f"chain {k} {key}")
        ps, os_ = batch.chain_summary(k), e.summary()
        assert ps["iteration"] == os_["iteration"]
        assert ps["num_isolates"] == os_["num_isolates"], f"chain {k}"
        np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"], err_msg=f"chain {k}")
        np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"], err_msg=f"chain {k}")
        np.testing.assert_array_equal(ps["theta"], os_["theta"], err_msg=f"chain {k}")
        assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9), f"chain {k}"
    if mass:
        m, R = batch.link_mass(), batch.num_records
        assert m.shape == (batch.num_chains * R,)
        for k, e in zip(chains, ones):
            assert_same_mass(m[k * R:(k + 1) * R], e.link_mass(), f"chain {k}")


# (link mode, graph mode): every link kernel eagerly, and the default kernels replayed from a captured graph
MODES = [(0, 1), (1, 1), (2, 1), (0, 2)]


@pytest.mark.parametrize("pop_extra", [0, 150])
@pytest.mark.parametrize("K", [2, 3])
@pytest.mark.parametrize("sampler", ["PCG-I", "PCG-II", "Gibbs"])
def test_every_chain_equals_its_one_chain_run(sampler, K, pop_extra):
    g = synth_problem(seed=5, R=450, n_files=2)
    R = len(g["values"])
    seeds = [77 + 1000 * k for k in range(K)]
    for link_mode, graph_mode in MODES:
        batch, ones, part, rc, x, file = chains_setup(g, seeds, 2, (2, 3), R + pop_extra if pop_extra else 0)
        assert batch.num_chains == K
        assert batch.num_records == R and batch.num_entities == R + pop_extra
        assert batch.num_partitions == K * part.num_partitions
        for e in [batch] + ones:
            e.set_link_mode(link_mode)
            e.set_graph_mode(graph_mode)
            e.set_link_mass_capture(True)
        assert batch.link_kernel(sampler) == ones[0].link_kernel(sampler)
        assert_chains_equal(batch, ones)
        for it in range(3):
            for e in [batch] + ones:
                e.sweep(sampler, 1)
            assert_chains_equal(batch, ones, mass=True)
        for e in [batch] + ones:  # several sweeps per call (a replayed graph in graph mode 2)
            e.sweep(sampler, 3)
        assert_chains_equal(batch, ones, mass=True)
        assert batch.iteration == 6
        for e in [batch] + ones:
            e.close()


def test_chain_one_against_the_oracle(oracle):
    """chain 1 of a batch against the oracle run with seed s_1 and the tree fitted on chain 0's initial values"""
    g = synth_problem(seed=9, R=500, n_files=2)
    seeds = [5, 123456789012345]
    levels, attr_ids = 2, (2, 3)
    batch, _, part, rc, x, file = chains_setup(g, seeds, levels, attr_ids, singles=False)
    idx = oracle_indexes(oracle, g)
    ox, ofile, F = encode(idx, g)
    np.testing.assert_array_equal(x, ox)
    alpha = [a.alpha for a in g["attributes"]]
    beta = [a.beta for a in g["attributes"]]
    m0 = oracle.Model(idx, alpha, beta, None, seeds[0], F)
    tree = oracle.KDTree.fit(oracle.State.init(m0, ox, ofile, 0).y, levels, list(attr_ids))
    m1 = oracle.Model(idx, alpha, beta, None, seeds[1], F)
    s1 = oracle.State.init(m1, ox, ofile, 0)
    m = oracle.Model(idx, alpha, beta, tree, seeds[1], F)
    st = oracle.State.from_arrays(m, ox, ofile, s1.z, s1.link, s1.y, s1.theta, 0)
    for sampler in ("PCG-II", "PCG-I", "Gibbs", "PCG-II"):
        batch.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        d = batch.download_chains()[1]
        for key in ("theta", "link", "y", "z", "block"):
            np.testing.assert_array_equal(d[key], getattr(st, key), err_msg=key)
        ps, os_ = batch.chain_summary(1), st.summary()
        assert ps["num_isolates"] == os_["num_isolates"]
        np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"])
        np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"])
        assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9)
    batch.close()


def _many_chains(indexes, alpha, beta, x, file, F, more_ids_than):
    """-> (batch, seeds): K chains on a 2-leaf tree, K just large enough that the PCG-I inverted index of the batch has
    more than `more_ids_than` (block, attribute, value) ids (K B sum_a V_a), while the B sum_a V_a ids of one chain fit
    the dense pointer table"""
    import dblink_b200 as D

    probe = D.GibbsEngine(indexes, alpha, beta, None, 1000, F)
    probe.init_state(x, file)
    part = D.KDTreePartitioner(1, [2]).fit(probe.download_state()["y"])
    probe.close()
    B = part.num_partitions
    sum_v = sum(ix.num_values for ix in indexes)
    assert B * sum_v <= (1 << 25)
    K = more_ids_than // (B * sum_v) + 2
    assert K * B * sum_v > more_ids_than
    seeds = list(range(1000, 1000 + K))
    batch = D.GibbsEngine(indexes, alpha, beta, None, seeds[0], F)
    batch.init_chains(x, file, 0, seeds)
    batch.set_partitioner(part)
    assert batch.num_partitions == K * B
    assert batch.link_kernel("PCG-I") == "k_link_pruned"
    return batch, seeds


def _equal_their_one_chain_runs(batch, seeds, indexes, alpha, beta, x, file, F, pop=0, part=None):
    """chains 0, 1, K/2 and K-1 of the batch against one-chain runs: with the batch's partitioner (part=None), or with
    `part` installed before the state is initialised, as it was on the batch"""
    import dblink_b200 as D

    K = len(seeds)
    check = [0, 1, K // 2, K - 1]
    ones = []
    for k in check:
        e = D.GibbsEngine(indexes, alpha, beta, None, seeds[k], F)
        if part is not None:
            e.set_partitioner(part)
        e.init_state(x, file, pop)
        if part is None:
            e.set_partitioner(batch.partitioner)
        ones.append(e)
    for n in (1, 2):
        for e in [batch] + ones:
            e.sweep("PCG-I", n)
        assert_chains_equal(batch, ones, chains=check)
    for e in ones:
        e.close()


def test_many_chains_take_the_wide_index_keys():
    """enough chains that the PCG-I inverted index has more (block, attribute, value) ids than its dense pointer table
    holds (K B sum_a V_a > 2^25): posting lists found by binary search in 32-bit ids"""
    g = synth_problem(seed=21, R=40, n_files=2)
    rc, x, file, alpha, beta = _model(g)
    F = len(rc.file_ids)
    batch, seeds = _many_chains(rc.indexes, alpha, beta, x, file, F, 1 << 25)
    _equal_their_one_chain_runs(batch, seeds, rc.indexes, alpha, beta, x, file, F)
    batch.close()


def test_many_chains_take_the_64_bit_index_keys():
    """a constant attribute with 2^22 values and enough chains that the (block, attribute, value) ids exceed 2^32:
    the batch sorts 64-bit ids and finds posting lists by binary search, each one-chain run uses the pointer table.
    Then the same context on one leaf with twice the entities: fewer than 2^32 ids, so 32-bit keys over twice the
    slots -- as many key bytes as before, and the index buffers must still be resized for the new slot count."""
    import dblink_b200 as D

    g = synth_problem(seed=21, R=40, n_files=2)
    rc, x, file, alpha, beta = _model(g)
    V = 1 << 22
    wide = D.AttributeIndex.from_tables(np.full(V, 1.0 / V), constant=True, expected_max_cluster_size=1)
    s1 = x[:, 3].astype(np.int64)  # duplicates that agree on s1 agree on the new attribute too
    x = np.ascontiguousarray(np.column_stack([x, np.where(s1 >= 0, (s1 * 40503 + 7) % V, -1)]), dtype=np.int32)
    indexes, alpha, beta, F = list(rc.indexes) + [wide], alpha + [alpha[0]], beta + [beta[0]], len(rc.file_ids)
    batch, seeds = _many_chains(indexes, alpha, beta, x, file, F, 1 << 32)
    _equal_their_one_chain_runs(batch, seeds, indexes, alpha, beta, x, file, F)
    K, R, sum_v = len(seeds), x.shape[0], sum(ix.num_values for ix in indexes)
    assert (1 << 25) < K * sum_v < (1 << 32)
    one_leaf = D.KDTreePartitioner(0, []).fit(batch.download_chains()[0]["y"])
    batch.set_partitioner(one_leaf)
    batch.init_chains(x, file, 2 * R, seeds)
    assert batch.num_partitions == K and batch.num_entities == 2 * R
    _equal_their_one_chain_runs(batch, seeds, indexes, alpha, beta, x, file, F, pop=2 * R, part=one_leaf)
    batch.close()


@pytest.mark.parametrize("sampler", ["PCG-I", "Gibbs"])
def test_zero_mass_in_one_chain_abandons_every_chain(sampler):
    """an invalid state in chain 1 only (record 0 undistorted on attribute 0, no entity carries its value): the sweep
    is abandoned for every chain -- state, theta and the shared iteration stay; a valid re-upload continues"""
    g = synth_problem(seed=13, R=400, n_files=1, missing=0.0)
    seeds = [8, 9]
    batch, ones, part, rc, x, file = chains_setup(g, seeds, 1, (2,))
    for e in [batch] + ones:
        e.sweep(sampler, 2)
    good = batch.download_chains()
    V0 = rc.indexes[0].num_values
    xv = int(x[0, 0])
    bad = {k: v.copy() for k, v in good[1].items()}
    bad["y"][bad["y"][:, 0] == xv, 0] = (xv + 1) % V0
    bad["z"][0, 0] = 0
    batch.upload_chains(x, file, [good[0], bad], seeds, iteration=2)
    with pytest.raises(ValueError, match="zero probability mass"):
        batch.sweep(sampler, 3)
    assert batch.iteration == 2
    after = batch.download_chains()
    for k, ref in ((0, good[0]), (1, bad)):
        for key in ("z", "link", "y", "theta"):
            np.testing.assert_array_equal(after[k][key], ref[key], err_msg=f"chain {k} {key}")
    batch.upload_chains(x, file, good, seeds, iteration=2)
    for e in [batch] + ones:
        e.sweep(sampler, 2)
    assert_chains_equal(batch, ones)
    for e in [batch] + ones:
        e.close()


def test_resume_through_upload_continues_every_chain():
    g = synth_problem(seed=3, R=300, n_files=2)
    seeds = [41, 42, 43]
    batch, ones, part, rc, x, file = chains_setup(g, seeds, 2, (2, 3), pop=350)
    for e in [batch] + ones:
        e.sweep("PCG-II", 2)
    saved, it = batch.download_chains(), batch.iteration
    batch.init_state(x, file)  # back to one chain ...
    assert batch.num_chains == 1 and batch.num_partitions == part.num_partitions
    batch.upload_chains(x, file, saved, seeds, iteration=it)  # ... and the three chains again
    assert batch.num_chains == 3
    for e in [batch] + ones:
        e.sweep("PCG-I", 2)
    assert_chains_equal(batch, ones)
    for e in [batch] + ones:
        e.close()


def test_refusals():
    import dblink_b200 as D
    from dblink_b200 import _lib

    g = synth_problem(seed=17, R=200, n_files=2)
    rc, x, file, alpha, beta = _model(g)
    F = len(rc.file_ids)
    eng = D.GibbsEngine(rc.indexes, alpha, beta, None, 1, F)
    with pytest.raises(ValueError):
        eng.init_chains(x, file, 0, [])  # K = 0
    with pytest.raises(ValueError):
        eng.init_chains(x, file, 0, [4, 5, 4])  # duplicate seeds
    xs = np.ascontiguousarray(x, np.int32)
    fs = np.ascontiguousarray(file, np.int32)
    L = _lib.load()
    assert L.dbl_chains_init(eng._h, 2, None, xs.shape[0], xs.ctypes.data_as(_lib.i32p), fs.ctypes.data_as(_lib.i32p),
                             0) == _lib.ERR_INVALID  # NULL seeds
    eng.init_chains(x, file, 0, [4, 5])
    st = eng.download_chains()
    far = {k: v.copy() for k, v in st[1].items()}
    far["link"][3] = len(st[1]["y"])  # outside chain 1
    with pytest.raises(ValueError):
        eng.upload_chains(x, file, [st[0], far], [4, 5])
    for call in (eng.download_state, eng.links, eng.summary, eng.state_hash, lambda: eng.sweep_by_block("PCG-I")):
        with pytest.raises(D.DblinkError):
            call()
    with pytest.raises(ValueError):
        eng.chain_summary(2)
    eng.sweep("PCG-I", 1)  # the refusals left the batch usable
    assert eng.iteration == 1
    eng.init_state(x, file)  # a one-chain context again: every one-chain call works
    eng.download_state()
    eng.summary()
    eng.close()
    sharded = D.GibbsEngine(rc.indexes, alpha, beta, None, 1, F, rank=0, world_size=2)
    with pytest.raises(ValueError):
        sharded.init_chains(x, file, 0, [1, 2])
    sharded.close()


def test_one_chain_must_use_the_model_seed():
    """num_chains = 1 is the one-chain context, keyed by the model's seed: another key is refused, not ignored"""
    import dblink_b200 as D

    g = synth_problem(seed=19, R=200, n_files=2)
    rc, x, file, alpha, beta = _model(g)
    F = len(rc.file_ids)
    eng = D.GibbsEngine(rc.indexes, alpha, beta, None, 5, F)
    with pytest.raises(ValueError):
        eng.init_chains(x, file, 0, [123])
    eng.init_chains(x, file, 0, [5])
    one = D.GibbsEngine(rc.indexes, alpha, beta, None, 5, F)
    one.init_state(x, file)
    part = D.KDTreePartitioner(1, [2]).fit(one.download_state()["y"])
    for e in (eng, one):
        e.set_partitioner(part)
        e.sweep("PCG-II", 2)
    assert eng.num_chains == 1
    st = eng.download_chains()
    with pytest.raises(ValueError):
        eng.upload_chains(x, file, st, [123], iteration=2)
    assert_chains_equal(eng, [one])
    eng.close()
    one.close()


def test_rldata500_project_with_three_chains(tmp_path, monkeypatch):
    """numChains = 3 end to end: chain 0 is the numChains = 1 run, the pooled sMPC / match probabilities of the GPU
    equal the numpy ones byte for byte, R̂ is written, and resuming continues all three chains exactly"""
    import shutil

    import pyarrow.parquet as pq

    from dblink_b200 import analysis_arrays as aa, config, project, state_io
    from dblink_b200.project import Project
    from test_host_pipeline import GOLDEN, make_conf

    def conf(out, n, resume, chains):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 1, '["fname_c1"]', sample_size=n, thinning=5,
                      cutoff=10)
        c = c.replace("resume : false", "resume : %s" % resume)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["cluster-size-distribution", "partition-sizes", "shared-most-probable-clusters", '
                      '"pairwise-match-probabilities"%s]' % (', "convergence-diagnostics"' if chains > 1 else ""))
        return c.replace("randomSeed : 319158", "randomSeed : 319158\n    numChains : %d" % chains)

    one, three, host = str(tmp_path / "one") + "/", str(tmp_path / "three") + "/", str(tmp_path / "host") + "/"
    Project(config.parse_string(conf(one, 12, "false", 1)), base_dir="").execute(log=lambda *a: None)
    p3 = Project(config.parse_string(conf(three, 12, "false", 3)), base_dir="")
    p3.execute(log=lambda *a: None)
    assert not os.path.exists(one + "chain-0")
    rows = lambda d: pq.read_table(d).sort_by([("iteration", "ascending")]).to_pylist()  # noqa: E731
    t1 = rows(one + "linkage-chain.parquet")
    t0 = rows(three + "chain-0/linkage-chain.parquet")
    key = lambda rs: sorted((r["iteration"], r["partitionId"], sorted(map(sorted, r["linkageStructure"])))  # noqa
                            for r in rs)
    assert key(t0) == key(t1)
    for k in range(3):
        for f in ("linkage-chain.parquet", "diagnostics.csv", "state.npz", "cluster-size-distribution.csv",
                  "partition-sizes.csv"):
            assert os.path.exists(os.path.join(three, f"chain-{k}", f)), (k, f)
    assert key(rows(three + "chain-1/linkage-chain.parquet")) != key(t0)
    # R̂ over the three chains
    lines = open(three + "convergence-diagnostics.csv").read().splitlines()
    assert lines[0] == "quantity,splitRhat,rankNormalizedSplitRhat,numChains,drawsPerChain"
    rh = {ln.split(",")[0]: ln.split(",") for ln in lines[1:]}
    for q in ("numObservedEntities", "logLikelihood"):
        assert math.isfinite(float(rh[q][1])) and math.isfinite(float(rh[q][2])) and rh[q][3] == "3", rh[q]
    # the pooled summaries from the numpy path: byte-identical files
    os.makedirs(host)
    for k in range(3):
        shutil.copytree(os.path.join(three, f"chain-{k}"), os.path.join(host, f"chain-{k}"))
    monkeypatch.setattr(project, "pairwise_match_counts", aa.pairwise_match_counts)
    monkeypatch.setattr(project, "shared_most_probable_clusters", aa.shared_most_probable_clusters)
    ph = Project(config.parse_string(conf(host, 12, "false", 3)), base_dir="")
    ph.steps = lambda: [s for s in Project.steps(ph) if s[0] != "sample"]
    ph.execute(log=lambda *a: None)
    for f in ("shared-most-probable-clusters.csv", "pairwise-match-probabilities.csv", "evaluation-results.txt"):
        assert open(three + f, "rb").read() == open(host + f, "rb").read(), f
    # resume: 6 samples + 6 more == 12 in one go, every chain
    part = str(tmp_path / "part") + "/"
    Project(config.parse_string(conf(part, 6, "false", 3)), base_dir="").execute(log=lambda *a: None)
    Project(config.parse_string(conf(part, 6, "true", 3)), base_dir="").execute(log=lambda *a: None)
    for k in range(3):
        a = state_io.load_state(os.path.join(three, f"chain-{k}"))
        b = state_io.load_state(os.path.join(part, f"chain-{k}"))
        assert a["iteration"] == b["iteration"] == 60
        for f in ("theta", "z", "link", "y"):
            np.testing.assert_array_equal(a[f], b[f], err_msg=f"chain {k} {f}")
        assert key(rows(os.path.join(three, f"chain-{k}", "linkage-chain.parquet"))) == \
            key(rows(os.path.join(part, f"chain-{k}", "linkage-chain.parquet")))
