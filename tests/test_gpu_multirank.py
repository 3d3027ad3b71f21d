"""The sharded chain on ONE GPU: 2-4 contexts ("ranks") of a single device in one process, one host thread each,
wired through dbl_comm_export / dbl_comm_import.  Every part of the multi-GPU data plane runs for real -- clusters
written into the destination rank's buffer, remote cursors, the flag barrier, summary slots, the device-side LPT --
so multi-rank parity with the oracle is checked wherever the GPU tests run, not only on a multi-GPU box
(tests/test_distributed.py has the one-process-per-GPU variant over NCCL-bootstrapped peers)."""
import numpy as np
import pytest

from helpers import oracle_setup, state_hash_numpy, synth_problem

pytestmark = pytest.mark.gpu


def make(world, g, seed, levels, split, **kw):
    import dblink_b200 as D
    from dblink_b200.distributed import LocalShards

    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    x, file = rc.transform_records(g["values"], g["files"])
    alpha = [a.alpha for a in g["attributes"]]
    beta = [a.beta for a in g["attributes"]]
    sh = LocalShards(rc.indexes, alpha, beta, seed=seed, num_files=len(rc.file_ids), levels=levels, split_attrs=split,
                     world=world)
    sh.init_state(x, file, **kw)
    return sh, rc, x, file


def assert_same(sh, st):
    d = sh.download_state()
    for k in ("theta", "link", "y", "z", "block"):
        np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=k)
    ps, os_ = sh.summary(), st.summary()
    assert ps["iteration"] == os_["iteration"] and ps["num_isolates"] == os_["num_isolates"]
    np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"])
    np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"])
    assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9)
    return d


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("sampler", ["PCG-II", "PCG-I", "Gibbs"])
def test_sharded_chain_equals_oracle(oracle, world, sampler):
    g = synth_problem(seed=5, R=1500, n_files=2)
    sh, rc, x, file = make(world, g, 99, 3, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, 3, (2, 3))
    moved = 0
    for it in range(4):
        sh.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same(sh, st)
        moved += sum(e for e, _, _ in sh.last_exchange())
    assert moved > 0, "clusters should move between ranks in this test"
    sh.sweep(sampler, 3)  # several sweeps per call: enqueued back to back on every rank, one barrier per sweep
    st.sweep(oracle.SAMPLERS[sampler], 3)
    d = assert_same(sh, st)
    # the rank-count-invariant fingerprint equals the one computed from the oracle's state
    from dblink_b200.engine import combine_state_hash

    he, hr = state_hash_numpy(st.y, st.link, st.z)
    assert sh.state_hash() == combine_state_hash(he, hr, st.theta, st.iteration)
    # resume from host arrays, keep following the oracle
    sh.upload_state(x, file, d["z"], d["link"], d["y"], d["theta"], iteration=sh.iteration)
    sh.sweep(sampler, 2)
    st.sweep(oracle.SAMPLERS[sampler], 2)
    assert_same(sh, st)
    sh.close()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("sampler", ["PCG-I", "Gibbs"])
def test_sharded_chain_without_dense_pointers(oracle, world, sampler, monkeypatch):
    """the pruned link update of every rank with the (block, attribute, value) pointer table disabled: posting lists
    found by binary search in the record's block range of the sorted index ids, eagerly and replayed from a captured
    graph (several sweeps per call); the chain is the oracle's"""
    monkeypatch.setenv("DBL_INV_DENSE_MAX", "0")
    g = synth_problem(seed=5, R=1500, n_files=2)
    sh, rc, x, file = make(world, g, 99, 3, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, 3, (2, 3))
    for it in range(4):
        sh.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same(sh, st)
    sh.sweep(sampler, 3)
    assert st.sweep(oracle.SAMPLERS[sampler], 3) == 0
    assert_same(sh, st)
    sh.close()


def test_device_side_replacement_keeps_the_chain(oracle):
    """blocks start on a deliberately bad placement (everything on rank 0); the LPT kernel re-places them from the
    global block sizes and the blocks migrate as cluster messages; the chain is the oracle's throughout"""
    g = synth_problem(seed=7, R=2000, n_files=2)
    sh, rc, x, file = make(3, g, 11, 3, (2, 3), owner=np.zeros(8, np.int32))
    sh.set_rebalance(2, 1.0)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 11, 3, (2, 3))
    assert (sh.block_owners() == 0).all()
    for it in range(6):
        sh.sweep("PCG-II", 1)
        st.sweep(oracle.SAMPLERS["PCG-II"])
        assert_same(sh, st)
    owners = sh.block_owners()
    assert len(set(owners.tolist())) == 3, owners
    assert all(c >= 1 for _, _, c in sh.last_exchange())  # every rank adopted the same new table
    # the placement the ranks agreed on balances records x entities
    d = sh.download_state()
    cost = np.bincount(d["block"], minlength=8) * np.bincount(d["block"][d["link"]], minlength=8)
    load = np.bincount(owners, weights=cost, minlength=3)
    assert load.max() <= 1.6 * load.mean()
    for e in sh.engines:  # and each rank holds exactly the rows of its blocks
        p = e.download_owned()
        assert (owners[p["block"]] == e_rank(e, sh)).all()
    sh.close()


def e_rank(e, sh):
    return sh.engines.index(e)


def test_state_hash_single_context_equals_oracle(oracle):
    from dblink_b200.engine import combine_state_hash
    from helpers import product_setup

    g = synth_problem(seed=3, R=800, n_files=2)
    eng, rc, x, file = product_setup(g, 21, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 21, 2, (2, 3))
    for sampler in ("PCG-II", "PCG-I"):
        eng.sweep(sampler, 2)
        st.sweep(oracle.SAMPLERS[sampler], 2)
        he, hr = eng.state_hash()
        assert (he, hr) == state_hash_numpy(st.y, st.link, st.z)
        s = eng.summary()
        assert combine_state_hash(he, hr, s["theta"], s["iteration"]) == \
            combine_state_hash(*state_hash_numpy(st.y, st.link, st.z), st.theta, st.iteration)
    eng.close()


def test_asynchronous_sweeps(oracle):
    """dbl_sweep_async enqueues, dbl_sync collects: same chain as blocking sweeps"""
    from helpers import product_setup

    g = synth_problem(seed=9, R=600, n_files=2)
    eng, rc, x, file = product_setup(g, 4, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 4, 2, (2, 3))
    eng.sweep_async("PCG-II", 3)
    eng.sweep_async("PCG-I", 2)
    with pytest.raises(Exception):
        eng.sweep("PCG-I", 1)  # blocking call with sweeps pending
    eng.sync()
    st.sweep(oracle.SAMPLERS["PCG-II"], 3)
    st.sweep(oracle.SAMPLERS["PCG-I"], 2)
    d = eng.download_state()
    for k in ("theta", "link", "y", "z", "block"):
        np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=k)
    assert eng.iteration == 5 == st.iteration
    eng.close()


@pytest.mark.parametrize("sampler", ["PCG-I", "Gibbs"])
def test_zero_mass_abandons_the_sweep(oracle, sampler):
    """a categorical without mass: the reference fails the task and there is no new state
    (IndexNonUniformDiscreteDist.scala:78-79) -- here the sweep is abandoned: links, values, flags, theta and the
    iteration are those before the call, the sweeps queued behind it are skipped, and the next valid call works"""
    from helpers import product_setup

    g = synth_problem(seed=13, R=400, n_files=1, missing=0.0)
    eng, rc, x, file = product_setup(g, 8, 1, (2,))
    m, st0, tree, ox, ofile = oracle_setup(oracle, g, 8, 1, (2,))
    eng.sweep(sampler, 2)
    st0.sweep(oracle.SAMPLERS[sampler], 2)
    good = eng.download_state()
    # an INVALID state: record 0 claims to be undistorted on attribute 0 but no entity carries its value there
    V0 = rc.indexes[0].num_values
    xv = int(x[0, 0])
    y = good["y"].copy()
    y[y[:, 0] == xv, 0] = (xv + 1) % V0
    z = good["z"].copy()
    z[0, 0] = 0
    eng.upload_state(x, file, z, good["link"], y, good["theta"], iteration=2)
    st = oracle.State.from_arrays(m, x, file, z, good["link"], y, good["theta"], 2)
    with pytest.raises(ValueError, match="zero probability mass"):
        eng.sweep(sampler, 3)
    assert st.sweep(oracle.SAMPLERS[sampler]) != 0
    after = eng.download_state()
    assert eng.iteration == 2 == st.iteration
    for k, ref in (("link", good["link"]), ("y", y), ("z", z), ("theta", good["theta"])):
        np.testing.assert_array_equal(after[k], ref, err_msg=k)
        np.testing.assert_array_equal(getattr(st, k), ref, err_msg="oracle " + k)
    # repaired state: the chain goes on
    eng.upload_state(x, file, good["z"], good["link"], good["y"], good["theta"], iteration=2)
    st = oracle.State.from_arrays(m, x, file, good["z"], good["link"], good["y"], good["theta"], 2)
    eng.sweep(sampler, 2)
    assert st.sweep(oracle.SAMPLERS[sampler], 2) == 0
    d = eng.download_state()
    for k in ("theta", "link", "y", "z"):
        np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=k)
    eng.close()


@pytest.mark.parametrize("sampler", ["PCG-II", "PCG-I", "Gibbs", "Gibbs-Sequential"])
def test_graph_replay_gives_the_same_chain(oracle, sampler):
    """several sweeps per call replay ONE captured CUDA graph of a sweep (every per-sweep quantity is read from device
    memory): same chain as kernel-by-kernel launches, for every link mode"""
    from helpers import product_setup

    g = synth_problem(seed=15, R=800, n_files=2)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 31, 2, (2, 3))
    engs = []
    for graph_mode, link_mode in ((2, 0), (1, 0), (2, 2), (2, 1)):
        eng, rc, x, file = product_setup(g, 31, 2, (2, 3))
        eng.set_graph_mode(graph_mode)
        eng.set_link_mode(link_mode)
        engs.append(eng)
    for n in (5, 1, 7):  # first call: 1 eager + capture + replays; later calls replay only
        st.sweep(oracle.SAMPLERS[sampler], n)
        for eng in engs:
            eng.sweep(sampler, n)
            d = eng.download_state()
            for k in ("theta", "link", "y", "z", "block"):
                np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=k)
            s, os_ = eng.summary(), st.summary()
            assert s["iteration"] == os_["iteration"] and s["num_isolates"] == os_["num_isolates"]
            np.testing.assert_array_equal(s["agg_dist"], os_["agg_dist"])
    # a new state of the same shape keeps the graphs; a new partitioner drops them
    d = engs[0].download_state()
    engs[0].upload_state(x, file, d["z"], d["link"], d["y"], d["theta"], iteration=engs[0].iteration)
    engs[0].sweep(sampler, 4)
    st.sweep(oracle.SAMPLERS[sampler], 4)
    np.testing.assert_array_equal(engs[0].download_state()["link"], st.link)
    for eng in engs:
        eng.close()


def test_graph_replay_on_a_sharded_chain(oracle):
    g = synth_problem(seed=5, R=1500, n_files=2)
    sh, rc, x, file = make(2, g, 99, 3, (2, 3))
    for e in sh.engines:
        e.set_graph_mode(2)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, 3, (2, 3))
    for n in (6, 3):
        sh.sweep("PCG-II", n)
        st.sweep(oracle.SAMPLERS["PCG-II"], n)
        assert_same(sh, st)
    sh.close()


def test_upload_state_keeps_the_records(oracle):
    """the records never change along a chain (the reference broadcasts its RecordsCache once): a state upload without
    them -- x = file = None, or the very same host arrays as before -- leaves them on the device"""
    from helpers import product_setup

    g = synth_problem(seed=19, R=700, n_files=2)
    eng, rc, x, file = product_setup(g, 6, 2, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 6, 2, (2, 3))
    eng.sweep("PCG-II", 2)
    st.sweep(oracle.SAMPLERS["PCG-II"], 2)
    d = eng.download_state()
    for how in ("none", "same-arrays", "same-arrays"):
        if how == "none":
            eng.upload_state(None, None, d["z"], d["link"], d["y"], d["theta"], iteration=eng.iteration)
        else:
            eng.upload_state(x, file, d["z"], d["link"], d["y"], d["theta"], iteration=eng.iteration)
        eng.sweep("PCG-I", 2)
        st.sweep(oracle.SAMPLERS["PCG-I"], 2)
        d = eng.download_state()
        for k in ("theta", "link", "y", "z", "block"):
            np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=how + " " + k)
    with pytest.raises(Exception):  # another population size needs the records again
        eng.upload_state(None, None, d["z"], d["link"], d["y"][:-1], d["theta"], iteration=0)
    eng.close()
