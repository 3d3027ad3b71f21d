"""The Binder search on the GPU (dbl_pairs_binder_search in dbl_posterior.cu, analysis_gpu.binder_search) against the
numpy implementation in analysis_arrays.py: labels, round logs, convergence, n and K must be exactly equal on random
chains, on a 12 000-record cluster, on a 1 M-record chain and through Project.execute, for every cost and for start
labels in host and in device memory; a search never changes the held table or S, and neither does any refusal."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu

TS = (0.0, 0.25, 0.5, 0.7, 1.0)


def starts_of(ch):
    """A sample's labels and the sMPC's."""
    from dblink_b200 import analysis_arrays as aa

    mem, off, _ = ch.samples[len(ch.samples) // 2]
    return [aa.sample_labels(ch.num_records, mem, off), aa.shared_most_probable_clusters(ch)]


def assert_run_equal(g, w):
    assert g.labels.dtype == np.int64 and np.array_equal(g.labels, w.labels)
    for x, y in ((g.moves, w.moves), (g.dn, w.dn), (g.dK, w.dK)):
        assert x.dtype == np.int64 and np.array_equal(x, y)
    assert (g.converged, g.n, g.K) == (w.converged, w.n, w.K)


def assert_equal_to_numpy(ch, ts=TS, max_rounds=1000, starts=None):
    """The GPU search from every start at every t against numpy's, on one handle and one table; returns the runs."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    R, S = ch.num_records, len(ch.samples)
    first, second, count = aa.pairwise_match_counts(ch)
    starts = starts_of(ch) if starts is None else starts
    out = []
    with ag.Pairs(R) as pairs:
        ag._add_chain(pairs, ch)
        for t in ts:
            a, b = aa.search_cost(t)
            for st in starts:
                g = pairs.binder_search(a, b, st, max_rounds)
                w = aa.search_rounds(R, first, second, count, S, st, a, b, max_rounds)
                assert_run_equal(g, w)
                out.append(g)
    return out


@pytest.mark.parametrize("S", [1, 7, 64, 300])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    # at t = 0 everything connected merges, one record per cluster and round, so big chains are searched for a
    # bounded number of rounds (numpy takes about 2 s a round at R = 50 000, S = 300): equality over those rounds is
    # the same check
    big = R > 2500
    runs = assert_equal_to_numpy(random_chain(R, S, seed=R * 7919 + S), ts=(0.0, 0.5, 1.0) if big else TS,
                                 max_rounds=1000 if R <= 40 else 10 if big else 40)
    if R >= 40 and S > 1:  # a chain of one sample: that sample has loss 0, so no move lowers it
        assert sum(r.rounds for r in runs) > 0


def test_the_chosen_start_equals_numpy():
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    ch = random_chain(2500, 30, seed=11)
    for t in TS:
        g_best, g_runs = ag.binder_search(ch, t, starts_of(ch), 25)
        w_best, w_runs = aa.binder_search(ch, t, starts_of(ch), 25)
        assert g_best == w_best
        for g, w in zip(g_runs, w_runs):
            assert_run_equal(g, w)


def test_a_cluster_of_12000_records_next_to_small_ones():
    """From the sample holding the big cluster (72 M held pairs; numpy takes about 30 s a round), one round."""
    from dblink_b200 import analysis_arrays as aa
    from test_match_probabilities_host import random_chain as chain_with_big

    ch = chain_with_big(50_000, 3, seed=8, big=12_000)
    mem, off, _ = ch.samples[0]
    (run,) = assert_equal_to_numpy(ch, ts=(0.5,), max_rounds=1, starts=[aa.sample_labels(50_000, mem, off)])
    assert run.rounds == 1 and run.moves[0] > 1000


def test_million_records():
    """The chain of profiles/scripts/smpc_time.py (R = 1 M, 64 partitions), its first 30 samples."""
    from dblink_b200 import analysis_arrays as aa

    R, S = 1_000_000, 30
    rng = np.random.default_rng(12345)
    E = (3 * R) // 4
    blk = rng.integers(0, 64, E).astype(np.int32)
    base = rng.integers(0, E, R).astype(np.int32)
    samples = []
    for s in range(S):
        link = base.copy()
        move = rng.random(R) < 0.3
        link[move] = rng.integers(0, E, int(move.sum()))
        if s % 3 == 0:
            base = link
        samples.append(aa.sample_from_links(link, blk))
    runs = assert_equal_to_numpy(aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples),
                                 ts=(0.5, 0.7), max_rounds=5)
    assert all(r.rounds > 0 for r in runs)


def test_device_starts_and_refusals_leave_the_table_as_it_was():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    L = _lib.load()
    R = 40
    ch = random_chain(R, 9, seed=4)
    first, second, count = aa.pairwise_match_counts(ch)
    st = starts_of(ch)[1]
    a, b = aa.search_cost(0.5)

    def call(p, ptr, a=a, b=b, max_rounds=50):
        labels = np.full(R, -7, np.int32)
        logs = [np.full(max(max_rounds, 1), -7, np.int64) for _ in range(3)]
        rounds, conv, n, K = C.c_int32(-7), C.c_int32(-7), C.c_int64(-7), C.c_int64(-7)
        rc = L.dbl_pairs_binder_search(p._h, a, b, ptr, max_rounds, labels.ctypes.data, C.byref(rounds),
                                       C.byref(conv), *(x.ctypes.data_as(_lib.i64p) for x in logs), C.byref(n),
                                       C.byref(K))
        k = max(rounds.value, 0)
        return rc, aa.SearchRun(labels.astype(np.int64), *(x[:k] for x in logs), conv.value, n.value, K.value)

    with ag.Pairs(R) as p:
        host = np.ascontiguousarray(st, np.int32)
        assert call(p, host.ctypes.data)[0] == _lib.ERR_STATE  # no sample yet
        assert p.num_samples == 0
        ag._add_chain(p, ch)
        held = p.read()

        def unchanged():
            assert p.num_samples == 9
            for x, y in zip(p.read(), held):
                assert np.array_equal(x, y)

        want = aa.search_rounds(R, first, second, count, 9, st, a, b, 50)
        assert want.rounds > 0
        dev = torch.tensor(host, device="cuda")
        torch.cuda.synchronize()
        for ptr in (host.ctypes.data, dev.data_ptr()):
            rc, got = call(p, ptr)
            assert rc == _lib.OK
            assert_run_equal(got, want)
            unchanged()
        # refusals: labels outside [0, R), a cost outside 0 <= a <= b <= 2^16, max_rounds < 1
        for bad in (np.r_[host[:-1], R], np.r_[-1, host[1:]]):
            bad = np.ascontiguousarray(bad, np.int32)
            bad_dev = torch.tensor(bad, device="cuda")
            torch.cuda.synchronize()
            for ptr in (bad.ctypes.data, bad_dev.data_ptr()):
                assert call(p, ptr)[0] == _lib.ERR_INVALID
                unchanged()
        for kw in (dict(a=-1), dict(a=3, b=2), dict(b=0), dict(a=1, b=(1 << 16) + 1), dict(max_rounds=0)):
            assert call(p, host.ctypes.data, **kw)[0] == _lib.ERR_INVALID
            unchanged()
        # the search still works after the refusals, and adding a sample still works after the searches
        assert_run_equal(call(p, host.ctypes.data)[1], want)
        p.add_sample(np.zeros(R, np.int32))
        assert p.num_samples == 10


def test_the_size_bound_is_checked_before_the_device(monkeypatch):
    """S R < 2^44 is checked by both paths before any work (a chain of 2^44 record-samples is out of reach of a test;
    the ABI refuses it with DBL_ERR_INVALID by the same bound)."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    ch = random_chain(10, 4, seed=1)
    monkeypatch.setattr(aa, "MAX_SEARCH_SIZE", 40)
    for fn in (aa.binder_search, ag.binder_search):
        with pytest.raises(ValueError, match=r"samples x records < 2\^44"):
            fn(ch, 0.5, starts_of(ch))


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500: the GPU search writes the same bytes as analysis_arrays from the same
    chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["binder-search-clusters"], falseLinkCost : 0.7')
        return c.replace('metrics : ["pairwise", "cluster"]',
                         'metrics : ["binder-search-pairwise", "binder-search-cluster"], falseLinkCost : 0.7')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.binder_search
    monkeypatch.setattr(ag, "binder_search", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    gpu_res = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate
    names = ("binder-search-clusters.csv", "binder-search.csv", "evaluation-results.txt")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert gpu["binder-search.csv"].startswith(b"start,round,moves,linkedPairs,expectedLoss\nbinder-sample,0,0,")
    assert b"searched at 0.6999969482421875" in gpu["evaluation-results.txt"]

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    for name in ("binder_counts", "shared_most_probable_clusters", "binder_search"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    host_res = p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
    assert host_res == gpu_res and 0 < gpu_res["binder-search-pairwise"]["f1score"] <= 1
