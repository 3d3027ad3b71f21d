"""The VI search and the expected VI of any labelling on the GPU (dbl_vi_search / dbl_vi_score in dbl_posterior.cu,
analysis_gpu.VI) against the numpy implementation in analysis_arrays.py: labels, rounds, convergence, moves, clusters,
dJ, J0 and the cell histograms must be exactly equal on random chains, on a 12 000-record cluster, under several batch
budgets, for start labels in host and in device memory, on a 1 M-record chain and through Project.execute; every
refusal returns its documented status and leaves the held samples usable."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def starts_of(ch):
    """A sample's labels, the sMPC's and all singletons."""
    from dblink_b200 import analysis_arrays as aa

    mem, off, _ = ch.samples[len(ch.samples) // 2]
    R = ch.num_records
    return [aa.sample_labels(R, mem, off), aa.shared_most_probable_clusters(ch), np.arange(R)]


def assert_run_equal(g, w):
    assert g.labels.dtype == np.int64 and np.array_equal(g.labels, w.labels)
    for x, y in ((g.moves, w.moves), (g.clusters, w.clusters), (g.dJ, w.dJ)):
        assert x.dtype == np.int64 and np.array_equal(x, y)
    assert (g.converged, g.J0, g.rounds) == (w.converged, w.J0, w.rounds)


def assert_equal_to_numpy(ch, max_rounds=1000, starts=None, batch_keys=None):
    """The GPU search and scores from every start against numpy's, on one handle; returns the GPU runs."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    R = ch.num_records
    table = aa.vi_search_table(R)
    host = aa.VISamples(ch)
    width = aa.vi_width(ch)
    out = []
    with ag.vi_samples(ch, batch_keys) as vi:
        for st in starts_of(ch) if starts is None else starts:
            g = vi.search(table, st, max_rounds)
            w = host.search(table, st, max_rounds)
            assert_run_equal(g, w)
            for lab in (st, g.labels):
                assert np.array_equal(vi.score(lab, width), host.score(lab, width))
            out.append(g)
    return out


@pytest.mark.parametrize("S", [1, 7, 64])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    runs = assert_equal_to_numpy(random_chain(R, S, seed=R * 7907 + S), max_rounds=1000 if R <= 2500 else 4)
    if R >= 40:
        assert sum(r.rounds for r in runs) > 0


def test_a_cluster_of_12000_records_next_to_small_ones():
    from dblink_b200 import analysis_arrays as aa
    from test_match_probabilities_host import random_chain as chain_with_big

    ch = chain_with_big(50_000, 3, seed=8, big=12_000)
    mem, off, _ = ch.samples[0]
    (run,) = assert_equal_to_numpy(ch, max_rounds=2, starts=[aa.sample_labels(50_000, mem, off)])
    assert run.rounds >= 1


@pytest.mark.parametrize("batch_keys", [1, 5000, 1 << 20])
def test_batch_budgets_do_not_change_the_result(batch_keys):
    """A budget of 1 key takes one sample per batch; 5000 a few; 2^20 every sample of the chain in one batch."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    ch = random_chain(2500, 30, seed=17)
    R = ch.num_records
    table = aa.vi_search_table(R)
    width = aa.vi_width(ch)
    with ag.vi_samples(ch) as one:
        want = [one.search(table, st, 50) for st in starts_of(ch)]
        want_cells = one.score(want[0].labels, width)
    with ag.vi_samples(ch, batch_keys) as vi:
        for st, w in zip(starts_of(ch), want):
            assert_run_equal(vi.search(table, st, 50), w)
        assert np.array_equal(vi.score(want[0].labels, width), want_cells)


def test_the_chosen_start_equals_numpy():
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    ch = random_chain(2500, 20, seed=11)
    g_best, g_runs = ag.vi_search(ch, starts_of(ch)[:2], 30)
    w_best, w_runs = aa.vi_search(ch, starts_of(ch)[:2], 30)
    assert g_best == w_best
    for g, w in zip(g_runs, w_runs):
        assert_run_equal(g, w)


def test_million_records():
    """The chain of test_gpu_vi.py's million-record test (R = 1 M, 20 samples), three rounds from two starts."""
    from dblink_b200 import analysis_arrays as aa

    R, S = 1_000_000, 20
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
    ch = aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples)
    runs = assert_equal_to_numpy(ch, max_rounds=3, starts=starts_of(ch)[:2], batch_keys=1 << 23)
    assert all(r.rounds > 0 for r in runs)


def test_device_starts_and_refusals_leave_the_samples_as_they_were():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    L = _lib.load()
    R = 40
    ch = random_chain(R, 9, seed=4)
    st = starts_of(ch)[1]
    table = aa.vi_search_table(R)
    width = aa.vi_width(ch)

    def call(v, ptr, step=table, max_rounds=50):
        step = np.ascontiguousarray(step, np.int64)
        labels = np.full(R, -7, np.int32)
        logs = [np.full(max(max_rounds, 1), -7, np.int64) for _ in range(3)]
        rounds, conv, J0 = C.c_int32(-7), C.c_int32(-7), C.c_int64(-7)
        rc = L.dbl_vi_search(v._h, step.ctypes.data_as(_lib.i64p), ptr, max_rounds, labels.ctypes.data,
                             C.byref(rounds), C.byref(conv), *(x.ctypes.data_as(_lib.i64p) for x in logs),
                             C.byref(J0))
        k = max(rounds.value, 0)
        return rc, aa.VISearchRun(labels.astype(np.int64), *(x[:k] for x in logs), conv.value, J0.value)

    with ag.VI(R, 10) as v:
        host = np.ascontiguousarray(st, np.int32)
        G = np.zeros(width, np.int64)
        assert call(v, host.ctypes.data)[0] == _lib.ERR_STATE  # no sample yet
        assert L.dbl_vi_score(v._h, host.ctypes.data, width, G.ctypes.data) == _lib.ERR_STATE
        ag._add_chain(v, ch)
        held = v.cross(width)

        def unchanged():
            assert v.num_samples == 9 and np.array_equal(v.cross(width), held)

        want = aa.VISamples(ch).search(table, st, 50)
        want_cells = aa.vi_label_cells(ch, st, width)
        assert want.rounds > 0
        dev = torch.tensor(host, device="cuda")
        torch.cuda.synchronize()
        for ptr in (host.ctypes.data, dev.data_ptr()):
            rc, got = call(v, ptr)
            assert rc == _lib.OK
            assert_run_equal(got, want)
            assert L.dbl_vi_score(v._h, ptr, width, G.ctypes.data) == _lib.OK and np.array_equal(G, want_cells)
            unchanged()
        # refusals: labels outside [0, R); a table with D_q[0] != 0, decreasing, or past the int64 bound; max_rounds < 1
        for bad in (np.r_[host[:-1], R], np.r_[-1, host[1:]]):
            bad = np.ascontiguousarray(bad, np.int32)
            bad_dev = torch.tensor(bad, device="cuda")
            torch.cuda.synchronize()
            for ptr in (bad.ctypes.data, bad_dev.data_ptr()):
                assert call(v, ptr)[0] == _lib.ERR_INVALID
                assert L.dbl_vi_score(v._h, ptr, width, G.ctypes.data) == _lib.ERR_INVALID
                unchanged()
        decreasing = table.copy()
        decreasing[5] = decreasing[4] - 1
        huge = np.full(R, 1 << 55, np.int64)
        huge[0] = 0
        for step in (table + 1, decreasing, huge):
            assert call(v, host.ctypes.data, step=step)[0] == _lib.ERR_INVALID
            unchanged()
        assert call(v, host.ctypes.data, max_rounds=0)[0] == _lib.ERR_INVALID
        assert L.dbl_vi_score(v._h, host.ctypes.data, width - 1, G.ctypes.data) == _lib.ERR_INVALID
        unchanged()
        # still working after the refusals, and a sample can still be added
        assert_run_equal(call(v, host.ctypes.data)[1], want)
        v.add_sample(np.zeros(R, np.int32))
        assert v.num_samples == 10


def test_the_squares_cap_is_refused_by_the_device():
    """A sample of one cluster of 16 385 records: 16 385^2 > 2^28.  The ABI refuses it, the held samples stay usable,
    and both Python paths raise the same ValueError first."""
    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    R = 16_385
    ch = aa.ChainArrays(np.arange(R), np.arange(2, dtype=np.int64),
                        [aa.sample_from_links(np.arange(R, dtype=np.int32), np.zeros(R, np.int32)),
                         aa.sample_from_links(np.zeros(R, np.int32), np.zeros(1, np.int32))])
    msg = f"^the VI search refuses sample 1: its clusters' squared sizes sum to {R * R}, more than {1 << 28}$"
    for fn in (aa.vi_search, ag.vi_search):
        with pytest.raises(ValueError, match=msg):
            fn(ch, [np.arange(R)])
    with ag.vi_samples(ch) as vi:
        with pytest.raises(ag.DblinkError) as e:
            vi.search(aa.vi_search_table(R), np.arange(R), 5)
        assert e.value.status == _lib.ERR_INVALID
        # the score has no such cap, and its buffers grow with the records in clusters of two or more only
        assert np.array_equal(vi.score(np.arange(R), R + 1), np.zeros(R + 1, np.int64))
        G = vi.score(np.zeros(R, np.int32), R + 1)
        assert G.tolist() == aa.vi_label_cells(ch, np.zeros(R), R + 1).tolist() and G[R] == 1
        assert vi.cross(R + 1).shape == (2, R + 1)


def test_the_score_of_a_sample_with_one_huge_cluster():
    """A sample holding one cluster of 150 000 of 200 000 records (sum of |K|^2 about 2.25e10): the score's cell pass
    takes one key per record in a cluster of two or more, so it needs memory linear in R and equals numpy, under the
    default budget and one sample per batch; the search refuses the sample."""
    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    R = 200_000
    rng = np.random.default_rng(31)
    huge = rng.integers(0, R // 3, R).astype(np.int32)
    huge[rng.permutation(R)[:150_000]] = R - 1
    ch = aa.ChainArrays(np.arange(R), np.arange(3, dtype=np.int64),
                        [aa.sample_from_links(l, np.zeros(R, np.int32))
                         for l in (rng.integers(0, R // 2, R).astype(np.int32), huge,
                                   rng.integers(0, R // 4, R).astype(np.int32))])
    width = aa.vi_width(ch)
    assert width == 150_001 and aa.vi_sample_squares(ch)[1] > 150_000 ** 2
    labellings = [aa.sample_labels(R, *ch.samples[1][:2]), rng.integers(0, R // 5, R), np.arange(R) // 2]
    want = [aa.vi_label_cells(ch, lab, width) for lab in labellings]
    for batch_keys in (None, 1):
        with ag.vi_samples(ch, batch_keys) as vi:
            for lab, w in zip(labellings, want):
                assert np.array_equal(vi.score(lab, width), w)
            with pytest.raises(ag.DblinkError) as e:
                vi.search(aa.vi_search_table(R), labellings[1], 5)
            assert e.value.status == _lib.ERR_INVALID
            assert np.array_equal(vi.score(labellings[2], width), want[2])  # still usable


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500: the GPU path writes the same bytes as the numpy path from the same chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["vi-search-clusters"]')
        return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["vi-search-pairwise", "vi-search-cluster"]')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.vi_samples
    monkeypatch.setattr(ag, "vi_samples", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    gpu_res = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate
    names = ("vi-search-clusters.csv", "vi-search.csv", "evaluation-results.txt")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert gpu["vi-search.csv"].startswith(b"start,round,moves,numClusters,expectedLoss\nvi-sample,0,0,")

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "shared_most_probable_clusters", aa.shared_most_probable_clusters)
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    host_res = p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
    assert host_res == gpu_res and 0 < gpu_res["vi-search-pairwise"]["f1score"] <= 1
