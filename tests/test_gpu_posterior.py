"""Shared most probable clusters on the GPU (dbl_posterior.cu, analysis_gpu.py) against the numpy implementation in
analysis_arrays.py: labels and frequencies must be exactly equal, on random chains with repeated and tied modes, on
edge cases, on a chain large enough to need several record blocks, and through Project.execute."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu

PAIR_BLOCK = 1 << 26  # (signature, sample) pairs per record block in dbl_posterior.cu


def random_chain(R, S, seed):
    """ChainArrays of S samples over R records: samples share most clusters, so modes repeat and tie (the pattern of
    test_array_summaries_equal_the_set_based_ones)."""
    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(seed)
    E = max(1, (3 * R) // 4)
    blk = rng.integers(0, 4, E).astype(np.int32)
    base = rng.integers(0, E, R).astype(np.int32)
    samples = []
    for s in range(S):
        link = base.copy()
        move = rng.random(R) < 0.3
        link[move] = rng.integers(0, E, int(move.sum()))
        if s % 3 == 0:
            base = link
        samples.append(aa.sample_from_links(link, blk))
    return aa.ChainArrays(np.array(["r%d" % i for i in range(R)] if R <= 1000 else np.arange(R)),
                          np.arange(S, dtype=np.int64) * 10, samples)


def chain_from_links(links):
    from dblink_b200 import analysis_arrays as aa

    R = len(links[0])
    blk = np.zeros(R, np.int32)
    return aa.ChainArrays(np.arange(R), np.arange(len(links), dtype=np.int64),
                          [aa.sample_from_links(np.asarray(l, np.int32), blk) for l in links])


def assert_equal_to_numpy(ch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    labels, freq = ag.most_probable_clusters(ch)
    _, want_freq = aa.most_probable_signature(aa.cluster_signatures(ch))
    want_labels = aa.shared_most_probable_clusters(ch)
    assert labels.dtype == np.int64 and freq.dtype == np.float64
    assert np.array_equal(labels, want_labels)
    assert np.array_equal(freq, want_freq)
    assert np.array_equal(ag.shared_most_probable_clusters(ch), want_labels)
    return labels, freq


@pytest.mark.parametrize("R,S", [(1, 1), (1, 7), (2, 2), (6, 7), (40, 64), (300, 3000), (2500, 7), (50_000, 2),
                                 (50_000, 64), (4000, 3000)])
def test_random_chains_equal_numpy(R, S):
    ch = random_chain(R, S, seed=R * 7919 + S)
    labels, freq = assert_equal_to_numpy(ch)
    if S > 2 and R > 1:
        assert (freq < 1).any() and len(np.unique(labels)) > 1  # the chain has real choices to make


def test_edge_cases(tmp_path):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, writers as w

    # two equally frequent clusters: the one of the earlier sample wins (a and b together, c alone)
    ids = ["a", "b", "c"]
    blk = np.zeros(3, np.int32)
    path = os.path.join(tmp_path, "tie.parquet")
    lw = w.LinkageChainWriter(path)
    lw.append(0, w.linkage_structure_arrow(np.array([0, 0, 2], np.int32), blk, ids))   # {a,b} {c}
    lw.append(1, w.linkage_structure_arrow(np.array([0, 1, 1], np.int32), blk, ids))   # {a} {b,c}
    lw.close()
    ca = aa.read_chain_arrays(path)
    labels, freq = assert_equal_to_numpy(ca)
    got = {frozenset(c) for c in aa.labels_to_clusters(labels, ca.record_ids)}
    assert got == {frozenset("ab"), frozenset("c")}
    assert list(freq) == [0.5, 0.5, 0.5]
    # one record, one sample
    labels, freq = assert_equal_to_numpy(chain_from_links([[0]]))
    assert list(labels) == [0] and list(freq) == [1.0]
    # all singletons
    R = 1000
    labels, freq = assert_equal_to_numpy(chain_from_links([np.arange(R), np.arange(R)[::-1], np.arange(R)]))
    assert np.array_equal(labels, np.arange(R)) and (freq == 1.0).all()
    # one cluster of every record
    labels, freq = assert_equal_to_numpy(chain_from_links([np.zeros(R), np.full(R, 5)]))
    assert (labels == 0).all() and (freq == 1.0).all()
    # no sample, no record
    assert len(ag.shared_most_probable_clusters(aa.ChainArrays(np.arange(0), np.zeros(0, np.int64), []))) == 0


def test_million_records_several_blocks():
    R, S = 1_000_000, 100
    assert R * S > PAIR_BLOCK and R % (PAIR_BLOCK // S) != 0  # several blocks, the last one partial
    ch = random_chain(R, S, seed=2024)
    labels, freq = assert_equal_to_numpy(ch)
    assert len(np.unique(labels)) > R // 4 and (freq < 1).any()


def test_errors_leave_the_process_working():
    import torch

    from dblink_b200 import _lib, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    L = _lib.load()
    R = 5
    good = np.array([0, 0, 2, 3, 3], np.int32)

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    p = ag.Posterior(R, 2)
    try:
        assert status(p.smpc) == _lib.ERR_STATE                         # no sample yet
        for bad in ([0, 0, 5, 3, 3], [0, -1, 2, 3, 3]):                   # label == R, negative label
            assert status(p.add_sample, np.array(bad, np.int32)) == _lib.ERR_INVALID
            dev = torch.tensor(bad, dtype=torch.int32, device="cuda")    # the same check on device labels
            torch.cuda.synchronize()
            assert L.dbl_posterior_add_sample(p._h, dev.data_ptr()) == _lib.ERR_INVALID
        assert p.num_samples == 0
        p.add_sample(good)
        dev = torch.tensor(good, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert L.dbl_posterior_add_sample(p._h, dev.data_ptr()) == _lib.OK
        assert status(p.add_sample, good) == _lib.ERR_INVALID           # beyond max_samples
        assert p.num_samples == 2
        labels, freq = p.smpc()
        assert list(labels) == [0, 0, 2, 3, 3] and (freq == 1.0).all()
        assert L.dbl_posterior_smpc(p._h, None, None) == _lib.OK         # both outputs optional
    finally:
        p.close()
    assert status(ag.Posterior, 0, 1) == _lib.ERR_INVALID
    assert status(ag.Posterior, R, 0) == _lib.ERR_INVALID
    assert status(ag.Posterior, 1 << 30, 1 << 20) == _lib.ERR_CUDA        # an 8 PB signature matrix
    h = C.c_void_p()
    assert L.dbl_posterior_create(C.byref(h), 1 << 30, 1 << 20) == _lib.ERR_CUDA and not h
    # the process keeps working
    assert_equal_to_numpy(random_chain(300, 9, seed=5))


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize + evaluate on RLdata500: the GPU sMPC writes the same bytes as analysis_arrays from the same chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        return c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                         'quantities : ["cluster-size-distribution", "partition-sizes", '
                         '"shared-most-probable-clusters"]')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.shared_most_probable_clusters
    monkeypatch.setattr(ag, "shared_most_probable_clusters", lambda ch: calls.append(1) or real(ch))
    res_gpu = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate both took the GPU path

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "shared_most_probable_clusters", aa.shared_most_probable_clusters)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    res_host = p.execute(log=lambda *a: None)
    assert len(calls) == 2 and res_host == res_gpu
    for f in ("shared-most-probable-clusters.csv", "evaluation-results.txt", "cluster-size-distribution.csv",
              "partition-sizes.csv"):
        a, b = open(os.path.join(gpu_dir, f), "rb").read(), open(os.path.join(host_dir, f), "rb").read()
        assert len(a) > 0 and a == b, f
