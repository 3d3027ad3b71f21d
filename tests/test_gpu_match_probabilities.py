"""Posterior pairwise match counts on the GPU (dbl_pairs_* in dbl_posterior.cu, analysis_gpu.py) against the numpy
implementation in analysis_arrays.py: (first, second, count) must be exactly equal on random chains, on edge cases
(no pairs, one large cluster, a sample of ~7e7 pairs), on a 1 M-record chain and through Project.execute; every
refusal leaves the held table as it was."""
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import chain_from_links, random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def assert_equal_to_numpy(ch, **kw):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    got = ag.pairwise_match_counts(ch, **kw)
    want = aa.pairwise_match_counts(ch, **kw)
    for g, w in zip(got, want):
        assert g.dtype == np.int64 and np.array_equal(g, w)
    return got


@pytest.mark.parametrize("S", [1, 2, 7, 64, 300])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    first, second, count = assert_equal_to_numpy(random_chain(R, S, seed=R * 7919 + S))
    if R >= 40:
        assert len(first) > 0 and count.max() <= S
        if S > 2:
            assert (count < S).any() and (count > 1).any()  # the chain both keeps and breaks pairs


def test_min_count_selects_on_the_device():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(2500, 64, seed=11)
    for t in (0.0, 0.5, 2 / 3, 1.0):
        f, _, c = assert_equal_to_numpy(ch, min_count=aa.min_match_count(t, 64))
        assert (c / 64 >= t).all() and (t > 0 or len(f) > 0)


def test_edge_cases():
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    R = 1000
    # all singletons: no pair
    first, _, _ = assert_equal_to_numpy(chain_from_links([np.arange(R), np.arange(R)[::-1]]))
    assert len(first) == 0
    # one cluster of 1 000 records in every sample: every pair, S times
    first, second, count = assert_equal_to_numpy(chain_from_links([np.zeros(R), np.full(R, 7), np.full(R, 999)]))
    assert len(first) == R * (R - 1) // 2 and (count == 3).all()
    assert np.array_equal(first * R + second, np.flatnonzero(np.triu(np.ones((R, R), bool), 1)))
    # no sample, no record
    empty = aa.ChainArrays(np.arange(0), np.zeros(0, np.int64), [])
    assert all(len(a) == 0 for a in ag.pairwise_match_counts(empty))


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    ch = chain_with_big(50_000, 3, seed=8, big=12_000)
    first, _, count = assert_equal_to_numpy(ch)
    assert len(first) > 12_000 * 11_999 // 2 and (count == 1).any() and (count > 1).any()


def test_million_records():
    """The chain of profiles/scripts/smpc_time.py: R = 1 M, 64 partitions, S = 100."""
    from dblink_b200 import analysis_arrays as aa

    R, S = 1_000_000, 100
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
    first, _, count = assert_equal_to_numpy(aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples))
    assert len(first) > R // 2 and (count == 1).any() and (count >= 10).any()


def test_errors_leave_the_held_pairs_as_they_were():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    L = _lib.load()

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    def both(p, labels):
        """status of add_sample on host labels, then on the same labels on the device"""
        host = L.dbl_pairs_add_sample(p._h, np.ascontiguousarray(labels, np.int32).ctypes.data)
        dev = torch.tensor(np.asarray(labels, np.int32), device="cuda")
        torch.cuda.synchronize()
        return host, L.dbl_pairs_add_sample(p._h, dev.data_ptr())

    R = 10
    p = ag.Pairs(R, 12)  # 12 distinct pairs at most
    try:
        assert status(p.count) == _lib.ERR_STATE and status(p.read) == _lib.ERR_STATE  # no sample yet
        for bad in ([0] * 9 + [10], [0, -1] + [2] * 8):                                 # label == R, negative label
            assert both(p, bad) == (_lib.ERR_INVALID, _lib.ERR_INVALID)
        assert both(p, [0] * 6 + list(range(6, 10))) == (_lib.ERR_INVALID, _lib.ERR_INVALID)  # 15 pairs alone
        assert p.num_samples == 0
        first = [0, 0, 0, 0, 4, 4, 4, 7, 8, 9]                                          # 6 + 3 pairs
        assert both(p, first) == (_lib.OK, _lib.OK)
        held = p.read()
        assert len(held[0]) == 9 and (held[2] == 2).all() and p.num_samples == 2
        # 12 pairs, 3 of them new: 12 distinct pairs fit; then a sample of 5 pairs, one of them new, does not
        assert both(p, [1, 1, 1, 1, 4, 4, 4, 4, 8, 9]) == (_lib.OK, _lib.OK)
        held = p.read()
        assert len(held[0]) == 12 and p.num_samples == 4
        assert sorted(held[2]) == [2] * 3 + [4] * 9
        assert both(p, [0, 0, 3, 3, 5, 5, 6, 6, 8, 8]) == (_lib.ERR_INVALID, _lib.ERR_INVALID)
        assert p.num_samples == 4 and p.count() == 12
        for a, b in zip(p.read(), held):
            assert np.array_equal(a, b)
        assert p.count(3) == 9 and p.count(5) == 0
        f, s, c = p.read(3)
        assert len(f) == 9 and (c == 4).all() and (f < s).all()
    finally:
        p.close()

    # one cluster of 70 000 records: 2.45e9 pairs, beyond int32; refused by the int64 count, nothing allocated
    R = 70_000
    p = ag.Pairs(R, (1 << 31) - 1)
    try:
        torch.cuda.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        assert both(p, np.zeros(R, np.int32)) == (_lib.ERR_INVALID, _lib.ERR_INVALID)
        assert torch.cuda.mem_get_info()[0] > free_before - (1 << 30)  # the keys alone would take 19.6 GB
        assert p.num_samples == 0
        p.add_sample(np.arange(R) // 2)
        assert p.count() == R // 2
    finally:
        p.close()

    # both paths raise the same ValueError for the cap
    ch = random_chain(300, 9, seed=5)
    n = len(aa.pairwise_match_counts(ch)[0])
    for fn in (aa.pairwise_match_counts, ag.pairwise_match_counts):
        with pytest.raises(ValueError, match=f"^the chain puts more than {n - 1} distinct record pairs in a cluster$"):
            fn(ch, max_pairs=n - 1)
        with pytest.raises(ValueError, match="more than 5 distinct"):
            fn(chain_from_links([np.zeros(4), np.zeros(4)]), max_pairs=5)
    # the process keeps working
    assert_equal_to_numpy(random_chain(300, 9, seed=6))
    assert len(assert_equal_to_numpy(ch, max_pairs=n)[0]) == n


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize on RLdata500: the GPU pairs write the same bytes as analysis_arrays from the same chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out, threshold):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        return c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                         'quantities : ["pairwise-match-probabilities", "shared-most-probable-clusters"], '
                         'minMatchProbability : %r' % threshold)

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.pairwise_match_counts
    monkeypatch.setattr(ag, "pairwise_match_counts", lambda ch, **kw: calls.append(1) or real(ch, **kw))
    Project(config.parse_string(conf(gpu_dir, 0.0)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 1
    name = "pairwise-match-probabilities.csv"
    gpu_all = open(os.path.join(gpu_dir, name), "rb").read()

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "pairwise_match_counts", aa.pairwise_match_counts)
    for t in (0.0, 0.37):
        p = Project(config.parse_string(conf(host_dir, t)), base_dir="")
        p.steps = lambda: [s for s in Project.steps(p) if s[0] == "summarize"]
        p.execute(log=lambda *a: None)
        host = open(os.path.join(host_dir, name), "rb").read()
        if t == 0.0:
            assert host == gpu_all
            lines = gpu_all.decode().splitlines()
            assert len(lines) > 1
        else:
            monkeypatch.setattr(project, "pairwise_match_counts", lambda ch, **kw: calls.append(1) or real(ch, **kw))
            q = Project(config.parse_string(conf(gpu_dir, t)), base_dir="")
            q.steps = lambda: [s for s in Project.steps(q) if s[0] == "summarize"]
            q.execute(log=lambda *a: None)
            assert len(calls) == 2 and open(os.path.join(gpu_dir, name), "rb").read() == host
            assert len(host.splitlines()) <= len(lines)
