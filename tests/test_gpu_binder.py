"""The Binder-loss counts on the GPU (dbl_pairs_score_sample in dbl_posterior.cu, analysis_gpu.binder_counts) against
the numpy implementation in analysis_arrays.py: (n, K) per sample must be exactly equal on random chains, on a
12 000-record cluster, on a 1 M-record chain and through Project.execute; scoring never changes the held table, and
every refusal leaves it as it was."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def assert_equal_to_numpy(ch, **kw):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    got = ag.binder_counts(ch, **kw)
    want = aa.binder_counts(ch, **kw)
    for g, w in zip(got, want):
        assert g.dtype == np.int64 and g.shape == (len(ch.samples),) and np.array_equal(g, w)
    return got


@pytest.mark.parametrize("S", [1, 2, 7, 64, 300])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(R, S, seed=R * 7919 + S)
    n, K = assert_equal_to_numpy(ch)
    if R >= 40:
        _, _, count = aa.pairwise_match_counts(ch)
        assert int(n.sum()) == int(count.sum()) and int(K.sum()) == int((count ** 2).sum())
        assert (K >= n).all() and (n > 0).all()
        if S > 2:
            assert len(set(K.tolist())) > 1


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    n, K = assert_equal_to_numpy(chain_with_big(50_000, 3, seed=8, big=12_000))
    assert n[0] > 12_000 * 11_999 // 2 and K[0] >= n[0]


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
    n, K = assert_equal_to_numpy(aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples))
    assert (n > R // 2).all() and (K > n).all()


def test_scores_and_refusals_leave_the_table_as_it_was():
    import torch

    from dblink_b200 import _lib, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    L = _lib.load()

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    def both(p, labels):
        """(status, n, K) of score_sample on host labels, then on the same labels on the device"""
        out = []
        dev = torch.tensor(np.asarray(labels, np.int32), device="cuda")
        torch.cuda.synchronize()
        for ptr in (np.ascontiguousarray(labels, np.int32).ctypes.data, dev.data_ptr()):
            n, K = C.c_int64(-1), C.c_int64(-1)
            out.append((L.dbl_pairs_score_sample(p._h, ptr, C.byref(n), C.byref(K)), n.value, K.value))
        return out

    R = 10
    p = ag.Pairs(R, 12)  # 12 distinct pairs at most
    try:
        assert status(p.score_sample, np.zeros(R, np.int32)) == _lib.ERR_STATE  # no sample yet
        first = [0, 0, 0, 0, 4, 4, 4, 7, 8, 9]   # {0,1,2,3} {4,5,6}: 6 + 3 pairs
        second = [0, 0, 2, 2, 4, 4, 4, 7, 7, 9]  # (0,1) (2,3) (4,5) (4,6) (5,6) (7,8)
        p.add_sample(first)
        p.add_sample(second)
        held = p.read()
        assert len(held[0]) == 10 and p.num_samples == 2

        def unchanged():
            assert p.num_samples == 2
            for a, b in zip(p.read(), held):
                assert np.array_equal(a, b)

        # counts: (0,1) (2,3) (4,5) (4,6) (5,6) twice; (0,2) (0,3) (1,2) (1,3) (7,8) once
        assert both(p, first) == [(_lib.OK, 9, 5 * 2 + 4)] * 2
        assert both(p, second) == [(_lib.OK, 6, 5 * 2 + 1)] * 2
        unchanged()
        # labellings that are no sample: pairs the table does not hold count 0
        assert both(p, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9]) == [(_lib.OK, 0, 0)] * 2
        other = [1, 1, 1, 2, 3, 3, 6, 6, 9, 9]  # (0,1) (0,2) (1,2) (4,5) (6,7) (8,9): 2 + 1 + 1 + 2 + 0 + 0
        assert both(p, other) == [(_lib.OK, 6, 6)] * 2 and p.score_sample(np.array(other)) == (6, 6)
        unchanged()
        # refusals: a label == R, a negative label, and a labelling whose own pairs exceed the cap (45 > 12)
        for bad in ([0] * 9 + [10], [0, -1] + [2] * 8, [3] * R):
            assert [r[0] for r in both(p, bad)] == [_lib.ERR_INVALID] * 2
            unchanged()
        # 12 pairs exactly: scored
        assert both(p, [0, 0, 0, 0, 4, 4, 4, 4, 8, 9])[0][:2] == (_lib.OK, 12)
        unchanged()
        # adding still works after scores and refusals
        p.add_sample(first)
        assert p.num_samples == 3 and p.score_sample(first) == (9, 5 * 3 + 4 * 2)
    finally:
        p.close()

    # one cluster of 70 000 records: 2.45e9 pairs, refused by the int64 count before anything is allocated
    R = 70_000
    p = ag.Pairs(R, (1 << 31) - 1)
    try:
        p.add_sample(np.arange(R) // 2)
        torch.cuda.synchronize()
        free_before = torch.cuda.mem_get_info()[0]
        assert [r[0] for r in both(p, np.zeros(R, np.int32))] == [_lib.ERR_INVALID] * 2
        assert torch.cuda.mem_get_info()[0] > free_before - (1 << 30)
        assert p.num_samples == 1 and p.count() == R // 2
        assert p.score_sample(np.arange(R) // 2) == (R // 2, R // 2)
    finally:
        p.close()


def test_the_cap_refusal_is_the_numpy_one():
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    ch = random_chain(300, 9, seed=5)
    n = len(aa.pairwise_match_counts(ch)[0])
    for fn in (aa.binder_counts, ag.binder_counts):
        with pytest.raises(ValueError, match=f"^the chain puts more than {n - 1} distinct record pairs in a cluster$"):
            fn(ch, max_pairs=n - 1)
    assert_equal_to_numpy(ch, max_pairs=n)


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500: the GPU counts write the same bytes as analysis_arrays from the same
    chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["binder-clusters"], falseLinkCost : 0.7')
        return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["binder-pairwise", "binder-cluster"]')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.binder_counts
    monkeypatch.setattr(ag, "binder_counts", lambda ch, **kw: calls.append(1) or real(ch, **kw))
    gpu_res = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate
    names = ("binder-clusters.csv", "binder-loss.csv", "evaluation-results.txt")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert len(gpu["binder-loss.csv"].splitlines()) > 50

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "binder_counts", aa.binder_counts)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    host_res = p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
    assert host_res == gpu_res and 0 < gpu_res["binder-pairwise"]["f1score"] <= 1
