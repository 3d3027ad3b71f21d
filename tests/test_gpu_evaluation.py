"""Every posterior sample against the ground truth on the GPU (dbl_eval_* in dbl_posterior.cu, analysis_gpu.py)
against the numpy implementation in analysis_arrays.py: the per-sample counts (tp, pred_pairs, num_clusters) must be
exactly equal on random chains, on edge cases, on a 1 M-record chain and through Project.execute; every refusal leaves
the held counts as they were."""
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import chain_from_links, random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def assert_equal_to_numpy(ch, truth):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    got = ag.posterior_metric_counts(ch, truth)
    want = aa.posterior_metric_counts(ch, truth)
    for g, w in zip(got, want):
        assert g.dtype == np.int64 and np.array_equal(g, w)
    return got


@pytest.mark.parametrize("S", [1, 2, 7, 64])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    from dblink_b200 import analysis_gpu as ag

    ch = random_chain(R, S, seed=R * 7919 + S)
    # truth: the first sample's clusters with a fifth of the records moved, so the samples find some true pairs
    rng = np.random.default_rng(R + S)
    truth = ag.sample_clusters(R, *ch.samples[0][:2]).astype(np.int64)
    move = rng.random(R) < 0.2
    truth[move] = rng.integers(0, R, int(move.sum()))
    tp, pp, nc = assert_equal_to_numpy(ch, truth)
    assert (pp >= tp).all() and (nc >= 1).all()
    if R >= 40:
        assert tp[0] > 0 and (pp > tp).any() and (nc < R).all()
        if S > 2:
            assert len(set(tp)) > 1 and len(set(nc)) > 1


def test_edge_cases():
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    R = 1000
    truth = np.arange(R) // 3
    # all singletons: no predicted pair
    tp, pp, nc = assert_equal_to_numpy(chain_from_links([np.arange(R), np.arange(R)[::-1]]), truth)
    assert list(tp) == [0, 0] and list(pp) == [0, 0] and list(nc) == [R, R]
    # one cluster of every record: every true pair found
    tp, pp, nc = assert_equal_to_numpy(chain_from_links([np.zeros(R), np.full(R, 7)]), truth)
    assert list(tp) == [999] * 2 and list(pp) == [R * (R - 1) // 2] * 2 and list(nc) == [1, 1]
    # the truth itself, with labels that are not dense
    tp, pp, nc = assert_equal_to_numpy(chain_from_links([truth]), truth * 5 + 11)
    assert tp[0] == pp[0] == 999 and nc[0] == 334
    # no sample, no record
    empty = aa.ChainArrays(np.arange(0), np.zeros(0, np.int64), [])
    assert all(len(a) == 0 for a in ag.posterior_metric_counts(empty, np.zeros(0, np.int64)))


def million_chain():
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
    return aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples), base


def test_million_records():
    ch, last_base = million_chain()
    tp, pp, nc = assert_equal_to_numpy(ch, last_base)  # truth: the clustering the last samples move away from
    assert tp[0] < 10 and (pp[:-1] > tp[:-1]).all() and len(set(nc)) > 1
    assert tp[-1] == pp[-1] > 600_000 and nc[-1] == len(np.unique(last_base))  # the last sample is the truth
    # one cluster of all 1 M records in both: C(R, 2) pairs, beyond int32
    R = 1_000_000
    tp, pp, nc = assert_equal_to_numpy(chain_from_links([np.zeros(R, np.int32)]), np.zeros(R, np.int64))
    assert tp[0] == pp[0] == 499_999_500_000 and nc[0] == 1


def test_errors_leave_the_counts_as_they_were():
    import ctypes as C

    import torch

    from dblink_b200 import _lib, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    L = _lib.load()

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    def both(ev, labels):
        """status of add_sample on host labels, then on the same labels on the device"""
        host = L.dbl_eval_add_sample(ev._h, np.ascontiguousarray(labels, np.int32).ctypes.data)
        dev = torch.tensor(np.asarray(labels, np.int32), device="cuda")
        torch.cuda.synchronize()
        return host, L.dbl_eval_add_sample(ev._h, dev.data_ptr())

    R = 6
    truth = np.array([0, 0, 1, 1, 2, 3], np.int32)
    ev = ag.Evaluation(R, truth, 4)
    try:
        assert status(ev.read) == _lib.ERR_STATE                                    # no sample yet
        for bad in ([0, 0, 6, 3, 3, 3], [0, -1, 2, 3, 3, 3]):                        # label == R, negative label
            assert both(ev, bad) == (_lib.ERR_INVALID, _lib.ERR_INVALID)
        assert ev.num_samples == 0 and status(ev.read) == _lib.ERR_STATE
        assert both(ev, [0, 0, 0, 3, 4, 4]) == (_lib.OK, _lib.OK)                  # host and device: same counts
        assert both(ev, [0, 1, 2, 3, 4, 5]) == (_lib.OK, _lib.OK)
        held = ev.read()
        assert [list(a) for a in held] == [[1, 1, 0, 0], [4, 4, 0, 0], [3, 3, 6, 6]]
        assert both(ev, [0, 0, 2, 2, 4, 5]) == (_lib.ERR_INVALID, _lib.ERR_INVALID)  # beyond max_samples
        assert both(ev, [0, 0, 2, 2, 4, 6]) == (_lib.ERR_INVALID, _lib.ERR_INVALID)
        assert ev.num_samples == 4
        for a, b in zip(ev.read(), held):
            assert np.array_equal(a, b)
    finally:
        ev.close()
    # a bad true label: no object
    for bad in ([0, 0, 1, 1, 2, 6], [0, 0, 1, -1, 2, 3]):
        assert status(ag.Evaluation, R, np.array(bad, np.int32), 4) == _lib.ERR_INVALID
        h = C.c_void_p()
        dev = torch.tensor(bad, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert L.dbl_eval_create(C.byref(h), R, dev.data_ptr(), 4) == _lib.ERR_INVALID and not h
    # device truth: the same counts as host truth
    h = C.c_void_p()
    dev = torch.tensor(truth, device="cuda")
    torch.cuda.synchronize()
    assert L.dbl_eval_create(C.byref(h), R, dev.data_ptr(), 1) == _lib.OK and h
    try:
        assert L.dbl_eval_add_sample(h, np.array([0, 0, 0, 3, 4, 4], np.int32).ctypes.data) == _lib.OK
        out = [np.zeros(1, np.int64) for _ in range(3)]
        assert L.dbl_eval_read(h, *(a.ctypes.data_as(_lib.i64p) for a in out)) == _lib.OK
        assert [int(a[0]) for a in out] == [1, 4, 3]
    finally:
        L.dbl_eval_free(h)
    # the process keeps working
    assert_equal_to_numpy(random_chain(300, 9, seed=5), np.arange(300) // 2)


METRICS = '["pairwise", "cluster", "posterior-pairwise", "posterior-cluster"]'


def conf(out, metrics=METRICS, chains=1):
    c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                  sampler="PCG-I", cutoff=100)
    c = c.replace('metrics : ["pairwise", "cluster"]', "metrics : " + metrics)
    return c.replace("randomSeed : 319158", "randomSeed : 319158\n    numChains : %d" % chains)


def read(path):
    with open(path, "rb") as fh:
        return fh.read()


def copy_chains(src, dst, dirs):
    os.makedirs(dst)
    for d in dirs:
        shutil.copytree(os.path.join(src, d, "linkage-chain.parquet"), os.path.join(dst, d, "linkage-chain.parquet"))


def evaluate_only(out, monkeypatch, counts, metrics=METRICS, chains=1):
    from dblink_b200 import config, project
    from dblink_b200.project import Project

    monkeypatch.setattr(project, "posterior_metric_counts", counts)
    p = Project(config.parse_string(conf(out, metrics, chains)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] == "evaluate"]
    return p.execute(log=lambda *a: None)


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """RLdata500: the GPU counts write the same bytes as analysis_arrays from the same chain, and the sMPC sections
    are those of a run with the reference metrics only."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    gpu_dir, host_dir, ref_dir = (str(tmp_path / d) + "/" for d in ("gpu", "host", "ref"))
    calls = []
    real = ag.posterior_metric_counts
    monkeypatch.setattr(ag, "posterior_metric_counts", lambda ch, t: calls.append(1) or real(ch, t))
    res_gpu = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 1  # the platform choice took the GPU path
    rows = read(gpu_dir + "evaluation-samples.csv").decode().splitlines()
    assert rows[0] == "iteration,numClusters,TP,FP,FN,precision,recall,f1score,adjRandIndex" and len(rows) == 1 + 91
    assert [int(r.split(",")[0]) for r in rows[1:]] == list(range(100, 1001, 10))
    s = res_gpu["posterior-pairwise"]["f1score"]
    assert s["n"] == 91 and 0.5 < s["mean"] < 1 and s["sd"] > 0 and s["q025"] <= s["median"] <= s["q975"]
    assert res_gpu["posterior-cluster"]["trueNumClusters"] == 450

    copy_chains(gpu_dir, host_dir, ["."])
    res_host = evaluate_only(host_dir, monkeypatch, aa.posterior_metric_counts)
    assert len(calls) == 1 and res_host == res_gpu
    for f in ("evaluation-samples.csv", "evaluation-results.txt", "shared-most-probable-clusters.csv"):
        assert read(gpu_dir + f) == read(host_dir + f), f

    copy_chains(gpu_dir, ref_dir, ["."])
    evaluate_only(ref_dir, monkeypatch, project.posterior_metric_counts, '["pairwise", "cluster"]')
    ref = read(ref_dir + "evaluation-results.txt")
    assert read(gpu_dir + "evaluation-results.txt").startswith(ref)
    assert read(ref_dir + "shared-most-probable-clusters.csv") == read(gpu_dir + "shared-most-probable-clusters.csv")
    assert not os.path.exists(ref_dir + "evaluation-samples.csv")


def test_two_chains_pool_their_samples(tmp_path, monkeypatch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config
    from dblink_b200.project import Project

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.posterior_metric_counts
    monkeypatch.setattr(ag, "posterior_metric_counts", lambda ch, t: calls.append(1) or real(ch, t))
    res = Project(config.parse_string(conf(gpu_dir, chains=2)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # one call per chain
    per_chain = []
    for k in range(2):
        rows = read(gpu_dir + f"chain-{k}/evaluation-samples.csv").decode().splitlines()[1:]
        assert len(rows) == 91
        per_chain.append([float(r.split(",")[7]) for r in rows])
    assert per_chain[0] != per_chain[1]
    f1 = [x for xs in per_chain for x in xs if x == x]
    assert res["posterior-pairwise"]["f1score"]["n"] == len(f1) and res["posterior-pairwise"]["f1score"]["mean"] == \
        pytest.approx(np.mean(f1), rel=1e-12)
    assert " Samples:         182\n" in read(gpu_dir + "evaluation-results.txt").decode()
    assert not os.path.exists(gpu_dir + "evaluation-samples.csv")

    copy_chains(gpu_dir, host_dir, ["chain-0", "chain-1"])
    assert evaluate_only(host_dir, monkeypatch, aa.posterior_metric_counts, chains=2) == res
    for f in ("chain-0/evaluation-samples.csv", "chain-1/evaluation-samples.csv", "evaluation-results.txt",
              "shared-most-probable-clusters.csv"):
        assert read(gpu_dir + f) == read(host_dir + f), f
