"""The variation-of-information cell histograms on the GPU (dbl_vi_* in dbl_posterior.cu,
analysis_gpu.vi_cross_histograms) against the numpy implementation in analysis_arrays.py: G must be exactly equal on
random chains, on a 12 000-record cluster, on a 1 M-record chain in several batches per sample and through
Project.execute; every refusal returns its documented status and leaves the held samples usable."""
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

    got = ag.vi_cross_histograms(ch, **kw)
    want = aa.vi_cross_histograms(ch)
    assert got.dtype == np.int64 and got.shape == want.shape and np.array_equal(got, want)
    return got


@pytest.mark.parametrize("S", [1, 2, 7, 64])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    G = assert_equal_to_numpy(random_chain(R, S, seed=R * 7919 + S))
    assert (G[:, :2] == 0).all()
    if R >= 40 and S >= 2:
        assert G[:, 2].sum() > 0


def test_small_batches_equal_numpy():
    """One sort per sample s, and batches that leave a remainder."""
    ch = random_chain(2500, 20, seed=3)
    want = assert_equal_to_numpy(ch)
    for keys in (1, 3000, 7 * 1800):
        assert np.array_equal(assert_equal_to_numpy(ch, batch_keys=keys), want)


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    G = assert_equal_to_numpy(chain_with_big(50_000, 3, seed=8, big=12_000))
    assert G.shape[1] > 12_000


def test_million_records_in_several_batches():
    """The chain of profiles/scripts/smpc_time.py (R = 1 M, 64 partitions), its first 20 samples, with a batch of
    2^21 keys: about 736 000 records of every sample are in clusters of two or more, so each t takes several
    batches."""
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
    big = (np.bincount(aa.sample_labels(R, *samples[0][:2]), minlength=R)[aa.sample_labels(R, *samples[0][:2])] >= 2)
    assert 3 * int(big.sum()) > 1 << 21  # at least three batches for t = 0
    G = assert_equal_to_numpy(ch, batch_keys=1 << 21)
    assert (G[:, 2] > R // 10).all()


def test_refusals_leave_the_held_samples_usable():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    L = _lib.load()

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    def add_both(v, labels):
        """status of add_sample on host labels, then on the same labels on the device"""
        dev = torch.tensor(np.asarray(labels, np.int32), device="cuda")
        torch.cuda.synchronize()
        return [L.dbl_vi_add_sample(v._h, ptr) for ptr in (np.ascontiguousarray(labels, np.int32).ctypes.data,
                                                           dev.data_ptr())]

    R = 8
    links = [[0, 0, 1, 1, 1, 5, 6, 7], [0, 1, 2, 2, 4, 4, 4, 4], [0, 0, 2, 2, 4, 4, 6, 6]]
    ch = aa.ChainArrays(np.arange(R), np.arange(3, dtype=np.int64),
                        [aa.sample_from_links(np.array(l, np.int32), np.zeros(R, np.int32)) for l in links])
    want = aa.vi_cross_histograms(ch)
    v = ag.VI(R, 3)
    try:
        assert status(v.cross, 5) == _lib.ERR_STATE and v.num_samples == 0  # reading before any sample
        v.add_sample(links[0])
        # a bad label: a label == R, a negative one; nothing is added
        for bad in ([0] * 7 + [8], [0, -1] + [2] * 6):
            assert add_both(v, bad) == [_lib.ERR_INVALID] * 2 and v.num_samples == 1
        assert add_both(v, links[1]) == [_lib.OK, _lib.OK] and v.num_samples == 3
        # a sample beyond max_samples
        assert status(v.add_sample, links[2]) == _lib.ERR_INVALID and v.num_samples == 3
        # width too small: M = 4, so 5 is the least width
        assert status(v.cross, 4) == _lib.ERR_INVALID
        assert status(v.cross, 0) == _lib.ERR_INVALID
        assert status(v.set_batch_keys, 0) == _lib.ERR_INVALID
        got = v.cross(5)
        two = aa.ChainArrays(np.arange(R), np.arange(3, dtype=np.int64), [ch.samples[0], ch.samples[1], ch.samples[1]])
        assert np.array_equal(got, aa.vi_cross_histograms(two))
        assert np.array_equal(v.cross(9)[:, :5], got) and not v.cross(9)[:, 5:].any()
        # device output
        G = torch.zeros((3, 5), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        assert L.dbl_vi_cross(v._h, 5, G.data_ptr()) == _lib.OK
        assert np.array_equal(G.cpu().numpy(), got) and v.num_samples == 3
    finally:
        v.close()
    # a fresh handle with every sample of the chain gives the numpy histograms
    with ag.VI(R, 3) as v:
        for l in links:
            v.add_sample(l)
        assert np.array_equal(v.cross(want.shape[1]), want)


def test_the_cap_refusal_is_the_numpy_one(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag
    from test_vi_host import giant_chain

    for fn in (aa.vi_cross_histograms, ag.vi_cross_histograms):
        with pytest.raises(ValueError, match=r"^the VI histograms need 256 x 1048577 entries, more than 268435456$"):
            fn(giant_chain())
    ch = random_chain(300, 9, seed=5)
    width = aa.vi_width(ch)
    monkeypatch.setattr(aa, "MAX_VI_ENTRIES", 9 * width - 1)
    for fn in (aa.vi_cross_histograms, ag.vi_cross_histograms):
        with pytest.raises(ValueError, match="^the VI histograms need 9 x"):
            fn(ch)


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500: the GPU histograms write the same bytes as analysis_arrays from the same
    chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]', 'quantities : ["vi-clusters"]')
        return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["vi-pairwise", "vi-cluster"]')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.vi_cross_histograms
    monkeypatch.setattr(ag, "vi_cross_histograms", lambda ch, **kw: calls.append(1) or real(ch, **kw))
    gpu_res = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate
    names = ("vi-clusters.csv", "vi-loss.csv", "evaluation-results.txt")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert len(gpu["vi-loss.csv"].splitlines()) > 50

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "vi_cross_histograms", aa.vi_cross_histograms)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    host_res = p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
    assert host_res == gpu_res and 0 < gpu_res["vi-pairwise"]["f1score"] <= 1
