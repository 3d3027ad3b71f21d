"""The cells of a labelling with every held sample, kept per sample, on the GPU (dbl_vi_score_samples in
dbl_posterior.cu, analysis_gpu.VI.score_samples) against numpy's analysis_arrays.vi_sample_cells: exactly equal on
random chains, on a 12 000-record cluster, under several batch budgets, for labels in host and in device memory, for
centers of one cluster and of singletons, on samples of singletons and on a 1 M-record chain; the rows sum to
dbl_vi_score; every refusal returns its documented status and leaves the held samples usable; the project's
credible-ball files are the same bytes on the GPU path and the numpy path."""
import os
import shutil

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def centers_of(ch, seed=0):
    """A sample's labels, the sMPC's, all singletons, one cluster and random labels."""
    from dblink_b200 import analysis_arrays as aa

    R = ch.num_records
    mem, off, _ = ch.samples[len(ch.samples) // 2]
    rng = np.random.default_rng(seed)
    return [aa.sample_labels(R, mem, off), aa.shared_most_probable_clusters(ch), np.arange(R), np.zeros(R, np.int64),
            rng.integers(0, max(R // 3, 1), R)]


def assert_equal_to_numpy(ch, centers=None, batch_keys=None):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    width = aa.vi_width(ch)
    with ag.vi_samples(ch, batch_keys) as vi:
        for lab in centers_of(ch) if centers is None else centers:
            got = vi.score_samples(lab, width)
            want = aa.vi_sample_cells(ch, lab, width)
            assert got.dtype == np.int64 and got.shape == want.shape and np.array_equal(got, want)
            assert np.array_equal(got.sum(axis=0), vi.score(lab, width))


@pytest.mark.parametrize("S", [1, 7, 64])
@pytest.mark.parametrize("R", [1, 2, 6, 40, 2500, 50_000])
def test_random_chains_equal_numpy(R, S):
    assert_equal_to_numpy(random_chain(R, S, seed=R * 7919 + S))


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    assert_equal_to_numpy(chain_with_big(50_000, 3, seed=8, big=12_000))


@pytest.mark.parametrize("batch_keys", [1, 5000, 1 << 20])
def test_batch_budgets_do_not_change_the_result(batch_keys):
    """A budget of 1 key takes one sample per batch; 5000 a few; 2^20 every sample of the chain in one batch."""
    assert_equal_to_numpy(random_chain(2500, 30, seed=17), batch_keys=batch_keys)


def test_samples_of_singletons():
    """Samples of singletons only give no keys; they sit between samples that do, in one batch and in several."""
    from dblink_b200 import analysis_arrays as aa

    R = 3000
    base = random_chain(R, 4, seed=5)
    single = aa.sample_from_links(np.arange(R, dtype=np.int32), np.zeros(R, np.int32))
    samples = [single, base.samples[0], single, single, base.samples[1], single]
    ch = aa.ChainArrays(base.record_ids, np.arange(len(samples), dtype=np.int64), samples)
    for batch_keys in (None, 1):
        assert_equal_to_numpy(ch, batch_keys=batch_keys)
    only = aa.ChainArrays(base.record_ids, np.arange(3, dtype=np.int64), [single] * 3)
    assert_equal_to_numpy(only)


def test_million_records():
    """The chain of test_gpu_vi.py's million-record test (R = 1 M, 20 samples), in several batches and in one."""
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
    centers = centers_of(ch)[:3]
    assert_equal_to_numpy(ch, centers, batch_keys=1 << 23)
    assert_equal_to_numpy(ch, centers[:1])


def test_device_labels_and_refusals_leave_the_samples_as_they_were():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    L = _lib.load()
    R = 40
    ch = random_chain(R, 9, seed=4)
    lab = centers_of(ch)[1]
    width = aa.vi_width(ch)
    with ag.VI(R, 10) as v:
        host = np.ascontiguousarray(lab, np.int32)
        G = np.full((9, width), -7, np.int64)
        assert L.dbl_vi_score_samples(v._h, host.ctypes.data, width, G.ctypes.data) == _lib.ERR_STATE  # no sample yet
        assert (G == -7).all()
        ag._add_chain(v, ch)
        held = v.cross(width)

        def unchanged():
            assert v.num_samples == 9 and np.array_equal(v.cross(width), held)

        want = aa.vi_sample_cells(ch, lab, width)
        dev = torch.tensor(host, device="cuda")
        out_dev = torch.full((9, width), -7, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        for ptr in (host.ctypes.data, dev.data_ptr()):
            G[:] = -7
            assert L.dbl_vi_score_samples(v._h, ptr, width, G.ctypes.data) == _lib.OK and np.array_equal(G, want)
            assert L.dbl_vi_score_samples(v._h, ptr, width, out_dev.data_ptr()) == _lib.OK
            torch.cuda.synchronize()
            assert np.array_equal(out_dev.cpu().numpy(), want)
            unchanged()
        # refusals: NULL pointers, width < M + 1, S width 8 bytes past INT64_MAX, labels outside [0, R)
        G[:] = -7
        assert L.dbl_vi_score_samples(v._h, None, width, G.ctypes.data) == _lib.ERR_INVALID
        assert L.dbl_vi_score_samples(v._h, host.ctypes.data, width, None) == _lib.ERR_INVALID
        assert L.dbl_vi_score_samples(v._h, host.ctypes.data, width - 1, G.ctypes.data) == _lib.ERR_INVALID
        assert L.dbl_vi_score_samples(v._h, host.ctypes.data, (1 << 63) // 8 // 9 + 1, G.ctypes.data) == \
            _lib.ERR_INVALID
        assert (G == -7).all()
        unchanged()
        for bad in (np.r_[host[:-1], R], np.r_[-1, host[1:]]):
            bad = np.ascontiguousarray(bad, np.int32)
            bad_dev = torch.tensor(bad, device="cuda")
            torch.cuda.synchronize()
            for ptr in (bad.ctypes.data, bad_dev.data_ptr()):
                assert L.dbl_vi_score_samples(v._h, ptr, width, G.ctypes.data) == _lib.ERR_INVALID
                assert (G == -7).all()
                unchanged()
        # still working after the refusals, and a sample can still be added
        assert np.array_equal(v.score_samples(lab, width), want)
        v.add_sample(np.zeros(R, np.int32))
        assert v.num_samples == 10 and v.score_samples(lab, R + 1).shape == (10, R + 1)


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500: the GPU path writes the same bytes as the numpy path from the same chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["credible-ball"], credibleLevel : 0.9')
        return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["credible-ball"]')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.vi_samples
    monkeypatch.setattr(ag, "vi_samples", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    gpu_res = Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 4  # summarize and evaluate: the VI search's center, then the ball
    names = ["credible-ball-samples.csv", "credible-ball.csv", "evaluation-results.txt"] + [
        f"credible-ball-{d}-{b}.csv" for d in aa.CREDIBLE_BALL_DISTANCES for b in aa.CREDIBLE_BALL_BOUNDS]
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert gpu["credible-ball.csv"].count(b"\n") == 7 and b"vi-search-clusters,0.9," in gpu["credible-ball.csv"]

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "shared_most_probable_clusters", aa.shared_most_probable_clusters)
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    host_res = p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
    assert host_res == gpu_res and gpu_res["credible-ball"]["samples"] > 0
