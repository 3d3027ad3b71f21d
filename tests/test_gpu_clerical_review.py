"""The clerical review on the GPU (dbl_pairs_record_links and dbl_posterior_cluster_counts in dbl_posterior.cu,
analysis_gpu.record_links / cluster_appearances) against the numpy path in analysis_arrays.py: every integer exactly,
from 1 record to 1 M, with a 12 000-record cluster, with host and device labels and outputs and an all-singleton
center; every refusal leaves the handle usable; the project's files equal the host path's."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def assert_equal_to_numpy(ch, labels):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    labels = aa.canonical_clusters(labels)
    C = int(labels.max()) + 1
    got = ag.record_links(ch, labels)
    want = aa.record_links(*aa.pairwise_match_counts(ch), labels, C)
    for name in ("W", "I", "partner", "partner_count", "inner", "least"):
        g, w = getattr(got, name), getattr(want, name)
        assert g.dtype == np.int64 and np.array_equal(g, w), name
    A = ag.cluster_appearances(ch, labels)
    assert A.dtype == np.int64 and np.array_equal(A, aa.cluster_appearances(ch, labels))
    return got, A


def centers(ch):
    from dblink_b200 import analysis_arrays as aa

    R = ch.num_records
    mem, off, _ = ch.samples[len(ch.samples) // 2]
    rng = np.random.default_rng(R)
    return [aa.shared_most_probable_clusters(ch), aa.sample_labels(R, mem, off), rng.integers(0, max(1, R // 2), R)]


@pytest.mark.parametrize("R,S", [(1, 1), (2, 3), (40, 1), (700, 17), (5000, 40), (50_000, 12)])
def test_random_chains_equal_numpy(R, S):
    ch = random_chain(R, S, seed=R + S)
    for labels in centers(ch):
        links, A = assert_equal_to_numpy(ch, labels)
    if R >= 700:
        assert (links.partner >= 0).any() and (links.inner > 0).any() and (A > 0).any()


def test_an_all_singleton_center_and_a_sample_as_the_center():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(3000, 9, seed=5)
    links, _ = assert_equal_to_numpy(ch, np.arange(3000))
    assert (links.I == 0).all() and (links.inner == 0).all() and (links.least == 0).all()
    mem, off, _ = ch.samples[4]
    _, A = assert_equal_to_numpy(ch, aa.sample_labels(3000, mem, off))
    assert (A >= 1).all()


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    ch = chain_with_big(50_000, 6, seed=8, big=12_000)
    mem, off, _ = ch.samples[0]
    from dblink_b200 import analysis_arrays as aa

    links, A = assert_equal_to_numpy(ch, aa.sample_labels(50_000, mem, off))
    assert links.inner.max() == 12_000 * 11_999 // 2 and links.W.max() >= 11_999
    assert_equal_to_numpy(ch, centers(ch)[0])


def test_million_records():
    """The chain of profiles/scripts/smpc_time.py: R = 1 M, 64 partitions, S = 100, against its sMPC."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

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
    ch = aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples)
    links, A = assert_equal_to_numpy(ch, ag.shared_most_probable_clusters(ch))
    assert (links.partner >= 0).sum() > R // 10 and (A >= 1).all() and (A < S).any()


def test_device_labels_and_outputs_equal_host_ones():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    L = _lib.load()
    ch = random_chain(4000, 30, seed=21)
    R = ch.num_records
    labels = aa.canonical_clusters(centers(ch)[0])
    C = int(labels.max()) + 1
    dev = torch.tensor(labels.astype(np.int32), device="cuda")
    with ag.Pairs(R) as p:
        ag._add_chain(p, ch)
        want = p.record_links(labels, C)
        r64 = [torch.zeros(R, dtype=torch.int64, device="cuda") for _ in range(2)]
        r32 = [torch.zeros(R, dtype=torch.int32, device="cuda") for _ in range(2)]
        c64, c32 = torch.zeros(C, dtype=torch.int64, device="cuda"), torch.zeros(C, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert L.dbl_pairs_record_links(p._h, dev.data_ptr(), C, *(a.data_ptr() for a in r64 + r32 + [c64, c32])) \
            == _lib.OK
        for a, name in zip(r64 + r32 + [c64, c32], ("W", "I", "partner", "partner_count", "inner", "least")):
            assert np.array_equal(a.cpu().numpy(), getattr(want, name)), name
    with ag.Posterior(R, len(ch.samples)) as post:
        ag._add_chain(post, ch)
        want = post.cluster_counts(labels, C)
        out = torch.zeros(R, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        assert L.dbl_posterior_cluster_counts(post._h, dev.data_ptr(), C, out.data_ptr()) == _lib.OK
        assert np.array_equal(out.cpu().numpy(), want)


def test_refusals_leave_the_handle_usable():
    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    ch = random_chain(400, 12, seed=4)
    R = ch.num_records
    labels = aa.canonical_clusters(centers(ch)[0]).astype(np.int32)
    C = int(labels.max()) + 1
    gap = labels.copy()
    gap[gap == 1] = 0  # cluster 1 empty
    wide = labels.copy()
    wide[7] = C
    neg = labels.copy()
    neg[3] = -1
    for cls, call in ((ag.Pairs, lambda h, lab, c: h.record_links(lab, c)),
                      (ag.Posterior, lambda h, lab, c: h.cluster_counts(lab, c))):
        h = cls(R) if cls is ag.Pairs else cls(R, len(ch.samples))
        try:
            assert status(call, h, labels, C) == _lib.ERR_STATE  # no sample yet
            ag._add_chain(h, ch)
            for bad, c in ((labels, 0), (labels, R + 1), (labels, C - 1), (labels, C + 1), (gap, C), (wide, C),
                           (neg, C)):
                assert status(call, h, bad, c) == _lib.ERR_INVALID
            got = call(h, labels, C)
            if cls is ag.Pairs:
                want = aa.record_links(*aa.pairwise_match_counts(ch), labels, C)
                assert all(np.array_equal(getattr(got, n), getattr(want, n)) for n in ("W", "I", "partner", "least"))
            else:
                assert np.array_equal(got, aa.cluster_appearances(ch, labels))
            assert h.num_samples == len(ch.samples)
        finally:
            h.close()
    L = _lib.load()
    out = np.zeros(R, np.int32)
    with ag.Posterior(R, len(ch.samples)) as post:
        ag._add_chain(post, ch)
        assert L.dbl_posterior_cluster_counts(post._h, None, C, out.ctypes.data) == _lib.ERR_INVALID
        assert L.dbl_posterior_cluster_counts(post._h, labels.ctypes.data, C, None) == _lib.ERR_INVALID
    with ag.Pairs(R) as p:
        ag._add_chain(p, ch)
        bufs = [np.zeros(R, np.int64), np.zeros(R, np.int64), np.zeros(R, np.int32), np.zeros(R, np.int32),
                np.zeros(C, np.int64), np.zeros(C, np.int32)]
        for hole in range(len(bufs)):
            args = [None if i == hole else b.ctypes.data for i, b in enumerate(bufs)]
            assert L.dbl_pairs_record_links(p._h, labels.ctypes.data, C, *args) == _lib.ERR_INVALID
        assert L.dbl_pairs_record_links(p._h, None, C, *(b.ctypes.data for b in bufs)) == _lib.ERR_INVALID


def test_new_kernels_do_not_spill():
    from dblink_b200 import _lib

    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--dump-resource-usage", _lib.SO_PATH], capture_output=True, text=True).stdout
    lines = out.splitlines()
    for name in ("k_record_links", "k_links_out", "k_match_center", "k_flag_emptyIi", "k_flag_emptyIj"):
        at = [i for i, line in enumerate(lines) if name in line and "Function" in line]
        assert len(at) == 1, name
        assert " LOCAL:0 " in lines[at[0] + 1] and " STACK:0 " in lines[at[0] + 1], lines[at[0] + 1]


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize and evaluate on RLdata500 sampled on the GPU: the device review writes the same bytes as the numpy
    path."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                      'quantities : ["clerical-review", "shared-most-probable-clusters"], falseLinkCost : 0.3')
        return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["pairwise", "clerical-review"], '
                         'falseLinkCost : 0.3')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    for name in ("record_links", "cluster_appearances"):
        real = getattr(ag, name)
        monkeypatch.setattr(ag, name, lambda ch, lab, real=real: calls.append(1) or real(ch, lab))
    Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 4  # summarize and evaluate, two calls each
    names = ("clerical-review.csv", "clerical-review-records.csv", "clerical-review-clusters.csv",
             "clerical-review-evaluation.csv", "evaluation-results.txt", "shared-most-probable-clusters.csv")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert len(gpu[names[0]].splitlines()) > 100 and b"Clerical review" in gpu["evaluation-results.txt"]

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "shared_most_probable_clusters", aa.shared_most_probable_clusters)
    monkeypatch.setattr(project, "cluster_appearances", aa.cluster_appearances)
    monkeypatch.setattr(project, "record_links", lambda ch, labels: aa.record_links(
        *aa.pairwise_match_counts(ch), labels, int(np.max(labels)) + 1))
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "sample"]
    p.execute(log=lambda *a: None)
    assert len(calls) == 4
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
