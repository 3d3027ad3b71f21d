"""The variation-of-information point estimate on the host: analysis_arrays.vi_cross_histograms / vi_losses /
vi_estimate against a worked example and the set-based analysis.vi_clusters; the histogram cap; the summarize quantity
vi-clusters and the evaluate metrics vi-pairwise / vi-cluster with their output files; the C ABI's checks that come
before any device work."""
import csv
import ctypes as C
import os

import numpy as np
import pytest

from test_binder_host import WORKED, chain_of, project_of
from test_match_probabilities_host import as_set_chain, random_chain


def numpy_losses(ch):
    from dblink_b200 import analysis_arrays as aa

    G = aa.vi_cross_histograms(ch)
    g = aa.vi_cluster_histograms(ch, G.shape[1])
    return aa.vi_losses(g, G, ch.num_records)


def assert_equal_to_sets(ch):
    """The numpy losses equal the entropy / mutual-information definition to 1e-9 relative, and the choice is the
    same unless the best two losses are closer than that."""
    from dblink_b200 import analysis, analysis_arrays as aa

    losses = numpy_losses(ch)
    best, clusters, want = analysis.vi_clusters(as_set_chain(ch)[0])
    assert losses.dtype == np.float64 and np.allclose(losses, want, rtol=1e-9, atol=1e-12)
    s = aa.vi_estimate(losses)
    top = sorted(want)
    if len(top) < 2 or top[1] - top[0] > 1e-9 * max(abs(top[1]), 1e-300):
        assert s == best
        mem, off, _ = ch.samples[s]
        ids = list(ch.record_ids)
        got = {frozenset(ids[i] for i in g) for g in aa.labels_to_clusters(aa.sample_labels(ch.num_records, mem, off))}
        assert got == set(clusters)
    return losses


def test_worked_example():
    from dblink_b200 import analysis_arrays as aa

    # s0 = {0,1}{2}{3}, s1 = {0,1,2}{3}, s2 = {0}{1}{2,3}: only s0 ^ s1 has a cell of two, {0,1}
    ch = chain_of(WORKED)
    G = aa.vi_cross_histograms(ch)
    assert G.dtype == np.int64 and G.tolist() == [[0, 0, 1, 0], [0, 0, 1, 0], [0, 0, 0, 0]]
    g = aa.vi_cluster_histograms(ch, 4)
    assert g.tolist() == [[0, 0, 1, 0], [0, 0, 0, 1], [0, 0, 1, 0]]
    # A = 2, 3 log2 3, 2; D_t[n] = g_t[n] + sum_s g_s[n] - 2 G_t[n]
    a3 = 3 * np.log2(3)
    want = [(2 + a3) / 12, 2 * a3 / 12, (6 + a3) / 12]
    losses = aa.vi_losses(g, G, 4)
    assert np.allclose(losses, want, rtol=1e-15) and aa.vi_estimate(losses) == 0
    assert_equal_to_sets(ch)


@pytest.mark.parametrize("R,S", [(2, 3), (7, 12), (25, 30), (60, 9), (40, 20), (150, 6)])
def test_random_chains_equal_the_set_based_losses(R, S):
    assert_equal_to_sets(random_chain(R, S, seed=R * 31 + S))


def test_a_big_cluster_next_to_small_ones():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 5, seed=4, big=120)
    G = aa.vi_cross_histograms(ch)
    assert G.shape == (5, aa.vi_width(ch)) and G.shape[1] > 120
    assert_equal_to_sets(ch)


def test_edge_cases():
    from dblink_b200 import analysis_arrays as aa

    # one sample: VI against itself is 0
    one = chain_of([[0, 0, 1, 1, 1, 5, 6, 7]])
    assert numpy_losses(one).tolist() == [0.0] and assert_equal_to_sets(one).tolist() == [0.0]
    # two samples: each is the other's only partner, so their losses are equal and the first is chosen
    two = chain_of([[0, 0, 1, 1, 1, 5, 6, 7], [0, 1, 2, 2, 4, 4, 4, 4]])
    losses = numpy_losses(two)
    assert losses[0] == losses[1] > 0 and aa.vi_estimate(losses) == 0
    # identical samples tie exactly, and the earliest wins
    ch = chain_of([WORKED[1], WORKED[0], WORKED[2], WORKED[0]])
    losses = numpy_losses(ch)
    assert losses[1] == losses[3] and aa.vi_estimate(losses) == 1
    # all singletons, or one cluster, in every sample: nothing to choose
    for link in (np.arange(5), np.zeros(5)):
        assert numpy_losses(chain_of([link] * 3)).tolist() == [0.0] * 3
    # all singletons: width 2, nothing to count
    assert aa.vi_cross_histograms(chain_of([np.arange(5)] * 2)).shape == (2, 2)
    with pytest.raises(ValueError, match="at least one sample"):
        aa.vi_estimate(np.zeros(0))


def test_the_cap_refuses_before_counting(monkeypatch):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 9, seed=5)
    width = aa.vi_width(ch)
    monkeypatch.setattr(aa, "MAX_VI_ENTRIES", 9 * width - 1)
    with pytest.raises(ValueError, match=f"^the VI histograms need 9 x {width} entries, more than {9 * width - 1}$"):
        aa.vi_cross_histograms(ch)
    monkeypatch.setattr(aa, "MAX_VI_ENTRIES", 9 * width)
    assert aa.vi_cross_histograms(ch).shape == (9, width)


def giant_chain():
    """256 samples, each one cluster of 2^20 records: 256 x (2^20 + 1) entries, past the cap of 2^28."""
    from dblink_b200 import analysis_arrays as aa

    R = 1 << 20
    one = aa.sample_from_links(np.zeros(R, np.int32), np.zeros(1, np.int32))
    return aa.ChainArrays(np.arange(R), np.arange(256, dtype=np.int64), [one] * 256)


def test_a_giant_cluster_is_refused():
    from dblink_b200 import analysis_arrays as aa

    with pytest.raises(ValueError, match=r"^the VI histograms need 256 x 1048577 entries, more than 268435456$"):
        aa.vi_cross_histograms(giant_chain())


def test_config_and_run_txt(tmp_path):
    (_, s), (_, e) = project_of(tmp_path, quantities='["vi-clusters"]', metrics='["vi-cluster", "vi-pairwise"]').steps()
    assert s["quantities"] == ["vi-clusters"] and e["metrics"] == ["vi-cluster", "vi-pairwise"]
    with pytest.raises(ValueError, match="quantities"):
        project_of(tmp_path, quantities='["vi-cluster"]').steps()
    with pytest.raises(ValueError, match="metrics"):
        project_of(tmp_path, metrics='["vi-clusters"]').steps()
    p = project_of(tmp_path, quantities='["vi-clusters", "partition-sizes"]', metrics='["pairwise", "vi-pairwise"]')
    assert p.steps_mk_string().splitlines()[2:] == [
        "  * SummarizeStep: Calculating summary quantities {'vi-clusters', 'partition-sizes'} along the chain for "
        "iterations >= 10",
        "  * SummarizeStep: vi-clusters is the sample of least posterior expected variation of information",
        "  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= 10) using {'pairwise'} "
        "metrics",
        "  * EvaluateStep: Evaluating the sample of least posterior expected variation of information (iterations >= "
        "10) using {'vi-pairwise'} metrics"]
    assert "variation of information" not in project_of(tmp_path).steps_mk_string()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("vi_cross_histograms", "shared_most_probable_clusters", "pairwise_match_counts",
                 "posterior_metric_counts", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))


def read_loss(path):
    with open(path) as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["chain", "iteration", "numClusters", "expectedLoss"]
    return [(int(k), int(it), int(n)) for k, it, n, _ in rows[1:]], [float(x[3]) for x in rows[1:]]


def assert_outputs_are_the_set_based_ones(p, out, want_rows):
    from dblink_b200 import analysis

    ch = p.read_chain(10)
    best, clusters, want = analysis.vi_clusters(as_set_chain(ch)[0])
    rows, losses = read_loss(out + "vi-loss.csv")
    assert rows == want_rows and np.allclose(losses, want, rtol=1e-9)
    assert open(out + "vi-clusters.csv").read() == "".join(
        ", ".join(sorted(c)) + "\n" for c in sorted(clusters, key=lambda c: min(int(r[1:]) for r in c)))
    return best, losses


# 6 records, truth {r0,r1} {r2,r3} {r4} {r5}; a sample at iteration 0 that the cutoff drops, then s0 = the truth,
# s1 = {0,1} and singletons, s2 = {0,1} {2,3} {4,5}.  R VI(s0, s1) = 4 + 2 - 2 * 2 = 2, R VI(s0, s2) = 4 + 6 - 2 * 4 = 2,
# R VI(s1, s2) = 2 + 6 - 2 * 2 = 4: the truth lies between the other two and is chosen.  The second chain holds the
# truth at iteration 20 only, so pooled, chain 0's s0 and it tie.
CHAIN = [(0, [0, 0, 0, 0, 0, 0]), (10, [0, 0, 2, 2, 4, 5]), (20, [0, 0, 2, 3, 4, 5]), (30, [0, 0, 2, 2, 4, 4])]


def write_chain(tmp_path, p):
    from dblink_b200 import writers as w

    with open(os.path.join(tmp_path, "data.csv"), "w") as fh:
        fh.write("rec_id,ent_id,a\n" + "".join(f"r{i},e{t},v{i % 2}\n" for i, t in enumerate([0, 0, 1, 1, 2, 3])))
    ids = ["r%d" % i for i in range(6)]
    for k, dr in enumerate(p.chain_dirs()):
        lw = w.LinkageChainWriter(os.path.join(dr, "linkage-chain.parquet"))
        for it, link in CHAIN if k == 0 else [CHAIN[0], (20, CHAIN[1][1])]:
            lw.append(it, w.linkage_structure_arrow(np.array(link, np.int32), np.zeros(6, np.int32), ids))
        lw.close()


def test_project_writes_the_estimate_and_its_metrics(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, quantities='["vi-clusters"]', metrics='["vi-cluster", "vi-pairwise"]')
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    best, losses = assert_outputs_are_the_set_based_ones(p, out, [(0, 10, 4), (0, 20, 5), (0, 30, 3)])
    assert best == 0 and losses[0] < min(losses[1:]) and open(out + "vi-clusters.csv").read() == "r0, r1\nr2, r3\nr4\nr5\n"
    text = open(out + "evaluation-results.txt").read()
    line = f" Estimate:        sample at iteration 10 of chain 0, expected VI {losses[0]!r}\n"
    assert text == ("=====================================\n         VI cluster metrics\n"
                    "-------------------------------------\n" + line + " Adj. Rand index: 1.0\n"
                    "=====================================\n\n"
                    "=====================================\n        VI pairwise metrics\n"
                    "-------------------------------------\n" + line + " Precision:      1.0\n Recall:         1.0\n"
                    " F1-score:       1.0\n=====================================\n\n")
    assert set(res) == {"vi-cluster", "vi-pairwise"} and res["vi-cluster"] == 1.0
    assert not os.path.exists(out + "shared-most-probable-clusters.csv")


def test_two_chains_pool_the_estimate(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, chains=2, quantities='["vi-clusters"]', metrics='["vi-pairwise"]')
    write_chain(tmp_path, p)
    p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    # chain 1 holds the truth at iteration 20 only; it ties with chain 0's s0, which comes first
    best, losses = assert_outputs_are_the_set_based_ones(p, out, [(0, 10, 4), (0, 20, 5), (0, 30, 3), (1, 20, 4)])
    assert best == 0 and losses[0] == losses[3] < min(losses[1:3])
    assert f" Estimate:        sample at iteration 10 of chain 0, expected VI {losses[0]!r}\n" in open(
        out + "evaluation-results.txt").read()


def test_no_sample_after_the_cutoff(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    for kw in (dict(quantities='["vi-clusters"]'), dict(metrics='["vi-pairwise"]')):
        p = project_of(tmp_path, **kw)
        write_chain(tmp_path, p)
        p.steps = lambda p=p: [(n, dict(prm, lower_iteration_cutoff=100)) for n, prm in type(p).steps(p)]
        with pytest.raises(ValueError, match="at least one sample at or after lowerIterationCutoff"):
            p.execute(log=lambda *a: None)


def test_other_outputs_do_not_change(tmp_path, monkeypatch):
    """The same steps with and without the new names write the same bytes in every other file; the evaluation text
    only gains the VI sections at its end."""
    host_paths(monkeypatch)
    quantities = ["shared-most-probable-clusters", "pairwise-match-probabilities", "cluster-size-distribution",
                  "partition-sizes", "binder-clusters"]
    metrics = ["pairwise", "cluster", "posterior-pairwise", "posterior-cluster", "binder-pairwise"]

    def run(out, q, m):
        p = project_of(tmp_path, quantities=str(q).replace("'", '"'), metrics=str(m).replace("'", '"'), out=out)
        write_chain(tmp_path, p)
        p.execute(log=lambda *a: None)
        d = str(tmp_path / out)
        return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d)) if f.endswith((".csv", ".txt"))}

    plain = run("plain", quantities, metrics)
    mixed = run("mixed", quantities[:2] + ["vi-clusters"] + quantities[2:],
                metrics[:1] + ["vi-pairwise"] + metrics[1:] + ["vi-cluster"])
    assert set(mixed) - set(plain) == {"vi-clusters.csv", "vi-loss.csv"}
    text = "evaluation-results.txt"
    for f in plain:
        if f != text:
            assert mixed[f] == plain[f], f
    assert mixed[text].startswith(plain[text]) and b"VI pairwise metrics" in mixed[text][len(plain[text]):]


def test_abi_checks_before_any_device_work():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import VI

    L = _lib.load()
    h = C.c_void_p()
    for R, S in ((0, 1), (1, 0), (1 << 31, 1), (-1, 4)):
        assert L.dbl_vi_create(C.byref(h), R, S) == _lib.ERR_INVALID and not h.value
    assert L.dbl_vi_create(None, 4, 1) == _lib.ERR_INVALID
    G = np.zeros(8, np.int64)
    assert L.dbl_vi_cross(None, 4, G.ctypes.data) == _lib.ERR_INVALID
    assert L.dbl_vi_add_sample(None, np.zeros(4, np.int32).ctypes.data) == _lib.ERR_INVALID
    assert L.dbl_vi_set_batch_keys(None, 5) == _lib.ERR_INVALID
    assert L.dbl_vi_num_samples(None) == 0
    L.dbl_vi_free(None)
    v = VI.__new__(VI)  # an owner without a handle: the shape check comes first
    v.num_records = 4
    with pytest.raises(ValueError, match="one cluster label per record"):
        v.add_sample(np.zeros(3, np.int32))


def test_project_uses_the_host_path_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(chain, **kw):
        raise AssertionError("the GPU histograms were called on a host without a device")

    monkeypatch.setattr(ag, "vi_cross_histograms", no_gpu)
    assert project.vi_cross_histograms(chain_of(WORKED)).tolist() == [[0, 0, 1, 0], [0, 0, 1, 0], [0, 0, 0, 0]]
    s, labels, num_clusters, losses = project.vi_estimate(chain_of(WORKED))
    assert s == 0 and list(labels) == [0, 0, 2, 3] and list(num_clusters) == [3, 2, 3] and losses[0] < losses[2]
