"""The Binder-loss point estimate on the host: analysis_arrays.binder_counts / binder_losses / binder_estimate against
the worked example, the set-based analysis.binder_clusters and a brute-force least-squares search; the summarize
quantity binder-clusters and the evaluate metrics binder-pairwise / binder-cluster with their output files; the C
ABI's checks that come before any device work."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from test_match_probabilities_host import as_set_chain, random_chain


def chain_of(links, iterations=None, chains=None):
    from dblink_b200 import analysis_arrays as aa

    R = len(links[0])
    its = np.arange(len(links), dtype=np.int64) if iterations is None else np.asarray(iterations, np.int64)
    return aa.ChainArrays(np.array(["r%d" % i for i in range(R)]), its,
                          [aa.sample_from_links(np.asarray(l, np.int32), np.zeros(R, np.int32)) for l in links], chains)


# R = 4, S = 3: s0 = {0,1}{2}{3}, s1 = {0,1,2}{3}, s2 = {0}{1}{2,3}
WORKED = [[0, 0, 2, 3], [0, 0, 0, 3], [0, 1, 2, 2]]


def test_worked_example():
    from dblink_b200 import analysis_arrays as aa

    ch = chain_of(WORKED)
    n, K = aa.binder_counts(ch)
    assert n.dtype == K.dtype == np.int64 and list(n) == [1, 3, 1] and list(K) == [2, 4, 1]
    _, _, count = aa.pairwise_match_counts(ch)
    assert int(n.sum()) == int(count.sum()) == 5 and int(K.sum()) == int((count ** 2).sum()) == 7
    for t, want, best in ((0.5, [2 / 3, 1, 1], 0), (0.2, [2.6 / 3, 0.6, 1.2], 1), (0.9, [0.4, 4.6 / 3, 2.2 / 3], 0)):
        got = aa.binder_losses(n, K, t)
        assert got.dtype == np.float64 and np.abs(got - want).max() < 1e-15
        assert aa.binder_estimate(n, K, t) == best


def set_based(ch, t):
    from dblink_b200 import analysis

    return analysis.binder_clusters(as_set_chain(ch)[0], t)


def assert_choice_equal_to_sets(ch, t):
    from dblink_b200 import analysis_arrays as aa

    n, K = aa.binder_counts(ch)
    s = aa.binder_estimate(n, K, t)
    best, clusters, losses = set_based(ch, t)
    assert s == best
    mem, off, _ = ch.samples[s]
    ids = list(ch.record_ids)
    got = {frozenset(ids[i] for i in g) for g in aa.labels_to_clusters(aa.sample_labels(ch.num_records, mem, off))}
    assert got == set(clusters)
    assert np.allclose(aa.binder_losses(n, K, t), losses, rtol=0, atol=1e-12)
    return s


@pytest.mark.parametrize("R,S", [(2, 3), (7, 12), (25, 30), (60, 9), (60, 30)])
def test_random_chains_choose_the_set_based_sample(R, S):
    ch = random_chain(R, S, seed=R * 31 + S)
    chosen = {assert_choice_equal_to_sets(ch, t) for t in (0.0, 0.1, 0.5, 0.9, 1.0)}
    if R >= 25:
        assert len(chosen) > 1  # the cost moves the choice


@pytest.mark.parametrize("seed", range(6))
def test_half_cost_is_the_least_squares_sample(seed):
    """At t = 1/2 the estimate minimises sum over pairs of (delta - p)^2 (Dahl 2006), by brute force over all pairs."""
    from dblink_b200 import analysis_arrays as aa

    R, S = 15, 20
    ch = random_chain(R, S, seed=100 + seed)
    delta = np.zeros((S, R, R), np.int64)
    for s, (mem, off, _) in enumerate(ch.samples):
        lab = aa.sample_labels(R, mem, off)
        delta[s] = lab[:, None] == lab[None, :]
    count = delta.sum(0)
    iu = np.triu_indices(R, 1)
    sq = [int(((S * delta[s] - count)[iu] ** 2).sum()) for s in range(S)]  # S^2 sum (delta - p)^2, exact
    n, K = aa.binder_counts(ch)
    assert aa.binder_estimate(n, K, 0.5) == min(range(S), key=lambda s: (sq[s], s))
    assert int(K.sum()) == int((count[iu] ** 2).sum())


@pytest.mark.parametrize("R,S", [(40, 20), (300, 9)])
def test_count_sums_are_the_sum_of_squared_counts(R, S):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(R, S, seed=R + S)
    n, K = aa.binder_counts(ch)
    _, _, count = aa.pairwise_match_counts(ch)
    assert int(n.sum()) == int(count.sum()) and int(K.sum()) == int((count ** 2).sum())


def test_edge_cases():
    from dblink_b200 import analysis_arrays as aa

    R = 8
    # one sample: every pair it links has p = 1, every other p = 0, so its loss is 0 whatever t
    one = chain_of([[0, 0, 1, 1, 1, 5, 6, 7]])
    n, K = aa.binder_counts(one)
    assert list(n) == [4] and list(K) == [4]
    for t in (0.0, 0.3, 1.0):
        assert aa.binder_losses(n, K, t).tolist() == [0.0] and assert_choice_equal_to_sets(one, t) == 0
    # all singletons, and one big cluster, in every sample: nothing to choose, losses 0
    for link in (np.arange(R), np.zeros(R)):
        ch = chain_of([link] * 3)
        n, K = aa.binder_counts(ch)
        assert list(n) == [int(link[0] == link[1]) * R * (R - 1) // 2] * 3 and list(K) == list(3 * n)
        assert aa.binder_losses(n, K, 0.5).tolist() == [0.0] * 3 and aa.binder_estimate(n, K, 0.5) == 0
    # ties go to the earliest sample: s0 and its copy s3 tie; at t = 1/2 the singletons (s0) tie with {0,1}{2}{3} (s1)
    ch = chain_of(WORKED + [WORKED[0]])
    n, K = aa.binder_counts(ch)
    losses = aa.binder_losses(n, K, 0.5)
    assert losses[0] == losses[3] and aa.binder_estimate(n, K, 0.5) == 0 == assert_choice_equal_to_sets(ch, 0.5)
    tie = chain_of([[0, 1, 2, 3], [0, 0, 2, 3]])  # counts (0,1) = 1, S = 2: losses 1/4 and 1/4
    n, K = aa.binder_counts(tie)
    assert aa.binder_losses(n, K, 0.5).tolist() == [0.25, 0.25] and assert_choice_equal_to_sets(tie, 0.5) == 0
    assert assert_choice_equal_to_sets(tie, 0.4) == 1 and assert_choice_equal_to_sets(tie, 0.6) == 0
    # t = 1/10 is not exact in binary; the choice compares the exact binary fraction, as the set-based one does
    assert assert_choice_equal_to_sets(chain_of([[0, 1, 2, 3]] + [[0, 0, 2, 3]] * 9), 0.1) == 1
    # no sample
    empty = chain_of([np.arange(3)])
    empty.samples, empty.iterations, empty.chains = [], np.zeros(0, np.int64), np.zeros(0, np.int64)
    n, K = aa.binder_counts(empty)
    assert len(n) == len(K) == 0
    with pytest.raises(ValueError, match="at least one sample"):
        aa.binder_estimate(n, K, 0.5)


def test_sample_labels():
    from dblink_b200 import analysis_arrays as aa

    mem, off, _ = aa.sample_from_links(np.array([3, 0, 3, 2, 0, 3], np.int32), np.zeros(4, np.int32))
    assert list(aa.sample_labels(6, mem, off)) == [0, 1, 0, 3, 1, 0]
    with pytest.raises(ValueError, match="exactly once"):
        aa.sample_labels(6, mem[:-1], off[:-1])
    with pytest.raises(ValueError, match="exactly once"):
        aa.sample_labels(6, np.r_[mem[:-1], mem[0]], off)


def test_the_cap_is_the_pairwise_one():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 9, seed=5)
    n = len(aa.pairwise_match_counts(ch)[0])
    with pytest.raises(ValueError, match=f"^the chain puts more than {n - 1} distinct record pairs in a cluster$"):
        aa.binder_counts(ch, max_pairs=n - 1)
    assert len(aa.binder_counts(ch, max_pairs=n)[0]) == 9


CONF = """
dblink : {
  data : { path : "%s", recordIdentifier : "rec_id", entityIdentifier : "ent_id", nullValue : "NA",
           matchingAttributes : [ {name : "a", similarityFunction : { name : "ConstantSimilarityFn" },
                                   distortionPrior : {alpha : 0.5, beta : 50.0}} ] }
  outputPath : "%s"
  randomSeed : 1
  numChains : %d
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [
    {name : "summarize", parameters : { lowerIterationCutoff : 10, quantities : %s %s }}
    {name : "evaluate", parameters : { lowerIterationCutoff : 10, metrics : %s %s }}
  ]
}
"""


def project_of(tmp_path, chains=1, quantities='["partition-sizes"]', metrics='["pairwise"]', summarize_extra="",
               evaluate_extra="", out="out"):
    from dblink_b200 import config
    from dblink_b200.project import Project

    data = os.path.join(tmp_path, "data.csv")
    return Project(config.parse_string(CONF % (data, str(tmp_path / out) + "/", chains, quantities, summarize_extra,
                                               metrics, evaluate_extra)), base_dir="")


def test_config(tmp_path):
    def steps(**kw):
        return project_of(tmp_path, **kw).steps()

    (_, s), (_, e) = steps(quantities='["binder-clusters"]', metrics='["binder-cluster", "binder-pairwise"]')
    assert s["quantities"] == ["binder-clusters"] and s["false_link_cost"] == 0.5
    assert e["metrics"] == ["binder-cluster", "binder-pairwise"] and e["false_link_cost"] == 0.5
    (_, s), (_, e) = steps(quantities='["binder-clusters"]', summarize_extra=", falseLinkCost : 0.7",
                           metrics='["binder-cluster"]', evaluate_extra=", falseLinkCost : 1")
    assert s["false_link_cost"] == 0.7 and e["false_link_cost"] == 1.0
    assert steps(summarize_extra=", falseLinkCost : 0")[0][1]["false_link_cost"] == 0.0
    for bad in ("-0.1", "1.5", "2"):
        for kw in (dict(summarize_extra=", falseLinkCost : " + bad), dict(evaluate_extra=", falseLinkCost : " + bad)):
            with pytest.raises(ValueError, match=r"^falseLinkCost must be in \[0, 1\]\.$"):
                steps(**kw)
    with pytest.raises(ValueError, match="quantities"):
        steps(quantities='["binder-cluster"]')
    with pytest.raises(ValueError, match="metrics"):
        steps(metrics='["binder-clusters"]')
    # the step descriptions mention the estimate only when it is asked for
    p = project_of(tmp_path, quantities='["binder-clusters", "partition-sizes"]',
                   summarize_extra=", falseLinkCost : 0.25", metrics='["pairwise", "binder-pairwise"]')
    assert p.steps_mk_string().splitlines()[2:] == [
        "  * SummarizeStep: Calculating summary quantities {'binder-clusters', 'partition-sizes'} along the chain for "
        "iterations >= 10",
        "  * SummarizeStep: binder-clusters is the sample of least posterior expected Binder loss with "
        "falseLinkCost=0.25",
        "  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= 10) using {'pairwise'} "
        "metrics",
        "  * EvaluateStep: Evaluating the sample of least posterior expected Binder loss (falseLinkCost=0.5, "
        "iterations >= 10) using {'binder-pairwise'} metrics"]
    assert "Binder" not in project_of(tmp_path).steps_mk_string()


# 6 records, truth {r0,r1} {r2,r3} {r4} {r5}; a sample at iteration 0 that the cutoff drops, then s0 = singletons,
# s1 = the truth, s2 = {0,1,2} {3} {4,5}.  Counts (0,1) = 2, (0,2) = (1,2) = (2,3) = (4,5) = 1, C = 6, S = 3;
# n = 0, 2, 4 and K = 0, 3, 5.  t = 0.4: losses (3.6 + 1.2 n - K) / 3 = 1.2, 1, 3.4/3: s1.  t = 0.3: losses
# (4.2 + 0.9 n - K) / 3 = 1.4, 1, 2.8/3: s2.
CHAIN = [(0, [0, 0, 0, 0, 0, 0]), (10, [0, 1, 2, 3, 4, 5]), (20, [0, 0, 2, 2, 4, 5]), (30, [0, 0, 0, 3, 4, 4])]

BINDER_CLUSTERS_CSV = "r0, r1\nr2, r3\nr4\nr5\n"

BINDER_LOSS_CSV = """chain,iteration,linkedPairs,expectedLoss
0,10,0,1.2
0,20,2,1.0
0,30,4,1.1333333333333335
"""

# the second chain holds the truth at iteration 20 only: pooled S = 4, C = 8, counts (0,1) = 3, (2,3) = 2;
# n = 0, 2, 4, 2 and K = 0, 5, 6, 5; t = 0.4: losses (4.8 + 1.6 n - K) / 4 = 1.2, 0.75, 1.3, 0.75: chain 0's s1
BINDER_LOSS_TWO_CHAINS_CSV = """chain,iteration,linkedPairs,expectedLoss
0,10,0,1.2
0,20,2,0.75
0,30,4,1.2999999999999998
1,20,2,0.75
"""

BINDER_RESULTS_TXT = """=====================================
       Binder cluster metrics
-------------------------------------
 Estimate:        sample at iteration 30 of chain 0, falseLinkCost 0.3
 Adj. Rand index: 0.18918918918918917
=====================================

=====================================
      Binder pairwise metrics
-------------------------------------
 Estimate:        sample at iteration 30 of chain 0, falseLinkCost 0.3
 Precision:      0.25
 Recall:         0.5
 F1-score:       0.3333333333333333
=====================================

"""


def write_chain(tmp_path, p):
    from dblink_b200 import writers as w

    with open(os.path.join(tmp_path, "data.csv"), "w") as fh:
        fh.write("rec_id,ent_id,a\n" + "".join(f"r{i},e{t},v{i % 2}\n" for i, t in enumerate([0, 0, 1, 1, 2, 3])))
    ids = ["r%d" % i for i in range(6)]
    for k, dr in enumerate(p.chain_dirs()):
        lw = w.LinkageChainWriter(os.path.join(dr, "linkage-chain.parquet"))
        for it, link in CHAIN if k == 0 else CHAIN[:1] + CHAIN[2:3]:
            lw.append(it, w.linkage_structure_arrow(np.array(link, np.int32), np.zeros(6, np.int32), ids))
        lw.close()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("binder_counts", "shared_most_probable_clusters", "pairwise_match_counts", "posterior_metric_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))


def test_project_writes_the_estimate_and_its_metrics(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, quantities='["binder-clusters"]', summarize_extra=", falseLinkCost : 0.4",
                   metrics='["binder-cluster", "binder-pairwise"]', evaluate_extra=", falseLinkCost : 0.3")
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "binder-clusters.csv").read() == BINDER_CLUSTERS_CSV
    assert open(out + "binder-loss.csv").read() == BINDER_LOSS_CSV
    assert open(out + "evaluation-results.txt").read() == BINDER_RESULTS_TXT
    assert set(res) == {"binder-cluster", "binder-pairwise"}
    assert res["binder-cluster"] == pytest.approx(7 / 37)
    assert (res["binder-pairwise"]["TP"], res["binder-pairwise"]["FP"], res["binder-pairwise"]["FN"]) == (1, 3, 1)
    assert not os.path.exists(out + "shared-most-probable-clusters.csv")


def test_two_chains_pool_the_estimate(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, chains=2, quantities='["binder-clusters"]', summarize_extra=", falseLinkCost : 0.4",
                   metrics='["binder-pairwise"]', evaluate_extra=", falseLinkCost : 0.4")
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "binder-loss.csv").read() == BINDER_LOSS_TWO_CHAINS_CSV
    assert open(out + "binder-clusters.csv").read() == BINDER_CLUSTERS_CSV
    assert " Estimate:        sample at iteration 20 of chain 0, falseLinkCost 0.4\n" in open(
        out + "evaluation-results.txt").read()
    assert res["binder-pairwise"]["precision"] == 1.0 and res["binder-pairwise"]["recall"] == 1.0


def test_pooled_reader_names_each_samples_chain(tmp_path):
    from dblink_b200 import analysis_arrays as aa

    p = project_of(tmp_path, chains=2)
    write_chain(tmp_path, p)
    pooled = p.read_chain(10)
    assert list(pooled.chains) == [0, 0, 0, 1] and list(pooled.iterations) == [10, 20, 30, 20]
    one = aa.read_chain_arrays(os.path.join(p.chain_dirs()[1], "linkage-chain.parquet"), 0)
    assert list(one.chains) == [0, 0] and list(one.iterations) == [0, 20]


def test_no_sample_after_the_cutoff(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    for kw in (dict(quantities='["binder-clusters"]'), dict(metrics='["binder-pairwise"]')):
        p = project_of(tmp_path, **kw)
        write_chain(tmp_path, p)
        p.steps = lambda p=p: [(n, dict(prm, lower_iteration_cutoff=100)) for n, prm in type(p).steps(p)]
        with pytest.raises(ValueError, match="at least one sample at or after lowerIterationCutoff"):
            p.execute(log=lambda *a: None)


def test_other_outputs_do_not_change(tmp_path, monkeypatch):
    """The same steps with and without the new names write the same bytes in every other file; the evaluation text
    only gains the Binder sections at its end."""
    host_paths(monkeypatch)
    quantities = ["shared-most-probable-clusters", "pairwise-match-probabilities", "cluster-size-distribution",
                  "partition-sizes"]
    metrics = ["pairwise", "cluster", "posterior-pairwise", "posterior-cluster"]

    def run(out, q, m):
        p = project_of(tmp_path, quantities=str(q).replace("'", '"'), metrics=str(m).replace("'", '"'), out=out)
        write_chain(tmp_path, p)
        p.execute(log=lambda *a: None)
        d = str(tmp_path / out)
        return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d)) if f.endswith((".csv", ".txt"))}

    plain = run("plain", quantities, metrics)
    mixed = run("mixed", quantities[:2] + ["binder-clusters"] + quantities[2:],
                metrics[:1] + ["binder-pairwise"] + metrics[1:] + ["binder-cluster"])
    assert set(mixed) - set(plain) == {"binder-clusters.csv", "binder-loss.csv"}
    text = "evaluation-results.txt"
    for f in plain:
        if f != text:
            assert mixed[f] == plain[f], f
    assert mixed[text].startswith(plain[text]) and b"Binder pairwise metrics" in mixed[text][len(plain[text]):]


def test_abi_checks_before_any_device_work():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Pairs

    L = _lib.load()
    labels = np.zeros(4, np.int32)
    n, K = C.c_int64(-1), C.c_int64(-1)
    for args in itertools.product((None,), (None, labels.ctypes.data), (None, C.byref(n)), (None, C.byref(K))):
        assert L.dbl_pairs_score_sample(*args) == _lib.ERR_INVALID
    assert (n.value, K.value) == (-1, -1)
    p = Pairs.__new__(Pairs)  # an owner without a handle: the shape check comes first
    p.num_records = 4
    with pytest.raises(ValueError, match="one cluster label per record"):
        p.score_sample(np.zeros(3, np.int32))


def test_binder_counts_need_a_device():
    import torch

    from dblink_b200 import _lib, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(DblinkError) as e:
        ag.binder_counts(chain_of(WORKED))
    assert e.value.status == _lib.ERR_CUDA


def test_project_uses_the_host_counts_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(chain, **kw):
        raise AssertionError("the GPU counts were called on a host without a device")

    monkeypatch.setattr(ag, "binder_counts", no_gpu)
    n, K = project.binder_counts(chain_of(WORKED))
    assert list(n) == [1, 3, 1] and list(K) == [2, 4, 1]
    s, labels, n, losses = project.binder_estimate(chain_of(WORKED), 0.2)
    assert s == 1 and list(labels) == [0, 0, 0, 3] and list(n) == [1, 3, 1] and losses[1] == pytest.approx(0.6)
