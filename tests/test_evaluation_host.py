"""Every posterior sample against the ground truth, on the host: analysis_arrays.posterior_metric_counts against the
set-based analysis.pairwise_metrics / adjusted_rand_index, the posterior summary, the evaluate metrics
posterior-pairwise / posterior-cluster and their output files, and the C ABI's checks that come before any device
work."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from test_match_probabilities_host import as_set_chain, random_chain


def same(a, b):
    return a == b or (isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b))


def sample_rows(ch, truth):
    from dblink_b200 import analysis_arrays as aa

    tp, pp, nc = aa.posterior_metric_counts(ch, truth)
    assert tp.dtype == pp.dtype == nc.dtype == np.int64 and len(tp) == len(ch.samples)
    return aa.sample_metrics(tp, pp, nc, truth)


@pytest.mark.parametrize("R,S", [(2, 3), (6, 7), (40, 20), (300, 9)])
def test_counts_give_the_set_based_metrics_on_every_sample(R, S):
    from dblink_b200 import analysis

    ch = random_chain(R, S, seed=R * 13 + S)
    truth = np.random.default_rng(R + S).integers(0, max(1, R // 2), R)
    chain, ids = as_set_chain(ch)
    true_sets = analysis.membership_to_clusters(ids, truth)
    rows = sample_rows(ch, truth)
    for (_, parts), row in zip(chain, rows):
        pred = [frozenset(c) for cl in parts.values() for c in cl]
        want = dict(analysis.pairwise_metrics(pred, true_sets), adjRandIndex=analysis.adjusted_rand_index(pred, true_sets),
                    numClusters=len(pred))
        assert set(row) == set(want)
        for k in want:
            assert same(row[k], want[k]), (k, row[k], want[k])
    if R >= 40:
        assert len({r["TP"] for r in rows}) > 1 and len({r["numClusters"] for r in rows}) > 1


def test_summary_by_hand():
    from dblink_b200 import analysis_arrays as aa

    # truth {0,1} {2,3} {4} {5}: 2 true pairs out of C(6, 2) = 15
    truth = np.array([0, 0, 1, 1, 2, 3])
    blk = np.zeros(6, np.int32)
    links = [[0, 1, 2, 3, 4, 5],   # singletons: no predicted pair, precision undefined
             [0, 0, 2, 2, 4, 5],   # the truth
             [0, 0, 0, 3, 4, 4]]   # {0,1,2} {3} {4,5}: 4 predicted pairs, 1 true
    ch = aa.ChainArrays(np.arange(6), np.array([10, 20, 30]),
                        [aa.sample_from_links(np.array(l, np.int32), blk) for l in links])
    tp, pp, nc = aa.posterior_metric_counts(ch, truth)
    assert list(tp) == [0, 2, 1] and list(pp) == [0, 2, 4] and list(nc) == [6, 4, 3]
    rows = aa.sample_metrics(tp, pp, nc, truth)
    assert math.isnan(rows[0]["precision"]) and rows[0]["recall"] == 0.0 and rows[0]["f1score"] == 0.0
    assert rows[0]["adjRandIndex"] == 0.0 and (rows[0]["FP"], rows[0]["FN"]) == (0, 2)
    assert [rows[1][k] for k in ("precision", "recall", "f1score", "adjRandIndex")] == [1.0, 1.0, 1.0, 1.0]
    assert (rows[2]["precision"], rows[2]["recall"]) == (0.25, 0.5) and rows[2]["f1score"] == pytest.approx(1 / 3)
    assert rows[2]["adjRandIndex"] == pytest.approx(7 / 37)  # (1 - 8/15) / (3 - 8/15)
    s = aa.posterior_summary(rows)
    p = s["precision"]
    assert (p["n"], p["undefined"]) == (2, 1)
    assert p["mean"] == 0.625 and p["sd"] == pytest.approx(0.75 / math.sqrt(2))
    assert (p["q025"], p["median"], p["q975"]) == pytest.approx((0.26875, 0.625, 0.98125))
    r = s["recall"]
    assert (r["n"], r["undefined"]) == (3, 0) and r["mean"] == 0.5 and r["sd"] == 0.5 and r["median"] == 0.5
    assert (r["q025"], r["q975"]) == pytest.approx((0.025, 0.975))
    n = s["numClusters"]
    assert n["mean"] == pytest.approx(13 / 3) and n["median"] == 4.0 and n["sd"] == pytest.approx(math.sqrt(7 / 3))
    assert (n["q025"], n["q975"]) == pytest.approx((3.05, 5.9))
    assert s["adjRandIndex"]["mean"] == pytest.approx((1 + 7 / 37) / 3)
    # one sample: no sd; no defined value: every statistic NaN
    one = aa.posterior_summary(rows[1:2])
    assert one["f1score"]["mean"] == 1.0 and math.isnan(one["f1score"]["sd"]) and one["f1score"]["q025"] == 1.0
    none = aa.posterior_summary(rows[0:1])["precision"]
    assert (none["n"], none["undefined"]) == (0, 1)
    assert all(math.isnan(none[k]) for k in ("mean", "sd", "q025", "median", "q975"))


def test_repeated_clustering_summarises_to_its_own_metrics():
    from dblink_b200 import analysis_arrays as aa

    R = 200
    rng = np.random.default_rng(7)
    link = rng.integers(0, 120, R).astype(np.int32)
    truth = rng.integers(0, 150, R)
    # eight copies: numpy sums eight equal floats exactly, so the mean is the value itself and the sd is 0
    ch = aa.ChainArrays(np.arange(R), np.arange(8), [aa.sample_from_links(link, np.zeros(120, np.int32))] * 8)
    s = aa.posterior_summary(sample_rows(ch, truth))
    pw, ari = aa.pairwise_metrics(link, truth), aa.adjusted_rand_index(link, truth)
    for k in ("precision", "recall", "f1score"):
        assert s[k]["mean"] == pw[k] and s[k]["median"] == pw[k] and s[k]["sd"] == 0.0
    assert s["adjRandIndex"]["mean"] == ari and s["adjRandIndex"]["sd"] == 0.0
    assert s["numClusters"]["mean"] == len(np.unique(link)) and s["numClusters"]["sd"] == 0.0


def test_one_record_has_no_adjusted_rand_index():
    from dblink_b200 import analysis_arrays as aa

    ch = aa.ChainArrays(np.arange(1), np.arange(2), [aa.sample_from_links(np.zeros(1, np.int32), np.zeros(1))] * 2)
    rows = sample_rows(ch, np.zeros(1, np.int64))
    assert all(math.isnan(r["adjRandIndex"]) and r["numClusters"] == 1 for r in rows)
    assert aa.posterior_summary(rows)["adjRandIndex"]["undefined"] == 2


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
    {name : "evaluate", parameters : { lowerIterationCutoff : 10, metrics : %s }}
  ]
}
"""


def test_config_accepts_the_posterior_metrics():
    from dblink_b200 import config
    from dblink_b200.project import Project

    def steps(metrics):
        return Project(config.parse_string(CONF % ("x.csv", "out/", 1, metrics)), base_dir="").steps()

    (name, prm), = steps('["posterior-cluster", "pairwise", "posterior-pairwise"]')
    assert name == "evaluate" and prm["metrics"] == ["posterior-cluster", "pairwise", "posterior-pairwise"]
    for bad in ('["accuracy"]', '["posterior-pairwise", "accuracy"]', "[]"):
        with pytest.raises(ValueError, match="metrics"):
            steps(bad)
    p = Project(config.parse_string(CONF % ("x.csv", "out/", 1, '["cluster", "posterior-pairwise"]')), base_dir="")
    assert p.steps_mk_string().splitlines()[2:] == [
        "  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= 10) using {'cluster'} "
        "metrics",
        "  * EvaluateStep: Evaluating every sample of the chain for iterations >= 10 using {'posterior-pairwise'} "
        "metrics"]


def test_abi_checks_before_any_device_work():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Evaluation

    L = _lib.load()
    truth = np.zeros(4, np.int32)
    h = C.c_void_p()
    assert L.dbl_eval_create(None, 4, truth.ctypes.data, 1) == _lib.ERR_INVALID
    for R, t, S in ((0, truth, 1), (-3, truth, 1), (1 << 31, truth, 1), (4, None, 1), (4, truth, 0), (4, truth, -1)):
        assert L.dbl_eval_create(C.byref(h), R, None if t is None else t.ctypes.data, S) == _lib.ERR_INVALID and not h
    assert L.dbl_eval_add_sample(None, truth.ctypes.data) == _lib.ERR_INVALID
    assert L.dbl_eval_read(None, None, None, None) == _lib.ERR_INVALID
    assert L.dbl_eval_num_samples(None) == 0
    L.dbl_eval_free(None)
    with pytest.raises(ValueError, match="one label per record"):
        Evaluation(4, np.zeros(3, np.int32), 1)


def test_eval_needs_a_device():
    import torch

    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Evaluation
    from dblink_b200.engine import DblinkError

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(DblinkError) as e:
        Evaluation(4, np.zeros(4, np.int32), 2)
    assert e.value.status == _lib.ERR_CUDA
    h = C.c_void_p()
    assert _lib.load().dbl_eval_create(C.byref(h), 4, np.zeros(4, np.int32).ctypes.data, 2) == _lib.ERR_CUDA and not h


# 6 records, truth {r0,r1} {r2,r3} {r4} {r5}; the samples of test_summary_by_hand at iterations 10, 20, 30, after one
# at iteration 0 that the cutoff drops
CHAIN = [(0, [0, 0, 0, 0, 0, 0]), (10, [0, 1, 2, 3, 4, 5]), (20, [0, 0, 2, 2, 4, 5]), (30, [0, 0, 0, 3, 4, 4])]

SAMPLES_CSV = """iteration,numClusters,TP,FP,FN,precision,recall,f1score,adjRandIndex
10,6,0,0,2,nan,0.0,0.0,0.0
20,4,2,0,0,1.0,1.0,1.0,1.0
30,3,1,3,1,0.25,0.5,0.3333333333333333,0.18918918918918917
"""

# the sections of metrics ["posterior-cluster", "posterior-pairwise"] over the samples above (adjusted Rand indices
# 0, 1 and 7/37; precisions undefined, 1 and 1/4; numbers checked by hand in test_summary_by_hand)
RESULTS_TXT = """=====================================
      Posterior cluster metrics
-------------------------------------
 Samples:         3
 Adj. Rand index: 0.3963963963963964 (sd 0.5312260536146151, 95% interval [0.00945945945945946, 0.9594594594594594], median 0.18918918918918917)
 Clusters:        4.333333333333333 (sd 1.5275252316519465, 95% interval [3.05, 5.9], median 4.0) (true: 4)
=====================================

=====================================
     Posterior pairwise metrics
-------------------------------------
 Samples:         3
 Precision:       0.625 (sd 0.5303300858899106, 95% interval [0.26875, 0.98125], median 0.625), undefined in 1 samples
 Recall:          0.5 (sd 0.5, 95% interval [0.025, 0.975], median 0.5)
 F1-score:        0.4444444444444444 (sd 0.5091750772173156, 95% interval [0.016666666666666666, 0.9666666666666667], median 0.3333333333333333)
=====================================

"""  # noqa: E501


def write_project(tmp_path, chains, metrics):
    from dblink_b200 import config, writers as w
    from dblink_b200.project import Project

    data = os.path.join(tmp_path, "data.csv")
    with open(data, "w") as fh:
        fh.write("rec_id,ent_id,a\n" + "".join(f"r{i},e{t},v{i % 2}\n" for i, t in enumerate([0, 0, 1, 1, 2, 3])))
    out = str(tmp_path / "out") + "/"
    p = Project(config.parse_string(CONF % (data, out, chains, metrics)), base_dir="")
    ids = ["r%d" % i for i in range(6)]
    for k, dr in enumerate(p.chain_dirs()):
        lw = w.LinkageChainWriter(os.path.join(dr, "linkage-chain.parquet"))
        for it, link in CHAIN if k == 0 else CHAIN[:1] + CHAIN[2:3]:
            lw.append(it, w.linkage_structure_arrow(np.array(link, np.int32), np.zeros(6, np.int32), ids))
        lw.close()
    return p, out


def test_project_writes_the_samples_and_the_summary(tmp_path, monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    monkeypatch.setattr(project, "posterior_metric_counts", aa.posterior_metric_counts)
    p, out = write_project(tmp_path, 1, '["posterior-cluster", "posterior-pairwise"]')
    res = p.execute(log=lambda *a: None)
    assert open(out + "evaluation-samples.csv").read() == SAMPLES_CSV
    assert open(out + "evaluation-results.txt").read() == RESULTS_TXT
    assert not os.path.exists(out + "shared-most-probable-clusters.csv")  # no sMPC metric, no sMPC
    assert res["posterior-pairwise"]["precision"]["undefined"] == 1 and res["posterior-cluster"]["trueNumClusters"] == 4
    assert set(res) == {"posterior-pairwise", "posterior-cluster"}


def test_two_chains_write_their_samples_and_pool_the_summary(tmp_path, monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    monkeypatch.setattr(project, "posterior_metric_counts", aa.posterior_metric_counts)
    p, out = write_project(tmp_path, 2, '["posterior-pairwise"]')
    res = p.execute(log=lambda *a: None)
    lines = SAMPLES_CSV.splitlines(keepends=True)
    assert open(out + "chain-0/evaluation-samples.csv").read() == SAMPLES_CSV
    assert open(out + "chain-1/evaluation-samples.csv").read() == lines[0] + lines[2]
    r = res["posterior-pairwise"]["recall"]
    assert r["n"] == 4 and r["mean"] == 0.625 and r["median"] == 0.75  # recalls 0, 1, 0.5 and 1
    assert " Samples:         4\n" in open(out + "evaluation-results.txt").read()
    assert not os.path.exists(out + "evaluation-samples.csv")
