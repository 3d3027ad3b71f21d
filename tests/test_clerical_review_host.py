"""The clerical review of a point estimate on the host (analysis_arrays.record_links / cluster_appearances /
ClericalReview) against the literal restatement in analysis.py, its identities (W is the sum of the sample cluster
sizes, I sums to twice K, the cluster losses add up to the Binder loss), every tie rule, the config refusals, and the
project's files and evaluation on RLdata500."""
import gzip
import os
import shutil
from fractions import Fraction

import numpy as np
import pytest

from test_binder_host import chain_of, project_of
from test_match_probabilities_host import as_set_chain, random_chain

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def review_of(ch, labels, t=0.5):
    from dblink_b200 import analysis_arrays as aa

    labels = aa.canonical_clusters(labels)
    first, second, count = aa.pairwise_match_counts(ch)
    links = aa.record_links(first, second, count, labels, int(labels.max()) + 1)
    return aa.ClericalReview(links, aa.cluster_appearances(ch, labels), labels, len(ch.samples), t), links


def assert_equal_to_literal(ch, labels, t=0.5):
    from dblink_b200 import analysis

    rv, links = review_of(ch, labels, t)
    chain, ids = as_set_chain(ch)
    center = [frozenset(ids[i] for i in np.flatnonzero(rv.labels == k)) for k in range(len(rv.size))]
    recs, clusters, order = analysis.clerical_review(chain, center, t, ids)
    S = len(ch.samples)
    for i, r in enumerate(ids):
        want = recs[r]
        assert (links.W[i], links.I[i], rv.record_appearances[i]) == (want["W"], want["I"], want["A"])
        assert (Fraction(int(rv.record_fl[i]), S), Fraction(int(rv.record_ml[i]), S)) == (want["FL"], want["ML"])
        assert (ids[rv.partner[i]] if rv.partner[i] >= 0 else None, rv.partner_count[i]) == (want["partner"],
                                                                                           want["partner_count"])
    for k, want in enumerate(clusters):
        assert rv.size[k] == want["size"] and Fraction(int(rv.appearances[k]), S) == want["probability"]
        assert (Fraction(int(rv.fl[k]), S), Fraction(int(rv.ml[k]), S)) == (want["FL"], want["ML"])
        assert rv.losses()[k] == float(want["loss"])
        assert (None if rv.weakest[k] < 0 else Fraction(int(rv.weakest[k]), S)) == want["weakest"]
        got = (None if rv.inside[k] < 0 else
               (ids[rv.inside[k]], ids[rv.outside[k]], Fraction(int(rv.outside_count[k]), S)))
        assert got == want["strongest"]
    assert rv.order.tolist() == order
    return rv, links


def centers_of(ch, rng):
    from dblink_b200 import analysis_arrays as aa

    R = ch.num_records
    mem, off, _ = ch.samples[len(ch.samples) // 2]
    return [aa.shared_most_probable_clusters(ch), aa.sample_labels(R, mem, off), np.arange(R), np.zeros(R, np.int64),
            rng.integers(0, max(1, R // 3), R)]


@pytest.mark.parametrize("seed", range(6))
def test_numpy_equals_the_literal_restatement(seed):
    rng = np.random.default_rng(seed)
    R, S = int(rng.integers(1, 28)), int(rng.integers(1, 9))
    ch = random_chain(R, S, seed)
    for labels in centers_of(ch, rng):
        for t in (0.5, 0.0, 1.0, 0.7):
            assert_equal_to_literal(ch, labels, t)


def test_all_singletons_and_one_giant_cluster():
    singles = chain_of([[0, 1, 2, 3, 4]] * 3)
    rv, links = assert_equal_to_literal(singles, np.arange(5))
    assert (links.W == 0).all() and (rv.record_appearances == 3).all() and (rv.partner == -1).all()
    assert (rv.weakest == -1).all() and (rv.inside == -1).all() and rv.order.tolist() == [0, 1, 2, 3, 4]
    giant = chain_of([[0, 0, 0, 0, 0], [0, 0, 0, 2, 2]])
    rv, links = assert_equal_to_literal(giant, np.zeros(5, np.int64))
    assert rv.size.tolist() == [5] and rv.appearances.tolist() == [1] and rv.weakest.tolist() == [1]
    rv, _ = assert_equal_to_literal(giant, np.arange(5))  # every pair of the giant cluster is a missed link
    assert rv.ml.tolist() == [4 + 2, 4 + 2, 4 + 2, 4 + 1, 4 + 1] and (rv.fl == 0).all()


def test_a_sample_as_the_center_has_no_error_when_it_is_the_only_sample():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(40, 1, seed=3)
    mem, off, _ = ch.samples[0]
    rv, _ = assert_equal_to_literal(ch, aa.sample_labels(40, mem, off))
    assert (rv.fl == 0).all() and (rv.ml == 0).all() and (rv.record_appearances == 1).all()
    assert (rv.record_fl == 0).all() and (rv.record_ml == 0).all()


@pytest.mark.parametrize("seed", range(4))
def test_the_identities(seed):
    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(seed)
    ch = random_chain(200, 11, seed + 50)
    first, second, count = aa.pairwise_match_counts(ch)
    S, C = len(ch.samples), int(count.sum())
    # W(i) = sum over the samples of (|C_s(i)| - 1)
    W = np.zeros(200, np.int64)
    for mem, off, _ in ch.samples:
        W[mem] += np.repeat(np.diff(off) - 1, np.diff(off))
    for labels in centers_of(ch, rng):
        for t in (0.5, 0.25, 0.1):
            rv, links = review_of(ch, labels, t)
            assert np.array_equal(links.W, W)
            n, K = aa.search_result_counts(first, second, count, rv.labels)
            assert int(links.I.sum()) == 2 * K
            a, b = Fraction(t).numerator, Fraction(t).denominator
            total = sum(Fraction(a * int(f) * 2 + (b - a) * int(m), 2 * b * S) for f, m in zip(rv.fl, rv.ml))
            assert total == Fraction((b - a) * C + a * S * n - b * K, b * S)
            assert abs(float(total) - aa.expected_losses(n, K, C, S, t)) <= 1e-9 * max(1.0, float(total))


def test_every_tie_rule():
    from dblink_b200 import analysis_arrays as aa

    # record 0's partners 1 and 2 each linked in 1 of 2 samples: the smaller partner wins
    ch = chain_of([[0, 0, 2, 3], [0, 1, 0, 3]])
    rv, links = assert_equal_to_literal(ch, np.arange(4))
    assert (links.partner[0], links.partner_count[0]) == (1, 1)
    # cluster {0, 3}: its members 0 and 3 both reach an outside record with count 1: the smaller inside record wins;
    # record 0 reaches 1 and 2 with count 1: the smaller outside record wins
    ch = chain_of([[0, 0, 0, 3], [0, 1, 1, 1]])
    rv, _ = assert_equal_to_literal(ch, [0, 1, 2, 0])
    k = rv.labels[0]
    assert (rv.inside[k], rv.outside[k], rv.outside_count[k]) == (0, 1, 1)
    # equal losses: the smaller cluster first
    rv, _ = assert_equal_to_literal(chain_of([[0, 0, 2, 2]]), [0, 1, 2, 3])
    assert rv.order.tolist() == [0, 1, 2, 3]
    # the review order compares exactly, past int64: a S FL + (b - a) S ML with t = 0.1 (b = 2^55)
    assert aa.review_order([3, 0], [0, 1 << 40], 0.1).tolist() == [1, 0]
    assert aa.review_order([1 << 62, 1 << 62], [0, 1], 1e-300).tolist() == [1, 0]
    # weakest internal link: 0 when a pair of the cluster was never linked
    rv, _ = assert_equal_to_literal(chain_of([[0, 0, 2], [0, 1, 1]]), [0, 0, 0])
    assert rv.weakest.tolist() == [0]
    rv, _ = assert_equal_to_literal(chain_of([[0, 0, 2], [0, 0, 0]]), [0, 0, 1])
    assert rv.weakest.tolist() == [2, -1]


def test_non_canonical_labels_are_refused():
    from dblink_b200 import analysis_arrays as aa

    ch = chain_of([[0, 0, 2, 3]])
    first, second, count = aa.pairwise_match_counts(ch)
    for labels, C in (([0, 0, 2, 3], 4), ([0, 0, 1, 4], 4), ([0, -1, 1, 2], 3), ([0, 0, 1, 1], 3)):
        with pytest.raises(ValueError, match="cluster"):
            aa.record_links(first, second, count, labels, C)
    with pytest.raises(ValueError, match="not canonical"):
        aa.cluster_appearances(ch, [0, 0, 2, 3])


def test_erroneous_clusters_and_the_evaluation():
    from dblink_b200 import analysis_arrays as aa

    truth = np.array([7, 7, 5, 5, 9, 3])
    # clusters {0, 1} exact, {2} half of 5, {3, 4} two entities, {5} exact
    labels = np.array([0, 0, 1, 2, 2, 3])
    assert aa.erroneous_clusters(labels, truth).tolist() == [False, True, True, False]

    class Review:
        pass

    rv = Review()
    rv.labels, rv.order, rv.appearances = labels, np.array([2, 0, 1, 3]), np.array([1, 5, 3, 3])
    rows, res = aa.clerical_review_evaluation(rv, truth)
    assert rows == [[1, 2, 1, 1], [2, 0, 0, 1], [3, 1, 1, 2], [4, 3, 0, 2]]
    # one of the two erroneous clusters in the first ceil(p 4 / 100) = 1 position; area: the (erroneous, correct)
    # pairs in that order, (2 before 0, 2 before 3, 1 before 3) of 4
    assert res == dict(clusters=4, erroneous=2, found=[0.5, 0.5, 0.5], area=0.75, baseline=[0.0, 0.0, 0.0])
    rv.labels, rv.order, rv.appearances = np.array([0, 1]), np.array([0, 1]), np.array([1, 1])
    res = aa.clerical_review_evaluation(rv, np.array([4, 5]))[1]
    assert res["erroneous"] == 0 and all(np.isnan(x) for x in res["found"] + res["baseline"] + [res["area"]])


def test_config_refusals_and_defaults(tmp_path):
    (_, s), (_, e) = project_of(tmp_path, quantities='["clerical-review"]', metrics='["clerical-review"]').steps()
    assert s["clerical_review_center"] == e["clerical_review_center"] == "shared-most-probable-clusters"
    extra = ', clericalReviewCenter : "vi-search-clusters"'
    (_, s), (_, e) = project_of(tmp_path, summarize_extra=extra, evaluate_extra=extra).steps()
    assert s["clerical_review_center"] == e["clerical_review_center"] == "vi-search-clusters"
    for bad in ('clericalReviewCenter : "clerical-review"', 'clericalReviewCenter : "sMPC"'):
        for kw in (dict(summarize_extra=", " + bad), dict(evaluate_extra=", " + bad)):
            with pytest.raises(ValueError, match="^clericalReviewCenter must be one of"):
                project_of(tmp_path, quantities='["clerical-review"]', metrics='["clerical-review"]', **kw).steps()
    for bad in ("-0.1", "1.5"):
        for kw in (dict(summarize_extra=", falseLinkCost : " + bad), dict(evaluate_extra=", falseLinkCost : " + bad)):
            with pytest.raises(ValueError, match=r"^falseLinkCost must be in \[0, 1\]\.$"):
                project_of(tmp_path, quantities='["clerical-review"]', metrics='["clerical-review"]', **kw).steps()


def write_rldata500_chain(tmp_path, p, S=12, seed=0):
    """RLdata500 as the data and a chain of S samples around its truth: each sample relinks a fifth of the records."""
    import csv

    from dblink_b200 import writers as w

    with gzip.open(os.path.join(GOLDEN, "RLdata500.csv.gz"), "rt") as fh:
        rows = list(csv.DictReader(fh))
    with open(os.path.join(tmp_path, "data.csv"), "w") as fh:
        fh.write("rec_id,ent_id,a\n" + "".join(f"{r['rec_id']},{r['ent_id']},v\n" for r in rows))
    ids = [r["rec_id"] for r in rows]
    _, truth = np.unique([r["ent_id"] for r in rows], return_inverse=True)
    R, E = len(ids), int(truth.max()) + 1
    rng = np.random.default_rng(seed)
    lw = w.LinkageChainWriter(os.path.join(p.chain_dirs()[0], "linkage-chain.parquet"))
    for s in range(S):
        link = truth.copy()
        move = rng.random(R) < 0.2
        link[move] = rng.integers(0, E, int(move.sum()))
        lw.append(10 * (s + 1), w.linkage_structure_arrow(link.astype(np.int32), np.zeros(R, np.int32), ids))
    lw.close()
    return ids, truth


def output_files(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            path = os.path.join(d, f)
            out[os.path.relpath(path, root)] = open(path, "rb").read()
    return out


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("vi_cross_histograms", "shared_most_probable_clusters", "pairwise_match_counts",
                 "posterior_metric_counts", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)
    monkeypatch.setattr(project, "cluster_appearances", aa.cluster_appearances)
    monkeypatch.setattr(project, "record_links", lambda ch, labels: aa.record_links(
        *aa.pairwise_match_counts(ch), labels, int(np.max(labels)) + 1))


@pytest.mark.parametrize("center", ["shared-most-probable-clusters", "vi-clusters"])
def test_project_writes_the_review_on_rldata500(tmp_path, monkeypatch, center):
    from dblink_b200 import analysis, analysis_arrays as aa, project

    host_paths(monkeypatch)
    extra = f', clericalReviewCenter : "{center}", falseLinkCost : 0.25'
    p = project_of(tmp_path, quantities='["clerical-review", "partition-sizes", "shared-most-probable-clusters"]',
                   metrics='["pairwise", "clerical-review"]', summarize_extra=extra, evaluate_extra=extra)
    ids, truth = write_rldata500_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    ch = p.read_chain(10)
    S, R = len(ch.samples), ch.num_records
    chain_ids = [str(x) for x in ch.record_ids.to_pylist()]
    labels = aa.canonical_clusters(project.credible_ball_center(ch, center, 0.25, 1000))
    C = int(labels.max()) + 1
    center_sets = [frozenset(chain_ids[i] for i in np.flatnonzero(labels == k)) for k in range(C)]
    chain, _ = as_set_chain(ch)
    recs, clusters, order = analysis.clerical_review(chain, center_sets, 0.25, chain_ids)

    assert open(out + "clerical-review-clusters.csv").read().splitlines() == [
        ", ".join(sorted(c)) for c in center_sets]
    lines = open(out + "clerical-review.csv").read().splitlines()
    assert lines[0] == ("rank,cluster,size,clusterProbability,expectedFalseLinks,expectedMissedLinks,expectedLoss,"
                        "weakestInternalLinkProbability,strongestLinkInsideRecordId,strongestLinkOutsideRecordId,"
                        "strongestOutsideLinkProbability")
    assert len(lines) == C + 1 and C > 50
    for rank, (line, k) in enumerate(zip(lines[1:], order), 1):
        w = clusters[k]
        top = w["strongest"]
        assert line.split(",") == [
            str(rank), str(k), str(w["size"]), repr(float(w["probability"])), repr(float(w["FL"])),
            repr(float(w["ML"])), repr(float(w["loss"])), "" if w["weakest"] is None else repr(float(w["weakest"])),
            "" if top is None else top[0], "" if top is None else top[1], "" if top is None else repr(float(top[2]))]
    records = open(out + "clerical-review-records.csv").read().splitlines()
    assert records[0] == ("recordId,cluster,clusterProbability,expectedFalseLinks,expectedMissedLinks,"
                          "strongestOutsideRecordId,strongestOutsideLinkProbability")
    assert len(records) == R + 1
    for i, line in enumerate(records[1:]):
        w = recs[chain_ids[i]]
        assert line.split(",") == [chain_ids[i], str(labels[i]), repr(w["A"] / S), repr(float(w["FL"])),
                                   repr(float(w["ML"])), w["partner"] or "",
                                   "" if w["partner"] is None else repr(w["partner_count"] / S)]

    # the evaluation: erroneous = not exactly a true entity, counted along the queue
    ent = dict(zip(ids, truth))
    true_sets = {frozenset(r for r in chain_ids if ent[r] == e) for e in set(truth.tolist())}
    err = [c not in true_sets for c in center_sets]
    ev = open(out + "clerical-review-evaluation.csv").read().splitlines()
    assert ev[0] == "rank,cluster,erroneous,erroneousFound"
    found = np.cumsum([err[k] for k in order])
    assert ev[1:] == [f"{r + 1},{k},{int(err[k])},{found[r]}" for r, k in enumerate(order)]
    E = sum(err)
    r = res["clerical-review"]
    assert (r["center"], r["clusters"], r["erroneous"]) == (center, C, E) and 0 < E < C
    assert r["found"] == [found[-(-q * C // 100) - 1] / E for q in (1, 5, 10)]
    worse = sum(1 for a in range(C) for b in range(a + 1, C) if err[order[a]] and not err[order[b]])
    assert r["area"] == worse / (E * (C - E))
    by_p = sorted(range(C), key=lambda k: (clusters[k]["probability"], k))
    base = np.cumsum([err[k] for k in by_p])
    assert r["baseline"] == [base[-(-q * C // 100) - 1] / E for q in (1, 5, 10)]
    text = open(out + "evaluation-results.txt").read()
    assert analysis.format_clerical_review(r) in text and " not a true entity\n" in text

    run = p.steps_mk_string().splitlines()
    settings = f"clericalReviewCenter={center}, ranked at falseLinkCost=0.25"
    assert ("  * SummarizeStep: clerical-review ranks the clusters of a point estimate by their expected false and "
            f"missed links, with {settings}") in run
    assert ("  * EvaluateStep: Evaluating how soon the clerical review queue of a point estimate reaches its clusters "
            f"that are not a true entity ({settings}, iterations >= 10) using {{'clerical-review'}} metrics") in run

    # every other file is the one a run without the quantity and metric writes
    q = project_of(tmp_path, quantities='["partition-sizes", "shared-most-probable-clusters"]', metrics='["pairwise"]',
                   summarize_extra=extra, evaluate_extra=extra, out="out2")
    os.makedirs(q.output_path, exist_ok=True)
    shutil.copytree(os.path.join(p.output_path, "linkage-chain.parquet"),
                    os.path.join(q.output_path, "linkage-chain.parquet"))
    q.execute(log=lambda *a: None)
    with_q, without = output_files(out), output_files(str(tmp_path / "out2") + "/")
    assert set(with_q) - set(without) == {"clerical-review.csv", "clerical-review-records.csv",
                                          "clerical-review-clusters.csv", "clerical-review-evaluation.csv"}
    assert with_q.pop("evaluation-results.txt").startswith(without.pop("evaluation-results.txt"))
    assert len(without) > 2 and all(with_q[f] == without[f] for f in without)


def test_an_empty_chain_is_refused():
    from dblink_b200 import project

    ch = chain_of([[0, 0, 2]])
    with pytest.raises(ValueError, match="clerical review needs at least one sample"):
        project.clerical_review_estimate(type(ch)(ch.record_ids, np.zeros(0, np.int64), []),
                                         "shared-most-probable-clusters", 0.5, 10)


def test_abi_refuses_a_null_handle():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Pairs, Posterior

    L = _lib.load()
    labels = np.zeros(4, np.int32)
    out64, out32 = np.zeros(4, np.int64), np.zeros(4, np.int32)
    assert L.dbl_pairs_record_links(None, labels.ctypes.data, 1, *(a.ctypes.data for a in
                                                                   (out64, out64, out32, out32, out64, out32))) \
        == _lib.ERR_INVALID
    assert L.dbl_posterior_cluster_counts(None, labels.ctypes.data, 1, out32.ctypes.data) == _lib.ERR_INVALID
    assert (out64 == 0).all() and (out32 == 0).all()
    for cls, call in ((Pairs, lambda h: h.record_links(np.zeros(5, np.int32), 1)),
                      (Posterior, lambda h: h.cluster_counts(np.zeros(5, np.int32), 1))):
        h = cls.__new__(cls)  # an owner without a handle: the shape check comes first
        h.num_records = 4
        with pytest.raises(ValueError, match="one cluster label per record"):
            call(h)
