"""The credible ball on the host: the numpy distances (vi_sample_cells, credible_ball_distances) and ball
(credible_ball) against the literal analysis.credible_ball (entropies over sets, every record pair enumerated) on random
small chains; the identities that tie the per-sample cells to the existing histograms; the radius rule, its ties and
the tie rule of every bound; the config refusals; the files, run.txt lines and evaluation lines that Project.execute
writes on RLdata500; the C ABI's NULL-handle refusal."""
import gzip
import os

import numpy as np
import pytest

from test_binder_host import chain_of, project_of
from test_match_probabilities_host import as_set_chain, random_chain

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
BOUNDS = ("vertical-upper", "horizontal-upper", "horizontal-lower")


def numpy_ball(ch, labels, level):
    """{distance: (distances, radius, in-ball mask, bounds)} of the numpy path around labels."""
    from dblink_b200 import analysis_arrays as aa

    width = aa.vi_width(ch)
    G = aa.VISamples(ch).score_samples(labels, width)
    g = aa.vi_cluster_histograms(ch, width)
    d = aa.credible_ball_distances(np.bincount(np.bincount(labels)), g, G, ch.num_records)
    k = [len(off) - 1 for _, off, _ in ch.samples]
    return {name: (x,) + aa.credible_ball(x, k, level) for name, x in zip(("vi", "binder"), d)}


def centers_of(ch, rng):
    from dblink_b200 import analysis_arrays as aa

    R = ch.num_records
    mem, off, _ = ch.samples[len(ch.samples) // 2]
    return [aa.sample_labels(R, mem, off), aa.shared_most_probable_clusters(ch), np.arange(R),
            np.zeros(R, np.int64), rng.integers(0, max(R // 2, 1), R)]


@pytest.mark.parametrize("seed", range(10))
def test_numpy_equals_the_literal_ball(seed):
    from dblink_b200 import analysis

    rng = np.random.default_rng(seed)
    R, S = int(rng.integers(1, 30)), [1, 2, 3, 7, 12][seed % 5]
    ch = random_chain(R, S, seed=5000 + seed)
    chain, ids = as_set_chain(ch)
    for labels in centers_of(ch, rng):
        center = [frozenset(ids[i] for i in np.flatnonzero(labels == x)) for x in np.unique(labels)]
        for level in (0.1, 0.5, 0.7, 0.95, 1.0):
            got = numpy_ball(ch, labels, level)
            want = analysis.credible_ball(chain, center, level)
            for name in ("vi", "binder"):
                d, radius, inside, bounds = got[name]
                w = want[name]
                if name == "binder":
                    assert d.dtype == np.int64 and d.tolist() == w["distances"] and radius == w["radius"]
                else:
                    assert d.dtype == np.float64 and np.abs(d - w["distances"]).max() <= 1e-12
                    assert abs(radius - w["radius"]) <= 1e-12
                assert inside.tolist() == w["in_ball"] and bounds == w["bounds"]


def test_a_sample_is_at_distance_zero_from_itself():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 9, seed=3)
    for t, (mem, off, _) in enumerate(ch.samples):
        balls = numpy_ball(ch, aa.sample_labels(300, mem, off), 0.5)
        assert balls["vi"][0][t] == 0.0 and balls["binder"][0][t] == 0
        assert (balls["vi"][0] >= 0).all() and (balls["binder"][0] >= 0).all()


@pytest.mark.parametrize("R,S", [(1, 1), (7, 4), (400, 13)])
def test_the_cells_per_sample_add_up_to_the_existing_histograms(R, S):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(R, S, seed=R + S)
    width = aa.vi_width(ch)
    rng = np.random.default_rng(R)
    for labels in centers_of(ch, rng):
        G = aa.vi_sample_cells(ch, labels, width)
        assert G.dtype == np.int64 and G.shape == (S, width) and (G[:, :2] == 0).all()
        assert G.sum(axis=0).tolist() == aa.vi_label_cells(ch, labels, width).tolist()
    # c = C_t: the rows s != t are the cells of C_t ^ C_s, which vi_cross_histograms sums into its row t
    cross = aa.vi_cross_histograms(ch)
    for t, (mem, off, _) in enumerate(ch.samples):
        G = aa.vi_sample_cells(ch, aa.sample_labels(R, mem, off), width)
        assert (G.sum(axis=0) - G[t]).tolist() == cross[t].tolist()
        assert G[t].tolist() == aa.vi_cluster_histograms(ch, width)[t].tolist()


def test_the_linked_pairs_of_the_cells_are_the_binder_count_sum():
    """The pairs c ^ C_s links, summed over s, are K(c): the sum over c's pairs of their match counts."""
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(500, 11, seed=21)
    first, second, count = aa.pairwise_match_counts(ch)
    width = aa.vi_width(ch)
    n = np.arange(width)
    for labels in centers_of(ch, np.random.default_rng(2)):
        G = aa.vi_sample_cells(ch, labels, width)
        _, K = aa.search_result_counts(first, second, count, labels)
        assert int((G * (n * (n - 1) // 2)).sum()) == K


def test_the_radius_rule_and_its_ties():
    from dblink_b200 import analysis_arrays as aa

    assert [aa.credible_level_rank(p, 10) for p in (0.1, 0.7, 0.95, 1)] == [1, 7, 10, 10]
    assert [aa.credible_level_rank(p, 1) for p in (0.1, 0.7, 0.95, 1)] == [1, 1, 1, 1]
    assert aa.credible_level_rank(0.3, 10) == 3 and aa.credible_level_rank(0.01, 100) == 1
    d = np.array([5, 1, 3, 3, 9, 0, 3, 7, 2, 8], np.int64)
    k = np.arange(10) % 3 + 1
    for level, radius, members in ((0.1, 0, [5]), (0.2, 1, [1, 5]), (0.5, 3, [1, 2, 3, 5, 6, 8]),
                                   (0.7, 5, [0, 1, 2, 3, 5, 6, 8]), (0.95, 9, list(range(10))),
                                   (1, 9, list(range(10)))):
        r, inside, _ = aa.credible_ball(d, k, level)
        assert r == radius and np.flatnonzero(inside).tolist() == members
    # S = 1: every level gives the one sample
    for level in (0.1, 0.7, 0.95, 1):
        r, inside, b = aa.credible_ball(np.array([0.25]), [4], level)
        assert r == 0.25 and inside.tolist() == [True] and b == {x: (0, 1) for x in BOUNDS}
    for bad in (0, -0.5, 1.5):
        with pytest.raises(ValueError, match=r"^credibleLevel must be in \(0, 1\]\.$"):
            aa.credible_ball(d, k, bad)


def test_the_tie_rule_of_every_bound():
    """Samples 2, 4 and 6 tie at the largest distance; among the fewest clusters (2: samples 1, 4, 6) 4 and 6 are the
    farthest; among the most (5: samples 0, 2, 3) 2 is the farthest.  The earliest sample wins every tie."""
    from dblink_b200 import analysis_arrays as aa

    d = np.array([0.5, 0.25, 1.0, 0.75, 1.0, 0.0, 1.0, 2.0])
    k = np.array([5, 2, 5, 5, 2, 3, 2, 1])
    r, inside, b = aa.credible_ball(d, k, 0.875)
    assert r == 1.0 and inside.tolist() == [True] * 7 + [False]
    assert b == {"vertical-upper": (2, 3), "horizontal-upper": (4, 2), "horizontal-lower": (2, 1)}
    # ties in both keys of a horizontal bound
    r, _, b = aa.credible_ball(np.array([3, 3, 1, 3]), np.array([4, 4, 4, 2]), 1)
    assert b == {"vertical-upper": (0, 3), "horizontal-upper": (3, 1), "horizontal-lower": (0, 2)}


def test_config_refusals_and_defaults(tmp_path):
    (_, s), (_, e) = project_of(tmp_path, quantities='["credible-ball"]', metrics='["credible-ball"]').steps()
    assert (s["credible_ball_center"], s["credible_level"]) == ("vi-search-clusters", 0.95)
    assert (e["credible_ball_center"], e["credible_level"]) == ("vi-search-clusters", 0.95)
    (_, s), (_, e) = project_of(tmp_path, quantities='["credible-ball"]',
                                summarize_extra=', credibleBallCenter : "binder-clusters", credibleLevel : 0.5',
                                evaluate_extra=", credibleLevel : 1").steps()
    assert (s["credible_ball_center"], s["credible_level"], e["credible_level"]) == ("binder-clusters", 0.5, 1.0)
    for extra in ('credibleBallCenter : "credible-ball"', 'credibleBallCenter : "sMPC"'):
        for kw in (dict(summarize_extra=", " + extra), dict(evaluate_extra=", " + extra)):
            with pytest.raises(ValueError, match="^credibleBallCenter must be one of"):
                project_of(tmp_path, **kw).steps()
    for bad in ("0", "-0.25", "1.5", "true"):
        for kw in (dict(summarize_extra=", credibleLevel : " + bad), dict(evaluate_extra=", credibleLevel : " + bad)):
            with pytest.raises(ValueError, match=r"^credibleLevel must be in \(0, 1\]\.$"):
                project_of(tmp_path, **kw).steps()


def write_rldata500_chain(tmp_path, p, S=12, seed=0):
    """RLdata500 as the data and a chain of S samples around its truth: each sample relinks a fifth of the records
    and merges a few entities."""
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


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("vi_cross_histograms", "shared_most_probable_clusters", "pairwise_match_counts",
                 "posterior_metric_counts", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)


def test_project_writes_the_ball_on_rldata500(tmp_path, monkeypatch):
    from dblink_b200 import analysis, analysis_arrays as aa, project

    host_paths(monkeypatch)
    extra = ', credibleBallCenter : "shared-most-probable-clusters", credibleLevel : 0.75'
    p = project_of(tmp_path, quantities='["credible-ball", "partition-sizes"]', metrics='["pairwise", "credible-ball"]',
                   summarize_extra=extra, evaluate_extra=extra)
    ids, truth = write_rldata500_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    ch = p.read_chain(10)
    S, R = len(ch.samples), ch.num_records
    assert (S, R) == (12, 500)
    smpc = aa.shared_most_probable_clusters(ch)
    chain, chain_ids = as_set_chain(ch)
    center = [frozenset(chain_ids[i] for i in np.flatnonzero(smpc == x)) for x in np.unique(smpc)]
    want = analysis.credible_ball(chain, center, 0.75)

    samples = open(out + "credible-ball-samples.csv").read().splitlines()
    assert samples[0] == "chain,iteration,numClusters,viDistance,binderDistance" and len(samples) == S + 1
    for s, line in enumerate(samples[1:]):
        k, it, n, v, b = line.split(",")
        assert (int(k), int(it), int(n)) == (0, 10 * (s + 1), len(ch.samples[s][1]) - 1)
        assert abs(float(v) - want["vi"]["distances"][s]) <= 1e-12 and int(b) == want["binder"]["distances"][s]

    ball = open(out + "credible-ball.csv").read().splitlines()
    assert ball[0] == ("distance,bound,center,level,radius,samplesInBall,samples,chain,iteration,numClusters,"
                       "distanceToCenter,ties")
    assert [tuple(x.split(",")[:2]) for x in ball[1:]] == [(d, b) for d in ("vi", "binder") for b in BOUNDS]
    for line in ball[1:]:
        name, bound, c, level, radius, inside, samples_, k, it, n, dist, ties = line.split(",")
        w = want[name]
        s, t = w["bounds"][bound]
        assert (c, level, int(inside), int(samples_), int(k), int(it), int(ties)) == (
            "shared-most-probable-clusters", "0.75", sum(w["in_ball"]), S, 0, 10 * (s + 1), t)
        assert int(n) == len(ch.samples[s][1]) - 1
        if name == "binder":
            assert (int(radius), int(dist)) == (w["radius"], w["distances"][s])
        else:
            assert abs(float(radius) - w["radius"]) <= 1e-12 and abs(float(dist) - w["distances"][s]) <= 1e-12
        mem, off, _ = ch.samples[s]
        want_lines = sorted(", ".join(sorted(chain_ids[i] for i in mem[off[c]:off[c + 1]])) for c in range(len(off) - 1))
        assert sorted(open(out + f"credible-ball-{name}-{bound}.csv").read().splitlines()) == want_lines

    # the evaluation: the truth's distances from the center, by one contingency table
    ent = dict(zip(ids, truth))
    truth = np.array([ent[r] for r in chain_ids])  # in the chain's record order, as the center's labels
    tc = [frozenset(chain_ids[i] for i in np.flatnonzero(truth == e)) for e in np.unique(truth)]
    truth_ball = analysis.credible_ball([(0, {0: [list(c) for c in tc]})], center, 1)
    t_vi, t_binder = truth_ball["vi"]["distances"][0], truth_ball["binder"]["distances"][0]
    r = res["credible-ball"]
    assert abs(r["vi"]["truthDistance"] - t_vi) <= 1e-12 and r["binder"]["truthDistance"] == t_binder
    assert (r["center"], r["level"], r["samples"]) == ("shared-most-probable-clusters", 0.75, S)
    for name in ("vi", "binder"):
        assert r[name]["truthInBall"] == (r[name]["truthDistance"] <= r[name]["radius"])
        assert r[name]["samplesInBall"] == sum(want[name]["in_ball"])
    text = open(out + "evaluation-results.txt").read()
    section = text.split("\n\n")[1]
    where = {n: "inside" if r[n]["truthInBall"] else "outside" for n in ("vi", "binder")}
    assert section == (
        "=====================================\n           Credible ball\n"
        "-------------------------------------\n"
        f" Center:          shared-most-probable-clusters, level 0.75, {S} samples\n"
        f" VI:              truth at {r['vi']['truthDistance']!r} bits from the center, radius {r['vi']['radius']!r}, "
        f"{where['vi']} the ball of {r['vi']['samplesInBall']} samples\n"
        f" Binder:          truth at {t_binder} pairs from the center, radius {r['binder']['radius']}, "
        f"{where['binder']} the ball of {r['binder']['samplesInBall']} samples\n"
        "=====================================")
    assert project.credible_ball_truth(smpc, truth) == (r["vi"]["truthDistance"], t_binder)

    run = p.steps_mk_string().splitlines()
    assert ("  * SummarizeStep: credible-ball is the smallest ball around a point estimate, in variation of information "
            "and in Binder distance, that holds a share of the samples, with "
            "credibleBallCenter=shared-most-probable-clusters, credibleLevel=0.75") in run
    assert ("  * EvaluateStep: Evaluating whether the ground truth lies in the credible ball around a point estimate "
            "(credibleBallCenter=shared-most-probable-clusters, credibleLevel=0.75, iterations >= 10) using "
            "{'credible-ball'} metrics") in run


def test_run_txt_names_the_settings_of_the_center(tmp_path):
    def lines(center):
        extra = f', credibleBallCenter : "{center}", falseLinkCost : 0.25, maxSearchRounds : 9'
        p = project_of(tmp_path, quantities='["credible-ball"]', summarize_extra=extra)
        return [x for x in p.steps_mk_string().splitlines() if "credible-ball is" in x][0]

    assert lines("binder-search-clusters").endswith(
        "credibleBallCenter=binder-search-clusters, falseLinkCost=0.25, maxSearchRounds=9, credibleLevel=0.95")
    assert lines("binder-clusters").endswith("credibleBallCenter=binder-clusters, falseLinkCost=0.25, "
                                             "credibleLevel=0.95")
    assert lines("vi-search-clusters").endswith("credibleBallCenter=vi-search-clusters, maxSearchRounds=9, "
                                                "credibleLevel=0.95")
    assert lines("vi-clusters").endswith("credibleBallCenter=vi-clusters, credibleLevel=0.95")
    assert "credible" not in project_of(tmp_path).steps_mk_string()


@pytest.mark.parametrize("center", ["shared-most-probable-clusters", "binder-clusters", "binder-search-clusters",
                                    "vi-clusters", "vi-search-clusters"])
def test_every_center_is_its_own_estimate(tmp_path, monkeypatch, center):
    from dblink_b200 import project

    host_paths(monkeypatch)
    ch = chain_of([[0, 0, 2, 3, 4, 4], [0, 0, 0, 3, 4, 5], [0, 1, 2, 2, 4, 4], [0, 0, 2, 2, 4, 4]])
    labels, k, balls = project.credible_ball_estimate(ch, center, 0.5, 0.5, 100)
    want = {"shared-most-probable-clusters": lambda: project.shared_most_probable_clusters(ch),
            "binder-clusters": lambda: project.binder_estimate(ch, 0.5)[1],
            "binder-search-clusters": lambda: project.binder_search_estimate(ch, 0.5, 100)[1].labels,
            "vi-clusters": lambda: project.vi_estimate(ch)[1],
            "vi-search-clusters": lambda: project.vi_search_estimate(ch, 100)[1].labels}[center]()
    assert labels.tolist() == list(want) and k.tolist() == [4, 4, 4, 3]
    assert set(balls) == {"vi", "binder"}
    with pytest.raises(ValueError, match="at least one sample at or after lowerIterationCutoff"):
        project.credible_ball_estimate(type(ch)(ch.record_ids, np.zeros(0, np.int64), []), center, 0.5, 0.5, 100)


def test_abi_refuses_a_null_handle():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import VI

    L = _lib.load()
    labels = np.zeros(4, np.int32)
    G = np.zeros((2, 8), np.int64)
    assert L.dbl_vi_score_samples(None, labels.ctypes.data, 8, G.ctypes.data) == _lib.ERR_INVALID
    assert (G == 0).all()
    v = VI.__new__(VI)  # an owner without a handle: the shape check comes first
    v.num_records = 4
    with pytest.raises(ValueError, match="one cluster label per record"):
        v.score_samples(np.zeros(5, np.int32), 8)
