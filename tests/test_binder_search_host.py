"""The Binder search on the host: analysis_arrays.binder_search (numpy) against the literal analysis.binder_search
(sets and fractions over every cluster) on random small chains; a brute-force check that no single-record move
lowers the loss of a converged result; J falling every round; truncation by maxSearchRounds; the rounding of t and
the samples x records bound; the summarize quantity binder-search-clusters and the evaluate metrics
binder-search-pairwise / binder-search-cluster with their config and output files; the C ABI's checks that come
before any device work."""
import ctypes as C
import fractions
import itertools
import os

import numpy as np
import pytest

from test_binder_host import CONF, write_chain
from test_match_probabilities_host import as_set_chain, random_chain

TS = (0.0, 0.25, 0.5, 0.7, 1.0)


def starts_of(ch):
    """The two starts the project uses: the Binder sample at t = 1/2 and the sMPC."""
    from dblink_b200 import analysis_arrays as aa

    s = aa.binder_estimate(*aa.binder_counts(ch), 0.5)
    mem, off, _ = ch.samples[s]
    return [aa.sample_labels(ch.num_records, mem, off), aa.shared_most_probable_clusters(ch)]


def as_sets(labels, ids):
    from dblink_b200 import analysis_arrays as aa

    return {frozenset(ids[i] for i in g) for g in aa.labels_to_clusters(labels)}


def literal(ch, t, starts, max_rounds=1000):
    from dblink_b200 import analysis

    chain, ids = as_set_chain(ch)
    return analysis.binder_search(chain, t, [as_sets(s, ids) for s in starts], max_rounds, records=ids)


def assert_equal_to_literal(ch, t, starts, max_rounds=1000):
    from dblink_b200 import analysis_arrays as aa

    best, runs = aa.binder_search(ch, t, starts, max_rounds)
    lit_best, lit = literal(ch, t, starts, max_rounds)
    ids = as_set_chain(ch)[1]
    assert best == lit_best
    for run, want in zip(runs, lit):
        assert as_sets(run.labels, ids) == want["clusters"]
        assert list(run.labels) == list(aa.canonical_labels(run.labels))  # canonical
        assert list(zip(run.moves.tolist(), run.dn.tolist(), run.dK.tolist())) == want["rounds"]
        assert (run.converged, run.n, run.K) == (want["converged"], want["n"], want["K"])
    return best, runs


def literal_loss(ch, t, clusters):
    """E[L] of a partition (sets of ids) by the definition, over every pair of records."""
    chain, ids = as_set_chain(ch)
    count = _counts(chain)
    S = len(chain)
    of = {r: c for c in clusters for r in c}
    loss = fractions.Fraction(0)
    for i, j in itertools.combinations(ids, 2):
        p = fractions.Fraction(count.get(frozenset((i, j)), 0), S)
        loss += t * (1 - p) if of[i] == of[j] else (1 - t) * p
    return loss


def _counts(chain):
    from dblink_b200 import analysis

    out = {}
    for s in chain:
        for c in analysis.clusters_of_sample(s):
            for p in itertools.combinations(c, 2):
                out[frozenset(p)] = out.get(frozenset(p), 0) + 1
    return out


@pytest.mark.parametrize("seed", range(8))
def test_numpy_equals_the_literal_search(seed):
    rng = np.random.default_rng(seed)
    R, S = int(rng.integers(2, 31)), int(rng.integers(1, 9))
    ch = random_chain(R, S, seed=1000 + seed)
    starts = starts_of(ch)
    for t in TS:
        assert_equal_to_literal(ch, t, starts)


def test_singletons_and_one_cluster_as_starts():
    """Starts that are no sample: everything apart, everything together, and a start whose clusters hold no pair."""
    ch = random_chain(14, 5, seed=77)
    R = ch.num_records
    for t in TS:
        best, runs = assert_equal_to_literal(ch, t, [np.arange(R), np.zeros(R, np.int64), np.arange(R) % 3])
        assert all(r.converged for r in runs)


@pytest.mark.parametrize("seed", range(4))
def test_no_single_move_lowers_a_converged_result(seed):
    """Brute force: from every converged result, moving any record to ANY other cluster or to a singleton does not
    lower the loss of the definition at the rounded t."""
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(16 + 3 * seed, 6, seed=2000 + seed)
    ids = as_set_chain(ch)[1]
    for t in TS:
        tr = fractions.Fraction(*aa.search_cost(t))
        _, runs = aa.binder_search(ch, t, starts_of(ch))
        for run in runs:
            assert run.converged
            part = as_sets(run.labels, ids)
            base = literal_loss(ch, tr, part)
            for r in ids:
                A = next(c for c in part if r in c)
                rest = [c for c in part if c != A] + ([A - {r}] if len(A) > 1 else [])
                for X in [c for c in part if c != A] + ([frozenset()] if len(A) > 1 else []):
                    moved = [c for c in rest if c != X] + [X | {r}]
                    assert literal_loss(ch, tr, moved) >= base


@pytest.mark.parametrize("R,S", [(30, 8), (200, 20), (2000, 40)])
def test_every_round_lowers_J_and_no_result_is_above_its_start(R, S):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(R, S, seed=R + S)
    first, second, count = aa.pairwise_match_counts(ch)
    n_s, K_s = aa.binder_counts(ch)
    C = int(n_s.sum())
    starts = starts_of(ch)
    moved = 0
    for t in TS:
        a, b = aa.search_cost(t)
        best, runs = aa.binder_search(ch, t, starts, max_rounds=60)
        for st, run in zip(starts, runs):
            n, K = run.linked_pairs(), run.count_sums()
            assert (n[0], K[0]) == aa.search_result_counts(first, second, count, st)
            assert (n[-1], K[-1]) == (run.n, run.K) == aa.search_result_counts(first, second, count, run.labels)
            J = [a * S * int(x) - b * int(y) for x, y in zip(n, K)]
            assert all(j1 < j0 for j0, j1 in zip(J, J[1:])) and (run.moves > 0).all()
            loss = aa.expected_losses(n, K, C, S, t)
            assert (np.diff(loss) <= 1e-9 * max(1.0, abs(loss[0]))).all()
            moved += run.rounds
        J = [a * S * r.n - b * r.K for r in runs]
        assert J[best] == min(J) and (J[0] > J[1] or best == 0)
    assert moved > 0


def test_the_binder_sample_start_is_scored_as_binder_counts_scores_it():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(60, 9, seed=3)
    n, K = aa.binder_counts(ch)
    s = aa.binder_estimate(n, K, 0.5)
    _, (run, _) = aa.binder_search(ch, 0.5, starts_of(ch))
    assert (run.linked_pairs()[0], run.count_sums()[0]) == (n[s], K[s])


def test_truncation_is_a_prefix():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 12, seed=9)
    starts = starts_of(ch)
    for t in (0.0, 0.5):
        _, full = aa.binder_search(ch, t, starts)
        assert max(r.rounds for r in full) >= 3
        for k in (1, 2, 3):
            _, cut = aa.binder_search(ch, t, starts, max_rounds=k)
            for f, c in zip(full, cut):
                assert c.rounds == min(k, f.rounds)
                for x, y in ((f.moves, c.moves), (f.dn, c.dn), (f.dK, c.dK)):
                    assert list(y) == list(x[:k])
                # a search whose k-th round is its last finds no move after it: it converged within the limit
                assert c.converged == (f.rounds <= k)
                if f.rounds <= k:
                    assert list(c.labels) == list(f.labels)
    small = random_chain(18, 6, seed=4)
    for k in (1, 2):
        assert_equal_to_literal(small, 0.0, starts_of(small), max_rounds=k)


def test_cost_rounding():
    from dblink_b200 import analysis_arrays as aa

    b = 1 << 16
    for t, a in ((0.0, 0), (0.25, b // 4), (0.5, b // 2), (0.75, 3 * b // 4), (1.0, b), (0.7, 45875), (0.1, 6554)):
        assert aa.search_cost(t) == (a, b)
    assert aa.search_cost(0.7)[0] / b == 0.6999969482421875
    assert aa.search_cost(2.5 / b) == (3, b) and aa.search_cost(3.5 / b) == (4, b)  # halves up
    assert aa.search_cost(2.4999 / b) == (2, b)
    for bad in (-0.01, 1.01):
        with pytest.raises(ValueError, match=r"falseLinkCost must be in \[0, 1\]"):
            aa.search_cost(bad)


def test_samples_times_records_bound(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    aa.check_search_size((1 << 22) - 1, 1 << 22)
    aa.check_search_size(1 << 20, (1 << 24) - 1)
    for S, R in ((1 << 22, 1 << 22), (1, 1 << 44), (1 << 24, 1 << 20)):
        with pytest.raises(ValueError, match=r"samples x records < 2\^44"):
            aa.check_search_size(S, R)
    ch = random_chain(10, 4, seed=1)
    monkeypatch.setattr(aa, "MAX_SEARCH_SIZE", 40)
    for fn in (aa.binder_search, ag.binder_search):  # both paths refuse before any work
        with pytest.raises(ValueError, match=r"here 4 x 10"):
            fn(ch, 0.5, starts_of(ch))
    monkeypatch.setattr(aa, "MAX_SEARCH_SIZE", 41)
    assert aa.binder_search(ch, 0.5, starts_of(ch))[0] in (0, 1)


def test_bad_starts():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(10, 4, seed=1)
    with pytest.raises(ValueError, match="one cluster label per record"):
        aa.binder_search(ch, 0.5, [np.zeros(9, np.int64)])


# ---- the project: config, run.txt and output files ------------------------------------------------------------------
def project_of(tmp_path, quantities='["partition-sizes"]', metrics='["pairwise"]', summarize_extra="",
               evaluate_extra="", out="out", chains=1):
    from dblink_b200 import config
    from dblink_b200.project import Project

    data = os.path.join(tmp_path, "data.csv")
    return Project(config.parse_string(CONF % (data, str(tmp_path / out) + "/", chains, quantities, summarize_extra,
                                               metrics, evaluate_extra)), base_dir="")


def test_config(tmp_path):
    def steps(**kw):
        return project_of(tmp_path, **kw).steps()

    (_, s), (_, e) = steps(quantities='["binder-search-clusters"]',
                           metrics='["binder-search-cluster", "binder-search-pairwise"]')
    assert s["quantities"] == ["binder-search-clusters"] and s["max_search_rounds"] == 1000
    assert e["metrics"] == ["binder-search-cluster", "binder-search-pairwise"] and e["max_search_rounds"] == 1000
    (_, s), (_, e) = steps(summarize_extra=", maxSearchRounds : 7", evaluate_extra=", maxSearchRounds : 1")
    assert s["max_search_rounds"] == 7 and e["max_search_rounds"] == 1
    for bad in ("0", "-3", "1.5", "true", '"10"'):
        for kw in (dict(summarize_extra=", maxSearchRounds : " + bad), dict(evaluate_extra=", maxSearchRounds : " + bad)):
            with pytest.raises(ValueError, match=r"^maxSearchRounds must be a positive integer\.$"):
                steps(**kw)
    with pytest.raises(ValueError, match="quantities"):
        steps(quantities='["binder-search"]')
    with pytest.raises(ValueError, match="metrics"):
        steps(metrics='["binder-search-clusters"]')


def test_run_txt_mentions_the_search_only_when_asked(tmp_path):
    p = project_of(tmp_path, quantities='["binder-search-clusters", "partition-sizes"]',
                   summarize_extra=", falseLinkCost : 0.7, maxSearchRounds : 20",
                   metrics='["pairwise", "binder-search-pairwise"]')
    assert p.steps_mk_string().splitlines()[2:] == [
        "  * SummarizeStep: Calculating summary quantities {'binder-search-clusters', 'partition-sizes'} along the "
        "chain for iterations >= 10",
        "  * SummarizeStep: binder-search-clusters is the least posterior expected Binder loss found by single-record "
        "moves from the Binder sample and the sMPC, with falseLinkCost=0.7 (searched at 0.6999969482421875) and "
        "maxSearchRounds=20",
        "  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= 10) using {'pairwise'} "
        "metrics",
        "  * EvaluateStep: Evaluating the least posterior expected Binder loss found by single-record moves from the "
        "Binder sample and the sMPC (falseLinkCost=0.5, searched at 0.5, maxSearchRounds=1000, iterations >= 10) "
        "using {'binder-search-pairwise'} metrics"]
    for kw in (dict(), dict(quantities='["binder-clusters"]', metrics='["binder-pairwise", "cluster"]'),
               dict(summarize_extra=", maxSearchRounds : 20", evaluate_extra=", maxSearchRounds : 3")):
        assert "search" not in project_of(tmp_path, **kw).steps_mk_string()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("binder_counts", "shared_most_probable_clusters", "pairwise_match_counts", "posterior_metric_counts",
                 "binder_search"):
        monkeypatch.setattr(project, name, getattr(aa, name))


# The chain of test_binder_host: 6 records, truth {r0,r1} {r2,r3} {r4} {r5}; after the cutoff s0 = singletons, s1 = the
# truth, s2 = {0,1,2} {3} {4,5}.  Counts (0,1) = 2, (0,2) = (1,2) = (2,3) = (4,5) = 1, S = 3, C = 6; a move of i from A
# to X changes E[L] by sum over j in X of (t - p_ij) - sum over j in A \ {i} of (t - p_ij).  At t = 0.3 the Binder
# sample is s2, and no move lowers its loss: 0 rounds.  The sMPC is all singletons (every record's clusters tie, the
# earliest wins).  From it, round 1: r0 -> {1} (-0.37) holds clusters 0 and 1, r4 -> {5} (-0.03) holds 4 and 5; r1,
# r2, r3 and r5 lose a claim: 2 moves, dn = 2, dK = 2 + 1.  Round 2: r2 -> {0,1} (-0.07) beats r3 -> {2} (-0.03) on
# cluster 2: 1 move, dn = 2, dK = 2.  That is s2 again; J ties, so the Binder-sample start is kept.  Losses
# (4.2 + 0.9 n - K) / 3: n = 4, K = 5 gives 2.8 / 3; n = 0, 2 gives 1.4, 1.
BINDER_SEARCH_CSV = """start,round,moves,linkedPairs,expectedLoss
binder-sample,0,0,4,0.933333333333333
smpc,0,0,0,1.3999999999999997
smpc,1,2,2,0.9999999999999997
smpc,2,1,4,0.933333333333333
"""

BINDER_SEARCH_RESULTS_TXT = """=====================================
    Binder search cluster metrics
-------------------------------------
 Estimate:        search from the binder-sample start, 0 rounds, converged, falseLinkCost 0.3 (searched at 0.3000030517578125)
 Adj. Rand index: 0.18918918918918917
=====================================

=====================================
   Binder search pairwise metrics
-------------------------------------
 Estimate:        search from the binder-sample start, 0 rounds, converged, falseLinkCost 0.3 (searched at 0.3000030517578125)
 Precision:      0.25
 Recall:         0.5
 F1-score:       0.3333333333333333
=====================================

"""

# Two chains, the second holding the truth at iteration 20 only: S = 4, C = 8, p(0,1) = 3/4, p(2,3) = 1/2, the other
# three 1/4.  At t = 0.4 the Binder sample is the truth, a local minimum; the sMPC is {0,1} {2} {3} {4} {5} (r3's
# clusters {3} and {2,3} tie and {3} comes first).  From it r2 -> {3} (-0.1) and r3 -> {2} (-0.1) claim the same two
# clusters and r2, the smaller index, moves: 1 move, dn = 1, dK = 2, and the result is the truth.  Losses
# (4.8 + 1.6 n - K) / 4.
BINDER_SEARCH_TWO_CHAINS_CSV = """start,round,moves,linkedPairs,expectedLoss
binder-sample,0,0,2,0.75
smpc,0,0,1,0.8500000000000001
smpc,1,1,2,0.75
"""


def test_project_writes_the_search_files(tmp_path, monkeypatch):
    from dblink_b200 import analysis_arrays as aa

    host_paths(monkeypatch)
    p = project_of(tmp_path, quantities='["binder-search-clusters"]', summarize_extra=", falseLinkCost : 0.3",
                   metrics='["binder-search-cluster", "binder-search-pairwise"]', evaluate_extra=", falseLinkCost : 0.3")
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "binder-search-clusters.csv").read() == "r0, r1, r2\nr3\nr4, r5\n"
    assert open(out + "binder-search.csv").read() == BINDER_SEARCH_CSV
    assert open(out + "evaluation-results.txt").read() == BINDER_SEARCH_RESULTS_TXT
    assert set(res) == {"binder-search-cluster", "binder-search-pairwise"}
    assert (res["binder-search-pairwise"]["TP"], res["binder-search-pairwise"]["FP"]) == (1, 3)
    assert not os.path.exists(out + "binder-clusters.csv") and not os.path.exists(out + "binder-loss.csv")
    # the rows agree with the literal restatement from the same starts
    ch = p.read_chain(10)
    best, lit = literal(ch, 0.3, starts_of_at(ch, 0.3))
    assert best == 0 and [r["rounds"] for r in lit] == [[], [(2, 2, 3), (1, 2, 2)]]


def starts_of_at(ch, t):
    from dblink_b200 import analysis_arrays as aa

    s = aa.binder_estimate(*aa.binder_counts(ch), t)
    mem, off, _ = ch.samples[s]
    return [aa.sample_labels(ch.num_records, mem, off), aa.shared_most_probable_clusters(ch)]


def test_two_chains_pool_the_search(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, chains=2, quantities='["binder-search-clusters"]', summarize_extra=", falseLinkCost : 0.4",
                   metrics='["binder-search-pairwise"]', evaluate_extra=", falseLinkCost : 0.4")
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "binder-search-clusters.csv").read() == "r0, r1\nr2, r3\nr4\nr5\n"
    assert open(out + "binder-search.csv").read() == BINDER_SEARCH_TWO_CHAINS_CSV
    assert res["binder-search-pairwise"]["precision"] == 1.0 and res["binder-search-pairwise"]["recall"] == 1.0


def test_other_outputs_do_not_change(tmp_path, monkeypatch):
    """The same steps with and without the new names write the same bytes in every other file; the evaluation text
    only gains the search sections at its end."""
    host_paths(monkeypatch)
    quantities = ["shared-most-probable-clusters", "binder-clusters", "pairwise-match-probabilities",
                  "partition-sizes"]
    metrics = ["pairwise", "binder-pairwise", "posterior-cluster"]

    def run(out, q, m):
        p = project_of(tmp_path, quantities=str(q).replace("'", '"'), metrics=str(m).replace("'", '"'), out=out)
        write_chain(tmp_path, p)
        p.execute(log=lambda *a: None)
        d = str(tmp_path / out)
        return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d)) if f.endswith((".csv", ".txt"))}

    plain = run("plain", quantities, metrics)
    mixed = run("mixed", quantities[:1] + ["binder-search-clusters"] + quantities[1:],
                metrics[:1] + ["binder-search-cluster"] + metrics[1:] + ["binder-search-pairwise"])
    assert set(mixed) - set(plain) == {"binder-search-clusters.csv", "binder-search.csv"}
    text = "evaluation-results.txt"
    for f in plain:
        if f != text:
            assert mixed[f] == plain[f], f
    assert mixed[text].startswith(plain[text]) and b"Binder search pairwise metrics" in mixed[text][len(plain[text]):]


def test_abi_checks_before_any_device_work():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Pairs

    L = _lib.load()
    lab = np.zeros(4, np.int32)
    r, c = C.c_int32(-1), C.c_int32(-1)
    logs = [np.zeros(2, np.int64) for _ in range(3)]
    n, K = C.c_int64(-1), C.c_int64(-1)
    ok = [lab.ctypes.data, 2, lab.ctypes.data, C.byref(r), C.byref(c)] + [x.ctypes.data_as(_lib.i64p) for x in logs] \
        + [C.byref(n), C.byref(K)]
    for k in range(len(ok)):  # a NULL handle, and every other NULL pointer
        args = list(ok)
        if k != 1:
            args[k] = None
        assert L.dbl_pairs_binder_search(None, 1, 2, *args[:1], *args[1:]) == _lib.ERR_INVALID
    assert (r.value, c.value, n.value, K.value) == (-1, -1, -1, -1)
    p = Pairs.__new__(Pairs)  # an owner without a handle: the shape check comes first
    p.num_records = 4
    with pytest.raises(ValueError, match="one cluster label per record"):
        p.binder_search(1, 2, np.zeros(3, np.int32), 5)


def test_the_search_needs_a_device():
    import torch

    from dblink_b200 import _lib, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    ch = random_chain(10, 4, seed=1)
    with pytest.raises(DblinkError) as e:
        ag.binder_search(ch, 0.5, starts_of(ch))
    assert e.value.status == _lib.ERR_CUDA


def test_project_uses_the_host_search_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(*a, **kw):
        raise AssertionError("the GPU search was called on a host without a device")

    monkeypatch.setattr(ag, "binder_search", no_gpu)
    ch = random_chain(40, 6, seed=2)
    start, run, rows = project.binder_search_estimate(ch, 0.5, 1000)
    best, runs = aa.binder_search(ch, 0.5, starts_of(ch))
    assert start == aa.SEARCH_STARTS[best] and list(run.labels) == list(runs[best].labels)
    assert [r[:2] for r in rows] == [(name, k) for name, x in zip(aa.SEARCH_STARTS, runs) for k in range(x.rounds + 1)]
