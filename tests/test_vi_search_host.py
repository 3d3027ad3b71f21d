"""The VI search on the host: analysis_arrays.vi_search (numpy) against the literal analysis.vi_search (sets, every
cluster a candidate, every change recomputed from scratch) on random small chains and a hand-worked example; a
brute-force check that no single-record move lowers J_q of a converged result; J_q falling every round and E_q
against the entropy definition of the expected VI; the quantised table; the size and squares refusals; the exact
expected VI of any labelling (vi_label_cells / vi_label_loss) against vi_losses; the summarize quantity
vi-search-clusters and the evaluate metrics vi-search-pairwise / vi-search-cluster with their config and files; the C
ABI's checks that come before any device work."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from test_binder_host import WORKED, chain_of, project_of
from test_match_probabilities_host import as_set_chain, random_chain
from test_vi_host import write_chain

Q = 20


def starts_of(ch):
    """The two starts the project uses: the VI sample and the sMPC."""
    from dblink_b200 import analysis_arrays as aa

    G = aa.vi_cross_histograms(ch)
    s = aa.vi_estimate(aa.vi_losses(aa.vi_cluster_histograms(ch, G.shape[1]), G, ch.num_records))
    mem, off, _ = ch.samples[s]
    return [aa.sample_labels(ch.num_records, mem, off), aa.shared_most_probable_clusters(ch)]


def as_sets(labels, ids):
    from dblink_b200 import analysis_arrays as aa

    return {frozenset(ids[i] for i in g) for g in aa.labels_to_clusters(labels)}


def assert_equal_to_literal(ch, starts, max_rounds=1000):
    from dblink_b200 import analysis, analysis_arrays as aa

    best, runs = aa.vi_search(ch, starts, max_rounds)
    chain, ids = as_set_chain(ch)
    lit_best, lit = analysis.vi_search(chain, [as_sets(s, ids) for s in starts], max_rounds, records=ids)
    assert best == lit_best
    for run, want in zip(runs, lit):
        assert as_sets(run.labels, ids) == want["clusters"]
        assert list(run.labels) == list(aa.canonical_labels(run.labels))  # canonical
        assert list(zip(run.moves.tolist(), run.clusters.tolist(), run.dJ.tolist())) == want["rounds"]
        assert (run.converged, run.J0, run.J) == (want["converged"], want["J0"], want["J"])
    return best, runs


def J_of(ch, labels, table):
    """J_q by the definition, over the clusters of labels and the cells with every sample."""
    from dblink_b200 import analysis_arrays as aa

    F = aa.vi_search_prefix(table)
    R, S = ch.num_records, len(ch.samples)
    labels = np.asarray(labels, np.int64)
    J = S * int(F[np.bincount(labels)].sum())
    for mem, off, _ in ch.samples:
        _, n = np.unique(aa.sample_labels(R, mem, off) * R + labels, return_counts=True)
        J -= 2 * int(F[n].sum())
    return J


def entropy_vi(ch, labels):
    """The expected VI of a labelling by the entropy definition: mean over the samples of H(c) + H(C_s) - 2 I(c, C_s)."""
    from dblink_b200 import analysis_arrays as aa

    R = ch.num_records

    def H(n):
        return -sum(k / R * math.log2(k / R) for k in n)

    labels = np.asarray(labels, np.int64)
    c = np.bincount(labels)
    total = 0.0
    for mem, off, _ in ch.samples:
        ls = aa.sample_labels(R, mem, off)
        cells, n = np.unique(ls * R + labels, return_counts=True)
        s = np.bincount(ls)
        mi = sum(k / R * math.log2(k * R / (c[x % R] * s[x // R])) for x, k in zip(cells, n))
        total += H(c[c > 0]) + H(s[s > 0]) - 2 * mi
    return total / len(ch.samples)


def test_table():
    from dblink_b200 import analysis_arrays as aa

    for R in (1, 2, 5, 1000, 1 << 20):
        D = aa.vi_search_table(R)
        assert D.dtype == np.int64 and D.shape == (R,) and D[0] == 0 and (np.diff(D) >= 0).all()
        if R > 1:
            assert D[1] == 1 << (Q + 1)
    D = aa.vi_search_table(4096)
    F = aa.vi_search_prefix(D)
    n = np.arange(1, 4097)
    exact = n * np.log2(n) * 2.0 ** Q
    assert F.shape == (4097,) and F[0] == 0 and (np.abs(F[1:] - exact) <= n / 2).all()


def test_worked_example():
    """R = 4, S = 3 (s0 = {0,1}{2}{3}, s1 = {0,1,2}{3}, s2 = {0}{1}{2,3}), D_q = [0, D1, D2, D3] =
    [0, 2097152, 2888709, 3402747].
    From all singletons (J0 = 0): record 0 to {1} changes J_q by S D1 - 2 (D1 + D1) = -D1 (s0 and s1 hold 0 and 1
    together), record 1 to {0} likewise; both touch {0} and {1}, the lower record index wins: one move, 3 clusters,
    dJ = -2097152.  Then no move lowers J_q (record 2 to {0,1}: 3 D2 - 2 D2 > 0): the result is s0.
    From one cluster (J0 = 3 F(4) - 2 (F(2) + F(3) + F(2)) = 6805494): every record proposes a singleton, record 3 the
    least, -3 D3 + 2 D1 = -6013937; then record 2 leaves {0,1,2}, -3 D2 + 2 D2 = -2888709; then s0 again.  The two
    results tie at J_q = -2097152 and the VI-sample start is kept."""
    from dblink_b200 import analysis_arrays as aa

    ch = chain_of(WORKED)
    assert aa.vi_search_table(4).tolist() == [0, 2097152, 2888709, 3402747]
    best, runs = assert_equal_to_literal(ch, [np.arange(4), np.zeros(4, np.int64)])
    a, b = runs
    assert best == 0 and list(a.labels) == list(b.labels) == [0, 0, 2, 3]
    assert (a.J0, a.moves.tolist(), a.clusters.tolist(), a.dJ.tolist(), a.converged) == (
        0, [1], [3], [-2097152], True)
    assert (b.J0, b.moves.tolist(), b.clusters.tolist(), b.dJ.tolist(), b.converged) == (
        6805494, [1, 1], [2, 3], [-6013937, -2888709], True)
    assert a.J == b.J == -2097152
    # E_q of the result: (J + sum_s F(|K|)) / (2^Q R S), next to the expected VI of s0, (2 + 3 log2 3) / 12
    A = aa.vi_sample_sum(ch, aa.vi_search_table(4))
    assert A == 2097152 + 4985861 + 2097152
    (e,) = aa.vi_search_losses([a.J], A, 3, 4)
    assert e == (A - 2097152) / (12 << Q) and abs(e - (2 + 3 * math.log2(3)) / 12) <= 2.0 ** (1 - Q)


@pytest.mark.parametrize("seed", range(8))
def test_numpy_equals_the_literal_search(seed):
    rng = np.random.default_rng(seed)
    R, S = int(rng.integers(2, 26)), [1, 2, 3, 5, 8][seed % 5]
    ch = random_chain(R, S, seed=3000 + seed)
    assert_equal_to_literal(ch, starts_of(ch) + [np.arange(R), np.zeros(R, np.int64)])


def test_ties():
    """Identical samples and symmetric records: equal dJ proposals resolved by (dJ, record) and (dJ, destination)."""
    for links in ([[0, 0, 1, 1], [0, 0, 1, 1]], [[0, 0, 0, 0, 4, 4], [0, 1, 0, 1, 4, 4]], [[0, 1, 0, 1, 4, 5]] * 3):
        ch = chain_of(links)
        R = ch.num_records
        assert_equal_to_literal(ch, [np.arange(R), np.zeros(R, np.int64), starts_of(ch)[1]])


def test_truncated_rounds_are_a_prefix():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(60, 6, seed=21)
    _, full = aa.vi_search(ch, [np.arange(60)])
    assert full[0].converged and full[0].rounds >= 2
    for k in range(1, full[0].rounds):
        _, (run,) = aa.vi_search(ch, [np.arange(60)], max_rounds=k)
        assert not run.converged and run.rounds == k and run.J0 == full[0].J0
        assert run.moves.tolist() == full[0].moves[:k].tolist() and run.dJ.tolist() == full[0].dJ[:k].tolist()


@pytest.mark.parametrize("seed", range(4))
def test_no_single_move_lowers_a_converged_result(seed):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(14 + 3 * seed, 5, seed=4000 + seed)
    R = ch.num_records
    table = aa.vi_search_table(R)
    _, runs = aa.vi_search(ch, starts_of(ch))
    for run in runs:
        assert run.converged
        base = J_of(ch, run.labels, table)
        assert base == run.J
        for r in range(R):
            for dest in set(run.labels.tolist()) | {R}:  # every cluster, and R: a new singleton
                if dest == run.labels[r] or (dest == R and (run.labels == run.labels[r]).sum() == 1):
                    continue
                moved = run.labels.copy()
                moved[r] = dest
                assert J_of(ch, moved, table) >= base


@pytest.mark.parametrize("R,S", [(30, 8), (200, 20), (1500, 30)])
def test_J_falls_every_round_and_E_q_is_the_expected_vi(R, S):
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(R, S, seed=R + S)
    table = aa.vi_search_table(R)
    starts = starts_of(ch)
    best, runs = aa.vi_search(ch, starts, max_rounds=60)
    A = aa.vi_sample_sum(ch, table)
    moved = 0
    for st, run in zip(starts, runs):
        J = run.objectives()
        assert J[0] == run.J0 == J_of(ch, st, table) and J[-1] == run.J == J_of(ch, run.labels, table)
        assert all(j1 < j0 for j0, j1 in zip(J, J[1:])) and (run.moves > 0).all()
        e0, e1 = aa.vi_search_losses([J[0], J[-1]], A, S, R)
        assert abs(e0 - entropy_vi(ch, st)) <= 2.0 ** (1 - Q) and abs(e1 - entropy_vi(ch, run.labels)) <= 2.0 ** (1 - Q)
        if run.rounds:
            assert run.clusters[-1] == len(np.unique(run.labels))
        moved += run.rounds
    assert moved > 0 and best == aa.vi_search_choice(runs)


def test_label_loss_is_the_sample_loss():
    """vi_label_loss of each sample's own labels, from vi_label_cells, equals vi_losses exactly."""
    from dblink_b200 import analysis_arrays as aa

    for ch in (random_chain(40, 9, seed=6), random_chain(300, 5, seed=4, big=120), chain_of(WORKED)):
        R, S = ch.num_records, len(ch.samples)
        G = aa.vi_cross_histograms(ch)
        width = G.shape[1]
        g = aa.vi_cluster_histograms(ch, width)
        losses = aa.vi_losses(g, G, R)
        for s, (mem, off, _) in enumerate(ch.samples):
            lab = aa.sample_labels(R, mem, off)
            cells = aa.vi_label_cells(ch, lab, width)
            assert np.array_equal(cells, G[s] + g[s])
            assert aa.vi_label_loss(np.bincount(np.bincount(lab)), cells, g.sum(axis=0), S, R) == losses[s]
        other = np.arange(R) % 3
        e = aa.vi_label_loss(np.bincount(np.bincount(other)), aa.vi_label_cells(ch, other, width), g.sum(axis=0), S, R)
        assert abs(e - entropy_vi(ch, other)) < 1e-9


def test_refusals_have_one_message(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    # the size bound, S R (ceil(log2 R) + 2) 2^22 < 2^63: about 100 k samples at 1 M records
    R = 1_000_000
    edge = ((1 << 63) - 1) // (R * 22 << 22)
    aa.check_vi_search_size(edge, R)
    one = aa.sample_from_links(np.arange(R, dtype=np.int32), np.zeros(R, np.int32))
    big = aa.ChainArrays(np.arange(R), np.arange(edge + 1, dtype=np.int64), [one] * (edge + 1))
    msgs = []
    for fn in (aa.vi_search, ag.vi_search):
        with pytest.raises(ValueError, match=r"samples x records x \(ceil\(log2 records\) \+ 2\) x 2\^22 < 2\^63") as e:
            fn(big, [np.arange(R)])
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1] == f"the VI search needs samples x records x (ceil(log2 records) + 2) x 2^22 < 2^63 " \
                                 f"(here {edge + 1} x {R})"
    # the squares cap: sample 1 holds a cluster of 5 and one of 2, 25 + 4 + 3 singletons = 32
    ch = chain_of([np.arange(10), [0, 0, 0, 0, 0, 5, 5, 7, 8, 9]])
    assert aa.vi_sample_squares(ch).tolist() == [10, 32]
    monkeypatch.setattr(aa, "MAX_VI_SEARCH_SQUARES", 31)
    msgs = []
    for fn in (aa.vi_search, ag.vi_search):
        with pytest.raises(ValueError, match="^the VI search refuses sample 1: its clusters' squared sizes sum to 32, "
                                             "more than 31$") as e:
            fn(ch, [np.arange(10)])
        msgs.append(str(e.value))
    assert msgs[0] == msgs[1]
    monkeypatch.setattr(aa, "MAX_VI_SEARCH_SQUARES", 32)
    assert aa.vi_search(ch, [np.arange(10)])[1][0].converged


def test_config_and_run_txt(tmp_path):
    (_, s), (_, e) = project_of(tmp_path, quantities='["vi-search-clusters"]',
                                metrics='["vi-search-cluster", "vi-search-pairwise"]',
                                evaluate_extra=", maxSearchRounds : 7").steps()
    assert s["quantities"] == ["vi-search-clusters"] and s["max_search_rounds"] == 1000
    assert e["metrics"] == ["vi-search-cluster", "vi-search-pairwise"] and e["max_search_rounds"] == 7
    p = project_of(tmp_path, quantities='["vi-search-clusters", "partition-sizes"]',
                   metrics='["pairwise", "vi-search-pairwise"]', summarize_extra=", maxSearchRounds : 3")
    assert p.steps_mk_string().splitlines()[2:] == [
        "  * SummarizeStep: Calculating summary quantities {'vi-search-clusters', 'partition-sizes'} along the chain "
        "for iterations >= 10",
        "  * SummarizeStep: vi-search-clusters is the least posterior expected variation of information found by "
        "single-record moves from the VI sample and the sMPC, with maxSearchRounds=3",
        "  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= 10) using {'pairwise'} "
        "metrics",
        "  * EvaluateStep: Evaluating the least posterior expected variation of information found by single-record "
        "moves from the VI sample and the sMPC (maxSearchRounds=1000, iterations >= 10) using {'vi-search-pairwise'} "
        "metrics"]
    assert "single-record moves from the VI" not in project_of(tmp_path).steps_mk_string()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("vi_cross_histograms", "shared_most_probable_clusters", "pairwise_match_counts",
                 "posterior_metric_counts", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)


def test_project_writes_the_search_and_its_metrics(tmp_path, monkeypatch):
    """The chain of test_vi_host (6 records; s0 = the truth {0,1}{2,3}{4}{5}, s1 = {0,1} and singletons, s2 =
    {0,1}{2,3}{4,5}): the VI sample is s0, and no single move lowers it; the sMPC is s0 too."""
    from dblink_b200 import analysis_arrays as aa

    host_paths(monkeypatch)
    p = project_of(tmp_path, quantities='["vi-search-clusters"]', metrics='["vi-search-cluster", "vi-search-pairwise"]')
    write_chain(tmp_path, p)
    res = p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "vi-search-clusters.csv").read() == "r0, r1\nr2, r3\nr4\nr5\n"
    ch = p.read_chain(10)
    R, S = 6, 3
    table = aa.vi_search_table(R)
    A = aa.vi_sample_sum(ch, table)
    J = J_of(ch, [0, 0, 2, 2, 4, 5], table)
    e = (J + A) / (R * S << Q)
    assert open(out + "vi-search.csv").read() == f"start,round,moves,numClusters,expectedLoss\nvi-sample,0,0,4,{e!r}\n" \
                                                 f"smpc,0,0,4,{e!r}\n"
    G = aa.vi_cross_histograms(ch)
    exact = float(aa.vi_losses(aa.vi_cluster_histograms(ch, G.shape[1]), G, R)[0])  # the expected VI of s0
    assert abs(e - exact) <= 2.0 ** (1 - Q)
    lines = (" Estimate:        search from the vi-sample start, 0 rounds, converged\n"
             f" Expected VI:     vi-sample start {exact!r}, smpc start {exact!r}, from vi-sample {exact!r}, "
             f"from smpc {exact!r}\n")
    assert open(out + "evaluation-results.txt").read() == (
        "=====================================\n      VI search cluster metrics\n"
        "-------------------------------------\n" + lines + " Adj. Rand index: 1.0\n"
        "=====================================\n\n"
        "=====================================\n     VI search pairwise metrics\n"
        "-------------------------------------\n" + lines + " Precision:      1.0\n Recall:         1.0\n"
        " F1-score:       1.0\n=====================================\n\n")
    assert set(res) == {"vi-search-cluster", "vi-search-pairwise"} and res["vi-search-cluster"] == 1.0
    assert not os.path.exists(out + "shared-most-probable-clusters.csv")


def test_the_search_leaves_a_sample(tmp_path, monkeypatch):
    """A chain whose samples all over-link: the search from them splits records off and lowers E_q below both starts;
    the rows of vi-search.csv follow the runs."""
    from dblink_b200 import analysis_arrays as aa, project

    host_paths(monkeypatch)
    rng = np.random.default_rng(9)
    R, S = 80, 12
    truth = np.repeat(np.arange(40), 2)
    links = [np.where(rng.random(R) < 0.2, rng.integers(0, 40, R), truth) for _ in range(S)]
    ch = chain_of(links)
    start, run, rows, exact = project.vi_search_estimate(ch, 1000)
    assert rows[0][:2] == ("vi-sample", 0) and len(rows) == sum(r.rounds for r in project_vi_runs(ch)) + 2
    by = {name: [r for r in rows if r[0] == name] for name in aa.VI_SEARCH_STARTS}
    for name in aa.VI_SEARCH_STARTS:
        losses = [r[4] for r in by[name]]
        assert [r[1] for r in by[name]] == list(range(len(losses))) and all(b < a for a, b in zip(losses, losses[1:]))
    assert min(exact[2:]) < min(exact[:2]) and run.converged
    assert exact[aa.VI_SEARCH_STARTS.index(start) + 2] == min(exact[2:])


def project_vi_runs(ch):
    from dblink_b200 import analysis_arrays as aa

    return aa.vi_search(ch, starts_of(ch))[1]


def test_two_chains_pool_the_search(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    p = project_of(tmp_path, chains=2, quantities='["vi-search-clusters"]', metrics='["vi-search-pairwise"]')
    write_chain(tmp_path, p)
    p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    assert open(out + "vi-search-clusters.csv").read() == "r0, r1\nr2, r3\nr4\nr5\n"
    rows = open(out + "vi-search.csv").read().splitlines()
    assert rows[0] == "start,round,moves,numClusters,expectedLoss" and rows[1].startswith("vi-sample,0,0,4,")
    assert "search from the vi-sample start" in open(out + "evaluation-results.txt").read()


def test_no_sample_after_the_cutoff(tmp_path, monkeypatch):
    host_paths(monkeypatch)
    for kw in (dict(quantities='["vi-search-clusters"]'), dict(metrics='["vi-search-pairwise"]')):
        p = project_of(tmp_path, **kw)
        write_chain(tmp_path, p)
        p.steps = lambda p=p: [(n, dict(prm, lower_iteration_cutoff=100)) for n, prm in type(p).steps(p)]
        with pytest.raises(ValueError, match="at least one sample at or after lowerIterationCutoff"):
            p.execute(log=lambda *a: None)


def test_other_outputs_do_not_change(tmp_path, monkeypatch):
    """The same steps with and without the new names write the same bytes in every other file; the evaluation text
    only gains the VI search sections at its end."""
    host_paths(monkeypatch)
    quantities = ["shared-most-probable-clusters", "pairwise-match-probabilities", "cluster-size-distribution",
                  "partition-sizes", "binder-clusters", "vi-clusters"]
    metrics = ["pairwise", "cluster", "posterior-pairwise", "posterior-cluster", "binder-pairwise", "vi-pairwise"]

    def run(out, q, m):
        p = project_of(tmp_path, quantities=str(q).replace("'", '"'), metrics=str(m).replace("'", '"'), out=out)
        write_chain(tmp_path, p)
        p.execute(log=lambda *a: None)
        d = str(tmp_path / out)
        return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d)) if f.endswith((".csv", ".txt"))}

    plain = run("plain", quantities, metrics)
    mixed = run("mixed", quantities[:2] + ["vi-search-clusters"] + quantities[2:],
                metrics[:1] + ["vi-search-pairwise"] + metrics[1:] + ["vi-search-cluster"])
    assert set(mixed) - set(plain) == {"vi-search-clusters.csv", "vi-search.csv"}
    text = "evaluation-results.txt"
    for f in plain:
        if f != text:
            assert mixed[f] == plain[f], f
    assert mixed[text].startswith(plain[text]) and b"VI search pairwise metrics" in mixed[text][len(plain[text]):]


def test_abi_checks_before_any_device_work():
    from dblink_b200 import _lib, analysis_arrays as aa
    from dblink_b200.analysis_gpu import VI

    L = _lib.load()
    R = 4
    step = np.zeros(R, np.int64)
    start = np.zeros(R, np.int32)
    labels = np.zeros(R, np.int32)
    logs = [np.zeros(4, np.int64) for _ in range(3)]
    rounds, conv, J0 = C.c_int32(-7), C.c_int32(-7), C.c_int64(-7)
    args = [None, step.ctypes.data_as(_lib.i64p), start.ctypes.data, 4, labels.ctypes.data, C.byref(rounds),
            C.byref(conv), *(x.ctypes.data_as(_lib.i64p) for x in logs), C.byref(J0)]
    assert L.dbl_vi_search(*args) == _lib.ERR_INVALID
    assert (rounds.value, conv.value, J0.value) == (-7, -7, -7)
    G = np.zeros(8, np.int64)
    assert L.dbl_vi_score(None, labels.ctypes.data, 8, G.ctypes.data) == _lib.ERR_INVALID
    v = VI.__new__(VI)  # an owner without a handle: the shape checks come first
    v.num_records = R
    with pytest.raises(ValueError, match="one cluster label per record"):
        v.search(step, np.zeros(3, np.int32), 5)
    with pytest.raises(ValueError, match="^the VI search table needs one entry per record$"):
        v.search(step[:3], start, 5)
    with pytest.raises(ValueError, match="^the VI search table needs one entry per record$"):
        aa.vi_search_rounds(R, [start], step[:3], start, 5)
    with pytest.raises(ValueError, match="one cluster label per record"):
        v.score(np.zeros(5, np.int32), 8)


def test_project_uses_the_host_path_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(*a, **kw):
        raise AssertionError("the GPU handle was used on a host without a device")

    monkeypatch.setattr(ag, "vi_samples", no_gpu)
    start, run, rows, exact = project.vi_search_estimate(chain_of(WORKED), 10)
    assert start == "vi-sample" and list(run.labels) == [0, 0, 2, 3] and rows[0][:4] == ("vi-sample", 0, 0, 3)
