"""Capture histories on the host: the numpy counts (analysis_arrays.capture_histories) against the literal
analysis.capture_histories on random partitions with random files; the identities between H, L and the file sizes;
the population-size estimators against their definitions and scipy; the files Project.execute writes for the
summarize quantity and the evaluate metric on 3-file synthetic data with one and two chains, every other output file
unchanged; every refusal."""
import csv
import os
import shutil

import numpy as np
import pytest

from test_entity_values_host import ScriptedEngine
from test_match_probabilities_host import as_set_chain, random_chain


def literal(ch, file, F):
    from dblink_b200 import analysis

    chain, ids = as_set_chain(ch)
    H, L = analysis.capture_histories(chain, {ids[i]: int(file[i]) for i in range(len(ids))}, F)
    return np.asarray(H, np.int64).reshape(-1, 1 << F), np.asarray([L[r] for r in ids], np.int64).reshape(-1, F)


def one_sample(labels):
    """A ChainArrays of the single labelling labels[R]."""
    from dblink_b200 import analysis_arrays as aa

    labels = np.asarray(labels)
    return aa.ChainArrays(np.array(["r%d" % i for i in range(len(labels))]), np.zeros(1, np.int64),
                          [aa.sample_from_links(labels, np.zeros(labels.max() + 1, np.int32))])


def cases():
    rng = np.random.default_rng(7)
    out = []
    for F in (1, 2, 3, 12):
        for seed in range(3):
            ch = random_chain(60, 6, seed + 10 * F, big=20 if seed == 2 else 0)
            out.append((f"random-F{F}-{seed}", ch, rng.integers(0, F, 60), F))
    out.append(("one-sample", random_chain(50, 1, 3), rng.integers(0, 3, 50), 3))
    out.append(("singletons", one_sample(np.arange(30)), rng.integers(0, 4, 30), 4))
    out.append(("giant", one_sample(np.zeros(40, np.int64)), rng.integers(0, 3, 40), 3))
    out.append(("one-file", random_chain(45, 4, 5), np.full(45, 2), 3))
    return out


CASES = cases()


@pytest.mark.parametrize("name,ch,file,F", CASES, ids=[c[0] for c in CASES])
def test_numpy_counts_equal_the_literal_counts(name, ch, file, F):
    from dblink_b200 import analysis_arrays as aa

    H, L = aa.capture_histories(ch, file, F)
    assert H.dtype == L.dtype == np.int64
    want_H, want_L = literal(ch, file, F)
    assert np.array_equal(H, want_H)
    assert np.array_equal(L, want_L)


@pytest.mark.parametrize("name,ch,file,F", CASES, ids=[c[0] for c in CASES])
def test_identities(name, ch, file, F):
    from dblink_b200 import analysis_arrays as aa

    H, L = aa.capture_histories(ch, file, F)
    S, R = len(ch.samples), ch.num_records
    assert (H[:, 0] == 0).all()
    assert H.sum(axis=1).tolist() == [len(off) - 1 for _, off, _ in ch.samples]  # one history per cluster
    per_file = np.bincount(file, minlength=F)
    summary = aa.CaptureSummary(H, L, per_file)
    cols = dict(zip(summary.names, summary.columns))
    for f in range(F):
        assert (cols[f"entities[{f}]"] + cols[f"duplicates[{f}]"] == per_file[f]).all()
    assert ((0 <= L) & (L <= S)).all()
    for mem, off, _ in ch.samples[:1] if S == 1 else []:
        for c in range(len(off) - 1):  # S = 1: records of one cluster have equal links into other files
            rec = mem[off[c]:off[c + 1]]
            for g in range(F):
                other = rec[file[rec] != g]
                assert len(set(L[other, g].tolist())) <= 1
    if S == 1:
        return
    # two records sharing a cluster in every sample have the same links into every file but their own ones
    lab = [aa.sample_labels(R, m, o) for m, o, _ in ch.samples]
    always = np.all([x == lab[0] for x in lab], axis=0)
    for a in range(R):
        for b in range(a + 1, R):
            if always[a] and always[b] and lab[0][a] == lab[0][b]:
                keep = [g for g in range(F) if g not in (file[a], file[b])]
                assert (L[a, keep] == L[b, keep]).all()


def test_the_estimators():
    from scipy.optimize import minimize_scalar
    from scipy.special import xlogy

    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(3)
    # two files: Lincoln-Petersen
    for _ in range(50):
        n0, n1 = rng.integers(5, 500, 2)
        m = int(rng.integers(1, min(n0, n1) + 1))
        D = n0 + n1 - m
        est = aa.independence_estimate(np.array([[n0, n1]]), np.array([D]))[0]
        assert est == pytest.approx(n0 * n1 / m, rel=1e-12, abs=0)
    # three and five files: the maximum of the profiled conditional likelihood
    for F in (3, 5):
        for _ in range(10):
            N = int(rng.integers(200, 2000))
            caught = rng.random((N, F)) < rng.uniform(0.1, 0.6, F)
            seen = caught.any(axis=1)
            n, D = caught.sum(axis=0), int(seen.sum())

            def nll(x):
                return -((1 - F) * xlogy(x, x) - xlogy(x - D, x - D) + xlogy(x - n, x - n).sum())

            opt = minimize_scalar(nll, bounds=(D, 100 * N), method="bounded", options={"xatol": 1e-10})
            est = aa.independence_estimate(n[None], np.array([D]))[0]
            assert est == pytest.approx(opt.x, rel=1e-6)
            assert nll(est) <= nll(opt.x) + 1e-9
    # +inf exactly when no file overlaps another
    n = np.array([[3, 4, 5], [3, 4, 5], [12, 1, 1], [0, 0, 7]])
    D = np.array([12, 11, 12, 7])
    est = aa.independence_estimate(n, D)
    assert np.isinf(est).tolist() == [True, False, False, True]
    assert est[2] == 12  # a file holding every observed entity
    # Chapman on a table
    H = np.zeros((1, 4), np.int64)
    H[0, 1:] = [5, 7, 3]  # file 0 only, file 1 only, both
    s = aa.CaptureSummary(H, np.zeros((0, 2), np.int64), [8, 10])
    cols = dict(zip(s.names, s.columns))
    assert cols["chapman[0,1]"][0] == (8 + 1) * (10 + 1) / (3 + 1) - 1
    assert cols["overlap[0,1]"][0] == 3 and cols["observed-entities"][0] == 15
    assert cols["independence"][0] == pytest.approx(8 * 10 / 3, rel=1e-12)
    assert s.names == ["observed-entities", "entities[0]", "entities[1]", "duplicates[0]", "duplicates[1]",
                       "overlap[0,1]", "chapman[0,1]", "independence"]
    one = aa.CaptureSummary(np.array([[0, 4]]), np.zeros((5, 1), np.int64), [5])
    assert one.names == ["observed-entities", "entities[0]", "duplicates[0]"]


def test_infinite_estimates_are_counted_not_averaged():
    from dblink_b200 import analysis_arrays as aa

    H = np.array([[0, 5, 5, 0], [0, 4, 4, 1], [0, 3, 3, 2]], np.int64)
    s = aa.CaptureSummary(H, np.zeros((0, 2), np.int64), [5, 5])
    ind = s.quantity_summary()[s.names.index("independence")]
    assert ind[5] == 1
    finite = [5 * 5 / 1, 5 * 5 / 2]
    assert ind[0] == pytest.approx(np.mean(finite), rel=1e-12) and ind[1] == pytest.approx(np.std(finite), rel=1e-12)


def test_refusals():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(10, 2, 0)
    with pytest.raises(ValueError, match="1 to 12 files"):
        aa.capture_histories(ch, np.zeros(10, np.int64), 13)
    with pytest.raises(ValueError, match="outside"):
        aa.capture_histories(ch, np.full(10, 3), 3)
    with pytest.raises(ValueError, match="at least one sample"):
        aa.capture_histories(aa.ChainArrays(ch.record_ids, np.zeros(0, np.int64), []), np.zeros(10, np.int64), 1)


# ---- the project on 3-file synthetic data -------------------------------------------------------------------------
CONF = """
dblink : {
  data : { path : "%s", recordIdentifier : "rec_id", fileIdentifier : "file_id", %s nullValue : "NA",
           matchingAttributes : [ {name : "a0", similarityFunction : { name : "ConstantSimilarityFn" },
                                   distortionPrior : {alpha : 0.5, beta : 50.0}} ] }
  outputPath : "%s"
  randomSeed : 1
  numChains : %d
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [
    {name : "summarize", parameters : { lowerIterationCutoff : %d, quantities : [%s] }}
    {name : "evaluate", parameters : { lowerIterationCutoff : %d, metrics : [%s] }}
  ]
}
"""
OTHER_QUANTITIES = '"shared-most-probable-clusters", "pairwise-match-probabilities", "cluster-size-distribution"'


def synthetic_data(tmp_path, F=3, R=300, seed=5):
    from dblink_b200 import synth

    g = synth.generate(seed, R, [synth.SynthAttr("a0", "constant", 20, 1.0)], n_files=F)
    path = tmp_path / "data.csv"
    with open(path, "w", newline="") as fh:
        out = csv.writer(fh, lineterminator="\n")
        out.writerow(["rec_id", "file_id", "ent_id", "a0"])
        for r, f, e, v in zip(g["rec_ids"], g["files"], g["ent_ids"], g["values"]):
            out.writerow([f"id{r}", f"f{f}", e, v[0] if v[0] is not None else "NA"])
    return path, [f"id{r}" for r in g["rec_ids"]], np.asarray(g["ent_ids"]), [f"f{f}" for f in g["files"]]


def project(tmp_path, out, chains, quantities, metrics, cutoff=0, entity=True):
    from dblink_b200 import config
    from dblink_b200.project import Project

    path = tmp_path / "data.csv"
    c = CONF % (path, 'entityIdentifier : "ent_id",' if entity else "", str(out) + "/", chains, cutoff, quantities,
                cutoff, metrics)
    return Project(config.parse_string(c), base_dir="")


def write_chains(p, ids, truth, chains, S=8, seed=0):
    """Each chain directory gets a linkage chain of S samples around the truth, sampled through the scripted
    engine."""
    from dblink_b200 import sampler

    rng = np.random.default_rng(seed)
    _, truth = np.unique(truth, return_inverse=True)
    R, E = len(ids), int(truth.max()) + 1
    for d in p.chain_dirs():
        script = []
        for s in range(S + 1):
            link = truth.copy()
            move = rng.random(R) < 0.15
            link[move] = rng.integers(0, E + 20, int(move.sum()))
            script.append((link.astype(np.int32), np.zeros(E + 20, np.int32), None))
        sampler.sample(ScriptedEngine(script, A=1, F=3), ids, ["a0"], S, d)


def snapshot(out):
    got = {}
    for root, _, files in os.walk(out):
        for f in files:
            with open(os.path.join(root, f), "rb") as fh:
                got[os.path.relpath(os.path.join(root, f), out)] = fh.read()
    return got


NEW_FILES = {"capture-histories-samples.csv", "capture-histories.csv", "population-size.csv",
             "population-size-samples.csv", "file-links.csv", "capture-histories-evaluation.csv"}


@pytest.fixture
def host_only(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project as pj

    for name in ("shared_most_probable_clusters", "pairwise_match_counts", "posterior_metric_counts",
                 "capture_histories"):
        monkeypatch.setattr(pj, name, getattr(aa, name))


def read_csv(path):
    with open(path, newline="") as fh:
        return list(csv.reader(fh))


@pytest.mark.parametrize("chains", [1, 2])
def test_project_files(tmp_path, host_only, chains):
    from dblink_b200 import analysis, analysis_arrays as aa

    _, ids, ent, files = synthetic_data(tmp_path)
    base, new = tmp_path / "base", tmp_path / "new"
    p0 = project(tmp_path, base, chains, OTHER_QUANTITIES, '"pairwise"')
    p1 = project(tmp_path, new, chains, OTHER_QUANTITIES + ', "capture-histories"', '"pairwise", "capture-histories"')
    write_chains(p0, ids, ent, chains)
    shutil.copytree(base, new)  # the same chain for both runs
    p0.execute(log=lambda *a: None)
    res = p1.execute(log=lambda *a: None)
    a, b = snapshot(base), snapshot(new)
    assert set(b) - set(a) == NEW_FILES
    text_a, text_b = a.pop("evaluation-results.txt"), b.pop("evaluation-results.txt")
    assert {k: b[k] for k in a} == a  # every other file is byte-identical
    assert text_b.startswith(text_a) and b"Capture histories" in text_b[len(text_a):]

    out = str(new) + "/"
    ch = p1.read_chain(0)
    S, R, F = len(ch.samples), ch.num_records, 3
    assert S == 9 * chains
    fids = ["f0", "f1", "f2"]
    file_of = dict(zip(ids, files))
    cid = [str(x) for x in ch.record_ids.to_pylist()]
    file_num = np.array([fids.index(file_of[r]) for r in cid])
    want_H, want_L = literal(ch, file_num, F)

    rows = read_csv(out + "capture-histories-samples.csv")
    assert rows[0] == ["chain", "iteration", "f0", "f1", "f2", "entities"]
    got = np.zeros_like(want_H)
    seen = []
    for row in rows[1:]:
        s = [i for i, (k, it) in enumerate(zip(ch.chains, ch.iterations)) if (int(k), int(it)) == (int(row[0]),
                                                                                                    int(row[1]))]
        h = sum(int(x) << f for f, x in enumerate(row[2:5]))
        got[s[0], h] = int(row[5])
        seen.append((s[0], h))
    assert seen == sorted(seen) and (got == want_H).all()

    summary = aa.CaptureSummary(want_H, want_L, np.bincount(file_num, minlength=F))
    rows = read_csv(out + "capture-histories.csv")
    assert rows[0] == fids + ["mean", "sd", "q2.5", "q50", "q97.5"]
    assert len(rows) == 8
    for h, row in enumerate(rows[1:], start=1):
        assert [int(x) for x in row[:3]] == [(h >> f) & 1 for f in range(3)]
        v = want_H[:, h].astype(float)
        assert row[3:] == [repr(float(x)) for x in (v.mean(), v.std(), *np.quantile(v, [0.025, 0.5, 0.975]))]

    rows = read_csv(out + "population-size.csv")
    assert rows[0] == ["quantity", "mean", "sd", "q2.5", "q50", "q97.5", "infinite"]
    names = [r[0] for r in rows[1:]]
    assert names == (["observed-entities"] + [f"entities[{f}]" for f in fids] + [f"duplicates[{f}]" for f in fids]
                     + ["overlap[f0,f1]", "overlap[f0,f2]", "overlap[f1,f2]", "chapman[f0,f1]", "chapman[f0,f2]",
                        "chapman[f1,f2]", "independence"])
    D = want_H.sum(axis=1).astype(float)
    assert rows[1][1:] == [repr(float(x)) for x in (D.mean(), D.std(), *np.quantile(D, [0.025, 0.5, 0.975]))] + ["0"]
    samples = read_csv(out + "population-size-samples.csv")
    assert samples[0] == ["chain", "iteration"] + names and len(samples) == S + 1
    assert [int(r[2]) for r in samples[1:]] == want_H.sum(axis=1).tolist()
    ind = summary.columns[-1]
    assert [r[-1] for r in samples[1:]] == [repr(float(x)) for x in ind]

    rows = read_csv(out + "file-links.csv")
    assert rows[0] == ["recordId", "fileId"] + fids
    assert [r[0] for r in rows[1:]] == ids  # data order
    where = {r: i for i, r in enumerate(cid)}
    for row in rows[1:]:
        i = where[row[0]]
        assert row[1] == file_of[row[0]]
        assert row[2:] == [repr(float(x / S)) for x in want_L[i]]

    # the evaluation: the truth counted through the same code as one sample
    truth_H, truth_L = literal(one_sample(np.unique(ent[[ids.index(r) for r in cid]], return_inverse=True)[1]),
                               file_num, F)
    rows = read_csv(out + "capture-histories-evaluation.csv")
    assert rows[0] == ["quantity", "truth", "mean", "q2.5", "q97.5", "inside"]
    assert len(rows) == 1 + 7 + len(names)
    assert rows[1][0] == "history[f0]" and rows[7][0] == "history[f0,f1,f2]"
    assert [r[0] for r in rows[8:]] == names
    for h, row in enumerate(rows[1:8], start=1):
        assert int(row[1]) == truth_H[0, h]
        lo, hi = float(row[3]), float(row[4])
        assert row[5] == str(int(lo <= truth_H[0, h] <= hi))
    brier = ((want_L / S - truth_L) ** 2).mean(axis=0)
    assert res["capture-histories"]["brier"] == pytest.approx(brier, rel=1e-12)
    section = text_b[len(text_a):].decode()
    assert f" Observed:        truth {int(truth_H[0].sum())}," in section
    assert all(f" Brier [{f}]:" in section for f in fids)
    assert section == analysis.format_capture_histories(res["capture-histories"], fids) + "\n"

    run = p1.steps_mk_string().splitlines()
    assert any(x.startswith("  * SummarizeStep: capture-histories counts every sample's clusters") for x in run)
    assert any(x.startswith("  * EvaluateStep: Evaluating the capture histories") for x in run)
    assert not any("capture" in x for x in p0.steps_mk_string().splitlines())


def test_project_refusals(tmp_path, host_only):
    _, ids, ent, _ = synthetic_data(tmp_path)
    p = project(tmp_path, tmp_path / "late", 1, '"capture-histories"', '"capture-histories"', cutoff=10 ** 6)
    write_chains(p, ids, ent, 1, S=2)
    with pytest.raises(ValueError, match="capture-histories needs at least one sample"):
        p.execute(log=lambda *a: None)
    p = project(tmp_path, tmp_path / "noent", 1, '"shared-most-probable-clusters"', '"capture-histories"',
                entity=False)
    write_chains(p, ids, ent, 1, S=2)
    with pytest.raises(ValueError, match="Ground truth entity ids are required"):
        p.execute(log=lambda *a: None)


@pytest.mark.parametrize("where", ["summarize", "evaluate"])
def test_more_than_twelve_files_are_refused(tmp_path, where):
    synthetic_data(tmp_path, F=13, R=400)
    q = '"capture-histories"' if where == "summarize" else '"shared-most-probable-clusters"'
    m = '"capture-histories"' if where == "evaluate" else '"pairwise"'
    p = project(tmp_path, tmp_path / "out", 1, q, m)
    with pytest.raises(ValueError, match="capture-histories supports 1 to 12 files"):
        p.steps()
