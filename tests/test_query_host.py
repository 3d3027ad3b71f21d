"""New records linked to a finished chain, on the host: the numpy path (analysis_arrays.QueryScores) against the exact
posterior of a tiny model, against the oracle's literal PCG-II link weight, and against the literal restatement
(analysis.query_link_probabilities); the distortion-probabilities chain file and its summary; the refusals."""
import csv
import os

import numpy as np
import pytest

from helpers import oracle_setup, synth_problem
from test_oracle_distribution import exact_partition_posterior, tiny_model


def oracle_tables(ix):
    return {"phi": ix.phi, "norm": ix.norm, "rowptr": ix.rowptr, "col": ix.col, "expsim": ix.expsim}


def chain_samples(R, draws):
    """(labels, values[K][A], theta) per recorded (link, y, theta): the non-empty entities as clusters."""
    out = []
    for link, y, theta in draws:
        ent, labels = np.unique(link, return_inverse=True)
        out.append((labels.astype(np.int64), y[ent].astype(np.int32), theta))
    return out


def numpy_result(tab, samples, R, M, t=0.05):
    from dblink_b200 import analysis_arrays as aa

    return aa.link_queries(tab, lambda: iter(samples), R, M, t)


def literal_result(tab, tables, constant, samples, M):
    from dblink_b200 import analysis

    queries = [(int(tab.file[q]), {a: int(v) for a, v in enumerate(tab.x[q]) if v >= 0}) for q in range(len(tab.x))]
    lit = [([np.flatnonzero(lab == k).tolist() for k in range(len(vals))], vals, theta) for lab, vals, theta in samples]
    return analysis.query_link_probabilities(queries, lit, tables, constant, M)


@pytest.mark.parametrize("query", ["near-match", "missing"])
def test_against_the_exact_posterior(oracle, query):
    """Three records sampled with PCG-II (E = 3); the fourth scored as a query.  p(q, r) and p_new match the 4-record
    enumeration's probabilities that the fourth record shares a block with r, and that it is alone."""
    from dblink_b200 import analysis_arrays as aa

    lev, con, x4 = tiny_model(oracle)
    if query == "near-match":  # data ANNA, BOB, ANNE; the query ANNE: an exact and a Levenshtein near match
        x4 = np.array([x4[0], x4[2], x4[1], x4[3]], np.int32)
        x4[3] = [lev.value_id("ANNE"), 0]
    E, alpha, beta = 3, 1.0, 4.0
    exact = exact_partition_posterior(lev, con, x4, E, alpha, beta)
    m = oracle.Model([lev, con], [alpha, alpha], [beta, beta], None, 4242, 1)
    st = oracle.State.init(m, x4[:3], np.zeros(3, np.int32), E)
    st.sweep(oracle.PCG_II, 300)
    draws = []
    for _ in range(6000):
        st.sweep(oracle.PCG_II, 3)
        draws.append((st.link, st.y, st.theta))
    tab = aa.QueryTables(x4[3:4], [0], [oracle_tables(lev), oracle_tables(con)], [False, True], 1)
    res = numpy_result(tab, chain_samples(3, draws), 3, E, t=1e-6)
    p = dict(zip(res.record.tolist(), res.probability.tolist()))
    for r in range(3):
        want = sum(v for part, v in exact.items() if any(3 in b and r in b for b in part))
        assert abs(p.get(r, 0.0) - want) < 0.02, (r, p.get(r), want)
    alone = sum(v for part, v in exact.items() if (3,) in part)
    assert abs(res.new_entity_probability[0] - alone) < 0.02


def test_weights_equal_the_oracle_literal_link_weight(oracle):
    """On a 2-file synthetic problem with missing values and constant, Levenshtein and Jaro-Winkler attributes, the
    numpy w(q, e) = m rho of existing records against every entity equals the oracle's literal PCG-II weight."""
    from dblink_b200 import analysis_arrays as aa, synth

    C = synth.SynthAttr
    g = synth_problem(seed=5, R=200, n_files=2, missing=0.1,
                      attrs=[C("c", "constant", 6), C("lev", "levenshtein", 40), C("jw", "jaro-winkler", 30)])
    m, st, tree, x, file = oracle_setup(oracle, g, 3)
    tables = [oracle_tables(ix) for ix in m.indexes]
    constant = [ix.is_const for ix in m.indexes]
    qs = np.arange(0, st.R, 9)
    tab = aa.QueryTables(x[qs], file[qs], tables, constant, 2)
    theta = np.random.default_rng(1).uniform(0.02, 0.4, (m.A, 2))
    st = oracle.State.from_arrays(m, x, file, st.z, st.link, st.y, theta, 0)
    coef = aa.query_coefficients(tab, theta)
    w = aa.query_rho(tab, coef, st.y, np.arange(len(qs))) * np.exp(coef[2])[:, None]
    for i, r in enumerate(qs):
        want = st.link_weights(int(r), oracle.PCG_II, np.arange(st.E, dtype=np.int32), literal=True)
        np.testing.assert_allclose(w[i], want, rtol=1e-12, atol=0)
    pr = aa.query_pair_rho(tab, coef, st.y, np.repeat(np.arange(len(qs)), 5), np.tile(np.arange(5), len(qs)))
    np.testing.assert_allclose(pr, aa.query_rho(tab, coef, st.y[:5], np.arange(len(qs))).ravel(), rtol=1e-15)


def random_case(oracle, seed, S=4, singletons=False):
    from dblink_b200 import analysis_arrays as aa, synth

    C = synth.SynthAttr
    g = synth_problem(seed=seed, R=60, n_files=2, missing=0.1,
                      attrs=[C("c", "constant", 4), C("lev", "levenshtein", 12), C("jw", "jaro-winkler", 10)])
    m, st, tree, x, file = oracle_setup(oracle, g, seed)
    tables = [oracle_tables(ix) for ix in m.indexes]
    constant = [ix.is_const for ix in m.indexes]
    rng = np.random.default_rng(seed)
    R, M = 40, 55
    samples = []
    for _ in range(S):
        K = R if singletons else int(rng.integers(5, R))
        lab = np.r_[np.arange(K), rng.integers(0, K, R - K)] if not singletons else np.arange(R)
        rng.shuffle(lab)
        vals = np.stack([rng.integers(0, ix.V, K) for ix in m.indexes], 1).astype(np.int32)
        samples.append((lab.astype(np.int64), vals, rng.uniform(0.05, 0.6, (m.A, 2))))
    qx = x[R:].copy()
    tab = aa.QueryTables(qx, file[R:], tables, constant, 2)
    return tab, tables, constant, samples, R, M


@pytest.mark.parametrize("seed", range(4))
def test_numpy_equals_the_literal_restatement(oracle, seed):
    from dblink_b200 import analysis_arrays as aa

    tab, tables, constant, samples, R, M = random_case(oracle, seed)
    p_lit, new_lit, ess_lit = literal_result(tab, tables, constant, samples, M)
    for t in (1e-300, 0.05, 0.3):
        res = numpy_result(tab, samples, R, M, t)
        np.testing.assert_allclose(res.new_entity_probability, new_lit, rtol=1e-12)
        np.testing.assert_allclose(res.effective_samples, ess_lit, rtol=1e-12)
        got = dict(zip(zip(res.query.tolist(), res.record.tolist()), res.probability.tolist()))
        for key, v in got.items():
            assert v == pytest.approx(p_lit[key], rel=1e-12)
        assert t < 1e-200 or not any(abs(v - t) < 1e-9 for v in p_lit.values())
        q, r, p = aa.query_link_rows(res, t, np.arange(R))
        assert set(zip(q.tolist(), r.tolist())) == {k for k, v in p_lit.items() if v >= t}


def test_one_sample_of_singletons_sums_to_one(oracle):
    tab, tables, constant, samples, R, M = random_case(oracle, 7, S=1, singletons=True)
    res = numpy_result(tab, samples, R, M, 1e-300)
    total = np.bincount(res.query, weights=res.probability, minlength=len(tab.x)) + res.new_entity_probability
    np.testing.assert_allclose(total, 1.0, rtol=1e-12)


def test_a_query_with_every_attribute_missing(oracle):
    tab, tables, constant, samples, R, M = random_case(oracle, 3)
    tab.x[0] = -1
    tab.psi[0] = 0.0
    res = numpy_result(tab, samples, R, M, 1e-9)
    np.testing.assert_allclose(res.probability[res.query == 0], 1.0 / M, rtol=1e-12)
    want = sum(M - len(v) for _, v, _ in samples) / (len(samples) * M)
    assert res.new_entity_probability[0] == pytest.approx(want, rel=1e-12)


def test_refusals(oracle):
    from dblink_b200 import analysis_arrays as aa

    tab, tables, constant, samples, R, M = random_case(oracle, 1)
    lab, vals, th = samples[0]
    for t in (0.0, -0.1, 1.5, True):
        with pytest.raises(ValueError, match="minLinkProbability"):
            aa.QueryScores(tab, R, M, t)
    qs = aa.QueryScores(tab, R, M, 0.05)
    with pytest.raises(ValueError, match="more than the population size"):
        aa.QueryScores(tab, R, R - 1, 0.05).add_sample(np.arange(R), np.zeros((R, 3), np.int32), th)
    with pytest.raises(ValueError, match="labels"):
        qs.add_sample(np.r_[lab[:-1], len(vals)], vals, th)
    bad = vals.copy()
    bad[0, 1] = tab.num_values[1]
    with pytest.raises(ValueError, match="value id"):
        qs.add_sample(lab, bad, th)
    with pytest.raises(ValueError, match=r"\[0, 1\]"):
        qs.add_sample(lab, vals, th + 1.0)
    with pytest.raises(ValueError, match="every sample of pass 1"):
        qs.read()
    small = aa.QueryScores(tab, R, M, 1e-9, max_candidates=3)
    with pytest.raises(ValueError, match="candidate"):
        small.add_sample(lab, vals, th)
    assert small.num_samples == 0 and len(small.keys) == 0
    qs.add_sample(lab, vals, th)
    qs.score_sample(lab, vals, th)
    with pytest.raises(ValueError, match="more samples than pass 1"):
        qs.score_sample(lab, vals, th)
    with pytest.raises(ValueError, match="at least one sample"):
        aa.link_queries(tab, lambda: iter(()), R, M, 0.05)


def test_distortion_chain_writer_and_summary(tmp_path):
    from dblink_b200 import analysis_arrays as aa, writers

    cols = writers.distortion_columns(["a", "b,c"], ["0", "1"])
    assert cols == ["a[0]", "a[1]", "b,c[0]", "b,c[1]"]
    path = str(tmp_path / writers.DISTORTION_CHAIN)
    rng = np.random.default_rng(0)
    th = rng.uniform(0, 1, (5, 2, 2))
    w = writers.DistortionChainWriter(path, cols)
    for i in range(3):
        w.write_row(i * 10, th[i])
    w.close()
    w = writers.DistortionChainWriter(path, cols, append=True)  # resume appends
    for i in range(3, 5):
        w.write_row(i * 10, th[i])
    w.close()
    with open(path, newline="") as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["iteration"] + cols and len(rows) == 6
    assert [float(v) for v in rows[3][1:]] == th[2].ravel().tolist()

    class Ch:
        iterations = np.array([20, 30, 40])
        chains = np.zeros(3, np.int64)
        samples = [None] * 3

    got = aa.read_distortion_probabilities([str(tmp_path)], Ch, 2, 2)
    np.testing.assert_array_equal(got, th[2:])
    Ch.iterations = np.array([20, 35])
    Ch.samples = [None] * 2
    with pytest.raises(ValueError, match="iteration 35 has no distortion probabilities"):
        aa.read_distortion_probabilities([str(tmp_path)], Ch, 2, 2)
    summ = aa.distortion_summary(th)
    flat = th.reshape(5, -1)
    for j, (mean, sd, lo, mid, hi, S) in enumerate(summ):
        assert (mean, sd, S) == (flat[:, j].mean(), flat[:, j].std(), 5)
        assert (lo, mid, hi) == tuple(np.quantile(flat[:, j], [0.025, 0.5, 0.975]))
    writers.save_distortion_probabilities([("a", "0", s[:5], s[5]) for s in summ[:1]], str(tmp_path))
    with open(tmp_path / "distortion-probabilities.csv") as fh:
        assert fh.readline() == "attribute,file,mean,sd,q2.5,q50,q97.5,samples\n"


class _Engine:
    """A scripted engine: links, blocks and a summary with theta, one iteration per sweep."""

    def __init__(self, R=6, A=2, F=2, iteration=0):
        self.iteration, self.R, self.A, self.F = iteration, R, A, F
        self.num_entities = R

    def links(self):
        return np.arange(self.R) % 3, np.zeros(self.R, np.int32)

    def summary(self):
        th = np.full((self.A, self.F), 0.1) + self.iteration / 1000
        return {"iteration": self.iteration, "num_isolates": 0, "log_likelihood": 0.0,
                "agg_dist": np.zeros((self.A, self.F), np.int64), "rec_dist": np.zeros(self.A + 1, np.int64),
                "theta": th}

    def sweep(self, sampler, n):
        self.iteration += n


def test_sampler_writes_and_removes_the_theta_chain(tmp_path):
    from dblink_b200 import sampler, writers

    cols = writers.distortion_columns(["a", "b"], ["0", "1"])
    out = str(tmp_path / "o")
    sampler.sample(_Engine(), [str(i) for i in range(6)], ["a", "b"], 3, out, distortion_columns=cols)
    path = os.path.join(out, writers.DISTORTION_CHAIN)
    with open(path) as fh:
        lines = fh.read().splitlines()
    assert lines[0] == "iteration,a[0],a[1],b[0],b[1]" and [l.split(",")[0] for l in lines[1:]] == ["0", "1", "2",
                                                                                                     "3"]
    sampler.sample(_Engine(iteration=3), [str(i) for i in range(6)], ["a", "b"], 2, out, distortion_columns=cols)
    with open(path) as fh:
        assert [l.split(",")[0] for l in fh.read().splitlines()[1:]] == ["0", "1", "2", "3", "4", "5"]
    before = sorted(os.listdir(out))
    sampler.sample(_Engine(), [str(i) for i in range(6)], ["a", "b"], 2, out)  # a new chain without the option
    assert not os.path.exists(path) and sorted(os.listdir(out)) == [f for f in before if f != writers.DISTORTION_CHAIN]
    class K2(_Engine):
        num_chains = 2

        def download_chains(self, links_only=False):
            return [{"link": np.arange(self.R) % 2, "block": np.zeros(self.R, np.int32)} for _ in range(2)]

        def chain_summary(self, k):
            return self.summary()

    out2 = str(tmp_path / "k2")
    sampler.sample(K2(), [str(i) for i in range(6)], ["a", "b"], 1, out2, distortion_columns=cols)
    for k in range(2):
        assert os.path.exists(os.path.join(out2, f"chain-{k}", writers.DISTORTION_CHAIN))


# ---- the step on RLdata500, on the host -------------------------------------------------------------------------
PROJECT_CONF = """
dblink : {
  data : { path : "%s", recordIdentifier : "rec_id", nullValue : "NA", %s
           matchingAttributes : [
             {name : "fname_c1", similarityFunction : {name : "LevenshteinSimilarityFn",
              parameters : {threshold : 7.0, maxSimilarity : 10.0}}, distortionPrior : {alpha : 1.0, beta : 50.0}},
             {name : "lname_c1", similarityFunction : {name : "JaroWinklerSimilarityFn",
              parameters : {threshold : 7.0, maxSimilarity : 10.0}}, distortionPrior : {alpha : 1.0, beta : 50.0}},
             {name : "by", similarityFunction : {name : "ConstantSimilarityFn"},
              distortionPrior : {alpha : 1.0, beta : 50.0}} ] }
  outputPath : "%s"
  randomSeed : 1
  numChains : %d
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [ %s ]
}
"""
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def rldata500(tmp_path, files=False):
    """RLdata500 as data.csv (with a file column of two files when `files`), and its first 50 records as queries.csv,
    two of them with values the data never holds."""
    import gzip

    with gzip.open(os.path.join(GOLDEN, "RLdata500.csv.gz"), "rt") as fh:
        rows = list(csv.DictReader(fh))
    cols = ["rec_id", "fname_c1", "lname_c1", "by"] + (["file"] if files else [])
    for i, r in enumerate(rows):
        r["file"] = "ab"[i % 2]
    with open(tmp_path / "data.csv", "w", newline="") as fh:
        w = csv.writer(fh)
        w.writerow(cols)
        w.writerows([[r[c] for c in cols] for r in rows])
    queries = [dict(r) for r in rows[:50]]
    queries[3]["fname_c1"] = "ZZYZX"
    queries[7]["by"] = "1234"
    queries[7]["lname_c1"] = "QQQQQQ"
    for q in queries:
        q["rec_id"] = "q-" + q["rec_id"]
    with open(tmp_path / "queries.csv", "w", newline="") as fh:
        w = csv.writer(fh)
        w.writerow(cols)
        w.writerows([[q[c] for c in cols] for q in queries])
    return rows


def project_at(tmp_path, out, steps, chains=1, files=False):
    from dblink_b200 import config
    from dblink_b200.project import Project

    fid = 'fileIdentifier : "file",' if files else ""
    return Project(config.parse_string(PROJECT_CONF % (tmp_path / "data.csv", fid, str(tmp_path / out) + "/", chains,
                                                       steps)), base_dir="")


class _RecordsEngine:
    """A scripted engine over R records and E = R entities: every sweep draws new links near `truth`, entity values
    near each entity's records and theta, from the iteration alone."""

    def __init__(self, truth, x, V, F, seed):
        self.truth, self.x, self.V, self.F, self.seed = np.asarray(truth), x, np.asarray(V), F, seed
        self.iteration, self.num_entities = 0, len(truth)

    def _state(self):
        rng = np.random.default_rng((self.seed, self.iteration))
        R = len(self.truth)
        link = self.truth.copy()
        move = rng.random(R) < 0.1
        link[move] = rng.integers(0, R, int(move.sum()))
        y = (rng.random((R, len(self.V))) * self.V).astype(np.int32)
        own = np.where(self.x >= 0, self.x, y[link])
        y[link] = own
        return link.astype(np.int32), y, rng.uniform(0.005, 0.05, (len(self.V), self.F))

    def links(self):
        return self._state()[0], np.zeros(self.num_entities, np.int32)

    def download_state(self, keys=None):
        link, y, _ = self._state()
        return {"link": link, "y": y, "block": np.zeros(self.num_entities, np.int32)}

    def summary(self):
        A = len(self.V)
        return {"iteration": self.iteration, "num_isolates": 0, "log_likelihood": 0.0,
                "agg_dist": np.zeros((A, self.F), np.int64), "rec_dist": np.zeros(A + 1, np.int64),
                "theta": self._state()[2]}

    def sweep(self, sampler, n):
        self.iteration += n


def sample_project(p, on, seed=0, size=12):
    """The sample step of p over _RecordsEngine (one per chain), with both options on or off."""
    from dblink_b200 import sampler

    d = p.load()
    R = len(d["rec_ids"])
    V = [ix.num_values for ix in d["cache"].indexes]
    for k, dr in enumerate(p.chain_dirs()):
        eng = _RecordsEngine(np.arange(R) // 2 * 2, d["x"], V, len(d["cache"].file_ids), seed + k)
        sampler.sample(eng, d["rec_ids"], [a.name for a in p.matching_attributes], size, dr, 2, 3, sampler="PCG-II",
                       entity_values=p.attribute_values() if on else None,
                       distortion_columns=p.distortion_columns() if on else None)


def tree_bytes(root, skip=()):
    got = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            rel = os.path.relpath(os.path.join(d, f), root)
            if rel in skip:
                continue
            with open(os.path.join(d, f), "rb") as fh:
                data = fh.read()
            if f == "diagnostics.csv":  # the wall-clock column aside
                data = b"\n".join(b",".join(l.split(b",")[:1] + l.split(b",")[2:]) for l in data.splitlines())
            got[rel] = data
    return got


def host_link_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    monkeypatch.setattr(project, "link_queries", aa.link_queries)
    monkeypatch.setattr(project, "pairwise_match_counts", aa.pairwise_match_counts)


OLD_STEPS = '{name : "summarize", parameters : { lowerIterationCutoff : 0, quantities : ["pairwise-match-probabilities"]}}'
NEW_STEPS = ('{name : "summarize", parameters : { lowerIterationCutoff : 0, quantities : ["pairwise-match-probabilities",'
             ' "distortion-probabilities"]}}, {name : "link-records", parameters : {queryPath : "%s"}}')


@pytest.mark.parametrize("chains,files", [(1, False), (2, True)])
def test_project_on_rldata500(tmp_path, monkeypatch, chains, files):
    """Sample with both options, summarize and link 50 records: every file a run without them writes is unchanged;
    the links equal the literal restatement's pairs at p >= 0.05, unseen values are listed and count as missing; with
    two chains and two files the samples of both chain directories are pooled."""
    from dblink_b200 import analysis, analysis_arrays as aa

    host_link_paths(monkeypatch)
    rldata500(tmp_path, files)
    off = project_at(tmp_path, "off", OLD_STEPS, chains, files)
    sample_project(off, False)
    off.execute(log=lambda *a: None)
    on = project_at(tmp_path, "on", NEW_STEPS % (tmp_path / "queries.csv"), chains, files)
    sample_project(on, True)
    on.execute(log=lambda *a: None)
    new = {"distortion-probabilities.csv", "query-links.csv", "query-summary.csv"}
    per_chain = {"distortion-probabilities-chain.csv"}
    a = tree_bytes(tmp_path / "off")
    b = tree_bytes(tmp_path / "on")
    extra = {k for k in b if k not in a}
    assert {k for k in extra if "entity-values-chain" not in k and os.path.basename(k) not in per_chain} == new
    for k, v in a.items():
        assert b[k] == v, k

    # the literal restatement over the samples read back from the files
    ch = on.read_chain(0)
    assert len(ch.samples) == 12 * chains and set(ch.chains.tolist()) == set(range(chains))
    names = [x.name for x in on.matching_attributes]
    d = on.load()
    F = len(d["cache"].file_ids)
    theta = aa.read_distortion_probabilities(on.chain_dirs(), ch, 3, F)
    samples = []
    for s, v in enumerate(aa.read_entity_values(on.chain_dirs(), ch, names, on.attribute_values())):
        mem, off_, _ = ch.samples[s]
        lab, vals = aa.query_sample_arrays(ch.num_records, mem, off_, v)
        samples.append(([np.flatnonzero(lab == k).tolist() for k in range(len(vals))], vals, theta[s]))
    ids, x, file, unseen = on.read_queries(str(tmp_path / "queries.csv"))
    assert unseen[3] == ["fname_c1"] and unseen[7] == ["lname_c1", "by"] and x[3, 0] == -1 and (x[7, 1:] == -1).all()
    assert all(not u for i, u in enumerate(unseen) if i not in (3, 7))
    tables = [ix.tables() for ix in d["cache"].indexes]
    constant = [x_.is_constant for x_ in on.matching_attributes]
    queries = [(int(file[q]), {a: int(v) for a, v in enumerate(x[q]) if v >= 0}) for q in range(len(ids))]
    p_lit, new_lit, ess_lit = analysis.query_link_probabilities(queries, samples, tables, constant, ch.num_records)
    chain_ids = ch.record_ids.to_pylist()
    with open(tmp_path / "on" / "query-links.csv", newline="") as fh:
        rows = list(csv.reader(fh))
    assert rows[0] == ["queryId", "recordId", "probability"]
    got = {(r[0], r[1]): float(r[2]) for r in rows[1:]}
    want = {(ids[q], chain_ids[r]): v for (q, r), v in p_lit.items() if v >= 0.05}
    assert not any(abs(v - 0.05) < 1e-9 for v in p_lit.values())
    assert set(got) == set(want) and len(got) > 30
    for k, v in got.items():
        assert v == pytest.approx(want[k], rel=1e-10)
    order = [ids.index(r[0]) for r in rows[1:]]
    assert order == sorted(order)  # query-file order
    with open(tmp_path / "on" / "query-summary.csv", newline="") as fh:
        summ = list(csv.reader(fh))
    assert summ[0] == ["queryId", "newEntityProbability", "bestRecordId", "bestProbability", "effectiveSamples",
                       "unseenAttributes"]
    assert [r[0] for r in summ[1:]] == ids
    assert summ[4][5] == "fname_c1" and summ[8][5] == "lname_c1;by"
    for q, r in enumerate(summ[1:]):
        assert float(r[1]) == pytest.approx(new_lit[q], rel=1e-10)
        assert float(r[4]) == pytest.approx(ess_lit[q], rel=1e-10)
        mine = [row for row in rows[1:] if row[0] == ids[q]]
        assert r[2:4] == (mine[0][1:3] if mine else ["", ""])
    with open(tmp_path / "on" / "distortion-probabilities.csv", newline="") as fh:
        dp = list(csv.reader(fh))
    assert len(dp) == 1 + 3 * F and dp[1][:2] == ["fname_c1", d["cache"].file_ids[0]]
    assert dp[1][-1] == str(len(ch.samples))
    run = on.steps_mk_string()
    assert "LinkRecordsStep" in run and "queries are not linked to each other" in run


STEP = '{name : "link-records", parameters : {queryPath : "%s"%s}}'


def test_project_refusals(tmp_path, monkeypatch):
    host_link_paths(monkeypatch)
    rows = rldata500(tmp_path, files=True)
    q = str(tmp_path / "queries.csv")
    p = project_at(tmp_path, "out", STEP % (q, ""), 1, True)
    sample_project(p, True, size=3)

    def run(path=q, extra="", out="out"):
        project_at(tmp_path, out, STEP % (path, extra), 1, True).execute(log=lambda *a: None)

    run()  # the baseline works
    for t in ("0.0", "1.5", "-1"):
        with pytest.raises(ValueError, match=r"minLinkProbability must be in \(0, 1\]"):
            run(extra=", minLinkProbability : " + t)
    with pytest.raises(ValueError, match="needs queryPath"):
        project_at(tmp_path, "out", '{name : "link-records", parameters : {}}', 1, True).steps()
    text = open(q).read().splitlines()

    def variant(name, lines):
        path = tmp_path / name
        path.write_text("\n".join(lines) + "\n")
        return str(path)

    with pytest.raises(ValueError, match="lacks the column"):
        run(variant("nocol.csv", [",".join(l.split(",")[:3]) for l in text]))
    with pytest.raises(ValueError, match="lacks the column"):
        run(variant("nofile.csv", [",".join(l.split(",")[:4]) for l in text]))
    with pytest.raises(ValueError, match="duplicate record ids"):
        run(variant("dup.csv", text + [text[1]]))
    with pytest.raises(ValueError, match="file id 'c'"):
        run(variant("badfile.csv", text[:2] + [text[2].rsplit(",", 1)[0] + ",c"]))
    with pytest.raises(ValueError, match="has no records"):
        run(variant("empty.csv", text[:1]))
    with pytest.raises(ValueError, match="at least one sample"):
        run(extra=", lowerIterationCutoff : 1000")
    # a chain without theta, and one without entity values, past the cutoff
    p2 = project_at(tmp_path, "bare", STEP % (q, ""), 1, True)
    sample_project(p2, False, size=3)
    with pytest.raises(ValueError, match="has no distortion probabilities"):
        run(out="bare")
    os.remove(tmp_path / "out" / "entity-values-chain.parquet" / os.listdir(
        tmp_path / "out" / "entity-values-chain.parquet")[0] / "part-00000.parquet")
    with pytest.raises(ValueError, match="no entity values|do not match"):
        run()
    assert len(rows) == 500
