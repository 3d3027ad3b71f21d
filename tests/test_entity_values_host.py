"""The posterior of the entity values of a point estimate's clusters, on the host: the numpy counts
(analysis_arrays.EntityValueCounts) against the literal analysis.entity_value_counts on random chains with random
values, and the identity sum over v of count(c, v) = |c| S; entity-values-chain.parquet written beside the linkage
chain and read back aligned with its samples (empty partitions, partition ids of two digits, several files, append on
resume, pooled chains); every refusal; sampler.sample over a scripted engine; the files and run.txt lines that
Project.execute writes on RLdata500; the C ABI's NULL-handle refusal."""
import csv
import gzip
import os

import numpy as np
import pytest

from test_binder_host import project_of
from test_credible_ball_host import centers_of
from test_match_probabilities_host import as_set_chain, random_chain

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def random_values(ch, A, V, seed):
    """Per sample: int32[A][R] (each record gets the value of its cluster's entity) and, for analysis.py, per attribute
    {frozenset of the cluster's ids: value}."""
    rng = np.random.default_rng(seed)
    _, ids = as_set_chain(ch)
    arrays, dicts = [], []
    for mem, off, _ in ch.samples:
        nc = len(off) - 1
        per_cluster = rng.integers(0, V, (A, nc)).astype(np.int32)
        out = np.empty((A, ch.num_records), np.int32)
        out[:, mem] = np.repeat(per_cluster, np.diff(off), axis=1)
        arrays.append(out)
        dicts.append([{frozenset(ids[i] for i in mem[off[c]:off[c + 1]]): int(per_cluster[a, c]) for c in range(nc)}
                      for a in range(A)])
    return arrays, dicts


@pytest.mark.parametrize("seed", range(12))
def test_numpy_counts_equal_the_literal_counts(seed):
    from dblink_b200 import analysis, analysis_arrays as aa

    rng = np.random.default_rng(seed)
    R, S = int(rng.integers(1, 31)), int(rng.integers(1, 13))
    A, V = 2, [2, 3, 5][seed % 3]  # few values: ties are common
    ch = random_chain(R, S, seed=7000 + seed)
    chain, ids = as_set_chain(ch)
    arrays, dicts = random_values(ch, A, V, seed)
    for labels in centers_of(ch, rng):
        lab = aa.canonical_clusters(labels)
        C = int(lab.max()) + 1
        center = [frozenset(ids[i] for i in np.flatnonzero(lab == k)) for k in range(C)]
        want = analysis.entity_value_counts(chain, dicts, center)
        modes = analysis.entity_value_modes(want, C, A)
        for a in range(A):
            with aa.EntityValueCounts(lab, C, V) as h:
                for x in arrays:
                    h.add_sample(x[a])
                cl, v, n = h.table()
                assert n.dtype == np.int64
                assert {(int(k), a, int(x)): int(c) for k, x, c in zip(cl, v, n)} == {
                    key: c for key, c in want.items() if key[1] == a}
                # every record of c counts once per sample
                assert np.bincount(cl, weights=n, minlength=C).astype(np.int64).tolist() == [
                    len(c) * S for c in center]
                mode, count = h.modes()
                assert mode.tolist() == [modes[(k, a)][0] for k in range(C)]
                assert count.tolist() == [modes[(k, a)][1] for k in range(C)]
        m, c, s = aa.entity_value_modes(lab, iter(arrays), [V] * A)
        assert s == S and m.shape == c.shape == (A, C) and m.dtype == np.int32 and c.dtype == np.int64
        assert m.tolist() == [[modes[(k, a)][0] for k in range(C)] for a in range(A)]


def test_ties_go_to_the_smallest_value():
    from dblink_b200 import analysis_arrays as aa

    lab = np.array([0, 0, 1, 1, 1, 2])
    h = aa.EntityValueCounts(lab, 3, 4)
    h.add_sample([3, 1, 2, 2, 0, 3])
    h.add_sample([1, 3, 0, 0, 2, 3])
    mode, count = h.modes()
    assert mode.tolist() == [1, 0, 3] and count.tolist() == [2, 3, 2]
    with pytest.raises(ValueError, match="outside"):
        h.add_sample([0, 0, 0, 0, 0, 4])
    with pytest.raises(ValueError, match="no sample added"):
        aa.EntityValueCounts(lab, 3, 4).modes()


# ---- entity-values-chain.parquet ---------------------------------------------------------------------------------
NAMES = ["fname", "by"]
VALUES = [["ann", "bob", "carl, jr", 'dee "d"', "eve"], ["1950", "1961", "1972"]]


def engine_states(R, E, S, seed, blocks=12):
    """S (iteration, link, block_of_entity, y) of R records and E entities over `blocks` partitions, some empty."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(S):
        link = rng.integers(0, E, R).astype(np.int32)
        blk = rng.integers(0, blocks, E).astype(np.int32)
        blk[blk == 3] = 11  # partitions 3 and 7 (usually) hold isolated entities only, or none
        blk[link[link % 5 == 0]] = 7
        blk[link] = np.where(blk[link] == 7, 8, blk[link])
        y = np.stack([rng.integers(0, len(v), E) for v in VALUES], 1).astype(np.int32)
        out.append((10 * (s + 1), link, blk, y))
    return out


def write_chain(d, states, ids, buffer=2, append=False, values=True):
    from dblink_b200 import writers as w

    lw = w.LinkageChainWriter(os.path.join(d, "linkage-chain.parquet"), buffer, append)
    ew = (w.EntityValuesChainWriter(os.path.join(d, "entity-values-chain.parquet"), NAMES, buffer, append, lw.file_no)
          if values else None)
    for it, link, blk, y in states:
        lw.append(it, w.linkage_structure_arrow(link, blk, ids))
        if ew:
            ew.append(it, w.entity_values_arrow(link, blk, y, VALUES))
    lw.close()
    if ew:
        ew.close()


def attribute_values():
    import pyarrow as pa

    return [pa.array(v, pa.string()) for v in VALUES]


def expected(ch, states, ids):
    """Per sample int32[A][R] in the chain's record order: y of the entity each record links to."""
    pos = {r: i for i, r in enumerate(ch.record_ids.to_pylist())}
    order = np.array([pos[r] for r in ids])
    out = []
    for _, link, _, y in states:
        x = np.empty((len(NAMES), len(ids)), np.int32)
        x[:, order] = y[link].T
        out.append(x)
    return out


def test_the_writer_and_reader_round_trip(tmp_path):
    from dblink_b200 import analysis_arrays as aa

    R, E = 60, 45
    ids = [f"r{i}" for i in range(R)]
    states = engine_states(R, E, 7, seed=1)
    d = str(tmp_path)
    write_chain(d, states, ids)
    parts = sorted(os.listdir(os.path.join(d, "entity-values-chain.parquet")))
    assert parts == sorted(os.listdir(os.path.join(d, "linkage-chain.parquet")))
    assert "partitionId=11" in parts and "partitionId=3" not in parts
    for p in parts:  # the same files, flush by flush
        assert (sorted(os.listdir(os.path.join(d, "entity-values-chain.parquet", p)))
                == sorted(os.listdir(os.path.join(d, "linkage-chain.parquet", p))))
    assert len(os.listdir(os.path.join(d, "linkage-chain.parquet", parts[0]))) == 4  # 7 samples, 2 per file

    import pyarrow.parquet as pq

    t = pq.read_table(os.path.join(d, "entity-values-chain.parquet", "partitionId=11"))
    assert t.schema.names == ["iteration"] + NAMES and t.schema.field("fname").type.value_type == "string"
    ch = aa.read_chain_arrays(os.path.join(d, "linkage-chain.parquet"))
    got = list(aa.read_entity_values([d], ch, NAMES, attribute_values()))
    want = expected(ch, states, ids)
    assert len(got) == len(want) == 7
    for g, x in zip(got, want):
        assert g.dtype == np.int32 and (g == x).all()

    # resume: the new samples append files numbered after the linkage chain's
    more = engine_states(R, E, 3, seed=2)
    more = [(it + 70, l, b, y) for it, l, b, y in more]
    write_chain(d, more, ids, append=True)
    ch = aa.read_chain_arrays(os.path.join(d, "linkage-chain.parquet"), 30)
    got = list(aa.read_entity_values([d], ch, NAMES, attribute_values()))
    want = expected(ch, (states + more)[2:], ids)
    assert [int(i) for i in ch.iterations] == [30, 40, 50, 60, 70, 80, 90, 100]
    assert all((g == x).all() for g, x in zip(got, want)) and len(got) == 8


def test_an_empty_partition_has_empty_lists(tmp_path):
    import pyarrow.parquet as pq

    from dblink_b200 import analysis_arrays as aa

    ids = ["a", "b", "c"]
    link, blk = np.array([0, 0, 2], np.int32), np.array([1, 10, 1], np.int32)  # entity 1 (partition 10) is isolated
    y = np.array([[4, 0], [1, 1], [2, 2]], np.int32)
    write_chain(str(tmp_path), [(5, link, blk, y)], ids)
    t = pq.read_table(os.path.join(tmp_path, "entity-values-chain.parquet", "partitionId=10")).to_pydict()
    assert t == {"iteration": [5], "fname": [[]], "by": [[]]}
    t = pq.read_table(os.path.join(tmp_path, "entity-values-chain.parquet", "partitionId=1")).to_pydict()
    assert t == {"iteration": [5], "fname": [["eve", "carl, jr"]], "by": [["1950", "1972"]]}
    ch = aa.read_chain_arrays(os.path.join(tmp_path, "linkage-chain.parquet"))
    (got,) = aa.read_entity_values([str(tmp_path)], ch, NAMES, attribute_values())
    pos = {r: i for i, r in enumerate(ch.record_ids.to_pylist())}
    assert got[:, [pos["a"], pos["b"], pos["c"]]].tolist() == [[4, 4, 2], [0, 0, 2]]


def test_pooled_chains_are_read_chain_major(tmp_path):
    from dblink_b200 import analysis_arrays as aa

    R, E = 40, 30
    ids = [f"r{i}" for i in range(R)]
    dirs, states = [], []
    for k in range(2):
        dirs.append(str(tmp_path / f"chain-{k}"))
        states.append(engine_states(R, E, 5, seed=10 + k))
        write_chain(dirs[-1], states[-1], ids[::-1] if k else ids)  # the second chain meets the records in another order
    ch = aa.read_pooled_chain_arrays([os.path.join(d, "linkage-chain.parquet") for d in dirs], 20)
    got = list(aa.read_entity_values(dirs, ch, NAMES, attribute_values()))
    assert ch.chains.tolist() == [0] * 4 + [1] * 4
    one = [aa.read_chain_arrays(os.path.join(d, "linkage-chain.parquet"), 20) for d in dirs]
    want = []
    for k in range(2):
        wk = expected(one[k], states[k][1:], ids[::-1] if k else ids)
        # into the pooled record order
        pos = {r: i for i, r in enumerate(ch.record_ids.to_pylist())}
        perm = np.array([pos[r] for r in one[k].record_ids.to_pylist()])
        for x in wk:
            y = np.empty_like(x)
            y[:, perm] = x
            want.append(y)
    assert len(got) == 8 and all((g == x).all() for g, x in zip(got, want))


def test_refusals_of_the_reader(tmp_path):
    import pyarrow as pa
    import pyarrow.parquet as pq

    from dblink_b200 import analysis_arrays as aa

    R, E = 30, 20
    ids = [f"r{i}" for i in range(R)]
    states = engine_states(R, E, 4, seed=3)
    # the first two samples without entity values: a run resumed with saveEntityValues switched on
    d = str(tmp_path / "resumed")
    write_chain(d, states[:2], ids, values=False)
    write_chain(d, states[2:], ids, append=True)
    path = os.path.join(d, "linkage-chain.parquet")
    with pytest.raises(ValueError, match="iteration 10 has no entity values.*raise lowerIterationCutoff"):
        list(aa.read_entity_values([d], aa.read_chain_arrays(path), NAMES, attribute_values()))
    ch = aa.read_chain_arrays(path, 30)
    assert len(list(aa.read_entity_values([d], ch, NAMES, attribute_values()))) == 2

    # a value the attribute's index lacks
    short = attribute_values()
    short[0] = pa.array(VALUES[0][:-1], pa.string())
    d = str(tmp_path / "whole")
    write_chain(d, states, ids)
    ch = aa.read_chain_arrays(os.path.join(d, "linkage-chain.parquet"))
    with pytest.raises(ValueError, match="'fname' has the value 'eve', which its index lacks"):
        list(aa.read_entity_values([d], ch, NAMES, short))

    # a row with one value too many
    f = os.path.join(d, "entity-values-chain.parquet", "partitionId=11", "part-00000.parquet")
    t = pq.read_table(f).to_pydict()
    t["by"][0] = t["by"][0] + ["1950"]
    pq.write_table(pa.table(t, schema=pq.read_schema(f)), f)
    with pytest.raises(ValueError, match="partition 11: the value lists do not have one entry per cluster"):
        list(aa.read_entity_values([d], ch, NAMES, attribute_values()))


def test_config_refusals_and_defaults(tmp_path):
    from dblink_b200 import config
    from dblink_b200.project import Project

    (_, s), _ = project_of(tmp_path, quantities='["entity-values"]').steps()
    assert s["entity_values_center"] == "shared-most-probable-clusters"
    (_, s), _ = project_of(tmp_path, quantities='["entity-values"]',
                           summarize_extra=', entityValuesCenter : "vi-search-clusters"').steps()
    assert s["entity_values_center"] == "vi-search-clusters"
    for bad in ('"credible-ball"', '"sMPC"', "1"):
        with pytest.raises(ValueError, match="^entityValuesCenter must be one of"):
            project_of(tmp_path, summarize_extra=", entityValuesCenter : " + bad).steps()

    def sample_step(extra):
        conf = ('dblink : { data : { path : "x.csv", recordIdentifier : "id", nullValue : "NA", matchingAttributes : '
                '[ {name : "a", similarityFunction : { name : "ConstantSimilarityFn" }, distortionPrior : '
                '{alpha : 0.5, beta : 50.0}} ] }, outputPath : "%s", randomSeed : 1, partitioner : { name : '
                '"KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }, steps : [ {name : '
                '"sample", parameters : { sampleSize : 10 %s }} ] }') % (tmp_path, extra)
        return Project(config.parse_string(conf), base_dir="")

    p = sample_step("")
    assert p.steps()[0][1] == dict(sample_size=10, burnin_interval=0, thinning_interval=1, resume=True, sampler="PCG-I")
    line = p.steps_mk_string().splitlines()[2]
    assert line.endswith("thinningInterval=1 and sampler=PCG-I")
    p = sample_step(", saveEntityValues : false")
    assert "save_entity_values" not in p.steps()[0][1] and p.steps_mk_string().splitlines()[2] == line
    p = sample_step(", saveEntityValues : true")
    assert p.steps()[0][1]["save_entity_values"] is True
    assert p.steps_mk_string().splitlines()[2] == line + ", saving every sample's entity values (saveEntityValues=true)"
    for bad in ('"true"', "1", "0"):
        with pytest.raises(ValueError, match="^saveEntityValues must be a boolean.$"):
            sample_step(", saveEntityValues : " + bad).steps()


# ---- the sampler over a scripted engine --------------------------------------------------------------------------
class ScriptedEngine:
    """Stands in for GibbsEngine: each sweep moves to the next scripted state."""

    def __init__(self, states, A=2, F=1):
        self.states, self.i, self.A, self.F = states, 0, A, F
        self.downloads = 0

    @property
    def iteration(self):
        return self.i

    @property
    def num_entities(self):
        return len(self.states[0][1])

    def sweep(self, sampler, n):
        self.i += n

    def links(self):
        link, blk, _ = self.states[self.i]
        return link, blk

    def download_state(self):
        self.downloads += 1
        link, blk, y = self.states[self.i]
        return {"link": link, "block": blk, "y": y, "z": None, "theta": None}

    def summary(self):
        return {"iteration": self.i, "num_isolates": 0, "log_likelihood": 0.0,
                "agg_dist": np.zeros((self.A, self.F), np.int64), "rec_dist": np.zeros(self.A + 1, np.int64)}


def test_the_sampler_writes_the_entity_values_chain(tmp_path):
    from dblink_b200 import analysis_arrays as aa, sampler

    R, E = 25, 18
    ids = [f"r{i}" for i in range(R)]
    st = engine_states(R, E, 8, seed=4)
    script = [(link, blk, y) for _, link, blk, y in st]
    on, off = str(tmp_path / "on"), str(tmp_path / "off")
    eng = ScriptedEngine(script)
    assert sampler.sample(eng, ids, NAMES, 3, on, burnin_interval=1, thinning_interval=2, write_buffer_size=2,
                          entity_values=VALUES) == 5
    assert eng.downloads == 3
    sampler.sample(ScriptedEngine(script), ids, NAMES, 3, off, burnin_interval=1, thinning_interval=2,
                   write_buffer_size=2)
    assert not os.path.exists(os.path.join(off, "entity-values-chain.parquet"))
    a = aa.read_chain_arrays(os.path.join(on, "linkage-chain.parquet"))
    b = aa.read_chain_arrays(os.path.join(off, "linkage-chain.parquet"))
    assert a.iterations.tolist() == b.iterations.tolist() == [1, 3, 5]
    assert all((x[0] == y[0]).all() and (x[1] == y[1]).all() for x, y in zip(a.samples, b.samples))
    got = list(aa.read_entity_values([on], a, NAMES, attribute_values()))
    want = expected(a, [(it, *script[it]) for it in (1, 3, 5)], ids)
    assert all((g == x).all() for g, x in zip(got, want))


# ---- the summarize quantity on RLdata500 -------------------------------------------------------------------------
CONF = """
dblink : {
  data : { path : "%s", recordIdentifier : "rec_id", entityIdentifier : "ent_id", nullValue : "NA",
           matchingAttributes : [ {name : "fname_c1", similarityFunction : { name : "ConstantSimilarityFn" },
                                   distortionPrior : {alpha : 0.5, beta : 50.0}},
                                  {name : "by", similarityFunction : { name : "ConstantSimilarityFn" },
                                   distortionPrior : {alpha : 0.5, beta : 50.0}} ] }
  outputPath : "%s"
  randomSeed : 1
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [
    {name : "summarize", parameters : { lowerIterationCutoff : 10, quantities : ["entity-values"] %s }}
  ]
}
"""


def rldata500_project(tmp_path, extra=""):
    from dblink_b200 import config
    from dblink_b200.project import Project

    with gzip.open(os.path.join(GOLDEN, "RLdata500.csv.gz"), "rt") as fh:
        rows = list(csv.DictReader(fh))
    with open(os.path.join(tmp_path, "data.csv"), "w") as fh:
        fh.write("rec_id,ent_id,fname_c1,by\n" + "".join(f"{r['rec_id']},{r['ent_id']},{r['fname_c1']},{r['by']}\n"
                                                        for r in rows))
    p = Project(config.parse_string(CONF % (tmp_path / "data.csv", str(tmp_path / "out") + "/", extra)), base_dir="")
    return p, rows


def write_rldata500_values(p, rows, S=10, seed=0):
    """A chain of S samples around RLdata500's truth with entity values drawn near each entity's recorded values."""
    from dblink_b200 import writers as w

    ids = [r["rec_id"] for r in rows]
    _, truth = np.unique([r["ent_id"] for r in rows], return_inverse=True)
    R, E = len(ids), int(truth.max()) + 1
    values = p.attribute_values()
    pos = [{v: i for i, v in enumerate(vals.to_pylist())} for vals in values]
    own = np.zeros((E, 2), np.int32)
    for r, e in zip(rows, truth):
        own[e] = [pos[0][r["fname_c1"]], pos[1][r["by"]]]
    rng = np.random.default_rng(seed)
    d = p.chain_dirs()[0]
    lw = w.LinkageChainWriter(os.path.join(d, "linkage-chain.parquet"), 4)
    ew = w.EntityValuesChainWriter(os.path.join(d, "entity-values-chain.parquet"), ["fname_c1", "by"], 4, False,
                                   lw.file_no)
    for s in range(S):
        link = truth.copy()
        move = rng.random(R) < 0.2
        link[move] = rng.integers(0, E, int(move.sum()))
        y = own.copy()
        noisy = rng.random((E, 2)) < 0.3
        y[noisy] = rng.integers(0, [len(v) for v in values], (E, 2))[noisy]
        blk = np.zeros(E, np.int32)
        lw.append(10 * (s + 1), w.linkage_structure_arrow(link.astype(np.int32), blk, ids))
        ew.append(10 * (s + 1), w.entity_values_arrow(link.astype(np.int32), blk, y, values))
    lw.close()
    ew.close()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("shared_most_probable_clusters", "entity_value_modes", "vi_cross_histograms", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    monkeypatch.setattr(project, "vi_samples", aa.VISamples)


def test_project_writes_the_entity_values_on_rldata500(tmp_path, monkeypatch):
    from dblink_b200 import analysis, analysis_arrays as aa

    host_paths(monkeypatch)
    p, rows = rldata500_project(tmp_path)
    write_rldata500_values(p, rows)
    p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    ch = p.read_chain(10)
    S, R = len(ch.samples), ch.num_records
    assert (S, R) == (10, 500)
    values = [v.to_pylist() for v in p.attribute_values()]
    assert values[1] == sorted(values[1])  # value ids in byte order

    # the literal counts, over sets of record ids and per-sample value dicts read back from the chain
    chain, ids = as_set_chain(ch)
    arrays = list(aa.read_entity_values(p.chain_dirs(), ch, ["fname_c1", "by"], p.attribute_values()))
    dicts = []
    for (mem, off, _), x in zip(ch.samples, arrays):
        dicts.append([{frozenset(ids[i] for i in mem[off[c]:off[c + 1]]): values[a][x[a, mem[off[c]]]]
                       for c in range(len(off) - 1)} for a in range(2)])
    lab = aa.canonical_clusters(aa.shared_most_probable_clusters(ch))
    C = int(lab.max()) + 1
    center = [frozenset(ids[i] for i in np.flatnonzero(lab == k)) for k in range(C)]
    counts = analysis.entity_value_counts(chain, dicts, center)
    # ties in string order are ties in value-id order: value ids are the byte order of the values
    modes = analysis.entity_value_modes(counts, C, 2)

    clusters = open(out + "entity-values-clusters.csv").read().splitlines()
    assert clusters == [", ".join(sorted(c)) for c in center]
    with open(out + "entity-values.csv", newline="") as fh:
        table = list(csv.reader(fh))
    assert table[0] == ["cluster", "size", "fname_c1", "fname_c1Probability", "by", "byProbability"]
    assert len(table) == C + 1
    for k, row in enumerate(table[1:]):
        size = len(center[k])
        assert row[:2] == [str(k), str(size)]
        for a in range(2):
            v, n = modes[(k, a)]
            assert row[2 + 2 * a] == v and row[3 + 2 * a] == repr(n / (size * S))
    run = p.steps_mk_string().splitlines()
    assert ("  * SummarizeStep: entity-values is the most probable value of each attribute of the entity of each "
            "cluster of a point estimate, from the entity values saved with the samples, with "
            "entityValuesCenter=shared-most-probable-clusters") in run


def test_run_txt_names_the_settings_of_the_center(tmp_path):
    p, _ = rldata500_project(tmp_path, ', entityValuesCenter : "binder-search-clusters", falseLinkCost : 0.25, '
                                       'maxSearchRounds : 9')
    (line,) = [x for x in p.steps_mk_string().splitlines() if "entity-values is" in x]
    assert line.endswith("entityValuesCenter=binder-search-clusters, falseLinkCost=0.25, maxSearchRounds=9")


def test_values_with_commas_and_quotes_are_quoted(tmp_path):
    from dblink_b200 import analysis_arrays as aa, writers as w

    lab = np.array([0, 0, 1])
    modes, counts = np.array([[2, 3], [0, 1]], np.int32), np.array([[3, 1], [4, 2]], np.int64)
    rows = aa.entity_value_rows(lab, modes, counts, 2, VALUES)
    assert rows == [[0, 2, "carl, jr", repr(3 / 4), "1950", repr(4 / 4)], [1, 1, 'dee "d"', repr(1 / 2), "1961", "1.0"]]
    w.save_entity_values(NAMES, rows, str(tmp_path))
    assert open(tmp_path / "entity-values.csv").read() == (
        "cluster,size,fname,fnameProbability,by,byProbability\n"
        '0,2,"carl, jr",0.75,1950,1.0\n'
        '1,1,"dee ""d""",0.5,1961,1.0\n')


def test_no_sample_is_refused():
    from dblink_b200 import analysis_arrays as aa

    with pytest.raises(ValueError, match="at least one sample at or after lowerIterationCutoff"):
        aa.entity_value_modes(np.zeros(3, np.int64), iter([]), [2])


def test_abi_refuses_a_null_handle():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import EntityValues

    L = _lib.load()
    values = np.zeros(4, np.int32)
    mode, count = np.full(2, 7, np.int32), np.full(2, 7, np.int64)
    assert L.dbl_values_add_sample(None, values.ctypes.data) == _lib.ERR_INVALID
    assert L.dbl_values_modes(None, mode.ctypes.data, count.ctypes.data) == _lib.ERR_INVALID
    assert L.dbl_values_create(None, 4, values.ctypes.data, 2, 2) == _lib.ERR_INVALID
    assert L.dbl_values_num_samples(None) == 0
    assert (mode == 7).all() and (count == 7).all()
    v = EntityValues.__new__(EntityValues)  # an owner without a handle: the shape check comes first
    v.num_records = 4
    with pytest.raises(ValueError, match="one value per record"):
        v.add_sample(np.zeros(5, np.int32))


def test_synthetic_data_gives_the_true_entity_values():
    """generate_encoded's ent_values take no random draw: every other key is what the same seed gave without them
    (the digest was taken before they existed), and a record that is neither distorted nor missing carries its
    entity's true value."""
    import hashlib

    from dblink_b200 import synth

    e = synth.generate_encoded(5, 3000, synth.config_attrs(4), n_files=2)
    digest = hashlib.sha256(e["codes"].tobytes() + e["files"].tobytes() + e["ent_ids"].tobytes()
                            + repr(e["vocabs"]).encode()).hexdigest()
    assert digest == "39ca1b51faf6c049181571965a04b28f108f713cb3efa8bd96c8f1d8139b62b9"
    true = e["ent_values"][e["ent_ids"]]
    assert e["ent_values"].shape == (int(e["ent_ids"].max()) + 1, 10) and e["ent_values"].dtype == np.int32
    present = e["codes"] >= 0
    agree = (e["codes"] == true)[present].mean()
    assert 0.9 < agree < 1.0  # distortion 0.05 per attribute; a distorted draw may land on the true value
    for a, vocab in enumerate(e["vocabs"]):
        assert 0 <= e["ent_values"][:, a].min() and e["ent_values"][:, a].max() < len(vocab)


def test_a_new_chain_without_values_removes_the_old_values(tmp_path):
    from dblink_b200 import sampler

    R, E = 25, 18
    ids = [f"r{i}" for i in range(R)]
    script = [(link, blk, y) for _, link, blk, y in engine_states(R, E, 4, seed=5)]
    d = str(tmp_path)
    sampler.sample(ScriptedEngine(script), ids, NAMES, 2, d, entity_values=VALUES)
    assert os.path.isdir(os.path.join(d, "entity-values-chain.parquet"))
    sampler.sample(ScriptedEngine(script), ids, NAMES, 2, d)
    assert not os.path.exists(os.path.join(d, "entity-values-chain.parquet"))


def test_values_of_another_chain_are_refused(tmp_path):
    import shutil

    from dblink_b200 import analysis_arrays as aa

    R, E = 30, 20
    ids = [f"r{i}" for i in range(R)]
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    write_chain(a, engine_states(R, E, 2, seed=6), ids)
    write_chain(b, engine_states(R, E, 2, seed=7, blocks=5), ids)  # same iterations and file names, other partitions
    shutil.rmtree(os.path.join(a, "entity-values-chain.parquet"))
    shutil.copytree(os.path.join(b, "entity-values-chain.parquet"), os.path.join(a, "entity-values-chain.parquet"))
    ch = aa.read_chain_arrays(os.path.join(a, "linkage-chain.parquet"))
    with pytest.raises(ValueError, match="the partitions do not match those of linkage-chain.parquet"):
        list(aa.read_entity_values([a], ch, NAMES, attribute_values()))
