"""JaroWinklerSimilarityFn on the GPU: the all-pairs index build (k_jw_tiles) against the host loop, models with
Jaro-Winkler attributes swept against the oracle (given the rows of jw_reference.py), and a Project run on
RLdata10000."""
import collections
import os

import numpy as np
import pytest

import jw_reference as ref
from helpers import product_setup, synth_problem
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu

JW = "JaroWinklerSimilarityFn"


def test_gpu_index_build_equals_host(monkeypatch):
    import dblink_b200 as D
    from dblink_b200 import synth

    rng = np.random.default_rng(3)
    strings, _ = synth._string_vocab(rng, 1600)
    strings += ["", "A", "AB", "BB", "John Smith", "Jane Smith", "Zoë", "Zoe", "José", "Jose", "x" * 64,
                "x" * 63 + "y", "ab" * 32, "ba" * 32, "a" * 33 + "b" * 31, "MARTHA", "MARHTA", "DWAYNE", "DUANE",
                "aaaaab", "baaaaa", "张伟", "张伟a"]
    vw = {s: float(1 + (i * 7919) % 13) for i, s in enumerate(dict.fromkeys(strings))}
    nnz = []
    for thr in (8.5, 7.0, 0.0):
        monkeypatch.setenv("DBL_INDEX_GPU", "0")
        host = D.AttributeIndex.build(vw, "jaro-winkler", thr, 10.0).tables()
        monkeypatch.setenv("DBL_INDEX_GPU", "1")
        dev = D.AttributeIndex.build(vw, "jaro-winkler", thr, 10.0).tables()
        for k in ("phi", "norm", "rowptr", "col", "expsim"):
            np.testing.assert_array_equal(host[k], dev[k], err_msg=f"{k} at threshold {thr}")
        nnz.append(len(host["col"]))
    assert nnz[0] < nnz[1] < nnz[2]
    # a string longer than 64 bytes: the device path declines, the host loop builds the same index
    vw2 = dict(list(vw.items())[:50])
    vw2["q" * 80] = 2.0
    vw2["q" * 79 + "r"] = 1.0
    tabs = []
    for flag in ("1", "0"):
        monkeypatch.setenv("DBL_INDEX_GPU", flag)
        tabs.append(D.AttributeIndex.build(vw2, "jaro-winkler", 7.0, 10.0).tables())
    for k in ("phi", "norm", "rowptr", "col", "expsim"):
        np.testing.assert_array_equal(tabs[0][k], tabs[1][k], err_msg=k)


def jw_problem():
    g = synth_problem(seed=6, R=700, n_files=2)
    from dblink_b200.records import SimilarityFn

    g["attributes"][2].similarity_fn = SimilarityFn(JW, 8.5, 10.0)
    g["attributes"][3].similarity_fn = SimilarityFn(JW, 7.0, 10.0)
    return g


def oracle_jw_setup(O, g, seed, levels, attr_ids):
    """helpers.oracle_setup with the Jaro-Winkler attributes' rows from the literal restatement (jw_reference)"""
    idx, ids = [], []
    for a, attr in enumerate(g["attributes"]):
        cnt = collections.Counter(v[a] for v in g["values"] if v[a] is not None)
        vw = {k: float(c) for k, c in cnt.items()}
        sf = attr.similarity_fn
        if sf.name == JW:
            ix, vid = ref.oracle_index(O, vw, sf.threshold, sf.max_similarity)
        else:
            ix = O.Index.build(vw, sf.is_constant, sf.threshold, sf.max_similarity, 10)
            vid = {k: ix.value_id(k) for k in vw}
        idx.append(ix)
        ids.append(vid)
    x = np.array([[-1 if v is None else ids[a][v] for a, v in enumerate(rec)] for rec in g["values"]], np.int32)
    fids = sorted(set(g["files"]))
    file = np.array([fids.index(f) for f in g["files"]], np.int32)
    F = len(fids)
    alpha = [a.alpha for a in g["attributes"]]
    beta = [a.beta for a in g["attributes"]]
    m0 = O.Model(idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    tree = O.KDTree.fit(s0.y, levels, list(attr_ids))
    m = O.Model(idx, alpha, beta, tree, seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0, tree, idx)
    return st


@pytest.mark.parametrize("sampler", ["PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential"])
def test_jaro_winkler_model_sweeps_equal_oracle(oracle, sampler):
    g = jw_problem()
    eng, rc, x, file = product_setup(g, 21, 1, (2,))
    st = oracle_jw_setup(oracle, g, 21, 1, (2,))
    np.testing.assert_array_equal(x, st.x)
    assert eng.link_kernel("PCG-II") == "k_link_pcg2<A=4,NS=2,HC=32,PK=1>", (eng.link_kernel(), eng.link_tile_format())
    for _ in range(3):
        eng.sweep(sampler, 1)
        st.sweep(oracle.SAMPLERS[sampler])
        d = eng.download_state()
        for k in ("link", "y", "z", "theta"):
            np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=f"{k} after a {sampler} sweep")
    eng.close()


def jw_conf(data, out, sample_size, thinning, sampler, quantities):
    conf = make_conf(data, out, 2, '["fname_c1", "lname_c1"]', sample_size=sample_size, thinning=thinning,
                     sampler=sampler, cutoff=0)
    conf = conf.replace("lowDistortion : {alpha : 0.5, beta : 50.0}", "lowDistortion : {alpha : 10.0, beta : 1000.0}")
    conf = conf.replace('quantities : ["cluster-size-distribution", "partition-sizes"]', f"quantities : {quantities}")
    return conf.replace('name : "LevenshteinSimilarityFn",', f'name : "{JW}",').replace("threshold : 7.0",
                                                                                       "threshold : 8.5")


def test_rldata10000_project_with_jaro_winkler_names(tmp_path):
    from dblink_b200 import config
    from dblink_b200.project import Project

    out = str(tmp_path) + "/"
    conf = jw_conf(os.path.join(GOLDEN, "RLdata10000.csv.gz"), out, 20, 10, "PCG-II",
                   '["shared-most-probable-clusters"]')
    proj = Project(config.parse_string(conf), base_dir="")
    assert [a.similarity_fn.name for a in proj.matching_attributes][3:] == [JW, JW]
    proj.write_run_txt()
    res = proj.execute(log=lambda *a: None)
    for f in ("run.txt", "linkage-chain.parquet", "diagnostics.csv", "shared-most-probable-clusters.csv",
              "evaluation-results.txt", "state.npz"):
        assert os.path.exists(os.path.join(out, f)), f
    assert "JaroWinklerSimilarityFn(threshold=8.5, maxSimilarity=10.0)" in open(out + "run.txt").read()
    assert len(open(out + "diagnostics.csv").read().splitlines()) == 1 + 21
    pw = res["pairwise"]
    assert 0.0 <= pw["precision"] <= 1.0 and 0.0 <= pw["recall"] <= 1.0, pw
    clusters = open(out + "shared-most-probable-clusters.csv").read().splitlines()
    assert sum(len(c.split(",")) for c in clusters) == 10000


def test_state_saved_under_levenshtein_is_refused(tmp_path):
    """the fingerprint covers the tables: switching the names to Jaro-Winkler refuses the saved Levenshtein state"""
    from dblink_b200 import config
    from dblink_b200.project import Project

    data, out = os.path.join(GOLDEN, "RLdata500.csv.gz"), str(tmp_path) + "/"
    lev = make_conf(data, out, 0, "[]", sample_size=2, thinning=1, cutoff=0)
    Project(config.parse_string(lev), base_dir="").execute(log=lambda *a: None)
    jw = lev.replace('name : "LevenshteinSimilarityFn",', f'name : "{JW}",').replace("resume : false",
                                                                                    "resume : true")
    with pytest.raises(ValueError, match="saved state does not match"):
        Project(config.parse_string(jw), base_dir="").execute(log=lambda *a: None)
    # the same configuration resumes
    Project(config.parse_string(lev.replace("resume : false", "resume : true")), base_dir="").execute(
        log=lambda *a: None)
