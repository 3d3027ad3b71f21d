"""JaroWinklerSimilarityFn on the host (no GPU): the unit similarity and its truncation through the library against a
literal Python restatement (jw_reference.py); the symmetry of the counts the GPU index build relies on; host-built
index tables against the oracle's tables of the restated rows; configuration parsing, run.txt and the rejection of bad
parameters and unknown kinds."""
import ctypes as C
import itertools
import math
import os

import numpy as np
import pytest

import jw_reference as ref
from test_host_pipeline import GOLDEN, make_conf

JW = "JaroWinklerSimilarityFn"

# (a, b, (m, h, l), unit at threshold 0 / maxSimilarity 1); the first three are Winkler's 0.961 / 0.840 / 0.813
GOLDEN_PAIRS = [
    ("MARTHA", "MARHTA", (6, 2, 3), 0.9611111111111111),
    ("DWAYNE", "DUANE", (4, 0, 1), 0.8400000000000001),
    ("DIXON", "DICKSONX", (4, 0, 2), 0.8133333333333332),
    ("JELLYFISH", "SMELLYFISH", (8, 0, 0), 0.8962962962962964),
    ("ABC", "XYZ", (0, 0, 0), 0.0),
]


def vocabulary():
    from dblink_b200 import synth

    strings, _ = synth._string_vocab(np.random.default_rng(11), 360)
    strings += ["", "A", "B", "AB", "BA", "AA", "MARTHA", "MARHTA", "DWAYNE", "DUANE", "DIXON", "DICKSONX",
                "x" * 64, "x" * 63 + "y", "ab" * 32, "ba" * 32, "a" * 33 + "b" * 31, "aaaaab", "baaaaa",
                "Zoë", "Zoe", "José", "Jose", "Müller", "Mueller", "张伟", "张伟a"]
    return list(dict.fromkeys(strings))


def test_golden_pairs():
    import dblink_b200 as D

    for a, b, counts, unit in GOLDEN_PAIRS:
        assert ref.counts(a.encode(), b.encode()) == counts
        assert ref.counts(b.encode(), a.encode()) == counts
        assert ref.unit(a, b) == unit
        assert ref.similarity(a, b, 0.0, 1.0) == unit
        assert D.similarity(a, b, JW, 0.0, 1.0) == unit
        assert D.similarity(b, a, JW, 0.0, 1.0) == unit
    # the shipped Levenshtein transform sends DWAYNE / DUANE to zero; Jaro-Winkler 7/10 keeps it
    assert D.similarity("DWAYNE", "DUANE", "LevenshteinSimilarityFn", 7.0, 10.0) == 0.0
    assert D.similarity("DWAYNE", "DUANE", JW, 7.0, 10.0) > 0.0


def test_library_equals_literal():
    import dblink_b200 as D

    vocab = vocabulary()
    rng = np.random.default_rng(5)
    pairs = [(vocab[i], vocab[j]) for i, j in rng.integers(0, len(vocab), (3000, 2))]
    edge = ["", "A", "x" * 64, "ab" * 32, "aaaaab", "Zoë", "张伟"]
    pairs += list(itertools.product(edge, edge))
    for thr, ms in ((8.5, 10.0), (7.0, 10.0), (0.0, 10.0), (0.0, 1.0)):
        for a, b in pairs:
            want = ref.similarity(a, b, thr, ms)
            assert D.similarity(a, b, JW, thr, ms) == want, (a, b, thr)
    assert D.similarity("", "", JW, 7.0, 10.0) == 10.0
    assert D.similarity("", "A", JW, 0.0, 10.0) == 0.0


def test_counts_are_symmetric():
    """(m, h) of (a, b) equal those of (b, a): the GPU build scans the other string of each pair and mirrors it, and the
    library's similarity is symmetric"""
    import dblink_b200 as D

    rng = np.random.default_rng(8)
    for alphabet in ("ab", "abc", "abcd"):
        for _ in range(4000):
            a = "".join(rng.choice(list(alphabet), rng.integers(0, 15)))
            b = "".join(rng.choice(list(alphabet), rng.integers(0, 15)))
            ab, ba = ref.counts(a.encode(), b.encode()), ref.counts(b.encode(), a.encode())
            assert ab == ba, (a, b)
            assert D.similarity(a, b, JW, 0.0, 10.0) == D.similarity(b, a, JW, 0.0, 10.0)
    words = [b""] + [bytes(p) for n in range(1, 6) for p in itertools.product(b"abc", repeat=n)]
    for a, b in itertools.combinations(words, 2):
        assert ref.counts(a, b)[:2] == ref.counts(b, a)[:2], (a, b)


@pytest.mark.parametrize("threshold", [8.5, 7.0, 0.0])
def test_host_index_equals_oracle(oracle, monkeypatch, threshold):
    import dblink_b200 as D

    monkeypatch.setenv("DBL_INDEX_GPU", "0")
    vw = {s: float(1 + (i * 7919) % 13) for i, s in enumerate(vocabulary())}
    got = D.AttributeIndex.build(vw, "jaro-winkler", threshold, 10.0).tables()
    want, ids = ref.oracle_index(oracle, vw, threshold, 10.0)
    for k in ("phi", "norm", "rowptr", "col", "expsim"):
        np.testing.assert_array_equal(got[k], getattr(want, k), err_msg=k)
    ix = D.AttributeIndex.build(vw, "jaro-winkler", threshold, 10.0)
    assert all(ix.value_idx_of(v) == i for v, i in ids.items())
    lev = D.AttributeIndex.build(vw, "levenshtein", threshold, 10.0).tables()
    assert not np.array_equal(lev["rowptr"], got["rowptr"])  # a different function gives different rows
    # every stored pair is the library's own similarity of the two values
    for v in (0, 5, len(vw) - 1):
        for c, e in ix.sim_values_of(v).items():
            assert e == math.exp(D.similarity(ix.value_of(v), ix.value_of(c), JW, threshold, 10.0))


def test_records_cache_builds_jaro_winkler_indexes(oracle, monkeypatch):
    """RecordsCache.build and the columnar build pass the attribute's similarity function to the index build"""
    import pyarrow as pa

    import dblink_b200 as D
    from dblink_b200 import records
    from helpers import synth_problem

    monkeypatch.setenv("DBL_INDEX_GPU", "0")
    g = synth_problem(seed=3, R=500)
    for a in g["attributes"][2:]:
        a.similarity_fn = D.SimilarityFn(JW, 8.5, 10.0)
    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    cols = [pa.array([v[a] for v in g["values"]], pa.string()) for a in range(len(g["attributes"]))]
    rc2, _, _ = records.build_cache_from_columns(cols, pa.array(g["files"], pa.string()), g["attributes"])
    for a in (2, 3):
        vw = {}
        for v in g["values"]:
            if v[a] is not None:
                vw[v[a]] = vw.get(v[a], 0.0) + 1.0
        want, _ = ref.oracle_index(oracle, vw, 8.5, 10.0)
        for t in (rc.indexes[a].tables(), rc2.indexes[a].tables()):
            for k in ("phi", "norm", "rowptr", "col", "expsim"):
                np.testing.assert_array_equal(t[k], getattr(want, k), err_msg=k)


def jw_conf(out="out/", threshold="8.5", max_sim="10.0"):
    conf = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out)
    return conf.replace('name : "LevenshteinSimilarityFn",', f'name : "{JW}",').replace(
        "threshold : 7.0", f"threshold : {threshold}").replace("maxSimilarity : 10.0", f"maxSimilarity : {max_sim}")


def test_config_and_run_txt(tmp_path):
    from dblink_b200 import config
    from dblink_b200.project import Project

    proj = Project(config.parse_string(jw_conf(str(tmp_path) + "/")), base_dir="")
    fns = [a.similarity_fn for a in proj.matching_attributes]
    assert [f.name for f in fns] == ["ConstantSimilarityFn"] * 3 + [JW] * 2
    assert (fns[3].threshold, fns[3].max_similarity) == (8.5, 10.0)
    assert fns[3].index_kind == "jaro-winkler"
    proj.write_run_txt()
    txt = open(os.path.join(str(tmp_path), "run.txt")).read()
    assert ("  * 'fname_c1' (id=3) with JaroWinklerSimilarityFn(threshold=8.5, maxSimilarity=10.0) and "
            "BetaShapeParameters(alpha=0.5, beta=50.0)\n") in txt


def test_bad_parameters_are_rejected():
    import dblink_b200 as D
    from dblink_b200 import config
    from dblink_b200.project import Project

    for thr, ms in ((10.0, 10.0), (-1.0, 10.0), (1.0, 0.0), (12.0, 10.0)):
        with pytest.raises(ValueError):
            D.SimilarityFn(JW, thr, ms)
        with pytest.raises(ValueError):
            D.similarity("a", "b", JW, thr, ms)
        with pytest.raises(ValueError):
            D.AttributeIndex.build({"a": 1.0, "b": 1.0}, "jaro-winkler", thr, ms)
    with pytest.raises(ValueError):
        Project(config.parse_string(jw_conf(threshold="10.0")), base_dir="")
    with pytest.raises(ValueError):
        D.SimilarityFn("JaroSimilarityFn", 7.0, 10.0)
    with pytest.raises(ValueError):
        D.similarity("a", "b", "JaroSimilarityFn")
    with pytest.raises(ValueError):
        D.AttributeIndex.build({"a": 1.0, "b": 1.0}, "jaro")
    with pytest.raises(config.ConfigError):
        Project(config.parse_string(jw_conf().replace(JW, "SoundexSimilarityFn")), base_dir="")


def test_unknown_similarity_kind_through_the_abi():
    """similarity values other than 0, 1, 2 are DBL_ERR_INVALID (NaN from dbl_similarity)"""
    from dblink_b200 import _lib

    L = _lib.load()
    arr = (C.c_char_p * 2)(b"a", b"b")
    w = np.ones(2)
    probs = np.full(2, 0.5)
    rowptr, col, es = np.array([0, 1, 2], np.int32), np.array([0, 1], np.int32), np.ones(2)
    for sim in (3, -1):
        h = C.c_void_p()
        assert L.dbl_index_build(C.byref(h), arr, w.ctypes.data_as(_lib.f64p), 2, sim, 7.0, 10.0, 10) == \
            _lib.ERR_INVALID
        assert np.isnan(L.dbl_similarity(sim, b"a", b"b", 7.0, 10.0))
        assert L.dbl_index_from_tables(C.byref(h), 2, sim, probs.ctypes.data_as(_lib.f64p),
                                       rowptr.ctypes.data_as(_lib.i32p), col.ctypes.data_as(_lib.i32p),
                                       es.ctypes.data_as(_lib.f64p), 10) == _lib.ERR_INVALID
    for sim in (0, 1, 2):
        h = C.c_void_p()
        assert L.dbl_index_build(C.byref(h), arr, w.ctypes.data_as(_lib.f64p), 2, sim, 7.0, 10.0, 10) == _lib.OK
        L.dbl_index_free(h)
