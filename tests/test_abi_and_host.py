"""CPU-only: the C-ABI library loads and exports every symbol include/dblink_b200.h declares; the host-side
pieces of the product (attribute index, similarity, k-d tree, RecordsCache, synthetic generator) agree with the
reference's golden vectors and with the oracle.  No GPU compute is called here."""
import collections
import ctypes as C
import os
import re

import numpy as np
import pytest

from helpers import oracle_indexes, synth_problem
from test_oracle_golden import STATE_SIM_NORMS, STATE_WEIGHTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "dblink_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(dbl_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_declared_abi():
    from dblink_b200 import _lib

    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 30
    for s in syms:
        assert hasattr(lib, s), f"{s} is declared in include/dblink_b200.h but not exported"
    assert set(_lib.SIGNATURES) == set(syms), "python binding and header disagree"
    assert b"sm_90a" in lib.dbl_version()


def test_sm90a_code_in_library():
    import subprocess

    from dblink_b200 import _lib

    out = subprocess.run(["cuobjdump", "--list-elf", _lib.SO_PATH], capture_output=True, text=True)
    if out.returncode != 0:
        pytest.skip("cuobjdump unavailable")
    assert "sm_90a" in out.stdout


def test_no_cpu_fallback_without_gpu():
    """without a CUDA device the context constructor fails loudly (DBL_ERR_CUDA); it never computes on the CPU"""
    import torch

    import dblink_b200 as D

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    ix = D.AttributeIndex.build({"a": 1.0, "b": 1.0})
    with pytest.raises(D.DblinkError):
        D.GibbsEngine([ix], [1.0], [1.0])


def test_product_does_not_import_oracle():
    """the product never imports, includes, links or calls anything under oracle/ (comments may mention it)"""
    pkg = os.path.join(ROOT, "dblink_b200")
    bad = re.compile(r"(^\s*(from|import)\s+oracle\b)|(#include\s+\"dbl_oracle)|(\borc_[a-z_0-9]+\s*\()|(liboracle)", re.M)
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".cuh")):
                src = open(os.path.join(dp, f)).read()
                assert not bad.search(src), f"{f} uses the oracle"


def test_similarity_golden_through_abi():
    """SimilarityFnTest.scala:25-75 through dbl_similarity"""
    import dblink_b200 as D

    assert D.similarity("TestValue", "TestValue", "ConstantSimilarityFn") == 0.0
    assert D.similarity("TestValue1", "TestValue2", "ConstantSimilarityFn") == 0.0
    s = lambda a, b, t=5.0: D.similarity(a, b, "LevenshteinSimilarityFn", t, 10.0)  # noqa: E731
    assert s("John Smith", "John Smith") == 10.0
    assert s("", "") == 10.0
    assert s("", "John Smith") == 0.0
    assert s("Jane Smith", "John Smith") == s("John Smith", "Jane Smith")
    assert s("AB", "BB") == 2.0
    assert s("AB", "BB", 0.0) == 6.0
    with pytest.raises(ValueError):
        D.similarity("a", "b", "LevenshteinSimilarityFn", 10.0, 10.0)  # threshold must be < maxSimilarity
    with pytest.raises(ValueError):
        D.similarity("a", "b", "LevenshteinSimilarityFn", 1.0, 0.0)


def test_attribute_index_golden_through_abi():
    """AttributeIndexTest.scala:38-99 + AttributeIndexBehaviors.scala through dbl_index_build"""
    import dblink_b200 as D

    const = D.AttributeIndex.build(STATE_WEIGHTS, "constant")
    lev = D.AttributeIndex.build(STATE_WEIGHTS, "levenshtein", 5.0, 10.0)
    total = sum(STATE_WEIGHTS.values())
    for ix in (const, lev):
        assert ix.num_values == 8
        assert {ix.value_idx_of(k) for k in STATE_WEIGHTS} == set(range(8))
        for k, w in STATE_WEIGHTS.items():
            assert ix.probability_of(ix.value_idx_of(k)) == pytest.approx(w / total, abs=1e-4)
        for fn in (ix.probability_of, ix.sim_normalization_of, ix.sim_values_of):
            with pytest.raises(IndexError):
                fn(ix.num_values + 1)
        with pytest.raises(IndexError):
            ix.exp_sim_of(ix.num_values + 1, 0)
        with pytest.raises(IndexError):
            ix.exp_sim_of(0, ix.num_values + 1)
    assert all(const.sim_normalization_of(v) == 1.0 for v in range(8))
    assert all(const.sim_values_of(v) == {} for v in range(8))
    assert all(const.exp_sim_of(i, j) == 1.0 for i in range(8) for j in range(8))
    for k, n in STATE_SIM_NORMS.items():
        assert lev.sim_normalization_of(lev.value_idx_of(k)) == pytest.approx(n, rel=1e-13)
    sa, wa = lev.value_idx_of("South Australia"), lev.value_idx_of("Western Australia")
    sv = lev.sim_values_of(sa)
    assert set(sv) == {7, 4}
    assert sv[7] == pytest.approx(39.813678188084864, rel=1e-13)
    assert sv[4] == pytest.approx(22026.465794806718, rel=1e-13)
    assert lev.exp_sim_of(sa, wa) == pytest.approx(39.813678188084864, rel=1e-13)
    assert lev.exp_sim_of(lev.value_idx_of("Victoria"), lev.value_idx_of("Tasmania")) == 1.0
    with pytest.raises(ValueError):
        D.AttributeIndex.build({})


def test_records_cache_and_index_match_oracle(oracle):
    import dblink_b200 as D

    g = synth_problem(seed=13, R=1500, n_files=2)
    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    oi = oracle_indexes(oracle, g)
    for a in range(rc.num_attributes):
        t = rc.indexes[a].tables()
        for k in ("phi", "norm", "rowptr", "col", "expsim", "invnorm", "pk", "cdf"):
            np.testing.assert_array_equal(t[k], getattr(oi[a], k))
        np.testing.assert_allclose(t["logphi"], np.log(oi[a].phi), rtol=1e-15, atol=1e-300)
        np.testing.assert_allclose(t["lognorm"], np.log(oi[a].norm), rtol=1e-15, atol=1e-300)
    x, file = rc.transform_records(g["values"], g["files"])
    assert x.shape == (1500, 4) and set(np.unique(file)) == {0, 1}
    assert rc.num_records == 1500 and sum(rc.file_sizes) == 1500
    miss = collections.Counter()
    for rec, f in zip(g["values"], g["files"]):
        for a, v in enumerate(rec):
            if v is None:
                miss[(f, a)] += 1
    assert rc.missing_counts == dict(miss)
    assert ((x < 0) == np.array([[v is None for v in rec] for rec in g["values"]])).all()
    with pytest.raises(ValueError):
        D.RecordsCache.build(g["values"], g["files"], g["attributes"][:2])
    with pytest.raises(ValueError):
        D.Attribute("bad", D.SimilarityFn(), alpha=0.0, beta=1.0)


@pytest.mark.parametrize("levels,attr_ids", [(0, []), (1, [0]), (3, [2, 3]), (4, [1, 2, 3, 0])])
def test_kdtree_matches_oracle(oracle, levels, attr_ids):
    import dblink_b200 as D

    rng = np.random.default_rng(levels)
    # attribute 0: 12 values (set splitter), 1: 25, 2: 200 (range splitter), 3: 400, Zipf-ish
    y = np.stack([rng.integers(0, 12, 4000), rng.integers(0, 25, 4000), (rng.pareto(1.0, 4000) * 10).astype(int) % 200,
                  rng.integers(0, 400, 4000)], axis=1).astype(np.int32)
    part = D.KDTreePartitioner(levels, attr_ids).fit(y)
    ot = oracle.KDTree.fit(y, levels, attr_ids)
    e = part.export()
    for k in ("attr", "kind", "split", "set_ptr", "set_val", "leaf_no"):
        np.testing.assert_array_equal(e[k], getattr(ot, k))
    assert part.num_partitions == ot.n_leaves == (1 << levels)
    ids = np.array([part.get_partition_id(r) for r in y[:500]])
    assert (ids == np.array([ot.leaf(r) for r in y[:500]])).all()
    if levels:
        sizes = np.bincount(np.array([part.get_partition_id(r) for r in y]), minlength=1 << levels)
        assert sizes.min() > 0.3 * sizes.mean()  # roughly balanced (KDTreePartitioner.scala:56-57 warns below 0.9)
    with pytest.raises(ValueError):
        D.KDTreePartitioner(-1, [])
    with pytest.raises(ValueError):
        D.KDTreePartitioner(2, [])


def test_kdtree_roundtrip_arrays():
    import dblink_b200 as D

    rng = np.random.default_rng(1)
    y = rng.integers(0, 50, (1000, 3)).astype(np.int32)
    p = D.KDTreePartitioner(3, [0, 1, 2]).fit(y)
    e = p.export()
    q = D.KDTreePartitioner.from_arrays(e["attr"], e["kind"], e["split"], e["set_ptr"], e["set_val"], e["leaf_no"])
    assert q.num_partitions == p.num_partitions
    assert all(p.get_partition_id(r) == q.get_partition_id(r) for r in y[:200])


def test_synth_is_deterministic_and_shaped():
    from dblink_b200 import synth

    a = synth.generate_encoded(5, 5000, synth.config_attrs(4), n_files=2)
    b = synth.generate_encoded(5, 5000, synth.config_attrs(4), n_files=2)
    np.testing.assert_array_equal(a["codes"], b["codes"])
    assert a["codes"].shape == (5000, 10)
    assert 0.003 < (a["codes"] < 0).mean() < 0.02
    n_ent = len(np.unique(a["ent_ids"]))
    assert 0.85 * 5000 <= n_ent <= 0.91 * 5000
    idx, x, f, F = synth.build_encoded(a)
    assert F == 2 and x.shape == (5000, 10) and [ix.is_constant for ix in idx] == [True] * 4 + [False] * 6
    g = synth.generate(5, 300, synth.config_attrs(3))
    assert len(g["values"]) == 300 and len(g["values"][0]) == 8


def test_every_entry_point_is_documented():
    """INTEGRATION.md maps every function the header declares to what it replaces in the reference."""
    import re

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "dblink_b200.h")).read()
    doc = open(os.path.join(root, "INTEGRATION.md")).read()
    fns = sorted(set(re.findall(r"\b(dbl_[a-z_0-9]+)\s*\(", header)))
    assert len(fns) >= 50
    assert [f for f in fns if f not in doc] == []


def test_theta_draw_of_the_product_equals_the_oracle_bit_for_bit(oracle):
    """updateDistProbs through the product's C ABI (host build of the function the device runs) against the oracle's
    own restatement: protocol log / exp and the whole Beta draw, shapes below and above 1"""
    import ctypes as C

    from dblink_b200 import _lib

    L, OL = _lib.load(), oracle.lib()
    rng = np.random.default_rng(5)
    for x in np.r_[rng.uniform(0, 1, 3000), 10.0 ** rng.uniform(-320, 300, 3000)]:
        assert L.dbl_det_log(float(x)) == OL.orc_det_log(float(x))
    for x in rng.uniform(-760, 720, 6000):
        assert L.dbl_det_exp(float(x)) == OL.orc_det_exp(float(x))
    ix = oracle.Index.build({"a": 1.0, "b": 2.0}, True)
    alpha, beta = np.array([0.5, 0.5, 10.0, 3.0]), np.array([50.0, 2.0, 1000.0, 1.0])
    m = oracle.Model([ix] * 4, alpha.tolist(), beta.tolist(), None, 0xC0FFEE12345, F=3)
    fs = np.array([200, 3000, 1], np.int64)
    for it in range(1, 400):
        agg = np.minimum(rng.integers(0, 50, (4, 3)), fs[None, :]).astype(np.int64)
        if it % 3 == 0:
            agg[:2] = 0  # shape < 1
        ref = oracle.draw_theta(m, agg, fs, it)
        out = np.zeros((4, 3))
        rc = L.dbl_draw_theta(4, 3, alpha.ctypes.data_as(_lib.f64p), beta.ctypes.data_as(_lib.f64p), 0xC0FFEE12345,
                              agg.ctypes.data_as(_lib.i64p), fs.ctypes.data_as(_lib.i64p), it,
                              out.ctypes.data_as(_lib.f64p))
        assert rc == 0
        np.testing.assert_array_equal(out, ref)

