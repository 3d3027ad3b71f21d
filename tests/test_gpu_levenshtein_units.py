"""LevenshteinSimilarityFn on non-ASCII values on the GPU.

The device kernel k_lev_tiles indexes its match masks by byte; the index build hands it one byte symbol per UTF-16
code unit (the identity below 256, otherwise a dense table of at most 256 distinct units) and the lengths in code
units.  Every case here equals lev_reference.index_rows bit for bit, and asserts which path built the pairs
(AttributeIndex.pairs_on_device), so a device path that quietly declines cannot pass.  Then models whose string
attributes hold accented, CJK, supplementary-plane and long values are swept against the oracle."""
import zlib

import numpy as np
import pytest

import lev_reference as ref
from helpers import (assert_literal_mass, assert_same_mass, literal_link_mass, oracle_setup, product_setup,
                     synth_problem)
from test_gpu_parity import assert_same_state
from test_levenshtein_units import LATIN, MIXED, weights

pytestmark = pytest.mark.gpu

TABLE_KEYS = ("phi", "norm", "rowptr", "col", "expsim")


def build(monkeypatch, vw, threshold, flag):
    import dblink_b200 as D

    monkeypatch.setenv("DBL_INDEX_GPU", flag)
    return D.AttributeIndex.build(vw, "levenshtein", threshold, 10.0)


def assert_literal_rows(ix, vw, threshold, what):
    vals, _, rowptr, col, expsim = ref.index_rows(vw, threshold, 10.0)
    got = ix.tables()
    for k, want in (("rowptr", rowptr), ("col", col), ("expsim", expsim)):
        np.testing.assert_array_equal(got[k], want, err_msg=f"{k}: {what} at threshold {threshold}")
    assert ix.value_of(0) == vals[0] and ix.value_of(len(vals) - 1) == vals[-1]


def bound_variants(threshold, m=40):
    """a string of m distinct Latin-1 units, and copies with k of its units replaced by ASCII letters it does not
    hold (distance exactly k) for k = maxd - 1, maxd, maxd + 1, maxd = k_lev_tiles' length bound of the pair"""
    t = threshold / 10.0
    maxd = int((m + m) * ((1.0 - t) / (1.0 + t))) + 1
    a = "".join(chr(0xC0 + q) for q in range(m))
    out = [a]
    for k in (maxd - 1, maxd, maxd + 1):
        b = "".join("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"[q] for q in range(k)) + a[k:]
        assert ref.distance(a, b) == k and len(ref.units(b)) == m
        out.append(b)
    return out


def latin_vocabulary(V=611):
    """V values (not a multiple of 32, above 256: pattern tiles straddle text tiles and the diagonal), every unit below
    256: synth strings through the Latin accenting map; lengths 0, 1, 63 and 64 units; 64 units in 128 bytes with
    one-edit variants; pairs at k_lev_tiles' length bound at thresholds 7 and 5"""
    from dblink_b200 import synth

    edge = ["", "é", "a", "é" * 63, "é" * 64, "é" * 63 + "e", "é" * 32 + "a" + "é" * 31, "e" + "é" * 63,
            "é" * 62 + "ÿ", "ab" * 32, "ÿ" * 64, "ÿ" * 63]
    edge += bound_variants(7.0) + bound_variants(5.0)
    strings, _ = synth._string_vocab(np.random.default_rng(17), 2 * V)
    vals = list(dict.fromkeys(edge + [s.translate(LATIN) for s in strings]))[:V]
    assert len(vals) == V and max(max(ref.units(s), default=0) for s in vals) < 256
    assert {0, 1, 63, 64} <= {len(ref.units(s)) for s in vals} and len(("é" * 64).encode()) == 128
    return vals


@pytest.mark.parametrize("threshold", [7.0, 5.0, 0.0])
def test_latin_vocabulary_on_device_equals_literal(monkeypatch, threshold):
    vw = weights(latin_vocabulary())
    ix = build(monkeypatch, vw, threshold, "1")
    assert ix.pairs_on_device, "64 code units in 128 bytes take the device kernel"
    assert_literal_rows(ix, vw, threshold, "Latin, device")
    host = build(monkeypatch, vw, threshold, "0")
    assert not host.pairs_on_device
    dt, ht = ix.tables(), host.tables()
    for k in TABLE_KEYS:
        np.testing.assert_array_equal(dt[k], ht[k], err_msg=k)


def test_65_code_units_take_the_host_loop(monkeypatch):
    vw = weights(latin_vocabulary(300) + ["é" * 65, "é" * 64 + "a"])
    ix = build(monkeypatch, vw, 7.0, "1")
    assert not ix.pairs_on_device, "a value of 65 code units is beyond the kernel's 64-bit columns"
    assert_literal_rows(ix, vw, 7.0, "65 units, host")


def distinct_units(vals):
    return {u for s in vals for u in ref.units(s)}


def wide_vocabulary():
    """a vocabulary with exactly 256 distinct code units, among them CJK characters and both halves of surrogate pairs
    (64 units in 128 bytes among them), and one more value that brings a 257th"""
    vals = latin_vocabulary(280)[:200] + ["张伟", "张伟a", "😀a", "😀b", "😀" * 32, "😀" * 31 + "a", "ω" * 10, "\U00020000"]
    fill = [cp for cp in range(0x4E00, 0x9FFF) if cp not in {ord("张"), ord("伟")}]
    need = 256 - len(distinct_units(vals))
    assert need > 0
    cjk = [chr(cp) for cp in fill[:need + 1]]
    vals += ["".join(cjk[q:min(q + 4, need)]) + "张" for q in range(0, need, 4)]
    assert len(distinct_units(vals)) == 256
    units = distinct_units(vals)
    assert any(0xD800 <= u < 0xDC00 for u in units) and any(0xDC00 <= u < 0xE000 for u in units)
    return vals, vals + [cjk[need] + "张伟"]


def test_256_distinct_code_units_on_device_257_on_host(monkeypatch):
    v256, v257 = wide_vocabulary()
    assert len(distinct_units(v257)) == 257
    for vals, on_device in ((v256, True), (v257, False)):
        vw = weights(vals)
        for threshold in (7.0, 0.0):
            ix = build(monkeypatch, vw, threshold, "1")
            assert ix.pairs_on_device == on_device, (len(distinct_units(vals)), threshold)
            assert_literal_rows(ix, vw, threshold, f"{len(distinct_units(vals))} distinct units")


def test_retry_path_beyond_the_initial_cap(monkeypatch):
    """threshold 0 at V = 1 600 gives ~1.28 M candidate pairs, more than the first output buffer of 2^20: the driver
    runs the kernel again with a larger one.  Compared with the host loop, which the CPU tests tie to the literal
    reference."""
    from test_levenshtein_units import vocabulary

    vals = vocabulary(MIXED, 1700)[:1600]
    assert len(vals) == 1600 and max(distinct_units(vals)) >= 256
    vw = weights(vals)
    dev = build(monkeypatch, vw, 0.0, "1")
    assert dev.pairs_on_device
    assert dev.nnz > 2 * (1 << 20)
    host = build(monkeypatch, vw, 0.0, "0")
    dt, ht = dev.tables(), host.tables()
    for k in TABLE_KEYS:
        np.testing.assert_array_equal(dt[k], ht[k], err_msg=k)


def accented(v):
    """the sweeps' value map: every value through the mixed accenting map (Latin-1, Greek, CJK, a supplementary-plane
    character); one value in 11 padded to 60 code units (more than 64 bytes), one in 11 prefixed by an emoji"""
    s = v.translate(MIXED)
    h = zlib.crc32(v.encode()) % 11
    if h == 0:
        return "é" * (60 - len(ref.units(s))) + s
    if h == 1:
        return "😀" + s
    return s


def accented_problem():
    g = synth_problem(seed=9, R=700, n_files=2)
    lev = [a for a, attr in enumerate(g["attributes"]) if not attr.is_constant]
    assert lev == [2, 3]
    for rec in g["values"]:
        for a in lev:
            if rec[a] is not None:
                rec[a] = accented(rec[a])
    vals = {rec[a] for rec in g["values"] for a in lev if rec[a] is not None}
    assert any(len(v.encode()) > 64 for v in vals) and any("😀" in v for v in vals)
    assert max(len(ref.units(v)) for v in vals) <= 64
    return g, lev


@pytest.mark.parametrize("sampler", ["PCG-II", "PCG-I", "Gibbs"])
def test_accented_model_sweeps_equal_oracle(oracle, monkeypatch, sampler):
    """from the initial state, 3 sweeps: state, theta and summaries equal the oracle's bit for bit after each, the link
    masses equal the oracle's and lie within LITERAL_MASS_REL of the literal conditionals; the same with the index
    pairs from the host loop and from the device kernel"""
    g, lev = accented_problem()
    finals = []
    for flag in ("0", "1"):
        monkeypatch.setenv("DBL_INDEX_GPU", flag)
        eng, rc, x, file = product_setup(g, 23, 1, (2,))
        assert [rc.indexes[a].pairs_on_device for a in lev] == [flag == "1"] * 2
        m, st, tree, ox, ofile = oracle_setup(oracle, g, 23, 1, (2,))
        np.testing.assert_array_equal(x, ox)
        for a in lev:
            t, o = rc.indexes[a].tables(), m.indexes[a]
            for k in TABLE_KEYS:
                np.testing.assert_array_equal(t[k], getattr(o, k), err_msg=f"attribute {a} {k}")
        eng.set_link_mass_capture(True)
        for it in range(3):
            y, z, link = st.y, st.z, st.link
            eng.sweep(sampler, 1)
            assert st.sweep(oracle.SAMPLERS[sampler]) == 0
            assert_same_state(eng, st)
            mass = eng.link_mass()
            assert_same_mass(mass, st.last_link_mass(), f"{sampler} sweep {it} index pairs {flag}")
            lit = literal_link_mass(oracle, m, st.x, st.file, y, z, link, st.theta, sampler)
            assert_literal_mass(mass, lit, f"{sampler} sweep {it} index pairs {flag}")
        finals.append(eng.download_state())
        eng.close()
    for k in ("link", "y", "z", "theta"):
        np.testing.assert_array_equal(finals[0][k], finals[1][k], err_msg=k)
