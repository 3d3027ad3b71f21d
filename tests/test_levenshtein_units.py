"""LevenshteinSimilarityFn on non-ASCII values, without a GPU.

The reference measures Java Strings, so lengths and edit distances count UTF-16 code units (lev_reference.py restates
it literally).  Here every Levenshtein path of the library (dbl_similarity, the host index build) and of the CPU
oracle (levenshtein, lev_similarity, its index build) is checked against that restatement bit for bit, on values
where UTF-8 bytes, code points and code units all differ: accented Latin, CJK, supplementary-plane characters
(surrogate pairs) and combining marks.  Invalid UTF-8 is refused through the C ABI."""
import ctypes as C
import itertools

import numpy as np
import pytest

import jw_reference
import lev_reference as ref

LEV = "LevenshteinSimilarityFn"

# Latin-1 letters only (one code unit below 256, two UTF-8 bytes each)
LATIN = str.maketrans({"A": "Á", "E": "é", "I": "Ï", "O": "Ø", "U": "ü", "C": "Ç", "N": "ñ", "S": "ß", "Y": "ÿ"})
# plus units above 255: Greek (two bytes), CJK (three bytes) and a supplementary-plane character (four bytes, two units)
MIXED = str.maketrans({"A": "Á", "E": "é", "I": "Ï", "O": "Ø", "U": "ü", "C": "Ç", "N": "ñ", "S": "ß", "Y": "ÿ",
                       "Q": "ω", "Z": "张", "X": "😀"})

NFC_JOSE, NFD_JOSE = "Jos\u00e9", "Jose\u0301"  # precomposed; e + combining acute

# (a, b, edit distance, |a|, |b| in UTF-16 code units, similarity at 7/10 to 4 decimals), worked out by hand:
# unit = 1 - 2 d / (|a| + |b| + d), similarity = 10 / 3 (10 unit - 7) truncated at 0
PINNED = [
    ("Müller", "Muller", 1, 6, 6, 4.8718),
    ("José", "Jose", 1, 4, 4, 2.5926),
    ("François", "Francois", 1, 8, 8, 6.0784),
    ("Zoë", "Zoe", 1, 3, 3, 0.4762),
    ("张伟", "张伟a", 1, 2, 3, 0.0),
    ("😀a", "😀b", 1, 3, 3, 0.4762),
    (NFC_JOSE, NFD_JOSE, 2, 4, 5, 0.0),
    ("😀", "😁", 1, 2, 2, 0.0),  # same high surrogate: one unit differs
    ("\U00020000", "", 2, 2, 0, 0.0),
]

# one-byte, two-byte, three-byte characters and two surrogate pairs
SMALL_ALPHABET = ["a", "é", "ß", "张", "😀", "\U00020000"]

EDGE = ["", "a", "é", "ß", "张", "😀", "\U00020000", "\x80", "\ud7ff", "\ue000", "\uffff", "\U0010ffff",
        "Müller", "Muller", "Mueller", "José", "Jose", NFD_JOSE, "François", "Francois", "Zoë", "Zoe", "张伟", "张伟a",
        "😀a", "😀b", "😀😀", "a😀", "é" * 64, "é" * 63 + "e", "é" * 63, "é" * 65, "😀" * 32, "😀" * 31 + "a",
        "ab" * 32, "é" * 20]


def random_strings(seed, n, max_units=70):
    """n strings of 0..max_units code units mixing ASCII, Latin-1, other BMP and supplementary-plane characters"""
    rng = np.random.default_rng(seed)
    pools = [[chr(c) for c in range(0x41, 0x5B)], [chr(c) for c in range(0xC0, 0x100)],
             [chr(c) for c in (0x3C9, 0x416, 0x5D0, 0x4E00, 0x4F1F, 0x5F20, 0xAC00, 0xFB01)],
             [chr(c) for c in (0x1F600, 0x1F601, 0x1F680, 0x20000, 0x2A6D6, 0x10348)]]
    out = []
    for _ in range(n):
        target, s = int(rng.integers(0, max_units + 1)), ""
        while True:
            pool = pools[int(rng.integers(0, 4))]
            c = pool[int(rng.integers(0, len(pool)))]
            if len(ref.units(s + c)) > target:
                break
            s += c
        out.append(s)
    return out


def vocabulary(table=MIXED, n=260, seed=11):
    """synth strings through an accenting map, plus the edge strings"""
    from dblink_b200 import synth

    strings, _ = synth._string_vocab(np.random.default_rng(seed), n)
    return list(dict.fromkeys([s.translate(table) for s in strings] + EDGE))


def weights(vals):
    return {s: float(1 + (i * 7919) % 13) for i, s in enumerate(vals)}


def test_pinned_by_hand(oracle):
    import dblink_b200 as D

    for a, b, d, la, lb, sim in PINNED:
        assert (len(ref.units(a)), len(ref.units(b))) == (la, lb), (a, b)
        assert ref.distance(a, b) == ref.distance(b, a) == d, (a, b)
        want = ref.similarity(a, b, 7.0, 10.0)
        assert round(want, 4) == sim, (a, b, want)
        assert D.similarity(a, b, LEV, 7.0, 10.0) == want, (a, b)
        assert D.similarity(b, a, LEV, 7.0, 10.0) == want, (a, b)
        assert oracle.levenshtein(a, b) == d, (a, b)
        assert oracle.lev_similarity(a, b, 7.0, 10.0) == want, (a, b)
    # the ASCII golden pairs of SimilarityFnTest.scala:46-74 keep their values
    for s in (lambda a, b, t=5.0: ref.similarity(a, b, t, 10.0), lambda a, b, t=5.0: D.similarity(a, b, LEV, t, 10.0)):
        assert s("John Smith", "John Smith") == 10.0
        assert s("", "") == 10.0
        assert s("", "John Smith") == 0.0
        assert s("Jane Smith", "John Smith") == s("John Smith", "Jane Smith")
        assert s("AB", "BB") == 2.0
        assert s("AB", "BB", 0.0) == 6.0
    assert ref.distance("kitten", "sitting") == 3


def pair_sets():
    words = [""] + ["".join(p) for n in range(1, 4) for p in itertools.product(SMALL_ALPHABET, repeat=n)]
    rnd = random_strings(5, 60)
    return {"small alphabet": list(itertools.product(words, words)),
            "random": list(itertools.product(rnd, rnd)) + list(itertools.product(rnd, EDGE))}


@pytest.mark.parametrize("threshold", [7.0, 0.0])
def test_library_and_oracle_equal_literal(oracle, threshold):
    import dblink_b200 as D

    for name, pairs in pair_sets().items():
        for a, b in pairs:
            want = ref.similarity(a, b, threshold, 10.0)
            assert D.similarity(a, b, LEV, threshold, 10.0) == want, (name, a, b)
            assert oracle.lev_similarity(a, b, threshold, 10.0) == want, (name, a, b)
            assert oracle.levenshtein(a, b) == ref.distance(a, b), (name, a, b)


@pytest.mark.parametrize("threshold", [7.0, 5.0, 0.0])
def test_host_index_equals_literal_rows(oracle, monkeypatch, threshold):
    import dblink_b200 as D

    monkeypatch.setenv("DBL_INDEX_GPU", "0")
    vw = weights(vocabulary())
    ix = D.AttributeIndex.build(vw, "levenshtein", threshold, 10.0)
    assert not ix.pairs_on_device
    got = ix.tables()
    vals, probs, rowptr, col, expsim = ref.index_rows(vw, threshold, 10.0)
    for k, want in (("rowptr", rowptr), ("col", col), ("expsim", expsim)):
        np.testing.assert_array_equal(got[k], want, err_msg=k)
    assert [ix.value_of(i) for i in range(len(vals))] == vals
    literal, _ = jw_reference.oracle_index(oracle, vw, threshold, 10.0, sim=ref.similarity)
    own = oracle.Index.build(vw, False, threshold, 10.0)
    for k in ("phi", "norm", "rowptr", "col", "expsim"):
        np.testing.assert_array_equal(got[k], getattr(own, k), err_msg=k)
        np.testing.assert_array_equal(getattr(literal, k), getattr(own, k), err_msg=k)
    assert [own.value(i) for i in range(len(vals))] == vals


INVALID_UTF8 = [
    b"\x80", b"ab\xbfcd",                 # stray continuation bytes
    b"\xc3", b"a\xe5\xbc", b"\xf0\x9f\x98", b"\xc3a",  # truncated sequences
    b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\xaf", b"\xf0\x80\x80\xaf",  # overlong forms
    b"\xc0\x80",                          # JNI's modified UTF-8 for NUL
    b"\xed\xa0\x80", b"\xed\xbf\xbf",     # encoded surrogates
    b"\xed\xa0\xbd\xed\xb8\x80",          # a surrogate pair encoded as two 3-byte sequences (CESU-8 / modified UTF-8)
    b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xfe", b"\xff",  # above U+10FFFF, bytes that never occur
]


def test_invalid_utf8_is_refused_through_the_abi(oracle):
    """similarity 1 decodes: invalid UTF-8 is DBL_ERR_INVALID from dbl_index_build and NaN from dbl_similarity (the
    oracle: -1, NaN, no index).  Constant and Jaro-Winkler indexes do not decode and accept the same bytes."""
    from dblink_b200 import _lib

    L, O = _lib.load(), oracle.lib()
    w = np.ones(3)
    for bad in INVALID_UTF8:
        with pytest.raises(UnicodeDecodeError):  # Python's strict decoder agrees
            bad.decode("utf-8")
        arr = (C.c_char_p * 3)(b"abc", bad, b"\xc3\xa9")
        h = C.c_void_p()
        assert L.dbl_index_build(C.byref(h), arr, w.ctypes.data_as(_lib.f64p), 3, 1, 7.0, 10.0, 10) == \
            _lib.ERR_INVALID, bad
        for a, b in ((bad, b"abc"), (b"abc", bad), (bad, bad)):
            assert np.isnan(L.dbl_similarity(1, a, b, 7.0, 10.0)), bad
            assert not np.isnan(L.dbl_similarity(2, a, b, 7.0, 10.0)), bad
            assert L.dbl_similarity(0, a, b, 7.0, 10.0) == 0.0
            assert O.orc_levenshtein(a, b) == -1, bad
            assert np.isnan(O.orc_lev_similarity(a, b, 7.0, 10.0)), bad
        assert not O.orc_index_build(arr, w.ctypes.data_as(oracle.c_dp), 3, 0, 7.0, 10.0, 10), bad
        for sim in (0, 2):
            h = C.c_void_p()
            assert L.dbl_index_build(C.byref(h), arr, w.ctypes.data_as(_lib.f64p), 3, sim, 7.0, 10.0, 10) == _lib.OK
            L.dbl_index_free(h)
        oix = O.orc_index_build(arr, w.ctypes.data_as(oracle.c_dp), 3, 1, 7.0, 10.0, 10)
        assert oix
        O.orc_index_free(oix)
    # the boundaries of the valid ranges decode
    for good in ("\x80", "\u07ff", "\u0800", "\ud7ff", "\ue000", "\uffff", "\U00010000", "\U0010ffff"):
        arr = (C.c_char_p * 3)(b"abc", good.encode(), b"\xc3\xa9")
        h = C.c_void_p()
        assert L.dbl_index_build(C.byref(h), arr, w.ctypes.data_as(_lib.f64p), 3, 1, 0.0, 10.0, 10) == _lib.OK
        L.dbl_index_free(h)
        assert L.dbl_similarity(1, good.encode(), b"a" + good.encode(), 0.0, 10.0) == ref.similarity(
            good, "a" + good, 0.0, 10.0)
