"""Entity-value draws of large clusters against the log-space reference (tests/value_reference.py).  CPU only.

probs(v) n(v)^k underflows and the product of the records' factors overflows once a cluster holds enough records
(about 91 records on six equally weighted letters, about 55 agreeing records at theta = 0.05); the draws rescale by
powers of two there (DESIGN.md section 4.7).  These tests reach those sizes with crafted clusters.
"""
import numpy as np
import pytest

from value_reference import SAMPLERS, base_pmf, value_pmf

SIZES = [1, 2, 10, 11, 50, 55, 91, 140, 300]  # kmax = 10 on the first attribute: 11 is its first uncached size
THETAS = [1e-4, 0.05, 0.5]
KINDS = ["agree", "distorted", "mixed"]
LETTERS = {c: 1.0 for c in "ABCDEF"}


def string_vocab(n=60):
    from dblink_b200 import synth

    strings, _ = synth._string_vocab(np.random.default_rng(1), n)
    return list(dict.fromkeys(strings))


def tables_of(ix):
    return {"phi": ix.phi, "norm": ix.norm, "rowptr": ix.rowptr, "col": ix.col, "expsim": ix.expsim,
            "is_const": ix.is_const}


def crafted_specs(oracle):
    """The attributes the crafted clusters live in: [(values -> weights, constant, kmax)] and, per attribute, a value c
    and a neighbour of c in its similarity row"""
    vocab = string_vocab()
    ix0 = oracle.Index.build({s: 1.0 for s in vocab}, False, 7.0, 10.0, 10)
    # c: the first value whose similarity row holds a larger id; it carries weight 40, every other value 1
    c = next(v for v in range(ix0.V) if (ix0.col[ix0.rowptr[v]:ix0.rowptr[v + 1]] > v).any())
    nb = next(int(v) for v in ix0.col[ix0.rowptr[c]:ix0.rowptr[c + 1]] if v != c)
    w = {s: (40.0 if s == ix0.value(c) else 1.0) for s in vocab}
    specs = [(w, False, 10),     # sizes above 10 take the uncached base distribution
             (w, False, 400),    # every size cached
             (LETTERS, False, 2),
             ({"p": 1.0, "q": 3.0, "r": 9.0, "s": 27.0, "t": 2.0}, True, 10)]
    picks = [(c, nb), (c, nb), (2, 3), (0, 2)]  # letters C and D; constants p and r
    return specs, picks


def crafted_attributes(oracle):
    specs, picks = crafted_specs(oracle)
    return [oracle.Index.build(vw, const, 7.0, 10.0, kmax) for vw, const, kmax in specs], picks


def crafted_records(picks, size, kind, rng):
    """x rows and z rows of one cluster: every record agreeing on c (z = 0), every record distorted with values
    alternating c and its neighbour, or distorted neighbours first then agreeing records, plus one missing value"""
    A = len(picks)
    xs, zs = [], []
    for i in range(size):
        x, z = [], []
        for c, nb in picks:
            if kind == "agree":
                x.append(c); z.append(0)
            elif kind == "distorted":
                x.append(c if i % 2 == 0 else nb); z.append(1)
            else:
                first = i < (size + 1) // 2
                x.append(nb if first else c); z.append(1 if first else 0)
        xs.append(x); zs.append(z)
    if kind == "mixed":
        xs.append([-1] * A); zs.append([int(rng.random() < 0.5)] * A)
    return xs, zs


def crafted_state(picks, sizes=SIZES, kinds=KINDS, thetas=THETAS, seed=0):
    """One cluster per (size, kind, theta); file f of every record of a cluster has theta[:, f] = thetas[f].
    -> x, file, z, link, y, theta, [(entity, size, kind, f)]"""
    rng = np.random.default_rng(seed)
    X, Z, file, link, Y, info = [], [], [], [], [], []
    for size in sizes:
        for kind in kinds:
            for f in range(len(thetas)):
                e = len(Y)
                xs, zs = crafted_records(picks, size, kind, rng)
                X += xs; Z += zs
                file += [f] * len(xs)
                link += [e] * len(xs)
                Y.append([nb if kind == "distorted" else c for c, nb in picks])
                info.append((e, size, kind, f))
    theta = np.tile(np.array(thetas, np.float64), (len(picks), 1))
    return (np.array(X, np.int32), np.array(file, np.int32), np.array(Z, np.uint8), np.array(link, np.int32),
            np.array(Y, np.int32), theta, info)


def test_base_pmfs_match_log_space_reference(oracle):
    """every cached row B_k, k <= 400, is finite, sums to 1 and equals the log-space B_k; the rows of the six letters
    underflow from k = 91 on, those of the states vocabulary from k = 140"""
    from dblink_b200 import synth
    from test_oracle_golden import STATE_WEIGHTS

    strings, _ = synth._string_vocab(np.random.default_rng(3), 1600)
    big = {s: float(1 + (i * 7919) % 13) for i, s in enumerate(dict.fromkeys(strings))}
    skewed = {s: (1e6 if i == 0 else 1e-3 * (1 + i % 7)) for i, s in enumerate(string_vocab())}
    cases = {"letters": (LETTERS, 7.0), "states": (STATE_WEIGHTS, 5.0), "synthetic1600": (big, 7.0),
             "skewed": (skewed, 7.0)}
    for name, (vw, thr) in cases.items():
        ix = oracle.Index.build(vw, False, thr, 10.0, 400)
        tab = tables_of(ix)
        for k in range(401):
            p = ix.pk[k]
            assert np.isfinite(p).all() and abs(p.sum() - 1.0) < 1e-12, (name, k)
            np.testing.assert_allclose(p, base_pmf(tab, k), rtol=1e-11, atol=1e-30, err_msg=f"{name} k={k}")
            np.testing.assert_allclose(ix.cdf[k], np.cumsum(p), rtol=1e-12, atol=1e-15, err_msg=f"{name} k={k}")
            assert ix.cdf[k][-1] == pytest.approx(1.0, abs=1e-12)


@pytest.fixture(scope="module")
def crafted(oracle):
    idx, picks = crafted_attributes(oracle)
    x, file, z, link, y, theta, info = crafted_state(picks)
    m = oracle.Model(idx, [1.0] * len(idx), [4.0] * len(idx), None, 99, theta.shape[1])
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    return idx, st, x, file, z, link, theta, info


def cluster_of(x, z, file, link, theta, e, a):
    recs = np.flatnonzero(link == e)
    obs = recs[x[recs, a] >= 0]
    return x[obs, a], z[obs, a], theta[a, file[obs]]


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_literal_value_pmf_matches_log_space_reference(oracle, crafted, sampler):
    """the oracle's literal conditional equals the log-space one to 1e-12 for every crafted cluster (1e-10 for
    probabilities below 1e-100)"""
    idx, st, x, file, z, link, theta, info = crafted
    for e, size, kind, f in info:
        for a, ix in enumerate(idx):
            got = st.ref_value_pmf(e, a, oracle.SAMPLERS[sampler])
            want = value_pmf(tables_of(ix), *cluster_of(x, z, file, link, theta, e, a), sampler)
            what = f"{sampler} size {size} {kind} theta {THETAS[f]} attribute {a}"
            big = want > 1e-100  # below, a logarithm's last bits (|log p| ulp) dominate the relative error
            np.testing.assert_allclose(got[big], want[big], rtol=1e-12, err_msg=what)
            np.testing.assert_allclose(got, want, rtol=1e-10, atol=1e-300, err_msg=what)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_large_cluster_value_draws_follow_log_space_conditional(oracle, crafted, sampler):
    """value draws over a (u0, u1) grid reproduce the log-space conditional for clusters of 1 to 300 records: all
    agreeing, all distorted or mixed; theta 1e-4, 0.05 and 0.5; string attributes with cached and uncached base
    distributions (the six letters from k = 3 on), and a constant attribute"""
    idx, st, x, file, z, link, theta, info = crafted
    n = 40
    us = (np.arange(n) + 0.5) / n
    for e, size, kind, f in info:
        for a, ix in enumerate(idx):
            pmf = value_pmf(tables_of(ix), *cluster_of(x, z, file, link, theta, e, a), sampler)
            cnt = np.zeros(ix.V)
            for u0 in us:
                for u1 in us:
                    cnt[st.value_draw(e, a, oracle.SAMPLERS[sampler], u0, u1)] += 1
            emp = cnt / cnt.sum()
            what = f"{sampler} size {size} {kind} theta {THETAS[f]} attribute {a}"
            assert np.abs(emp - pmf).max() < 2.5 / n, what
            assert not np.any((pmf == 0) & (cnt > 0)), what
