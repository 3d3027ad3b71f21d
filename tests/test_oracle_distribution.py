"""The draw PROTOCOL (what the CUDA path reproduces bit for bit) against LITERAL restatements of the reference's
conditionals, and against the exact posterior obtained by brute-force enumeration on a tiny model.  This is
what stands in for the sampler tests the reference does not have (SURVEY.md section 4 / 8c).  CPU only."""
import itertools
import math

import numpy as np
import pytest
from scipy.special import betaln

from helpers import oracle_setup, random_state, synth_problem

SAMPLERS = ["PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential"]


@pytest.fixture(scope="module")
def problem(oracle):
    g = synth_problem(seed=17, R=240, n_files=2, missing=0.06, distortion=0.2)
    m, st0, tree, x, file = oracle_setup(oracle, g, 5)
    Vs = [ix.V for ix in m.indexes]
    rng = np.random.default_rng(3)
    y, link, z = random_state(rng, x, 40, Vs)
    theta = rng.uniform(0.01, 0.3, (len(Vs), 2))
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    return m, st, x, Vs


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_link_weights_protocol_is_proportional_to_literal(oracle, problem, sampler):
    """protocol weights == GU:363-395 / GU:434-466 weights up to a record-constant factor"""
    m, st, x, Vs = problem
    cand = np.arange(st.E, dtype=np.int32)
    for r in range(0, st.R, 7):
        wp = st.link_weights(r, oracle.SAMPLERS[sampler], cand)
        wl = st.link_weights(r, oracle.SAMPLERS[sampler], cand, literal=True)
        assert ((wp > 0) == (wl > 0)).all()
        assert (wl > 0).any()  # invariant: the current entity is always a candidate (GU:262-263)
        pos = wl > 0
        ratio = wp[pos] / wl[pos]
        np.testing.assert_allclose(ratio, ratio[0], rtol=1e-11)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_value_draw_follows_literal_conditional(oracle, problem, sampler):
    """value draws over a dense grid of (u0, u1) reproduce the full-domain conditional (GU:534-599, 605-727)"""
    m, st, x, Vs = problem
    n = 96
    us = (np.arange(n) + 0.5) / n
    checked = 0
    for e in range(0, st.E, 3):
        for a in range(m.A):
            pmf = st.ref_value_pmf(e, a, oracle.SAMPLERS[sampler])
            cnt = np.zeros(Vs[a])
            for u0 in us:
                for u1 in us:
                    cnt[st.value_draw(e, a, oracle.SAMPLERS[sampler], u0, u1)] += 1
            emp = cnt / cnt.sum()
            assert np.abs(emp - pmf).max() < 2.5 / n, (e, a)
            assert not np.any((pmf == 0) & (cnt > 0))  # never draws a zero-probability value
            checked += 1
    assert checked > 40


def test_distortion_probability_literal(oracle, problem):
    """z draws of one sweep follow GU:324-359 given the post-sweep y/theta"""
    m, st0, x, Vs = problem
    st = oracle.State.from_arrays(m, st0.x, st0.file, st0.z, st0.link, st0.y, st0.theta, 0)
    st.sweep(oracle.PCG_I)
    z, theta = st.z, st.theta
    y, link = st.y, st.link
    # deterministic cases
    for r in range(st.R):
        for a in range(m.A):
            p = st.ref_dist_prob(r, a)
            if x[r, a] >= 0 and x[r, a] != y[link[r], a]:
                assert p == 1.0 and z[r, a] == 1
            # the protocol's uniform for this draw
            u0, _ = oracle.uniform2(m.seed, 4, 1, r, a)
            assert z[r, a] == (1 if (p == 1.0 or u0 < p) else 0)


def test_uniform_streams_are_independent_of_layout(oracle):
    """draws are keyed by global ids: permuting nothing but the number of blocks leaves PCG draws of records
    whose block content is unchanged... (smoke check: same seed/iteration/id -> same uniforms)"""
    a = oracle.uniform2(7, 2, 5, 123, 0)
    assert a == oracle.uniform2(7, 2, 5, 123, 0)
    assert a != oracle.uniform2(7, 2, 5, 124, 0)
    assert a != oracle.uniform2(7, 2, 6, 123, 0)
    assert a != oracle.uniform2(8, 2, 5, 123, 0)
    assert a != oracle.uniform2(7, 3, 5, 123, 0)


# ---------------------------------------------------------------------------------------------------
# exact posterior by enumeration
# ---------------------------------------------------------------------------------------------------
def tiny_model(oracle):
    vocab = {"ANNA": 3.0, "ANNE": 2.0, "BOB": 2.0, "ROB": 1.0}
    lev = oracle.Index.build(vocab, False, 7.0, 10.0)
    con = oracle.Index.build({"x": 3.0, "y": 2.0}, True)
    x = np.array([[lev.value_id("ANNA"), 0], [lev.value_id("ANNE"), 0], [lev.value_id("BOB"), 1], [-1, 1]], np.int32)
    return lev, con, x


def exact_partition_posterior(lev, con, x, E, alpha, beta):
    """p(partition of records | x) with theta integrated out; model of SURVEY.md section 0.1"""
    idx = [lev, con]
    R, A = x.shape
    post = {}
    e_lev = np.ones((lev.V, lev.V))
    for v in range(lev.V):
        for w, ev in lev.sim_values_of(v).items():
            e_lev[v, w] = ev
    for lam in itertools.product(range(E), repeat=R):
        part = tuple(sorted(tuple(r for r in range(R) if lam[r] == e) for e in set(lam)))
        tot = 0.0
        for ys in itertools.product(*[range(ix.V) for _ in range(E) for ix in idx]):
            y = np.array(ys).reshape(E, A)
            prior_y = np.prod([idx[a].phi[y[e, a]] for e in range(E) for a in range(A)])
            # per (r, a): factor for z=0 and z=1
            f0 = np.zeros((R, A))
            f1 = np.zeros((R, A))
            for r in range(R):
                for a in range(A):
                    xv, yv = x[r, a], y[lam[r], a]
                    if xv < 0:
                        f0[r, a] = f1[r, a] = 1.0
                    else:
                        f0[r, a] = 1.0 if xv == yv else 0.0
                        if idx[a].is_const:
                            f1[r, a] = idx[a].phi[xv]
                        else:
                            f1[r, a] = idx[a].phi[xv] * idx[a].norm[yv] * e_lev[xv, yv]
            like = 1.0
            for a in range(A):  # one file: sum over z of prod f * Beta-binomial(n_dist)
                s = 0.0
                for zs in itertools.product((0, 1), repeat=R):
                    w = np.prod([f1[r, a] if zs[r] else f0[r, a] for r in range(R)])
                    if w == 0.0:
                        continue
                    nd = sum(zs)
                    s += w * math.exp(betaln(alpha + nd, beta + R - nd) - betaln(alpha, beta))
                like *= s
            tot += prior_y * like
        post[part] = post.get(part, 0.0) + tot
    z = sum(post.values())
    return {k: v / z for k, v in post.items()}


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_chain_targets_exact_posterior(oracle, sampler):
    """the protocol chain's distribution over record partitions matches brute-force enumeration (all four
    samplers target the same posterior, ProjectStep.scala:54-57)"""
    lev, con, x = tiny_model(oracle)
    E, alpha, beta = 3, 1.0, 4.0
    exact = exact_partition_posterior(lev, con, x, E, alpha, beta)
    m = oracle.Model([lev, con], [alpha, alpha], [beta, beta], None, 20240 + SAMPLERS.index(sampler), 1)
    st = oracle.State.init(m, x, np.zeros(4, np.int32), E)
    n_burn, n_keep = 500, 40000
    st.sweep(oracle.SAMPLERS[sampler], n_burn)
    counts = {}
    for _ in range(n_keep):
        st.sweep(oracle.SAMPLERS[sampler])
        lam = st.link
        part = tuple(sorted(tuple(r for r in range(4) if lam[r] == e) for e in set(lam.tolist())))
        counts[part] = counts.get(part, 0) + 1
    tv = 0.5 * sum(abs(exact.get(k, 0.0) - counts.get(k, 0) / n_keep) for k in set(exact) | set(counts))
    assert tv < 0.03, (tv, sorted(exact.items(), key=lambda kv: -kv[1])[:4],
                       sorted(((k, v / n_keep) for k, v in counts.items()), key=lambda kv: -kv[1])[:4])


def test_threaded_link_phase_gives_the_same_chain(oracle, monkeypatch):
    """ORC_THREADS splits the link update over host threads; every record has its own counter-based stream, so the
    chain is the same for any split."""
    import numpy as np

    from helpers import oracle_setup, synth_problem

    g = synth_problem(seed=9, R=900, n_files=2)
    out = {}
    # "plain": the PCG-II weights through the literal per-pair form (binary search in the sparse rows) instead of the
    # per-record dense similarity tables the whole-sweep link phase uses for speed -- the same multiplications
    for nt in ("1", "3", "8", "plain"):
        monkeypatch.setenv("ORC_THREADS", "2" if nt == "plain" else nt)
        if nt == "plain":
            monkeypatch.setenv("ORC_NO_DENSE", "1")
        m, st, tree, ox, ofile = oracle_setup(oracle, g, 77, 2, (2, 3))
        for s in ("PCG-II", "PCG-I", "Gibbs", "Gibbs-Sequential"):
            assert st.sweep(oracle.SAMPLERS[s], 2) == 0
        out[nt] = (st.link.copy(), st.y.copy(), st.z.copy(), st.theta.copy())
    for nt in ("3", "8", "plain"):
        for a, b in zip(out["1"], out[nt]):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("row", ["hash64", "hash128", "hash256"])
def test_oracle_link_mass_matches_literal_conditionals(oracle, row):
    """the total mass the oracle's sweep draws each link from (protocol weights, its dense PCG-II tables, the
    lane/chunk summation order) equals the sum of the literal GU:384-389 / GU:444-459 weights over the record's block
    divided by the record constant, for every record of a 900-record, 2-file, 4-block problem; the models are those
    whose similarity rows need 64, 128 and 256 hash slots on the GPU"""
    from dblink_b200 import synth

    from helpers import assert_literal_mass, literal_link_mass, threshold_problem

    C = synth.SynthAttr
    g = {"hash64": lambda: threshold_problem(60, 3.0, extra=[C("c0", "constant", 5), C("c1", "constant", 9)], n_files=2),
         "hash128": lambda: threshold_problem(120, 3.0, extra=[C("s1", "levenshtein", 80)], n_files=2),
         "hash256": lambda: threshold_problem(400, 3.0, n_files=2)}[row]()
    m, st, tree, x, file = oracle_setup(oracle, g, 13, 2, (0,))
    assert tree.n_leaves == 4
    assert not st.last_link_mass().any()  # nothing drawn yet
    for sampler in SAMPLERS:
        for it in range(2):
            y, z, link = st.y, st.z, st.link
            assert st.sweep(oracle.SAMPLERS[sampler]) == 0
            ref = literal_link_mass(oracle, m, x, file, y, z, link, st.theta, sampler)
            assert (ref > 0).all()
            assert_literal_mass(st.last_link_mass(), ref, f"{row} {sampler} sweep {it}")
