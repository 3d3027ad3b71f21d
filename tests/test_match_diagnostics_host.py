"""Per-pair MCMC diagnostics of the match probabilities on the host: the numpy path (analysis_arrays.
pairwise_match_diagnostics) against the literal analysis.pairwise_match_diagnostics (autocovariances by their
definition in fractions, Geyer's sequences verbatim) on small chains of 1 to 3 chains; R̂ against
convergence.split_rhat; the ESS of iid and Markov draws; the size refusals; the files Project.execute writes on
RLdata500 with 1 and 2 chains; the C ABI's NULL-handle refusals."""
import csv
import gzip
import math
import os
import shutil

import numpy as np
import pytest

from test_binder_host import chain_of, project_of

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def close(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b or abs(a - b) <= 1e-12 * abs(b)


def crafted_chain(K, n, R, seed, extra=0):
    """K chains of n draws (chain k gets n + k * extra) over R > 6 records: records 0, 1 always linked; 2, 3 linked in
    chain 0 only; 4, 5 linked in a single draw; the others relinked at random with some persistence."""
    rng = np.random.default_rng(seed)
    links, chains = [], []
    for k in range(K):
        base = rng.integers(0, R - 6, R)
        for t in range(n + k * extra):
            link = base.copy()
            move = rng.random(R) < 0.3
            link[move] = rng.integers(0, R - 6, int(move.sum()))
            if t % 2 == 0:
                base = link
            link = link + 6  # labels 6 .. R - 1 for the random part, 0 .. 5 for the crafted pairs
            link[0] = link[1] = 0
            link[2], link[3] = (2, 2) if k == 0 else (2, 3)
            link[4], link[5] = (4, 4) if (k, t) == (0, 1) else (4, 5)
            links.append(link)
            chains.append(k)
    return chain_of(links, chains=chains)


def literal(ch):
    """analysis.pairwise_match_diagnostics of a pooled ChainArrays, keyed by (first, second) record indices."""
    from dblink_b200 import analysis, analysis_arrays as aa

    K = int(ch.chains.max()) + 1
    chains = [[] for _ in range(K)]
    for k, (mem, off, _) in zip(ch.chains, ch.samples):
        keys = aa.sample_pair_keys(ch.num_records, mem, off)
        chains[k].append({frozenset((int(x >> 32), int(x & 0xFFFFFFFF))) for x in keys})
    return {tuple(sorted(p)): v for p, v in analysis.pairwise_match_diagnostics(chains).items()}


CASES = [(1, 4, 0), (1, 9, 0), (1, 40, 0), (2, 4, 0), (2, 7, 3), (2, 30, 1), (3, 5, 0), (3, 12, 2), (3, 21, 0)]


@pytest.mark.parametrize("K,n,extra", CASES)
def test_numpy_equals_the_literal_restatement(K, n, extra):
    from dblink_b200 import analysis_arrays as aa

    ch = crafted_chain(K, n, 12, seed=100 * K + n, extra=extra)
    first, second, count, mix = aa.pairwise_match_diagnostics(ch)
    want = literal(ch)
    assert mix.M == 2 * K and mix.draws == n and mix.N == n // 2
    # every pair linked in a used draw is in the literal dict; a pair linked only in unused draws has no linked draw
    for i, (a, b) in enumerate(zip(first, second)):
        w = want.get((a, b))
        got = (mix.count[i], mix.chain_min[i], mix.chain_max[i], mix.max_t[i], mix.rhat[i], mix.ess[i])
        if w is None:
            assert got[:3] == (0, 0, 0) and math.isnan(got[4])
            continue
        assert got[:4] == w[:4], (a, b)
        assert close(got[4], w[4]) and close(got[5], w[5]), (a, b, got, w)
    at = {(a, b): i for i, (a, b) in enumerate(zip(first, second))}
    assert set(want) <= set(at)
    # the crafted pairs: always linked -> undefined; one chain only -> inf; a single draw
    i = at[(0, 1)]
    assert math.isnan(mix.rhat[i]) and math.isnan(mix.ess[i]) and mix.count[i] == 2 * K * (n // 2)
    if K > 1:
        i = at[(2, 3)]
        assert mix.rhat[i] == math.inf and mix.chain_min[i] == 0 and mix.chain_max[i] == 2 * (n // 2)
    i = at[(4, 5)]
    assert count[i] == 1 and mix.count[i] == 1 and mix.rhat[i] >= 1 and mix.ess[i] > 0


@pytest.mark.parametrize("K,n,extra", CASES)
def test_rhat_is_the_split_rhat_of_the_draws(K, n, extra):
    from dblink_b200 import analysis_arrays as aa, convergence

    ch = crafted_chain(K, n, 16, seed=7 * K + n, extra=extra)
    first, second, _, mix = aa.pairwise_match_diagnostics(ch)
    starts, n_used = aa.chain_draws(ch)
    assert n_used == n and list(starts) == [sum(n + j * extra for j in range(k)) for k in range(K)]
    x = aa.pairwise_match_trace(ch, (first << 32) | second)
    for i in range(len(first)):
        want = convergence.split_rhat(np.stack([x[i, s:s + n] for s in starts]).astype(float))
        if math.isnan(want):  # convergence.py leaves W = 0 undefined; here it is inf unless every draw is equal
            assert math.isinf(mix.rhat[i]) or math.isnan(mix.rhat[i])
        else:
            assert abs(mix.rhat[i] - want) <= 1e-12 * want


def test_iid_draws_have_an_ess_near_their_number():
    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(2024)
    K, n = 2, 400
    x = rng.random((300, K * n)) < rng.uniform(0.2, 0.8, (300, 1))
    mix = aa.mixing_from_trace(x, [0, n], n, aa.ess_floor(K, n))
    ratio = mix.ess / (K * n)
    assert 0.9 <= ratio.mean() <= 1.1 and (mix.rhat < 1.1).all()


def test_a_two_state_markov_chain_has_the_ess_of_its_correlation():
    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(7)
    K, n, H = 1, 2000, 200
    for phi in (0.5, 0.8):
        # stay with probability (1 + phi) / 2, else flip: a symmetric chain with lag-1 correlation phi
        x = np.zeros((H, K * n), bool)
        x[:, 0] = rng.random(H) < 0.5
        flip = rng.random((H, K * n)) >= (1 + phi) / 2
        for t in range(1, K * n):
            x[:, t] = x[:, t - 1] ^ flip[:, t]
        mix = aa.mixing_from_trace(x, [0], n, aa.ess_floor(K, n))
        want = K * n * (1 - phi) / (1 + phi)
        assert abs(np.median(mix.ess) / want - 1) <= 0.15, phi


def test_size_refusals():
    from dblink_b200 import analysis_arrays as aa

    ch = crafted_chain(1, 3, 8, seed=1)
    with pytest.raises(ValueError, match="^pairwise-match-diagnostics needs at least 4 draws per chain after the cutoff$"):
        aa.pairwise_match_diagnostics(ch)
    with pytest.raises(ValueError, match="at least 4 draws"):
        aa.pairwise_match_diagnostics(crafted_chain(2, 6, 8, seed=1, extra=-3))  # chain 1 has 3 draws
    # M N^2 < 2^30: 2 chains of 2N draws pass at N = 16383 and not at N = 16384
    aa.check_mixing_size(2, 2 * 16383)
    with pytest.raises(ValueError, match=r"^pairwise-match-diagnostics needs M N\^2 < 2\^30: 4 half-chains of 16384 "
                                         r"draws$"):
        aa.check_mixing_size(2, 2 * 16384)
    aa.check_trace_size(64, 1 << 30)
    with pytest.raises(ValueError, match=r"^the match trace needs 2147483650 words, more than 2147483648$"):
        aa.check_trace_size(64, (1 << 30) + 1)


def test_the_trace_cap_refuses_before_the_trace(monkeypatch):
    from dblink_b200 import analysis_arrays as aa

    ch = crafted_chain(2, 6, 10, seed=3)
    H = len(aa.pairwise_match_counts(ch)[0])
    monkeypatch.setattr(aa, "MAX_TRACE_WORDS", H - 1)  # 12 samples: one word per pair
    with pytest.raises(ValueError, match=f"^the match trace needs {H} words, more than {H - 1}$"):
        aa.pairwise_match_diagnostics(ch)
    monkeypatch.setattr(aa, "MAX_TRACE_WORDS", H)
    aa.pairwise_match_diagnostics(ch)


def test_pack_trace_is_word_major():
    from dblink_b200 import analysis_arrays as aa

    x = np.zeros((3, 40), bool)
    x[0, 0] = x[1, 31] = x[2, 32] = x[2, 39] = True
    w = aa.pack_trace(x)
    assert w.shape == (2, 3) and w.dtype == np.uint32
    assert w.tolist() == [[1, 1 << 31, 0], [0, 0, 1 | (1 << 7)]]


def test_abi_refuses_a_null_handle():
    from dblink_b200 import _lib

    L = _lib.load()
    starts = np.zeros(1, np.int32)
    out = [np.zeros(4, np.int32) for _ in range(4)] + [np.zeros(4) for _ in range(2)]
    assert L.dbl_pairs_trace_begin(None, 8) == _lib.ERR_INVALID
    assert L.dbl_pairs_trace_sample(None, np.zeros(4, np.int32).ctypes.data, 0) == _lib.ERR_INVALID
    assert L.dbl_pairs_mixing(None, 1, 1, starts.ctypes.data_as(_lib.i32p), 8, 0.5,
                              *(a.ctypes.data for a in out)) == _lib.ERR_INVALID
    assert all(not a.any() for a in out)


# ---- the project's files ---------------------------------------------------------------------------------
def write_chains(tmp_path, p, S=12, seed=0):
    """RLdata500 as the data, and in every chain directory S samples around its truth (each relinks a fifth of the
    records; chains differ in their seeds)."""
    from dblink_b200 import writers as w

    with gzip.open(os.path.join(GOLDEN, "RLdata500.csv.gz"), "rt") as fh:
        rows = list(csv.DictReader(fh))
    with open(os.path.join(tmp_path, "data.csv"), "w") as fh:
        fh.write("rec_id,ent_id,a\n" + "".join(f"{r['rec_id']},{r['ent_id']},v\n" for r in rows))
    ids = [r["rec_id"] for r in rows]
    _, truth = np.unique([r["ent_id"] for r in rows], return_inverse=True)
    R, E = len(ids), int(truth.max()) + 1
    for k, dr in enumerate(p.chain_dirs()):
        rng = np.random.default_rng(seed + k)
        lw = w.LinkageChainWriter(os.path.join(dr, "linkage-chain.parquet"))
        for s in range(S + k):
            link = truth.copy()
            move = rng.random(R) < 0.2
            link[move] = rng.integers(0, E, int(move.sum()))
            lw.append(10 * (s + 1), w.linkage_structure_arrow(link.astype(np.int32), np.zeros(R, np.int32), ids))
        lw.close()


def host_paths(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, project

    for name in ("pairwise_match_counts", "pairwise_match_diagnostics"):
        monkeypatch.setattr(project, name, getattr(aa, name))


def output_files(root):
    out = {}
    for d, _, files in os.walk(root):
        for f in files:
            path = os.path.join(d, f)
            out[os.path.relpath(path, root)] = open(path, "rb").read()
    return out


@pytest.mark.parametrize("chains", [1, 2])
def test_project_writes_both_files_on_rldata500(tmp_path, monkeypatch, chains):
    from dblink_b200 import analysis_arrays as aa

    host_paths(monkeypatch)
    extra = ", minMatchProbability : 0.2"
    p = project_of(tmp_path, chains=chains, quantities='["pairwise-match-probabilities", "pairwise-match-diagnostics"]',
                   summarize_extra=extra, metrics='["pairwise"]')
    p.steps = lambda: [s for s in type(p).steps(p) if s[0] == "summarize"]
    write_chains(tmp_path, p)
    p.execute(log=lambda *a: None)
    out = str(tmp_path / "out") + "/"
    probs = open(out + "pairwise-match-probabilities.csv").read().splitlines()
    diag = open(out + "pairwise-match-diagnostics.csv").read().splitlines()
    assert diag[0] == "recordId1,recordId2,probability,minChainProbability,maxChainProbability,splitRhat,ess,mcse"
    assert len(diag) == len(probs) > 50
    for a, b in zip(probs[1:], diag[1:]):
        assert b.split(",")[:3] == a.split(",")
    # the numbers are the numpy path's, in the file's order
    ch = p.read_chain(10)
    S = len(ch.samples)
    first, second, count, mix = aa.pairwise_match_diagnostics(ch, aa.min_match_count(0.2, S))
    ids = ch.record_ids.tolist()
    row = {}
    for i in range(len(first)):
        a, b = sorted((str(ids[first[i]]), str(ids[second[i]])))
        row[(a, b)] = i
    D = 2 * mix.N
    mcse = aa.mcse(mix.count, mix.M * mix.N, mix.ess)
    for line in diag[1:]:
        a, b, prob, lo, hi, rh, e, m = line.split(",")
        i = row[(a, b)]
        assert (prob, lo, hi) == tuple(repr(int(c) / d) for c, d in ((count[i], S), (mix.chain_min[i], D), (mix.chain_max[i], D)))
        assert (rh, e, m) == (repr(float(mix.rhat[i])), repr(float(mix.ess[i])), repr(float(mcse[i])))
    summary = dict(line.split(",") for line in open(out + "pairwise-match-diagnostics-summary.csv").read().splitlines())
    assert summary.pop("quantity") == "value"
    assert list(summary) == ["numChains", "drawsPerChain", "pairs", "pairsRhatAbove1.01", "pairsRhatAbove1.1",
                             "pairsRhatInf", "pairsRhatUndefined", "minEss", "medianEss", "pairsEssBelow100PerChain"]
    assert (int(summary["numChains"]), int(summary["drawsPerChain"]), int(summary["pairs"])) == (chains, 12,
                                                                                               len(diag) - 1)
    assert int(summary["pairsRhatUndefined"]) == int(np.isnan(mix.rhat).sum())
    assert int(summary["pairsRhatAbove1.01"]) == int((mix.rhat > 1.01).sum()) > 0
    assert float(summary["medianEss"]) == float(np.median(mix.ess[~np.isnan(mix.ess)]))

    # every other file is the one a run without the quantity writes
    q = project_of(tmp_path, chains=chains, quantities='["pairwise-match-probabilities"]', summarize_extra=extra,
                   metrics='["pairwise"]', out="out2")
    q.steps = lambda: [s for s in type(q).steps(q) if s[0] == "summarize"]
    for dr, dr2 in zip(p.chain_dirs(), q.chain_dirs()):
        shutil.copytree(os.path.join(dr, "linkage-chain.parquet"), os.path.join(dr2, "linkage-chain.parquet"))
    q.execute(log=lambda *a: None)
    with_q, without = output_files(out), output_files(str(tmp_path / "out2") + "/")
    assert set(with_q) - set(without) == {"pairwise-match-diagnostics.csv", "pairwise-match-diagnostics-summary.csv"}
    assert len(without) > 2 and all(with_q[f] == without[f] for f in without)


def test_the_step_describes_the_quantity(tmp_path):
    p = project_of(tmp_path, quantities='["pairwise-match-diagnostics"]', summarize_extra=", minMatchProbability : 0.5")
    assert ("pairwise-match-diagnostics gives split-R̂, effective sample size and Monte Carlo standard error of every "
            "pair's link indicator, for the pairs of minMatchProbability=0.5") in p.steps_mk_string()
    assert "pairwise-match-diagnostics" not in project_of(tmp_path).steps_mk_string()
