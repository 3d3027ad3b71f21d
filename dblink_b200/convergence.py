"""Convergence diagnostics across chains: split-R̂ (Gelman et al., BDA3 §11.4) and its rank-normalised, folded
variant (Vehtari, Gelman, Simpson, Carpenter & Bürkner 2021).

The chains of a run differ in their Philox keys (which also draw the missing initial entity values) and otherwise
start from State.deterministic: they are not over-dispersed, so an R̂ near 1 is weaker evidence of mixing than it
would be from over-dispersed starts.
"""
import csv
import math
import os
from statistics import NormalDist

import numpy as np

# diagnostics.csv columns that are not quantities of the chain
NOT_QUANTITIES = ("iteration", "systemTime-ms", "popSize")
MIN_DRAWS = 4


def _halves(draws):
    """K x n -> 2K x N halves, N = n // 2 (an odd n drops the middle draw)."""
    d = np.asarray(draws, np.float64)
    if d.ndim != 2:
        raise ValueError("draws must be chains x draws")
    n = d.shape[1]
    N = n // 2
    return np.concatenate([d[:, :N], d[:, n - N:]], axis=0)


def _rhat(h):
    """R̂ of the 2K halves (rows): W = mean of their variances (ddof 1), B/N = variance of their means (ddof 1),
    R̂ = sqrt(((N-1)/N W + B/N) / W); NaN when W = 0."""
    N = h.shape[1]
    W = float(np.mean(np.var(h, axis=1, ddof=1)))
    B_over_N = float(np.var(np.mean(h, axis=1), ddof=1))
    if not W > 0.0:
        return float("nan")
    return math.sqrt(((N - 1) / N * W + B_over_N) / W)


def split_rhat(draws):
    """Split-R̂ of a chains x draws array (BDA3 §11.4): R̂ over the 2K halves of the chains."""
    h = _halves(draws)
    if h.shape[1] < 2:
        raise ValueError(f"split-R̂ needs at least {MIN_DRAWS} draws per chain")
    return _rhat(h)


def _rank_normalise(h):
    """pooled ranks (ties averaged) -> z = Phi^-1((rank - 3/8) / (S + 1/4)), S = number of draws"""
    flat = h.ravel()
    order = np.argsort(flat, kind="stable")
    ranks = np.empty(len(flat))
    sv = flat[order]
    i = 0
    while i < len(sv):  # runs of equal values share the mean of their ranks (1-based)
        j = i
        while j + 1 < len(sv) and sv[j + 1] == sv[i]:
            j += 1
        ranks[order[i:j + 1]] = (i + j) / 2.0 + 1.0
        i = j + 1
    inv = NormalDist().inv_cdf
    S = len(flat)
    z = np.array([inv((r - 0.375) / (S + 0.25)) for r in ranks])
    return z.reshape(h.shape)


def rank_normalized_split_rhat(draws):
    """max(split-R̂ of the rank-normalised draws, split-R̂ of the rank-normalised folded draws |x - median|), both over
    the 2K split halves; NaN when the draws are constant."""
    h = _halves(draws)
    if h.shape[1] < 2:
        raise ValueError(f"split-R̂ needs at least {MIN_DRAWS} draws per chain")
    if not np.var(h) > 0.0:
        return float("nan")
    bulk = _rhat(_rank_normalise(h))
    folded = np.abs(h - np.median(h))
    tail = _rhat(_rank_normalise(folded)) if np.var(folded) > 0.0 else float("nan")
    if math.isnan(tail):
        return bulk
    return max(bulk, tail)


def read_diagnostics(path, lower_iteration_cutoff=0):
    """diagnostics.csv -> (column names, float64 rows at or after the cutoff)"""
    with open(path) as fh:
        rows = list(csv.reader(fh))
    head, body = rows[0], rows[1:]
    it = head.index("iteration")
    data = np.array([[float(v) for v in r] for r in body if int(r[it]) >= lower_iteration_cutoff], np.float64)
    return head, data.reshape(-1, len(head))


def convergence_diagnostics(paths, lower_iteration_cutoff=0):
    """One diagnostics.csv per chain -> [(quantity, splitRhat, rankNormalizedSplitRhat, numChains, drawsPerChain)]
    over the rows at or after the cutoff (every chain cut to the shortest one's draws)."""
    if len(paths) < 2:
        raise ValueError("convergence-diagnostics needs numChains >= 2")
    tables = [read_diagnostics(p, lower_iteration_cutoff) for p in paths]
    head = tables[0][0]
    if any(t[0] != head for t in tables):
        raise ValueError("the chains' diagnostics.csv files have different columns")
    n = min(len(t[1]) for t in tables)
    if n < MIN_DRAWS:
        raise ValueError(f"convergence-diagnostics needs at least {MIN_DRAWS} draws per chain after the cutoff")
    out = []
    for c, name in enumerate(head):
        if name in NOT_QUANTITIES:
            continue
        d = np.stack([t[1][:n, c] for t in tables])
        out.append((name, split_rhat(d), rank_normalized_split_rhat(d), len(paths), n))
    return out


def save_convergence_diagnostics(rows, output_path):
    with open(os.path.join(output_path, "convergence-diagnostics.csv"), "w") as fh:
        fh.write("quantity,splitRhat,rankNormalizedSplitRhat,numChains,drawsPerChain\n")
        for q, r, rn, k, n in rows:
            fh.write(f"{q},{r!r},{rn!r},{k},{n}\n")
