"""Literal Python restatement of JaroWinklerSimilarityFn and of the attribute-index rows it gives (test code only).

The CPU oracle restates the reference, which has no Jaro-Winkler function; the Jaro-Winkler rows come from here and
enter the oracle through orc_index_from_tables, which computes the normalisations and base pmfs as for any index."""
import math

import numpy as np


def counts(a: bytes, b: bytes):
    """(m, h, l): each a[i], left to right, matches the first unmatched b[j] with |i - j| <= w and a[i] == b[j],
    w = max(0, max(|a|, |b|) / 2 - 1); h = positions k where the k-th matched bytes of a and b differ; l = common
    prefix, at most 4"""
    la, lb = len(a), len(b)
    if la == 0 or lb == 0:
        return 0, 0, 0
    w = max(0, max(la, lb) // 2 - 1)
    ma, mb = [False] * la, [False] * lb
    for i in range(la):
        for j in range(lb):
            if not mb[j] and abs(i - j) <= w and a[i] == b[j]:
                ma[i] = mb[j] = True
                break
    sa = [a[i] for i in range(la) if ma[i]]
    sb = [b[j] for j in range(lb) if mb[j]]
    h = sum(x != y for x, y in zip(sa, sb))
    l = 0
    while l < min(4, la, lb) and a[l] == b[l]:
        l += 1
    return len(sa), h, l


def unit(a: str, b: str):
    """Jaro-Winkler unit similarity of the UTF-8 bytes, prefix scale 0.1 (Python floats: IEEE doubles, no FMA)"""
    a, b = a.encode(), b.encode()
    if not a and not b:
        return 1.0
    m, h, l = counts(a, b)
    if m == 0:
        return 0.0
    jaro = (m / len(a) + m / len(b) + (m - 0.5 * h) / m) / 3.0
    return jaro + (0.1 * l) * (1.0 - jaro)


def similarity(a, b, threshold, max_sim):
    """the truncation of SimilarityFn.scala:65-70 applied to the unit similarity"""
    factor = max_sim / (max_sim - threshold)
    s = factor * (max_sim * unit(a, b) - threshold)
    return s if s > 0.0 else 0.0


def index_rows(values_weights, threshold, max_sim):
    """AttributeIndex.scala:107-231 for Jaro-Winkler: value ids in byte order, probs = weight / total (total summed in
    id order), all pairs kept when exp(sim) > 1 (pairs j >= i scored, mirrored: the counts are symmetric).
    -> (values in id order, probs, rowptr, col, expsim)"""
    vals = sorted(values_weights, key=lambda s: s.encode())
    total = 0.0
    for v in vals:
        total += values_weights[v]
    probs = np.array([values_weights[v] / total for v in vals])
    rows = [[] for _ in vals]
    for i, a in enumerate(vals):
        for j in range(i, len(vals)):
            e = math.exp(similarity(a, vals[j], threshold, max_sim))
            if e > 1.0:
                rows[i].append((j, e))
                if j != i:
                    rows[j].append((i, e))
    rowptr = np.zeros(len(vals) + 1, np.int32)
    rowptr[1:] = np.cumsum([len(r) for r in rows])
    col = np.array([c for r in rows for c, _ in sorted(r)], np.int32)
    expsim = np.array([e for r in rows for _, e in sorted(r)], np.float64)
    return vals, probs, rowptr, col, expsim


def oracle_index(O, values_weights, threshold, max_sim, kmax=10):
    """-> (oracle Index built from the Jaro-Winkler rows, {value: id})"""
    vals, probs, rowptr, col, expsim = index_rows(values_weights, threshold, max_sim)
    return O.Index.from_tables(probs, rowptr, col, expsim, False, kmax), {v: i for i, v in enumerate(vals)}
