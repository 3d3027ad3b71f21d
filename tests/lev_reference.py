"""Literal Python restatement of LevenshteinSimilarityFn on Java Strings (test code only).

The reference computes it on java.lang.String (SimilarityFn.scala:92-98): `a.length` counts UTF-16 code units, and
commons-lang3 StringUtils.getLevenshteinDistance compares them with charAt, so a supplementary-plane character is two
units and "e" + U+0301 is two units (no normalisation).  Here a string's units come from its UTF-16 encoding, the
distance is the full (|a|+1)(|b|+1) DP with no length bound and no early exit, and the unit formula and truncation
run in the reference's order of operations (Python floats: IEEE doubles without FMA), so results compare with ==."""
import functools
import struct

import jw_reference


def units(s: str):
    """the UTF-16 code units of s: what a Java String holds"""
    b = s.encode("utf-16-le")
    return struct.unpack(f"<{len(b) // 2}H", b)


@functools.lru_cache(maxsize=None)
def distance(a: str, b: str):
    """getLevenshteinDistance over code units: d[i][j] = edit distance of the first i units of a and j units of b"""
    ua, ub = units(a), units(b)
    d = [[0] * (len(ub) + 1) for _ in range(len(ua) + 1)]
    for i in range(len(ua) + 1):
        d[i][0] = i
    for j in range(len(ub) + 1):
        d[0][j] = j
    for i in range(1, len(ua) + 1):
        for j in range(1, len(ub) + 1):
            cost = 0 if ua[i - 1] == ub[j - 1] else 1
            d[i][j] = min(d[i - 1][j] + 1, d[i][j - 1] + 1, d[i - 1][j - 1] + cost)
    return d[len(ua)][len(ub)]


def unit(a: str, b: str):
    """SimilarityFn.scala:92-98: 1 - 2 d / (|a| + |b| + d) in code units, 1 when both are empty"""
    total = len(units(a)) + len(units(b))
    if total > 0:
        dist = float(distance(a, b))
        return 1.0 - 2.0 * dist / (total + dist)
    return 1.0


def similarity(a, b, threshold, max_sim):
    """SimilarityFn.scala:69-72: the truncated transform of the unit similarity"""
    trans_factor = max_sim / (max_sim - threshold)
    trans = trans_factor * (max_sim * unit(a, b) - threshold)
    return trans if trans > 0.0 else 0.0


def index_rows(values_weights, threshold, max_sim):
    """computeSimValueIndex (AttributeIndex.scala:219-231) under this similarity: jw_reference.index_rows' layout"""
    return jw_reference.index_rows(values_weights, threshold, max_sim, similarity)
