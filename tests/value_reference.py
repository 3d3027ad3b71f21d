"""Log-space restatement of the entity-value conditionals, for clusters of any size.

The draws (oracle and CUDA) multiply doubles: probs(v) n(v)^k underflows and the product of the records' factors
overflows once a cluster holds enough records.  Here every weight is a logarithm, normalised through the largest one
and summed with math.fsum, so the reference stays exact where the doubles leave their range.

Tables are those of an attribute index (phi, norm, rowptr, col, expsim, is_const); phi stands in for probs (the
two differ by the constant Z_0, which every distribution below normalises away).
"""
import math

import numpy as np

SAMPLERS = ("PCG-I", "PCG-II", "Gibbs", "Gibbs-Sequential")


def normalise(logw):
    """exp(logw) / sum exp(logw), through the largest term and math.fsum"""
    logw = np.asarray(logw, np.float64)
    w = np.exp(logw - logw.max())
    return w / math.fsum(w.tolist())


def base_pmf(tab, k):
    """(a) B_k(v) = probs(v) n(v)^k / Z_k (getSimNormDist, AttributeIndex.scala:197-216); k is ignored for a constant
    attribute (n == 1)"""
    lw = np.log(tab["phi"])
    if not tab["is_const"]:
        lw = lw + k * np.log(tab["norm"])
    return normalise(lw)


def _row(tab, x):
    lo, hi = tab["rowptr"][x], tab["rowptr"][x + 1]
    return tab["col"][lo:hi], tab["expsim"][lo:hi]


def value_pmf(tab, xs, zs, thetas, sampler):
    """(b) the full-domain conditional of y[e, a] given the cluster's records.

    xs: observed values of the records linked to e (missing ones left out), zs: their distortion flags, thetas: the
    distortion probability of each record's file.
      PCG-I / PCG-II (updateEntityValueCollapsed, GU:534-599): p(v) ~ B_k(v) prod_r g_r(v), g_r(v) = E(x_r, v)
        + [v == x_r] (1/theta_r - 1) / (phi(x_r) n(x_r)) over the records whose similarity row holds v (constant
        attributes: g_r(x_r) = 1 + (1/theta_r - 1) / phi(x_r));
      Gibbs (updateEntityValue, GU:605-727): x_r of the first undistorted record, else B_k(v) prod_r E(x_r, v)
        (constant attributes: phi);
      Gibbs-Sequential (GU:689): x_r of the first undistorted record, else phi(v) prod_r E(x_r, v) n(v) phi(x_r).
    """
    V = len(tab["phi"])
    xs = [int(x) for x in xs]
    k = len(xs)
    collapsed = sampler in ("PCG-I", "PCG-II")
    if not collapsed:
        for x, z in zip(xs, zs):
            if not z:
                p = np.zeros(V)
                p[x] = 1.0
                return p
    logphi, lognorm = np.log(tab["phi"]), np.log(tab["norm"])
    if k == 0 or (not collapsed and tab["is_const"]):
        return normalise(logphi)
    terms = [[] for _ in range(V)]  # log factors of each value, summed with fsum
    for x, th in zip(xs, thetas):
        if tab["is_const"]:  # collapsed (non-collapsed constant attributes returned above)
            terms[x].append(math.log(1.0 + (1.0 / th - 1.0) / tab["phi"][x]))
            continue
        cols, es = _row(tab, x)
        for v, e in zip(cols.tolist(), es.tolist()):
            if collapsed and v == x:
                e = e + (1.0 / th - 1.0) / (tab["phi"][x] * tab["norm"][x])
            terms[v].append(math.log(e))
    if sampler == "Gibbs-Sequential":
        const = math.fsum(logphi[x] for x in xs)
        lw = [math.fsum([logphi[v], k * lognorm[v], const] + terms[v]) for v in range(V)]
    else:
        kn = 0.0 if tab["is_const"] else k
        lw = [math.fsum([logphi[v], kn * lognorm[v]] + terms[v]) for v in range(V)]
    return normalise(lw)
