"""Posterior summaries of a linkage chain (host side; small inputs).

  most_probable_clusters / shared_most_probable_clusters  <- LinkageChain.scala:52-109
  pairwise_match_probabilities                            <- posterior probability that two records are one entity
  binder_clusters                                         <- the sample of least posterior expected Binder loss
  binder_search                                           <- single-record moves that lower the expected Binder loss
  vi_clusters                                             <- the sample of least posterior expected variation of
                                                             information
  vi_search                                               <- single-record moves that lower the quantised expected
                                                             variation of information
  credible_ball                                           <- the samples within a VI or Binder radius of an estimate
  clerical_review                                         <- each record's and cluster's expected false and missed
                                                             links against an estimate, for a review queue
  entity_value_counts / entity_value_modes                <- the posterior of the entity values of an estimate's
                                                             clusters
  capture_histories                                       <- the sets of files each sample's clusters hold, and each
                                                             record's links into every file
  cluster_size_distribution / partition_sizes             <- LinkageChain.scala:118-154
  pairwise_metrics                                        <- analysis/PairwiseMetrics.scala:44-63,
                                                             BinaryClassificationMetrics.scala:23-37
  adjusted_rand_index                                     <- analysis/ClusteringMetrics.scala:41-74

A linkage chain is a list of samples; a sample is (iteration, {partition_id: [cluster, ...]}) with clusters as
collections of record ids (what linkage-chain.parquet stores, package.scala:94-96).
"""
import collections
import fractions
import itertools
import math


def clusters_of_sample(sample):
    for clusters in sample[1].values():
        for c in clusters:
            if len(c):
                yield frozenset(c)


def most_probable_clusters(chain):
    """record id -> (cluster, frequency): the cluster the record appears in most often along the chain
    (LinkageChain.scala:52-64; ties are broken by the reduce order there, by first occurrence here)."""
    n = len({s[0] for s in chain})
    freq = collections.Counter()
    order = {}
    for s in chain:
        for c in clusters_of_sample(s):
            freq[c] += 1.0 / n
            order.setdefault(c, len(order))
    best = {}
    for c, f in sorted(freq.items(), key=lambda kv: order[kv[0]]):
        for r in c:
            if r not in best or f > best[r][1]:
                best[r] = (c, f)
    return best


def shared_most_probable_clusters(chain_or_mpc):
    """Records grouped by their most probable cluster (LinkageChain.scala:75-95; the reference's stricter
    'shared' filter is commented out there, :88-94, and is not applied here either)."""
    mpc = chain_or_mpc if isinstance(chain_or_mpc, dict) else most_probable_clusters(chain_or_mpc)
    groups = collections.defaultdict(set)
    for r, (c, _) in mpc.items():
        groups[c].add(r)
    return [frozenset(v) for v in groups.values()]


def pairwise_match_probabilities(chain):
    """frozenset({id1, id2}) -> the fraction of samples in which the two records share a cluster, for every pair that
    shares one in at least one sample."""
    n = len({s[0] for s in chain})
    count = collections.Counter()
    for s in chain:
        for c in clusters_of_sample(s):
            for a, b in itertools.combinations(c, 2):
                count[frozenset((a, b))] += 1
    return {pair: k / n for pair, k in count.items()}


def pairwise_match_diagnostics(chains):
    """chains: K lists of samples, each sample the set of record pairs (frozensets) it puts in one cluster.  For every
    pair linked in some sample, its 0/1 draws, each chain cut to the shortest chain's n draws and split into halves
    [0, N) and [n - N, n), N = n // 2 -> (linked draws, least and largest per-chain count, max_t, split-R̂, ESS), by
    the definitions of Vehtari, Gelman, Simpson, Carpenter & Bürkner (2021) in exact fractions: biased autocovariances
    of each half, W = mean within-half variance, B / N = variance of the half means, var+ = (N - 1) / N W + B / N,
    R̂ = sqrt(var+ / W), rho[0] = 1 and rho[t] = 1 - (W - mean autocovariance at lag t) / var+, then Geyer's initial
    positive sequence, initial monotone sequence and truncated estimator, ESS = M N / max(tau, 1 / log10(M N))."""
    F = fractions.Fraction
    n = min(len(ch) for ch in chains)
    N, M = n // 2, 2 * len(chains)
    pairs = {p for ch in chains for s in ch for p in s}
    floor = 1.0 / math.log10(M * N)
    out = {}
    for pair in pairs:
        per_chain = [[int(pair in s) for s in ch[:n]] for ch in chains]
        halves = [x[:N] for x in per_chain] + [x[n - N:] for x in per_chain]
        means = [F(sum(h), N) for h in halves]
        acov = [[F(sum((h[t] - mu) * (h[t + tau] - mu) for t in range(N - tau)), N) for tau in range(N)]
                for h, mu in zip(halves, means)]
        W = sum(a[0] * F(N, N - 1) for a in acov) / M
        grand = sum(means) / M
        B_over_N = sum((mu - grand) ** 2 for mu in means) / (M - 1)
        var_plus = F(N - 1, N) * W + B_over_N
        count = sum(sum(h) for h in halves)
        chain_counts = [sum(x[:N]) + sum(x[n - N:]) for x in per_chain]
        if var_plus == 0:
            out[pair] = (count, min(chain_counts), max(chain_counts), 0, float("nan"), float("nan"))
            continue
        rhat = math.sqrt(var_plus / W) if W > 0 else float("inf")
        rho = [F(1)] + [1 - (W - sum(a[tau] for a in acov) / M) / var_plus for tau in range(1, N)]
        # Geyer's initial positive sequence
        rho_p = [F(0)] * N
        t = 0
        even, odd = rho[0], rho[1]
        rho_p[0], rho_p[1] = even, odd
        while t < N - 5 and even + odd > 0:
            t += 2
            even, odd = rho[t], rho[t + 1]
            if even + odd >= 0:
                rho_p[t], rho_p[t + 1] = even, odd
        max_t = t
        if even > 0:
            rho_p[max_t] = even
        # initial monotone sequence
        t = 2
        while t <= max_t - 2:
            if rho_p[t] + rho_p[t + 1] > rho_p[t - 2] + rho_p[t - 1]:
                rho_p[t] = rho_p[t + 1] = (rho_p[t - 2] + rho_p[t - 1]) / 2
            t += 2
        tau_hat = -1 + 2 * sum(rho_p[:max_t]) + rho_p[max_t]
        ess = float(F(M * N) / tau_hat) if tau_hat > floor else M * N / floor
        out[pair] = (count, min(chain_counts), max(chain_counts), max_t, rhat, ess)
    return out


def binder_clusters(chain, false_link_cost=0.5):
    """The sample of least posterior expected Binder loss, by the definition: a pair linked in the sample costs
    t (1 - p), a pair not linked costs (1 - t) p, summed over every pair of records, where t = false_link_cost and p
    = the fraction of samples linking the pair.  Exact rational arithmetic; ties go to the earliest sample.  Returns
    (position of the sample in the chain, its clusters as frozensets, every sample's loss as a float)."""
    t = fractions.Fraction(false_link_cost)
    S = len(chain)
    clusters = [list(clusters_of_sample(s)) for s in chain]
    records = sorted({r for cl in clusters for c in cl for r in c})
    linked = [{frozenset(p) for c in cl for p in itertools.combinations(c, 2)} for cl in clusters]
    count = collections.Counter(p for ls in linked for p in ls)
    losses = []
    for ls in linked:
        loss = fractions.Fraction(0)
        for a, b in itertools.combinations(records, 2):
            pair = frozenset((a, b))
            p = fractions.Fraction(count[pair], S)
            loss += t * (1 - p) if pair in ls else (1 - t) * p
        losses.append(loss)
    best = min(range(S), key=lambda s: (losses[s], s))
    return best, clusters[best], [float(x) for x in losses]


def binder_search(chain, false_link_cost, starts, max_rounds=1000, records=None):
    """Single-record moves from each start (a partition: clusters of ids) while they lower the posterior expected
    Binder loss, by the definition, in exact rational arithmetic, with t = false_link_cost rounded as
    analysis_arrays.search_cost rounds it.  `records` orders the record ids (a record's index is its position; default:
    sorted).  One round: every record takes its best move to ANY other cluster or, out of a cluster of two or more, to a
    singleton -- the least (change of loss, destination), a singleton counting as destination -1 and a cluster as its
    smallest record index -- and proposes it if it lowers the loss; a proposal is applied if it is the least (change,
    record index) among the proposals touching each cluster it touches (its source, and its destination unless that is
    a singleton).  Returns (position of the chosen start: least loss, ties to the earlier; per start a dict with the
    final clusters as frozensets, rounds = [(moves, change of linked pairs, change of count sum)], converged, n, K)."""
    from .analysis_arrays import search_cost

    t = fractions.Fraction(*search_cost(false_link_cost))
    S = len(chain)
    count = collections.Counter(p for s in chain for c in clusters_of_sample(s) for p in
                                (frozenset(q) for q in itertools.combinations(c, 2)))
    ids = sorted({r for s in chain for c in clusters_of_sample(s) for r in c}) if records is None else list(records)
    index = {r: k for k, r in enumerate(ids)}

    def pair_loss(i, j, linked):
        p = fractions.Fraction(count[frozenset((i, j))], S)
        return t * (1 - p) if linked else (1 - t) * p

    def counts(cluster_of):
        linked = [(i, j) for i, j in itertools.combinations(ids, 2) if cluster_of[i] == cluster_of[j]]
        return len(linked), sum(count[frozenset(q)] for q in linked)

    runs = []
    for start in starts:
        cluster_of = {r: frozenset(c) for c in start for r in c}
        rounds, converged = [], False
        while True:
            label = {c: min(index[r] for r in c) for c in set(cluster_of.values())}
            proposals = []
            for i in ids:
                A = cluster_of[i]
                dests = [(label[X], X) for X in set(cluster_of.values()) if X != A]
                if len(A) > 1:
                    dests.append((-1, None))
                best = None
                for dest, X in dests:
                    change = sum(pair_loss(i, j, j in (X or ())) - pair_loss(i, j, j in A) for j in ids if j != i)
                    if best is None or (change, dest) < best[:2]:
                        best = (change, dest, X)
                if best is not None and best[0] < 0:
                    proposals.append((best[0], index[i], i, A, best[2]))
            if not proposals:
                converged = True
                break
            if len(rounds) == max_rounds:
                break
            least = {}
            for change, k, i, A, X in proposals:
                for c in (A, X) if X is not None else (A,):
                    least[c] = min(least.get(c, (change, k)), (change, k))
            before = counts(cluster_of)
            new = dict(cluster_of)
            applied = 0
            for change, k, i, A, X in proposals:
                if all(least[c] == (change, k) for c in ((A, X) if X is not None else (A,))):
                    applied += 1
                    for r in A - {i}:
                        new[r] = A - {i}
                    joined = (X or frozenset()) | {i}
                    for r in joined:
                        new[r] = joined
            cluster_of = new
            after = counts(cluster_of)
            rounds.append((applied, after[0] - before[0], after[1] - before[1]))
        n, K = counts(cluster_of)
        runs.append(dict(clusters=set(cluster_of.values()), rounds=rounds, converged=converged, n=n, K=K,
                         loss=((1 - t) * sum(count.values()) + t * S * n - K) / S))
    return min(range(len(runs)), key=lambda k: (runs[k]["loss"], k)), runs


def vi_clusters(chain):
    """The sample of least posterior expected variation of information, by the definition: VI(c, c') = H(c) + H(c')
    - 2 I(c, c') in bits, with H(c) = - sum over clusters x of p log2 p, p = |x| / R, and I(c, c') = sum over the
    non-empty cells x ^ y of p_xy log2(p_xy / (p_x p_y)); the expected VI of a sample is the mean of its VI against
    every sample.  Floats; ties go to the earliest sample.  Returns (position of the sample in the chain, its clusters
    as frozensets, every sample's expected VI)."""
    S = len(chain)
    clusters = [list(clusters_of_sample(s)) for s in chain]
    R = len({r for cl in clusters for c in cl for r in c})

    def entropy(cl):
        return -sum(len(x) / R * math.log2(len(x) / R) for x in cl)

    def mutual_information(a, b):
        total = 0.0
        for x in a:
            for y in b:
                n = len(x & y)
                if n:
                    total += n / R * math.log2(n * R / (len(x) * len(y)))
        return total

    H = [entropy(cl) for cl in clusters]
    losses = [sum(H[t] + H[s] - 2 * mutual_information(clusters[t], clusters[s]) for s in range(S)) / S
              for t in range(S)]
    best = min(range(S), key=lambda s: (losses[s], s))
    return best, clusters[best], losses


def vi_search(chain, starts, max_rounds=1000, records=None):
    """Single-record moves from each start (a partition: clusters of ids) while they lower J_q, by the definition:
    J_q(c) = S sum over clusters X of F_q(|X|) - 2 sum over the samples s and the non-empty cells x ^ y (x of c, y of
    C_s) of F_q(|x ^ y|), F_q(n) = D_q[0] + ... + D_q[n - 1] with D_q = analysis_arrays.vi_search_table(R), in exact
    integers.  `records` orders the record ids (a record's index is its position; default: sorted).  One round: every
    record takes its best move to ANY other cluster or, out of a cluster of two or more, to a singleton -- the least
    (change of J_q, destination), the change recomputed from scratch as J_q(after) - J_q(before), a singleton counting
    as destination -1 and a cluster as its smallest record index -- and proposes it if it lowers J_q; a proposal is
    applied if it is the least (change, record index) among the proposals touching each cluster it touches.  Returns
    (position of the chosen start: least final J_q, ties to the earlier; per start a dict with the final clusters as
    frozensets, rounds = [(moves, clusters after the round, change of J_q)], converged, J0 and J)."""
    from .analysis_arrays import vi_search_table

    S = len(chain)
    samples = [list(clusters_of_sample(s)) for s in chain]
    ids = sorted({r for cl in samples for c in cl for r in c}) if records is None else list(records)
    index = {r: k for k, r in enumerate(ids)}
    F = [0]
    for d in vi_search_table(len(ids)).tolist():
        F.append(F[-1] + d)

    def J(parts):
        total = S * sum(F[len(x)] for x in parts)
        for cl in samples:
            total -= 2 * sum(F[len(x & y)] for x in parts for y in cl if x & y)
        return total

    runs = []
    for start in starts:
        parts = {frozenset(c) for c in start}
        rounds, converged, J0 = [], False, J(parts)
        while True:
            label = {c: min(index[r] for r in c) for c in parts}
            base = J(parts)
            proposals = []
            for i in ids:
                A = next(c for c in parts if i in c)
                dests = [(label[X], X) for X in parts if X != A] + ([(-1, None)] if len(A) > 1 else [])
                best = None
                for dest, X in dests:
                    moved = (parts - {A, X}) | ({A - {i}} if len(A) > 1 else set()) | {(X or frozenset()) | {i}}
                    change = J(moved) - base
                    if best is None or (change, dest) < best[:2]:
                        best = (change, dest, X)
                if best is not None and best[0] < 0:
                    proposals.append((best[0], index[i], i, A, best[2]))
            if not proposals:
                converged = True
                break
            if len(rounds) == max_rounds:
                break
            least = {}
            for change, k, i, A, X in proposals:
                for c in (A, X) if X is not None else (A,):
                    least[c] = min(least.get(c, (change, k)), (change, k))
            new = set(parts)
            applied = 0
            for change, k, i, A, X in proposals:
                if all(least[c] == (change, k) for c in ((A, X) if X is not None else (A,))):
                    applied += 1
                    new -= {A, X}
                    if len(A) > 1:
                        new.add(A - {i})
                    new.add((X or frozenset()) | {i})
            parts = new
            rounds.append((applied, len(parts), J(parts) - base))
        runs.append(dict(clusters=parts, rounds=rounds, converged=converged, J0=J0, J=J(parts)))
    return min(range(len(runs)), key=lambda k: (runs[k]["J"], k)), runs


def credible_ball(chain, center, level):
    """The credible ball around a partition `center` (clusters of ids), by the definitions (Wade and Ghahramani 2018):
    the distance of every sample from the center, VI(c, C_s) = H(c) + H(C_s) - 2 I(c, C_s) in bits as vi_clusters
    computes it, and the Binder distance, the record pairs one of them links and the other does not, by enumerating
    every pair; k = ceil(level S) with level the fraction its repr spells; the radius is the k-th smallest distance and
    the ball every sample within it.  The bounds are samples in the ball: vertical-upper the farthest from the center,
    horizontal-upper the farthest of those with the fewest clusters, horizontal-lower the farthest of those with the
    most clusters, each the earliest sample when several qualify; ties = how many qualify.  Entropies carry rounding, so
    VI distances within 1e-12 of each other count as equal (each is ranked as the smallest of its run of such values).
    Returns {"vi" | "binder": dict(distances, radius, in_ball, bounds = {bound: (sample position, ties)})}."""
    samples = [list(clusters_of_sample(s)) for s in chain]
    center = [frozenset(c) for c in center]
    S = len(samples)
    R = sum(len(c) for c in center)

    def entropy(cl):
        return -sum(len(x) / R * math.log2(len(x) / R) for x in cl)

    def mutual_information(a, b):
        return sum(len(x & y) / R * math.log2(len(x & y) * R / (len(x) * len(y))) for x in a for y in b if x & y)

    def pairs(cl):
        return {frozenset(p) for c in cl for p in itertools.combinations(c, 2)}

    k = math.ceil(fractions.Fraction(repr(float(level))) * S)
    num_clusters = [len(cl) for cl in samples]
    out = {}
    for name, dist in (("vi", lambda cl: entropy(center) + entropy(cl) - 2 * mutual_information(center, cl)),
                       ("binder", lambda cl: len(pairs(center) ^ pairs(cl)))):
        raw = [dist(cl) for cl in samples]
        d = list(raw)
        if name == "vi":
            for a, b in zip(sorted(range(S), key=lambda s: raw[s]), sorted(range(S), key=lambda s: raw[s])[1:]):
                if raw[b] - d[a] <= 1e-12:
                    d[b] = d[a]
        radius = sorted(d)[k - 1]
        ball = [s for s in range(S) if d[s] <= radius]
        farthest = lambda among: [s for s in among if d[s] == max(d[t] for t in among)]  # noqa: E731
        fewest = [s for s in ball if num_clusters[s] == min(num_clusters[t] for t in ball)]
        most = [s for s in ball if num_clusters[s] == max(num_clusters[t] for t in ball)]
        bounds = {bound: (tied[0], len(tied)) for bound, tied in (("vertical-upper", farthest(ball)),
                                                                   ("horizontal-upper", farthest(fewest)),
                                                                   ("horizontal-lower", farthest(most)))}
        out[name] = dict(distances=raw, radius=radius, in_ball=[d[s] <= radius for s in range(S)], bounds=bounds)
    return out


def clerical_review(chain, center, false_link_cost, records):
    """The clerical review of a point estimate by the definitions, with sets and Fractions: center = a list of sets of
    record ids (cluster k = center[k]), records = the record ids in index order (the tie rules go by index), t =
    false_link_cost, p(i, j) = the fraction of samples linking i and j.  Per record id i: W = the sum over the other
    records of the samples linking them to i, I = the same over its cluster, FL = the sum over its cluster's other
    records of 1 - p, ML = the sum over the records outside its cluster of p, A = the samples holding its cluster as
    a cluster, and its strongest outside partner (largest p > 0, ties to the smaller index; None) with its count.  Per
    cluster: size, probability (A / S), FL = half the members' FL, ML = the members' ML, loss = t FL + (1 - t) ML,
    weakest = the least p over its pairs (None for a singleton), strongest = (inside id, outside id, p) of largest
    p > 0, ties to the smaller inside then outside index (None).  Returns (records, clusters, review order: by loss
    highest first, ties to the smaller k)."""
    F = fractions.Fraction
    t, S = F(false_link_cost), len(chain)
    samples = [set(clusters_of_sample(s)) for s in chain]
    count = collections.Counter(frozenset(p) for cl in samples for c in cl for p in itertools.combinations(c, 2))
    index = {r: i for i, r in enumerate(records)}
    center = [frozenset(c) for c in center]
    cluster_of = {r: c for c in center for r in c}
    recs = {}
    for i in records:
        mine = cluster_of[i]
        n = {j: count[frozenset((i, j))] for j in records if j != i}
        outside = [(n[j], j) for j in records if j not in mine and n[j] > 0]
        best = min(outside, key=lambda x: (-x[0], index[x[1]])) if outside else (0, None)
        recs[i] = dict(W=sum(n.values()), I=sum(n[j] for j in mine if j != i),
                       FL=sum((1 - F(n[j], S) for j in mine if j != i), F(0)),
                       ML=sum((F(n[j], S) for j in records if j not in mine), F(0)),
                       A=sum(1 for cl in samples if mine in cl), partner=best[1], partner_count=best[0])
    clusters = []
    for c in center:
        fl, ml = sum(recs[i]["FL"] for i in c) / 2, sum(recs[i]["ML"] for i in c)
        links = [(count[frozenset((i, j))], i, j) for i in c for j in records
                 if j not in c and count[frozenset((i, j))] > 0]
        top = min(links, key=lambda x: (-x[0], index[x[1]], index[x[2]])) if links else None
        clusters.append(dict(size=len(c), probability=F(sum(1 for cl in samples if c in cl), S), FL=fl, ML=ml,
                             loss=t * fl + (1 - t) * ml,
                             weakest=min(F(count[frozenset(p)], S) for p in itertools.combinations(c, 2))
                             if len(c) > 1 else None,
                             strongest=None if top is None else (top[1], top[2], F(top[0], S))))
    order = sorted(range(len(center)), key=lambda k: (-clusters[k]["loss"], k))
    return recs, clusters, order


def cluster_size_distribution(chain):
    """iteration -> {cluster size: count} (LinkageChain.scala:137-154)."""
    out = {}
    for it, parts in chain:
        d = collections.Counter()
        for clusters in parts.values():
            for c in clusters:
                d[len(c)] += 1
        out[it] = dict(d)
    return out


def partition_sizes(chain):
    """iteration -> {partition id: number of clusters} (LinkageChain.scala:118-128)."""
    return {it: {p: len(cl) for p, cl in parts.items()} for it, parts in chain}


def to_pairwise_links(clusters):
    links = set()
    for c in clusters:
        for a, b in itertools.combinations(sorted(c), 2):
            links.add((a, b))
    return links


def pairwise_metrics(predicted_clusters, true_clusters):
    """precision / recall / F1 over record pairs (PairwiseMetrics.scala:44-63)."""
    pred, true = to_pairwise_links(predicted_clusters), to_pairwise_links(true_clusters)
    tp = len(pred & true)
    fp, fn = len(pred) - tp, len(true) - tp
    precision = tp / (tp + fp) if tp + fp else float("nan")
    recall = tp / (tp + fn) if tp + fn else float("nan")
    f1 = 2 * precision * recall / (precision + recall) if tp else (0.0 if (fp or fn) else float("nan"))
    return {"precision": precision, "recall": recall, "f1score": f1, "TP": tp, "FP": fp, "FN": fn}


def adjusted_rand_index(predicted_clusters, true_clusters):
    """ClusteringMetrics.AdjustedRandIndex (ClusteringMetrics.scala:44-74)."""
    comb2 = lambda x: x * (x - 1) // 2 if x >= 2 else 0  # noqa: E731
    pred_of, true_of = {}, {}
    for i, c in enumerate(predicted_clusters):
        for r in c:
            pred_of[r] = i
    for i, c in enumerate(true_clusters):
        for r in c:
            true_of[r] = i
    if set(pred_of) != set(true_of):
        raise ValueError("predicted and true clusterings must cover the same records")
    table = collections.Counter((pred_of[r], true_of[r]) for r in pred_of)
    pred_sum, true_sum = collections.Counter(), collections.Counter()
    for (p, t), n in table.items():
        pred_sum[p] += n
        true_sum[t] += n
    pc = sum(comb2(v) for v in pred_sum.values())
    tc = sum(comb2(v) for v in true_sum.values())
    total = sum(comb2(v) for v in table.values())
    expected = pc * tc / comb2(len(pred_of))
    max_index = (pc + tc) / 2.0
    return (total - expected) / (max_index - expected) if max_index != expected else 1.0


def membership_to_clusters(record_ids, membership):
    groups = collections.defaultdict(set)
    for r, m in zip(record_ids, membership):
        groups[m].add(r)
    return [frozenset(v) for v in groups.values()]


def format_pairwise(m):
    return ("=====================================\n        Pairwise metrics              \n"
            "-------------------------------------\n"
            f" Precision:      {m['precision']}\n Recall:         {m['recall']}\n F1-score:       {m['f1score']}\n"
            "=====================================\n")


def format_cluster(ari):
    return ("=====================================\n          Cluster metrics            \n"
            "-------------------------------------\n"
            f" Adj. Rand index: {ari}\n=====================================\n")


def _binder_estimate_line(iteration, chain, false_link_cost):
    return f" Estimate:        sample at iteration {iteration} of chain {chain}, falseLinkCost {false_link_cost}\n"


def format_binder_pairwise(m, iteration, chain, false_link_cost):
    """The binder-pairwise section: m = pairwise metrics of the sample chosen at (iteration, chain)."""
    return ("=====================================\n      Binder pairwise metrics\n"
            "-------------------------------------\n" + _binder_estimate_line(iteration, chain, false_link_cost)
            + f" Precision:      {m['precision']}\n Recall:         {m['recall']}\n F1-score:       {m['f1score']}\n"
            "=====================================\n")


def format_binder_cluster(ari, iteration, chain, false_link_cost):
    """The binder-cluster section: ari = adjusted Rand index of the sample chosen at (iteration, chain)."""
    return ("=====================================\n       Binder cluster metrics\n"
            "-------------------------------------\n" + _binder_estimate_line(iteration, chain, false_link_cost)
            + f" Adj. Rand index: {ari}\n=====================================\n")


def _binder_search_line(start, rounds, converged, false_link_cost, searched_cost):
    return (f" Estimate:        search from the {start} start, {rounds} rounds, "
            f"{'converged' if converged else 'not converged'}, falseLinkCost {false_link_cost} "
            f"(searched at {searched_cost!r})\n")


def format_binder_search_pairwise(m, start, rounds, converged, false_link_cost, searched_cost):
    """The binder-search-pairwise section: m = pairwise metrics of the search result chosen from `start`."""
    return ("=====================================\n   Binder search pairwise metrics\n"
            "-------------------------------------\n"
            + _binder_search_line(start, rounds, converged, false_link_cost, searched_cost)
            + f" Precision:      {m['precision']}\n Recall:         {m['recall']}\n F1-score:       {m['f1score']}\n"
            "=====================================\n")


def format_binder_search_cluster(ari, start, rounds, converged, false_link_cost, searched_cost):
    """The binder-search-cluster section: ari = adjusted Rand index of the search result chosen from `start`."""
    return ("=====================================\n    Binder search cluster metrics\n"
            "-------------------------------------\n"
            + _binder_search_line(start, rounds, converged, false_link_cost, searched_cost)
            + f" Adj. Rand index: {ari}\n=====================================\n")


def _vi_estimate_line(iteration, chain, expected_vi):
    return f" Estimate:        sample at iteration {iteration} of chain {chain}, expected VI {expected_vi!r}\n"


def format_vi_pairwise(m, iteration, chain, expected_vi):
    """The vi-pairwise section: m = pairwise metrics of the sample chosen at (iteration, chain)."""
    return ("=====================================\n        VI pairwise metrics\n"
            "-------------------------------------\n" + _vi_estimate_line(iteration, chain, expected_vi)
            + f" Precision:      {m['precision']}\n Recall:         {m['recall']}\n F1-score:       {m['f1score']}\n"
            "=====================================\n")


def format_vi_cluster(ari, iteration, chain, expected_vi):
    """The vi-cluster section: ari = adjusted Rand index of the sample chosen at (iteration, chain)."""
    return ("=====================================\n         VI cluster metrics\n"
            "-------------------------------------\n" + _vi_estimate_line(iteration, chain, expected_vi)
            + f" Adj. Rand index: {ari}\n=====================================\n")


def _vi_search_lines(start, rounds, converged, exact):
    return (f" Estimate:        search from the {start} start, {rounds} rounds, "
            f"{'converged' if converged else 'not converged'}\n"
            f" Expected VI:     vi-sample start {exact[0]!r}, smpc start {exact[1]!r}, from vi-sample {exact[2]!r}, "
            f"from smpc {exact[3]!r}\n")


def format_vi_search_pairwise(m, start, rounds, converged, exact):
    """The vi-search-pairwise section: m = pairwise metrics of the search result chosen from `start`; exact = the
    expected VI of the two starts and the two results (project.vi_search_estimate)."""
    return ("=====================================\n     VI search pairwise metrics\n"
            "-------------------------------------\n" + _vi_search_lines(start, rounds, converged, exact)
            + f" Precision:      {m['precision']}\n Recall:         {m['recall']}\n F1-score:       {m['f1score']}\n"
            "=====================================\n")


def format_vi_search_cluster(ari, start, rounds, converged, exact):
    """The vi-search-cluster section: ari = adjusted Rand index of the search result chosen from `start`."""
    return ("=====================================\n      VI search cluster metrics\n"
            "-------------------------------------\n" + _vi_search_lines(start, rounds, converged, exact)
            + f" Adj. Rand index: {ari}\n=====================================\n")


def format_credible_ball(res):
    """The credible-ball section: res = the center, the level, the samples and per distance the truth's distance from
    the center, the radius, whether the truth lies in the ball and the samples in it (project.py)."""
    def line(label, r, unit):
        where = "inside" if r["truthInBall"] else "outside"
        return (f" {label:<17}truth at {r['truthDistance']!r}{unit} from the center, radius {r['radius']!r}, {where} "
                f"the ball of {r['samplesInBall']} samples\n")

    return ("=====================================\n           Credible ball\n"
            "-------------------------------------\n"
            f" Center:          {res['center']}, level {res['level']!r}, {res['samples']} samples\n"
            + line("VI:", res["vi"], " bits") + line("Binder:", res["binder"], " pairs")
            + "=====================================\n")


def _posterior_line(label, s, extra=""):
    line = f" {label:<17}{s['mean']} (sd {s['sd']}, 95% interval [{s['q025']}, {s['q975']}], median {s['median']})"
    if s["undefined"]:
        line += f", undefined in {s['undefined']} samples"
    return line + extra + "\n"


def format_posterior_pairwise(summary, num_samples):
    """The posterior-pairwise section: summary = analysis_arrays.posterior_summary over num_samples samples."""
    return ("=====================================\n     Posterior pairwise metrics\n"
            "-------------------------------------\n"
            f" Samples:         {num_samples}\n" + _posterior_line("Precision:", summary["precision"])
            + _posterior_line("Recall:", summary["recall"]) + _posterior_line("F1-score:", summary["f1score"])
            + "=====================================\n")


def format_posterior_cluster(summary, num_samples, true_num_clusters):
    """The posterior-cluster section: summary = analysis_arrays.posterior_summary over num_samples samples."""
    return ("=====================================\n      Posterior cluster metrics\n"
            "-------------------------------------\n"
            f" Samples:         {num_samples}\n" + _posterior_line("Adj. Rand index:", summary["adjRandIndex"])
            + _posterior_line("Clusters:", summary["numClusters"], f" (true: {true_num_clusters})")
            + "=====================================\n")


def is_nan(x):
    return isinstance(x, float) and math.isnan(x)


def entity_value_counts(chain, values, center):
    """The entity-value counts of the point estimate `center` (a list of sets of record ids; cluster k = center[k]),
    restated with dicts: chain = [(iteration, {partition: [cluster of ids]})], values[s][a] = {frozenset of a cluster
    of sample s: the value of its entity for attribute a}.  Returns {(k, a, v): the number of (sample, record of
    center[k]) whose entity has value v}."""
    counts = collections.Counter()
    for (_, parts), vals in zip(chain, values):
        where = {r: frozenset(c) for cl in parts.values() for c in cl for r in c}
        for k, c in enumerate(center):
            for a, va in enumerate(vals):
                for r in c:
                    counts[(k, a, va[where[r]])] += 1
    return dict(counts)


def entity_value_modes(counts, num_clusters, num_attributes):
    """{(k, a): (mode, count)} from entity_value_counts: the value of largest count, ties to the smallest value."""
    out = {}
    for (k, a, v), n in counts.items():
        best = out.get((k, a))
        if best is None or n > best[1] or (n == best[1] and v < best[0]):
            out[(k, a)] = (v, n)
    assert len(out) == num_clusters * num_attributes
    return out


def capture_histories(chain, file, num_files):
    """The capture histories restated with sets and Python integers: chain = [(iteration, {partition: [cluster of
    ids]})], file = {record id: its file in [0, num_files)}.  Returns (H, L): H[s][h] = the clusters of sample s whose
    set of files, as the bits of h, is exactly h (H[s][0] = 0), and L = {record id: [the samples in which its cluster
    holds a record of file g other than itself, for g in files]}."""
    H, L = [], {r: [0] * num_files for r in file}
    for sample in chain:
        row = [0] * (1 << num_files)
        for c in clusters_of_sample(sample):
            files = {file[r] for r in c}
            row[sum(1 << f for f in files)] += 1
            for r in c:
                for g in {file[o] for o in c if o != r}:
                    L[r][g] += 1
        H.append(row)
    return H, L


def format_capture_histories(res, file_ids):
    """The capture-histories section: res = analysis_arrays.capture_evaluation's summary."""
    def interval(x):
        mean, _, lo, _, hi, inf = x
        return f"posterior mean {mean!r}, 95% interval [{lo!r}, {hi!r}]" + (f", infinite in {inf} samples" if inf
                                                                              else "")

    lines = (f" Samples:         {res['samples']}\n"
             f" Histories:       {res['histories_inside']} of {res['histories']} with the truth inside the 95% "
             f"interval\n"
             f" Quantities:      {res['quantities_inside']} of {res['quantities']} with the truth inside the 95% "
             f"interval\n"
             f" Observed:        truth {res['observed'][0]}, {interval(res['observed'][1])}\n")
    if "independence" in res:
        lines += f" Independence:    truth {res['independence'][0]!r}, {interval(res['independence'][1])}\n"
    lines += "".join(f" Brier [{f}]:{' ' * max(1, 8 - len(str(f)))}{b!r}\n" for f, b in zip(file_ids, res["brier"]))
    return ("=====================================\n         Capture histories\n"
            "-------------------------------------\n" + lines + "=====================================\n")


def format_clerical_review(res):
    """The clerical-review section: res = the center, the clusters, the erroneous ones, the shares of them found in the
    first 1 %, 5 % and 10 % of the review queue and of the queue by cluster probability, and the queue's normalised
    area under the found-curve (analysis_arrays.clerical_review_evaluation)."""
    def shares(x):
        return f"{x[0]!r} in the first 1%, {x[1]!r} in 5%, {x[2]!r} in 10%"

    return ("=====================================\n          Clerical review\n"
            "-------------------------------------\n"
            f" Center:          {res['center']}, {res['clusters']} clusters, {res['erroneous']} not a true entity\n"
            f" Review queue:    found {shares(res['found'])}, area {res['area']!r}\n"
            f" By probability:  found {shares(res['baseline'])}\n"
            "=====================================\n")


def query_link_probabilities(queries, samples, tables, constant, population_size):
    """The posterior predictive of new records, restated literally with dicts and Python floats for small chains.
    queries = [(file, {attribute: value id})] (missing attributes left out); samples = [(clusters, values, theta)]
    with clusters = lists of record indices, values[k] = the entity values of cluster k, theta[a][f]; tables[a] =
    AttributeIndex.tables() of attribute a.  Per sample, w(q, k) = prod over the observed a of (1 - theta) [x = y] +
    theta psi(x) norm(y) expsim(x, y) (expsim = 1 off x's row; norm = expsim = 1 when constant), m(q) = prod over the
    observed a of psi(x) ((1 - theta) + theta sigma(x)), sigma(x) = sum over y of psi(y) norm(y) expsim(x, y) (1 when
    constant), Z = sum_k w + (M - K) m.  Returns ({(q, r): p}, [p_new], [ESS]) over every pair, no threshold."""
    def expsim(a, x, y):
        t = tables[a]
        for j in range(t["rowptr"][x], t["rowptr"][x + 1]):
            if t["col"][j] == y:
                return float(t["expsim"][j])
        return 1.0

    def norm(a, y):
        return 1.0 if constant[a] else float(tables[a]["norm"][y])

    def sigma(a, x):
        if constant[a]:
            return 1.0
        return sum(float(tables[a]["phi"][y]) * norm(a, y) * expsim(a, x, y) for y in range(len(tables[a]["phi"])))

    M = population_size
    num, den, den2, new = {}, [0.0] * len(queries), [0.0] * len(queries), [0.0] * len(queries)
    for clusters, values, theta in samples:
        K = len(clusters)
        for q, (f, obs) in enumerate(queries):
            w = []
            for k in range(K):
                wk = 1.0
                for a, x in obs.items():
                    th, y = float(theta[a][f]), int(values[k][a])
                    wk *= (1.0 - th) * (1.0 if x == y else 0.0) + th * float(tables[a]["phi"][x]) * norm(a, y) * \
                        expsim(a, x, y)
                w.append(wk)
            m = 1.0
            for a, x in obs.items():
                th = float(theta[a][f])
                m *= float(tables[a]["phi"][x]) * ((1.0 - th) + th * sigma(a, x))
            Z = sum(w) + (M - K) * m
            for k, members in enumerate(clusters):
                for r in members:
                    num[(q, r)] = num.get((q, r), 0.0) + w[k]
            den[q] += Z
            den2[q] += Z * Z
            new[q] += (M - K) * m
    p = {key: v / den[key[0]] for key, v in num.items()}
    return p, [new[q] / den[q] for q in range(len(queries))], [den[q] ** 2 / den2[q] for q in range(len(queries))]
