"""Posterior summaries of a linkage chain (host side; small inputs).

  most_probable_clusters / shared_most_probable_clusters  <- LinkageChain.scala:52-109
  pairwise_match_probabilities                            <- posterior probability that two records are one entity
  binder_clusters                                         <- the sample of least posterior expected Binder loss
  binder_search                                           <- single-record moves that lower the expected Binder loss
  vi_clusters                                             <- the sample of least posterior expected variation of
                                                             information
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
