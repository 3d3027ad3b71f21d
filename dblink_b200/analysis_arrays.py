"""Posterior summaries on arrays (no Python loop over clusters or records): the same quantities as analysis.py --
LinkageChain.scala:52-154 and analysis/{PairwiseMetrics,ClusteringMetrics}.scala -- for chains of millions of records.

A sample is held as (members, offsets, partition_of_cluster): `members` = record INDICES (positions in the id
dictionary) of all clusters back to back, `offsets[c]:offsets[c+1]` = cluster c.  The simple set-based functions in
analysis.py stay as the readable restatement; tests compare the two on random chains.
"""
import math
import os

import numpy as np


# ---- reading the chain -------------------------------------------------------------------------------
class ChainArrays:
    def __init__(self, record_ids, iterations, samples, chains=None):
        self.record_ids = record_ids  # pyarrow string array: index -> record id
        self.iterations = iterations  # int64[S], ascending
        self.samples = samples        # list of (members int32[n], offsets int64[nc+1], partition int32[nc])
        # int64[S]: the chain each sample comes from (all 0 unless read_pooled_chain_arrays pooled several)
        self.chains = np.zeros(len(samples), np.int64) if chains is None else np.asarray(chains, np.int64)

    @property
    def num_records(self):
        return len(self.record_ids)


def read_chain_arrays(path, lower_iteration_cutoff=0):
    """linkage-chain.parquet (hive-partitioned by partitionId) -> ChainArrays, through Arrow only."""
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyarrow.parquet as pq

    rows = {}  # iteration -> list of (pid, ListArray of clusters)
    for d in sorted(os.listdir(path)):
        if not d.startswith("partitionId="):
            continue
        pid = int(d.split("=")[1])
        for f in sorted(os.listdir(os.path.join(path, d))):
            t = pq.ParquetFile(os.path.join(path, d, f)).read()
            its = t.column("iteration").to_numpy()
            ls = t.column("linkageStructure").combine_chunks()
            for i, it in enumerate(its):
                if it >= lower_iteration_cutoff:
                    rows.setdefault(int(it), []).append((pid, ls[i].values))  # list<string> of that row
    its = sorted(rows)
    if not its:
        return ChainArrays(pa.array([], pa.string()), np.zeros(0, np.int64), [])
    first = pa.concat_arrays([cl.flatten() for _, cl in rows[its[0]]])
    ids = pc.unique(first)
    samples = []
    for it in its:
        # one id lookup per sample over all its partitions: each index_in call hashes the R ids of the value set
        idx = pc.index_in(pa.concat_arrays([cl.flatten() for _, cl in rows[it]]), value_set=ids)
        if idx.null_count:
            raise ValueError("a sample mentions a record id that the first sample does not")
        mem = [idx.to_numpy(zero_copy_only=False).astype(np.int32)]
        sizes, part = [], []
        for pid, cl in rows[it]:
            off = cl.offsets.to_numpy().astype(np.int64)
            sz = np.diff(off)
            sizes.append(sz)
            part.append(np.full(len(sz), pid, np.int32))
        sizes = np.concatenate(sizes) if sizes else np.zeros(0, np.int64)
        keep = sizes > 0
        samples.append((np.concatenate(mem) if mem else np.zeros(0, np.int32),
                        np.r_[0, np.cumsum(sizes[keep])].astype(np.int64),
                        (np.concatenate(part) if part else np.zeros(0, np.int32))[keep]))
    return ChainArrays(ids, np.asarray(its, np.int64), samples)


def read_pooled_chain_arrays(paths, lower_iteration_cutoff=0):
    """The samples of several chains (one linkage-chain.parquet each) at or after the cutoff, pooled into ONE
    ChainArrays: chain-major, then by iteration (the order that defines the sMPC tie rule "earliest sample").  Every
    chain's ids are mapped through the first chain's record-id dictionary; chains that mention different records are
    refused.  `iterations` is then ascending within each chain only; `chains` gives each sample's chain (its position
    in `paths`)."""
    import pyarrow as pa
    import pyarrow.compute as pc

    chains = [read_chain_arrays(p, lower_iteration_cutoff) for p in paths]
    if not chains:
        raise ValueError("no chains to pool")
    ids = chains[0].record_ids
    its, samples, which = [], [], []
    for k, ch in enumerate(chains):
        if len(ch.record_ids) != len(ids):
            raise ValueError("the chains mention different records")
        pos = pc.index_in(ch.record_ids, value_set=ids)
        if pos.null_count:
            raise ValueError("the chains mention different records")
        remap = pos.to_numpy(zero_copy_only=False).astype(np.int32)
        for mem, off, part in ch.samples:
            samples.append((remap[mem], off, part))
        its.append(ch.iterations)
        which.append(np.full(len(ch.samples), k, np.int64))
    return ChainArrays(ids if len(ids) else pa.array([], pa.string()),
                       np.concatenate(its) if its else np.zeros(0, np.int64), samples, np.concatenate(which))


def sample_from_links(link, block_of_entity):
    """One sample straight from the engine's arrays (record index = position): (members, offsets, partition)."""
    link = np.asarray(link)
    order = np.argsort(link, kind="stable").astype(np.int32)
    sl = link[order]
    start = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]]) if len(sl) else np.zeros(0, np.int64)
    return order, np.r_[start, len(sl)].astype(np.int64), np.asarray(block_of_entity)[sl[start]].astype(np.int32)


# ---- LinkageChain.scala:118-154 ----------------------------------------------------------------------
def cluster_size_distribution(chain):
    """iteration -> {cluster size: count}."""
    out = {}
    for it, (_, off, _) in zip(chain.iterations, chain.samples):
        sz = np.diff(off)
        cnt = np.bincount(sz)
        out[int(it)] = {int(k): int(cnt[k]) for k in np.flatnonzero(cnt)}
    return out


def partition_sizes(chain):
    """iteration -> {partition id: number of clusters}."""
    out = {}
    for it, (_, _, part) in zip(chain.iterations, chain.samples):
        p, n = np.unique(part, return_counts=True)
        out[int(it)] = {int(a): int(b) for a, b in zip(p, n)}
    return out


# ---- most probable clusters (LinkageChain.scala:52-109) ------------------------------------------------
def _mix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = (x + np.uint64(0x9E3779B97F4A7C15))
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def cluster_signatures(chain):
    """uint64[S, R]: for every sample and record, a 64-bit signature of the SET of records it is clustered with
    (sum of mixed member indices, mixed with the size); equal sets <=> equal signatures up to 2^-64 collisions."""
    R = chain.num_records
    mix = _mix64(np.arange(R, dtype=np.uint64))
    sig = np.zeros((len(chain.samples), R), np.uint64)
    for s, (mem, off, _) in enumerate(chain.samples):
        if len(mem) != R:
            raise ValueError("every sample must mention every record exactly once")
        sizes = np.diff(off)
        with np.errstate(over="ignore"):
            h = np.add.reduceat(mix[mem], off[:-1]) if len(sizes) else np.zeros(0, np.uint64)
            h = _mix64(h ^ _mix64(sizes.astype(np.uint64)))
        sig[s, mem] = np.repeat(h, sizes)
    return sig


def most_probable_signature(sig, block=65536):
    """For every record the signature it carries most often along the chain (ties: the one seen first) and its
    frequency: (uint64[R], float64[R]).  Works on blocks of records to bound memory."""
    S, R = sig.shape
    best = np.zeros(R, np.uint64)
    freq = np.zeros(R)
    for lo in range(0, R, block):
        a = sig[:, lo:lo + block]
        n = a.shape[1]
        order = np.argsort(a, axis=0, kind="stable")       # equal signatures keep ascending sample order
        srt = np.take_along_axis(a, order, 0).T.reshape(-1)  # record-major: the S signatures of a record are adjacent
        first_sample = order.T.reshape(-1)
        new = np.ones(n * S, bool)
        new[1:] = srt[1:] != srt[:-1]
        new[::S] = True                                      # a run never crosses records
        run_start = np.flatnonzero(new)
        count = np.diff(np.r_[run_start, n * S])
        # winner per record: larger count first, then the earlier first sample (a lexicographic sort of the runs; a
        # packed integer key would overflow int64 for chains of ~50k samples)
        rec_of_run = run_start // S
        by = np.lexsort((first_sample[run_start], -count, rec_of_run))
        lead = np.ones(len(by), bool)
        lead[1:] = rec_of_run[by][1:] != rec_of_run[by][:-1]
        win = by[lead]                                       # one run per record, in record order
        best[lo:lo + n] = srt[run_start[win]]
        freq[lo:lo + n] = count[win] / S
    return best, freq


def shared_most_probable_clusters(chain):
    """Records grouped by their most probable cluster: int32 labels[R] (records with equal labels form a cluster),
    labelled by the smallest record index of the group."""
    sig = cluster_signatures(chain)
    best, _ = most_probable_signature(sig)
    return canonical_labels(best)


def canonical_labels(keys):
    """int64 labels[R]: records with equal keys grouped, each group labelled by its smallest record index."""
    _, inv = np.unique(keys, return_inverse=True)
    inv = inv.reshape(-1)
    rep = np.full(inv.max() + 1 if len(inv) else 0, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(rep, inv, np.arange(len(inv)))
    return rep[inv].astype(np.int64)


# ---- posterior pairwise match probabilities ------------------------------------------------------------
MAX_PAIRS = 1 << 28  # distinct record pairs a chain may put in a cluster (the GPU table: 12 bytes each, twice)


def too_many_pairs(max_pairs):
    return ValueError(f"the chain puts more than {max_pairs} distinct record pairs in a cluster")


def min_match_count(threshold, num_samples):
    """The smallest count c >= 1 with c / S >= threshold in float64, so that a pair is kept exactly when its
    probability count / S is at least the threshold (threshold in [0, 1])."""
    S = int(num_samples)
    if S <= 0:
        return 1
    c = max(1, min(S, math.ceil(threshold * S)))
    while c > 1 and (c - 1) / S >= threshold:
        c -= 1
    while c < S and c / S < threshold:
        c += 1
    return c


def sample_pair_keys(num_records, members, offsets):
    """Sorted int64 keys first << 32 | second (record indices, first < second) of the pairs of records that share a
    cluster in one sample.  The record at position t of a cluster of k records (members in ascending index) is paired
    with positions t+1 .. k-1: one row per record, generated without a loop over clusters."""
    members = np.asarray(members)
    sizes = np.diff(offsets).astype(np.int64)
    n = len(members)
    cl = np.repeat(np.arange(len(sizes), dtype=np.int64), sizes)
    srt = np.sort(cl * num_records + members) - cl * num_records  # members of a cluster in ascending index
    row = np.repeat(np.asarray(offsets[:-1], np.int64) + sizes, sizes) - 1 - np.arange(n)
    row_off = np.r_[0, np.cumsum(row)]
    shift = np.repeat(row_off[:-1] - np.arange(n) - 1, row)  # partner position = output index - shift
    return np.sort((np.repeat(srt, row) << 32) | srt[np.arange(row_off[-1]) - shift])


def pairwise_match_counts(chain, max_pairs=MAX_PAIRS, min_count=1):
    """(first, second, count), int64: every pair of record indices (first < second, ascending (first, second) order)
    that shares a cluster in at least min_count samples, and the number of samples in which it does.  The probability
    that the two records are one entity is count / S.  Raises ValueError when the chain puts more than max_pairs
    distinct pairs in a cluster; each sample's sum k(k-1)/2 is checked before its pairs are generated."""
    R = chain.num_records
    keys, cnt = np.zeros(0, np.int64), np.zeros(0, np.int64)
    for mem, off, _ in chain.samples:
        if len(mem) != R:
            raise ValueError("every sample must mention every record exactly once")
        if int(_comb2(np.diff(off)).sum()) > max_pairs:
            raise too_many_pairs(max_pairs)
        k = sample_pair_keys(R, mem, off)
        pos = np.searchsorted(keys, k)
        hit = np.zeros(len(k), bool)
        inside = pos < len(keys)
        hit[inside] = keys[pos[inside]] == k[inside]
        new = ~hit
        if len(keys) + int(new.sum()) > max_pairs:
            raise too_many_pairs(max_pairs)
        cnt[pos[hit]] += 1  # a sample's keys are distinct, so are their positions
        keys = np.insert(keys, pos[new], k[new])
        cnt = np.insert(cnt, pos[new], 1)
    keep = cnt >= min_count
    keys, cnt = keys[keep], cnt[keep]
    return keys >> 32, keys & 0xFFFFFFFF, cnt


def sample_labels(num_records, members, offsets):
    """int64 labels[R] of one sample: every record labelled by the smallest record index of its cluster, as the sMPC
    labels its groups (so labels_to_clusters orders both the same way)."""
    members = np.asarray(members)
    offsets = np.asarray(offsets, np.int64)
    sizes = np.diff(offsets)
    if len(members) != num_records or (sizes <= 0).any():
        raise ValueError("every sample must mention every record exactly once")
    labels = np.full(num_records, -1, np.int64)
    if num_records:
        labels[members] = np.repeat(np.minimum.reduceat(members, offsets[:-1]), sizes)
    if (labels < 0).any():
        raise ValueError("every sample must mention every record exactly once")
    return labels


# ---- the Binder-loss point estimate ---------------------------------------------------------------------
# With count(i, j) = the samples in which records i and j share a cluster (p_ij = count / S) and t = the cost of a
# false link (1 - t that of a missed link), the posterior expected Binder loss of a partition c is
#   E[L(c)] = sum over pairs linked in c of t (1 - p_ij) + sum over pairs not linked in c of (1 - t) p_ij
#           = ((1 - t) C + t S n(c) - K(c)) / S
# where n(c) = the pairs c links, K(c) = the sum of count over them and C = the sum of all counts = sum of n over the
# samples.  The estimate is the sample of least E[L] (Dahl's least-squares clustering at t = 1/2).

def binder_counts(chain, max_pairs=MAX_PAIRS):
    """(n, K), int64[S]: per sample the record pairs it puts together and the sum of their match counts over the
    chain.  Raises ValueError as pairwise_match_counts does when the chain has more than max_pairs distinct pairs."""
    first, second, count = pairwise_match_counts(chain, max_pairs)
    keys = (first << 32) | second
    S = len(chain.samples)
    n, K = np.zeros(S, np.int64), np.zeros(S, np.int64)
    for s, (mem, off, _) in enumerate(chain.samples):
        k = sample_pair_keys(chain.num_records, mem, off)
        pos = np.minimum(np.searchsorted(keys, k), max(len(keys) - 1, 0))
        hit = keys[pos] == k if len(keys) else np.zeros(len(k), bool)
        n[s], K[s] = len(k), int(count[pos[hit]].sum())
    return n, K


def binder_losses(n, K, false_link_cost):
    """float64[S]: the posterior expected Binder loss ((1 - t) C + t S n - K) / S of every sample, t = false_link_cost,
    C = sum of n."""
    n = np.asarray(n, np.int64)
    return expected_losses(n, K, int(n.sum()), len(n), false_link_cost)


def expected_losses(n, K, C, S, false_link_cost):
    """float64[]: the posterior expected Binder loss ((1 - t) C + t S n - K) / S of partitions with linked pairs n and
    count sums K, against a chain of S samples whose counts sum to C."""
    n, K, t = np.asarray(n, np.int64), np.asarray(K, np.int64), float(false_link_cost)
    return ((1.0 - t) * C + t * S * n.astype(np.float64) - K.astype(np.float64)) / S


def binder_estimate(n, K, false_link_cost):
    """The position of the sample of least expected Binder loss, ties going to the earliest.  t is a binary fraction
    a / b, so the losses are compared exactly, as the integers a S n - b K (the rest of S E[L] b is the same for every
    sample): two samples of equal loss tie whatever the rounding of binder_losses."""
    a, b = float(false_link_cost).as_integer_ratio()
    S = len(n)
    if S == 0:
        raise ValueError("the Binder-loss estimate needs at least one sample")
    score = [a * S * int(x) - b * int(y) for x, y in zip(n, K)]
    return min(range(S), key=lambda s: (score[s], s))


# ---- a search beyond the samples: parallel single-record moves ---------------------------------------------
# With t = a / b, S b E[L](c) = (b - a) C + J(c), J(c) = a S n(c) - b K(c).  Moving record i from its cluster A to a
# cluster B changes J by  dJ = a S (|B| - |A| + 1) - b (w_B - w_A),  w_X = sum of count(i, j) over j in X \ {i}; a new
# singleton is |B| = 0, w_B = 0.  A cluster holding none of i's partners is never better than the singleton, so the
# candidates are the clusters of i's partners in the table and, when |A| > 1, a singleton.  One round:
#   1. labels are canonical (smallest record index of the cluster);
#   2. every record finds its least (dJ, destination), a singleton counting as destination -1, and proposes it if
#      dJ < 0;
#   3. a proposal touches its source cluster and, unless it goes to a singleton, its destination cluster; it is applied
#      only if it has the least (dJ, i) among the proposals touching each cluster it touches.  Applied moves touch
#      disjoint clusters, so their dJ add exactly, and the least proposal always wins, so J falls every round;
#   4. relabel; log the moves and the sums of dn and dK.
# The search stops when no record proposes a move (converged) or after max_rounds rounds.
SEARCH_COST_BITS = 16          # t is rounded to a multiple of 2^-16 for the search, so a, b <= 2^16
MAX_SEARCH_SIZE = 1 << 44      # S R below this keeps every dJ and every round's sum of dJ inside int64
SEARCH_STARTS = ("binder-sample", "smpc")


def search_cost(false_link_cost):
    """(a, b): t rounded to the nearest multiple of 2^-16 (halves up) as a / b, b = 2^16.  Exact for 0, 1/4, 1/2, 3/4
    and 1; 0.7 becomes 45875 / 65536."""
    t = float(false_link_cost)
    if not 0.0 <= t <= 1.0:
        raise ValueError("falseLinkCost must be in [0, 1].")
    b = 1 << SEARCH_COST_BITS
    return int(math.floor(t * b + 0.5)), b


def check_search_size(num_samples, num_records):
    if int(num_samples) * int(num_records) >= MAX_SEARCH_SIZE:
        raise ValueError(f"the Binder search needs samples x records < 2^44 (here {num_samples} x {num_records})")


class SearchRun:
    """One search: labels int64[R] (canonical) where it stopped; per round the moves applied and the sums of dn and
    dK, int64[rounds]; whether it stopped because no record proposed a move; n and K of the result."""

    def __init__(self, labels, moves, dn, dK, converged, n, K):
        self.labels, self.converged, self.n, self.K = labels, bool(converged), int(n), int(K)
        self.moves, self.dn, self.dK = (np.asarray(x, np.int64) for x in (moves, dn, dK))

    @property
    def rounds(self):
        return len(self.moves)

    def linked_pairs(self):
        """int64[rounds + 1]: n of the start (round 0) and after every round."""
        return self.n - int(self.dn.sum()) + np.r_[0, np.cumsum(self.dn)].astype(np.int64)

    def count_sums(self):
        """int64[rounds + 1]: K of the start (round 0) and after every round."""
        return self.K - int(self.dK.sum()) + np.r_[0, np.cumsum(self.dK)].astype(np.int64)


def search_result_counts(first, second, count, labels):
    """(n, K) of a labelling: n from its cluster sizes, K = the counts of the held pairs whose records share a label."""
    labels = np.asarray(labels, np.int64)
    n = int(_comb2(np.bincount(labels)).sum()) if len(labels) else 0
    return n, int(np.asarray(count, np.int64)[labels[first] == labels[second]].sum())


def _run_starts(sorted_keys):
    """Positions where a run of equal values starts."""
    return np.flatnonzero(np.r_[True, sorted_keys[1:] != sorted_keys[:-1]]) if len(sorted_keys) else np.zeros(0, np.int64)


def search_rounds(num_records, first, second, count, num_samples, start, a, b, max_rounds):
    """The search from labels start[R] against the table (first, second, count) of a chain of num_samples samples,
    t = a / b: a SearchRun."""
    R, S = int(num_records), int(num_samples)
    first, second, count = (np.asarray(x, np.int64) for x in (first, second, count))
    src, dst, cnt = np.r_[first, second], np.r_[second, first], np.r_[count, count]
    if np.shape(start) != (R,):
        raise ValueError("a start needs one cluster label per record")
    lab = canonical_labels(np.asarray(start, np.int64))
    aS, big = a * S, np.iinfo(np.int64).max
    moves, dn, dK, converged = [], [], [], False
    while True:
        size = np.bincount(lab, minlength=R).astype(np.int64)
        # the sum of count per (record, partner label), in ascending (record, label) order
        keys = src * R + lab[dst]
        order = np.argsort(keys)
        keys = keys[order]
        runs = _run_starts(keys)
        keys, w = keys[runs], np.add.reduceat(cnt[order], runs) if len(runs) else np.zeros(0, np.int64)
        rec, X = keys // R, keys % R
        own = X == lab[rec]
        wA = np.zeros(R, np.int64)
        wA[rec[own]] = w[own]
        # candidates in ascending (record, destination) order: a record's singleton first, then its partner clusters
        multi = np.flatnonzero(size[lab] > 1)
        by = np.argsort(np.r_[2 * multi, 2 * rec[~own] + 1], kind="stable")
        c_rec = np.r_[multi, rec[~own]][by]
        c_dest = np.r_[np.full(len(multi), -1, np.int64), X[~own]][by]
        c_dK = np.r_[-wA[multi], w[~own] - wA[rec[~own]]][by]
        c_dn = np.where(c_dest >= 0, size[np.maximum(c_dest, 0)], 0) - size[lab[c_rec]] + 1
        c_dJ = aS * c_dn - b * c_dK
        # per record the first candidate of least dJ: the least (dJ, destination)
        seg = _run_starts(c_rec)
        least = np.repeat(np.minimum.reduceat(c_dJ, seg), np.diff(np.r_[seg, len(c_rec)])) if len(seg) else c_dJ
        at = np.flatnonzero(c_dJ == least)
        best = at[_run_starts(c_rec[at])]
        best = best[c_dJ[best] < 0]
        if not len(best):
            converged = True
            break
        if len(moves) == max_rounds:
            break
        i, X, dJ = c_rec[best], c_dest[best], c_dJ[best]
        A, to = lab[i], X >= 0
        touched, t_dJ, t_i = np.r_[A, X[to]], np.r_[dJ, dJ[to]], np.r_[i, i[to]]
        claim_dJ = np.full(R, big, np.int64)
        np.minimum.at(claim_dJ, touched, t_dJ)
        least = t_dJ == claim_dJ[touched]
        claim_i = np.full(R, big, np.int64)
        np.minimum.at(claim_i, touched[least], t_i[least])
        win = (claim_dJ[A] == dJ) & (claim_i[A] == i)
        win[to] &= (claim_dJ[X[to]] == dJ[to]) & (claim_i[X[to]] == i[to])
        key = lab.copy()
        key[i[win]] = np.where(to[win], X[win], R + i[win])
        moves.append(int(win.sum()))
        dn.append(int(c_dn[best][win].sum()))
        dK.append(int(c_dK[best][win].sum()))
        lab = canonical_labels(key)
    n, K = search_result_counts(first, second, count, lab)
    return SearchRun(lab, moves, dn, dK, converged, n, K)


def search_choice(runs, num_samples, a, b):
    """The position of the run of least J = a S n - b K, ties going to the earlier start."""
    return min(range(len(runs)), key=lambda k: (a * num_samples * runs[k].n - b * runs[k].K, k))


def binder_search(chain, false_link_cost, starts, max_rounds=1000, max_pairs=MAX_PAIRS):
    """The search from each of starts (labels[R] each) against the chain's pairwise match counts, with t rounded by
    search_cost: (the position of the chosen run, the SearchRuns)."""
    R, S = chain.num_records, len(chain.samples)
    check_search_size(S, R)
    a, b = search_cost(false_link_cost)
    first, second, count = pairwise_match_counts(chain, max_pairs)
    runs = [search_rounds(R, first, second, count, S, st, a, b, max_rounds) for st in starts]
    return search_choice(runs, S, a, b), runs


# ---- the variation-of-information point estimate -----------------------------------------------------------
# With A(c) = sum over the blocks of c of n log2 n, the variation of information of two partitions of R records is
#   VI(c, c') = (A(c) + A(c') - 2 A(c ^ c')) / R,   c ^ c' = the non-empty cells (cluster of c, cluster of c'),
# and the posterior expected VI of sample t against the S samples is E_t = (1/S) sum_s VI(C_t, C_s).  In integers:
#   g_s[n] = the clusters of n records in sample s,  G_t[n] = sum over s != t of the cells of n records in C_t ^ C_s,
#   D_t[n] = (S - 2) g_t[n] + sum_s g_s[n] - 2 G_t[n],  E_t = sum over n >= 2 of D_t[n] n log2 n / (R S)
# (n log2 n is 0 at n = 0, 1, so those entries stay 0).  The estimate is the sample of least E_t, ties going to the
# earliest.  A cell is never larger than its clusters, so every histogram has width M + 1, M = the largest cluster.
MAX_VI_ENTRIES = 1 << 28  # S x (M + 1) histogram entries (the GPU's int64 matrix: 2 GB at the cap)


def vi_width(chain):
    """M + 1, M = the largest cluster of any sample of the chain (1 without records); ValueError when the S x (M + 1)
    histograms would exceed MAX_VI_ENTRIES."""
    S = len(chain.samples)
    M = max((int(np.diff(off).max()) for _, off, _ in chain.samples if len(off) > 1), default=0)
    if S * (M + 1) > MAX_VI_ENTRIES:
        raise ValueError(f"the VI histograms need {S} x {M + 1} entries, more than {MAX_VI_ENTRIES}")
    return M + 1


def vi_cluster_histograms(chain, width):
    """g, int64[S, width]: per sample the number of clusters of each size n >= 2 (entries 0 and 1 are 0)."""
    g = np.zeros((len(chain.samples), width), np.int64)
    for s, (_, off, _) in enumerate(chain.samples):
        g[s] = np.bincount(np.diff(off), minlength=width)[:width]
    g[:, :2] = 0
    return g


def vi_cross_histograms(chain):
    """G, int64[S, M + 1]: per sample t and cell size n >= 2, the number of cells of n records in C_t ^ C_s summed
    over the samples s != t.  Each pair t < s is counted once and added to both rows; only the records in clusters of
    two or more of C_t can be in a cell of two or more.  ValueError as vi_width raises it."""
    R, S = chain.num_records, len(chain.samples)
    width = vi_width(chain)
    G = np.zeros((S, width), np.int64)
    labels = [sample_labels(R, mem, off) for mem, off, _ in chain.samples]
    for t in range(S):
        big = np.flatnonzero(np.bincount(labels[t], minlength=R)[labels[t]] >= 2)
        if not len(big):
            continue
        hi = labels[t][big] * R
        for s in range(t + 1, S):
            _, n = np.unique(hi + labels[s][big], return_counts=True)
            h = np.bincount(n[n >= 2], minlength=width)
            G[t] += h
            G[s] += h
    return G


def vi_losses(g, G, num_records):
    """float64[S]: the posterior expected VI of every sample, from the cluster histograms g and the cell histograms G
    (int64[S, width] each): E_t = fsum over n >= 2 of float(D_t[n]) (n log2 n), divided by R S.  fsum is correctly
    rounded and does not depend on the order, so equal integers give equal losses."""
    g, G = np.asarray(g, np.int64), np.asarray(G, np.int64)
    S, width = G.shape
    if num_records == 0:
        return np.zeros(S)
    D = (S - 2) * g + g.sum(axis=0) - 2 * G
    weight = np.array([0.0, 0.0] + [n * math.log2(n) for n in range(2, width)])[:width]
    out = np.zeros(S)
    for t in range(S):
        nz = np.flatnonzero(D[t])
        out[t] = math.fsum(D[t, nz].astype(np.float64) * weight[nz]) / (num_records * S)
    return out


def vi_estimate(losses):
    """The position of the sample of least expected VI, ties going to the earliest."""
    if len(losses) == 0:
        raise ValueError("the VI estimate needs at least one sample")
    return min(range(len(losses)), key=lambda s: (losses[s], s))


def labels_to_clusters(labels, record_ids=None):
    """labels -> list of clusters (arrays of record indices, or lists of ids when record_ids is given)."""
    order = np.argsort(labels, kind="stable")
    sl = np.asarray(labels)[order]
    start = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]]) if len(sl) else np.zeros(0, np.int64)
    groups = np.split(order, start[1:])
    if record_ids is None:
        return groups
    ids = np.asarray(record_ids.to_pylist() if hasattr(record_ids, "to_pylist") else record_ids, dtype=object)
    return [list(ids[g]) for g in groups]


# ---- metrics (PairwiseMetrics.scala:44-63, ClusteringMetrics.scala:44-74) ------------------------------
def _comb2(x):
    x = np.asarray(x, np.int64)
    return x * (x - 1) // 2


def contingency(pred_labels, true_labels):
    _, p = np.unique(pred_labels, return_inverse=True)
    _, t = np.unique(true_labels, return_inverse=True)
    nt = int(t.max()) + 1 if len(t) else 0
    _, n = np.unique(p.astype(np.int64) * max(nt, 1) + t, return_counts=True)
    return n, np.bincount(p), np.bincount(t)


PAIRWISE_KEYS = ("precision", "recall", "f1score", "TP", "FP", "FN")


def metrics_from_counts(tp, pred_pairs, true_pairs, num_records):
    """Pairwise precision / recall / F1 / TP / FP / FN and the adjusted Rand index (key adjRandIndex) of one clustering,
    from its pair counts: tp = pairs put together by both clusterings, pred_pairs / true_pairs = pairs put together by
    each.  Undefined values are NaN: precision without a predicted pair, recall without a true pair, F1 without either,
    the adjusted Rand index with fewer than two records."""
    tp, pc, tc = int(tp), int(pred_pairs), int(true_pairs)
    fp, fn = pc - tp, tc - tp
    precision = tp / (tp + fp) if tp + fp else float("nan")
    recall = tp / (tp + fn) if tp + fn else float("nan")
    f1 = 2 * precision * recall / (precision + recall) if tp else (0.0 if (fp or fn) else float("nan"))
    all_pairs = int(_comb2(num_records))
    if all_pairs:
        expected = pc * tc / all_pairs
        max_index = (pc + tc) / 2.0
        ari = (tp - expected) / (max_index - expected) if max_index != expected else 1.0
    else:
        ari = float("nan")
    return {"precision": precision, "recall": recall, "f1score": f1, "TP": tp, "FP": fp, "FN": fn,
            "adjRandIndex": ari}


def _label_counts(pred_labels, true_labels):
    n, pn, tn = contingency(pred_labels, true_labels)
    return metrics_from_counts(_comb2(n).sum(), _comb2(pn).sum(), _comb2(tn).sum(), len(pred_labels))


def pairwise_metrics(pred_labels, true_labels):
    m = _label_counts(pred_labels, true_labels)
    return {k: m[k] for k in PAIRWISE_KEYS}


def adjusted_rand_index(pred_labels, true_labels):
    return _label_counts(pred_labels, true_labels)["adjRandIndex"]


# ---- every sample against the ground truth ---------------------------------------------------------------
def true_pairs(true_labels):
    """The number of record pairs the ground truth puts together."""
    return int(_comb2(np.unique(np.asarray(true_labels), return_counts=True)[1]).sum())


def posterior_metric_counts(chain, truth):
    """(tp, pred_pairs, num_clusters), int64[S]: per sample, the record pairs it shares with the ground truth
    (truth[r] = true label of record index r), the pairs it puts together and its number of clusters."""
    R = chain.num_records
    truth = np.asarray(truth)
    S = len(chain.samples)
    out = [np.zeros(S, np.int64) for _ in range(3)]
    for s, (mem, off, _) in enumerate(chain.samples):
        if len(mem) != R:
            raise ValueError("every sample must mention every record exactly once")
        sizes = np.diff(off)
        n, pn, _ = contingency(np.repeat(np.arange(len(sizes)), sizes), truth[mem])
        out[0][s], out[1][s], out[2][s] = _comb2(n).sum(), _comb2(pn).sum(), len(pn)
    return tuple(out)


SAMPLE_METRICS = ("precision", "recall", "f1score", "adjRandIndex", "numClusters")


def sample_metrics(tp, pred_pairs, num_clusters, truth):
    """One dict per sample: metrics_from_counts of its counts, and numClusters."""
    tc, R = true_pairs(truth), len(truth)
    return [dict(metrics_from_counts(t, p, tc, R), numClusters=int(c)) for t, p, c in zip(tp, pred_pairs, num_clusters)]


def posterior_summary(rows):
    """For each of SAMPLE_METRICS over the samples (dicts of sample_metrics) where it is defined (not NaN): mean, sd
    (ddof = 1; NaN below two values), the 2.5 %, 50 % and 97.5 % quantiles (np.quantile's default method), the number
    of defined values n and of undefined ones."""
    out = {}
    for k in SAMPLE_METRICS:
        v = np.asarray([r[k] for r in rows], np.float64)
        d = v[~np.isnan(v)]
        q = np.quantile(d, [0.025, 0.5, 0.975]) if len(d) else np.full(3, np.nan)
        out[k] = {"mean": float(d.mean()) if len(d) else float("nan"),
                  "sd": float(d.std(ddof=1)) if len(d) >= 2 else float("nan"),
                  "q025": float(q[0]), "median": float(q[1]), "q975": float(q[2]),
                  "n": len(d), "undefined": len(v) - len(d)}
    return out
