"""Posterior summaries on arrays (no Python loop over clusters or records): the same quantities as analysis.py --
LinkageChain.scala:52-154 and analysis/{PairwiseMetrics,ClusteringMetrics}.scala -- for chains of millions of records.

A sample is held as (members, offsets, partition_of_cluster): `members` = record INDICES (positions in the id
dictionary) of all clusters back to back, `offsets[c]:offsets[c+1]` = cluster c.  The simple set-based functions in
analysis.py stay as the readable restatement; tests compare the two on random chains.
"""
import fractions
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


def chain_files(path):
    """(partition id, file name, file path) of every file of a chain written hive-partitioned by partitionId, in the
    order the readers take them: partitionId= directories sorted by name (as strings, so 10 comes before 2), then
    their files by name."""
    for d in sorted(os.listdir(path)):
        if not d.startswith("partitionId="):
            continue
        for f in sorted(os.listdir(os.path.join(path, d))):
            yield int(d.split("=")[1]), f, os.path.join(path, d, f)


def kept_clusters(sizes):
    """The clusters of a linkage-chain row that a ChainArrays sample keeps: the non-empty ones."""
    return np.asarray(sizes) > 0


def read_chain_arrays(path, lower_iteration_cutoff=0):
    """linkage-chain.parquet (hive-partitioned by partitionId) -> ChainArrays, through Arrow only."""
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyarrow.parquet as pq

    rows = {}  # iteration -> list of (pid, ListArray of clusters)
    for pid, _, f in chain_files(path):
        t = pq.ParquetFile(f).read()
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
        keep = kept_clusters(sizes)
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


# ---- per-pair MCMC diagnostics of the match probabilities ------------------------------------------------
# For a pair, x_s = 1[the two records share a cluster in sample s].  Each of K chains, cut to the first n draws (n =
# the shortest chain's), gives two halves [0, N) and [n - N, n), N = n // 2: M = 2K halves, as convergence.split_rhat
# splits them.  With c_m the linked draws of half m, per lag tau in [0, N) the integers
#   L_m[tau] = sum_{t < N - tau} x_t x_{t + tau},  h_m[tau] = sum_{t < N - tau} x_t,  g_m[tau] = sum_{t >= tau} x_t,
#   Q_m[tau] = N^2 L - N c (h + g) + (N - tau) c^2 = N^3 x the half's biased autocovariance at lag tau,
# A = sum_m Q_m, Bn = M sum c_m^2 - (sum c_m)^2, V = (M - 1)(N - 1) A[0] + N (N - 1) Bn and Wn = (M - 1) N A[0]
# (var+ and W of Vehtari et al. 2021, scaled by M (M - 1) N^3 (N - 1)) give split-R̂ = sqrt(V / Wn) and, from
# u[tau] = 2 (V - Wn + (M - 1)(N - 1) A[tau]) (u[0] = 2 V, so rho[tau] = u[tau] / 2V), the effective sample size by
# Geyer's initial positive and initial monotone sequences.  Every comparison is on int64 u, and the monotone step keeps
# each pair sum at the running minimum of the pair sums before it, so one pass over the lags suffices.
MAX_TRACE_WORDS = 1 << 31    # uint32 words of the GPU's bit trace, [ceil(S / 32)][held pairs]
MIXING_SIZE_BOUND = 1 << 30  # M N^2 below this keeps every integer above inside int64 (M^2 N^4 < 2^60)
MIN_DRAWS = 4                # convergence.MIN_DRAWS


def chain_draws(chain):
    """(starts int32[K], n) of a pooled ChainArrays: chain k's draws are pooled positions starts[k] .. starts[k] + n - 1,
    n = the shortest chain's number of samples.  The one place that decides which draws the diagnostics use."""
    chains = np.asarray(chain.chains, np.int64)
    K = int(chains.max()) + 1 if len(chains) else 1
    counts = np.bincount(chains, minlength=K)
    if len(chains) and (np.diff(chains) < 0).any():
        raise ValueError("the pooled samples are not chain-major")
    n = int(counts.min())
    if n < MIN_DRAWS:
        raise ValueError(f"pairwise-match-diagnostics needs at least {MIN_DRAWS} draws per chain after the cutoff")
    return np.r_[0, np.cumsum(counts)[:-1]].astype(np.int32), n


def check_mixing_size(num_chains, draws):
    M, N = 2 * int(num_chains), int(draws) // 2
    if M * N * N >= MIXING_SIZE_BOUND:
        raise ValueError(f"pairwise-match-diagnostics needs M N^2 < 2^30: {M} half-chains of {N} draws")


def check_trace_size(num_samples, num_pairs):
    words = -(-int(num_samples) // 32) * int(num_pairs)
    if words > MAX_TRACE_WORDS:
        raise ValueError(f"the match trace needs {words} words, more than {MAX_TRACE_WORDS}")


def ess_floor(num_chains, draws):
    """1 / log10(M N), the least autocorrelation time the ESS divides by."""
    return 1.0 / math.log10(2 * int(num_chains) * (int(draws) // 2))


def pairwise_match_trace(chain, keys):
    """bool[len(keys), S]: x[i, s] = 1 when the pair keys[i] (first << 32 | second, sorted) shares a cluster in pooled
    sample s."""
    keys = np.asarray(keys, np.int64)
    x = np.zeros((len(keys), len(chain.samples)), bool)
    if len(keys) == 0:
        return x
    for s, (mem, off, _) in enumerate(chain.samples):
        k = sample_pair_keys(chain.num_records, mem, off)
        pos = np.minimum(np.searchsorted(keys, k), len(keys) - 1)
        hit = keys[pos] == k
        x[pos[hit], s] = True
    return x


def pack_trace(x):
    """bool[H, P] -> uint32[ceil(P / 32), H], the GPU's word-major bit trace (bit p % 32 of word p // 32)."""
    H, P = x.shape
    W = -(-P // 32)
    pad = np.zeros((H, 32 * W), bool)
    pad[:, :P] = x
    return np.packbits(pad.reshape(H, W, 4, 8), axis=-1, bitorder="little").reshape(H, W * 4).view("<u4").T.copy()


class MatchMixing:
    """Per pair, int64 arrays count (linked draws of the 2 K N used), chain_min / chain_max (the least and largest of
    one chain's), max_t (the lag where the initial positive sequence truncates) and float64 rhat, ess; with M halves
    of N = draws // 2 draws from each chain's first `draws`."""

    def __init__(self, count, chain_min, chain_max, max_t, rhat, ess, M, draws):
        self.count, self.chain_min, self.chain_max, self.max_t = count, chain_min, chain_max, max_t
        self.rhat, self.ess, self.M, self.draws, self.N = rhat, ess, M, draws, draws // 2


def mixing_from_trace(x, starts, n, floor):
    """The diagnostics of every row of a bool trace x[H, P] over the chains starts[k] .. starts[k] + n - 1: a
    MatchMixing, equal bit for bit to dbl_pairs_mixing.  The per-lag integers are taken vectorised over the pairs, one
    lag pair at a time, while any pair's sequence has not truncated."""
    starts = [int(s) for s in starts]
    K, n = len(starts), int(n)
    N, M = n // 2, 2 * len(starts)
    check_mixing_size(K, n)
    H = x.shape[0]
    halves = [np.ascontiguousarray(x[:, s + o:s + o + N], np.uint8) for s in starts for o in (0, n - N)]
    c = np.stack([h.sum(1, dtype=np.int64) for h in halves]).reshape(M, H)  # [M, H]
    chain_c = c[0::2] + c[1::2]                                    # halves of one chain are adjacent
    S1, S2 = c.sum(0), (c * c).sum(0)
    A0 = sum(N * c[m] - c[m] * c[m] for m in range(M)) * N         # Q_m[0] = N (N c - c^2)
    V = (M - 1) * (N - 1) * A0 + N * (N - 1) * (M * S2 - S1 * S1)
    Wn = (M - 1) * N * A0

    def u_at(tau, rows):
        if tau == 0:
            return 2 * V[rows]
        A = np.zeros(len(rows), np.int64)
        for m, h in enumerate(halves):
            hm = h[rows]
            L = (hm[:, :N - tau] & hm[:, tau:]).sum(1, dtype=np.int64)
            hh, gg = hm[:, :N - tau].sum(1, dtype=np.int64), hm[:, tau:].sum(1, dtype=np.int64)
            cm = c[m, rows]
            A += N * N * L - N * cm * (hh + gg) + (N - tau) * cm * cm
        return 2 * (V[rows] - Wn[rows] + (M - 1) * (N - 1) * A)

    max_t = np.zeros(H, np.int64)
    acc = np.zeros(H, np.float64)
    last = np.zeros(H, np.int64)
    live = np.flatnonzero(V != 0)
    even, odd = u_at(0, live), u_at(1, live)
    P = even + odd
    cur = P.copy()                                                 # the pair sum after the monotone step
    t = 0
    while len(live):
        stop = ~((t < N - 5) & (P > 0))
        done = live[stop]
        max_t[done] = t
        last[done] = np.where((P[stop] >= 0) | (even[stop] > 0), even[stop], 0)
        keep = ~stop
        live, cur = live[keep], cur[keep]
        if not len(live):
            break
        acc[live] = acc[live] + cur.astype(np.float64)            # the pair before max_t, in ascending lag order
        t += 2
        even, odd = u_at(t, live), u_at(t + 1, live)
        P = even + odd
        cur = np.minimum(P, cur)
    rhat = np.full(H, np.nan)
    ess = np.full(H, np.nan)
    pos = V != 0
    with np.errstate(divide="ignore"):
        rhat[pos] = np.sqrt(V[pos].astype(np.float64) / Wn[pos].astype(np.float64))
    num = (acc + acc) + last.astype(np.float64)
    tau_hat = -1.0 + num[pos] / (2 * V[pos]).astype(np.float64)
    ess[pos] = np.float64(M * N) / np.where(tau_hat > floor, tau_hat, floor)
    return MatchMixing(S1, chain_c.min(0), chain_c.max(0), max_t, rhat, ess, M, n)


def mcse(count, num_draws, ess):
    """Monte Carlo standard error of a probability count / num_draws with effective sample size ess:
    sqrt(count (D - count) / (D (D - 1)) / ess), D = num_draws."""
    count = np.asarray(count, np.int64)
    D = int(num_draws)
    var = (count * (D - count)).astype(np.float64) / float(D * (D - 1))
    with np.errstate(invalid="ignore"):
        return np.sqrt(var / np.asarray(ess, np.float64))


def match_diagnostics_summary(mix, num_chains, draws):
    """The (quantity, value) rows of pairwise-match-diagnostics-summary.csv over the pairs of a MatchMixing: the pairs
    with R̂ above 1.01 and 1.1 (inf included), with R̂ = inf and with R̂ undefined (NaN), the least and the median of
    the defined ESS, and the pairs with ESS below 100 per chain."""
    K = int(num_chains)
    rhat, ess = np.asarray(mix.rhat), np.asarray(mix.ess)
    defined = ess[~np.isnan(ess)]
    return [("numChains", K), ("drawsPerChain", int(draws)), ("pairs", len(rhat)),
            ("pairsRhatAbove1.01", int((rhat > 1.01).sum())), ("pairsRhatAbove1.1", int((rhat > 1.1).sum())),
            ("pairsRhatInf", int(np.isinf(rhat).sum())), ("pairsRhatUndefined", int(np.isnan(rhat).sum())),
            ("minEss", float(defined.min()) if len(defined) else float("nan")),
            ("medianEss", float(np.median(defined)) if len(defined) else float("nan")),
            ("pairsEssBelow100PerChain", int((defined < 100 * K).sum()))]


def pairwise_match_diagnostics(chain, min_count=1, max_pairs=MAX_PAIRS):
    """(first, second, count, MatchMixing) over the pairs with count >= min_count (pairwise_match_counts' rows, count
    over every pooled sample), the diagnostics over the draws chain_draws picks.  Raises ValueError for fewer than
    MIN_DRAWS draws per chain, M N^2 >= 2^30 or a trace of more than MAX_TRACE_WORDS words."""
    starts, n = chain_draws(chain)
    check_mixing_size(len(starts), n)
    first, second, count = pairwise_match_counts(chain, max_pairs)
    check_trace_size(len(chain.samples), len(first))
    keep = count >= min_count
    first, second, count = first[keep], second[keep], count[keep]
    x = pairwise_match_trace(chain, (first << 32) | second)
    return first, second, count, mixing_from_trace(x, starts, n, ess_floor(len(starts), n))


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
    aS = a * S
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
        win, lab = claim_moves(lab, c_rec[best], c_dest[best], c_dJ[best])
        moves.append(int(win.sum()))
        dn.append(int(c_dn[best][win].sum()))
        dK.append(int(c_dK[best][win].sum()))
    n, K = search_result_counts(first, second, count, lab)
    return SearchRun(lab, moves, dn, dK, converged, n, K)


def claim_moves(lab, i, X, dJ):
    """One round's claims, shared by both searches: records i propose moving from their clusters lab[i] to X (-1: a
    new singleton) with changes dJ < 0.  A proposal wins if it holds the least (dJ, i) among the proposals touching each
    cluster it touches (its source, and its destination unless a singleton).  Returns (win mask, the canonical labels
    after the winning moves)."""
    R, big = len(lab), np.iinfo(np.int64).max
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
    return win, canonical_labels(key)


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
    S = G.shape[0]
    g_sum = g.sum(axis=0)
    # against every sample including itself, sample t has G[t] + g[t] cells of each size (C_t ^ C_t = C_t)
    return np.array([vi_label_loss(g[t], G[t] + g[t], g_sum, S, num_records) for t in range(S)], np.float64)


def vi_label_loss(g_c, G_c, g_sum, num_samples, num_records):
    """The posterior expected VI of a labelling c against S samples, from integer histograms indexed by size n: g_c[n] =
    the clusters of n records of c, G_c[n] = the cells of n >= 2 records of c ^ C_s summed over every sample s, g_sum[n]
    = the clusters of n records summed over the samples.  D[n] = S g_c[n] + g_sum[n] - 2 G_c[n], E = fsum over n >= 2 of
    float(D[n]) (n log2 n), divided by R S.  fsum is correctly rounded and does not depend on the order, so equal
    integers give equal losses."""
    S, R = int(num_samples), int(num_records)
    if R == 0 or S == 0:
        return 0.0
    width = max(len(g_c), len(G_c), len(g_sum))
    pad = lambda x: np.pad(np.asarray(x, np.int64), (0, width - len(x)))  # noqa: E731
    D = S * pad(g_c) + pad(g_sum) - 2 * pad(G_c)
    D[:2] = 0
    nz = np.flatnonzero(D)
    return math.fsum(D[nz].astype(np.float64) * np.array([n * math.log2(n) for n in nz.tolist()])) / (R * S)


def vi_sample_cells(chain, labels, width):
    """G, int64[S, width]: per sample s the cells of n >= 2 records of labels ^ C_s (width at least M + 1, M = the
    largest cluster of any sample, as every cell lies inside one)."""
    R = chain.num_records
    labels = np.asarray(labels, np.int64)
    G = np.zeros((len(chain.samples), int(width)), np.int64)
    for s, (mem, off, _) in enumerate(chain.samples):
        lab_s = sample_labels(R, mem, off)
        big = np.flatnonzero(np.bincount(lab_s, minlength=R)[lab_s] >= 2)
        _, n = np.unique(lab_s[big] * R + labels[big], return_counts=True)
        G[s] = np.bincount(n[n >= 2], minlength=width)[:width]
    return G


def vi_label_cells(chain, labels, width):
    """G, int64[width]: the cells of n >= 2 records of labels ^ C_s summed over the samples s of the chain: the row sum
    of vi_sample_cells."""
    return vi_sample_cells(chain, labels, width).sum(axis=0)


def vi_estimate(losses):
    """The position of the sample of least expected VI, ties going to the earliest."""
    if len(losses) == 0:
        raise ValueError("the VI estimate needs at least one sample")
    return min(range(len(losses)), key=lambda s: (losses[s], s))


# ---- the credible ball around a point estimate (Wade and Ghahramani 2018, section 4) --------------------------------
# Per sample s and cell size n, with g_x[n] = the clusters of n records of x and G_s[n] = the cells of n >= 2 records of
# c ^ C_s: D_s[n] = g_c[n] + g_s[n] - 2 G_s[n].  Then VI(c, C_s) = sum over n of D_s[n] n log2 n / R bits, and the
# Binder distance, the record pairs one of c, C_s links and the other does not, is sum over n of D_s[n] n (n - 1) / 2,
# exact in int64.  The ball of level p holds every sample within the radius, the k-th smallest distance, k = ceil(p S)
# (an exact fraction of repr(p)); ties at the radius are inside.  Its bounds are samples in the ball: the farthest from
# c (vertical upper), the farthest of those with the fewest clusters (horizontal upper) and the farthest of those with
# the most clusters (horizontal lower); ties go to the earliest sample in pooled order.
CREDIBLE_BALL_BOUNDS = ("vertical-upper", "horizontal-upper", "horizontal-lower")
CREDIBLE_BALL_DISTANCES = ("vi", "binder")


def credible_ball_distances(g_c, g, G_rows, num_records):
    """(vi float64[S], binder int64[S]): the distances of a labelling c from every sample, from integer histograms
    indexed by size n: g_c[n] = the clusters of n records of c, g[s][n] those of sample s, G_rows[s][n] = the cells of
    n >= 2 records of c ^ C_s.  The VI is fsum over n >= 2 of float(D_s[n]) (n log2 n), divided by R: correctly rounded
    and order-free, so equal integers give equal distances."""
    g_c, g, G = np.asarray(g_c, np.int64), np.asarray(g, np.int64), np.asarray(G_rows, np.int64)
    S, R = G.shape[0], int(num_records)
    width = max(len(g_c), g.shape[1], G.shape[1])
    D = (np.pad(g_c, (0, width - len(g_c)))[None, :] + np.pad(g, ((0, 0), (0, width - g.shape[1])))
         - 2 * np.pad(G, ((0, 0), (0, width - G.shape[1]))))
    D[:, :2] = 0
    n = np.arange(width, dtype=np.int64)
    binder = (D * (n * (n - 1) // 2)).sum(axis=1) if S else np.zeros(0, np.int64)
    f = np.array([k * math.log2(k) if k >= 2 else 0.0 for k in range(width)])
    vi = np.zeros(S, np.float64)
    for s in range(S):
        nz = np.flatnonzero(D[s])
        vi[s] = math.fsum(D[s, nz].astype(np.float64) * f[nz]) / R if R else 0.0
    return vi, binder.astype(np.int64)


def credible_level_rank(level, num_samples):
    """k = ceil(level S), exact: level is taken as the fraction its repr spells (0.7 is 7/10, so 0.7 x 10 gives 7)."""
    level = float(level)
    if not 0.0 < level <= 1.0:
        raise ValueError("credibleLevel must be in (0, 1].")
    return math.ceil(fractions.Fraction(repr(level)) * int(num_samples))


def credible_ball(distances, num_clusters, level):
    """The credible ball of one distance: (radius, in-ball bool[S], {bound: (sample position, ties)}).  ties counts the
    samples of the ball that equal the chosen one in what the bound ranks them by."""
    d = np.asarray(distances)
    k = np.asarray(num_clusters, np.int64)
    S = len(d)
    if S == 0:
        raise ValueError("the credible ball needs at least one sample")
    radius = np.sort(d, kind="stable")[credible_level_rank(level, S) - 1].item()
    inside = d <= radius
    members = np.flatnonzero(inside).tolist()
    rank = {"vertical-upper": lambda s: (-d[s],),
            "horizontal-upper": lambda s: (k[s], -d[s]),
            "horizontal-lower": lambda s: (-k[s], -d[s])}
    bounds = {}
    for name in CREDIBLE_BALL_BOUNDS:
        best = min(members, key=lambda s: (rank[name](s), s))
        bounds[name] = (best, sum(rank[name](s) == rank[name](best) for s in members))
    return radius, inside, bounds


# ---- the VI search: parallel single-record moves ----------------------------------------------------------------
# With f(n) = n log2 n, A(x) = sum over the blocks of x of f(|block|) and samples C_1 .. C_S, R S E[VI](c) = S A(c) +
# sum_s A(C_s) - 2 sum_s A(c ^ C_s).  The search works on the quantised table D_q[m] = round(2^Q (f(m + 1) - f(m))),
# m = 0 .. R - 1, with F_q(n) = D_q[0] + ... + D_q[n - 1] in place of f, and lowers
#   J_q(c) = S sum over clusters X of F_q(|X|) - 2 sum_s sum over the cells of c ^ C_s of F_q(n).
# Moving record i from A (|A| = a) to B (|B| = beta; a new singleton is beta = 0) changes J_q by exactly
#   dJ = S (D_q[beta] - D_q[a - 1]) - 2 (w_B - w_A),  w_B = sum_s D_q[|B ^ C_s(i)|],  w_A = sum_s D_q[|A ^ C_s(i)| - 1].
# D_q[0] = 0 and D_q is non-decreasing, so a cluster sharing no sample cluster with i is never better than the
# singleton: the candidates are the clusters of the records that share a sample cluster with i and, when a > 1, a
# singleton; only samples where i is in a cluster of two or more add to w.  Moves that touch disjoint clusters of c
# touch disjoint cells of every c ^ C_s, so the claims of the Binder search (claim_moves) apply unchanged, their dJ add
# exactly and J_q falls every round.  The quantised expected VI E_q(c) = (J_q(c) + sum_s A_q(C_s)) / (2^Q R S) is
# within 2^(1-Q) bits of E[VI](c): each F_q(n) is off f(n) 2^Q by at most n / 2.
VI_SEARCH_BITS = 20             # Q
MAX_VI_SEARCH_SQUARES = 1 << 28  # a sample's sum over its clusters of |K|^2: bounds its contributions to one round
VI_SEARCH_STARTS = ("vi-sample", "smpc")


def vi_search_table(num_records):
    """D_q, int64[R]: round(2^Q (f(m + 1) - f(m))) for m = 0 .. R - 1, f(m + 1) - f(m) = log2(m + 1) + m log2(1 + 1/m)
    evaluated without cancellation, halves rounded up."""
    R = int(num_records)
    d = np.zeros(R)
    m = np.arange(1, R, dtype=np.float64)
    d[1:] = np.log2(m + 1) + m * np.log1p(1.0 / m) / math.log(2)
    return np.floor(d * float(1 << VI_SEARCH_BITS) + 0.5).astype(np.int64)


def check_vi_search_size(num_samples, num_records):
    """S R (ceil(log2 R) + 2) 2^(Q+2) < 2^63 keeps every dJ, round sum, J_q and sum_s A_q(C_s) inside int64."""
    S, R = int(num_samples), int(num_records)
    if S * R * ((max(R, 1) - 1).bit_length() + 2) << (VI_SEARCH_BITS + 2) >= 1 << 63:
        raise ValueError(f"the VI search needs samples x records x (ceil(log2 records) + 2) x 2^22 < 2^63 "
                         f"(here {S} x {R})")


def check_vi_search_squares(squares):
    """squares[s] = sum over the clusters of sample s of |K|^2; ValueError past MAX_VI_SEARCH_SQUARES."""
    for s, q in enumerate(squares):
        if int(q) > MAX_VI_SEARCH_SQUARES:
            raise ValueError(f"the VI search refuses sample {s}: its clusters' squared sizes sum to {int(q)}, more "
                             f"than {MAX_VI_SEARCH_SQUARES}")


def vi_sample_squares(chain):
    """int64[S]: per sample the sum over its clusters of |K|^2."""
    return np.array([int((np.diff(off).astype(np.int64) ** 2).sum()) for _, off, _ in chain.samples], np.int64)


def vi_search_prefix(table):
    """F_q, int64[R + 1]: F_q(n) = D_q[0] + ... + D_q[n - 1]."""
    return np.r_[0, np.cumsum(np.asarray(table, np.int64))].astype(np.int64)


def vi_sample_sum(chain, table):
    """sum over the samples and their clusters K of F_q(|K|): the J_q-independent part of R S 2^Q E_q."""
    F = vi_search_prefix(table)
    return sum(int(F[np.diff(off)].sum()) for _, off, _ in chain.samples)


class VISearchRun:
    """One VI search: labels int64[R] (canonical) where it stopped; per round the moves applied, the clusters after it
    and the change of J_q, int64[rounds]; whether it stopped because no record proposed a move; J_q of the start."""

    def __init__(self, labels, moves, clusters, dJ, converged, J0):
        self.labels, self.converged, self.J0 = labels, bool(converged), int(J0)
        self.moves, self.clusters, self.dJ = (np.asarray(x, np.int64) for x in (moves, clusters, dJ))

    @property
    def rounds(self):
        return len(self.moves)

    @property
    def J(self):
        return self.J0 + int(self.dJ.sum())

    def objectives(self):
        """[J_q of the start (round 0), then after every round], Python ints."""
        return [self.J0 + int(x) for x in np.r_[0, np.cumsum(self.dJ)]]


def vi_search_losses(objectives, sample_sum, num_samples, num_records):
    """E_q = (J_q + sum_s A_q(C_s)) / (2^Q R S) for each J_q: one correctly rounded division of integers."""
    den = (int(num_records) * int(num_samples)) << VI_SEARCH_BITS
    return [(int(J) + int(sample_sum)) / den for J in objectives]


def _vi_contributions(R, lab_s, big, lab, table):
    """One sample's contributions to w: for each record i in a cluster K of two or more of the sample and each cell
    (K, B) of m records, (i R + B, D_q[m]), or D_q[m - 1] for i's own cell; and the sum of F_q over the cells is left to
    the caller through the cell sizes.  Returns (keys, values, cell sizes)."""
    if not len(big):
        return (np.zeros(0, np.int64),) * 3
    key = lab_s[big] * R + lab[big]
    order = np.argsort(key, kind="stable")
    ks, rec = key[order], big[order]
    cs = _run_starts(ks)
    cn = np.diff(np.r_[cs, len(ks)])
    cK, cB = ks[cs] // R, ks[cs] % R
    ks_K = _run_starts(cK)                                # first cell of each sample cluster
    nK = np.diff(np.r_[ks_K, len(cs)])                    # its number of cells
    kidx = np.repeat(np.repeat(np.arange(len(ks_K)), nK), cn)  # per sorted record, its sample cluster
    cnt = nK[kidx]
    total = int(cnt.sum())
    first = np.repeat(np.cumsum(cnt) - cnt, cnt)
    j = np.arange(total) - first + np.repeat(ks_K[kidx], cnt)
    i = np.repeat(rec, cnt)
    B, m = cB[j], cn[j]
    return i * R + B, table[m - (B == lab[i])], cn


def vi_search_rounds(num_records, sample_labels_list, table, start, max_rounds):
    """The VI search from labels start[R] against the samples (a list of int64 labels[R], one per sample) with the
    table D_q: a VISearchRun."""
    R, S = int(num_records), len(sample_labels_list)
    table = np.asarray(table, np.int64)
    if table.shape != (R,):
        raise ValueError("the VI search table needs one entry per record")
    if np.shape(start) != (R,):
        raise ValueError("a start needs one cluster label per record")
    F = vi_search_prefix(table)
    bigs = [np.flatnonzero(np.bincount(ls, minlength=R)[ls] >= 2) for ls in sample_labels_list]
    lab = canonical_labels(np.asarray(start, np.int64))
    moves, clusters, dJs, converged, J0 = [], [], [], False, None
    while True:
        size = np.bincount(lab, minlength=R).astype(np.int64)
        keys, vals, cell_F = [], [], 0
        for ls, big in zip(sample_labels_list, bigs):
            k, v, cn = _vi_contributions(R, ls, big, lab, table)
            keys.append(k)
            vals.append(v)
            cell_F += int(F[cn].sum())
        if J0 is None:
            J0 = S * int(F[size].sum()) - 2 * cell_F
        keys = np.concatenate(keys) if keys else np.zeros(0, np.int64)
        vals = np.concatenate(vals) if vals else np.zeros(0, np.int64)
        order = np.argsort(keys, kind="stable")
        keys = keys[order]
        runs = _run_starts(keys)
        keys, w = keys[runs], np.add.reduceat(vals[order], runs) if len(runs) else np.zeros(0, np.int64)
        rec, X = keys // R, keys % R
        own = X == lab[rec]
        wA = np.zeros(R, np.int64)
        wA[rec[own]] = w[own]
        a = size[lab]
        dA = table[a - 1]
        # candidates in ascending (record, destination) order: a record's singleton first, then its clusters
        multi = np.flatnonzero(a > 1)
        by = np.argsort(np.r_[2 * multi, 2 * rec[~own] + 1], kind="stable")
        c_rec = np.r_[multi, rec[~own]][by]
        c_dest = np.r_[np.full(len(multi), -1, np.int64), X[~own]][by]
        r_o, x_o = rec[~own], X[~own]
        c_dJ = np.r_[-S * dA[multi] + 2 * wA[multi],
                     S * (table[size[x_o]] - dA[r_o]) - 2 * (w[~own] - wA[r_o])][by]
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
        win, lab = claim_moves(lab, c_rec[best], c_dest[best], c_dJ[best])
        moves.append(int(win.sum()))
        clusters.append(int(len(np.unique(lab))))
        dJs.append(int(c_dJ[best][win].sum()))
    return VISearchRun(lab, moves, clusters, dJs, converged, J0)


def vi_search_choice(runs):
    """The position of the run of least final J_q, ties going to the earlier start."""
    return min(range(len(runs)), key=lambda k: (runs[k].J, k))


class VISamples:
    """The held samples of a chain on the host, with the methods of analysis_gpu.VI: cross (the cell histograms of
    every pair of samples), search (the VI search), score (the cells of a labelling with every sample) and
    score_samples (those cells per sample)."""

    def __init__(self, chain):
        self.chain = chain
        self.num_records, self.num_samples = chain.num_records, len(chain.samples)
        self._labels = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        pass

    def labels(self):
        if self._labels is None:
            self._labels = [sample_labels(self.num_records, mem, off) for mem, off, _ in self.chain.samples]
        return self._labels

    def cross(self, width):
        G = vi_cross_histograms(self.chain)
        return np.pad(G, ((0, 0), (0, int(width) - G.shape[1])))

    def search(self, table, start, max_rounds):
        return vi_search_rounds(self.num_records, self.labels(), table, start, max_rounds)

    def score(self, labels, width):
        return vi_label_cells(self.chain, labels, width)

    def score_samples(self, labels, width):
        return vi_sample_cells(self.chain, labels, width)


def vi_search(chain, starts, max_rounds=1000):
    """The VI search from each of starts (labels[R] each) against the chain's samples: (the position of the chosen run,
    the VISearchRuns).  ValueError before any work for the size bound or a sample past the squares cap."""
    R, S = chain.num_records, len(chain.samples)
    check_vi_search_size(S, R)
    check_vi_search_squares(vi_sample_squares(chain))
    vi = VISamples(chain)
    runs = [vi.search(vi_search_table(R), st, max_rounds) for st in starts]
    return vi_search_choice(runs), runs


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


# ---- the posterior of the entity values of a point estimate's clusters ------------------------------------------
# For a point estimate with clusters c (canonical labels 0 .. C-1), a matching attribute and its value v:
#   count(c, v) = sum over samples s and records r of c of 1[y_s(link_s(r)) = v]
# so count / (|c| S) is the probability that the entity a uniformly chosen record of c links to has value v, and the
# counts of c sum to |c| S.  The mode of c is the v of largest count, ties going to the smallest value id (the first
# value in byte order).
ENTITY_VALUES_CHAIN = "entity-values-chain.parquet"


def _no_entity_values(iteration):
    return ValueError(f"the sample at iteration {iteration} has no entity values (it was recorded with "
                      f"saveEntityValues off): raise lowerIterationCutoff past it, or sample again with "
                      f"saveEntityValues on")


def _entity_value_index(chain_dir):
    """iteration -> the name of the files of entity-values-chain.parquet under chain_dir holding it."""
    import pyarrow.parquet as pq

    path = os.path.join(chain_dir, ENTITY_VALUES_CHAIN)
    index = {}
    if os.path.isdir(path):
        for _, name, f in chain_files(path):
            for it in pq.read_table(f, columns=["iteration"]).column("iteration").to_numpy():
                index.setdefault(int(it), name)
    return index


def _entity_value_group(chain_dir, name, attribute_names):
    """The rows of the files called `name` of a chain directory, one flush of its two writers: (the cluster sizes of
    each linkage row, the attribute value lists of each entity-values row), both keyed by (iteration, partition id)
    and in chain_files order."""
    import pyarrow.parquet as pq

    sizes, values = {}, {}
    for pid, f_name, f in chain_files(os.path.join(chain_dir, "linkage-chain.parquet")):
        if f_name == name:
            t = pq.ParquetFile(f).read()
            ls = t.column("linkageStructure").combine_chunks()
            for i, it in enumerate(t.column("iteration").to_numpy()):
                sizes[(int(it), pid)] = np.diff(ls[i].values.offsets.to_numpy())
    for pid, f_name, f in chain_files(os.path.join(chain_dir, ENTITY_VALUES_CHAIN)):
        if f_name == name:
            t = pq.ParquetFile(f).read()
            cols = [t.column(a).combine_chunks() for a in attribute_names]
            for i, it in enumerate(t.column("iteration").to_numpy()):
                values[(int(it), pid)] = [c[i].values for c in cols]
    return sizes, values


def read_entity_values(chain_dirs, chain, attribute_names, attribute_values):
    """Yields, for every sample of `chain` in order, int32[A][R]: the value id, per matching attribute, of the entity
    each record links to.  chain = read_chain_arrays of chain_dirs[0]'s linkage chain, or read_pooled_chain_arrays of
    every chain directory's (chain.chains[s] = the directory of sample s).  The values come from each directory's
    entity-values-chain.parquet, walked as read_chain_arrays walks the linkage chain (chain_files) with the same kept
    clusters; attribute_values[a] = the pyarrow string array of attribute a's values in value-id order.  One flush of
    files is read at a time, so no more than a write buffer of samples is held.  Raises ValueError for a row whose
    lists do not have one entry per cluster of its linkage row, a value the attribute lacks, or a sample without
    entity values."""
    import pyarrow as pa
    import pyarrow.compute as pc

    A, R = len(attribute_names), chain.num_records
    indexes, loaded, group = {}, None, None
    for s, (it, k) in enumerate(zip(chain.iterations, chain.chains)):
        it, k = int(it), int(k)
        if k not in indexes:
            indexes[k] = _entity_value_index(chain_dirs[k])
        name = indexes[k].get(it)
        if name is None:
            raise _no_entity_values(it)
        if loaded != (k, name):
            loaded, group = (k, name), _entity_value_group(chain_dirs[k], name, attribute_names)
        sizes, values = group
        mem, off, _ = chain.samples[s]
        cols = [[] for _ in range(A)]
        rows_of = [key for key in sizes if key[0] == it]
        if {key for key in values if key[0] == it} != set(rows_of):
            # files of one name that are not one flush of the two writers, e.g. values left by another chain
            raise ValueError(f"entity-values-chain.parquet, iteration {it}, files {name}: the partitions do not match "
                             f"those of linkage-chain.parquet")
        for key in rows_of:
            row = values[key]
            if any(len(v) != len(sizes[key]) for v in row):
                raise ValueError(f"entity-values-chain.parquet, iteration {it}, partition {key[1]}: the value lists "
                                 f"do not have one entry per cluster of the linkage row ({len(sizes[key])})")
            keep = pa.array(kept_clusters(sizes[key]))
            for a in range(A):
                cols[a].append(row[a].filter(keep))
        out = np.empty((A, R), np.int32)
        for a in range(A):
            got = pa.concat_arrays(cols[a]) if cols[a] else pa.array([], pa.string())
            if len(got) != len(off) - 1:
                raise ValueError(f"entity-values-chain.parquet, iteration {it}: {len(got)} values of "
                                 f"'{attribute_names[a]}' for {len(off) - 1} clusters")
            ids = pc.index_in(got, value_set=attribute_values[a])
            if ids.null_count:
                bad = got.filter(pc.is_null(ids))[0].as_py()
                raise ValueError(f"entity-values-chain.parquet, iteration {it}: '{attribute_names[a]}' has the value "
                                 f"{bad!r}, which its index lacks")
            out[a, mem] = np.repeat(ids.to_numpy(zero_copy_only=False).astype(np.int32), np.diff(off))
        yield out


class EntityValueCounts:
    """count(c, v) of one attribute over the samples added, for the clusters of labels[R] in [0, C): the integers of
    the dbl_values handle (analysis_gpu.EntityValues), held as a sorted table of keys c V + v and int64 counts."""

    def __init__(self, labels, num_clusters, num_values):
        self.labels = np.asarray(labels, np.int64)
        self.num_clusters, self.num_values = int(num_clusters), int(num_values)
        if len(self.labels) and (self.labels.min() < 0 or self.labels.max() >= self.num_clusters):
            raise ValueError("a cluster label outside [0, num_clusters)")
        self.keys, self.counts = np.zeros(0, np.int64), np.zeros(0, np.int64)
        self.num_samples = 0

    def add_sample(self, values):
        values = np.asarray(values, np.int64)
        if values.shape != self.labels.shape:
            raise ValueError("a sample needs one value per record")
        if len(values) and (values.min() < 0 or values.max() >= self.num_values):
            raise ValueError("a value outside [0, num_values)")
        k, n = np.unique(self.labels * self.num_values + values, return_counts=True)
        self.keys, inv = np.unique(np.r_[self.keys, k], return_inverse=True)
        counts = np.zeros(len(self.keys), np.int64)
        np.add.at(counts, inv, np.r_[self.counts, n.astype(np.int64)])
        self.counts = counts
        self.num_samples += 1

    def table(self):
        """(cluster, value, count), int64, in ascending (cluster, value) order."""
        return self.keys // self.num_values, self.keys % self.num_values, self.counts.copy()

    def modes(self):
        """(mode int32[C], count int64[C]): per cluster the value of largest count, ties to the smallest value; -1
        and 0 for a label no record has."""
        if not self.num_samples:
            raise ValueError("no sample added")
        cl, v, n = self.table()
        by = np.lexsort((v, -n, cl))
        lead = by[np.r_[True, cl[by][1:] != cl[by][:-1]]] if len(by) else by
        mode, count = np.full(self.num_clusters, -1, np.int32), np.zeros(self.num_clusters, np.int64)
        mode[cl[lead]], count[cl[lead]] = v[lead], n[lead]
        return mode, count

    def close(self):
        pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def canonical_clusters(labels):
    """int64 labels 0 .. C-1 of any labelling, cluster k being the k-th group of labels_to_clusters(labels)."""
    return np.unique(np.asarray(labels), return_inverse=True)[1].reshape(-1).astype(np.int64)


def entity_value_modes(labels, value_samples, num_values, counter=EntityValueCounts):
    """(modes int32[A][C], counts int64[A][C], S) of the canonical labels[R] (0 .. C-1) over the samples of
    value_samples, an iterable of int32[A][R] (read_entity_values) consumed once: one counter per attribute (of
    num_values[a] values), all alive while the samples stream through.  counter = EntityValueCounts on the host,
    analysis_gpu.EntityValues on the device; both give the same integers."""
    import contextlib

    labels = np.asarray(labels, np.int64)
    C = int(labels.max()) + 1 if len(labels) else 0
    with contextlib.ExitStack() as stack:
        handles = [stack.enter_context(counter(labels, C, V)) for V in num_values]
        S = 0
        for vals in value_samples:
            for h, v in zip(handles, vals):
                h.add_sample(v)
            S += 1
        if S == 0:
            raise ValueError("the entity values need at least one sample at or after lowerIterationCutoff")
        out = [h.modes() for h in handles]
    return (np.array([m for m, _ in out], np.int32).reshape(len(out), C),
            np.array([n for _, n in out], np.int64).reshape(len(out), C), S)


def entity_value_rows(labels, modes, counts, num_samples, attribute_values):
    """The rows of entity-values.csv from the integers: per cluster k of the canonical labels, (k, its size, then per
    attribute its mode's value string and repr(count / (size S)))."""
    sizes = np.bincount(np.asarray(labels, np.int64), minlength=modes.shape[1])
    strings = [np.asarray(v.to_pylist() if hasattr(v, "to_pylist") else list(v), dtype=object)
               for v in attribute_values]
    rows = []
    for k, size in enumerate(sizes.tolist()):
        row = [k, size]
        for a in range(len(strings)):
            row += [strings[a][modes[a, k]], repr(int(counts[a, k]) / (size * num_samples))]
        rows.append(row)
    return rows


# ---- clerical review of a point estimate ---------------------------------------------------------------
# With count(i, j) the pair table of S samples and c a point estimate with canonical labels 0 .. C-1 (record i in
# cluster c(i) of n(i) records), per record, in integers:
#   W(i) = sum over j != i of count(i, j) = sum over the samples of (|C_s(i)| - 1),
#   I(i) = the same sum over the j in c(i),
#   S FL(i) = S (n(i) - 1) - I(i)   (S x the expected false links: partners in c that a sample does not link),
#   S ML(i) = W(i) - I(i)           (S x the expected missed links: partners a sample links that c does not),
#   A(i) = the samples in which i's cluster equals c(i) as a set (the cluster signatures of the sMPC).
# Per cluster k: S FL_k = sum of S FL(i) / 2 (the sum is even), S ML_k = sum of S ML(i); the review order is by the
# expected loss t FL_k + (1 - t) ML_k, highest first, ties to the smaller k, compared exactly with t = a / b.  Since
# sum over k of S FL_k = S n(c) - K(c) and sum of S ML_k = 2 (C - K(c)), the sum over k of t FL_k + (1 - t) ML_k / 2 is
# the expected Binder loss of c.
REVIEW_SHARES = (1, 5, 10)  # the first 1 %, 5 % and 10 % of a review queue, in the evaluation


def check_canonical(labels, num_clusters):
    """Raise ValueError unless labels lie in [0, num_clusters) and every cluster holds a record."""
    labels = np.asarray(labels, np.int64)
    C = int(num_clusters)
    if len(labels) and (labels.min() < 0 or labels.max() >= C):
        raise ValueError("a cluster label outside [0, num_clusters)")
    if C < 1 or C > max(len(labels), 1) or (np.bincount(labels, minlength=C) == 0).any():
        raise ValueError("the labels are not canonical: a cluster in [0, num_clusters) holds no record")


class RecordLinks:
    """The integers of dbl_pairs_record_links, int64: per record W, I, the strongest partner outside its cluster (-1
    when there is none) and its count; per cluster the held pairs inside it and their least count (0 when none)."""

    def __init__(self, W, I, partner, partner_count, inner, least):  # noqa: E741
        self.W, self.I, self.partner, self.partner_count, self.inner, self.least = (
            np.asarray(x, np.int64) for x in (W, I, partner, partner_count, inner, least))


def record_links(first, second, count, labels, num_clusters):
    """RecordLinks of the canonical labels[R] (0 .. C-1) against the pair table (first, second, count)
    (pairwise_match_counts): the same integers as analysis_gpu.record_links.  Strongest outside partner: the largest
    count, ties to the smallest partner index."""
    labels = np.asarray(labels, np.int64)
    R, C = len(labels), int(num_clusters)
    check_canonical(labels, C)
    first, second, count = (np.asarray(x, np.int64) for x in (first, second, count))
    W, I = np.zeros(R, np.int64), np.zeros(R, np.int64)  # noqa: E741
    np.add.at(W, first, count)
    np.add.at(W, second, count)
    same = labels[first] == labels[second]
    np.add.at(I, first[same], count[same])
    np.add.at(I, second[same], count[same])
    inner = np.bincount(labels[first[same]], minlength=C).astype(np.int64)
    least = np.full(C, np.iinfo(np.int64).max, np.int64)
    np.minimum.at(least, labels[first[same]], count[same])
    least[inner == 0] = 0
    a, b = np.r_[first[~same], second[~same]], np.r_[second[~same], first[~same]]
    n = np.r_[count[~same], count[~same]]
    by = np.lexsort((b, -n, a))
    lead = by[np.r_[True, a[by][1:] != a[by][:-1]]] if len(by) else by
    partner, partner_count = np.full(R, -1, np.int64), np.zeros(R, np.int64)
    partner[a[lead]], partner_count[a[lead]] = b[lead], n[lead]
    return RecordLinks(W, I, partner, partner_count, inner, least)


def cluster_appearances(chain, labels):
    """A, int64[R]: for the canonical labels[R], the samples of a ChainArrays in which each record's cluster equals
    its cluster in labels as a set, by the cluster signatures of the sMPC (cluster_signatures): the same integers as
    analysis_gpu.cluster_appearances."""
    labels = np.asarray(labels, np.int64)
    R = chain.num_records
    if len(labels) != R:
        raise ValueError("the labels need one cluster label per record")
    C = int(labels.max()) + 1 if R else 0
    check_canonical(labels, C)
    center = ChainArrays(chain.record_ids, np.zeros(1, np.int64), [sample_from_links(labels, np.zeros(C, np.int32))])
    return (cluster_signatures(chain) == cluster_signatures(center)[0]).sum(axis=0).astype(np.int64)


class ClericalReview:
    """The review of a point estimate with canonical labels[R] (0 .. C-1) over S samples, in integers: per record
    S FL, S ML and A; per cluster size, A, S FL, S ML, the least internal count (-1 for a singleton), the strongest
    outside link (inside record, outside record, count; -1, -1, 0 when there is none) and the review order."""

    def __init__(self, links, appearances, labels, num_samples, false_link_cost):
        labels = np.asarray(labels, np.int64)
        S, C = int(num_samples), len(links.inner)
        check_canonical(labels, C)
        self.labels, self.num_samples, self.false_link_cost = labels, S, float(false_link_cost)
        self.size = np.bincount(labels, minlength=C).astype(np.int64)
        self.record_fl = S * (self.size[labels] - 1) - links.I
        self.record_ml = links.W - links.I
        self.record_appearances = np.asarray(appearances, np.int64)
        self.partner, self.partner_count = links.partner, links.partner_count
        self.appearances = np.zeros(C, np.int64)
        self.appearances[labels] = self.record_appearances
        fl2, self.ml = np.zeros(C, np.int64), np.zeros(C, np.int64)
        np.add.at(fl2, labels, self.record_fl)
        np.add.at(self.ml, labels, self.record_ml)
        if (fl2 % 2).any():
            raise ValueError("the false links of a cluster do not add up to an even number")
        self.fl = fl2 // 2
        self.weakest = np.where(self.size == 1, -1, np.where(links.inner == _comb2(self.size), links.least, 0))
        # strongest outside link: over the members' own strongest partners, the largest count, ties to the smaller
        # inside record, then to the smaller outside record (each member's partner is already its smallest of the count)
        has = np.flatnonzero(self.partner >= 0)
        by = has[np.lexsort((self.partner[has], has, -self.partner_count[has], labels[has]))]
        lead = by[np.r_[True, labels[by][1:] != labels[by][:-1]]] if len(by) else by
        self.inside, self.outside = np.full(C, -1, np.int64), np.full(C, -1, np.int64)
        self.outside_count = np.zeros(C, np.int64)
        self.inside[labels[lead]], self.outside[labels[lead]] = lead, self.partner[lead]
        self.outside_count[labels[lead]] = self.partner_count[lead]
        self.order = review_order(self.fl, self.ml, false_link_cost)

    def losses(self):
        """Per cluster t FL_k + (1 - t) ML_k as the float nearest the exact value."""
        a, b = float(self.false_link_cost).as_integer_ratio()
        return [float(fractions.Fraction(a * f + (b - a) * m, b * self.num_samples))
                for f, m in zip(self.fl.tolist(), self.ml.tolist())]


def review_order(fl, ml, false_link_cost):
    """int64[C]: the clusters by expected loss t FL_k + (1 - t) ML_k, highest first, ties to the smaller k, compared
    exactly: t = a / b and the integers a S FL_k + (b - a) S ML_k in Python integers (they may pass int64)."""
    a, b = float(false_link_cost).as_integer_ratio()
    score = [a * f + (b - a) * m for f, m in zip(np.asarray(fl).tolist(), np.asarray(ml).tolist())]
    return np.array(sorted(range(len(score)), key=lambda k: (-score[k], k)), np.int64)


def _ids(record_ids):
    return [str(r) for r in (record_ids.to_pylist() if hasattr(record_ids, "to_pylist") else record_ids)]


def clerical_review_rows(review, record_ids):
    """The rows of clerical-review.csv: per cluster in review order (rank from 1, cluster, size, cluster probability,
    expected false links, expected missed links, expected loss, weakest internal link probability, strongest outside
    link's inside and outside record ids and probability); an empty field where a cluster has no such link."""
    ids, S = _ids(record_ids), review.num_samples
    losses = review.losses()
    rows = []
    for rank, k in enumerate(review.order.tolist(), 1):
        w, i = int(review.weakest[k]), int(review.inside[k])
        rows.append([rank, k, int(review.size[k]), repr(int(review.appearances[k]) / S), repr(int(review.fl[k]) / S),
                     repr(int(review.ml[k]) / S), repr(losses[k]), "" if w < 0 else repr(w / S),
                     "" if i < 0 else ids[i], "" if i < 0 else ids[int(review.outside[k])],
                     "" if i < 0 else repr(int(review.outside_count[k]) / S)])
    return rows


def clerical_review_record_rows(review, record_ids):
    """The rows of clerical-review-records.csv: per record in chain record order (record id, cluster, cluster
    probability, expected false links, expected missed links, strongest outside record id and its probability)."""
    ids, S = _ids(record_ids), review.num_samples
    rows = []
    for r, (k, a, f, m, j, n) in enumerate(zip(review.labels.tolist(), review.record_appearances.tolist(),
                                                review.record_fl.tolist(), review.record_ml.tolist(),
                                                review.partner.tolist(), review.partner_count.tolist())):
        rows.append([ids[r], k, repr(a / S), repr(f / S), repr(m / S), "" if j < 0 else ids[j],
                     "" if j < 0 else repr(n / S)])
    return rows


def erroneous_clusters(labels, truth):
    """bool[C]: the clusters of the canonical labels that are not exactly one true entity."""
    labels = np.asarray(labels, np.int64)
    truth = np.unique(np.asarray(truth), return_inverse=True)[1].reshape(-1).astype(np.int64)
    C, T = (int(labels.max()) + 1 if len(labels) else 0), (int(truth.max()) + 1 if len(truth) else 1)
    cells, n = np.unique(labels * T + truth, return_counts=True)
    cl, tr = cells // T, cells % T
    cells_of = np.bincount(cl, minlength=C)
    single = cells_of[cl] == 1
    correct = np.zeros(C, bool)
    correct[cl[single]] = n[single] == np.bincount(truth, minlength=T)[tr[single]]
    return ~correct


def _found_shares(found, erroneous):
    """The share of the erroneous clusters in the first ceil(p C / 100) of a queue, p in REVIEW_SHARES (NaN when
    there is none)."""
    C = len(found)
    return [found[-(-p * C // 100) - 1] / erroneous if erroneous else float("nan") for p in REVIEW_SHARES]


def clerical_review_evaluation(review, truth):
    """How well the review order finds the clusters that are not exactly a true entity: (rows of
    clerical-review-evaluation.csv -- per queue position its rank, cluster, whether it is erroneous and the erroneous
    clusters found so far -- and a summary dict: clusters, erroneous, the shares found in the first 1 %, 5 % and 10 %
    of the queue, the normalised area under the found-curve and the same shares for the queue by cluster probability
    alone, lowest first, ties to the smaller cluster).  The area is (sum of found(r) - worst) / (best - worst): the
    share of (erroneous, correct) cluster pairs the queue puts in that order; NaN when every or no cluster is
    erroneous."""
    err = erroneous_clusters(review.labels, truth)
    C, E = len(err), int(err.sum())
    found = np.cumsum(err[review.order]).tolist()
    rows = [[r + 1, k, int(err[k]), f] for r, (k, f) in enumerate(zip(review.order.tolist(), found))]
    area = (float(fractions.Fraction(sum(found) - E * (E + 1) // 2, E * (C - E))) if 0 < E < C else float("nan"))
    by_probability = np.lexsort((np.arange(C), review.appearances))
    summary = dict(clusters=C, erroneous=E, found=_found_shares(found, E), area=area,
                   baseline=_found_shares(np.cumsum(err[by_probability]).tolist(), E))
    return rows, summary


# ---- new records linked to a finished chain ----------------------------------------------------------------------
# A query record has value ids x_qa in the data's vocabularies (-1 = missing, or a value the data never holds) and a
# file f(q).  For a sample with clusters k of entity values y_ka and distortion probabilities theta_af, the collapsed
# PCG-II link weight of q against cluster k is w(q, k) = prod over the observed a of
#   g(y) = (1 - theta) [x = y] + theta psi(x) norm(y) expsim(x, y)     (norm(y) = 1/n(y), expsim = 1 off x's sparse row;
#                                                                       norm = expsim = 1 for a constant attribute)
# and an entity no record links to has expected weight m(q) = prod over the observed a of h = psi(x) ((1 - theta) +
# theta sigma(x)), sigma(x) = sum_y psi(y) norm(y) expsim(x, y) (1 for a constant attribute).  With M the population
# size and K the sample's clusters, Z(q) = sum_k w(q, k) + (M - K) m(q).  Weights are carried relative to m:
# rho(q, k) = w / m = prod_a r(y), r = c0 [x = y] + c1 norm(y) expsim(x, y), c0 = (1 - theta) / h, c1 = theta psi(x) / h,
# so log w = log m + log rho and log Z = log m + log(sum_k rho + M - K).  Over the samples s, with L_q = max_s log Z_s
# and Z~ = exp(log Z - L_q):
#   p(q, r) = sum_s w_s(q, c_s(r)) / sum_s Z_s(q),  p_new(q) = sum_s (M - K_s) m_s(q) / sum_s Z_s(q),
#   ESS(q) = (sum_s Z_s)^2 / sum_s Z_s^2.
# p(q, r) >= t needs some sample with w_s >= t Z_s: pass 1 collects those (q, r) as candidates (at most floor(1/t)
# clusters per query and sample), pass 2 sums w over every sample for the candidates only.
MAX_QUERY_CANDIDATES = MAX_PAIRS
QUERY_BLOCK = 1 << 22  # query x cluster entries of one dense block of the numpy scan


class QueryTables:
    """The per-query tables, built once from the attribute indexes: x int32[Q][A] (-1 = missing or unseen), file
    int32[Q], psi and sigma float64[Q][A], the hit rows (x's sparse row: value ids ascending and their expsim) as
    hit_offsets int64[Q A + 1], hit_values, hit_expsim, and per attribute its norm table (ones when constant).
    tables[a] = AttributeIndex.tables() of attribute a; constant[a] = whether it is constant."""

    def __init__(self, x, file, tables, constant, num_files):
        x = np.array(x, np.int32, ndmin=2)
        Q, A = x.shape
        self.x, self.file = x, np.asarray(file, np.int32).reshape(Q)
        self.num_files = int(num_files)
        self.num_values = np.array([len(t["phi"]) for t in tables], np.int32)
        if len(tables) != A or len(constant) != A:
            raise ValueError("one table per matching attribute")
        if Q and (self.file.min() < 0 or self.file.max() >= self.num_files):
            raise ValueError("a query's file is not one of the data's files")
        if ((x < -1) | (x >= self.num_values[None, :])).any():
            raise ValueError("a query value id is outside its attribute's index")
        self.norm = [np.ones(len(t["phi"])) if c else np.asarray(t["norm"], np.float64) for t, c in zip(tables, constant)]
        self.psi, self.sigma = np.zeros((Q, A)), np.ones((Q, A))
        rows = []  # (q, a) -> (values, expsim)
        for a, (t, c) in enumerate(zip(tables, constant)):
            obs = x[:, a] >= 0
            self.psi[obs, a] = np.asarray(t["phi"])[x[obs, a]]
            if c:
                continue
            base = float(np.dot(t["phi"], self.norm[a]))
            for v in np.unique(x[obs, a]):
                lo, hi = t["rowptr"][v], t["rowptr"][v + 1]
                cols, es = np.asarray(t["col"][lo:hi]), np.asarray(t["expsim"][lo:hi])
                keep = es != 1.0
                rows.append((a, int(v), cols[keep], es[keep]))
                self.sigma[x[:, a] == v, a] = base + float(np.dot(t["phi"][cols] * self.norm[a][cols], es - 1.0))
        row_of = {(a, v): (cols, es) for a, v, cols, es in rows}
        lens = np.zeros(Q * A, np.int64)
        for q, a in zip(*np.nonzero(x >= 0)):
            if (a, int(x[q, a])) in row_of:
                lens[q * A + a] = len(row_of[(a, int(x[q, a]))][0])
        self.hit_offsets = np.r_[0, np.cumsum(lens)].astype(np.int64)
        self.hit_values = np.zeros(int(self.hit_offsets[-1]), np.int32)
        self.hit_expsim = np.zeros(int(self.hit_offsets[-1]))
        for i in np.flatnonzero(lens):
            q, a = divmod(int(i), A)
            cols, es = row_of[(a, int(x[q, a]))]
            lo = self.hit_offsets[i]
            order = np.argsort(cols, kind="stable")
            self.hit_values[lo:lo + len(cols)] = cols[order]
            self.hit_expsim[lo:lo + len(cols)] = es[order]

    @property
    def num_queries(self):
        return self.x.shape[0]

    @property
    def num_attributes(self):
        return self.x.shape[1]

    def hits(self, q, a):
        lo, hi = self.hit_offsets[q * self.num_attributes + a], self.hit_offsets[q * self.num_attributes + a + 1]
        return self.hit_values[lo:hi], self.hit_expsim[lo:hi]


def query_coefficients(tab, theta):
    """(c0, c1 float64[Q][A], log m float64[Q]) of one sample's theta[A][F]; c0 = c1 = 0 where x is not observed."""
    theta = np.asarray(theta, np.float64).reshape(tab.num_attributes, tab.num_files)
    th = theta[np.arange(tab.num_attributes)[None, :], tab.file[:, None]]
    obs = tab.x >= 0
    with np.errstate(divide="ignore", invalid="ignore"):
        h = tab.psi * ((1.0 - th) + th * tab.sigma)
        c0 = np.where(obs, (1.0 - th) / h, 0.0)
        c1 = np.where(obs, th * tab.psi / h, 0.0)
        logm = np.zeros(tab.num_queries)
        for a in range(tab.num_attributes):  # attribute order, as on the device
            logm += np.where(obs[:, a], np.log(np.where(obs[:, a], h[:, a], 1.0)), 0.0)
    return c0, c1, logm


def query_rho(tab, coef, values, qs):
    """rho(q, k) float64[len(qs)][K] of the queries qs against the K rows of values int32[K][A]: the product over the
    observed attributes, in attribute order, of c0 [x = y] + c1 norm(y) expsim(x, y)."""
    c0, c1, _ = coef
    values = np.asarray(values)
    qs = np.asarray(qs, np.int64)
    rho = np.ones((len(qs), len(values)))
    for a in range(tab.num_attributes):
        x = tab.x[qs, a]
        obs = x >= 0
        if not obs.any():
            continue
        y = values[:, a]
        t = c1[qs, a][:, None] * tab.norm[a][y][None, :]
        lens = tab.hit_offsets[qs * tab.num_attributes + a + 1] - tab.hit_offsets[qs * tab.num_attributes + a]
        if lens.any():
            E = np.ones((len(qs), tab.num_values[a]))
            for i in np.flatnonzero(lens):
                cols, es = tab.hits(int(qs[i]), a)
                E[i, cols] = es
            t = t * E[:, y]
        r = np.where(y[None, :] == x[:, None], c0[qs, a][:, None], 0.0) + t
        rho *= np.where(obs[:, None], r, 1.0)
    return rho


def _attribute_hit_keys(tab, a):
    """Attribute a's hits of every query as sorted keys q V_a + y, with their expsim."""
    A, Q, V = tab.num_attributes, tab.num_queries, int(tab.num_values[a])
    starts = tab.hit_offsets[np.arange(Q) * A + a]
    n = tab.hit_offsets[np.arange(Q) * A + a + 1] - starts
    idx = np.repeat(starts, n) + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n))
    return np.repeat(np.arange(Q, dtype=np.int64), n) * V + tab.hit_values[idx], tab.hit_expsim[idx]


def query_pair_rho(tab, coef, values, q, k):
    """rho(q[i], k[i]) for pairs (query, cluster): as query_rho, one entry per pair."""
    c0, c1, _ = coef
    q, k = np.asarray(q, np.int64), np.asarray(k, np.int64)
    values = np.asarray(values)
    rho = np.ones(len(q))
    for a in range(tab.num_attributes):
        x = tab.x[q, a]
        y = values[k, a].astype(np.int64)
        t = c1[q, a] * tab.norm[a][y]
        keys, es = _attribute_hit_keys(tab, a)
        if len(keys):
            want = q * int(tab.num_values[a]) + y
            pos = np.minimum(np.searchsorted(keys, want), len(keys) - 1)
            t = np.where(keys[pos] == want, t * es[pos], t)
        rho *= np.where(x >= 0, np.where(y == x, c0[q, a], 0.0) + t, 1.0)
    return rho


def _check_min_link_probability(t):
    if isinstance(t, bool) or not isinstance(t, (int, float)) or not 0.0 < float(t) <= 1.0:
        raise ValueError("minLinkProbability must be in (0, 1].")
    return float(t)


def check_query_sample(tab, labels, values, theta, num_records, population_size):
    """The refusals of both passes for one sample: (labels int64[R] in [0, K), values int32[K][A], theta[A][F])."""
    labels, values = np.asarray(labels), np.asarray(values)
    theta = np.asarray(theta, np.float64)
    K = len(values)
    if labels.shape != (num_records,) or values.ndim != 2 or values.shape[1] != tab.num_attributes:
        raise ValueError("a sample needs one cluster label per record and one value row per cluster")
    if K < 1 or K > population_size:
        raise ValueError(f"a sample has {K} clusters, more than the population size {population_size}"
                         if K else "a sample has no clusters")
    if labels.min() < 0 or labels.max() >= K or (np.bincount(labels, minlength=K) == 0).any():
        raise ValueError("a sample's cluster labels must cover [0, K) exactly")
    if ((values < 0) | (values >= tab.num_values[None, :])).any():
        raise ValueError("an entity value id is outside its attribute's index")
    if theta.size != tab.num_attributes * tab.num_files or not ((theta >= 0.0) & (theta <= 1.0)).all():
        raise ValueError("distortion probabilities must be [A][F] values in [0, 1]")


class QueryResult:
    """What both passes give: the candidates (query, record) in (query, record) order with their sums, and per query
    L_q, sum Z~, sum Z~^2, the new-entity sum and every sample's log Z ([S][Q])."""

    def __init__(self, query, record, sums, scale, zsum, zsq, fresh, logz):
        self.query, self.record, self.sums = np.asarray(query, np.int64), np.asarray(record, np.int64), sums
        self.scale, self.zsum, self.zsq, self.fresh, self.logz = scale, zsum, zsq, fresh, logz

    @property
    def probability(self):
        return self.sums / self.zsum[self.query]

    @property
    def new_entity_probability(self):
        return self.fresh / self.zsum

    @property
    def effective_samples(self):
        return self.zsum * self.zsum / self.zsq


class QueryScores:
    """The numpy path of the two passes (analysis_gpu.Query is the device's): add_sample for every sample (pass 1),
    then score_sample for the same samples in the same order (pass 2), then read()."""

    def __init__(self, tables, num_records, population_size, min_link_probability,
                 max_candidates=MAX_QUERY_CANDIDATES):
        self.tab, self.R, self.M = tables, int(num_records), int(population_size)
        self.t = _check_min_link_probability(min_link_probability)
        self.max_candidates = int(max_candidates)
        self.logz, self.logm, self.kcount = [], [], []
        self.keys = np.zeros(0, np.int64)
        self.S2, self.sums, self.scale = 0, None, None

    @property
    def num_samples(self):
        return len(self.logz)

    def add_sample(self, labels, values, theta):
        if self.S2:
            raise ValueError("pass 2 has begun")
        check_query_sample(self.tab, labels, values, theta, self.R, self.M)
        labels, values = np.asarray(labels, np.int64), np.asarray(values)
        tab, K, Q = self.tab, len(values), self.tab.num_queries
        coef = query_coefficients(tab, theta)
        step = max(1, QUERY_BLOCK // max(K, 1))
        total = np.zeros(Q)
        emitted = []
        for lo in range(0, Q, step):
            qs = np.arange(lo, min(Q, lo + step))
            rho = query_rho(tab, coef, values, qs)
            s = rho.sum(axis=1) + (self.M - K)
            total[qs] = s
            qi, ki = np.nonzero(rho >= self.t * s[:, None])
            emitted.append((qs[qi], ki))
        with np.errstate(divide="ignore"):
            logz = coef[2] + np.log(total)
        q = np.concatenate([e[0] for e in emitted]).astype(np.int64)
        k = np.concatenate([e[1] for e in emitted]).astype(np.int64)
        order = np.argsort(labels, kind="stable")
        start = np.searchsorted(labels[order], np.arange(K))
        size = np.bincount(labels, minlength=K)
        n = size[k]
        rec = order[np.repeat(start[k], n) + (np.arange(n.sum()) - np.repeat(np.cumsum(n) - n, n))]
        new = np.union1d(self.keys, (np.repeat(q, n) << 32) | rec)
        if len(new) > self.max_candidates:
            raise ValueError(f"more than {self.max_candidates} candidate (query, record) pairs: raise "
                             f"minLinkProbability")
        self.keys = new
        self.logz.append(logz)
        self.logm.append(coef[2])
        self.kcount.append(K)

    def score_sample(self, labels, values, theta):
        if self.S2 >= self.num_samples:
            raise ValueError("pass 2 has more samples than pass 1")
        if len(values) != self.kcount[self.S2]:
            raise ValueError("pass 2 must score the samples of pass 1, in the same order")
        check_query_sample(self.tab, labels, values, theta, self.R, self.M)
        if self.S2 == 0:
            self.scale = np.max(np.asarray(self.logz), axis=0)
            self.sums = np.zeros(len(self.keys))
        labels = np.asarray(labels, np.int64)
        coef = query_coefficients(self.tab, theta)
        q, r = self.keys >> 32, self.keys & 0xffffffff
        with np.errstate(divide="ignore"):
            self.sums += np.exp(coef[2][q] + np.log(query_pair_rho(self.tab, coef, values, q, labels[r])) -
                                self.scale[q])
        self.S2 += 1

    def read(self):
        if self.num_samples == 0 or self.S2 != self.num_samples:
            raise ValueError("pass 2 must score every sample of pass 1 before the results are read")
        logz, logm = np.asarray(self.logz), np.asarray(self.logm)
        zt = np.exp(logz - self.scale[None, :])
        un = self.M - np.asarray(self.kcount, np.int64)
        with np.errstate(divide="ignore"):
            fresh = np.where(un[:, None] > 0, np.exp(np.log(np.maximum(un, 1))[:, None] + logm - self.scale[None, :]),
                             0.0)
        zsum, zsq, fsum = np.zeros(len(self.scale)), np.zeros(len(self.scale)), np.zeros(len(self.scale))
        for s in range(len(zt)):  # sample order, as on the device
            zsum += zt[s]
            zsq += zt[s] * zt[s]
            fsum += fresh[s]
        return QueryResult(self.keys >> 32, self.keys & 0xffffffff, self.sums, self.scale, zsum, zsq, fsum, logz)


def query_sample_arrays(num_records, members, offsets, values):
    """(labels int64[R] in [0, K), cluster values int32[K][A]) of one sample: members / offsets of the chain and the
    per-record values int32[A][R] read_entity_values gives."""
    members = np.asarray(members)
    sizes = np.diff(np.asarray(offsets, np.int64))
    labels = np.full(num_records, -1, np.int64)
    labels[members] = np.repeat(np.arange(len(sizes)), sizes)
    return labels, np.ascontiguousarray(np.asarray(values)[:, members[np.asarray(offsets[:-1], np.int64)]].T,
                                        np.int32)


def link_queries(tables, samples, num_records, population_size, min_link_probability, scorer=QueryScores):
    """Both passes over the samples: samples() yields (labels, values[K][A], theta[A][F]) per sample, the same each time
    it is called; scorer = QueryScores or analysis_gpu.Query.  Returns the QueryResult."""
    if scorer is QueryScores:
        qs = scorer(tables, num_records, population_size, min_link_probability)
        return _two_passes(qs, samples)
    with scorer(tables, num_records, population_size, min_link_probability) as qs:
        return _two_passes(qs, samples)


def _two_passes(qs, samples):
    for s in samples():
        qs.add_sample(*s)
    if qs.num_samples == 0:
        raise ValueError("linking records needs at least one sample at or after lowerIterationCutoff")
    for s in samples():
        qs.score_sample(*s)
    return qs.read()


def query_link_rows(result, min_link_probability, data_position):
    """The reported pairs: (query, record, p) with p >= t, in query order, then p descending, then the record's data
    position (data_position[r] = its row in the data file)."""
    p = result.probability
    keep = p >= min_link_probability
    q, r, p = result.query[keep], result.record[keep], p[keep]
    order = np.lexsort((np.asarray(data_position)[r], -p, q))
    return q[order], r[order], p[order]


def read_distortion_probabilities(chain_dirs, chain, num_attributes, num_files):
    """float64[S][A][F]: theta of every sample of `chain` (pooled as read_entity_values takes it), from each chain
    directory's distortion-probabilities-chain.csv.  Raises ValueError for a sample past the cutoff without a row, or
    a file whose columns are not A F."""
    import csv

    rows = {}
    out = np.empty((len(chain.samples), num_attributes, num_files))
    for s, (it, k) in enumerate(zip(chain.iterations, chain.chains)):
        k = int(k)
        if k not in rows:
            rows[k] = {}
            path = os.path.join(chain_dirs[k], "distortion-probabilities-chain.csv")
            if os.path.exists(path):
                with open(path, newline="") as fh:
                    rd = csv.reader(fh)
                    head = next(rd, None)
                    if head is None or len(head) != 1 + num_attributes * num_files:
                        raise ValueError(f"{path}: expected iteration and {num_attributes * num_files} columns")
                    for row in rd:
                        rows[k][int(row[0])] = [float(v) for v in row[1:]]
        got = rows[k].get(int(it))
        if got is None:
            raise ValueError(f"the sample at iteration {int(it)} has no distortion probabilities (it was recorded with "
                             f"saveDistortionProbabilities off): raise lowerIterationCutoff past it, or sample again "
                             f"with saveDistortionProbabilities on")
        out[s] = np.asarray(got).reshape(num_attributes, num_files)
    return out


def distortion_summary(theta):
    """Per (attribute, file), attribute-major: (mean, sd, 2.5 %, 50 %, 97.5 % quantiles) of theta[S][A][F] over the
    samples (numpy quantile, default method; sd with ddof 0) and S."""
    theta = np.asarray(theta, np.float64)
    S = theta.shape[0]
    if S == 0:
        raise ValueError("distortion-probabilities needs at least one sample at or after lowerIterationCutoff")
    flat = theta.reshape(S, -1)
    q = np.quantile(flat, [0.025, 0.5, 0.975], axis=0)
    return [(float(flat[:, j].mean()), float(flat[:, j].std()), float(q[0, j]), float(q[1, j]), float(q[2, j]), S)
            for j in range(flat.shape[1])]


# ---- capture histories: how the files overlap ---------------------------------------------------------------------
# Files are numbered f = 0 .. F-1 (RecordsCache.file_ids order).  Per sample s and cluster c the history is
# h(c) = OR over records r of c of (1 << file[r]), a non-empty subset of the files:
#   H[s][h]  the clusters of sample s whose history is h (H[s][0] = 0), and
#   L[r][g]  the samples in which r's cluster holds a record of file g other than r itself,
# so L / S is the probability that r has a counterpart in file g (a duplicate in its own file when g = file[r]).  Every
# number written is computed from H and L by CaptureSummary, whichever path counted them.
MAX_CAPTURE_FILES = 12  # 2^12 histories: the GPU's shared-memory histogram


def check_capture_files(num_files):
    """ValueError unless 1 <= F <= MAX_CAPTURE_FILES."""
    if not 1 <= int(num_files) <= MAX_CAPTURE_FILES:
        raise ValueError(f"capture-histories supports 1 to {MAX_CAPTURE_FILES} files (2^F histories); the data has "
                         f"{int(num_files)}")


class CaptureCounts:
    """The numpy counter with analysis_gpu.Capture's interface: add_sample(cluster[R]) per sample, read() gives
    (H int64[S, 2^F], L int64[R, F])."""

    def __init__(self, file, num_files):
        check_capture_files(num_files)
        self.file = np.asarray(file, np.int64)
        self.F = int(num_files)
        if len(self.file) and (self.file.min() < 0 or self.file.max() >= self.F):
            raise ValueError("a file number is outside [0, F)")
        self.H = []
        self.L = np.zeros((len(self.file), self.F), np.int64)

    def add_sample(self, cluster):
        R, F, file = len(self.file), self.F, self.file
        lab = np.asarray(cluster, np.int64)
        if lab.shape != (R,) or (R and (lab.min() < 0 or lab.max() >= R)):
            raise ValueError("a sample needs one cluster label in [0, R) per record")
        bit = np.left_shift(1, file)
        hist = np.zeros(R, np.int64)
        np.bitwise_or.at(hist, lab, bit)
        twice = np.bincount(lab * F + file, minlength=R * F).reshape(R, F) >= 2
        dup = (twice << np.arange(F)).sum(axis=1)
        self.H.append(np.bincount(hist[hist > 0], minlength=1 << F))
        links = (hist[lab] & ~bit) | (dup[lab] & bit)
        self.L += (links[:, None] >> np.arange(F)) & 1

    @property
    def num_samples(self):
        return len(self.H)

    def read(self):
        return np.asarray(self.H, np.int64).reshape(-1, 1 << self.F), self.L.copy()


def capture_histories(chain, file, num_files, counter=CaptureCounts):
    """(H int64[S, 2^F], L int64[R, F]) of a ChainArrays whose record i is in file[i]; counter = CaptureCounts or
    analysis_gpu.Capture."""
    R = chain.num_records
    if not chain.samples:
        raise ValueError("capture-histories needs at least one sample at or after lowerIterationCutoff")
    cc = counter(file, num_files)
    try:
        for mem, off, _ in chain.samples:
            lab = np.empty(R, np.int32)
            lab[mem] = np.repeat(np.arange(len(off) - 1, dtype=np.int32), np.diff(off))
            cc.add_sample(lab)
        return cc.read()
    finally:
        if hasattr(cc, "close"):
            cc.close()


def independence_estimate(n, D):
    """Darroch's (1958) Mt estimate of the population size per row: n int64[S, F] entities per file, D int64[S]
    observed entities.  It maximises the conditional likelihood of the independence model with the capture
    probabilities profiled out, l(N) = (1 - F) N log N - (N - D) log(N - D) + sum_f (N - n_f) log(N - n_f), whose
    derivative is g(N) = sum_f log1p(-n_f / N) - log1p(-D / N): the root of g on N > D, found by bisection on x = D / N
    in (0, 1) to the last bit.  +inf when sum_f n_f = D (no file overlaps another); D when a file holds every observed
    entity (g < 0 on N > D, so l falls from N = D)."""
    n = np.asarray(n, np.float64)
    D = np.asarray(D, np.float64)
    S = len(D)
    out = np.full(S, np.inf)
    total = n.sum(axis=1)
    finite = total > D
    whole = finite & (n.max(axis=1, initial=0.0) >= D)
    out[whole] = D[whole]
    todo = np.flatnonzero(finite & ~whole)
    a = n[todo] / D[todo, None]
    lo, hi = np.zeros(len(todo)), np.ones(len(todo))
    for _ in range(2000):
        mid = 0.5 * (lo + hi)
        live = (mid > lo) & (mid < hi)
        if not live.any():
            break
        g = np.log1p(-mid[:, None] * a).sum(axis=1) - np.log1p(-mid)
        up = live & (g > 0)
        hi = np.where(up, mid, hi)
        lo = np.where(live & ~up, mid, lo)
    out[todo] = D[todo] / (0.5 * (lo + hi))
    return out


def _moments(v):
    """(mean, sd with ddof 0, 2.5 %, 50 %, 97.5 % quantiles -- numpy's default method, as distortion_summary) over the
    finite values of v, NaN when there is none, and the number of infinite ones."""
    v = np.asarray(v, np.float64)
    f = v[np.isfinite(v)]
    if not len(f):
        return (float("nan"),) * 5 + (len(v),)
    q = np.quantile(f, [0.025, 0.5, 0.975])
    return (float(f.mean()), float(f.std()), float(q[0]), float(q[1]), float(q[2]), int(len(v) - len(f)))


class CaptureSummary:
    """Every number the capture-histories files hold, from H[S, 2^F], L[R, F] and the records of each file:
    per sample the quantities (quantity names and int64 or float64 columns, in population-size.csv's order) and their
    summaries, the history summaries and the record link probabilities L / S."""

    def __init__(self, H, L, records_per_file):
        H = np.asarray(H, np.int64)
        self.H, self.L = H, np.asarray(L, np.int64)
        self.S, cells = H.shape
        self.F = F = cells.bit_length() - 1
        self.records_per_file = np.asarray(records_per_file, np.int64)
        hs = np.arange(cells)
        member = ((hs[:, None] >> np.arange(F)) & 1).astype(np.int64)  # [2^F, F]
        self.histories = member[1:]
        D = H.sum(axis=1)
        n = H @ member
        names, cols = ["observed-entities"], [D]
        names += [f"entities[{f}]" for f in range(F)]
        cols += [n[:, f] for f in range(F)]
        names += [f"duplicates[{f}]" for f in range(F)]
        cols += [self.records_per_file[f] - n[:, f] for f in range(F)]
        pairs = [(f, g) for f in range(F) for g in range(f + 1, F)]
        m = {(f, g): H @ (member[:, f] & member[:, g]) for f, g in pairs}
        names += [f"overlap[{f},{g}]" for f, g in pairs]
        cols += [m[p] for p in pairs]
        names += [f"chapman[{f},{g}]" for f, g in pairs]
        cols += [(n[:, f] + 1.0) * (n[:, g] + 1.0) / (m[(f, g)] + 1.0) - 1.0 for f, g in pairs]
        if F >= 2:
            names.append("independence")
            cols.append(independence_estimate(n, D))
        self.names, self.columns = names, cols

    def quantity_names(self, file_ids):
        """The quantity names with file numbers replaced by file ids."""
        out = []
        for name in self.names:
            if "[" in name:
                head, idx = name[:-1].split("[")
                out.append(head + "[" + ",".join(str(file_ids[int(i)]) for i in idx.split(",")) + "]")
            else:
                out.append(name)
        return out

    def quantity_summary(self):
        """Per quantity (mean, sd, q2.5, q50, q97.5, infinite)."""
        return [_moments(c) for c in self.columns]

    def history_summary(self):
        """Per history h = 1 .. 2^F - 1 (mean, sd, q2.5, q50, q97.5) of its cluster count, zeros included."""
        return [_moments(self.H[:, h])[:5] for h in range(1, self.H.shape[1])]

    def link_probabilities(self):
        """float64[R, F]: L / S."""
        return self.L / self.S


def capture_evaluation(post, truth):
    """The posterior against the ground truth (both CaptureSummary; truth of one sample): (rows of
    capture-histories-evaluation.csv -- per history, then per quantity: index, truth, posterior mean, 2.5 % and
    97.5 % quantiles, truth inside the interval -- and a summary dict: histories and quantities with the truth inside,
    the truth's observed entities and independence estimate with their posterior summaries, and the Brier score of
    L / S against the truth's 0/1 links per file)."""
    rows_h, rows_q = [], []
    for h, (mean, _, lo, _, hi) in enumerate(post.history_summary(), start=1):
        t = int(truth.H[0, h])
        rows_h.append((h, t, mean, lo, hi, bool(lo <= t <= hi)))
    for j, (col, (mean, _, lo, _, hi, _)) in enumerate(zip(truth.columns, post.quantity_summary())):
        t = col[0].item()
        rows_q.append((j, t, mean, lo, hi, bool(lo <= t <= hi)))
    brier = ((post.link_probabilities() - truth.L) ** 2).mean(axis=0) if len(post.L) else np.full(post.F, np.nan)
    summary = dict(samples=post.S, histories=len(rows_h), histories_inside=sum(r[5] for r in rows_h),
                   quantities=len(rows_q), quantities_inside=sum(r[5] for r in rows_q),
                   observed=(rows_q[0][1], post.quantity_summary()[0]), brier=[float(b) for b in brier])
    if "independence" in post.names:
        j = post.names.index("independence")
        summary["independence"] = (float(truth.columns[j][0]), post.quantity_summary()[j])
    return rows_h, rows_q, summary
