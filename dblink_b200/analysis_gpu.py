"""Posterior summaries of chains of millions of records on the GPU: the shared most probable clusters
(LinkageChain.scala:52-95) and the pairwise match counts.

Same results as analysis_arrays.shared_most_probable_clusters / most_probable_signature, bit for bit: the device
computes the same 64-bit cluster signatures (dbl_posterior.cu), the same per-record mode with ties going to the
earliest sample, and the same smallest-record-index labels.  The (S x R) signature matrix lives in device memory,
filled one sample at a time; the host only turns each sample's (members, offsets) into a cluster label per record.
The pairwise match counts equal analysis_arrays.pairwise_match_counts exactly: the device keeps the sorted table of
(pair, count) and merges each sample's pairs into it.  The per-sample counts against the ground truth equal
analysis_arrays.posterior_metric_counts exactly: they are integers, counted on the device from one radix sort of
(sample label, true label) per record.  The Binder-loss counts (n, K) per sample equal analysis_arrays.binder_counts
exactly: every sample goes into one pairs table, then every sample is scored against it.  The Binder search
(single-record moves from a start) equals analysis_arrays.binder_search exactly, in labels, round logs, n and K: the
rule is in integers, and the device applies it to the same table.  The cell histograms of the variation-of-information
estimate equal analysis_arrays.vi_cross_histograms exactly: they are integers, counted on the device from radix-sorted
(sample, label, label) keys of every pair of held samples.  The VI search (single-record moves on a quantised table)
and the cells of any labelling with every held sample, summed or per sample, equal analysis_arrays.vi_search_rounds /
vi_label_cells / vi_sample_cells exactly, on the same handle.  The entity-value counts of a point estimate's clusters
equal analysis_arrays.EntityValueCounts exactly: the device keeps the sorted table of (cluster, value) keys and int64
counts per attribute and merges each sample's run-length-encoded keys into it; the modes are a segmented arg-max.
The per-pair split-R̂ and ESS equal analysis_arrays.pairwise_match_diagnostics bit for bit: a bit trace per held pair,
then integer lag statistics and the same rounded double operations per pair on the device.  The links of every record
against a point estimate and the appearances of its clusters, for clerical review, equal analysis_arrays.record_links
and cluster_appearances exactly: integer atomics over the held pair table, and the sMPC's signatures compared.  The
capture histories and record links equal analysis_arrays.capture_histories exactly: integer atomics on per-cluster
file words, then a shared-memory histogram of the words.
"""
import ctypes as C

import numpy as np

from . import _lib
from . import analysis_arrays
from .analysis_arrays import (MAX_PAIRS, SearchRun, VISearchRun, check_search_size, check_vi_search_size,
                              check_vi_search_squares, search_choice, search_cost, too_many_pairs, vi_sample_squares,
                              vi_search_choice, vi_search_table, vi_width)
from .engine import DblinkError

_STATUS = {_lib.ERR_INVALID: "invalid argument (bad size, label out of range, too many samples or pairs)",
           _lib.ERR_CUDA: "CUDA failure (no device, or a device buffer does not fit on it)",
           _lib.ERR_STATE: "no sample added"}


def _check(rc, what):
    if rc == _lib.OK:
        return
    err = DblinkError(f"{what}: {_STATUS.get(rc, 'error %d' % rc)}")
    err.status = rc
    raise err


def sample_clusters(num_records, members, offsets):
    """One sample as int32 cluster[R]: the position of each record's cluster in (members, offsets)."""
    R = num_records
    members = np.asarray(members)
    offsets = np.asarray(offsets, np.int64)
    if len(members) != R or (R and (members.min() < 0 or members.max() >= R)):
        raise ValueError("every sample must mention every record exactly once")
    cluster = np.full(R, -1, np.int32)
    cluster[members] = np.repeat(np.arange(len(offsets) - 1, dtype=np.int32), np.diff(offsets))
    if (cluster < 0).any():  # R members, one record missing: another is mentioned twice
        raise ValueError("every sample must mention every record exactly once")
    return cluster


class _Handle:
    """Owner of one handle of dbl_posterior.cu, whose C functions are named <_prefix>_<name>: samples go in one at a
    time, close() (or leaving a with block) frees it."""

    _prefix = None

    def __init__(self, num_records, *create_args):
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.num_records = int(num_records)
        self._call("create", C.byref(self._h), self.num_records, *create_args)

    def _fn(self, name):
        return getattr(self._lib, f"{self._prefix}_{name}")

    def _call(self, name, *args):
        _check(self._fn(name)(*args), f"{self._prefix}_{name}")

    def add_sample(self, cluster):
        cluster = np.ascontiguousarray(cluster, np.int32)
        if cluster.shape != (self.num_records,):
            raise ValueError("a sample needs one cluster label per record")
        self._call("add_sample", self._h, cluster.ctypes.data)

    @property
    def num_samples(self):
        return self._fn("num_samples")(self._h)

    def close(self):
        if self._h:
            self._fn("free")(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()


def _add_chain(handle, chain):
    """Every sample of a ChainArrays into handle, in chain order."""
    for mem, off, _ in chain.samples:
        handle.add_sample(sample_clusters(handle.num_records, mem, off))


class Posterior(_Handle):
    """Owner of a dbl_posterior handle: samples go in one at a time, smpc() reads the summary."""

    _prefix = "dbl_posterior"

    def __init__(self, num_records, max_samples):
        super().__init__(num_records, int(max_samples))

    def smpc(self):
        """(labels int64[R], freq float64[R])."""
        labels = np.empty(self.num_records, np.int32)
        freq = np.empty(self.num_records, np.float64)
        self._call("smpc", self._h, labels.ctypes.data_as(_lib.i32p), freq.ctypes.data_as(_lib.f64p))
        return labels.astype(np.int64), freq

    def cluster_counts(self, labels, num_clusters):
        """A, int64[R]: for labels[R] canonical in [0, num_clusters), the held samples in which each record's cluster
        equals its cluster in labels as a set."""
        labels = np.ascontiguousarray(labels, np.int32)
        if labels.shape != (self.num_records,):
            raise ValueError("the labels need one cluster label per record")
        count = np.empty(self.num_records, np.int32)
        self._call("cluster_counts", self._h, labels.ctypes.data, int(num_clusters), count.ctypes.data)
        return count.astype(np.int64)


def most_probable_clusters(chain):
    """(labels, freq) of a ChainArrays: labels = the sMPC labels (the smallest record index of each group of records
    sharing their most probable cluster), freq = how often each record is in its most probable cluster."""
    R = chain.num_records
    if R == 0:
        return np.zeros(0, np.int64), np.zeros(0)
    with Posterior(R, len(chain.samples)) as post:
        _add_chain(post, chain)
        return post.smpc()


def shared_most_probable_clusters(chain):
    """int64 labels[R], identical to analysis_arrays.shared_most_probable_clusters(chain)."""
    return most_probable_clusters(chain)[0]


class Pairs(_Handle):
    """Owner of a dbl_pairs handle: samples go in one at a time, read() gives the pairwise match counts."""

    _prefix = "dbl_pairs"

    def __init__(self, num_records, max_pairs=MAX_PAIRS):
        super().__init__(num_records, int(max_pairs))

    def count(self, min_count=1):
        n = C.c_int64()
        self._call("count", self._h, int(min_count), C.byref(n))
        return n.value

    def read(self, min_count=1):
        """(first, second, count), int64, the pairs with count >= min_count in ascending (first, second) order."""
        n = self.count(min_count)
        out = [np.empty(n, np.int32) for _ in range(3)]
        if n:
            self._call("read", self._h, int(min_count), *(a.ctypes.data for a in out))
        return tuple(a.astype(np.int64) for a in out)

    def score_sample(self, cluster):
        """(n, K) of any labelling cluster[R] against the held table: the pairs it puts together and the sum of their
        counts (0 for a pair the table does not hold).  The table does not change."""
        cluster = np.ascontiguousarray(cluster, np.int32)
        if cluster.shape != (self.num_records,):
            raise ValueError("a sample needs one cluster label per record")
        n, K = C.c_int64(), C.c_int64()
        self._call("score_sample", self._h, cluster.ctypes.data, C.byref(n), C.byref(K))
        return n.value, K.value

    def binder_search(self, a, b, start, max_rounds):
        """The single-record-move search from labels start[R] against the held table at t = a / b: an
        analysis_arrays.SearchRun.  The table does not change."""
        start = np.ascontiguousarray(start, np.int32)
        if start.shape != (self.num_records,):
            raise ValueError("a start needs one cluster label per record")
        max_rounds = int(max_rounds)
        labels = np.empty(self.num_records, np.int32)
        logs = [np.zeros(max(max_rounds, 0), np.int64) for _ in range(3)]
        rounds, converged, n, K = C.c_int32(), C.c_int32(), C.c_int64(), C.c_int64()
        self._call("binder_search", self._h, int(a), int(b), start.ctypes.data, max_rounds, labels.ctypes.data,
                   C.byref(rounds), C.byref(converged), *(x.ctypes.data_as(_lib.i64p) for x in logs), C.byref(n),
                   C.byref(K))
        return SearchRun(labels.astype(np.int64), *(x[:rounds.value] for x in logs), converged.value, n.value, K.value)

    def trace_begin(self, num_positions):
        """A zeroed bit trace of num_positions bits per held pair (dropped by the next add_sample)."""
        self._call("trace_begin", self._h, int(num_positions))

    def trace_sample(self, cluster, position):
        """Sets bit `position` of every held pair that labelling cluster[R] puts together."""
        cluster = np.ascontiguousarray(cluster, np.int32)
        if cluster.shape != (self.num_records,):
            raise ValueError("a sample needs one cluster label per record")
        self._call("trace_sample", self._h, cluster.ctypes.data, int(position))

    def mixing(self, min_count, starts, draws, floor):
        """An analysis_arrays.MatchMixing of the held pairs with count >= min_count, in read() order, over the chains
        of `draws` trace positions from starts[k]."""
        starts = np.ascontiguousarray(starts, np.int32)
        n = self.count(min_count)
        i32 = [np.empty(n, np.int32) for _ in range(4)]
        f64 = [np.empty(n, np.float64) for _ in range(2)]
        self._call("mixing", self._h, int(min_count), len(starts), starts.ctypes.data_as(_lib.i32p), int(draws),
                   float(floor), *(a.ctypes.data for a in i32 + f64))
        return analysis_arrays.MatchMixing(*(a.astype(np.int64) for a in i32), *f64, 2 * len(starts), int(draws))

    def record_links(self, labels, num_clusters):
        """An analysis_arrays.RecordLinks of labels[R], canonical in [0, num_clusters), against the held table.  The
        table does not change."""
        labels = np.ascontiguousarray(labels, np.int32)
        if labels.shape != (self.num_records,):
            raise ValueError("the labels need one cluster label per record")
        R, C = self.num_records, int(num_clusters)
        W, I, inner = np.empty(R, np.int64), np.empty(R, np.int64), np.empty(max(C, 0), np.int64)  # noqa: E741
        partner, partner_count, least = np.empty(R, np.int32), np.empty(R, np.int32), np.empty(max(C, 0), np.int32)
        self._call("record_links", self._h, labels.ctypes.data, C,
                   *(a.ctypes.data for a in (W, I, partner, partner_count, inner, least)))
        return analysis_arrays.RecordLinks(W, I, partner, partner_count, inner, least)


def _add_pairs(pairs, chain, max_pairs):
    """Every sample of a ChainArrays into a Pairs handle; the cap refusal as analysis_arrays raises it."""
    try:
        _add_chain(pairs, chain)
    except DblinkError as e:  # the labels are valid, so DBL_ERR_INVALID means the cap
        if e.status == _lib.ERR_INVALID:
            raise too_many_pairs(max_pairs) from e
        raise


def pairwise_match_counts(chain, max_pairs=MAX_PAIRS, min_count=1):
    """(first, second, count), identical to analysis_arrays.pairwise_match_counts(chain, max_pairs, min_count)."""
    R = chain.num_records
    if R == 0 or not chain.samples:
        return tuple(np.zeros(0, np.int64) for _ in range(3))
    with Pairs(R, max_pairs) as pairs:
        _add_pairs(pairs, chain, max_pairs)
        return pairs.read(min_count)


def binder_counts(chain, max_pairs=MAX_PAIRS):
    """(n, K), int64[S], identical to analysis_arrays.binder_counts(chain, max_pairs): pass 1 adds every sample to one
    handle, pass 2 scores every sample against the full table."""
    R, S = chain.num_records, len(chain.samples)
    n, K = np.zeros(S, np.int64), np.zeros(S, np.int64)
    if R == 0 or S == 0:
        return n, K
    with Pairs(R, max_pairs) as pairs:
        _add_pairs(pairs, chain, max_pairs)
        for s, (mem, off, _) in enumerate(chain.samples):
            n[s], K[s] = pairs.score_sample(sample_clusters(R, mem, off))
    return n, K


def pairwise_match_diagnostics(chain, min_count=1, max_pairs=MAX_PAIRS):
    """(first, second, count, MatchMixing), identical to analysis_arrays.pairwise_match_diagnostics(chain, min_count,
    max_pairs), refusals included: pass 1 adds every sample to one handle, the trace pass marks every pooled sample's
    held pairs, then one mixing call."""
    starts, n = analysis_arrays.chain_draws(chain)
    analysis_arrays.check_mixing_size(len(starts), n)
    R, S = chain.num_records, len(chain.samples)
    with Pairs(R, max_pairs) as pairs:
        _add_pairs(pairs, chain, max_pairs)
        analysis_arrays.check_trace_size(S, pairs.count())
        pairs.trace_begin(S)
        for s, (mem, off, _) in enumerate(chain.samples):
            pairs.trace_sample(sample_clusters(R, mem, off), s)
        first, second, count = pairs.read(min_count)
        mix = pairs.mixing(min_count, starts, n, analysis_arrays.ess_floor(len(starts), n))
    return first, second, count, mix


def record_links(chain, labels, max_pairs=MAX_PAIRS):
    """RecordLinks of the canonical labels[R] (0 .. C-1), identical to analysis_arrays.record_links(
    *analysis_arrays.pairwise_match_counts(chain, max_pairs), labels, C): every sample goes into one handle, then one
    pass over its table."""
    labels = np.asarray(labels, np.int64)
    R = chain.num_records
    with Pairs(R, max_pairs) as pairs:
        _add_pairs(pairs, chain, max_pairs)
        return pairs.record_links(labels, int(labels.max()) + 1)


def cluster_appearances(chain, labels):
    """A, int64[R], identical to analysis_arrays.cluster_appearances(chain, labels): every sample's signatures go
    into one dbl_posterior handle, then every record's row is compared with the signature of its cluster in labels."""
    labels = np.asarray(labels, np.int64)
    with Posterior(chain.num_records, len(chain.samples)) as post:
        _add_chain(post, chain)
        return post.cluster_counts(labels, int(labels.max()) + 1)


def binder_search(chain, false_link_cost, starts, max_rounds=1000, max_pairs=MAX_PAIRS):
    """(chosen position, SearchRuns), identical to analysis_arrays.binder_search(chain, false_link_cost, starts,
    max_rounds, max_pairs): pass 1 adds every sample to one handle, then the search runs from each start on it."""
    R, S = chain.num_records, len(chain.samples)
    check_search_size(S, R)
    a, b = search_cost(false_link_cost)
    with Pairs(R, max_pairs) as pairs:
        _add_pairs(pairs, chain, max_pairs)
        runs = [pairs.binder_search(a, b, st, max_rounds) for st in starts]
    return search_choice(runs, S, a, b), runs


class Evaluation(_Handle):
    """Owner of a dbl_eval handle: the ground truth goes in once, samples one at a time, read() gives the per-sample
    counts."""

    _prefix = "dbl_eval"

    def __init__(self, num_records, truth, max_samples):
        truth = np.ascontiguousarray(truth, np.int32)
        if truth.shape != (int(num_records),):
            raise ValueError("the ground truth needs one label per record")
        super().__init__(num_records, truth.ctypes.data, int(max_samples))

    def read(self):
        """(tp, pred_pairs, num_clusters), int64[S]."""
        out = [np.empty(self.num_samples, np.int64) for _ in range(3)]
        self._call("read", self._h, *(a.ctypes.data_as(_lib.i64p) for a in out))
        return tuple(out)


def posterior_metric_counts(chain, truth):
    """(tp, pred_pairs, num_clusters), identical to analysis_arrays.posterior_metric_counts(chain, truth)."""
    R = chain.num_records
    if R == 0 or not chain.samples:
        return tuple(np.zeros(len(chain.samples), np.int64) for _ in range(3))
    _, dense = np.unique(np.asarray(truth), return_inverse=True)  # any labels -> [0, number of entities)
    with Evaluation(R, dense, len(chain.samples)) as ev:
        _add_chain(ev, chain)
        return ev.read()


class VI(_Handle):
    """Owner of a dbl_vi handle: samples go in one at a time, cross() gives the cell histograms G."""

    _prefix = "dbl_vi"

    def __init__(self, num_records, max_samples):
        super().__init__(num_records, int(max_samples))

    def set_batch_keys(self, max_keys):
        """The keys one sort of cross() may hold: bounds its memory, not its result."""
        self._call("set_batch_keys", self._h, int(max_keys))

    def cross(self, width):
        """G, int64[S, width]: per sample t and cell size n >= 2, the cells of n records in C_t ^ C_s over s != t."""
        G = np.empty((self.num_samples, int(width)), np.int64)
        self._call("cross", self._h, int(width), G.ctypes.data)
        return G

    def score(self, labels, width):
        """G, int64[width]: the cells of n >= 2 records of labels ^ C_s summed over the held samples s."""
        labels = np.ascontiguousarray(labels, np.int32)
        if labels.shape != (self.num_records,):
            raise ValueError("a labelling needs one cluster label per record")
        G = np.empty(int(width), np.int64)
        self._call("score", self._h, labels.ctypes.data, int(width), G.ctypes.data)
        return G

    def score_samples(self, labels, width):
        """G, int64[S, width]: per held sample s the cells of n >= 2 records of labels ^ C_s."""
        labels = np.ascontiguousarray(labels, np.int32)
        if labels.shape != (self.num_records,):
            raise ValueError("a labelling needs one cluster label per record")
        G = np.empty((self.num_samples, int(width)), np.int64)
        self._call("score_samples", self._h, labels.ctypes.data, int(width), G.ctypes.data)
        return G

    def search(self, table, start, max_rounds):
        """The VI search from labels start[R] with the table D_q (analysis_arrays.vi_search_table): an
        analysis_arrays.VISearchRun.  The held samples do not change."""
        table = np.ascontiguousarray(table, np.int64)
        start = np.ascontiguousarray(start, np.int32)
        if table.shape != (self.num_records,):
            raise ValueError("the VI search table needs one entry per record")
        if start.shape != (self.num_records,):
            raise ValueError("a start needs one cluster label per record")
        max_rounds = int(max_rounds)
        labels = np.empty(self.num_records, np.int32)
        logs = [np.zeros(max(max_rounds, 0), np.int64) for _ in range(3)]
        rounds, converged, J0 = C.c_int32(), C.c_int32(), C.c_int64()
        self._call("search", self._h, table.ctypes.data_as(_lib.i64p), start.ctypes.data, max_rounds,
                   labels.ctypes.data, C.byref(rounds), C.byref(converged), *(x.ctypes.data_as(_lib.i64p) for x in logs),
                   C.byref(J0))
        return VISearchRun(labels.astype(np.int64), *(x[:rounds.value] for x in logs), converged.value, J0.value)


def vi_samples(chain, batch_keys=None):
    """A VI handle holding every sample of a ChainArrays (R > 0 and S > 0), with the methods of
    analysis_arrays.VISamples."""
    vi = VI(chain.num_records, len(chain.samples))
    try:
        if batch_keys is not None:
            vi.set_batch_keys(batch_keys)
        _add_chain(vi, chain)
    except BaseException:
        vi.close()
        raise
    return vi


def vi_search(chain, starts, max_rounds=1000, batch_keys=None):
    """(chosen position, VISearchRuns), identical to analysis_arrays.vi_search(chain, starts, max_rounds), refusals
    included: every sample is added to one handle, then the search runs from each start on it."""
    R, S = chain.num_records, len(chain.samples)
    check_vi_search_size(S, R)
    check_vi_search_squares(vi_sample_squares(chain))
    with vi_samples(chain, batch_keys) as vi:
        runs = [vi.search(vi_search_table(R), st, max_rounds) for st in starts]
    return vi_search_choice(runs), runs


def vi_cross_histograms(chain, batch_keys=None):
    """G, int64[S, M + 1], identical to analysis_arrays.vi_cross_histograms(chain), refusals included; batch_keys
    bounds the keys of one device sort (VI.set_batch_keys)."""
    R, S = chain.num_records, len(chain.samples)
    width = vi_width(chain)
    if R == 0 or S == 0:
        return np.zeros((S, width), np.int64)
    with VI(R, S) as vi:
        if batch_keys is not None:
            vi.set_batch_keys(batch_keys)
        _add_chain(vi, chain)
        return vi.cross(width)


class EntityValues(_Handle):
    """Owner of a dbl_values handle, one attribute: the estimate's labels go in once, each sample's value per record
    one at a time, modes() reads every cluster's mode and its count."""

    _prefix = "dbl_values"

    def __init__(self, labels, num_clusters, num_values):
        labels = np.ascontiguousarray(labels, np.int32)
        super().__init__(len(labels), labels.ctypes.data, int(num_clusters), int(num_values))
        self.num_clusters = int(num_clusters)

    def add_sample(self, values):
        values = np.ascontiguousarray(values, np.int32)
        if values.shape != (self.num_records,):
            raise ValueError("a sample needs one value per record")
        self._call("add_sample", self._h, values.ctypes.data)

    def modes(self):
        """(mode int32[C], count int64[C]), as analysis_arrays.EntityValueCounts.modes."""
        mode, count = np.empty(self.num_clusters, np.int32), np.empty(self.num_clusters, np.int64)
        self._call("modes", self._h, mode.ctypes.data, count.ctypes.data)
        return mode, count


def entity_value_modes(labels, value_samples, num_values):
    """(modes, counts, S), identical to analysis_arrays.entity_value_modes(labels, value_samples, num_values): one
    handle per attribute, all alive while the samples stream through."""
    return analysis_arrays.entity_value_modes(labels, value_samples, num_values, EntityValues)


class Query(_Handle):
    """Owner of a dbl_query handle: the query tables (analysis_arrays.QueryTables) go in once; add_sample for every
    sample (pass 1), score_sample for the same samples in the same order (pass 2), read() gives the
    analysis_arrays.QueryResult.  Labels and values may be numpy arrays or device pointers (int)."""

    _prefix = "dbl_query"

    def __init__(self, tables, num_records, population_size, min_link_probability,
                 max_candidates=analysis_arrays.MAX_QUERY_CANDIDATES):
        t = analysis_arrays._check_min_link_probability(min_link_probability)
        tab = tables
        self._keep = [np.ascontiguousarray(tab.num_values, np.int32),
                      np.ascontiguousarray(np.concatenate(tab.norm), np.float64),
                      np.ascontiguousarray(tab.file, np.int32), np.ascontiguousarray(tab.x, np.int32),
                      np.ascontiguousarray(tab.psi, np.float64), np.ascontiguousarray(tab.sigma, np.float64),
                      np.ascontiguousarray(tab.hit_offsets, np.int64),
                      np.ascontiguousarray(np.r_[tab.hit_values, 0], np.int32),
                      np.ascontiguousarray(np.r_[tab.hit_expsim, 0.0], np.float64)]
        ptrs = [_lib.i32p, _lib.f64p, _lib.i32p, _lib.i32p, _lib.f64p, _lib.f64p, _lib.i64p, _lib.i32p, _lib.f64p]
        self.tab, self.Q, self.A = tab, tab.num_queries, tab.num_attributes
        super().__init__(num_records, int(population_size), self.Q, self.A, int(tab.num_files),
                         *[a.ctypes.data_as(p) for a, p in zip(self._keep, ptrs)], t, int(max_candidates))

    def _sample(self, name, labels, values, theta):
        theta = np.ascontiguousarray(theta, np.float64)
        if theta.size != self.A * self.tab.num_files:
            raise ValueError("distortion probabilities must be [A][F]")
        if isinstance(labels, int):
            lab = labels
        else:
            labels = np.ascontiguousarray(labels, np.int32)
            if labels.shape != (self.num_records,):
                raise ValueError("a sample needs one cluster label per record")
            lab = labels.ctypes.data
        if isinstance(values, tuple):  # (device pointer, K)
            val, K = values
        else:
            values = np.ascontiguousarray(values, np.int32)
            if values.ndim != 2 or values.shape[1] != self.A:
                raise ValueError("a sample needs one value row of A ids per cluster")
            val, K = values.ctypes.data, len(values)
        self._call(name, self._h, lab, int(K), val, theta.ctypes.data_as(_lib.f64p))

    def add_sample(self, labels, values, theta):
        self._sample("add_sample", labels, values, theta)

    def score_sample(self, labels, values, theta):
        self._sample("score_sample", labels, values, theta)

    def num_candidates(self):
        n = C.c_int64(0)
        self._call("num_candidates", self._h, C.byref(n))
        return n.value

    def read(self):
        H, Q, S = self.num_candidates(), self.Q, self.num_samples
        q, r = np.zeros(H, np.int32), np.zeros(H, np.int32)
        sums = np.zeros(H)
        scale, zsum, zsq, fresh = (np.zeros(Q) for _ in range(4))
        logz = np.zeros((S, Q))
        self._call("read", self._h, q.ctypes.data, r.ctypes.data, sums.ctypes.data, scale.ctypes.data,
                   zsum.ctypes.data, zsq.ctypes.data, fresh.ctypes.data, logz.ctypes.data)
        return analysis_arrays.QueryResult(q, r, sums, scale, zsum, zsq, fresh, logz)


def link_queries(tables, samples, num_records, population_size, min_link_probability):
    """analysis_arrays.link_queries on the device."""
    return analysis_arrays.link_queries(tables, samples, num_records, population_size, min_link_probability, Query)


class Capture(_Handle):
    """Owner of a dbl_capture handle: the records' files go in once, samples one at a time, read() gives (H int64[S,
    2^F], L int64[R, F]) as analysis_arrays.CaptureCounts.read.  file may be a numpy array or a device pointer (int)
    with num_records given."""

    _prefix = "dbl_capture"

    def __init__(self, file, num_files, max_samples=1 << 16, num_records=None):
        if isinstance(file, int):
            ptr, R = file, int(num_records)
        else:
            file = np.ascontiguousarray(file, np.int32)
            ptr, R = file.ctypes.data, len(file)
        self.F = int(num_files)
        super().__init__(R, ptr, self.F, int(max_samples))

    def add_sample(self, cluster):
        if isinstance(cluster, int):  # a device pointer
            self._call("add_sample", self._h, cluster)
        else:
            super().add_sample(cluster)

    def read(self, record_links=True):
        H = np.empty((self.num_samples, 1 << self.F), np.int64)
        L = np.empty((self.num_records, self.F), np.int32) if record_links else None
        self._call("read", self._h, H.ctypes.data, None if L is None else L.ctypes.data)
        return H, None if L is None else L.astype(np.int64)


def capture_histories(chain, file, num_files):
    """(H, L), identical to analysis_arrays.capture_histories(chain, file, num_files): every sample goes into one
    handle."""
    analysis_arrays.check_capture_files(num_files)
    return analysis_arrays.capture_histories(
        chain, file, num_files, lambda f, F: Capture(f, F, max(len(chain.samples), 1)))
