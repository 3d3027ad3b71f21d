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
(sample, label, label) keys of every pair of held samples.
"""
import ctypes as C

import numpy as np

from . import _lib
from .analysis_arrays import (MAX_PAIRS, SearchRun, check_search_size, search_choice, search_cost,
                              too_many_pairs, vi_width)
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
