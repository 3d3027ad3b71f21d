"""Host-side mirror of the reference's objects around the Gibbs sweep, backed by the C ABI.

  AttributeIndex      <- AttributeIndex.scala:39-245
  KDTreePartitioner   <- partitioning/KDTreePartitioner.scala:28-69
  GibbsEngine         <- State.scala:56-99 (nextState), GibbsUpdates.scala (all update* functions)

Errors follow the reference's conventions: argument problems raise ValueError (Scala `require` ->
IllegalArgumentException), out-of-range value ids raise IndexError (AttributeIndex.scala:137).
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import PCG_I, PCG_II, GIBBS, GIBBS_SEQ, SAMPLERS  # noqa: F401


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _p(a, t):
    return a.ctypes.data_as(t)


class DblinkError(RuntimeError):
    pass


def _check(rc, what, ctx=None):
    if rc == _lib.OK:
        return
    msg = ""
    if ctx:
        msg = _lib.load().dbl_last_error(ctx).decode()
    if rc == _lib.ERR_INVALID:
        raise ValueError(f"{what}: invalid argument {msg}")
    if rc == _lib.ERR_ZERO_MASS:
        raise ValueError(f"{what}: zero probability mass {msg}")  # IndexNonUniformDiscreteDist.scala:78-79
    if rc == _lib.ERR_CUDA:
        raise DblinkError(f"{what}: CUDA failure (dblink_b200 needs a CUDA device; there is no CPU fallback) {msg}")
    raise DblinkError(f"{what}: error {rc} {msg}")


SIMILARITY_KINDS = {"constant": _lib.SIM_CONSTANT, "levenshtein": _lib.SIM_LEVENSHTEIN,
                    "jaro-winkler": _lib.SIM_JARO_WINKLER}
SIMILARITY_FNS = {"ConstantSimilarityFn": _lib.SIM_CONSTANT, "LevenshteinSimilarityFn": _lib.SIM_LEVENSHTEIN,
                  "JaroWinklerSimilarityFn": _lib.SIM_JARO_WINKLER}


class AttributeIndex:
    """Index of one attribute domain (AttributeIndex.scala:39-104)."""

    def __init__(self, handle, is_constant):
        self._h = handle
        self.is_constant = bool(is_constant)
        L = _lib.load()
        self.num_values = L.dbl_index_num_values(handle)
        self.hash_slots = L.dbl_index_hash_slots(handle)
        self.nnz = L.dbl_index_nnz(handle)

    @classmethod
    def build(cls, values_weights, similarity="constant", threshold=7.0, max_similarity=10.0,
              expected_max_cluster_size=10):
        """AttributeIndex.apply (AttributeIndex.scala:107-127).  similarity: 'constant' | 'levenshtein' |
        'jaro-winkler'."""
        if not values_weights:
            raise ValueError("index cannot be empty")  # AttributeIndex.scala:111
        if similarity not in SIMILARITY_KINDS:
            raise ValueError(f"unsupported similarity {similarity!r}")
        L = _lib.load()
        vals = list(values_weights.keys())
        arr = (C.c_char_p * len(vals))(*[v.encode() for v in vals])
        w = _f64([values_weights[v] for v in vals])
        h = C.c_void_p()
        sim = SIMILARITY_KINDS[similarity]
        _check(L.dbl_index_build(C.byref(h), arr, _p(w, _lib.f64p), len(vals), sim, threshold, max_similarity,
                                 expected_max_cluster_size), "AttributeIndex.build")
        return cls(h, sim == 0)

    @classmethod
    def from_tables(cls, probs, rowptr=None, col=None, expsim=None, constant=True, expected_max_cluster_size=10):
        L = _lib.load()
        probs = _f64(probs)
        h = C.c_void_p()
        if constant:
            rc = L.dbl_index_from_tables(C.byref(h), len(probs), 0, _p(probs, _lib.f64p), None, None, None,
                                         expected_max_cluster_size)
        else:
            rowptr, col, expsim = _i32(rowptr), _i32(col), _f64(expsim)
            rc = L.dbl_index_from_tables(C.byref(h), len(probs), 1, _p(probs, _lib.f64p), _p(rowptr, _lib.i32p),
                                         _p(col, _lib.i32p), _p(expsim, _lib.f64p), expected_max_cluster_size)
        _check(rc, "AttributeIndex.from_tables")
        return cls(h, constant)

    def __del__(self):
        try:
            if self._h:
                _lib.load().dbl_index_free(self._h)
                self._h = None
        except Exception:
            pass

    def tables(self):
        V, nnz = self.num_values, self.nnz
        phi, norm = np.zeros(V), np.zeros(V)
        rowptr = np.zeros(V + 1, np.int32)
        col = np.zeros(max(nnz, 1), np.int32)
        es = np.zeros(max(nnz, 1))
        L = _lib.load()
        _check(L.dbl_index_tables(self._h, _p(phi, _lib.f64p), _p(norm, _lib.f64p), _p(rowptr, _lib.i32p),
                                    _p(col, _lib.i32p), _p(es, _lib.f64p)), "AttributeIndex.tables")
        kmax = C.c_int32(0)
        _check(L.dbl_index_base_tables(self._h, C.byref(kmax), None, None, None, None, None), "AttributeIndex.tables")
        invnorm, logphi, lognorm = np.zeros(V), np.zeros(V), np.zeros(V)
        pk, cdf = np.zeros((kmax.value + 1, V)), np.zeros((kmax.value + 1, V))
        _check(L.dbl_index_base_tables(self._h, None, _p(invnorm, _lib.f64p), _p(logphi, _lib.f64p),
                                       _p(lognorm, _lib.f64p), _p(pk, _lib.f64p), _p(cdf, _lib.f64p)),
               "AttributeIndex.tables")
        return {"phi": phi, "norm": norm, "rowptr": rowptr, "col": col[:nnz], "expsim": es[:nnz], "invnorm": invnorm,
                "logphi": logphi, "lognorm": lognorm, "pk": pk, "cdf": cdf}

    @property
    def slot_codes(self):
        """Slot codes of the 32-slot hash tables (int32, one per value id; code & 31 is the value's slot in every
        row's table), or None when the index has none."""
        out = np.zeros(self.num_values, np.int32)
        rc = _lib.load().dbl_index_slot_codes(self._h, _p(out, _lib.i32p))
        if rc == _lib.ERR_STATE:
            return None
        _check(rc, "AttributeIndex.slot_codes")
        return out

    @property
    def pairs_on_device(self):
        """True when build() found the similarity pairs with the device kernel, False when the host loop did."""
        return bool(_lib.load().dbl_index_pairs_on_device(self._h))

    def _require(self, v):
        if not 0 <= v < self.num_values:
            raise IndexError("valueId is not in the index")  # AttributeIndex.scala:137

    def value_idx_of(self, value):
        return _lib.load().dbl_index_value_id(self._h, value.encode())

    def value_of(self, v):
        self._require(v)
        r = _lib.load().dbl_index_value(self._h, v)
        return r.decode() if r is not None else None

    def probability_of(self, v):
        self._require(v)
        return float(self.tables()["phi"][v])

    def sim_normalization_of(self, v):
        self._require(v)
        return float(self.tables()["norm"][v])

    def sim_values_of(self, v):
        self._require(v)
        t = self.tables()
        lo, hi = t["rowptr"][v], t["rowptr"][v + 1]
        return {int(c): float(e) for c, e in zip(t["col"][lo:hi], t["expsim"][lo:hi])}

    def exp_sim_of(self, v1, v2):
        self._require(v1)
        self._require(v2)
        return _lib.load().dbl_index_exp_sim(self._h, v1, v2)


def similarity(a, b, name="LevenshteinSimilarityFn", threshold=7.0, max_similarity=10.0):
    """SimilarityFn.getSimilarity (SimilarityFn.scala:50-98); name: 'ConstantSimilarityFn' |
    'LevenshteinSimilarityFn' | 'JaroWinklerSimilarityFn'."""
    if name not in SIMILARITY_FNS:
        raise ValueError(f"unsupported similarity function {name}")
    if name == "ConstantSimilarityFn":
        return 0.0
    if not (max_similarity > 0.0):
        raise ValueError("`maxSimilarity` must be positive")
    if not (0.0 <= threshold < max_similarity):
        raise ValueError("`threshold` must be in the interval [0, maxSimilarity)")
    return _lib.load().dbl_similarity(SIMILARITY_FNS[name], a.encode(), b.encode(), threshold, max_similarity)


class KDTreePartitioner:
    """partitioning/KDTreePartitioner.scala:28-69."""

    def __init__(self, num_levels=0, attribute_ids=()):
        if num_levels < 0:
            raise ValueError("`numLevels` must be non-negative.")
        if num_levels > 0 and len(attribute_ids) == 0:
            raise ValueError("`attributeIds` must be non-empty if `numLevels` > 0")
        self.num_levels = num_levels
        self.attribute_ids = list(attribute_ids)
        self._h = None

    def fit(self, entity_values):
        y = _i32(entity_values)
        ids = _i32(self.attribute_ids if self.attribute_ids else [0])
        h = C.c_void_p()
        _check(_lib.load().dbl_kdtree_fit(C.byref(h), _p(y, _lib.i32p), y.shape[0], y.shape[1], self.num_levels,
                                          _p(ids, _lib.i32p), len(self.attribute_ids)), "KDTreePartitioner.fit")
        self._free()
        self._h = h
        return self

    @classmethod
    def from_arrays(cls, attr, kind, split, set_ptr, set_val, leaf_no):
        self = cls(0, ())
        a, k, s, sp, ln = _i32(attr), _i32(kind), _i32(split), _i32(set_ptr), _i32(leaf_no)
        sv = _i32(set_val if len(set_val) else [0])
        h = C.c_void_p()
        _check(_lib.load().dbl_kdtree_from_arrays(C.byref(h), len(a), _p(a, _lib.i32p), _p(k, _lib.i32p),
                                                  _p(s, _lib.i32p), _p(sp, _lib.i32p), _p(sv, _lib.i32p),
                                                  _p(ln, _lib.i32p)), "KDTreePartitioner.from_arrays")
        self._h = h
        return self

    def _free(self):
        if self._h:
            _lib.load().dbl_kdtree_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self._free()
        except Exception:
            pass

    @property
    def num_partitions(self):
        return _lib.load().dbl_kdtree_num_leaves(self._h) if self._h else 1

    def get_partition_id(self, values):
        v = _i32(values)
        return _lib.load().dbl_kdtree_partition_id(self._h, _p(v, _lib.i32p)) if self._h else 0

    def export(self):
        L = _lib.load()
        n, sl = L.dbl_kdtree_num_nodes(self._h), L.dbl_kdtree_set_len(self._h)
        out = {k: np.zeros(n, np.int32) for k in ("attr", "kind", "split", "leaf_no")}
        out["set_ptr"] = np.zeros(n + 1, np.int32)
        out["set_val"] = np.zeros(max(sl, 1), np.int32)
        _check(L.dbl_kdtree_export(self._h, _p(out["attr"], _lib.i32p), _p(out["kind"], _lib.i32p),
                                   _p(out["split"], _lib.i32p), _p(out["set_ptr"], _lib.i32p),
                                   _p(out["set_val"], _lib.i32p), _p(out["leaf_no"], _lib.i32p)), "KDTree.export")
        out["set_val"] = out["set_val"][:sl]
        return out


class _OwnedRows(dict):
    """dict of the owned rows that also carries the host buffers behind them (reused by the next download)."""


class GibbsEngine:
    """The Markov chain state on one GPU and its transition operator (State.scala:56-99)."""

    def __init__(self, indexes, alpha, beta, partitioner=None, seed=0, num_files=1, rank=0, world_size=1):
        if len(indexes) == 0 or len(indexes) > _lib.MAX_ATTRS:
            raise ValueError("between 1 and 32 matching attributes are supported")
        self.indexes = list(indexes)
        self.A = len(self.indexes)
        self.F = int(num_files)
        self.alpha, self.beta = _f64(alpha), _f64(beta)
        if np.any(self.alpha <= 0) or np.any(self.beta <= 0):
            raise ValueError("shape parameters must be positive")  # package.scala:165
        self.partitioner = partitioner
        self.seed = int(seed)
        L = _lib.load()
        arr = (C.c_void_p * self.A)(*[ix._h for ix in self.indexes])
        d = _lib.ModelDesc()
        d.num_attrs, d.num_files = self.A, self.F
        d.indexes = C.cast(arr, C.POINTER(C.c_void_p))
        d.alpha, d.beta = _p(self.alpha, _lib.f64p), _p(self.beta, _lib.f64p)
        d.tree = partitioner._h if (partitioner is not None and partitioner._h) else None
        d.seed = self.seed
        d.rank, d.world_size = rank, world_size
        h = C.c_void_p()
        rc = L.dbl_ctx_create(C.byref(h), C.byref(d))
        self._h = h if h else None
        _check(rc, "GibbsEngine", self._h)

    def close(self):
        if getattr(self, "_h", None):
            _lib.load().dbl_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state ------------------------------------------------------------------------------------
    def init_state(self, x, file_ids=None, population_size=0):
        """State.deterministic (State.scala:205-334)."""
        x = _i32(x)
        if x.ndim != 2 or x.shape[1] != self.A:
            raise ValueError("attribute specifications do not match the records")  # RecordsCache.scala:72
        f = _i32(file_ids if file_ids is not None else np.zeros(x.shape[0], np.int32))
        _check(_lib.load().dbl_state_init(self._h, x.shape[0], _p(x, _lib.i32p), _p(f, _lib.i32p),
                                          int(population_size)), "init_state", self._h)
        self._records_src = (None, None)

    def upload_state(self, x, file_ids, z, link, y, theta, iteration=0):
        """State.read: an arbitrary state.  x = file_ids = None keeps the records already on the device (they never
        change along a chain); passing the very same host arrays as last time has the same effect."""
        link, y = _i32(link), _i32(y)
        z = np.ascontiguousarray(z, dtype=np.uint8)
        theta = _f64(theta)
        if y.shape[1] != self.A or theta.size != self.A * self.F:
            raise ValueError("state arrays do not match the model")
        keep = x is None or (x is getattr(self, "_records_src", (None, None))[0] and
                             file_ids is self._records_src[1] and y.shape[0] == self.num_entities)
        if keep:
            xp, fp, R = None, None, self.num_records
            if z.shape[0] != R:
                raise ValueError("state arrays do not match the records on the device")
        else:
            xs, fs = _i32(x), _i32(file_ids)
            if xs.shape[1] != self.A:
                raise ValueError("state arrays do not match the model")
            xp, fp, R = _p(xs, _lib.i32p), _p(fs, _lib.i32p), xs.shape[0]
        _check(_lib.load().dbl_state_upload(self._h, R, y.shape[0], xp, fp, _p(z, _lib.u8p), _p(link, _lib.i32p),
                                            _p(y, _lib.i32p), _p(theta, _lib.f64p), int(iteration)), "upload_state",
               self._h)
        if not keep:
            self._records_src = (x, file_ids)

    def upload_state_device(self, R, E, x_ptr, file_ptr, z_ptr, link_ptr, y_ptr, theta, iteration=0):
        """upload_state from DEVICE buffers (raw addresses of int32 x[R,A], file[R], uint8 z[R,A], int32 link[R],
        y[E,A]); theta stays a host array."""
        theta = _f64(theta)
        if theta.size != self.A * self.F:
            raise ValueError("state arrays do not match the model")
        cast = lambda p, t: C.cast(C.c_void_p(int(p)), t) if p else None
        _check(_lib.load().dbl_state_upload(self._h, int(R), int(E), cast(x_ptr, _lib.i32p), cast(file_ptr, _lib.i32p),
                                            cast(z_ptr, _lib.u8p), cast(link_ptr, _lib.i32p), cast(y_ptr, _lib.i32p),
                                            _p(theta, _lib.f64p), int(iteration)), "upload_state", self._h)

    # ---- batched chains ---------------------------------------------------------------------------
    def init_chains(self, x, file_ids=None, population_size=0, seeds=(0, 1)):
        """State.deterministic for K = len(seeds) independent chains of the model in this one context, chain k drawn
        with key seeds[k].  Chain k is bit-equal to a one-chain engine created with seed=seeds[k] and given the same
        partitioner.  x / file_ids are the records once; the device replicates them."""
        x = _i32(x)
        if x.ndim != 2 or x.shape[1] != self.A:
            raise ValueError("attribute specifications do not match the records")  # RecordsCache.scala:72
        f = _i32(file_ids if file_ids is not None else np.zeros(x.shape[0], np.int32))
        s = np.ascontiguousarray(seeds, dtype=np.uint64)
        _check(_lib.load().dbl_chains_init(self._h, len(s), _p(s, _lib.u64p), x.shape[0], _p(x, _lib.i32p),
                                           _p(f, _lib.i32p), int(population_size)), "init_chains", self._h)
        self._records_src = (None, None)

    def upload_chains(self, x, file_ids, states, seeds, iteration=0):
        """Resume K = len(seeds) chains: `states` = one dict per chain in download_state's format (z, link with
        chain-local entity ids, y, theta)."""
        if len(states) != len(seeds):
            raise ValueError("one state per chain")
        xs, fs = _i32(x), _i32(file_ids)
        z = np.ascontiguousarray(np.concatenate([st["z"] for st in states]), dtype=np.uint8)
        link = _i32(np.concatenate([st["link"] for st in states]))
        y = _i32(np.concatenate([st["y"] for st in states]))
        theta = _f64(np.stack([np.asarray(st["theta"], np.float64).reshape(self.A, self.F) for st in states]))
        R, E = xs.shape[0], len(states[0]["y"])
        if (xs.ndim != 2 or xs.shape[1] != self.A or y.shape[1] != self.A or
                any(len(st["link"]) != R or len(st["y"]) != E for st in states)):
            raise ValueError("state arrays do not match the model")
        s = np.ascontiguousarray(seeds, dtype=np.uint64)
        _check(_lib.load().dbl_chains_upload(self._h, len(s), _p(s, _lib.u64p), R, E, _p(xs, _lib.i32p),
                                             _p(fs, _lib.i32p), _p(z, _lib.u8p), _p(link, _lib.i32p), _p(y, _lib.i32p),
                                             _p(theta, _lib.f64p), int(iteration)), "upload_chains", self._h)
        self._records_src = (None, None)

    @property
    def num_chains(self):
        return _lib.load().dbl_num_chains(self._h)

    def download_chains(self, links_only=False):
        """Every chain's state at once: a list of K dicts in download_state's format (chain-local link and entity ids,
        block = leaf id of the shared tree).  links_only: only link and block (the linkage structure of each chain)."""
        K, R, E, A = self.num_chains, self.num_records, self.num_entities, self.A
        link, blk = np.zeros(K * R, np.int32), np.zeros(K * E, np.int32)
        z = y = theta = None
        if not links_only:
            z, y, theta = np.zeros((K * R, A), np.uint8), np.zeros((K * E, A), np.int32), np.zeros((K, A, self.F))
        ptr = lambda a, t: _p(a, t) if a is not None else None
        _check(_lib.load().dbl_chains_download(self._h, ptr(z, _lib.u8p), _p(link, _lib.i32p), ptr(y, _lib.i32p),
                                               ptr(theta, _lib.f64p), _p(blk, _lib.i32p)), "download_chains", self._h)
        out = [{"link": link[k * R:(k + 1) * R], "block": blk[k * E:(k + 1) * E]} for k in range(K)]
        if not links_only:
            for k, d in enumerate(out):
                d.update(z=z[k * R:(k + 1) * R], y=y[k * E:(k + 1) * E], theta=theta[k])
        return out

    def chain_summary(self, k):
        """summary() of chain k."""
        head = _lib.SummaryHead()
        agg = np.zeros((self.A, self.F), np.int64)
        rec = np.zeros(self.A + 1, np.int64)
        theta = np.zeros((self.A, self.F))
        _check(_lib.load().dbl_chain_summary(self._h, int(k), C.byref(head), _p(agg, _lib.i64p), _p(rec, _lib.i64p),
                                             _p(theta, _lib.f64p)), "chain_summary", self._h)
        return {"iteration": head.iteration, "num_isolates": head.num_isolates, "log_likelihood": head.log_likelihood,
                "pairs_scored": head.pairs_scored, "agg_dist": agg, "rec_dist": rec, "theta": theta}

    def set_partitioner(self, partitioner):
        """Install the partition function fitted on the initial entity values (State.scala:309-316)."""
        self.partitioner = partitioner
        h = partitioner._h if (partitioner is not None and partitioner._h) else None
        _check(_lib.load().dbl_set_partitioner(self._h, h), "set_partitioner", self._h)

    @property
    def num_partitions(self):
        return _lib.load().dbl_num_partitions(self._h)

    @property
    def num_records(self):
        return _lib.load().dbl_num_records(self._h)

    @property
    def num_entities(self):
        return _lib.load().dbl_num_entities(self._h)

    @property
    def iteration(self):
        return _lib.load().dbl_iteration(self._h)

    def download_state(self, out=None):
        """Full state on the host (State.save, State.scala:122-150).  `out` may hold preallocated (e.g. pinned)
        arrays under the keys z, link, y, theta, block; they are filled in place."""
        R, E, A = self.num_records, self.num_entities, self.A
        out = out if out is not None else {}
        z = out.get("z") if out.get("z") is not None else np.zeros((R, A), np.uint8)
        link = out.get("link") if out.get("link") is not None else np.zeros(R, np.int32)
        y = out.get("y") if out.get("y") is not None else np.zeros((E, A), np.int32)
        theta = out.get("theta") if out.get("theta") is not None else np.zeros((A, self.F))
        blk = out.get("block") if out.get("block") is not None else np.zeros(E, np.int32)
        assert z.dtype == np.uint8 and link.dtype == np.int32 and y.dtype == np.int32 and blk.dtype == np.int32
        _check(_lib.load().dbl_state_download(self._h, _p(z, _lib.u8p), _p(link, _lib.i32p), _p(y, _lib.i32p),
                                              _p(theta, _lib.f64p), _p(blk, _lib.i32p)), "download_state", self._h)
        return {"z": z, "link": link, "y": y, "theta": theta, "block": blk}

    def links(self):
        """(link[R], block_of_entity[E]) -- the input of State.getLinkageStructure (State.scala:102-112)."""
        link = np.zeros(self.num_records, np.int32)
        blk = np.zeros(self.num_entities, np.int32)
        _check(_lib.load().dbl_links_download(self._h, _p(link, _lib.i32p), _p(blk, _lib.i32p)), "links", self._h)
        return link, blk

    # ---- transition -------------------------------------------------------------------------------
    def sweep(self, sampler="PCG-I", n=1):
        """n applications of State.nextState (State.scala:78-99)."""
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        _check(_lib.load().dbl_sweep(self._h, s, int(n)), "sweep", self._h)

    def sweep_async(self, sampler="PCG-I", n=1):
        """Enqueue n sweeps without waiting (nothing in a sweep needs the host); `sync()` collects them."""
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        _check(_lib.load().dbl_sweep_async(self._h, s, int(n)), "sweep_async", self._h)

    def sync(self):
        _check(_lib.load().dbl_sync(self._h), "sync", self._h)

    def state_hash(self):
        """(entities, records): order-independent 64-bit fingerprints of the rows this context owns; summed over
        ranks mod 2^64 they identify the global state for any number of ranks (`combine_state_hash`)."""
        h = np.zeros(2, np.uint64)
        _check(_lib.load().dbl_state_hash(self._h, _p(h, _lib.u64p)), "state_hash", self._h)
        return int(h[0]), int(h[1])

    def owned_counts(self):
        """(entities, records) in the blocks this context owns."""
        ne, nr = C.c_int64(0), C.c_int64(0)
        _check(_lib.load().dbl_download_owned(self._h, C.byref(ne), None, None, None, C.byref(nr), None, None, None),
               "owned_counts", self._h)
        return ne.value, nr.value

    def download_owned(self, out=None):
        """The rows this context owns, compacted: {ent_ids, y, block, rec_ids, link, z}.  `out` = the dict returned by
        an earlier call: its (pinned) buffers are reused when they are large enough."""
        A = self.A
        ne, nr = self.owned_counts()
        buf = getattr(out, "_buffers", None) if out is not None else None
        if buf is None or buf["cap_e"] < ne or buf["cap_r"] < nr:
            cap_e, cap_r = int(ne * 1.25) + 16, int(nr * 1.25) + 16

            def alloc(shape, dtype):
                try:  # pinned host memory: the copies are plain DMA
                    import torch

                    return torch.empty(shape, dtype=getattr(torch, np.dtype(dtype).name), pin_memory=True).numpy()
                except Exception:
                    return np.empty(shape, dtype)

            buf = {"cap_e": cap_e, "cap_r": cap_r, "eid": alloc(cap_e, np.int32), "y": alloc((cap_e, A), np.int32),
                   "blk": alloc(cap_e, np.int32), "rid": alloc(cap_r, np.int32), "link": alloc(cap_r, np.int32),
                   "z": alloc((cap_r, A), np.uint8)}
        ne2, nr2 = C.c_int64(0), C.c_int64(0)
        _check(_lib.load().dbl_download_owned(self._h, C.byref(ne2), _p(buf["eid"], _lib.i32p), _p(buf["y"], _lib.i32p),
                                              _p(buf["blk"], _lib.i32p), C.byref(nr2), _p(buf["rid"], _lib.i32p),
                                              _p(buf["link"], _lib.i32p), _p(buf["z"], _lib.u8p)),
               "download_owned", self._h)
        res = _OwnedRows({"ent_ids": buf["eid"][:ne], "y": buf["y"][:ne], "block": buf["blk"][:ne],
                          "rec_ids": buf["rid"][:nr], "link": buf["link"][:nr], "z": buf["z"][:nr]})
        res._buffers = buf
        return res

    def sweep_by_block(self, sampler="PCG-I", order=None):
        """One application of State.nextState driven block by block, the way the reference runs one task per
        partition (GibbsUpdates.updatePartition, GU:156-211).  `order` = the order the blocks are updated in
        (default ascending); the resulting state does not depend on it."""
        L = _lib.load()
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        _check(L.dbl_block_sweep_begin(self._h, s), "block_sweep_begin", self._h)
        for b in (range(self.num_partitions) if order is None else order):
            _check(L.dbl_update_block(self._h, int(b)), "update_block", self._h)
        _check(L.dbl_block_sweep_end(self._h), "block_sweep_end", self._h)

    def summary(self):
        """SummaryVars (package.scala:116-119) of the current state + theta."""
        head = _lib.SummaryHead()
        agg = np.zeros((self.A, self.F), np.int64)
        rec = np.zeros(self.A + 1, np.int64)
        theta = np.zeros((self.A, self.F))
        _check(_lib.load().dbl_summary(self._h, C.byref(head), _p(agg, _lib.i64p), _p(rec, _lib.i64p),
                                       _p(theta, _lib.f64p)), "summary", self._h)
        return {"iteration": head.iteration, "num_isolates": head.num_isolates, "log_likelihood": head.log_likelihood,
                "pairs_scored": head.pairs_scored, "agg_dist": agg, "rec_dist": rec, "theta": theta}

    def kernel_launches(self):
        return _lib.load().dbl_kernel_launches(self._h)

    def set_link_mode(self, mode):
        """0 = automatic kernel choice, 1 = force the generic fallback link kernel (same draws)."""
        _check(_lib.load().dbl_set_link_mode(self._h, int(mode)), "set_link_mode", self._h)

    def link_kernel(self, sampler="PCG-II"):
        """Name of the link kernel a sweep with this sampler launches."""
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        k = _lib.load().dbl_link_kernel(self._h, s)
        base = {0: "k_link_generic", 1: "k_link_match", 2: "k_link_pruned", 3: "k_link_pcg2"}[k & 3]
        if (k & 3) == 3:
            base += "<A=%d,NS=%d,HC=%s,PK=%d>" % (self.A, sum(not ix.is_constant for ix in self.indexes),
                                                  "32" if k & 8 else "0", 1 if k & 4 else 0)
        return base

    def link_tile_format(self, sampler="PCG-II"):
        """Tile format of the k_link_pcg2 instantiation a sweep with this sampler launches: {"id16": 16-bit
        non-constant values, "slot_codes": slot codes instead of value ids, "paired": the warp's two records share
        their key tables, "records_per_warp": 1 or 2}; None when the sampler gets another link kernel."""
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        k = _lib.load().dbl_link_kernel(self._h, s)
        if (k & 3) != 3:
            return None
        return {"id16": bool(k & 16), "slot_codes": bool(k & 32), "paired": bool(k & 64),
                "records_per_warp": 2 if k & 128 else 1}

    def set_link_mass_capture(self, on=True):
        """Checking aid: make every link kernel store the total mass of each record's categorical (off by default)."""
        _check(_lib.load().dbl_set_link_mass_capture(self._h, int(bool(on))), "set_link_mass_capture", self._h)

    def link_mass(self):
        """float64[R]: the total mass of each record's link categorical in the last sweep run with the capture on
        (K R totals, chain-major, on an engine holding K chains)."""
        out = np.zeros(self.num_chains * self.num_records, np.float64)
        _check(_lib.load().dbl_link_mass(self._h, _p(out, _lib.f64p)), "link_mass", self._h)
        return out

    def set_graph_mode(self, mode):
        """0 = automatic (CUDA graph replay of a sweep for launch-bound sizes), 1 = never, 2 = whenever possible."""
        _check(_lib.load().dbl_set_graph_mode(self._h, int(mode)), "set_graph_mode", self._h)

    def last_sweep_ms(self):
        return _lib.load().dbl_last_sweep_ms(self._h)

    def link_kernel_ms(self):
        n = C.c_int64(0)
        ms = _lib.load().dbl_link_kernel_ms(self._h, C.byref(n))
        return ms, n.value

    def phase_ms(self):
        """Per-phase CUDA-event time of the eager sweeps since the last call: ({phase: ms per sweep}, sweeps)."""
        out = (C.c_double * 4)()
        n = _lib.load().dbl_phase_ms(self._h, out)
        names = ("link", "values_distortions_summary", "exchange", "relayout")
        return {k: (out[i] / n if n else 0.0) for i, k in enumerate(names)}, int(n)


def combine_state_hash(ent_hash, rec_hash, theta, iteration):
    """One hex string for a whole state: the (summed) row fingerprints, theta's bits and the iteration."""
    import hashlib

    h = hashlib.blake2b(digest_size=8)
    h.update(np.array([ent_hash % (1 << 64), rec_hash % (1 << 64)], np.uint64).tobytes())
    h.update(np.ascontiguousarray(theta, np.float64).tobytes())
    h.update(np.int64(iteration).tobytes())
    return h.hexdigest()
