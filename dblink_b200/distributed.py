"""Multi-GPU Gibbs sweep: k-d-tree blocks sharded over ranks, one process per GPU.

Replaces, for the sweep, what Spark does in the reference:
  - one task per partition (GibbsUpdates.scala:137)            -> blocks placed on ranks by LPT on R_b * E_b, re-placed
                                                                  on the device every few sweeps
  - the shuffle `.partitionBy(partitioner)` (GU:144)           -> clusters whose new block is owned by another rank are
                                                                  written into that rank's receive buffer over
                                                                  NVLink/NVSwitch by the kernel that finds them
  - accumulators (SummaryAccumulators.scala:54-63)             -> every rank sums the partial summaries of all ranks
  - broadcast of theta (State.scala:84)                        -> nothing: every rank draws the same theta from the
                                                                  same counter-based stream

The data plane is INSIDE libdblink_b200.so (`dbl_comm_export / dbl_comm_import`, then plain `dbl_sweep`): the only
thing this module moves is the 192-byte description of each rank's communication buffer, once.  torch.distributed is
the out-of-band channel for that handshake and for read-out conveniences (gathering a full state on every rank).
`exchange="host"` selects the host-mediated fallback for machines without peer access: the library packs / unpacks,
this module moves the messages with NCCL all-to-alls.  The pure host logic (handshake, host-mediated exchange, merging
of owned rows, hashing) is exercised on CPU with the gloo backend by tests/test_distributed.py.
"""
import ctypes as C
import os

import numpy as np

from . import _lib
from .engine import GibbsEngine, KDTreePartitioner, SAMPLERS, _check, _p, combine_state_hash


def lpt_assign(costs, world):
    """Longest-processing-time placement of blocks on ranks (the reference ships the same heuristic in
    partitioning/LPTScheduler.scala:57-76).  Deterministic: ties by block id, then lowest rank."""
    costs = np.asarray(costs, dtype=np.float64)
    order = sorted(range(len(costs)), key=lambda b: (-costs[b], b))
    load = np.zeros(world)
    owner = np.zeros(len(costs), np.int32)
    for b in order:
        r = int(np.argmin(load))
        owner[b] = r
        load[r] += costs[b]
    return owner


def gather_blobs(dist, blob, device, torch):
    """All-gather of the ranks' communication-buffer descriptions (bytes) in rank order."""
    world = dist.get_world_size()
    mine = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(device)
    out = torch.empty(world * mine.numel(), dtype=torch.uint8, device=device)
    dist.all_gather_into_tensor(out, mine)
    return bytes(out.cpu().numpy().tobytes())


def exchange(dist, send_ent, ent_counts, send_rec, rec_counts, ent_words, device, torch):
    """Host-mediated exchange: all-to-all of the packed messages.  send_* are int32 tensors concatenated by
    destination rank; *_counts are per-destination MESSAGE counts.  Returns (recv_ent, n_ent, recv_rec, n_rec)."""
    world = dist.get_world_size()
    mine = torch.tensor(np.stack([ent_counts, rec_counts], axis=1).reshape(-1), dtype=torch.int64, device=device)
    theirs = torch.empty_like(mine)
    dist.all_to_all_single(theirs, mine)  # counts first
    theirs_h = theirs.cpu().numpy().reshape(world, 2)
    in_ent, in_rec = theirs_h[:, 0], theirs_h[:, 1]
    recv_ent = torch.empty(int(in_ent.sum()) * ent_words, dtype=torch.int32, device=device)
    recv_rec = torch.empty(int(in_rec.sum()) * 3, dtype=torch.int32, device=device)
    dist.all_to_all_single(recv_ent, send_ent, output_split_sizes=[int(c) * ent_words for c in in_ent],
                           input_split_sizes=[int(c) * ent_words for c in ent_counts])
    dist.all_to_all_single(recv_rec, send_rec, output_split_sizes=[int(c) * 3 for c in in_rec],
                           input_split_sizes=[int(c) * 3 for c in rec_counts])
    return recv_ent, int(in_ent.sum()), recv_rec, int(in_rec.sum())


def allreduce_summary(dist, counts, loglik, device, torch, failed=0):
    """One all-reduce for the integer summary words, the log-likelihood and an error flag: the counts travel as
    float64 (exact below 2^53; they are bounded by records x attributes).  Returns (counts, loglik, n_failed)."""
    buf = np.empty(len(counts) + 2, np.float64)
    buf[:-2] = counts
    buf[-2] = loglik
    buf[-1] = float(failed)
    t = torch.from_numpy(buf).to(device)
    dist.all_reduce(t)
    out = t.cpu().numpy()
    return np.rint(out[:-2]).astype(np.int64), float(out[-2]), int(round(out[-1]))


def merge_owned(parts, R, E, A):
    """Full state arrays from the ranks' compacted owned rows (`GibbsEngine.download_owned`)."""
    y = np.zeros((E, A), np.int32)
    blk = np.zeros(E, np.int32)
    link = np.zeros(R, np.int32)
    z = np.zeros((R, A), np.uint8)
    ne = nr = 0
    for p in parts:
        y[p["ent_ids"]] = p["y"]
        blk[p["ent_ids"]] = p["block"]
        link[p["rec_ids"]] = p["link"]
        z[p["rec_ids"]] = p["z"]
        ne += len(p["ent_ids"])
        nr += len(p["rec_ids"])
    if ne != E or nr != R:
        raise RuntimeError(f"shards do not cover the state: {ne}/{E} entities, {nr}/{R} records")
    return {"y": y, "block": blk, "link": link, "z": z}


LINK_MASS_UNSCORED = np.uint64(0xFFFFFFFFFFFFFFFF)  # dbl_link_mass on a shard: a record another rank scored


def merge_link_mass(parts):
    """R totals from the ranks' `dbl_link_mass` arrays, each holding the totals of the records its rank scored and
    the all-ones bit pattern everywhere else.  Raises unless exactly one rank scored each record."""
    bits = np.stack([np.asarray(p, np.float64).view(np.uint64) for p in parts])
    scored = bits != LINK_MASS_UNSCORED
    n = scored.sum(axis=0)
    bad = np.flatnonzero(n != 1)
    if bad.size:
        raise RuntimeError(f"link masses: {bad.size} records not scored by exactly one rank "
                           f"(record {bad[0]}: {n[bad[0]]} ranks)")
    return bits[scored.argmax(axis=0), np.arange(bits.shape[1])].view(np.float64)


def sum_hashes(dist, he, hr, device, torch):
    """Sum of the ranks' row fingerprints mod 2^64 (two's-complement int64 addition wraps the same way)."""
    t = torch.from_numpy(np.array([he, hr], np.uint64).view(np.int64).copy()).to(device)
    dist.all_reduce(t)
    out = t.cpu().numpy().view(np.uint64)
    return int(out[0]), int(out[1])


class ShardedGibbs:
    """Same surface as GibbsEngine (init_state / sweep / summary / links / download_state), block-sharded over the
    ranks of the default process group."""

    def __init__(self, indexes, alpha, beta, seed=0, num_files=1, levels=0, split_attrs=(), exchange=None):
        import torch
        import torch.distributed as dist

        self.torch, self.dist = torch, dist
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.levels, self.split_attrs = levels, list(split_attrs)
        self.eng = GibbsEngine(indexes, alpha, beta, None, seed, num_files, rank=self.rank, world_size=self.world)
        self.A, self.F = self.eng.A, self.eng.F
        self.owner = None
        self.exchange_mode = exchange or os.environ.get("DBL_EXCHANGE", "p2p")  # "p2p" | "host"
        self.connected = False
        self._ms = 0.0
        self._stage = {}  # device staging buffers of upload_state
        self.trace = {}   # host-mediated mode: wall-clock ms per phase of the sweep, accumulated (rank-local)
        self.last_exchange = (0, 0)

    # ---- state ---------------------------------------------------------------------------------------
    def init_state(self, x, file_ids=None, population_size=0):
        """Every rank builds the same replicated initial state (State.deterministic), fits the same k-d tree on it,
        then keeps only the blocks LPT assigns to it."""
        e = self.eng
        e.init_state(x, file_ids, population_size)
        part = KDTreePartitioner(self.levels, self.split_attrs).fit(e.download_state()["y"])
        e.set_partitioner(part)
        self.partitioner = part
        link, blk = e.links()
        P = e.num_partitions
        ent = np.bincount(blk, minlength=P).astype(np.float64)
        rec = np.bincount(blk[link], minlength=P).astype(np.float64)
        self.set_owners(lpt_assign(ent * rec, self.world))
        self.connect()

    def connect(self):
        """The handshake of the peer-to-peer data plane: export this rank's buffer, all-gather the descriptions, map
        the peers.  Falls back to the host-mediated exchange when peers cannot be mapped."""
        if self.exchange_mode != "p2p":
            return
        L, h = _lib.load(), self.eng._h
        blob = (C.c_uint8 * _lib.COMM_BLOB_BYTES)()
        _check(L.dbl_comm_export(h, blob), "comm_export", h)
        blobs = gather_blobs(self.dist, bytes(blob), self.device, self.torch)
        rc = L.dbl_comm_import(h, blobs, self.world)
        ok = self.torch.tensor([1 if rc == _lib.OK else 0], device=self.device)
        self.dist.all_reduce(ok, op=self.dist.ReduceOp.MIN)
        if int(ok[0]) == 1:
            self.connected = True
        else:  # some rank could not map a peer: everybody uses the host path
            import warnings

            warnings.warn("dblink_b200: peer-to-peer mapping unavailable (%s); using the host-mediated exchange"
                          % L.dbl_last_error(h).decode())
            self.exchange_mode = "host"

    def _gather_upload(self, name, a, dtype):
        """Full device copy of the host array `a` (identical on every rank): each rank copies 1/world of it over
        PCIe, one in-place all-gather over NVLink completes it."""
        torch, dist, W = self.torch, self.dist, self.world
        flat = np.ascontiguousarray(a, dtype=dtype).reshape(-1)
        n = flat.size
        chunk = (n + W - 1) // W
        key = (name, n)
        full = self._stage.get(key)
        if full is None:
            full = self._stage[key] = torch.empty(W * chunk, dtype=torch.from_numpy(flat[:0].copy()).dtype,
                                                  device=self.device)
        lo, hi = min(n, self.rank * chunk), min(n, (self.rank + 1) * chunk)
        if hi > lo:
            full[lo:hi].copy_(torch.from_numpy(flat[lo:hi]), non_blocking=True)
        dist.all_gather_into_tensor(full, full[self.rank * chunk:(self.rank + 1) * chunk])
        return full

    def upload_state(self, x, file_ids, z, link, y, theta, iteration=0):
        """Every rank is handed the same full state (State.read) and keeps the blocks it owns.  The host-to-device
        traffic is shared: a rank copies its 1/world slice of each array and the slices are all-gathered."""
        if self.owner is None:
            raise RuntimeError("upload_state needs the partitioner and block placement of init_state first")
        y = np.asarray(y)
        if y.ndim != 2 or y.shape[1] != self.A:
            raise ValueError("state arrays do not match the model")
        # the records never change along a chain: the same host arrays as last time stay on the devices
        keep = x is None or (x is getattr(self, "_records_src", (None, None))[0] and file_ids is self._records_src[1]
                             and y.shape[0] == self.eng.num_entities)
        R = self.eng.num_records if keep else np.asarray(x).shape[0]
        if not keep:
            x = np.asarray(x)
            if x.ndim != 2 or x.shape[1] != self.A:
                raise ValueError("state arrays do not match the model")
            dx = self._gather_upload("x", x, np.int32)
            df = self._gather_upload("file", file_ids, np.int32)
        dz = self._gather_upload("z", z, np.uint8)
        dl = self._gather_upload("link", link, np.int32)
        dy = self._gather_upload("y", y, np.int32)
        self.torch.cuda.current_stream().synchronize()  # the engine copies from these buffers on its own stream
        self.eng.upload_state_device(R, y.shape[0], dx.data_ptr() if not keep else 0, df.data_ptr() if not keep else 0,
                                     dz.data_ptr(), dl.data_ptr(), dy.data_ptr(), theta, iteration)
        if not keep:
            self._records_src = (x, file_ids)
        # carve the shards out again with the block -> rank table the devices hold (no host round trip)
        _check(_lib.load().dbl_set_block_owners(self.eng._h, None), "set_block_owners", self.eng._h)

    def set_owners(self, owner):
        owner = np.ascontiguousarray(owner, dtype=np.int32)
        self.owner = owner
        _check(_lib.load().dbl_set_block_owners(self.eng._h, _p(owner, _lib.i32p)), "set_block_owners", self.eng._h)

    def block_owners(self):
        """Current block -> rank table (the device-side LPT may have changed it since `set_owners`)."""
        out = np.zeros(self.eng.num_partitions, np.int32)
        _check(_lib.load().dbl_block_owners(self.eng._h, _p(out, _lib.i32p)), "block_owners", self.eng._h)
        return out

    def set_rebalance(self, period, threshold=1.03):
        _check(_lib.load().dbl_set_rebalance(self.eng._h, int(period), float(threshold)), "set_rebalance", self.eng._h)

    # ---- transition ----------------------------------------------------------------------------------
    def sweep(self, sampler="PCG-I", n=1):
        s = SAMPLERS[sampler] if isinstance(sampler, str) else int(sampler)
        if self.connected:
            L, h = _lib.load(), self.eng._h
            _check(L.dbl_sweep(h, s, int(n)), "sweep", h)  # the whole transition, exchange included, on the devices
            self._ms = self.eng.last_sweep_ms()
            e, r = C.c_int64(0), C.c_int64(0)
            L.dbl_last_exchange(h, C.byref(e), C.byref(r), None)
            self.last_exchange = (e.value, r.value)
            return
        self._sweep_host_mediated(s, n)

    def _sweep_host_mediated(self, s, n):
        """Fallback without peer access: the library packs and unpacks, NCCL all-to-alls move the messages.  A failure
        on one rank (e.g. a categorical without mass) is carried through the collectives of the sweep and raised on
        EVERY rank afterwards, so nobody is left waiting in a collective."""
        import time

        torch, dist, L, h = self.torch, self.dist, _lib.load(), self.eng._h
        W, ew = self.world, self.A + 1
        total_ms = 0.0
        tr = self.trace
        for _ in range(n):
            ec = np.zeros(W, np.int64)
            rc = np.zeros(W, np.int64)
            t0 = time.perf_counter()
            rc_begin = L.dbl_sweep_begin(h, s, _p(ec, _lib.i64p), _p(rc, _lib.i64p))
            err = L.dbl_last_error(h).decode() if rc_begin != _lib.OK else ""
            t1 = time.perf_counter()
            send_ent = torch.empty(int(ec.sum()) * ew, dtype=torch.int32, device=self.device)
            send_rec = torch.empty(int(rc.sum()) * 3, dtype=torch.int32, device=self.device)
            if rc_begin == _lib.OK:
                _check(L.dbl_exchange_pack(h, send_ent.data_ptr() if send_ent.numel() else None,
                                           send_rec.data_ptr() if send_rec.numel() else None), "exchange_pack", h)
            t2 = time.perf_counter()
            recv_ent, ne, recv_rec, nr = exchange(dist, send_ent, ec, send_rec, rc, ew, self.device, torch)
            torch.cuda.synchronize()
            t3 = time.perf_counter()
            if rc_begin == _lib.OK:
                _check(L.dbl_exchange_unpack(h, recv_ent.data_ptr() if ne else None, ne,
                                             recv_rec.data_ptr() if nr else None, nr), "exchange_unpack", h)
            nwords = L.dbl_summary_words(h)
            counts = np.zeros(nwords, np.int64)
            ll = C.c_double(0.0)
            L.dbl_partial_summary(h, _p(counts, _lib.i64p), C.byref(ll))
            g, gll, failed = allreduce_summary(dist, counts, ll.value, self.device, torch, failed=int(rc_begin != _lib.OK))
            g = np.ascontiguousarray(g, dtype=np.int64)
            t4 = time.perf_counter()
            rc_end = L.dbl_sweep_end(h, _p(g, _lib.i64p), gll, failed)
            if rc_begin != _lib.OK:
                _check(rc_begin, f"sweep_begin ({err})", None)
            _check(rc_end, "sweep_end", h)
            t5 = time.perf_counter()
            total_ms += self.eng.last_sweep_ms()
            for k, v in (("begin", t1 - t0), ("pack", t2 - t1), ("exchange", t3 - t2), ("unpack_summary", t4 - t3),
                         ("end", t5 - t4), ("sweeps", 1e-3)):
                tr[k] = tr.get(k, 0.0) + v * 1e3
            self.last_exchange = (int(ec.sum()), int(rc.sum()))
        self._ms = total_ms

    def last_sweep_ms(self):
        return self._ms

    # ---- read-out ------------------------------------------------------------------------------------
    def summary(self):
        return self.eng.summary()

    def kernel_launches(self):
        return self.eng.kernel_launches()

    def link_kernel_ms(self):
        return self.eng.link_kernel_ms()

    def phase_ms(self):
        return self.eng.phase_ms()

    @property
    def iteration(self):
        return self.eng.iteration

    @property
    def num_records(self):
        return self.eng.num_records

    @property
    def num_entities(self):
        return self.eng.num_entities

    @property
    def num_partitions(self):
        return self.eng.num_partitions

    def owned_masks(self):
        e = self.eng
        em = np.zeros(e.num_entities, np.uint8)
        rm = np.zeros(e.num_records, np.uint8)
        _check(_lib.load().dbl_owned_masks(e._h, _p(em, _lib.u8p), _p(rm, _lib.u8p)), "owned_masks", e._h)
        return em.astype(bool), rm.astype(bool)

    def state_hash(self):
        """Rank-count-invariant fingerprint of the global state (hex string, identical on every rank)."""
        he, hr = self.eng.state_hash()
        he, hr = sum_hashes(self.dist, he, hr, self.device, self.torch)
        s = self.eng.summary()
        return combine_state_hash(he, hr, s["theta"], s["iteration"])

    def download_owned(self, out=None):
        """Only this rank's rows (State.save of a distributed state): the device-to-host traffic of the whole job is
        one copy of the state, not one per rank.  `out` = an earlier result whose pinned buffers are reused."""
        return self.eng.download_owned(out)

    def links(self):
        """(link[R], block_of_entity[E]) of the global state on every rank."""
        d = self.download_state(keys=("link", "block"))
        return d["link"], d["block"]

    def download_state(self, out=None, keys=("y", "block", "link", "z")):
        """The full state on every rank: each rank exports the rows it owns into device buffers (zeros elsewhere),
        one all-reduce (NCCL) per array sums them, one device-to-host copy brings them back.  `out` may hold
        preallocated (e.g. pinned) host arrays under the keys z, link, y, block; they are filled in place."""
        torch, dist, e = self.torch, self.dist, self.eng
        R, E, A = e.num_records, e.num_entities, self.A
        y = torch.empty(E * A, dtype=torch.int32, device=self.device)
        blk = torch.empty(E, dtype=torch.int32, device=self.device)
        link = torch.empty(R, dtype=torch.int32, device=self.device)
        z = torch.empty(R * A, dtype=torch.uint8, device=self.device)
        _check(_lib.load().dbl_export_owned_dev(e._h, y.data_ptr(), blk.data_ptr(), link.data_ptr(), z.data_ptr()),
               "export_owned", e._h)
        dev = {"y": (y, (E, A)), "block": (blk, (E,)), "link": (link, (R,)), "z": (z, (R, A))}
        for k in keys:
            dist.all_reduce(dev[k][0])  # exactly one rank owns each row
        theta = np.zeros((A, self.F))
        _check(_lib.load().dbl_summary(e._h, None, None, None, _p(theta, _lib.f64p)), "summary", e._h)
        res = {"theta": theta}
        for k in keys:
            t, shape = dev[k]
            host = out.get(k) if out else None
            if host is None:
                res[k] = t.cpu().numpy().reshape(shape)
            else:
                torch.from_numpy(host.reshape(-1)).copy_(t, non_blocking=True)
                res[k] = host
        torch.cuda.current_stream().synchronize()
        if out and out.get("theta") is not None:
            out["theta"][...] = theta
            res["theta"] = out["theta"]
        return res


class LocalShards:
    """The same sharded chain driven from ONE process: one context per rank, one host thread per context while a
    sweep runs (a JVM host would do the same: one thread per GPU, all through the C ABI).  `devices[r]` is the CUDA
    device of rank r; several ranks may share a device (the tests shard a chain over 2-3 contexts of a single GPU and
    still go through the complete exchange: remote cursors, message buffers, flag barrier, summary slots)."""

    def __init__(self, indexes, alpha, beta, seed=0, num_files=1, levels=0, split_attrs=(), world=2, devices=None):
        self.world = world
        self.devices = list(devices) if devices is not None else [0] * world
        self.levels, self.split_attrs = levels, list(split_attrs)
        L = _lib.load()
        self.engines = []
        for r in range(world):
            _check(L.dbl_set_device(self.devices[r]), "set_device")
            self.engines.append(GibbsEngine(indexes, alpha, beta, None, seed, num_files, rank=r, world_size=world))
        self.A, self.F = self.engines[0].A, self.engines[0].F

    def _each(self, fn):
        """fn(rank, engine) on one thread per rank (ctypes releases the GIL inside the library)."""
        import threading

        errs = [None] * self.world

        def run(r):
            try:
                fn(r, self.engines[r])
            except BaseException as e:  # noqa: BLE001 -- re-raised on the calling thread
                errs[r] = e

        th = [threading.Thread(target=run, args=(r,)) for r in range(self.world)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for e in errs:
            if e is not None:
                raise e

    def init_state(self, x, file_ids=None, population_size=0, owner=None):
        e0 = self.engines[0]
        for e in self.engines:
            e.init_state(x, file_ids, population_size)
        y0 = e0.download_state()["y"]
        self.partitioners = []
        for e in self.engines:
            part = KDTreePartitioner(self.levels, self.split_attrs).fit(y0)
            e.set_partitioner(part)
            self.partitioners.append(part)
        if owner is None:
            link, blk = e0.links()
            P = e0.num_partitions
            ent = np.bincount(blk, minlength=P).astype(np.float64)
            rec = np.bincount(blk[link], minlength=P).astype(np.float64)
            owner = lpt_assign(ent * rec, self.world)
        self.set_owners(owner)
        self.connect()

    def upload_state(self, x, file_ids, z, link, y, theta, iteration=0, owner=None):
        """owner = the block -> rank table to carve the shards with (default: the current one).  A state of another
        shape closes the communication buffers (they are sized by the state): the ranks connect again."""
        owner = self.block_owners() if owner is None else owner
        for e in self.engines:
            e.upload_state(x, file_ids, z, link, y, theta, iteration)
        self.set_owners(owner)
        e0 = self.engines[0]
        if (e0.num_records, e0.num_entities) != self._connected_shape:
            self.connect()

    def set_owners(self, owner):
        owner = np.ascontiguousarray(owner, dtype=np.int32)
        for e in self.engines:
            _check(_lib.load().dbl_set_block_owners(e._h, _p(owner, _lib.i32p)), "set_block_owners", e._h)

    def block_owners(self):
        e = self.engines[0]
        out = np.zeros(e.num_partitions, np.int32)
        _check(_lib.load().dbl_block_owners(e._h, _p(out, _lib.i32p)), "block_owners", e._h)
        return out

    def set_rebalance(self, period, threshold=1.03):
        for e in self.engines:
            _check(_lib.load().dbl_set_rebalance(e._h, int(period), float(threshold)), "set_rebalance", e._h)

    def connect(self):
        L = _lib.load()
        blobs = b""
        for e in self.engines:
            blob = (C.c_uint8 * _lib.COMM_BLOB_BYTES)()
            _check(L.dbl_comm_export(e._h, blob), "comm_export", e._h)
            blobs += bytes(blob)
        for e in self.engines:
            _check(L.dbl_comm_import(e._h, blobs, self.world), "comm_import", e._h)
        self._connected_shape = (self.engines[0].num_records, self.engines[0].num_entities)

    def sweep(self, sampler="PCG-I", n=1):
        self._each(lambda r, e: e.sweep(sampler, n))

    def set_link_mass_capture(self, on=True):
        """Checking aid: every rank's link kernels store the total mass of each record they score."""
        for e in self.engines:
            e.set_link_mass_capture(on)

    def link_mass(self):
        """float64[R]: the total mass of each record's link categorical in the last sweep, from the rank that scored it."""
        return merge_link_mass([e.link_mass() for e in self.engines])

    @property
    def iteration(self):
        return self.engines[0].iteration

    def summary(self):
        return self.engines[0].summary()

    def last_exchange(self):
        out = []
        for e in self.engines:
            a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
            _lib.load().dbl_last_exchange(e._h, C.byref(a), C.byref(b), C.byref(c))
            out.append((a.value, b.value, c.value))
        return out

    def download_state(self):
        e0 = self.engines[0]
        parts = [e.download_owned() for e in self.engines]
        d = merge_owned(parts, e0.num_records, e0.num_entities, self.A)
        d["theta"] = e0.summary()["theta"]
        return d

    def state_hash(self):
        he = hr = 0
        for e in self.engines:
            a, b = e.state_hash()
            he, hr = (he + a) % (1 << 64), (hr + b) % (1 << 64)
        s = self.summary()
        return combine_state_hash(he, hr, s["theta"], s["iteration"])

    def close(self):
        for e in self.engines:
            e.close()
