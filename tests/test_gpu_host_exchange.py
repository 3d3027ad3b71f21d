"""The host-mediated exchange on ONE GPU: 2-3 contexts ("ranks") of a single device in one process, driven through
dbl_sweep_begin / dbl_exchange_pack / dbl_exchange_unpack / dbl_partial_summary / dbl_sweep_end without
dbl_comm_*.  The transport between the ranks is written here: every rank gets the slices of the send buffers
addressed to it, concatenated in source-rank order, and the partial summaries are summed in rank order.  None of the
calls waits for another rank, so one host thread drives all of them in turn.  The chain must be the oracle's after
every sweep (tests/test_distributed.py runs the same transport over NCCL with one process per GPU)."""
import ctypes as C

import numpy as np
import pytest

from helpers import oracle_setup, state_hash_numpy, synth_problem

pytestmark = pytest.mark.gpu


def make(world, g, seed, levels, split):
    import dblink_b200 as D

    rc = D.RecordsCache.build(g["values"], g["files"], g["attributes"])
    x, file = rc.transform_records(g["values"], g["files"])
    alpha = [a.alpha for a in g["attributes"]]
    beta = [a.beta for a in g["attributes"]]
    return make_engines(world, rc.indexes, alpha, beta, seed, len(rc.file_ids), x, file, levels, split), x, file


def make_engines(world, indexes, alpha, beta, seed, F, x, file, levels, split):
    """One context per rank from the initial state of the records, k-d blocks fitted on it, placed by LPT."""
    import dblink_b200 as D
    from dblink_b200.distributed import lpt_assign

    engines = [D.GibbsEngine(indexes, alpha, beta, None, seed, F, rank=r, world_size=world) for r in range(world)]
    for e in engines:
        e.init_state(x, file)
    y0 = engines[0].download_state()["y"]
    for e in engines:
        e.set_partitioner(D.KDTreePartitioner(levels, list(split)).fit(y0))
    link, blk = engines[0].links()
    P = engines[0].num_partitions
    cost = np.bincount(blk, minlength=P).astype(np.float64) * np.bincount(blk[link], minlength=P)
    set_owners(engines, lpt_assign(cost, world))
    return engines


def set_owners(engines, owner):
    from dblink_b200 import _lib
    from dblink_b200.engine import _check, _p

    owner = np.ascontiguousarray(owner, dtype=np.int32)
    for e in engines:
        _check(_lib.load().dbl_set_block_owners(e._h, _p(owner, _lib.i32p)), "set_block_owners", e._h)


def host_sweep(engines, sampler):
    """One sweep of every rank through the host-mediated calls -> messages sent (entities, records)."""
    import torch

    from dblink_b200 import _lib
    from dblink_b200.engine import SAMPLERS, _check, _p

    L, W = _lib.load(), len(engines)
    ew = engines[0].A + 1
    counts = []
    for e in engines:
        ec, rc = np.zeros(W, np.int64), np.zeros(W, np.int64)
        _check(L.dbl_sweep_begin(e._h, SAMPLERS[sampler], _p(ec, _lib.i64p), _p(rc, _lib.i64p)), "sweep_begin", e._h)
        counts.append((ec, rc))
    sent = []  # sent[s] = (entity slices, record slices) of rank s, by destination
    for e, (ec, rc) in zip(engines, counts):
        send_ent = torch.empty(int(ec.sum()) * ew, dtype=torch.int32, device="cuda")
        send_rec = torch.empty(int(rc.sum()) * 3, dtype=torch.int32, device="cuda")
        _check(L.dbl_exchange_pack(e._h, send_ent.data_ptr() if send_ent.numel() else None,
                                   send_rec.data_ptr() if send_rec.numel() else None), "exchange_pack", e._h)
        oe = np.concatenate([[0], np.cumsum(ec)]) * ew
        orc = np.concatenate([[0], np.cumsum(rc)]) * 3
        sent.append(([send_ent[oe[d]:oe[d + 1]] for d in range(W)], [send_rec[orc[d]:orc[d + 1]] for d in range(W)]))
    for d, e in enumerate(engines):
        recv_ent = torch.cat([sent[s][0][d] for s in range(W)])
        recv_rec = torch.cat([sent[s][1][d] for s in range(W)])
        torch.cuda.synchronize()  # the library reads the buffers on its own stream
        ne, nr = recv_ent.numel() // ew, recv_rec.numel() // 3
        _check(L.dbl_exchange_unpack(e._h, recv_ent.data_ptr() if ne else None, ne,
                                     recv_rec.data_ptr() if nr else None, nr), "exchange_unpack", e._h)
    nw = L.dbl_summary_words(engines[0]._h)
    total, ll = np.zeros(nw, np.int64), 0.0
    for e in engines:
        c, l = np.zeros(nw, np.int64), C.c_double(0.0)
        _check(L.dbl_partial_summary(e._h, _p(c, _lib.i64p), C.byref(l)), "partial_summary", e._h)
        total += c
        ll += l.value
    for e in engines:
        _check(L.dbl_sweep_end(e._h, _p(total, _lib.i64p), ll, 0), "sweep_end", e._h)
    return sum(int(ec.sum()) for ec, _ in counts), sum(int(rc.sum()) for _, rc in counts)


def assert_same(engines, st):
    from dblink_b200.distributed import merge_owned

    e0 = engines[0]
    d = merge_owned([e.download_owned() for e in engines], e0.num_records, e0.num_entities, e0.A)
    for k in ("link", "y", "z", "block"):
        np.testing.assert_array_equal(d[k], getattr(st, k), err_msg=k)
    os_ = st.summary()
    for e in engines:
        ps = e.summary()
        np.testing.assert_array_equal(ps["theta"], st.theta, err_msg="theta")
        assert ps["iteration"] == os_["iteration"] and ps["num_isolates"] == os_["num_isolates"]
        np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"])
        np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"])
        assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9)
    return d


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("sampler", ["PCG-II", "PCG-I", "Gibbs"])
def test_host_mediated_chain_equals_oracle(oracle, world, sampler):
    from dblink_b200 import _lib
    from dblink_b200.engine import _check, combine_state_hash

    g = synth_problem(seed=5, R=1500, n_files=2)
    engines, x, file = make(world, g, 99, 3, (2, 3))
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, 3, (2, 3))
    moved = 0
    for it in range(6):
        ent, rec = host_sweep(engines, sampler)
        moved += ent + rec
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        d = assert_same(engines, st)
    assert moved > 0, "clusters should move between ranks in this test"
    # the rank-count-invariant fingerprint equals the one computed from the oracle's state
    he = hr = 0
    for e in engines:
        a, b = e.state_hash()
        he, hr = (he + a) % (1 << 64), (hr + b) % (1 << 64)
    s = engines[0].summary()
    assert combine_state_hash(he, hr, s["theta"], s["iteration"]) == \
        combine_state_hash(*state_hash_numpy(st.y, st.link, st.z), st.theta, st.iteration)
    # resume from host arrays with the block -> rank table the contexts hold on the device, keep following the oracle
    for e in engines:
        e.upload_state(x, file, d["z"], d["link"], d["y"], st.theta, iteration=st.iteration)
        _check(_lib.load().dbl_set_block_owners(e._h, None), "set_block_owners", e._h)
    for it in range(2):
        host_sweep(engines, sampler)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        assert_same(engines, st)
    for e in engines:
        e.close()
