"""Sharded sweeps on every link-kernel family and value-draw path, with every record's link mass.

The models of tests/test_gpu_link_kernels.py (hash tables of 64 / 128 / 256 slots, both generic fall-backs, 255 / 256
constant values, A = 32, the pruned kernel's crafted branches) and the crafted large clusters of
tests/test_value_reference.py, each sharded over 2-3 contexts of one GPU (LocalShards, and the host-mediated calls of
tests/test_gpu_host_exchange.py).  Several paths only run on a shard: entity messages of A + 1 words, record messages
whose z mask uses bit 31 at A = 32, k_link_pruned / k_link_heavy and k_values_rescaled over a rank's owned rows, and
blocks that migrate while they hold heavy records or large clusters.

After every sweep the merged state equals the oracle's and so does every record's link-categorical total, merged from
the ranks' dbl_link_mass arrays (distributed.merge_link_mass) and compared bit for bit: a draw only moves when its
uniform falls into the interval a wrong weight shifts, the total sees every candidate's weight.
"""
import numpy as np
import pytest

import test_gpu_host_exchange as HX
import test_gpu_multirank as MR
from helpers import assert_same_mass, oracle_model_setup, oracle_setup, random_state, synth_problem
from test_gpu_link_kernels import (HEAVY_MIN_CANDIDATES, PRUNED_SCAP, ROWS, SAMPLERS, crafted_pruned_state,
                                   expected_kernel, survivors)
from test_gpu_value_reference import crafted_setup

pytestmark = pytest.mark.gpu

LAYOUTS = ((2, 0), (2, 1), (2, 2), (3, 0))  # (ranks, link mode)
LEVELS = 2  # 4 blocks: every rank of 3 owns one
# k-d split attributes per row: a string attribute with enough values to split twice
SPLIT = dict({row: (0,) for row in ROWS}, a32=(1, 3), pruned=(1,), pruned_bsearch=(1,))
PRUNED_E = 1200  # crafted pruned states: more entities than records, blocks beyond 256 entities on ranks 1 and 2


def check(sh, st, what):
    MR.assert_same(sh, st)
    assert_same_mass(sh.link_mass(), st.last_link_mass(), what)


def run_chain(oracle, shards, st, sampler, n, call, what):
    """n single sweeps, then one call of `call` sweeps (a replayed graph); -> cluster messages sent per shard"""
    moved = [0] * len(shards)
    for it in range(n):
        for sh in shards:
            sh.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        for i, sh in enumerate(shards):
            check(sh, st, f"{what} {sh.world} ranks sweep {it}")
            moved[i] += sum(e + r for e, r, _ in sh.last_exchange())
    for sh in shards:
        sh.sweep(sampler, call)
    assert st.sweep(oracle.SAMPLERS[sampler], call) == 0
    for sh in shards:
        check(sh, st, f"{what} {sh.world} ranks, {call} sweeps in one call")
    return moved


def pruned_start(oracle, m, x, file, Vs):
    """A crafted pruned state over several blocks -> (y, link, z, theta, block of each record, {branch: records})"""
    rng = np.random.default_rng(5)
    y, link, z = crafted_pruned_state(rng, x, PRUNED_E, Vs)
    theta = rng.uniform(0.01, 0.3, (len(Vs), int(file.max()) + 1))
    block = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0).block
    assert len(np.unique(block)) >= 2
    nmm, ns, nb = survivors(x, z, y, link, block).T
    branches = {"re-walk": (nmm > 0) & (ns > PRUNED_SCAP),  # pass 2 walks the postings again
                "single survivor": (nmm > 0) & (ns == 1),
                "k_link_heavy": (nmm == 0) & (nb > HEAVY_MIN_CANDIDATES)}
    return y, link, z, theta, block[link], branches


def branch_owner(rec_block, branches, world):
    """blocks placed so that the single-survivor record's block is on rank 1, the others round robin"""
    first = rec_block[np.flatnonzero(branches["single survivor"])[0]]
    return (np.arange(int(rec_block.max()) + 1) - first + 1) % world


def assert_branches_off_rank0(owners, rec_block, branches):
    """every branch happens in a block the context's own block -> rank table gives to a rank other than 0"""
    off0 = owners[rec_block] != 0
    for name, sel in branches.items():
        assert (off0 & sel).any(), name


@pytest.mark.parametrize("sampler", SAMPLERS)
@pytest.mark.parametrize("row", list(ROWS))
def test_sharded_link_kernel_against_oracle(oracle, monkeypatch, row, sampler):
    recipe, _, slots, _, _, env = ROWS[row]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = recipe()
    split = SPLIT[row]
    shards = []
    for world, mode in LAYOUTS:
        sh, rc, x, file = MR.make(world, g, 31, LEVELS, split)
        for e in sh.engines:
            e.set_link_mode(mode)
        sh.set_link_mass_capture(True)
        shards.append(sh)
    # routing first, on every rank: the row tests what it says it tests
    for (world, mode), sh in zip(LAYOUTS, shards):
        assert set(sh.block_owners().tolist()) == set(range(world))
        for e in sh.engines:
            assert [ix.hash_slots for ix in e.indexes] == slots
            for s in SAMPLERS:
                assert e.link_kernel(s) == expected_kernel(row, s, mode), (row, world, s, mode)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 31, LEVELS, split)
    np.testing.assert_array_equal(x, ox)
    moved = run_chain(oracle, shards, st, sampler, 3, 3, f"{row} {sampler} init")
    assert all(moved), f"clusters should move between ranks: {moved}"

    # the next states have another number of entities than the chain so far: the sweeps after them reallocate
    if row.startswith("pruned"):
        Vs = [ix.num_values for ix in rc.indexes]
        y, link, z, theta, rec_block, branches = pruned_start(oracle, m, x, file, Vs)
        for sh in shards:
            sh.upload_state(x, file, z, link, y, theta, iteration=10, owner=branch_owner(rec_block, branches, sh.world))
            assert_branches_off_rank0(sh.block_owners(), rec_block, branches)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10)
        run_chain(oracle, shards, st, sampler, 2, 2, f"{row} {sampler} crafted")
        if row == "pruned":
            # every block on rank 0, re-placed after every sweep: blocks holding heavy records migrate
            sh = shards[-1]
            sh.upload_state(x, file, z, link, y, theta, iteration=10, owner=np.zeros(int(rec_block.max()) + 1))
            sh.set_rebalance(1, 1.0)
            st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10)
            assert (sh.block_owners() == 0).all()
            run_chain(oracle, [sh], st, sampler, 3, 2, f"{row} {sampler} re-placed")
            heavy_blocks = np.unique(rec_block[branches["k_link_heavy"]])
            assert (sh.block_owners()[heavy_blocks] != 0).any(), "no block holding k_link_heavy records migrated"
    else:
        # a random valid state of R / 3 entities: many distorted records (A = 32: z mask bit 31) in clusters that
        # change block
        rng = np.random.default_rng(5)
        Vs = [ix.num_values for ix in rc.indexes]
        y, link, z = random_state(rng, x, x.shape[0] // 3, Vs)
        theta = rng.uniform(0.01, 0.3, (len(Vs), int(file.max()) + 1))
        for sh in shards:
            sh.upload_state(x, file, z, link, y, theta, iteration=10)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10)
        run_chain(oracle, shards, st, sampler, 2, 2, f"{row} {sampler} random state")
    for sh in shards:
        sh.close()


def crafted_shards(oracle, world, sizes=None, pad=0, owner0=False):
    """the crafted clusters of tests/test_gpu_value_reference.py on `world` ranks (two blocks: the k-d tree fitted on
    the records' initial state splits the constant attribute), block b on rank (b + 1) % world, or every block on
    rank 0 -> (shards, oracle state, entities of the 300-record clusters)"""
    from dblink_b200.distributed import LocalShards

    dix, part, (m,), arrays, info = crafted_setup(oracle, pad=pad, sizes=sizes, initial_tree=True)
    x, file, z, link, y, theta = arrays
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    P = int(st.block.max()) + 1
    assert P == 2
    big = np.array([e for e, size, _, _ in info if size == 300])
    sh = LocalShards(dix, m.alpha, m.beta, seed=m.seed, num_files=m.F, levels=1, split_attrs=[3], world=world)
    sh.init_state(x, file)
    sh.upload_state(x, file, z, link, y, theta, 0, owner=np.zeros(P) if owner0 else (np.arange(P) + 1) % world)
    sh.set_link_mass_capture(True)
    if owner0:
        assert (sh.block_owners() == 0).all()
    else:
        assert_big_clusters_off_rank0(sh, big)
    return sh, st, big


def assert_big_clusters_off_rank0(sh, big):
    """a rank other than 0 holds a 300-record cluster: it draws that entity's values (rescaled at this size)"""
    held = [np.intersect1d(e.download_owned()["ent_ids"], big).size for e in sh.engines]
    assert sum(held) == big.size and sum(held[1:]) > 0, held


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("sampler", SAMPLERS)
def test_sharded_crafted_clusters(oracle, world, sampler):
    """81 crafted clusters of 1 to 300 records in two blocks on different ranks: k_values<8> and k_values_rescaled"""
    sh, st, big = crafted_shards(oracle, world)
    MR.assert_same(sh, st)
    run_chain(oracle, [sh], st, sampler, 2, 2, f"crafted {sampler}")
    sh.close()


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("sampler", ["PCG-II", "PCG-I"])
def test_sharded_crafted_clusters_among_isolated_entities(oracle, world, sampler):
    """the largest crafted clusters with 300 000 isolated entities: E * A beyond sm_count * 8192, so k_values<2>"""
    sh, st, big = crafted_shards(oracle, world, sizes=[2, 55, 91, 300], pad=300_000)
    sh.sweep(sampler, 1)
    assert st.sweep(oracle.SAMPLERS[sampler]) == 0
    check(sh, st, f"crafted among isolated entities {sampler}")
    sh.close()


def test_sharded_crafted_clusters_re_placed(oracle):
    """the crafted clusters from every block on rank 0, re-placed after every sweep: large clusters migrate"""
    sh, st, big = crafted_shards(oracle, 3, owner0=True)
    sh.set_rebalance(1, 1.0)
    run_chain(oracle, [sh], st, "PCG-I", 3, 2, "crafted re-placed")
    assert_big_clusters_off_rank0(sh, big)
    sh.close()


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_sharded_population_and_files(oracle, sampler):
    """3 files, a population of 1.3 R (isolated entities from the start), 3 ranks: every rank's reduction of the summary
    slots gives the oracle's per-file distortion counts, isolates and log-likelihood"""
    g = synth_problem(seed=21, R=1500, n_files=3)
    pop = 1950
    sh, rc, x, file = MR.make(3, g, 77, 3, (2, 3), population_size=pop)
    sh.set_link_mass_capture(True)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 77, 3, (2, 3), pop=pop)
    assert st.y.shape[0] == pop and st.summary()["agg_dist"].shape == (4, 3)
    assert set(sh.block_owners().tolist()) == {0, 1, 2}
    for it in range(4):
        sh.sweep(sampler, 1)
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        check(sh, st, f"population {sampler} sweep {it}")
        os_ = st.summary()
        assert os_["num_isolates"] > 0
        for r, e in enumerate(sh.engines):
            ps = e.summary()
            assert ps["iteration"] == os_["iteration"] and ps["num_isolates"] == os_["num_isolates"], r
            np.testing.assert_array_equal(ps["agg_dist"], os_["agg_dist"], err_msg=f"rank {r}")
            np.testing.assert_array_equal(ps["rec_dist"], os_["rec_dist"], err_msg=f"rank {r}")
            assert ps["log_likelihood"] == pytest.approx(os_["log_likelihood"], rel=1e-9)
    sh.close()


def test_sharded_state_of_another_size(oracle):
    """after sweeps, states with more and with fewer entities: a state of another shape closes the communication
    buffers and dbl_sweep refuses it until the ranks connect again; then the sweeps, which reallocate buffers while a
    peer context of the same device may wait in the exchange barrier, follow the oracle"""
    import dblink_b200 as D

    g = synth_problem(seed=5, R=1500, n_files=2)
    sh, rc, x, file = MR.make(2, g, 99, 3, (2, 3))
    sh.set_link_mass_capture(True)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 99, 3, (2, 3))
    run_chain(oracle, [sh], st, "PCG-II", 2, 2, "initial")
    rng = np.random.default_rng(3)
    Vs = [ix.num_values for ix in rc.indexes]
    theta = rng.uniform(0.01, 0.3, (len(Vs), 2))
    y, link, z = random_state(rng, x, 2 * x.shape[0], Vs)
    owner = sh.block_owners()
    for e in sh.engines:  # uploaded without connecting again
        e.upload_state(x, file, z, link, y, theta, 4)
    sh.set_owners(owner)
    with pytest.raises(D.DblinkError, match="dbl_comm_export / dbl_comm_import first"):
        sh.sweep("PCG-II", 1)
    sh.upload_state(x, file, z, link, y, theta, iteration=4)  # connects again
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 4)
    run_chain(oracle, [sh], st, "PCG-I", 2, 2, "larger state")
    y, link, z = random_state(rng, x, x.shape[0] // 2, Vs)
    sh.upload_state(x, file, z, link, y, theta, iteration=8)  # connects again
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 8)
    run_chain(oracle, [sh], st, "Gibbs", 2, 2, "smaller state")
    sh.close()


def test_sharded_one_record_per_warp_shape(oracle):
    """k_link_pcg2 with 9 non-constant attributes (one record per warp) on 2 ranks"""
    from dblink_b200.distributed import LocalShards
    from test_gpu_link_shapes import _model, expected_format

    p_idx, o_idx, x, file, F, kpos = _model(oracle, 1, 9)
    A = len(p_idx)
    alpha, beta, seed, split = [10.0] * A, [1000.0] * A, 41, [kpos[1], kpos[2]]
    sh = LocalShards(p_idx, alpha, beta, seed=seed, num_files=F, levels=2, split_attrs=split, world=2)
    for e in sh.engines:
        assert e.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS=9,HC=32,PK=1>"
        assert e.link_tile_format("PCG-II") == expected_format(9, "sc16")
    sh.init_state(x, file)
    sh.set_link_mass_capture(True)
    assert set(sh.block_owners().tolist()) == {0, 1}
    m, st, tree = oracle_model_setup(oracle, o_idx, alpha, beta, seed, F, x, file, 2, split)
    run_chain(oracle, [sh], st, "PCG-II", 3, 3, "NS=9")
    sh.close()


# ---- host-mediated transport --------------------------------------------------------------------------------------
def host_chain(oracle, engines, st, sampler, n, what):
    from dblink_b200.distributed import merge_link_mass

    moved = 0
    for it in range(n):
        ent, rec = HX.host_sweep(engines, sampler)
        moved += ent + rec
        assert st.sweep(oracle.SAMPLERS[sampler]) == 0
        HX.assert_same(engines, st)
        assert_same_mass(merge_link_mass([e.link_mass() for e in engines]), st.last_link_mass(), f"{what} sweep {it}")
    return moved


def block_owners(engine):
    from dblink_b200 import _lib
    from dblink_b200.engine import _check, _p

    out = np.zeros(engine.num_partitions, np.int32)
    _check(_lib.load().dbl_block_owners(engine._h, _p(out, _lib.i32p)), "block_owners", engine._h)
    return out


def host_upload(engines, arrays, owner, iteration):
    x, file, z, link, y, theta = arrays
    for e in engines:
        e.upload_state(x, file, z, link, y, theta, iteration=iteration)
    HX.set_owners(engines, owner)


@pytest.mark.parametrize("sampler", SAMPLERS)
@pytest.mark.parametrize("row", ["a32", "pruned"])
def test_host_mediated_link_kernels(oracle, row, sampler):
    """entity messages of A + 1 words sized on the host, record messages with bit 31 of the z mask, and the crafted
    pruned branches on rank 1, through the host-mediated calls on 2 ranks"""
    g = ROWS[row][0]()
    split = SPLIT[row]
    engines, x, file = HX.make(2, g, 31, LEVELS, split)
    for e in engines:
        e.set_link_mass_capture(True)
    m, st, tree, ox, ofile = oracle_setup(oracle, g, 31, LEVELS, split)
    assert host_chain(oracle, engines, st, sampler, 3, f"host {row} {sampler}") > 0
    if row == "pruned":
        Vs = [ix.num_values for ix in engines[0].indexes]
        y, link, z, theta, rec_block, branches = pruned_start(oracle, m, x, file, Vs)
        host_upload(engines, (x, file, z, link, y, theta), branch_owner(rec_block, branches, 2), 10)
        assert_branches_off_rank0(block_owners(engines[0]), rec_block, branches)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10)
        host_chain(oracle, engines, st, sampler, 2, f"host {row} {sampler} crafted")
    else:
        rng = np.random.default_rng(5)
        Vs = [ix.num_values for ix in engines[0].indexes]
        y, link, z = random_state(rng, x, x.shape[0], Vs)
        theta = rng.uniform(0.01, 0.3, (len(Vs), int(file.max()) + 1))
        host_upload(engines, (x, file, z, link, y, theta), np.arange(4) % 2, 10)
        st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 10)
        host_chain(oracle, engines, st, sampler, 2, f"host {row} {sampler} random state")
    for e in engines:
        e.close()


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_host_mediated_crafted_clusters(oracle, sampler):
    dix, part, (m,), arrays, info = crafted_setup(oracle, initial_tree=True)
    x, file, z, link, y, theta = arrays
    engines = HX.make_engines(2, dix, m.alpha, m.beta, m.seed, m.F, x, file, 1, [3])
    for e in engines:
        e.set_link_mass_capture(True)
    st = oracle.State.from_arrays(m, x, file, z, link, y, theta, 0)
    host_upload(engines, arrays, (np.arange(int(st.block.max()) + 1) + 1) % 2, 0)
    host_chain(oracle, engines, st, sampler, 2, f"host crafted {sampler}")
    for e in engines:
        e.close()
