"""k_link_pcg2 on records with missing non-constant values: the 1/n(y) of every tile entity travel with the tiles as
one f64 column per non-constant attribute, and the producer stages the columns its work item's records miss in the
ring stage of each tile.  dbl_link_kernel reports that path (+256).  The records are grouped by the first attribute
they miss (k_rec_class), and the cases below reach what that grouping does not settle on its own: records missing
each non-constant attribute in turn, records missing several at once, work items whose 16 records miss all six
attributes between them (every record misses the first one and one other), warps whose two records miss different
attributes, and the block's last warp with one record (R odd, one block).  Each sweep must equal the oracle's state
and give every record's categorical the oracle's total, bit for bit, with the sweep replayed as a CUDA graph and
enqueued kernel by kernel, and in a 2-rank sharded chain.
"""
import numpy as np
import pytest

from helpers import assert_same_mass
from test_gpu_link_shapes import R, _model
from test_gpu_multirank import assert_same
from test_gpu_parity import assert_same_state

pytestmark = pytest.mark.gpu

N_CONST, N_STR = 4, 6  # the benchmark's shape: paired tables, two records per warp


def _records(O):
    """The _model of test_gpu_link_shapes at the benchmark's shape, with missing-value patterns of its own."""
    p_idx, o_idx, x, file, F, kpos = _model(O, N_CONST, N_STR, seed=3)
    strs = kpos[N_CONST:]
    x = x.copy()
    x[:, strs] = np.where(x[:, strs] < 0, 0, x[:, strs])  # start from records that miss no string value
    rng = np.random.default_rng(5)
    rows = rng.permutation(np.arange(255, R))
    k = 0
    for q in range(N_STR):  # each attribute in turn
        x[rows[k:k + 20], strs[q]] = -1
        k += 20
    for r in rows[k:k + 15]:  # several at once
        x[r, rng.choice(strs, rng.integers(2, 4), replace=False)] = -1
    k += 15
    for i, r in enumerate(rows[k:k + 32]):  # the first attribute and one other: 6 columns per work item
        x[r, strs[0]] = -1
        x[r, strs[1 + i % (N_STR - 1)]] = -1
    return p_idx, o_idx, np.ascontiguousarray(x), file, F, kpos


@pytest.mark.parametrize("graph", [1, 2], ids=["eager", "graph"])
def test_missing_columns_against_oracle(oracle, graph):
    import dblink_b200 as D
    from dblink_b200 import _lib

    O = oracle
    p_idx, o_idx, x, file, F, kpos = _records(O)
    strs = kpos[N_CONST:]
    miss = x[:, strs] < 0
    assert all(((miss.sum(axis=1) == 1) & miss[:, q]).sum() >= 20 for q in range(N_STR))
    assert (miss.sum(axis=1) >= 2).sum() >= 40
    A = N_CONST + N_STR
    alpha, beta, seed = [10.0] * A, [1000.0] * A, 17
    eng = D.GibbsEngine(p_idx, alpha, beta, None, seed, F)
    eng.init_state(x, file)
    eng.set_partitioner(D.KDTreePartitioner(0, []).fit(eng.download_state()["y"]))
    eng.set_link_mass_capture(True)
    eng.set_graph_mode(graph)
    assert eng.link_kernel("PCG-II") == f"k_link_pcg2<A={A},NS={N_STR},HC=32,PK=1>"
    k = _lib.load().dbl_link_kernel(eng._h, _lib.SAMPLERS["PCG-II"])
    assert k & 256, "the 1/n(y) columns are staged with the tiles"
    assert eng.link_tile_format("PCG-II") == {"id16": True, "slot_codes": True, "paired": True,
                                              "records_per_warp": 2}

    m0 = O.Model(o_idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    m = O.Model(o_idx, alpha, beta, O.KDTree.fit(s0.y, 0, []), seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0)
    for it in range(4):
        eng.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same_state(eng, st)
        assert_same_mass(eng.link_mass(), st.last_link_mass(), f"missing columns sweep {it}")
    eng.close()


def test_no_missing_value_no_columns(oracle):
    """A model whose records miss no non-constant value builds no columns and does not report them."""
    import dblink_b200 as D
    from dblink_b200 import _lib

    p_idx, o_idx, x, file, F, kpos = _records(oracle)
    strs = kpos[N_CONST:]
    x = x.copy()
    x[:, strs] = np.where(x[:, strs] < 0, 0, x[:, strs])
    A = N_CONST + N_STR
    eng = D.GibbsEngine(p_idx, [10.0] * A, [1000.0] * A, None, 17, F)
    eng.init_state(x, file)
    eng.set_partitioner(D.KDTreePartitioner(0, []).fit(eng.download_state()["y"]))
    eng.sweep("PCG-II", 1)
    assert not _lib.load().dbl_link_kernel(eng._h, _lib.SAMPLERS["PCG-II"]) & 256
    eng.close()


def test_missing_columns_sharded(oracle):
    from dblink_b200.distributed import LocalShards

    O = oracle
    p_idx, o_idx, x, file, F, kpos = _records(O)
    strs = kpos[N_CONST:]
    A = N_CONST + N_STR
    alpha, beta, seed, levels, split = [10.0] * A, [1000.0] * A, 23, 2, [strs[0], strs[1]]
    sh = LocalShards(p_idx, alpha, beta, seed=seed, num_files=F, levels=levels, split_attrs=split, world=2)
    sh.init_state(x, file)
    m0 = O.Model(o_idx, alpha, beta, None, seed, F)
    s0 = O.State.init(m0, x, file, 0)
    m = O.Model(o_idx, alpha, beta, O.KDTree.fit(s0.y, levels, split), seed, F)
    st = O.State.from_arrays(m, x, file, s0.z, s0.link, s0.y, s0.theta, 0)
    st._keep = (m0, s0)
    for it in range(3):
        sh.sweep("PCG-II", 1)
        assert st.sweep(O.PCG_II) == 0
        assert_same(sh, st)
    sh.close()
