"""Several chains without a GPU: split-R̂ and rank-normalised R̂ against a literal restatement, the project's
numChains settings and run.txt, the pooled reader of several linkage chains, and the ABI's argument checks."""
import math
import os
import statistics

import numpy as np
import pytest

from test_host_pipeline import GOLDEN, make_conf


# ---- R̂, restated with plain Python loops ----------------------------------------------------------------------
def _lit_halves(chains):
    out = []
    for c in chains:
        c = [float(v) for v in c]
        N = len(c) // 2
        out += [c[:N], c[len(c) - N:]]
    return out


def _lit_rhat(halves):
    M, N = len(halves), len(halves[0])
    means = [sum(h) / N for h in halves]
    W = sum(sum((v - m) ** 2 for v in h) / (N - 1) for h, m in zip(halves, means)) / M
    g = sum(means) / M
    BN = sum((m - g) ** 2 for m in means) / (M - 1)
    return float("nan") if W == 0 else math.sqrt(((N - 1) / N * W + BN) / W)


def _lit_z(halves):
    flat = [v for h in halves for v in h]
    S = len(flat)
    inv = statistics.NormalDist().inv_cdf
    z = []
    for v in flat:
        less = sum(1 for u in flat if u < v)
        eq = sum(1 for u in flat if u == v)
        z.append(inv((less + (eq + 1) / 2 - 0.375) / (S + 0.25)))
    N = len(halves[0])
    return [z[i * N:(i + 1) * N] for i in range(len(halves))]


def lit_split_rhat(chains):
    return _lit_rhat(_lit_halves(chains))


def lit_rank_rhat(chains):
    h = _lit_halves(chains)
    med = statistics.median([v for x in h for v in x])
    folded = [[abs(v - med) for v in x] for x in h]
    return max(_lit_rhat(_lit_z(h)), _lit_rhat(_lit_z(folded)))


@pytest.mark.parametrize("K,n", [(2, 8), (3, 9), (4, 21), (2, 5)])
def test_rhat_against_literal_loops(K, n):
    from dblink_b200 import convergence as cv

    rng = np.random.default_rng(K * 100 + n)
    for draws in (rng.normal(size=(K, n)), rng.integers(0, 4, size=(K, n)).astype(float)):  # the second has ties
        assert cv.split_rhat(draws) == pytest.approx(lit_split_rhat(draws), rel=1e-12)
        assert cv.rank_normalized_split_rhat(draws) == pytest.approx(lit_rank_rhat(draws), rel=1e-12)


def test_rhat_behaviour():
    from dblink_b200 import convergence as cv

    rng = np.random.default_rng(3)
    iid = rng.normal(size=(4, 4000))
    assert cv.split_rhat(iid) < 1.01 and cv.rank_normalized_split_rhat(iid) < 1.01
    shifted = iid + np.arange(4)[:, None]
    assert cv.split_rhat(shifted) > 1.1 and cv.rank_normalized_split_rhat(shifted) > 1.1
    const = np.full((3, 10), 7.0)
    assert math.isnan(cv.split_rhat(const)) and math.isnan(cv.rank_normalized_split_rhat(const))
    with pytest.raises(ValueError):
        cv.split_rhat(rng.normal(size=(2, 3)))


def test_convergence_diagnostics_file(tmp_path):
    from dblink_b200 import convergence as cv

    rng = np.random.default_rng(1)
    paths = []
    for k in range(3):
        p = tmp_path / f"d{k}.csv"
        rows = ["iteration,systemTime-ms,logLikelihood,popSize,numObservedEntities"]
        rows += [f"{10 * i},{i * 3},{rng.normal()!r},500,{400 + int(rng.integers(0, 5))}" for i in range(12)]
        p.write_text("\n".join(rows) + "\n")
        paths.append(str(p))
    out = cv.convergence_diagnostics(paths, lower_iteration_cutoff=30)
    assert [r[0] for r in out] == ["logLikelihood", "numObservedEntities"]
    assert all(r[3] == 3 and r[4] == 9 for r in out)
    cv.save_convergence_diagnostics(out, str(tmp_path))
    lines = (tmp_path / "convergence-diagnostics.csv").read_text().splitlines()
    assert lines[0] == "quantity,splitRhat,rankNormalizedSplitRhat,numChains,drawsPerChain"
    assert len(lines) == 3
    with pytest.raises(ValueError):
        cv.convergence_diagnostics(paths, lower_iteration_cutoff=90)  # 3 draws per chain
    with pytest.raises(ValueError):
        cv.convergence_diagnostics(paths[:1])


# ---- project settings ------------------------------------------------------------------------------------------
def _project(tmp_path, extra="", quantities=None):
    from dblink_b200 import config
    from dblink_b200.project import Project

    conf = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), str(tmp_path) + "/")
    conf = conf.replace("randomSeed : 319158", "randomSeed : 319158\n    " + extra)
    if quantities:
        conf = conf.replace('quantities : ["cluster-size-distribution", "partition-sizes"]', "quantities : " + quantities)
    return Project(config.parse_string(conf), base_dir="")


def test_num_chains_setting_and_run_txt(tmp_path):
    p1 = _project(tmp_path)
    assert p1.num_chains == 1 and p1.chain_dirs() == [str(tmp_path) + "/"]
    assert "numChains" not in p1.mk_string()
    p3 = _project(tmp_path, "numChains : 3")
    assert p3.num_chains == 3 and p3.chain_seeds() == [319158, 319159, 319160]
    assert [os.path.basename(d) for d in p3.chain_dirs()] == ["chain-0", "chain-1", "chain-2"]
    assert ("  * Running numChains=3 chains with seeds 319158, 319159, 319160 (one k-d tree, fitted on chain 0; "
            "chains start from State.deterministic, not over-dispersed), outputs under chain-<k>/") in p3.mk_string()
    assert p3.fingerprint() != p1.fingerprint()
    for bad in ("numChains : 0", "numChains : -2", 'numChains : "two"', "numChains : 1.5"):
        with pytest.raises(ValueError):
            _project(tmp_path, bad)
    q = '["convergence-diagnostics"]'
    with pytest.raises(ValueError):
        _project(tmp_path, "", q).steps()  # one chain: no R̂
    assert _project(tmp_path, "numChains : 2", q).steps()[1][1]["quantities"] == ["convergence-diagnostics"]


# ---- the pooled reader -----------------------------------------------------------------------------------------
def _write_chain(path, samples):
    """samples: [(iteration, {partition id: [[record ids], ...]})]"""
    import pyarrow as pa

    from dblink_b200.writers import LinkageChainWriter

    w = LinkageChainWriter(path, 10, False)
    for it, parts in samples:
        w.append(it, {pid: pa.array(cl, pa.list_(pa.string())) for pid, cl in parts.items()})
    w.close()


def test_pooled_reader(tmp_path):
    from dblink_b200 import analysis_arrays as aa

    a, b, c = str(tmp_path / "a"), str(tmp_path / "b"), str(tmp_path / "c")
    _write_chain(a, [(0, {0: [["r1", "r2"], ["r3"]]}), (10, {0: [["r1"], ["r2", "r3"]]})])
    # another record order and partition split: mapped through chain a's dictionary
    _write_chain(b, [(0, {0: [["r3", "r1"]], 1: [["r2"]]}), (10, {1: [["r2", "r1", "r3"]]})])
    ch = aa.read_pooled_chain_arrays([a, b], 0)
    ids = ch.record_ids.to_pylist()
    assert list(ch.iterations) == [0, 10, 0, 10]  # chain-major, then by iteration
    got = []
    for mem, off, part in ch.samples:
        got.append(sorted((int(part[i]), sorted(ids[m] for m in mem[off[i]:off[i + 1]])) for i in range(len(part))))
    assert got == [[(0, ["r1", "r2"]), (0, ["r3"])], [(0, ["r1"]), (0, ["r2", "r3"])],
                   [(0, ["r1", "r3"]), (1, ["r2"])], [(1, ["r1", "r2", "r3"])]]
    assert list(aa.read_pooled_chain_arrays([a, b], 10).iterations) == [10, 10]
    _write_chain(c, [(0, {0: [["r1", "r2"], ["r4"]]})])
    with pytest.raises(ValueError):
        aa.read_pooled_chain_arrays([a, c], 0)


# ---- ABI -------------------------------------------------------------------------------------------------------
def test_chains_abi_rejects_a_missing_context():
    from dblink_b200 import _lib

    L = _lib.load()
    x = np.zeros((4, 1), np.int32)
    f = np.zeros(4, np.int32)
    s = np.array([1, 2], np.uint64)
    xp, fp, sp = x.ctypes.data_as(_lib.i32p), f.ctypes.data_as(_lib.i32p), s.ctypes.data_as(_lib.u64p)
    assert L.dbl_chains_init(None, 2, sp, 4, xp, fp, 0) == _lib.ERR_INVALID
    assert L.dbl_chains_upload(None, 2, sp, 4, 4, xp, fp, None, None, None, None, 0) == _lib.ERR_INVALID
    assert L.dbl_chains_download(None, None, None, None, None, None) == _lib.ERR_INVALID
    assert L.dbl_chain_summary(None, 0, None, None, None, None) == _lib.ERR_INVALID
    assert L.dbl_num_chains(None) == 0
