"""Per-pair MCMC diagnostics on the GPU (dbl_pairs_trace_* and dbl_pairs_mixing in dbl_posterior.cu,
analysis_gpu.pairwise_match_diagnostics) against the numpy path in analysis_arrays.py: counts, per-chain counts and
max_t exactly, split-R̂ and ESS bit for bit, from 2 to 1 M records, 1 to 8 chains and 2 to 1000 draws per half with
half starts off word boundaries; the trace's bits through windows of the mixing call; host and device labels and
outputs; every refusal leaves the handle usable; the project's files equal the host path's."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_gpu_posterior import random_chain
from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu


def pooled(ch, K, n, extra):
    """ch's samples as K chains, chain k of n + k * extra samples (ch must hold enough)."""
    sizes = [n + k * extra for k in range(K)]
    S = sum(sizes)
    assert len(ch.samples) >= S
    return type(ch)(ch.record_ids, ch.iterations[:S], ch.samples[:S], np.repeat(np.arange(K), sizes))


def assert_equal_to_numpy(ch, min_count=1):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    *got, gm = ag.pairwise_match_diagnostics(ch, min_count)
    *want, wm = aa.pairwise_match_diagnostics(ch, min_count)
    for g, w in zip(got, want):
        assert g.dtype == np.int64 and np.array_equal(g, w)
    for name in ("count", "chain_min", "chain_max", "max_t"):
        assert np.array_equal(getattr(gm, name), getattr(wm, name)), name
    for name in ("rhat", "ess"):  # bit for bit, NaN and inf included
        assert np.array_equal(getattr(gm, name).view(np.int64), getattr(wm, name).view(np.int64)), name
    assert (gm.M, gm.draws) == (wm.M, wm.draws)
    return got, gm


# (R, K, n, extra): N = n // 2 in {2, 31, 32, 33, 64, 65, 1000}; extra > 0 puts later chains' starts off word
# boundaries
CASES = [(2, 1, 4, 0), (6, 3, 5, 1), (40, 1, 63, 0), (2500, 2, 64, 1), (50_000, 3, 66, 2), (500, 8, 129, 1),
         (300, 8, 130, 3), (300, 2, 2001, 5)]


@pytest.mark.parametrize("R,K,n,extra", CASES)
def test_random_chains_equal_numpy(R, K, n, extra):
    ch = pooled(random_chain(R, K * n + K * K * extra, seed=R + 31 * n), K, n, extra)
    (first, _, _), mix = assert_equal_to_numpy(ch)
    if R >= 40:
        assert len(first) > 0 and (mix.max_t > 0).any() and np.isfinite(mix.ess).any()


def test_min_counts_select_on_the_device():
    from dblink_b200 import analysis_arrays as aa

    ch = pooled(random_chain(2500, 210, seed=11), 3, 60, 7)
    S = len(ch.samples)
    sizes = []
    for t in (0.0, 0.1, 0.5, 0.9, 1.0):
        (first, _, count), _ = assert_equal_to_numpy(ch, aa.min_match_count(t, S))
        sizes.append(len(first))
    assert sizes[1] > 0 and sizes == sorted(sizes, reverse=True) and len(set(sizes)) > 2


def test_a_cluster_of_12000_records_next_to_small_ones():
    from test_match_probabilities_host import random_chain as chain_with_big

    ch = chain_with_big(50_000, 10, seed=8, big=12_000)
    ch = type(ch)(ch.record_ids, ch.iterations, ch.samples, np.repeat([0, 1], 5))
    (first, _, count), mix = assert_equal_to_numpy(ch)
    assert len(first) > 12_000 * 11_999 // 2 and (count == 1).sum() > 12_000 * 11_999 // 4


def test_million_records():
    """The chain of profiles/scripts/smpc_time.py: R = 1 M, 64 partitions, S = 100, as 1 chain and as 4 of 25."""
    from dblink_b200 import analysis_arrays as aa

    R, S = 1_000_000, 100
    rng = np.random.default_rng(12345)
    E = (3 * R) // 4
    blk = rng.integers(0, 64, E).astype(np.int32)
    base = rng.integers(0, E, R).astype(np.int32)
    samples = []
    for s in range(S):
        link = base.copy()
        move = rng.random(R) < 0.3
        link[move] = rng.integers(0, E, int(move.sum()))
        if s % 3 == 0:
            base = link
        samples.append(aa.sample_from_links(link, blk))
    ch = aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples)
    # the pairs seen in at least 8 samples: the device's trace still holds all 34 M pairs; numpy takes fewer
    _, mix = assert_equal_to_numpy(ch, 8)
    assert len(mix.count) > 10_000 and (mix.max_t > 0).any()
    assert_equal_to_numpy(type(ch)(ch.record_ids, ch.iterations, ch.samples, np.repeat(np.arange(4), 25)), 8)


def handle_with_trace(ch):
    from dblink_b200 import analysis_gpu as ag

    p = ag.Pairs(ch.num_records)
    for mem, off, _ in ch.samples:
        p.add_sample(ag.sample_clusters(ch.num_records, mem, off))
    p.trace_begin(len(ch.samples))
    return p


def test_the_trace_holds_numpy_bits_and_device_labels_and_outputs_work():
    import torch

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag

    L = _lib.load()
    ch = random_chain(3000, 70, seed=21)
    R, S = ch.num_records, len(ch.samples)
    first, second, count = aa.pairwise_match_counts(ch)
    x = aa.pairwise_match_trace(ch, (first << 32) | second)
    assert np.array_equal(x.sum(1), count)
    with handle_with_trace(ch) as p:
        # every sample from device labels; odd positions twice (repeating a position changes nothing)
        for s, (mem, off, _) in enumerate(ch.samples):
            dev = torch.tensor(ag.sample_clusters(R, mem, off), device="cuda")
            torch.cuda.synchronize()
            for _ in range(1 + s % 2):
                assert L.dbl_pairs_trace_sample(p._h, dev.data_ptr(), s) == _lib.OK
        # one chain over every even number of positions: each row's popcount is its held count
        m = p.mixing(1, [0], S, aa.ess_floor(1, S))
        assert np.array_equal(m.count, count)
        # windows of 4 positions from every start: the trace's bits are numpy's
        for s in range(S - 3):
            m = p.mixing(1, [s], 4, aa.ess_floor(1, 4))
            assert np.array_equal(m.count, x[:, s:s + 4].sum(1)), s
        # device outputs equal host outputs
        want = p.mixing(1, [0, 17, 35], 33, aa.ess_floor(3, 33))
        n = len(first)
        i32 = [torch.zeros(n, dtype=torch.int32, device="cuda") for _ in range(4)]
        f64 = [torch.zeros(n, dtype=torch.float64, device="cuda") for _ in range(2)]
        starts = np.array([0, 17, 35], np.int32)
        torch.cuda.synchronize()
        assert L.dbl_pairs_mixing(p._h, 1, 3, starts.ctypes.data_as(_lib.i32p), 33, aa.ess_floor(3, 33),
                                  *(a.data_ptr() for a in i32 + f64)) == _lib.OK
        for a, w in zip(i32, (want.count, want.chain_min, want.chain_max, want.max_t)):
            assert np.array_equal(a.cpu().numpy(), w)
        for a, w in zip(f64, (want.rhat, want.ess)):
            assert np.array_equal(a.cpu().numpy().view(np.int64), w.view(np.int64))
        wm = aa.mixing_from_trace(x, [0, 17, 35], 33, aa.ess_floor(3, 33))
        assert np.array_equal(want.ess.view(np.int64), wm.ess.view(np.int64))


def test_refusals_leave_the_handle_usable():
    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag
    from dblink_b200.engine import DblinkError

    def status(fn, *a):
        with pytest.raises(DblinkError) as e:
            fn(*a)
        return e.value.status

    ch = random_chain(400, 24, seed=4)
    R, S = ch.num_records, len(ch.samples)
    first, second, _ = aa.pairwise_match_counts(ch)
    x = aa.pairwise_match_trace(ch, (first << 32) | second)
    floor = aa.ess_floor(2, 12)
    p = ag.Pairs(R)
    try:
        lab = ag.sample_clusters(R, *ch.samples[0][:2])
        assert status(p.trace_begin, S) == _lib.ERR_STATE                # no sample yet
        for mem, off, _ in ch.samples:
            p.add_sample(ag.sample_clusters(R, mem, off))
        assert status(p.trace_sample, lab, 0) == _lib.ERR_STATE          # no trace yet
        assert status(p.mixing, 1, [0, 12], 12, floor) == _lib.ERR_STATE
        assert status(p.trace_begin, 0) == _lib.ERR_INVALID
        assert status(p.trace_begin, (1 << 31) - 1) == _lib.ERR_INVALID  # 2^26 words per pair, past 2^31 words
        p.trace_begin(S)
        for s, (mem, off, _) in enumerate(ch.samples):
            p.trace_sample(ag.sample_clusters(R, mem, off), s)
        assert status(p.trace_sample, lab, S) == _lib.ERR_INVALID
        assert status(p.trace_sample, lab, -1) == _lib.ERR_INVALID
        bad = lab.copy()
        bad[3] = R
        assert status(p.trace_sample, bad, 0) == _lib.ERR_INVALID
        assert status(p.mixing, 1, [0, 13], 12, floor) == _lib.ERR_INVALID  # 13 + 12 > 24 positions
        assert status(p.mixing, 1, [-1], 12, floor) == _lib.ERR_INVALID
        assert status(p.mixing, 1, [0], 3, floor) == _lib.ERR_INVALID        # N = 1
        assert status(p.mixing, 1, [], 12, floor) == _lib.ERR_INVALID        # no chain
        want = aa.mixing_from_trace(x, [0, 12], 12, floor)
        got = p.mixing(1, [0, 12], 12, floor)
        for name in ("count", "chain_min", "chain_max", "max_t"):
            assert np.array_equal(getattr(got, name), getattr(want, name))
        for name in ("rhat", "ess"):
            assert np.array_equal(getattr(got, name).view(np.int64), getattr(want, name).view(np.int64))
        # a new sample drops the trace
        p.add_sample(lab)
        assert status(p.mixing, 1, [0, 12], 12, floor) == _lib.ERR_STATE
        assert p.num_samples == S + 1 and len(p.read()[0]) == len(first)
    finally:
        p.close()
    # the size bound: M N^2 >= 2^30 refused by the ABI (4 halves of 16384 positions) and by both paths
    big = ag.Pairs(4)
    try:
        big.add_sample(np.zeros(4, np.int32))
        big.trace_begin(2 * 16384)
        assert big.mixing(1, [0], 2 * 16383, 0.5).count[0] == 0
        assert status(big.mixing, 1, [0, 0], 2 * 16384, 0.5) == _lib.ERR_INVALID
    finally:
        big.close()


def test_both_paths_raise_the_same_value_errors(monkeypatch):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    short = pooled(random_chain(300, 10, seed=5), 2, 3, 2)
    for fn in (aa.pairwise_match_diagnostics, ag.pairwise_match_diagnostics):
        with pytest.raises(ValueError, match="^pairwise-match-diagnostics needs at least 4 draws per chain"):
            fn(short)
    ch = pooled(random_chain(300, 12, seed=6), 2, 6, 0)
    H = len(aa.pairwise_match_counts(ch)[0])
    monkeypatch.setattr(aa, "MAX_TRACE_WORDS", H - 1)
    for fn in (aa.pairwise_match_diagnostics, ag.pairwise_match_diagnostics):
        with pytest.raises(ValueError, match=f"^the match trace needs {H} words, more than {H - 1}$"):
            fn(ch)
    monkeypatch.setattr(aa, "MIXING_SIZE_BOUND", 4 * 3 * 3)  # M N^2 = 36 with 2 chains of 6
    for fn in (aa.pairwise_match_diagnostics, ag.pairwise_match_diagnostics):
        with pytest.raises(ValueError, match=r"^pairwise-match-diagnostics needs M N\^2 < 2\^30: 4 half-chains of 3"):
            fn(ch)


def test_new_kernels_do_not_spill():
    from dblink_b200 import _lib

    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--dump-resource-usage", _lib.SO_PATH], capture_output=True, text=True).stdout
    lines = out.splitlines()
    for name in ("k_mark_pairs", "k_pair_mixing"):
        at = [i for i, line in enumerate(lines) if name in line and "Function" in line]
        assert len(at) == 1, name
        assert " LOCAL:0 " in lines[at[0] + 1] and " STACK:0 " in lines[at[0] + 1], lines[at[0] + 1]


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """summarize on RLdata500 sampled on the GPU: the device diagnostics write the same bytes as the numpy path."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 0, "[]", sample_size=100, thinning=10,
                      sampler="PCG-I", cutoff=100)
        return c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]',
                         'quantities : ["pairwise-match-probabilities", "pairwise-match-diagnostics"], '
                         'minMatchProbability : 0.1')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.pairwise_match_diagnostics
    monkeypatch.setattr(ag, "pairwise_match_diagnostics", lambda ch, **kw: calls.append(1) or real(ch, **kw))
    Project(config.parse_string(conf(gpu_dir)), base_dir="").execute(log=lambda *a: None)
    assert len(calls) == 1
    names = ("pairwise-match-probabilities.csv", "pairwise-match-diagnostics.csv",
             "pairwise-match-diagnostics-summary.csv")
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert len(gpu[names[1]].splitlines()) == len(gpu[names[0]].splitlines()) > 10

    os.makedirs(host_dir)
    shutil.copytree(os.path.join(gpu_dir, "linkage-chain.parquet"), os.path.join(host_dir, "linkage-chain.parquet"))
    monkeypatch.setattr(project, "pairwise_match_counts", aa.pairwise_match_counts)
    monkeypatch.setattr(project, "pairwise_match_diagnostics", aa.pairwise_match_diagnostics)
    p = Project(config.parse_string(conf(host_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] == "summarize"]
    p.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
