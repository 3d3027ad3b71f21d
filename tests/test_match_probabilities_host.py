"""Posterior pairwise match probabilities on the host: analysis_arrays.pairwise_match_counts against the set-based
analysis.pairwise_match_probabilities, the CSV writer, the summarize parameters, the C ABI's checks that come before
any device work and the platform choice in project.py."""
import ctypes as C
import os

import numpy as np
import pytest


def random_chain(R, S, seed, big=0):
    """ChainArrays of S samples over R records that share most clusters (the pattern of
    test_gpu_posterior.random_chain); with big > 0 the first sample also has one cluster of `big` records."""
    from dblink_b200 import analysis_arrays as aa

    rng = np.random.default_rng(seed)
    E = max(1, (3 * R) // 4)
    blk = rng.integers(0, 4, E).astype(np.int32)
    base = rng.integers(0, E, R).astype(np.int32)
    samples = []
    for s in range(S):
        link = base.copy()
        move = rng.random(R) < 0.3
        link[move] = rng.integers(0, E, int(move.sum()))
        if s % 3 == 0:
            base = link
        if s == 0 and big:
            link = link.copy()
            link[rng.permutation(R)[:big]] = 0
        samples.append(aa.sample_from_links(link, blk))
    return aa.ChainArrays(np.array(["r%d" % i for i in range(R)]), np.arange(S, dtype=np.int64) * 10, samples)


def as_set_chain(ch):
    """The same chain in analysis.py's form: [(iteration, {partition: [cluster of ids]})]."""
    ids = [str(x) for x in np.asarray(ch.record_ids.to_pylist() if hasattr(ch.record_ids, "to_pylist")
                                      else ch.record_ids)]
    out = []
    for it, (mem, off, part) in zip(ch.iterations, ch.samples):
        parts = {}
        for c in range(len(off) - 1):
            parts.setdefault(int(part[c]), []).append([ids[i] for i in mem[off[c]:off[c + 1]]])
        out.append((int(it), parts))
    return out, ids


def assert_equal_to_sets(ch):
    from dblink_b200 import analysis, analysis_arrays as aa

    first, second, count = aa.pairwise_match_counts(ch)
    assert first.dtype == second.dtype == count.dtype == np.int64
    assert (first < second).all()
    key = first * ch.num_records + second
    assert (np.diff(key) > 0).all()  # ascending (first, second), no pair twice
    chain, ids = as_set_chain(ch)
    S = len(ch.samples)
    got = {frozenset((ids[a], ids[b])): c / S for a, b, c in zip(first, second, count)}
    assert got == analysis.pairwise_match_probabilities(chain)
    return first, second, count


@pytest.mark.parametrize("R,S", [(1, 1), (2, 3), (6, 7), (40, 20), (300, 9)])
def test_array_counts_equal_the_set_based_ones(R, S):
    first, _, count = assert_equal_to_sets(random_chain(R, S, seed=R * 31 + S))
    if R >= 40:
        assert len(first) > 0 and (count < S).any() and (count > 1).any()


def test_counts_through_the_parquet_chain(tmp_path):
    from dblink_b200 import analysis_arrays as aa, writers as w

    R = 200
    rng = np.random.default_rng(9)
    ids = ["id%03d" % i for i in rng.permutation(R)]
    blk = rng.integers(0, 5, R).astype(np.int32)
    path = os.path.join(tmp_path, "linkage-chain.parquet")
    lw = w.LinkageChainWriter(path, write_buffer_size=3)
    for it in range(8):
        lw.append(it, w.linkage_structure_arrow(rng.integers(0, R // 3, R).astype(np.int32), blk, ids))
    lw.close()
    ch = aa.read_chain_arrays(path, lower_iteration_cutoff=2)
    assert len(ch.samples) == 6
    assert_equal_to_sets(ch)


def test_total_count_equals_pairs_per_sample():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(500, 12, seed=3, big=40)
    _, _, count = aa.pairwise_match_counts(ch)
    want = sum(k * (k - 1) // 2 * n for d in aa.cluster_size_distribution(ch).values() for k, n in d.items())
    assert int(count.sum()) == want and want > 780


def test_cap_and_min_count():
    from dblink_b200 import analysis_arrays as aa

    ch = random_chain(300, 9, seed=4)
    first, second, count = aa.pairwise_match_counts(ch)
    n = len(first)
    assert np.array_equal(np.column_stack(aa.pairwise_match_counts(ch, max_pairs=n)),
                          np.column_stack((first, second, count)))
    with pytest.raises(ValueError, match=f"more than {n - 1} distinct record pairs"):
        aa.pairwise_match_counts(ch, max_pairs=n - 1)
    # a single sample over the cap is refused before its pairs are generated
    big = random_chain(3000, 1, seed=5, big=2000)
    with pytest.raises(ValueError, match="more than 1000 distinct"):
        aa.pairwise_match_counts(big, max_pairs=1000)
    f3, s3, c3 = aa.pairwise_match_counts(ch, min_count=3)
    keep = count >= 3
    assert np.array_equal(f3, first[keep]) and np.array_equal(s3, second[keep]) and np.array_equal(c3, count[keep])


def test_min_match_count_is_exact():
    from dblink_b200.analysis_arrays import min_match_count

    for S in (1, 3, 7, 10, 100, 1000):
        for t in [0.0, 1.0, 0.1, 0.3, 1 / 3, 2 / 3, 0.7] + [c / S for c in range(S + 1)]:
            c = min_match_count(t, S)
            assert c / S >= t and (c == 1 or (c - 1) / S < t), (S, t, c)
    assert min_match_count(0.5, 0) == 1


def read_rows(path):
    with open(os.path.join(path, "pairwise-match-probabilities.csv")) as fh:
        lines = fh.read().split("\n")
    assert lines[0] == "recordId1,recordId2,probability" and lines[-1] == ""
    return [tuple(l.split(",")) for l in lines[1:-1]]


def test_writer_order_orientation_threshold_and_text(tmp_path):
    from dblink_b200 import writers as w

    ids = ["b", "a", "c", "ab", "Z"]  # index order differs from code-point order: Z < a < ab < b < c
    first = np.array([0, 0, 1, 2, 3, 1])
    second = np.array([1, 4, 2, 3, 4, 3])
    count = np.array([2, 3, 1, 2, 3, 2])
    w.save_pairwise_match_probabilities(first, second, count, 3, ids, 0.0, str(tmp_path))
    rows = read_rows(tmp_path)
    assert rows == [("Z", "ab", "1.0"), ("Z", "b", "1.0"), ("a", "ab", "0.6666666666666666"),
                    ("a", "b", "0.6666666666666666"), ("ab", "c", "0.6666666666666666"),
                    ("a", "c", "0.3333333333333333")]
    assert float(rows[2][2]) == 2 / 3
    for a, b, _ in rows:
        assert a < b
    # a probability exactly equal to the threshold is kept
    w.save_pairwise_match_probabilities(first, second, count, 3, ids, 2 / 3, str(tmp_path))
    assert [r[2] for r in read_rows(tmp_path)] == ["1.0", "1.0"] + ["0.6666666666666666"] * 3
    w.save_pairwise_match_probabilities(first, second, count, 3, ids, 1.0, str(tmp_path))
    assert len(read_rows(tmp_path)) == 2
    # a chain with no sample after the cutoff: the header only
    z = np.zeros(0, np.int64)
    w.save_pairwise_match_probabilities(z, z, z, 0, ids, 0.0, str(tmp_path))
    assert open(os.path.join(tmp_path, "pairwise-match-probabilities.csv")).read() == "recordId1,recordId2,probability\n"


def test_writer_accepts_arrow_ids(tmp_path):
    import pyarrow as pa

    from dblink_b200 import writers as w

    ids = pa.array(["r10", "r9", "é", "r1"])
    w.save_pairwise_match_probabilities(np.array([0, 1]), np.array([1, 2]), np.array([1, 1]), 4, ids, 0.25,
                                        str(tmp_path))
    assert read_rows(tmp_path) == [("r10", "r9", "0.25"), ("r9", "é", "0.25")]


CONF = """
dblink : {
  data : { path : "x.csv", recordIdentifier : "rec_id", nullValue : "NA", matchingAttributes : [] }
  outputPath : "out/"
  randomSeed : 1
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [
    {name : "summarize", parameters : { lowerIterationCutoff : 10, %s }}
  ]
}
"""


def test_summarize_parses_the_new_quantity_and_threshold():
    from dblink_b200 import config
    from dblink_b200.project import Project

    def steps(prm):
        return Project(config.parse_string(CONF % prm), base_dir="").steps()

    (name, prm), = steps('quantities : ["pairwise-match-probabilities", "partition-sizes"], minMatchProbability : 0.25')
    assert name == "summarize" and prm["quantities"] == ["pairwise-match-probabilities", "partition-sizes"]
    assert prm["min_match_probability"] == 0.25 and prm["lower_iteration_cutoff"] == 10
    assert steps('quantities : ["pairwise-match-probabilities"]')[0][1]["min_match_probability"] == 0.0
    assert steps('quantities : ["partition-sizes"], minMatchProbability : 1')[0][1]["min_match_probability"] == 1.0
    for bad in ("-0.1", "1.5", "2"):
        with pytest.raises(ValueError, match="minMatchProbability"):
            steps('quantities : ["pairwise-match-probabilities"], minMatchProbability : %s' % bad)
    with pytest.raises(ValueError, match="quantities"):
        steps('quantities : ["pairwise-match-probability"]')


def test_pairs_create_checks_sizes():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Pairs
    from dblink_b200.engine import DblinkError

    for R, P in ((0, 1), (-3, 1), (1 << 31, 1), (4, 0), (4, -1), (4, 1 << 31)):
        with pytest.raises(DblinkError) as e:
            Pairs(R, P)
        assert e.value.status == _lib.ERR_INVALID
    L = _lib.load()
    assert L.dbl_pairs_create(None, 4, 4) == _lib.ERR_INVALID
    assert L.dbl_pairs_add_sample(None, None) == _lib.ERR_INVALID
    assert L.dbl_pairs_count(None, 1, None) == _lib.ERR_INVALID
    assert L.dbl_pairs_num_samples(None) == 0
    L.dbl_pairs_free(None)


def test_pairs_need_a_device():
    import torch

    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Pairs
    from dblink_b200.engine import DblinkError

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(DblinkError) as e:
        Pairs(10, 100)
    assert e.value.status == _lib.ERR_CUDA
    h = C.c_void_p()
    assert _lib.load().dbl_pairs_create(C.byref(h), 10, 100) == _lib.ERR_CUDA and not h


def test_project_uses_the_host_pairs_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(chain, **kw):
        raise AssertionError("the GPU pairs were called on a host without a device")

    monkeypatch.setattr(ag, "pairwise_match_counts", no_gpu)
    link = np.array([3, 0, 3, 2, 0, 3], np.int32)
    ch = aa.ChainArrays(np.arange(6), np.zeros(1, np.int64), [aa.sample_from_links(link, np.zeros(5, np.int32))])
    first, second, count = project.pairwise_match_counts(ch)
    assert list(first) == [0, 0, 1, 2] and list(second) == [2, 5, 4, 5] and list(count) == [1, 1, 1, 1]
