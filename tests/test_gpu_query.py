"""New records linked to a finished chain on the GPU (dbl_query_*): the device's candidates, probabilities,
new-entity probabilities, effective samples and per-sample log Z against the numpy path, bit-identical reruns, the
refusals, 0 spills, and the project's files on RLdata500."""
import gzip
import os
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from test_query_host import numpy_result, oracle_tables  # noqa: E402


def problem(oracle, seed, R, Q, kinds, S=3, big=0, F=2):
    from dblink_b200 import analysis_arrays as aa, synth

    from helpers import oracle_setup, synth_problem

    C = synth.SynthAttr
    attrs = [C(f"a{i}", k, n) for i, (k, n) in enumerate(kinds)]
    g = synth_problem(seed=seed, R=R + Q, n_files=F, missing=0.05, attrs=attrs)
    m, st, tree, x, file = oracle_setup(oracle, g, seed)
    rng = np.random.default_rng(seed)
    samples = []
    for _ in range(S):
        K = int(rng.integers(max(1, R // 3), R + 1))
        lab = np.r_[np.arange(K), rng.integers(0, K, R - K)]
        if big:
            lab[:big] = 0
            K = len(np.unique(lab))
            lab = np.unique(lab, return_inverse=True)[1]
        rng.shuffle(lab)
        vals = np.stack([x[rng.integers(0, R + Q, K), a].clip(0) for a in range(m.A)], 1).astype(np.int32)
        samples.append((lab.astype(np.int64), vals, rng.uniform(0.02, 0.5, (m.A, F))))
    tab = aa.QueryTables(x[R:], file[R:], [oracle_tables(ix) for ix in m.indexes], [ix.is_const for ix in m.indexes],
                         F)
    return tab, samples


def device_result(tab, samples, R, M, t, device_labels=False):
    from dblink_b200 import analysis_gpu

    if not device_labels:
        return analysis_gpu.link_queries(tab, lambda: iter(samples), R, M, t)
    import torch

    dev = [(torch.as_tensor(l.astype(np.int32), device="cuda"), torch.as_tensor(v, device="cuda"), th)
           for l, v, th in samples]
    with analysis_gpu.Query(tab, R, M, t) as qh:
        for l, v, th in dev:
            qh.add_sample(l.data_ptr(), (v.data_ptr(), v.shape[0]), th)
        for l, v, th in dev:
            qh.score_sample(l.data_ptr(), (v.data_ptr(), v.shape[0]), th)
        torch.cuda.synchronize()
        return qh.read()


def assert_same(dev, ref, t):
    np.testing.assert_allclose(dev.logz, ref.logz, rtol=1e-10)
    np.testing.assert_allclose(dev.new_entity_probability, ref.new_entity_probability, rtol=1e-10)
    np.testing.assert_allclose(dev.effective_samples, ref.effective_samples, rtol=1e-10)
    a = dict(zip(zip(dev.query.tolist(), dev.record.tolist()), dev.probability.tolist()))
    b = dict(zip(zip(ref.query.tolist(), ref.record.tolist()), ref.probability.tolist()))
    for k in set(a) & set(b):
        assert a[k] == pytest.approx(b[k], rel=1e-10)
    far = lambda d: {k for k, v in d.items() if v >= t and abs(v - t) > 1e-9 * max(t, 1e-300)}
    assert far(a) == far(b)


LEV, JW, CON = ("levenshtein", 40), ("jaro-winkler", 30), ("constant", 5)


@pytest.mark.parametrize("R,Q,kinds,big,labels", [
    (1, 1, [CON], 0, False), (50, 7, [CON, ("constant", 3)], 0, False), (300, 40, [LEV, CON, JW], 0, True),
    (2000, 130, [LEV, JW, CON, LEV], 0, False), (13000, 200, [LEV, CON], 12000, True),
    (100000, 1000, [LEV, CON, JW, CON], 0, False)])
def test_device_equals_numpy(oracle, R, Q, kinds, big, labels):
    tab, samples = problem(oracle, R % 97 + Q, R, Q, kinds, S=2 if R > 20000 else 3, big=big)
    M = R + 5
    for t in (0.05, 0.5):
        ref = numpy_result(tab, samples, R, M, t)
        dev = device_result(tab, samples, R, M, t, labels)
        assert_same(dev, ref, t)


def test_bit_identical_reruns_and_refusals(oracle):
    from dblink_b200 import analysis_gpu
    from dblink_b200.engine import DblinkError

    tab, samples = problem(oracle, 3, 400, 60, [LEV, CON, JW])
    R, M = 400, 420
    a, b = (device_result(tab, samples, R, M, 0.05) for _ in range(2))
    for f in ("query", "record", "sums", "zsum", "zsq", "fresh", "logz"):
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    lab, vals, th = samples[0]
    with analysis_gpu.Query(tab, R, M, 0.05) as qh:
        bad = lab.copy()
        bad[0] = len(vals)
        for args in [(bad, vals, th), (lab, vals + tab.num_values[None, :], th), (lab, vals, th + 1.0)]:
            with pytest.raises(DblinkError):
                qh.add_sample(*args)
        with pytest.raises(DblinkError):
            qh.add_sample(lab, np.zeros((M + 1, tab.num_attributes), np.int32), th)
        with pytest.raises(DblinkError):
            qh.score_sample(lab, vals, th)  # before pass 1
        assert qh.num_samples == 0
        qh.add_sample(lab, vals, th)
        with pytest.raises(DblinkError):
            qh.read()
        qh.score_sample(lab, vals, th)
        with pytest.raises(DblinkError):
            qh.score_sample(lab, vals, th)
        qh.read()
    with analysis_gpu.Query(tab, R, M, 0.05) as qh:
        empty = lab.copy()
        empty[empty == len(vals) - 1] = 0  # labels in range, cluster K - 1 without records
        with pytest.raises(DblinkError):
            qh.add_sample(empty, vals, th)
        qh.add_sample(lab, vals, th)
        lab2, vals2, th2 = next(sm for sm in samples + [(lab[:0], vals[:1], th)] if len(sm[1]) != len(vals))
        with pytest.raises(DblinkError):
            qh.score_sample(lab2, vals2, th2)  # pass 2 with another sample's K
        assert qh.num_samples == 1
    with analysis_gpu.Query(tab, R, M, 1e-9, max_candidates=5) as qh:
        with pytest.raises(DblinkError):
            qh.add_sample(lab, vals, th)
        assert qh.num_samples == 0 and qh.num_candidates() == 0
    with pytest.raises(ValueError):
        analysis_gpu.Query(tab, R, M, 0.0)


def test_null_pointers_and_create_refusals(oracle):
    import ctypes as C

    from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu
    from dblink_b200.engine import DblinkError

    tab, samples = problem(oracle, 5, 200, 20, [LEV, CON])
    R, M = 200, 210
    lib = _lib.load()
    assert tab.hit_offsets[-1] > 0
    # create: a file out of range, a value id out of range, an unsorted hit row, a NULL table
    cases = []
    bad = aa.QueryTables.__new__(aa.QueryTables)
    bad.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in tab.__dict__.items()})
    bad.file = bad.file.copy()
    bad.file[0] = tab.num_files
    cases.append(bad)
    bad = aa.QueryTables.__new__(aa.QueryTables)
    bad.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in tab.__dict__.items()})
    bad.x[0, 0] = tab.num_values[0]
    cases.append(bad)
    bad = aa.QueryTables.__new__(aa.QueryTables)
    bad.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in tab.__dict__.items()})
    i = int(np.flatnonzero(np.diff(bad.hit_offsets) >= 2)[0])
    lo = bad.hit_offsets[i]
    bad.hit_values[lo], bad.hit_values[lo + 1] = bad.hit_values[lo + 1], bad.hit_values[lo]
    cases.append(bad)
    for b in cases:
        with pytest.raises(DblinkError) as e:
            analysis_gpu.Query(b, R, M, 0.05)
        assert e.value.status == _lib.ERR_INVALID
    h = C.c_void_p()
    assert lib.dbl_query_create(C.byref(h), R, M, 1, 1, 1, None, None, None, None, None, None, None, None, None, 0.05,
                                10) == _lib.ERR_INVALID
    with analysis_gpu.Query(tab, R, M, 0.05) as qh:
        lab, vals, th = samples[0]
        lab32 = np.ascontiguousarray(lab, np.int32)
        thp = np.ascontiguousarray(th).ctypes.data_as(_lib.f64p)
        assert lib.dbl_query_add_sample(qh._h, None, len(vals), vals.ctypes.data, thp) == _lib.ERR_INVALID
        assert lib.dbl_query_add_sample(qh._h, lab32.ctypes.data, len(vals), None, thp) == _lib.ERR_INVALID
        assert lib.dbl_query_add_sample(qh._h, lab32.ctypes.data, len(vals), vals.ctypes.data, None) == \
            _lib.ERR_INVALID
        assert lib.dbl_query_add_sample(None, lab32.ctypes.data, len(vals), vals.ctypes.data, thp) == _lib.ERR_INVALID
        assert lib.dbl_query_num_candidates(qh._h, None) == _lib.ERR_INVALID
        assert lib.dbl_query_read(qh._h, None, None, None, None, None, None, None, None) == _lib.ERR_INVALID
        assert qh.num_samples == 0


def test_pooled_chains_project_files_equal_numpy(tmp_path, monkeypatch):
    """Two chains and two files on RLdata500: link-records and distortion-probabilities pool the samples of both
    chain directories; the GPU path writes the numpy path's ids and values within 1e-10."""
    from dblink_b200 import analysis_arrays as aa, project

    from test_query_host import NEW_STEPS, project_at, rldata500, sample_project

    rldata500(tmp_path, True)
    p = project_at(tmp_path, "on", NEW_STEPS % (tmp_path / "queries.csv"), 2, True)
    sample_project(p, True)
    p.execute(log=lambda *a: None)
    gpu = {k: (tmp_path / "on" / k).read_text() for k in ("query-links.csv", "query-summary.csv")}
    monkeypatch.setattr(project, "link_queries", aa.link_queries)
    p._link_records([s for n, s in p.steps() if n == "link-records"][0])
    assert len(gpu["query-links.csv"].splitlines()) > 30
    for k, text in gpu.items():
        host = (tmp_path / "on" / k).read_text()
        ga, ha = [l.split(",") for l in text.splitlines()], [l.split(",") for l in host.splitlines()]
        assert len(ga) == len(ha)
        for x, y in zip(ga, ha):
            assert len(x) == len(y)
            for u, v in zip(x, y):
                try:
                    assert float(u) == pytest.approx(float(v), rel=1e-10, abs=1e-300)
                except ValueError:
                    assert u == v


def test_new_kernels_do_not_spill():
    from dblink_b200 import _lib

    so = _lib.SO_PATH
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "--dump-resource-usage", so], capture_output=True,
                         text=True).stdout
    lines = out.splitlines()
    usage = [(l, lines[i + 1]) for i, l in enumerate(lines[:-1]) if "Function" in l and "k_query" in l]
    assert len(usage) >= 10
    for name, res in usage:
        assert "STACK:0" in res and "LOCAL:0" in res, (name, res)


CONF = """dblink : {
  randomSeed : 319158
  expectedMaxClusterSize : 10
  data : {
    path : "%s"
    recordIdentifier : "rec_id"
    nullValue : "NA"
    matchingAttributes : [
      {name : "by", similarityFunction : {name : "ConstantSimilarityFn"}, distortionPrior : {alpha : 1.0, beta : 50.0}},
      {name : "fname_c1", similarityFunction : {name : "LevenshteinSimilarityFn", parameters : {threshold : 7.0, maxSimilarity : 10.0}}, distortionPrior : {alpha : 1.0, beta : 50.0}},
      {name : "lname_c1", similarityFunction : {name : "LevenshteinSimilarityFn", parameters : {threshold : 7.0, maxSimilarity : 10.0}}, distortionPrior : {alpha : 1.0, beta : 50.0}}
    ]
  }
  outputPath : "%s"
  partitioner : {name : "KDTreePartitioner", parameters : {numLevels : 0, matchingAttributes : []}}
  steps : [
    {name : "sample", parameters : {sampleSize : 20, burninInterval : 10, thinningInterval : 2, resume : false, sampler : "PCG-II"%s}}
    {name : "summarize", parameters : {lowerIterationCutoff : 0, quantities : ["cluster-size-distribution"%s]}}
    %s
  ]
}
"""


def run_project(tmp_path, name, on):
    from dblink_b200 import config
    from dblink_b200.project import Project

    data = tmp_path / "data.csv"
    if not data.exists():
        with gzip.open(os.path.join(os.path.dirname(__file__), "golden", "RLdata500.csv.gz"), "rt") as fh:
            text = fh.read()
        data.write_text(text)
        lines = text.splitlines()
        (tmp_path / "queries.csv").write_text("\n".join([lines[0]] + lines[1:51]) + "\n")
    out = tmp_path / name
    extra = (", saveEntityValues : true, saveDistortionProbabilities : true", ', "distortion-probabilities"',
             '{name : "link-records", parameters : {queryPath : "%s", minLinkProbability : 0.05}}'
             % (tmp_path / "queries.csv")) if on else ("", "", "")
    p = Project(config.parse_string(CONF % ((data, str(out) + "/") + extra)), base_dir="")
    p.write_run_txt()
    p.execute(log=lambda *_: None)
    return p, out


def files(root):
    got = {}
    for d, _, fs in os.walk(root):
        for f in fs:
            rel = os.path.relpath(os.path.join(d, f), root)
            if "diagnostics.csv" in rel or rel == "run.txt" or rel.startswith("entity-values-chain") or rel == "state.npz":
                continue
            with open(os.path.join(d, f), "rb") as fh:
                got[rel] = fh.read()
    return got


def test_project_files_on_rldata500(tmp_path, monkeypatch):
    from dblink_b200 import project

    _, off = run_project(tmp_path, "off", False)
    p, on = run_project(tmp_path, "on", True)
    a, b = files(off), files(on)
    for k, v in a.items():
        assert b[k] == v, k
    assert {"distortion-probabilities-chain.csv", "distortion-probabilities.csv", "query-links.csv",
            "query-summary.csv"} <= set(b)
    with open(on / "run.txt") as fh:
        txt = fh.read()
    assert "saveDistortionProbabilities=true" in txt and "LinkRecordsStep" in txt
    # the numpy path writes the same ids and values within 1e-10
    gpu = {k: b[k].decode() for k in ("query-links.csv", "query-summary.csv")}
    monkeypatch.setattr(project, "link_queries", lambda *a: project.analysis_arrays.link_queries(*a))
    prm = [s for n, s in p.steps() if n == "link-records"][0]
    p._link_records(prm)
    for k, text in gpu.items():
        with open(on / k) as fh:
            host = fh.read()
        ga, ha = [l.split(",") for l in text.splitlines()], [l.split(",") for l in host.splitlines()]
        assert len(ga) == len(ha)
        for x, y in zip(ga, ha):
            assert len(x) == len(y)
            for u, v in zip(x, y):
                try:
                    assert float(u) == pytest.approx(float(v), rel=1e-10, abs=1e-300)
                except ValueError:
                    assert u == v
