"""The entity-value counts on the GPU (dbl_values_* in dbl_posterior.cu, analysis_gpu.EntityValues) against numpy's
analysis_arrays.EntityValueCounts: modes and counts exactly equal on random labellings of up to 50 000 records and 64
samples over several attributes, on a 12 000-record cluster of many values, on all-singleton centers, on values at
V - 1, for host and device inputs and on a 1 M-record chain; every refusal returns its documented status and leaves
the handle usable.  A sample step with saveEntityValues on writes the linkage chain it writes with the option off,
and each cluster's recorded values are the entity values of that iteration, replayed from the seeded engine: on one
chain, on two chains and on a sharded engine.  The project's entity-values files are the same bytes on the GPU path
and the numpy path."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from test_host_pipeline import GOLDEN, make_conf

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def assert_equal_to_numpy(labels, samples, V, device=False):
    """samples = per sample int32[R] values of one attribute."""
    import torch

    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    C = int(labels.max()) + 1
    want = aa.EntityValueCounts(labels, C, V)
    lab = torch.from_numpy(np.ascontiguousarray(labels, np.int32)).cuda() if device else labels
    if device:
        h = ag.EntityValues.__new__(ag.EntityValues)  # the owner, with the labels passed as a device pointer
        from dblink_b200 import _lib
        import ctypes as C_

        h._lib, h._h, h.num_records, h.num_clusters = _lib.load(), C_.c_void_p(), len(labels), C
        h._call("create", C_.byref(h._h), len(labels), lab.data_ptr(), C, V)
    else:
        h = ag.EntityValues(labels, C, V)
    with h:
        for x in samples:
            want.add_sample(x)
            if device:
                d = torch.from_numpy(np.ascontiguousarray(x, np.int32)).cuda()
                h._call("add_sample", h._h, d.data_ptr())
            else:
                h.add_sample(x)
        assert h.num_samples == len(samples)
        got_mode, got_count = h.modes()
    mode, count = want.modes()
    assert got_mode.dtype == np.int32 and got_count.dtype == np.int64
    assert np.array_equal(got_mode, mode) and np.array_equal(got_count, count)
    return mode, count


@pytest.mark.parametrize("R,S,V,seed", [(1, 1, 1, 0), (7, 3, 2, 1), (300, 12, 5, 2), (5000, 40, 50, 3),
                                        (50000, 64, 1000, 4), (50000, 8, 70000, 5)])
def test_modes_equal_numpy(R, S, V, seed):
    rng = np.random.default_rng(seed)
    labels = np.unique(rng.integers(0, max(R // 3, 1), R), return_inverse=True)[1]
    for a in range(3):  # several attributes: one handle each
        samples = [rng.integers(0, V, R).astype(np.int32) for _ in range(S)]
        samples[0][: max(R // 10, 1)] = V - 1  # values at V - 1
        assert_equal_to_numpy(labels, samples, V)


def test_one_big_cluster_of_many_values_and_device_inputs():
    rng = np.random.default_rng(6)
    R, V = 20000, 9000
    labels = rng.integers(1, 4000, R)
    labels[rng.permutation(R)[:12000]] = 0  # one cluster of 12 000 records
    labels = np.unique(labels, return_inverse=True)[1]
    samples = [rng.integers(0, V, R).astype(np.int32) for _ in range(16)]
    for device in (False, True):
        mode, count = assert_equal_to_numpy(labels, samples, V, device)
    assert count[0] < 12000 * 16  # many values in the big cluster: its mode holds a fraction of its records
    # all singletons, and one cluster of every record
    assert_equal_to_numpy(np.arange(R), samples[:4], V)
    assert_equal_to_numpy(np.zeros(R, np.int64), samples[:4], V)


def test_a_million_records():
    rng = np.random.default_rng(7)
    R, V = 1_000_000, 30000
    labels = np.unique(rng.integers(0, 700_000, R), return_inverse=True)[1]
    ent = rng.integers(0, V, R)  # values that mostly agree across samples, as entity values do
    samples = []
    for _ in range(6):
        x = ent.copy()
        move = rng.random(R) < 0.2
        x[move] = rng.integers(0, V, int(move.sum()))
        samples.append(x.astype(np.int32))
    assert_equal_to_numpy(labels, samples, V)


def test_refusals_leave_the_handle_usable():
    import ctypes as C
    import torch

    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import EntityValues

    L = _lib.load()
    h = C.c_void_p()
    good = np.array([0, 1, 1, 2], np.int32)
    for R, lab, nc, nv in ((0, good, 3, 2), (4, good, 0, 2), (4, good, 3, 0), (1 << 31, good, 3, 2),
                           (4, np.array([0, 1, 3, 2], np.int32), 3, 2), (4, np.array([0, -1, 1, 2], np.int32), 3, 2)):
        assert L.dbl_values_create(C.byref(h), R, lab.ctypes.data, nc, nv) == _lib.ERR_INVALID and not h.value
    assert L.dbl_values_create(C.byref(h), 4, None, 3, 2) == _lib.ERR_INVALID
    with EntityValues(good, 3, 2) as v:
        mode, count = np.zeros(3, np.int32), np.zeros(3, np.int64)
        assert L.dbl_values_modes(v._h, mode.ctypes.data, count.ctypes.data) == _lib.ERR_STATE
        assert L.dbl_values_modes(v._h, None, count.ctypes.data) == _lib.ERR_INVALID
        assert L.dbl_values_add_sample(v._h, None) == _lib.ERR_INVALID
        for bad in ([0, 0, 2, 0], [0, -1, 0, 0]):
            assert L.dbl_values_add_sample(v._h, np.array(bad, np.int32).ctypes.data) == _lib.ERR_INVALID
            dev = torch.tensor(bad, dtype=torch.int32, device="cuda")
            assert L.dbl_values_add_sample(v._h, dev.data_ptr()) == _lib.ERR_INVALID
        assert v.num_samples == 0
        v.add_sample([1, 0, 1, 1])
        v.add_sample([1, 1, 0, 1])
        assert L.dbl_values_add_sample(v._h, np.array([2, 0, 0, 0], np.int32).ctypes.data) == _lib.ERR_INVALID
        assert v.num_samples == 2
        m, c = v.modes()
        assert m.tolist() == [1, 0, 1] and c.tolist() == [2, 2, 2]  # cluster 1: 0 and 1 twice each, the smaller wins


# ---- the sample step ----------------------------------------------------------------------------------------------
def sample_conf(out, chains=1, save=True, sample_size=4):
    c = make_conf(os.path.join(GOLDEN, "RLdata500.csv.gz"), out, 1, '["fname_c1"]', sample_size=sample_size,
                  thinning=5, sampler="PCG-II", cutoff=0)
    if save:
        c = c.replace("resume : false,", "resume : false, saveEntityValues : true,")
    if chains > 1:
        c = c.replace("randomSeed : 319158", f"randomSeed : 319158\n    numChains : {chains}")
    c = c.replace('quantities : ["cluster-size-distribution", "partition-sizes"]', 'quantities : ["entity-values"]')
    return c.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["pairwise"]')


def replay(p, iterations):
    """{iteration: [(link, y) per chain]} of the seeded engine swept to each iteration."""
    eng = p.generate_initial_state()
    out = {}
    for it in iterations:
        if it > eng.iteration:
            eng.sweep("PCG-II", it - eng.iteration)
        if p.num_chains == 1:
            d = eng.download_state()
            out[it] = [(d["link"], d["y"])]
        else:
            out[it] = [(d["link"], d["y"]) for d in eng.download_chains()]
    eng.close()
    return out


@pytest.mark.parametrize("chains", [1, 2])
def test_the_sample_step_records_the_entity_values(tmp_path, chains):
    from dblink_b200 import analysis_arrays as aa, config
    from dblink_b200.project import Project

    on, off = str(tmp_path / "on") + "/", str(tmp_path / "off") + "/"
    p = Project(config.parse_string(sample_conf(on, chains)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] == "sample"]
    p.execute(log=lambda *a: None)
    q = Project(config.parse_string(sample_conf(off, chains, save=False)), base_dir="")
    q.steps = lambda: [s for s in Project.steps(q) if s[0] == "sample"]
    q.execute(log=lambda *a: None)
    names = [a.name for a in p.matching_attributes]
    rec = p.load()["rec_ids"]
    for k, (d_on, d_off) in enumerate(zip(p.chain_dirs(), q.chain_dirs())):
        a = aa.read_chain_arrays(os.path.join(d_on, "linkage-chain.parquet"))
        b = aa.read_chain_arrays(os.path.join(d_off, "linkage-chain.parquet"))
        assert a.iterations.tolist() == b.iterations.tolist() == [0, 5, 10, 15, 20]
        assert a.record_ids.equals(b.record_ids)
        assert all(np.array_equal(x[i], y[i]) for x, y in zip(a.samples, b.samples) for i in range(3))
        assert open(os.path.join(d_on, "diagnostics.csv")).read().count("\n") == 6
        assert not os.path.exists(os.path.join(d_off, "entity-values-chain.parquet"))
        pos = {r: i for i, r in enumerate(a.record_ids.to_pylist())}
        order = np.array([pos[str(r)] for r in rec])
        truth = replay(p, [int(i) for i in a.iterations])
        for it, got in zip(a.iterations, aa.read_entity_values([d_on], a, names, p.attribute_values())):
            link, y = truth[int(it)][k]
            want = np.empty_like(got)
            want[:, order] = y[link].T
            assert np.array_equal(got, want), (k, it)


def test_the_sharded_sample_step_records_the_entity_values():
    """Sampler.sample over ShardedGibbs with entity values: a collective download of y, block and link on every rank,
    files on rank 0 (tests/entity_values_worker.py)."""
    import torch

    nproc = max(1, min(torch.cuda.device_count(), 2))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-port=29763", os.path.join(ROOT, "tests", "entity_values_worker.py")]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")]))
    res = subprocess.run(cmd, capture_output=True, text=True, env=env, timeout=900)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "sharded entity values ok" in res.stdout


def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch):
    """sample then summarize on RLdata500: the GPU path writes the same bytes as the numpy path from the same chain."""
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project
    from dblink_b200.project import Project

    def conf(out):
        c = sample_conf(out, sample_size=20)
        return c.replace('quantities : ["entity-values"]',
                         'quantities : ["entity-values"], entityValuesCenter : "binder-clusters"')

    gpu_dir, host_dir = str(tmp_path / "gpu") + "/", str(tmp_path / "host") + "/"
    calls = []
    real = ag.entity_value_modes
    monkeypatch.setattr(ag, "entity_value_modes", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    p = Project(config.parse_string(conf(gpu_dir)), base_dir="")
    p.steps = lambda: [s for s in Project.steps(p) if s[0] != "evaluate"]
    p.execute(log=lambda *a: None)
    assert len(calls) == 1
    names = ["entity-values.csv", "entity-values-clusters.csv"]
    gpu = {f: open(os.path.join(gpu_dir, f), "rb").read() for f in names}
    assert gpu["entity-values.csv"].startswith(b"cluster,size,by,byProbability,bm,bmProbability,bd,bdProbability,"
                                               b"fname_c1,fname_c1Probability,lname_c1,lname_c1Probability\n")
    assert gpu["entity-values.csv"].count(b"\n") == gpu["entity-values-clusters.csv"].count(b"\n") + 1

    os.makedirs(host_dir)
    for f in ("linkage-chain.parquet", "entity-values-chain.parquet"):
        shutil.copytree(os.path.join(gpu_dir, f), os.path.join(host_dir, f))
    for name in ("entity_value_modes", "binder_counts"):
        monkeypatch.setattr(project, name, getattr(aa, name))
    q = Project(config.parse_string(conf(host_dir)), base_dir="")
    q.steps = lambda: [s for s in Project.steps(q) if s[0] == "summarize"]
    q.execute(log=lambda *a: None)
    for f in names:
        assert open(os.path.join(host_dir, f), "rb").read() == gpu[f], f
