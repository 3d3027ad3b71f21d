"""Capture histories on the GPU (dbl_capture_* in dbl_posterior.cu, analysis_gpu.Capture / capture_histories) against
the numpy path in analysis_arrays.py: H and L exactly, from 1 record to 1 M, with 1, 2, 7 and 12 files, a 12 000-record
cluster, all singletons, labels and files in host and in device memory, pooled chains; bit-identical reruns; every
refusal leaves the handle as it was; 0 spills; the project's files equal the host path's."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from test_capture_histories_host import NEW_FILES, project, synthetic_data, write_chains
from test_gpu_posterior import random_chain

pytestmark = pytest.mark.gpu


def assert_equal_to_numpy(ch, file, F):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag

    H, L = ag.capture_histories(ch, file, F)
    want_H, want_L = aa.capture_histories(ch, file, F)
    assert H.dtype == L.dtype == np.int64
    assert np.array_equal(H, want_H) and np.array_equal(L, want_L)
    return H, L


@pytest.mark.parametrize("R,S,F", [(1, 1, 1), (2, 3, 2), (40, 1, 7), (700, 17, 12), (5000, 20, 2), (50_000, 8, 7),
                                   (1_000_000, 3, 12), (1_000_000, 2, 1)])
def test_random_chains_equal_numpy(R, S, F):
    ch = random_chain(R, S, seed=R + S + F)
    file = np.random.default_rng(R).integers(0, F, R)
    H, L = assert_equal_to_numpy(ch, file, F)
    assert H.sum() == sum(len(off) - 1 for _, off, _ in ch.samples)
    if R >= 700:
        assert (L > 0).any() and (H[:, (1 << F) - 1] >= 0).all()


def test_a_giant_cluster_and_all_singletons():
    from dblink_b200 import analysis_arrays as aa

    R = 30_000
    rng = np.random.default_rng(2)
    link = rng.integers(0, R, R).astype(np.int32)
    link[rng.permutation(R)[:12_000]] = 0  # one cluster of 12 000 records
    blk = np.zeros(R, np.int32)
    ch = aa.ChainArrays(np.arange(R), np.arange(3, dtype=np.int64),
                        [aa.sample_from_links(link, blk), aa.sample_from_links(np.arange(R, dtype=np.int32), blk),
                         aa.sample_from_links(np.zeros(R, np.int32), blk)])
    for F in (1, 2, 7, 12):
        file = rng.integers(0, F, R)
        H, L = assert_equal_to_numpy(ch, file, F)
        assert H[1].sum() == R  # all singletons: one cluster per record
        assert H[2].sum() == 1
        assert (L[:, :] <= 2).all()


def test_device_labels_and_files_and_reruns():
    import torch

    from dblink_b200 import analysis_arrays as aa
    from dblink_b200.analysis_gpu import Capture

    R, F = 20_000, 7
    ch = random_chain(R, 6, seed=9)
    file = np.random.default_rng(9).integers(0, F, R)
    want_H, want_L = aa.capture_histories(ch, file, F)
    labels = []
    for mem, off, _ in ch.samples:
        lab = np.empty(R, np.int32)
        lab[mem] = np.repeat(np.arange(len(off) - 1, dtype=np.int32), np.diff(off))
        labels.append(lab)
    dfile = torch.as_tensor(file.astype(np.int32), device="cuda")
    dlab = [torch.as_tensor(x, device="cuda") for x in labels]
    torch.cuda.synchronize()
    runs = []
    for device_file in (False, True):
        with Capture(dfile.data_ptr() if device_file else file, F, len(labels), num_records=R) as cap:
            for x, d in zip(labels, dlab):
                cap.add_sample(d.data_ptr() if device_file else x)
            H, L = cap.read()
            dL = torch.empty((R, F), dtype=torch.int32, device="cuda")
            cap._call("read", cap._h, H.ctypes.data, dL.data_ptr())
            torch.cuda.synchronize()
            assert np.array_equal(dL.cpu().numpy().astype(np.int64), want_L)
            H2, none = cap.read(record_links=False)
            assert none is None and np.array_equal(H2, H)
        assert np.array_equal(H, want_H) and np.array_equal(L, want_L)
        runs.append((H.tobytes(), L.tobytes()))
    assert runs[0] == runs[1]


def test_pooled_chains(tmp_path):
    from dblink_b200 import analysis_arrays as aa, writers as w

    R, F = 3000, 3
    ids = [f"r{i}" for i in range(R)]
    rng = np.random.default_rng(4)
    paths = []
    for k in range(2):
        path = str(tmp_path / f"c{k}" / "linkage-chain.parquet")
        lw = w.LinkageChainWriter(path, 3)
        for s in range(5):
            link = rng.integers(0, R // 2, R).astype(np.int32)
            lw.append(10 * s, w.linkage_structure_arrow(link, np.zeros(R // 2, np.int32), ids))
        lw.close()
        paths.append(path)
    ch = aa.read_pooled_chain_arrays(paths)
    assert len(ch.samples) == 10
    assert_equal_to_numpy(ch, rng.integers(0, F, R), F)


def test_refusals_leave_the_handle_unchanged():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Capture

    lib = _lib.load()
    R, F = 100, 3
    file = np.random.default_rng(0).integers(0, F, R).astype(np.int32)
    h = C.c_void_p()
    for args in [(R, None, F, 4), (0, file.ctypes.data, F, 4), (-1, file.ctypes.data, F, 4),
                 (R, file.ctypes.data, 0, 4), (R, file.ctypes.data, 13, 4), (R, file.ctypes.data, F, 0),
                 (R, (file + 1).ctypes.data, F, 4), (R, (file - 1).ctypes.data, F, 4)]:
        assert lib.dbl_capture_create(C.byref(h), *args) == _lib.ERR_INVALID
        assert not h.value
    assert lib.dbl_capture_create(None, R, file.ctypes.data, F, 4) == _lib.ERR_INVALID
    assert lib.dbl_capture_add_sample(None, file.ctypes.data) == _lib.ERR_INVALID
    assert lib.dbl_capture_num_samples(None) == 0
    assert lib.dbl_capture_read(None, file.ctypes.data, None) == _lib.ERR_INVALID
    lib.dbl_capture_free(None)

    with Capture(file, F, 2) as cap:
        H = np.zeros((1, 1 << F), np.int64)
        assert lib.dbl_capture_read(cap._h, H.ctypes.data, None) == _lib.ERR_STATE
        lab = np.random.default_rng(1).integers(0, R // 3, R).astype(np.int32)
        cap.add_sample(lab)
        before = cap.read()
        for bad in (np.full(R, R, np.int32), np.full(R, -1, np.int32)):
            assert lib.dbl_capture_add_sample(cap._h, bad.ctypes.data) == _lib.ERR_INVALID
        assert lib.dbl_capture_add_sample(cap._h, None) == _lib.ERR_INVALID
        assert lib.dbl_capture_read(cap._h, None, None) == _lib.ERR_INVALID
        assert cap.num_samples == 1
        after = cap.read()
        assert all(np.array_equal(a, b) for a, b in zip(before, after))
        cap.add_sample(lab)
        assert lib.dbl_capture_add_sample(cap._h, lab.ctypes.data) == _lib.ERR_INVALID  # max_samples = 2
        H, L = cap.read()
        assert cap.num_samples == 2 and np.array_equal(H[1], before[0][0]) and np.array_equal(L, 2 * before[1])


def test_new_kernels_do_not_spill():
    from dblink_b200 import _lib

    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    out = subprocess.run([tool, "--dump-resource-usage", _lib.SO_PATH], capture_output=True, text=True).stdout
    lines = out.splitlines()
    for name in ("k_capture_or", "k_capture_count"):
        at = [i for i, line in enumerate(lines) if name in line and "Function" in line]
        assert len(at) == 1, name
        assert " LOCAL:0 " in lines[at[0] + 1] and " STACK:0 " in lines[at[0] + 1], lines[at[0] + 1]


@pytest.mark.parametrize("chains", [1, 2])
def test_project_outputs_equal_the_host_ones(tmp_path, monkeypatch, chains):
    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, project as pj

    _, ids, ent, _ = synthetic_data(tmp_path)
    q, m = '"shared-most-probable-clusters", "capture-histories"', '"pairwise", "capture-histories"'
    gpu, host = tmp_path / "gpu", tmp_path / "host"
    p = project(tmp_path, gpu, chains, q, m)
    write_chains(p, ids, ent, chains)
    shutil.copytree(gpu, host)
    calls = []
    real = ag.capture_histories
    monkeypatch.setattr(ag, "capture_histories", lambda *a: calls.append(1) or real(*a))
    p.execute(log=lambda *a: None)
    assert len(calls) == 2  # summarize and evaluate
    monkeypatch.setattr(pj, "capture_histories", aa.capture_histories)
    project(tmp_path, host, chains, q, m).execute(log=lambda *a: None)
    assert len(calls) == 2
    for f in sorted(NEW_FILES) + ["evaluation-results.txt"]:
        assert open(os.path.join(host, f), "rb").read() == open(os.path.join(gpu, f), "rb").read(), f
