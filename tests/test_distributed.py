"""N>1 path: the host exchange logic under gloo (CPU, world_size 2) and, on a multi-GPU box, the sharded chain
against the oracle."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKER = os.path.join(ROOT, "tests", "mp_worker.py")


def run_workers(mode, nproc, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), WORKER, mode]
    env = dict(os.environ, OMP_NUM_THREADS="1")
    return subprocess.run(cmd, capture_output=True, text=True, timeout=600, env=env)


def test_exchange_logic_gloo_world2():
    res = run_workers("cpu", 2, 29731)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "cpu exchange ok" in res.stdout


def test_lpt_assign():
    import numpy as np

    from dblink_b200.distributed import lpt_assign

    costs = np.array([10.0, 9, 8, 7, 6, 5, 4, 3, 2, 1])
    owner = lpt_assign(costs, 3)
    loads = np.bincount(owner, weights=costs, minlength=3)
    assert loads.max() <= 1.1 * costs.sum() / 3
    assert (lpt_assign(costs, 1) == 0).all()
    assert lpt_assign([], 4).shape == (0,)


def test_merge_link_mass():
    """each record's total comes from the one rank that scored it; a record scored by no rank or by two is refused"""
    import numpy as np

    from dblink_b200.distributed import LINK_MASS_UNSCORED, merge_link_mass

    want = np.array([0.5, 3.0, 1e-300, 0.0, np.inf, 7.25])
    owner = np.array([0, 2, 1, 1, 0, 2])
    unscored = np.full(len(want), LINK_MASS_UNSCORED).view(np.float64)
    parts = [np.where(owner == r, want, unscored) for r in range(3)]
    got = merge_link_mass(parts)
    assert (got.view(np.uint64) == want.view(np.uint64)).all()
    # a NaN a kernel stores is a total, not the marker of a record another rank scored
    parts[0][0] = np.nan
    assert np.isnan(merge_link_mass(parts)[0])
    lost = [p.copy() for p in parts]
    lost[1][2] = unscored[0]
    with pytest.raises(RuntimeError, match="1 records"):
        merge_link_mass(lost)
    twice = [p.copy() for p in parts]
    twice[0][3] = 2.0
    with pytest.raises(RuntimeError, match="record 3: 2 ranks"):
        merge_link_mass(twice)


@pytest.mark.gpu
def test_sharded_chain_matches_oracle():
    import torch

    n = torch.cuda.device_count()
    if n < 2:
        # one rank still exercises begin/pack/unpack/end + the summary all-reduce (NCCL on a single device)
        res = run_workers("gpu", 1, 29741)
    else:
        res = run_workers("gpu", min(n, 4), 29741)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "sharded chain == oracle chain" in res.stdout


@pytest.mark.gpu
def test_chain_driver_on_a_sharded_engine():
    """Sampler.sample over ShardedGibbs (links() / num_entities on the sharded engine, outputs on rank 0 only)"""
    import torch

    res = run_workers("sample", max(1, min(torch.cuda.device_count(), 2)), 29751)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]
    assert "sharded sample ok" in res.stdout
