"""CPU-only checks of the host side of the GPU sMPC (analysis_gpu.py): sample validation, argument checks of the C
ABI that come before any device work, the failure without a device, and the platform choice in project.py."""
import numpy as np
import pytest


def test_sample_clusters_rejects_samples_that_miss_or_repeat_records():
    from dblink_b200 import analysis_gpu as ag

    c = ag.sample_clusters(5, np.array([1, 4, 0, 2, 3]), np.array([0, 2, 3, 5]))
    assert c.dtype == np.int32 and list(c) == [1, 0, 2, 2, 0]
    for mem, off in (([1, 4, 0, 2], [0, 2, 4]),             # a record missing
                     ([1, 4, 0, 2, 2], [0, 2, 3, 5]),       # a record twice
                     ([1, 4, 0, 2, 5], [0, 2, 3, 5]),       # an index out of range
                     ([1, 4, 0, 2, 3, 3], [0, 2, 3, 6])):   # too many
        with pytest.raises(ValueError):
            ag.sample_clusters(5, np.array(mem), np.array(off))


def test_posterior_create_checks_sizes():
    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Posterior
    from dblink_b200.engine import DblinkError

    for R, S in ((0, 1), (-3, 1), (1 << 31, 1), (4, 0), (4, (1 << 26) + 1)):
        with pytest.raises(DblinkError) as e:
            Posterior(R, S)
        assert e.value.status == _lib.ERR_INVALID


def test_posterior_needs_a_device():
    import torch

    from dblink_b200 import _lib
    from dblink_b200.analysis_gpu import Posterior
    from dblink_b200.engine import DblinkError

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(DblinkError) as e:
        Posterior(10, 2)
    assert e.value.status == _lib.ERR_CUDA


def test_project_uses_the_host_smpc_without_a_device(monkeypatch):
    import torch

    from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, project

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")

    def no_gpu(chain):
        raise AssertionError("the GPU sMPC was called on a host without a device")

    monkeypatch.setattr(ag, "shared_most_probable_clusters", no_gpu)
    link = np.array([3, 0, 3, 2, 0, 4], np.int32)
    ch = aa.ChainArrays(np.arange(6), np.zeros(1, np.int64), [aa.sample_from_links(link, np.zeros(5, np.int32))])
    assert list(project.shared_most_probable_clusters(ch)) == [0, 1, 0, 3, 1, 5]
