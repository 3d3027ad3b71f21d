"""Time of the Binder-loss counts (n, K) of a 1 M-record chain: the numpy path (analysis_arrays.binder_counts) and
the GPU path (analysis_gpu.binder_counts), host clock around work that ends in a synchronise.  Both run pass 1 (every
sample into the pair-count table) and pass 2 (every sample scored against it); the numpy pass 2 is its
binder_counts less its pairwise_match_counts.  The GPU pass 2 is timed three ways: as binder_counts runs it
(sample_clusters on the host + dbl_pairs_score_sample), dbl_pairs_score_sample alone on labels already in host memory,
and on labels already in device memory.

The chain is the S = 100 one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64
partitions, each sample moving 30 % of the records.  The card's name and power limit are read in the same run.

    python profiles/scripts/binder_time.py [--records 1000000]
"""
import argparse
import ctypes as C
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402

from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag  # noqa: E402
from smpc_time import card, links, timed  # noqa: E402


def gpu_passes(chain):
    """(n, K, pass 1 s, pass 2 s, score-only host labels s, score-only device labels s) on one handle."""
    import torch

    R, S = chain.num_records, len(chain.samples)
    L = _lib.load()
    n, K = np.zeros(S, np.int64), np.zeros(S, np.int64)
    with ag.Pairs(R) as pairs:
        t = time.perf_counter()
        for mem, off, _ in chain.samples:
            pairs.add_sample(ag.sample_clusters(R, mem, off))
        t1 = time.perf_counter() - t
        t = time.perf_counter()
        for s, (mem, off, _) in enumerate(chain.samples):
            n[s], K[s] = pairs.score_sample(ag.sample_clusters(R, mem, off))
        t2 = time.perf_counter() - t
        labels = [ag.sample_clusters(R, mem, off) for mem, off, _ in chain.samples]
        a, b = C.c_int64(), C.c_int64()
        t = time.perf_counter()
        for s, lab in enumerate(labels):
            assert L.dbl_pairs_score_sample(pairs._h, lab.ctypes.data, C.byref(a), C.byref(b)) == _lib.OK
            assert (a.value, b.value) == (n[s], K[s])
        t_host = time.perf_counter() - t
        dev = [torch.from_numpy(lab).cuda() for lab in labels]
        torch.cuda.synchronize()
        t = time.perf_counter()
        for s, lab in enumerate(dev):
            assert L.dbl_pairs_score_sample(pairs._h, lab.data_ptr(), C.byref(a), C.byref(b)) == _lib.OK
            assert (a.value, b.value) == (n[s], K[s])
        t_dev = time.perf_counter() - t
    return n, K, t1, t2, t_host, t_dev


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    args = ap.parse_args()
    R, S = args.records, 100
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    print(f"host: {len(os.sched_getaffinity(0))} cpus visible")

    lk, blk = links(R, S, seed=12345)
    ch = aa.ChainArrays(pa.array(["r%d" % i for i in range(R)]), np.arange(S, dtype=np.int64),
                        [aa.sample_from_links(l, blk) for l in lk])
    ag.binder_counts(aa.ChainArrays(np.arange(4), np.zeros(1, np.int64),
                                    [aa.sample_from_links(np.zeros(4, np.int32), blk)]))  # warm-up

    n, K, t1, t2, t_host, t_dev = gpu_passes(ch)
    print(f"GPU pass 1 (add): {t1:.2f} s, {t1 / S * 1e3:.1f} ms per sample")
    print(f"GPU pass 2 (sample_clusters + score): {t2:.2f} s, {t2 / S * 1e3:.1f} ms per sample")
    print(f"GPU dbl_pairs_score_sample alone: {t_host / S * 1e3:.2f} ms per sample with host labels, "
          f"{t_dev / S * 1e3:.2f} ms with device labels")
    print(f"pairs per sample: mean {n.mean():.0f}; sum of counts C = {int(n.sum())}")

    (hn, hK), t_np = timed(aa.binder_counts, ch)
    assert np.array_equal(hn, n) and np.array_equal(hK, K), "GPU counts differ from numpy's"
    _, t_np1 = timed(aa.pairwise_match_counts, ch)
    print(f"numpy binder_counts: {t_np:.2f} s = pass 1 {t_np1:.2f} s + pass 2 {t_np - t_np1:.2f} s "
          f"({(t_np - t_np1) / S * 1e3:.1f} ms per sample); (n, K) equal to the GPU's")
    for t in (0.5, 0.7):
        s = aa.binder_estimate(n, K, t)
        print(f"t = {t}: estimate = sample {s}, expected loss {aa.binder_losses(n, K, t)[s]!r}")


if __name__ == "__main__":
    main()
