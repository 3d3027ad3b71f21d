"""Time per sample of the counts behind the posterior-pairwise / posterior-cluster metrics on the 1 M-record chain of
smpc_time.py (R = 1 M, 64 partitions, S = 100), against a ground truth that is the chain's first sample:

  * numpy: analysis_arrays.posterior_metric_counts;
  * dbl_eval_add_sample alone, with each sample's labels already made: from host memory (the upload included) and
    from device memory;
  * sample_clusters (members / offsets -> labels on the host) + dbl_eval_add_sample, as analysis_gpu does.

Host clock around calls that end in a synchronise (dbl_eval_add_sample waits for its stream).  The card's name and
power limit are read in the same run.  The GPU counts are checked against numpy's.

    python profiles/scripts/eval_time.py [--records 1000000]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import smpc_time  # noqa: E402  (also puts the repository on sys.path)

from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag  # noqa: E402


def add_all(R, truth, labels, S):
    ev = ag.Evaluation(R, truth, S)
    try:
        t = time.perf_counter()
        for lab in labels:
            ev.add_sample(lab)
        dt = time.perf_counter() - t
        return ev.read(), dt
    finally:
        ev.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    args = ap.parse_args()
    R, S = args.records, 100
    L = _lib.load()
    if L.dbl_device_count() == 0:
        sys.exit("no CUDA device")
    import torch

    print("card:", smpc_time.card())
    lk, blk = smpc_time.links(R, S, seed=12345)
    ch = aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), [aa.sample_from_links(l, blk) for l in lk])
    truth = lk[0]

    want, t_np = smpc_time.timed(aa.posterior_metric_counts, ch, truth)
    print(f"numpy posterior_metric_counts: {t_np / S * 1e3:.1f} ms per sample (S = {S}, R = {R})")

    labels = [ag.sample_clusters(R, mem, off) for mem, off, _ in ch.samples]
    _, dense = np.unique(truth, return_inverse=True)
    add_all(R, dense, labels[:2], 2)  # warm-up: module load, sort kernels
    for name, lab in (("host", labels), ("device", [torch.from_numpy(x).cuda() for x in labels])):
        torch.cuda.synchronize()
        got, dt = _add_device(R, dense, lab, S) if name == "device" else add_all(R, dense, lab, S)
        assert all(np.array_equal(g, w) for g, w in zip(got, want)), "GPU counts differ from numpy's"
        print(f"dbl_eval_add_sample alone, labels in {name} memory: {dt / S * 1e3:.2f} ms per sample")

    ev = ag.Evaluation(R, dense, S)
    try:
        t = time.perf_counter()
        for mem, off, _ in ch.samples:
            ev.add_sample(ag.sample_clusters(R, mem, off))
        dt = time.perf_counter() - t
        assert all(np.array_equal(g, w) for g, w in zip(ev.read(), want))
    finally:
        ev.close()
    print(f"sample_clusters + dbl_eval_add_sample: {dt / S * 1e3:.2f} ms per sample (counts equal numpy's)")


def _add_device(R, truth, dev_labels, S):
    """dbl_eval_add_sample on device labels, through the C ABI (the owner class takes host arrays)."""
    L = _lib.load()
    ev = ag.Evaluation(R, truth, S)
    try:
        t = time.perf_counter()
        for x in dev_labels:
            assert L.dbl_eval_add_sample(ev._h, x.data_ptr()) == _lib.OK
        dt = time.perf_counter() - t
        return ev.read(), dt
    finally:
        ev.close()


if __name__ == "__main__":
    main()
