"""Time of the posterior pairwise match counts of a 1 M-record chain: the numpy path (analysis_arrays, S = 100 only)
and the GPU path (analysis_gpu), host clock around work that ends in a synchronise.  The GPU time is split into
adding the samples (host labels + upload + the per-sample pair generation, sort and merge) and reading the result.

The chain is the one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64 partitions,
each sample moving 30 % of the records; the S = 1 000 chain draws its samples (seeded) from the S = 100 ones.

    python profiles/scripts/match_prob_time.py [--records 1000000]
"""
import argparse
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


def gpu_split(chain):
    """The GPU pairs in their two halves: samples in, then the read."""
    R = chain.num_records
    pairs = ag.Pairs(R)
    try:
        t = time.perf_counter()
        for mem, off, _ in chain.samples:
            pairs.add_sample(ag.sample_clusters(R, mem, off))
        t_add = time.perf_counter() - t
        res, t_read = timed(pairs.read)
    finally:
        pairs.close()
    return res, t_add, t_read


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    args = ap.parse_args()
    R = args.records
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    print(f"host: {len(os.sched_getaffinity(0))} cpus visible")

    lk, blk = links(R, 100, seed=12345)
    ch100 = aa.ChainArrays(pa.array(["r%d" % i for i in range(R)]), np.arange(100, dtype=np.int64),
                           [aa.sample_from_links(l, blk) for l in lk])
    pool = np.random.default_rng(777).integers(0, 100, 1000)
    ch1000 = aa.ChainArrays(ch100.record_ids, np.arange(1000, dtype=np.int64), [ch100.samples[i] for i in pool])
    per_sample = [int(aa._comb2(np.diff(off)).sum()) for _, off, _ in ch100.samples]
    print(f"pairs per sample: mean {np.mean(per_sample):.0f}, min {min(per_sample)}, max {max(per_sample)} "
          f"(R = {R}, 64 partitions)")

    ag.pairwise_match_counts(aa.ChainArrays(np.arange(4), np.zeros(1, np.int64),
                                            [aa.sample_from_links(np.zeros(4, np.int32), blk)]))  # warm-up
    _, t_labels = timed(lambda: [ag.sample_clusters(R, m, o) for m, o, _ in ch100.samples])
    print(f"host labels alone (sample_clusters): {t_labels / 100 * 1e3:.1f} ms per sample")
    host, t_host = timed(aa.pairwise_match_counts, ch100)
    print(f"S = 100: numpy {t_host:.2f} s, {len(host[0])} distinct pairs")
    for S, ch in ((100, ch100), (1000, ch1000)):
        dev, t_add, t_read = gpu_split(ch)
        if S == 100:
            assert all(np.array_equal(a, b) for a, b in zip(dev, host)), "GPU pairs differ from numpy's"
        print(f"S = {S}: GPU {t_add + t_read:.2f} s = {t_add:.2f} s adding samples ({t_add / S * 1e3:.1f} ms each) "
              f"+ {t_read:.3f} s reading; {len(dev[0])} distinct pairs" + (" (equal to numpy's)" if S == 100 else ""))


if __name__ == "__main__":
    main()
