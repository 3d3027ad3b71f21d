"""Time of the variation-of-information cell histograms on a 1 M-record chain: the GPU path (dbl_vi_cross through
analysis_gpu.VI) against the numpy path (analysis_arrays.vi_cross_histograms).  Host clock around calls that end in a
synchronise.  Adding the samples (host labels + upload) is timed apart from dbl_vi_cross.  numpy is timed on the first
--numpy-samples samples only, (n choose 2) pairs, and scaled to the S (S - 1) / 2 pairs of the whole chain by the
number of pairs; the GPU's histograms of those samples are checked equal to numpy's.

The chain is the S = 100 one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64
partitions, each sample moving 30 % of the records.  The card's name and power limit are read in the same run.

    python profiles/scripts/vi_time.py [--records 1000000] [--numpy-samples 8]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--numpy-samples", type=int, default=8)
    args = ap.parse_args()
    R, S, Sn = args.records, 100, args.numpy_samples
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    print(f"host: {len(os.sched_getaffinity(0))} cpus visible")

    lk, blk = links(R, S, seed=12345)
    ch = aa.ChainArrays(pa.array(["r%d" % i for i in range(R)]), np.arange(S, dtype=np.int64),
                        [aa.sample_from_links(l, blk) for l in lk])
    width = aa.vi_width(ch)
    big = [int((np.bincount(lab, minlength=R)[lab] >= 2).sum())
           for lab in (aa.sample_labels(R, m, o) for m, o, _ in ch.samples[:5])]
    print(f"R = {R}, S = {S}, width M + 1 = {width}; records in clusters of two or more (first samples): {big}")

    ag.vi_cross_histograms(aa.ChainArrays(np.arange(4), np.zeros(2, np.int64),
                                          [aa.sample_from_links(np.array([0, 0, 1, 2], np.int32), blk)] * 2))  # warm-up
    with ag.VI(R, S) as vi:
        t0 = time.perf_counter()
        for m, o, _ in ch.samples:
            vi.add_sample(ag.sample_clusters(R, m, o))
        t_add = time.perf_counter() - t0
        G, t_cross = timed(vi.cross, width)
    pairs = S * (S - 1) // 2
    print(f"GPU: adding {S} samples {t_add:.2f} s ({t_add / S * 1e3:.1f} ms each); dbl_vi_cross {t_cross:.2f} s for "
          f"{pairs} pairs ({t_cross / pairs * 1e3:.2f} ms a pair)")
    g = aa.vi_cluster_histograms(ch, width)
    losses, t_loss = timed(aa.vi_losses, g, G, R)
    s = aa.vi_estimate(losses)
    print(f"host losses {t_loss * 1e3:.1f} ms; VI sample {s}, expected VI {losses[s]:.4f} (range {losses.min():.4f} "
          f"to {losses.max():.4f})")

    sub = aa.ChainArrays(ch.record_ids, ch.iterations[:Sn], ch.samples[:Sn])
    want, t_np = timed(aa.vi_cross_histograms, sub)
    sub_pairs = Sn * (Sn - 1) // 2
    assert np.array_equal(ag.vi_cross_histograms(sub), want), "GPU histograms differ from numpy's"
    print(f"numpy on the first {Sn} samples ({sub_pairs} pairs): {t_np:.2f} s ({t_np / sub_pairs * 1e3:.1f} ms a pair), "
          f"scaled to {pairs} pairs: {t_np / sub_pairs * pairs:.0f} s (not run); GPU histograms equal numpy's")


if __name__ == "__main__":
    main()
