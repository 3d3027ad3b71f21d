"""Time of the credible ball's cells on a 1 M-record chain: dbl_vi_score_samples (through analysis_gpu.VI) of the VI
sample and of the sMPC against every sample, next to dbl_vi_score of the same labellings, after a warm-up call of each;
numpy's vi_sample_cells on the first --numpy-samples samples, scaled to the whole chain by the number of samples (one
cell pass per sample), the GPU's rows checked equal on those.  Host clock around calls that end in a synchronise; the
samples are added once, before the timed calls; --repeats calls of each are timed.

The chain is the S = 100 one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64
partitions, each sample moving 30 % of the records.  The card's name and power limit are read in the same run.

    python profiles/scripts/credible_ball_time.py [--records 1000000] [--numpy-samples 5] [--repeats 3]
"""
import argparse
import os
import sys

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
    ap.add_argument("--numpy-samples", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
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
    g = aa.vi_cluster_histograms(ch, width)
    smpc = ag.shared_most_probable_clusters(ch)
    keys = sum(int(np.diff(off)[np.diff(off) >= 2].sum()) for _, off, _ in ch.samples)
    print(f"R = {R}, S = {S}, width {width}; records in clusters of two or more, summed over the samples: {keys}")

    with ag.vi_samples(ch) as vi:
        s = aa.vi_estimate(aa.vi_losses(g, vi.cross(width), R))
        mem, off, _ = ch.samples[s]
        centers = (("VI sample", aa.sample_labels(R, mem, off)), ("sMPC", smpc))
        vi.score_samples(smpc, width)  # warm-up
        vi.score(smpc, width)
        for name, lab in centers:
            t_rows, t_sum = [], []
            for _ in range(args.repeats):
                G, t = timed(vi.score_samples, lab, width)
                t_rows.append(t)
                G_sum, t = timed(vi.score, lab, width)
                t_sum.append(t)
            assert np.array_equal(G.sum(axis=0), G_sum), "rows do not sum to dbl_vi_score"
            d = aa.credible_ball_distances(np.bincount(np.bincount(lab)), g, G, R)
            print(f"GPU, center {name}: dbl_vi_score_samples {min(t_rows) * 1e3:.1f} ms (all {args.repeats}: "
                  f"{', '.join(f'{x * 1e3:.1f}' for x in t_rows)}); dbl_vi_score {min(t_sum) * 1e3:.1f} ms (all: "
                  f"{', '.join(f'{x * 1e3:.1f}' for x in t_sum)}); VI distances {d[0].min():.4f} .. {d[0].max():.4f} "
                  f"bits, Binder {d[1].min()} .. {d[1].max()} pairs")
    sub = aa.ChainArrays(ch.record_ids, ch.iterations[:Sn], ch.samples[:Sn])
    want, t_np = timed(aa.vi_sample_cells, sub, smpc, width)
    assert np.array_equal(G[:Sn], want), "GPU rows differ from numpy's"
    print(f"numpy vi_sample_cells of the sMPC on the first {Sn} samples: {t_np:.2f} s (GPU rows equal); scaled to "
          f"{S} samples: {t_np * S / Sn:.1f} s (not run)")


if __name__ == "__main__":
    main()
