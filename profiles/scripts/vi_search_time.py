"""Time of the VI search on a 1 M-record chain: the GPU path (dbl_vi_search through analysis_gpu.VI) from the VI sample
and from the sMPC, against one numpy round (analysis_arrays.vi_search_rounds, max_rounds = 1) on the first
--numpy-samples samples, scaled to the whole chain by the number of samples (a round is one pass over every sample);
the GPU's first round on those samples is checked equal to numpy's.  Host clock around calls that end in a
synchronise; the samples are added once, before the timed calls.

The chain is the S = 100 one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64
partitions, each sample moving 30 % of the records.  The card's name and power limit are read in the same run.

    python profiles/scripts/vi_search_time.py [--records 1000000] [--numpy-samples 10] [--max-rounds 1000]
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
    ap.add_argument("--numpy-samples", type=int, default=10)
    ap.add_argument("--max-rounds", type=int, default=1000)
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
    table = aa.vi_search_table(R)
    smpc = ag.shared_most_probable_clusters(ch)
    g = aa.vi_cluster_histograms(ch, width)
    A = aa.vi_sample_sum(ch, table)
    print(f"R = {R}, S = {S}; squares per sample (first 3): {aa.vi_sample_squares(ch)[:3].tolist()}")

    tiny = aa.ChainArrays(np.arange(4), np.zeros(2, np.int64),
                          [aa.sample_from_links(np.array([0, 0, 1, 2], np.int32), blk)] * 2)
    ag.vi_search(tiny, [np.arange(4)])  # warm-up
    with ag.vi_samples(ch) as vi:
        s = aa.vi_estimate(aa.vi_losses(g, vi.cross(width), R))
        mem, off, _ = ch.samples[s]
        starts = [aa.sample_labels(R, mem, off), smpc]
        for name, st in zip(aa.VI_SEARCH_STARTS, starts):
            run, t = timed(vi.search, table, st, args.max_rounds)
            e = aa.vi_search_losses(run.objectives(), A, S, R)
            print(f"GPU from {name}: {run.rounds} rounds, converged {run.converged}, {t:.2f} s "
                  f"({t / max(run.rounds + 1, 1) * 1e3:.1f} ms a round incl. the last, proposal-free one); "
                  f"E_q {e[0]:.6f} -> {e[-1]:.6f}; moves per round {run.moves.tolist()}")
    sub = aa.ChainArrays(ch.record_ids, ch.iterations[:Sn], ch.samples[:Sn])
    rows = [aa.sample_labels(R, m, o) for m, o, _ in sub.samples]
    want, t_np = timed(aa.vi_search_rounds, R, rows, table, smpc, 1)
    with ag.vi_samples(sub) as vi:
        got, t_gpu = timed(vi.search, table, smpc, 1)
    assert np.array_equal(got.labels, want.labels) and got.moves.tolist() == want.moves.tolist() \
        and got.dJ.tolist() == want.dJ.tolist() and got.J0 == want.J0, "GPU round differs from numpy's"
    print(f"numpy, one round from the sMPC on the first {Sn} samples: {t_np:.2f} s (GPU {t_gpu:.3f} s, equal); "
          f"scaled to {S} samples: {t_np * S / Sn:.0f} s a round (not run)")


if __name__ == "__main__":
    main()
