"""Time of the Binder search (single-record moves) on a 1 M-record chain: the GPU path (dbl_pairs_binder_search through
analysis_gpu.Pairs.binder_search) against the numpy path (analysis_arrays.search_rounds), from the two starts the
project uses (the Binder sample and the sMPC), at falseLinkCost 0.5 and 0.7.  Host clock around calls that end in a
synchronise.  Pass 1 (every sample into the pair-count table) is timed apart; each search call includes its own setup
(start labels, buffers) and the final (n, K) pass.  Rounds and moves per round are printed, and every GPU run is
checked equal to numpy's.  numpy runs from the Binder sample at t = 0.5 only: with 34 M held pairs it takes
seconds a round.

The chain is the S = 100 one of smpc_time.py: synthetic and seeded, R records linked to 3R/4 entities over 64
partitions, each sample moving 30 % of the records.  The card's name and power limit are read in the same run.

    python profiles/scripts/binder_search_time.py [--records 1000000]
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
    args = ap.parse_args()
    R, S = args.records, 100
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    print(f"host: {len(os.sched_getaffinity(0))} cpus visible")

    lk, blk = links(R, S, seed=12345)
    ch = aa.ChainArrays(pa.array(["r%d" % i for i in range(R)]), np.arange(S, dtype=np.int64),
                        [aa.sample_from_links(l, blk) for l in lk])
    n, K = ag.binder_counts(ch)
    s = aa.binder_estimate(n, K, 0.5)
    mem, off, _ = ch.samples[s]
    starts = {"binder-sample": aa.sample_labels(R, mem, off), "smpc": ag.shared_most_probable_clusters(ch)}
    first, second, count = aa.pairwise_match_counts(ch)
    print(f"held pairs H = {len(first)}; Binder sample (t = 0.5) = sample {s}")

    with ag.Pairs(R) as pairs:
        t0 = time.perf_counter()
        for m, o, _ in ch.samples:
            pairs.add_sample(ag.sample_clusters(R, m, o))
        print(f"GPU pass 1 (add): {time.perf_counter() - t0:.2f} s")
        a, b = aa.search_cost(0.5)
        pairs.binder_search(a, b, starts["smpc"], 1)  # warm-up
        for t in (0.5, 0.7):
            a, b = aa.search_cost(t)
            for name, st in starts.items():
                run, dt = timed(pairs.binder_search, a, b, st, 1000)
                print(f"t = {t} (searched at {a / b!r}), from {name}: {run.rounds} rounds, converged {run.converged}, "
                      f"GPU {dt * 1e3:.1f} ms ({dt * 1e3 / max(run.rounds, 1):.1f} ms a round); moves per round "
                      f"{run.moves.tolist()}")
                if t == 0.5 and name == "binder-sample":
                    want, dt_np = timed(aa.search_rounds, R, first, second, count, S, st, a, b, 1000)
                    same = (np.array_equal(want.labels, run.labels) and np.array_equal(want.moves, run.moves)
                            and np.array_equal(want.dn, run.dn) and np.array_equal(want.dK, run.dK)
                            and (want.n, want.K, want.converged) == (run.n, run.K, run.converged))
                    assert same, "the GPU search differs from numpy's"
                    print(f"    numpy {dt_np:.1f} s ({dt_np / max(run.rounds, 1):.2f} s a round); equal to the GPU's")


if __name__ == "__main__":
    main()
