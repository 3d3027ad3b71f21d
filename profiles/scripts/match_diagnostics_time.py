"""Time of the per-pair MCMC diagnostics (split-R̂, ESS) of the 1M-record chain of smpc_time.py (R = 1 M, 64
partitions, S = 100 samples that keep most clusters for three samples, so the pairs' draws are autocorrelated), read
as K = 1 chain of 100 and as K = 4 chains of 25: pass 1 (every sample into dbl_pairs), the trace pass per sample
(dbl_pairs_trace_sample), and dbl_pairs_mixing over the pairs seen in at least two samples, three calls after a
warm-up; numpy's mixing_from_trace on the first pairs, scaled by the number of pairs (marked as scaled), with the
device checked equal on those pairs.  Host clock around work that ends in a synchronise; the card's name and power
limit are read in the same run.

    python profiles/scripts/match_diagnostics_time.py [--records 1000000] [--numpy-pairs 200000]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag  # noqa: E402
from smpc_time import card, links  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--numpy-pairs", type=int, default=200_000)
    a = ap.parse_args()
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    R, S, min_count = a.records, 100, 2
    lk, blk = links(R, S, seed=12345)
    samples = [aa.sample_from_links(l, blk) for l in lk]
    labels = [ag.sample_clusters(R, mem, off) for mem, off, _ in samples]
    with ag.Pairs(R) as p:
        t = time.perf_counter()
        for lab in labels:
            p.add_sample(lab)
        t_add = time.perf_counter() - t
        H = p.count()
        first, second, count = p.read(min_count)
        print(f"R = {R}, S = {S}: {H} distinct pairs, {len(first)} seen in >= {min_count} samples; pass 1 "
              f"{t_add:.2f} s ({t_add / S * 1e3:.1f} ms per sample)")
        p.trace_begin(S)
        t = time.perf_counter()
        for s, lab in enumerate(labels):
            p.trace_sample(lab, s)
        t_trace = time.perf_counter() - t
        print(f"trace pass: {t_trace:.2f} s ({t_trace / S * 1e3:.1f} ms per sample, host labels), trace "
              f"{-(-S // 32) * H * 4 / 1e6:.0f} MB")
        x = None
        for K in (1, 4):
            n = S // K
            starts = np.arange(K, dtype=np.int32) * n
            floor = aa.ess_floor(K, n)
            p.mixing(min_count, starts, n, floor)  # warm-up
            times = []
            for _ in range(3):
                t = time.perf_counter()
                mix = p.mixing(min_count, starts, n, floor)
                times.append(time.perf_counter() - t)
            print(f"K = {K} x {n} draws: dbl_pairs_mixing {min(times) * 1e3:.1f} / {np.median(times) * 1e3:.1f} / "
                  f"{max(times) * 1e3:.1f} ms (min / median / max of 3); max_t: median {np.median(mix.max_t):.0f}, "
                  f"max {mix.max_t.max()}; R̂ > 1.01: {int((mix.rhat > 1.01).sum())}, undefined: "
                  f"{int(np.isnan(mix.rhat).sum())}; median ESS {np.nanmedian(mix.ess):.1f}")
            m = min(a.numpy_pairs, len(first))
            if x is None:
                x = aa.pairwise_match_trace(aa.ChainArrays(np.arange(R), np.arange(S), samples),
                                            (first[:m] << 32) | second[:m])
            t = time.perf_counter()
            want = aa.mixing_from_trace(x, starts, n, floor)
            t_np = time.perf_counter() - t
            for name in ("count", "chain_min", "chain_max", "max_t"):
                assert np.array_equal(getattr(mix, name)[:m], getattr(want, name)), name
            for name in ("rhat", "ess"):
                assert np.array_equal(getattr(mix, name)[:m].view(np.int64), getattr(want, name).view(np.int64))
            print(f"K = {K}: numpy mixing_from_trace {t_np:.2f} s on {m} pairs, scaled to all {len(first)}: "
                  f"{t_np * len(first) / m:.1f} s (scaled); the device equals numpy on those pairs")


if __name__ == "__main__":
    main()
