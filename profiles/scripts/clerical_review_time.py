"""Time of the clerical review of the 1M-record chain of smpc_time.py (R = 1 M, 64 partitions, S = 100 samples),
centered on its sMPC: the two device calls, dbl_pairs_record_links (one pass over the held pair table) and
dbl_posterior_cluster_counts (every record's row of the signature matrix against the center), three calls each after
a warm-up; numpy's record_links on the whole pair table and cluster_appearances on the first samples, scaled by the
number of samples (marked as scaled), the device checked equal; and the host review (ClericalReview: the per-cluster
sums, ties and the exact review order) that both paths share.  Host clock around work that ends in a synchronise; the
card's name and power limit are read in the same run.

    python profiles/scripts/clerical_review_time.py [--records 1000000] [--numpy-samples 10]
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


def best_of_3(fn):
    fn()  # warm-up
    times, out = [], None
    for _ in range(3):
        t = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t)
    return out, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--numpy-samples", type=int, default=10)
    a = ap.parse_args()
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    R, S = a.records, 100
    lk, blk = links(R, S, seed=12345)
    samples = [aa.sample_from_links(l, blk) for l in lk]
    ch = aa.ChainArrays(np.arange(R), np.arange(S, dtype=np.int64), samples)
    labels = aa.canonical_clusters(ag.shared_most_probable_clusters(ch))
    C = int(labels.max()) + 1
    cluster = [ag.sample_clusters(R, mem, off) for mem, off, _ in samples]
    fmt = lambda ts: f"{min(ts) * 1e3:.1f} / {np.median(ts) * 1e3:.1f} / {max(ts) * 1e3:.1f} ms"  # noqa: E731
    with ag.Pairs(R) as p, ag.Posterior(R, S) as post:
        for c in cluster:
            p.add_sample(c)
            post.add_sample(c)
        H = p.count()
        links_d, t_links = best_of_3(lambda: p.record_links(labels, C))
        A_d, t_counts = best_of_3(lambda: post.cluster_counts(labels, C))
    print(f"R = {R}, S = {S}, C = {C} sMPC clusters, {H} held pairs")
    print(f"dbl_pairs_record_links: {fmt(t_links)} (min / median / max of 3, host labels and outputs)")
    print(f"dbl_posterior_cluster_counts: {fmt(t_counts)} (min / median / max of 3, host labels and outputs)")
    first, second, count = aa.pairwise_match_counts(ch)
    t = time.perf_counter()
    links_h = aa.record_links(first, second, count, labels, C)
    t_np_links = time.perf_counter() - t
    for name in ("W", "I", "partner", "partner_count", "inner", "least"):
        assert np.array_equal(getattr(links_d, name), getattr(links_h, name)), name
    m = min(a.numpy_samples, S)
    t = time.perf_counter()
    A_h = aa.cluster_appearances(aa.ChainArrays(ch.record_ids, ch.iterations[:m], samples[:m]), labels)
    t_np_counts = time.perf_counter() - t
    with ag.Posterior(R, m) as post:
        for c in cluster[:m]:
            post.add_sample(c)
        assert np.array_equal(post.cluster_counts(labels, C), A_h)
    print(f"numpy record_links: {t_np_links:.2f} s on the whole table; the device equals it")
    print(f"numpy cluster_appearances: {t_np_counts:.2f} s on {m} samples, scaled to {S}: "
          f"{t_np_counts * S / m:.1f} s (scaled); the device equals it on those samples")
    t = time.perf_counter()
    review = aa.ClericalReview(links_d, A_d, labels, S, 0.5)
    t_host = time.perf_counter() - t
    print(f"host review (per-cluster sums, ties, exact order of {C} clusters): {t_host:.2f} s; top cluster "
          f"{int(review.order[0])} of size {int(review.size[review.order[0]])}")


if __name__ == "__main__":
    main()
