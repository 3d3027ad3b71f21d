"""RLdata10000 (tests/golden): the credible ball around every point estimate the summarize step offers, on the chains
of vi_f1.py (Levenshtein 7/10 and Jaro-Winkler 8.5/10 on fname_c1 / lname_c1, PCG-II, seed 319158) at credibleLevel
0.95, falseLinkCost 0.5.  Each chain is sampled once; per center, with the functions the summarize and evaluate steps
use: both radii and ball sizes, each bound's number of clusters and pairwise precision / recall / F1 against the ground
truth, and whether the truth lies in each ball.  The card's name and power limit are read in the same run.

    python profiles/scripts/credible_ball_f1.py [--burnin 1000] [--samples 100] [--thinning 10] [--level 0.95]
"""
import argparse
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dblink_b200 import analysis_arrays as aa, config, project  # noqa: E402
from dblink_b200.project import Project  # noqa: E402
from similarity_f1 import CONF, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burnin", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--thinning", type=int, default=10)
    ap.add_argument("--level", type=float, default=0.95)
    a = ap.parse_args()
    data = os.path.join(ROOT, "tests", "golden", "RLdata10000.csv.gz")
    print("card:", card())
    print(f"RLdata10000, PCG-II, burn-in {a.burnin}, {a.samples} samples every {a.thinning} sweeps, seed 319158, "
          f"credibleLevel {a.level}, falseLinkCost 0.5")
    for name, thr in (("LevenshteinSimilarityFn", "7.0"), ("JaroWinklerSimilarityFn", "8.5")):
        with tempfile.TemporaryDirectory() as out:
            conf = CONF % (name, thr, data, out + "/", a.samples, a.burnin, a.thinning)
            proj = Project(config.parse_string(conf), base_dir="")
            proj.steps = lambda p=proj: [s for s in Project.steps(p) if s[0] == "sample"]
            proj.execute(log=lambda *_: None)
            ch = proj.read_chain(0)
            truth = proj.true_labels()(ch.record_ids)
            R = ch.num_records
            print(f"{name}({thr}, 10): {len(ch.samples)} samples, true clusters {len(set(truth.tolist()))}")
            for center in project.CREDIBLE_BALL_CENTERS:
                t = time.perf_counter()
                labels, k, balls = project.credible_ball_estimate(ch, center, a.level, 0.5, 1000)
                dt = time.perf_counter() - t
                t_vi, t_binder = project.credible_ball_truth(labels, truth)
                print(f"  center {center} ({len(set(labels.tolist()))} clusters; {dt:.2f} s with the center)")
                for dist, t_d in zip(aa.CREDIBLE_BALL_DISTANCES, (t_vi, t_binder)):
                    d, radius, inside, bounds = balls[dist]
                    print(f"    {dist}: radius {radius:.6g}, {int(inside.sum())} samples in the ball; truth at "
                          f"{t_d:.6g}, {'inside' if t_d <= radius else 'outside'}")
                    for bound in aa.CREDIBLE_BALL_BOUNDS:
                        s, ties = bounds[bound]
                        mem, off, _ = ch.samples[s]
                        pw = aa.pairwise_metrics(aa.sample_labels(R, mem, off), truth)
                        print(f"      {bound}: iteration {ch.iterations[s]}, {k[s]} clusters, distance {d[s]:.6g}, "
                              f"ties {ties}; precision {pw['precision']:.4f} recall {pw['recall']:.4f} "
                              f"F1 {pw['f1score']:.4f}")


if __name__ == "__main__":
    main()
