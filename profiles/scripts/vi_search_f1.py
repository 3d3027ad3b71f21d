"""RLdata10000 (tests/golden): the VI search against the VI sample, the sMPC and the Binder search (falseLinkCost 0.5),
on the chains of vi_f1.py (Levenshtein 7/10 and Jaro-Winkler 8.5/10 on fname_c1 / lname_c1, PCG-II, seed 319158).
Each chain is sampled once; the estimates are computed with the functions the summarize and evaluate steps use and
scored against the ground truth (pairwise precision / recall / F1, the adjusted Rand index, the number of clusters) and
by their exact posterior expected VI (dbl_vi_score).  The card's name and power limit are read in the same run.

    python profiles/scripts/vi_search_f1.py [--burnin 1000] [--samples 100] [--thinning 10]
"""
import argparse
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from dblink_b200 import analysis_arrays as aa, analysis_gpu as ag, config, project  # noqa: E402
from dblink_b200.project import Project  # noqa: E402
from similarity_f1 import CONF, card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burnin", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--thinning", type=int, default=10)
    a = ap.parse_args()
    data = os.path.join(ROOT, "tests", "golden", "RLdata10000.csv.gz")
    print("card:", card())
    print(f"RLdata10000, PCG-II, burn-in {a.burnin}, {a.samples} samples every {a.thinning} sweeps, seed 319158")
    for name, thr in (("LevenshteinSimilarityFn", "7.0"), ("JaroWinklerSimilarityFn", "8.5")):
        with tempfile.TemporaryDirectory() as out:
            conf = CONF % (name, thr, data, out + "/", a.samples, a.burnin, a.thinning)
            proj = Project(config.parse_string(conf), base_dir="")
            proj.steps = lambda p=proj: [s for s in Project.steps(p) if s[0] == "sample"]
            proj.execute(log=lambda *_: None)
            ch = proj.read_chain(0)
            truth = proj.true_labels()(ch.record_ids)
            t = time.perf_counter()
            start, run, rows, exact = project.vi_search_estimate(ch, 1000)
            dt = time.perf_counter() - t
            s, vi_labels, _, _ = project.vi_estimate(ch)
            _, brun, _ = project.binder_search_estimate(ch, 0.5, 1000)
            R, S = ch.num_records, len(ch.samples)
            width = aa.vi_width(ch)
            g_sum = aa.vi_cluster_histograms(ch, width).sum(axis=0)
            with ag.vi_samples(ch) as vi:
                e_binder = aa.vi_label_loss(np.bincount(np.bincount(brun.labels)), vi.score(brun.labels, width), g_sum,
                                            S, R)
            by = {n: [r for r in rows if r[0] == n] for n in aa.VI_SEARCH_STARTS}
            for n in aa.VI_SEARCH_STARTS:
                print(f"{name}({thr}, 10) search from {n}: {by[n][-1][1]} rounds, moves {[r[2] for r in by[n][1:]]}, "
                      f"E_q {by[n][0][4]:.6f} -> {by[n][-1][4]:.6f}")
            for label, lab, e in (("sMPC", project.shared_most_probable_clusters(ch), exact[1]),
                                  (f"VI sample (iteration {ch.iterations[s]})", vi_labels, exact[0]),
                                  ("Binder search t = 0.5", brun.labels, e_binder),
                                  (f"VI search (from {start}, {run.rounds} rounds, converged {run.converged})",
                                   run.labels, exact[2 + aa.VI_SEARCH_STARTS.index(start)])):
                pw = aa.pairwise_metrics(lab, truth)
                print(f"{name}({thr}, 10) {label}: expected VI {e:.6f}, precision {pw['precision']:.4f} recall "
                      f"{pw['recall']:.4f} F1 {pw['f1score']:.4f} ARI {aa.adjusted_rand_index(lab, truth):.4f} "
                      f"clusters {len(np.unique(lab))}")
            print(f"  true clusters {len(np.unique(truth))}; expected VI of both search results {exact[2]:.6f} / "
                  f"{exact[3]:.6f}; the VI search estimate: {dt:.2f} s")


if __name__ == "__main__":
    main()
