"""RLdata10000 (tests/golden): the variation-of-information (VI) sample against the sMPC, the Binder sample and the
Binder search at falseLinkCost 0.5, on the chains of binder_f1.py (Levenshtein 7/10 and Jaro-Winkler 8.5/10 on
fname_c1 / lname_c1, PCG-II, seed 319158).  Each chain is sampled once; the estimates are computed from it with the
functions the summarize and evaluate steps use, and scored against the ground truth: pairwise precision / recall / F1,
the adjusted Rand index and the number of clusters.  The card's name and power limit are read in the same run.

    python profiles/scripts/vi_f1.py [--burnin 1000] [--samples 100] [--thinning 10]
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

from dblink_b200 import analysis_arrays as aa, config, project  # noqa: E402
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
            s, vi_labels, _, losses = project.vi_estimate(ch)
            dt = time.perf_counter() - t
            b, binder, _, _ = project.binder_estimate(ch, 0.5)
            start, run, _ = project.binder_search_estimate(ch, 0.5, 1000)
            for label, lab in (("sMPC", project.shared_most_probable_clusters(ch)),
                               (f"Binder sample t = 0.5 (iteration {ch.iterations[b]})", binder),
                               (f"Binder search t = 0.5 (from {start})", run.labels),
                               (f"VI sample (iteration {ch.iterations[s]}, expected VI {losses[s]:.4f})", vi_labels)):
                pw = aa.pairwise_metrics(lab, truth)
                print(f"{name}({thr}, 10) {label}: precision {pw['precision']:.4f} recall {pw['recall']:.4f} "
                      f"F1 {pw['f1score']:.4f} ARI {aa.adjusted_rand_index(lab, truth):.4f} "
                      f"clusters {len(np.unique(lab))}")
            print(f"  true clusters {len(np.unique(truth))}; the VI estimate: {dt:.2f} s; Binder sample is the VI "
                  f"sample: {b == s}")


if __name__ == "__main__":
    main()
