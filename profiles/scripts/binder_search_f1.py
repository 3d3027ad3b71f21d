"""RLdata10000 (tests/golden): the Binder search against the Binder sample and the sMPC at falseLinkCost t = 0.5 and
0.7, on the chains of binder_f1.py (Levenshtein 7/10 and Jaro-Winkler 8.5/10 on fname_c1 / lname_c1, PCG-II, seed
319158).  Each chain is sampled once; the estimates are computed from it with the functions the summarize and evaluate
steps use, and scored against the ground truth (pairwise precision / recall / F1 and the adjusted Rand index) and by
their posterior expected Binder loss at the user's t.  The card's name and power limit are read in the same run.

    python profiles/scripts/binder_search_f1.py [--burnin 1000] [--samples 100] [--thinning 10]
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
            first, second, count = project.pairwise_match_counts(ch)
            C, S = int(count.sum()), len(ch.samples)
            smpc = project.shared_most_probable_clusters(ch)
            for cost in (0.5, 0.7):
                t = time.perf_counter()
                s, sample, _, _ = project.binder_estimate(ch, cost)
                start, run, rows = project.binder_search_estimate(ch, cost, 1000)
                dt = time.perf_counter() - t
                for label, lab in (("sMPC", smpc), (f"Binder sample (iteration {ch.iterations[s]})", sample),
                                   (f"search (from {start}, {run.rounds} rounds, converged {run.converged})",
                                    run.labels)):
                    n, K = aa.search_result_counts(first, second, count, lab)
                    loss = aa.expected_losses([n], [K], C, S, cost)[0]
                    pw = aa.pairwise_metrics(lab, truth)
                    print(f"{name}({thr}, 10) t = {cost} {label}: precision {pw['precision']:.4f} recall "
                          f"{pw['recall']:.4f} F1 {pw['f1score']:.4f} ARI {aa.adjusted_rand_index(lab, truth):.4f} "
                          f"expected loss {loss:.2f}")
                for r in rows:
                    if r[1] == 0:
                        print(f"  start {r[0]}: expected loss {r[4]:.2f}")
                print(f"  Binder sample + search from both starts: {dt:.1f} s")


if __name__ == "__main__":
    main()
