"""RLdata10000 (tests/golden) with the similarity_f1.py model (PCG-II, Levenshtein 7/10 on fname_c1 / lname_c1,
seed 319158, 100 samples every 10 sweeps after 1000): the evaluate metric clerical-review centered on the sMPC and on
the VI search, as evaluation-results.txt reports it: the clusters that are not exactly a true entity, the share of
them in the first 1 %, 5 % and 10 % of the review queue and of the queue by cluster probability alone, and the
queue's normalised area under the found-curve.  The card's name and power limit are read in the same run.

    python profiles/scripts/clerical_review_rldata.py [--burnin 1000] [--samples 100] [--thinning 10]
"""
import argparse
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dblink_b200 import config  # noqa: E402
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
    with tempfile.TemporaryDirectory() as out:
        conf = CONF % ("LevenshteinSimilarityFn", "7.0", data, out + "/", a.samples, a.burnin, a.thinning)
        proj = Project(config.parse_string(conf), base_dir="")
        proj.steps = lambda p=proj: [s for s in Project.steps(p) if s[0] == "sample"]
        proj.execute(log=lambda *_: None)
        for center in ("shared-most-probable-clusters", "vi-search-clusters"):
            evaluate = conf.replace('metrics : ["pairwise", "cluster"]',
                                    f'metrics : ["clerical-review"], clericalReviewCenter : "{center}"')
            q = Project(config.parse_string(evaluate), base_dir="")
            q.steps = lambda p=q: [s for s in Project.steps(p) if s[0] == "evaluate"]
            start = time.perf_counter()
            res = q.execute(log=lambda *_: None)["clerical-review"]
            dt = time.perf_counter() - start
            print(f"{center}: evaluate step {dt:.1f} s (chain read and center included)")
            print(open(os.path.join(out, "evaluation-results.txt")).read().rstrip())
            print(f"  summary: {res}")


if __name__ == "__main__":
    main()
