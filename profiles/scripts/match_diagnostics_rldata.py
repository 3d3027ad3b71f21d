"""RLdata10000 (tests/golden) with 4 PCG-II chains of the binder_f1.py model (Levenshtein 7/10 on fname_c1 /
lname_c1, seed 319158, chain k keyed by the seed + k): the summarize step's pairwise-match-diagnostics over the pairs of
minMatchProbability 0.5 and over every pair seen, printed from its summary file, with the pairs above probability 0.5
that have R̂ > 1.01 and the time of the step.  The card's name and power limit are read in the same run.

    python profiles/scripts/match_diagnostics_rldata.py [--burnin 1000] [--samples 100] [--thinning 10]
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
    print(f"RLdata10000, 4 PCG-II chains, burn-in {a.burnin}, {a.samples} samples every {a.thinning} sweeps, "
          f"seed 319158")
    with tempfile.TemporaryDirectory() as out:
        conf = CONF % ("LevenshteinSimilarityFn", "7.0", data, out + "/", a.samples, a.burnin, a.thinning)
        conf = conf.replace("randomSeed : 319158", "randomSeed : 319158\n    numChains : 4")
        proj = Project(config.parse_string(conf), base_dir="")
        proj.steps = lambda p=proj: [s for s in Project.steps(p) if s[0] == "sample"]
        proj.execute(log=lambda *_: None)
        for t in (0.5, 0.0):
            summarize = conf.replace(
                '{name : "evaluate", parameters : {lowerIterationCutoff : 0, metrics : ["pairwise", "cluster"]}}',
                '{name : "summarize", parameters : {lowerIterationCutoff : 0, minMatchProbability : %r, '
                'quantities : ["pairwise-match-probabilities", "pairwise-match-diagnostics"]}}' % t)
            q = Project(config.parse_string(summarize), base_dir="")
            q.steps = lambda p=q: [s for s in Project.steps(p) if s[0] == "summarize"]
            start = time.perf_counter()
            q.execute(log=lambda *_: None)
            dt = time.perf_counter() - start
            print(f"minMatchProbability {t}: summarize step {dt:.1f} s (both quantities, chain read included)")
            for line in open(os.path.join(out, "pairwise-match-diagnostics-summary.csv")).read().splitlines()[1:]:
                print("  " + line)
            rows = [r.split(",") for r in open(os.path.join(out, "pairwise-match-diagnostics.csv")).read().splitlines()[1:]]
            above = [r for r in rows if float(r[2]) > 0.5]
            print(f"  pairs above probability 0.5: {len(above)}, with R̂ > 1.01: "
                  f"{sum(float(r[5]) > 1.01 for r in above)}, with R̂ > 1.1: {sum(float(r[5]) > 1.1 for r in above)}")


if __name__ == "__main__":
    main()
