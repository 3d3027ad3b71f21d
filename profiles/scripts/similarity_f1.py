"""RLdata10000 (tests/golden) under two similarity functions for the name attributes fname_c1 / lname_c1:
LevenshteinSimilarityFn(7, 10) and JaroWinklerSimilarityFn(8.5, 10).  The same model otherwise (by / bm / bd constant,
distortion prior Beta(10, 1000), 4 k-d-tree blocks on the two names, seed 319158), the same PCG-II sweeps; prints the
pairwise precision / recall / F1 and the adjusted Rand index of the sMPC point estimate of each, the card name and
power limit read in the same run.

    python profiles/scripts/similarity_f1.py [--burnin 1000] [--samples 100] [--thinning 10]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from dblink_b200 import config  # noqa: E402
from dblink_b200.project import Project  # noqa: E402

CONF = """
dblink : {
    dist : {alpha : 10.0, beta : 1000.0}
    const : {name : "ConstantSimilarityFn"}
    names : {name : "%s", parameters : {threshold : %s, maxSimilarity : 10.0}}
    data : {
        path : "%s", recordIdentifier : "rec_id", entityIdentifier : "ent_id", nullValue : "NA"
        matchingAttributes : [
            {name : "by", similarityFunction : ${dblink.const}, distortionPrior : ${dblink.dist}},
            {name : "bm", similarityFunction : ${dblink.const}, distortionPrior : ${dblink.dist}},
            {name : "bd", similarityFunction : ${dblink.const}, distortionPrior : ${dblink.dist}},
            {name : "fname_c1", similarityFunction : ${dblink.names}, distortionPrior : ${dblink.dist}},
            {name : "lname_c1", similarityFunction : ${dblink.names}, distortionPrior : ${dblink.dist}}
        ]
    }
    randomSeed : 319158
    expectedMaxClusterSize : 10
    partitioner : {name : "KDTreePartitioner", parameters : {numLevels : 2, matchingAttributes : ["fname_c1", "lname_c1"]}}
    outputPath : "%s"
    steps : [
        {name : "sample", parameters : {sampleSize : %d, burninInterval : %d, thinningInterval : %d, resume : false,
                                        sampler : "PCG-II"}},
        {name : "evaluate", parameters : {lowerIterationCutoff : 0, metrics : ["pairwise", "cluster"]}}
    ]
}
"""


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:
        return "unknown"


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
            t = time.time()
            res = proj.execute(log=lambda *_: None)
            pw = res["pairwise"]
            print(f"{name}({thr}, 10): precision {pw['precision']:.4f} recall {pw['recall']:.4f} "
                  f"F1 {pw['f1score']:.4f} ARI {res['cluster']:.4f} ({time.time() - t:.1f} s)")


if __name__ == "__main__":
    main()
