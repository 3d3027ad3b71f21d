"""Capture histories against a known truth: 3-file synthetic data (synth.generate, 2 000 records, 4 constant and 2
Levenshtein attributes, 25 % duplicates), PCG-II sampled on the GPU, then the summarize quantity and the evaluate
metric `capture-histories`: how many history counts and population-size quantities have the truth inside their 95 %
interval, the truth's observed entities and independence estimate beside the posterior's, and the Brier score of
each file column of file-links.csv.  Card name and power limit are read in the same run.

    python profiles/scripts/capture_histories_synth.py [--records 2000] [--samples 200] [--out report.json]
"""
import argparse
import csv
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dblink_b200 import _lib, config, synth  # noqa: E402
from dblink_b200.project import Project  # noqa: E402
from smpc_time import card  # noqa: E402

CONF = """
dblink : {
  data : { path : "%s", recordIdentifier : "rec_id", fileIdentifier : "file_id", entityIdentifier : "ent_id",
           nullValue : "NA", matchingAttributes : [ %s ] }
  outputPath : "%s"
  randomSeed : 3
  expectedMaxClusterSize : 10
  partitioner : { name : "KDTreePartitioner", parameters : { numLevels : 0, matchingAttributes : [] } }
  steps : [
    {name : "sample", parameters : { sampleSize : %d, burninInterval : %d, thinningInterval : 5, resume : false,
                                     sampler : "PCG-II" }}
    {name : "summarize", parameters : { lowerIterationCutoff : %d, quantities : ["capture-histories"] }}
    {name : "evaluate", parameters : { lowerIterationCutoff : %d, metrics : ["capture-histories"] }}
  ]
}
"""


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=2000)
    ap.add_argument("--samples", type=int, default=200)
    ap.add_argument("--burnin", type=int, default=500)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if _lib.load().dbl_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    attrs = [synth.SynthAttr(f"c{i}", "constant", v, 0.5) for i, v in enumerate((100, 12, 31, 50))]
    attrs += [synth.SynthAttr(f"s{i}", "levenshtein", 500, 1.0) for i in range(2)]
    g = synth.generate(11, args.records, attrs, dup=0.25, n_files=3)
    with tempfile.TemporaryDirectory() as tmp:
        data = os.path.join(tmp, "data.csv")
        with open(data, "w", newline="") as fh:
            out = csv.writer(fh, lineterminator="\n")
            out.writerow(["rec_id", "file_id", "ent_id"] + [a.name for a in attrs])
            for r, f, e, v in zip(g["rec_ids"], g["files"], g["ent_ids"], g["values"]):
                out.writerow([r, f, e] + ["NA" if x is None else x for x in v])
        ma = ", ".join(
            f'{{name : "{a.name}", similarityFunction : '
            + ('{ name : "ConstantSimilarityFn" }' if a.kind == "constant" else
               '{ name : "LevenshteinSimilarityFn", parameters : { threshold : 7.0, maxSimilarity : 10.0 } }')
            + ", distortionPrior : {alpha : 10.0, beta : 1000.0}}" for a in attrs)
        outp = os.path.join(tmp, "out") + "/"
        p = Project(config.parse_string(CONF % (data, ma, outp, args.samples, args.burnin, args.burnin,
                                                args.burnin)), base_dir="")
        res = p.execute(log=lambda *a: None)["capture-histories"]
        text = open(os.path.join(outp, "evaluation-results.txt")).read()
        with open(os.path.join(outp, "capture-histories-evaluation.csv"), newline="") as fh:
            rows = list(csv.DictReader(fh))
    report = {"card": card(), "records": args.records, "samples": res["samples"],
              "histories_inside": f"{res['histories_inside']} of {res['histories']}",
              "quantities_inside": f"{res['quantities_inside']} of {res['quantities']}",
              "observed_truth": res["observed"][0], "observed_posterior": res["observed"][1],
              "independence_truth": res["independence"][0], "independence_posterior": res["independence"][1],
              "brier": res["brier"], "rows": rows}
    print(text)
    print(json.dumps({k: v for k, v in report.items() if k != "rows"}))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(report, fh, indent=1)


if __name__ == "__main__":
    main()
