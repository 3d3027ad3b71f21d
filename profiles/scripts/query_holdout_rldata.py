"""Held-out records of RLdata10000 (tests/golden) linked back with link-records.  500 records, drawn with a fixed seed,
are held out; the similarity_f1.py model (PCG-II, Levenshtein 7/10 on fname_c1 / lname_c1, seed 319158) samples the
other 9 500 with saveEntityValues and saveDistortionProbabilities on, and link-records scores the 500 as queries.
Reported:
  * of the held-out records with a true partner among the 9 500, the share whose best record is one, with p >= 0.5;
  * of those without one, the share with p_new >= 0.5;
  * against a chain on all 10 000 records (same model and schedule): the mean |p(q, r) - pairwise match probability|
    over the pairs of a held-out record that either reports at >= minLinkProbability (a pair the other does not
    report counts as 0 there), and how often the best record equals the full chain's most probable partner, over the
    held-out records where either has one.
The card's name and power limit are read in the same run.

    python profiles/scripts/query_holdout_rldata.py [--burnin 1000] [--samples 100] [--thinning 10] [--seed 7]
"""
import argparse
import csv
import gzip
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dblink_b200 import config  # noqa: E402
from dblink_b200.project import Project  # noqa: E402
from similarity_f1 import CONF, card  # noqa: E402

T = 0.05


def write(path, header, rows):
    with open(path, "w", newline="") as fh:
        w = csv.DictWriter(fh, header)
        w.writeheader()
        w.writerows(rows)


def read(path):
    with open(path, newline="") as fh:
        return list(csv.DictReader(fh))


def run(conf):
    p = Project(config.parse_string(conf), base_dir="")
    start = time.perf_counter()
    p.execute(log=lambda *_: None)
    return time.perf_counter() - start


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--burnin", type=int, default=1000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--thinning", type=int, default=10)
    ap.add_argument("--seed", type=int, default=7)
    a = ap.parse_args()
    with gzip.open(os.path.join(ROOT, "tests", "golden", "RLdata10000.csv.gz"), "rt") as fh:
        rd = csv.DictReader(fh)
        header, rows = rd.fieldnames, list(rd)
    held = set(np.random.default_rng(a.seed).choice(len(rows), 500, replace=False).tolist())
    train = [r for i, r in enumerate(rows) if i not in held]
    queries = [rows[i] for i in sorted(held)]
    ent_of = {r["rec_id"]: r["ent_id"] for r in rows}
    train_ents = {r["ent_id"] for r in train}
    print("card:", card())
    print(f"RLdata10000, 500 records held out (seed {a.seed}), PCG-II, burn-in {a.burnin}, {a.samples} samples every "
          f"{a.thinning} sweeps, model seed 319158, minLinkProbability {T}")
    with tempfile.TemporaryDirectory() as tmp:
        write(os.path.join(tmp, "train.csv"), header, train)
        write(os.path.join(tmp, "queries.csv"), header, queries)
        sample = (f'sampler : "PCG-II", saveEntityValues : true, saveDistortionProbabilities : true}}}},\n'
                  f'        {{name : "link-records", parameters : {{queryPath : "{tmp}/queries.csv", '
                  f'minLinkProbability : {T}}}}}')
        conf = CONF % ("LevenshteinSimilarityFn", "7.0", os.path.join(tmp, "train.csv"), tmp + "/held/", a.samples,
                       a.burnin, a.thinning)
        conf = conf[:conf.index('sampler : "PCG-II"}},')] + sample + "\n    ]\n}\n"  # sample, then link-records
        dt = run(conf)
        print(f"chain on 9 500 records + link-records: {dt:.1f} s")
        links = read(os.path.join(tmp, "held", "query-links.csv"))
        summ = read(os.path.join(tmp, "held", "query-summary.csv"))
        full = CONF % ("LevenshteinSimilarityFn", "7.0", os.path.join(ROOT, "tests", "golden", "RLdata10000.csv.gz"),
                       tmp + "/full/", a.samples, a.burnin, a.thinning)
        full = full.replace('metrics : ["pairwise", "cluster"]', 'metrics : ["pairwise"]').replace(
            '{name : "evaluate"', '{name : "summarize", parameters : {lowerIterationCutoff : 0, quantities : '
            f'["pairwise-match-probabilities"], minMatchProbability : {T}}}}},\n        {{name : "evaluate"')
        dt = run(full)
        print(f"chain on 10 000 records: {dt:.1f} s")
        pmp = read(os.path.join(tmp, "full", "pairwise-match-probabilities.csv"))

    qids = [q["rec_id"] for q in queries]
    with_partner = [q for q in qids if ent_of[q] in train_ents]
    best = {r["queryId"]: (r["bestRecordId"], float(r["bestProbability"]) if r["bestRecordId"] else 0.0) for r in summ}
    new = {r["queryId"]: float(r["newEntityProbability"]) for r in summ}
    hit = sum(1 for q in with_partner if best[q][0] and ent_of[best[q][0]] == ent_of[q] and best[q][1] >= 0.5)
    alone = [q for q in qids if ent_of[q] not in train_ents]
    fresh = sum(1 for q in alone if new[q] >= 0.5)
    print(f"held-out records with a true partner among the 9 500: {len(with_partner)}; best record a true partner "
          f"with p >= 0.5: {hit} ({hit / max(len(with_partner), 1):.3f})")
    print(f"held-out records without one: {len(alone)}; p_new >= 0.5: {fresh} ({fresh / max(len(alone), 1):.3f})")

    qset = set(qids)
    p_q = {(r["queryId"], r["recordId"]): float(r["probability"]) for r in links}
    p_f, partner = {}, {}
    for r in pmp:
        a1, a2, v = r["recordId1"], r["recordId2"], float(r["probability"])
        for q, o in ((a1, a2), (a2, a1)):
            if q in qset and o not in qset:  # the held-out record's partners among the 9 500
                p_f[(q, o)] = v
                if q not in partner or v > partner[q][1]:
                    partner[q] = (o, v)
    keys = set(p_q) | set(p_f)
    diff = [abs(p_q.get(k, 0.0) - p_f.get(k, 0.0)) for k in keys]
    print(f"pairs reported by either at >= {T}: {len(keys)} (link-records {len(p_q)}, full chain {len(p_f)}); mean "
          f"|p - pairwise match probability| {np.mean(diff) if diff else float('nan'):.4f}")
    either = [q for q in qids if best[q][0] or q in partner]
    agree = sum(1 for q in either if best[q][0] and q in partner and best[q][0] == partner[q][0])
    print(f"held-out records with a best record in either: {len(either)}; the same best partner: {agree} "
          f"({agree / max(len(either), 1):.3f})")


if __name__ == "__main__":
    main()
