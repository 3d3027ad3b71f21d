"""Aggregate throughput of batched chains: K chains of one model swept together in one context (dbl_chains_*), in
chain-sweeps per second (K x sweeps/s), for K in {1, 2, 4, 8}, PCG-I and PCG-II, on RLdata10000 (2 k-d levels,
4 blocks) and on the synthetic 100k-record / 8-string-attribute / 16-block problem (bench.py --config 3).  K = 1 is
the ordinary one-chain context.  Each rate is the CUDA-event time of one dbl_sweep call of n sweeps after a warm-up
(graph mode automatic, as a user runs it).  The card's name and power limit are read in the same run.

usage: python profiles/scripts/chains_time.py [out.json]
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import dblink_b200 as D  # noqa: E402

KS = (1, 2, 4, 8)
SAMPLERS = ("PCG-I", "PCG-II")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True)
    except OSError:
        return "unknown"
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def rldata10000():
    from dblink_b200 import config
    from dblink_b200.project import Project
    from test_host_pipeline import GOLDEN, make_conf

    conf = make_conf(os.path.join(GOLDEN, "RLdata10000.csv.gz"), "/tmp/dbl_chains_time/", 2,
                     '["fname_c1", "lname_c1"]')
    proj = Project(config.parse_string(conf), base_dir="")
    d = proj.load()
    return dict(name="RLdata10000 / 4 blocks", indexes=d["cache"].indexes,
                alpha=[a.alpha for a in proj.matching_attributes], beta=[a.beta for a in proj.matching_attributes],
                F=len(d["cache"].file_ids), x=d["x"], file=d["file"], levels=proj.num_levels,
                split=list(proj.partition_attribute_ids), seed=proj.random_seed, warm=30, n=300)


def synthetic_100k():
    from dblink_b200 import synth

    attrs = synth.config_attrs(3)
    enc = synth.generate_encoded(1, 100_000, attrs, dup=0.10, distortion=0.05, missing=0.01, n_files=1)
    indexes, x, file, F = synth.build_encoded(enc)
    split = [i for i, a in enumerate(attrs) if a.kind == "levenshtein"][:4]
    return dict(name="synthetic 100k records / 8 string attrs / 16 blocks", indexes=indexes,
                alpha=[a.alpha for a in enc["attributes"]], beta=[a.beta for a in enc["attributes"]], F=F, x=x,
                file=file, levels=4, split=split, seed=2024, warm=5, n=30)


def rate(p, K, sampler):
    eng = D.GibbsEngine(p["indexes"], p["alpha"], p["beta"], None, p["seed"], p["F"])
    if K == 1:
        eng.init_state(p["x"], p["file"])
        y0 = eng.download_state()["y"]
    else:
        eng.init_chains(p["x"], p["file"], 0, [p["seed"] + k for k in range(K)])
        y0 = eng.download_chains()[0]["y"]
    part = D.KDTreePartitioner(p["levels"], p["split"]).fit(y0)
    eng.set_partitioner(part)
    eng.sweep(sampler, p["warm"])
    eng.sweep(sampler, p["n"])
    ms = eng.last_sweep_ms()
    eng.close()
    return p["n"] / (ms / 1e3)


def main():
    rows = []
    gpu = card()
    for make in (rldata10000, synthetic_100k):
        p = make()
        for sampler in SAMPLERS:
            for K in KS:
                r = rate(p, K, sampler)
                row = {"workload": p["name"], "sampler": sampler, "chains": K, "sweeps_per_s": round(r, 2),
                       "chain_sweeps_per_s": round(K * r, 2), "gpu": gpu}
                rows.append(row)
                print(json.dumps(row), flush=True)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
