"""Share of the PCG-II link kernel that the records with a missing value take: the bench.py workload (BASELINE.json
configs[3]: 1M records, 4 constant + 6 Levenshtein attributes, 64 blocks, 1 % of each attribute missing) against the
same data generated with no missing value (`missing=0.0`; synth.generate_encoded draws the same randoms, so every
other value, file and duplicate is the same).  Both engines are resident at once; each is timed three times, the two
alternating, over `n` eager sweeps per window (CUDA events around every link-kernel launch, dbl_link_kernel_ms).  The
difference between the two link-kernel times bounds what any change to the missing-value path can gain.  The card's
name and power limit are read in the same run.

usage: python profiles/scripts/missing_share.py [out.json] [--sweeps n]
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import dblink_b200 as D  # noqa: E402
from dblink_b200 import synth  # noqa: E402

REPEATS = 3


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True)
    except OSError:
        return "unknown"
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def engine(missing):
    """bench.py's single-GPU set-up of configs[3] (--config 4), with the given missing-value probability."""
    attrs = synth.config_attrs(4)
    enc = synth.generate_encoded(2, 1_000_000, attrs, dup=0.10, distortion=0.05, missing=missing, n_files=2)
    split = [i for i, a in enumerate(attrs) if a.kind == "levenshtein"][:6]
    indexes, x, file, F = synth.build_encoded(enc)
    eng = D.GibbsEngine(indexes, [a.alpha for a in enc["attributes"]], [a.beta for a in enc["attributes"]], None,
                        2024, F)
    eng.init_state(x, file)
    eng.set_partitioner(D.KDTreePartitioner(6, split).fit(eng.download_state()["y"]))
    eng.set_graph_mode(1)  # eager: every link launch is timed
    miss_rows = int(((x[:, [i for i, a in enumerate(attrs) if a.kind != "constant"]] < 0).any(axis=1)).sum())
    return eng, miss_rows / x.shape[0]


def window(eng, n):
    eng.link_kernel_ms()
    eng.sweep("PCG-II", n)
    ms, k = eng.link_kernel_ms()
    return ms / max(k, 1), eng.last_sweep_ms() / n


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    n = int(sys.argv[sys.argv.index("--sweeps") + 1]) if "--sweeps" in sys.argv else 8
    if "--sweeps" in sys.argv:
        args.remove(str(n))
    gpu = card()
    engines = {}
    for label, missing in (("missing=0.01", 0.01), ("missing=0.0", 0.0)):
        eng, frac = engine(missing)
        eng.sweep("PCG-II", 3)
        engines[label] = (eng, frac)
    rows = {label: [] for label in engines}
    for r in range(REPEATS):
        for label, (eng, _) in engines.items():
            link_ms, sweep_ms = window(eng, n)
            rows[label].append({"link_kernel_ms": round(link_ms, 3), "sweep_ms": round(sweep_ms, 3)})
            print(json.dumps({"run": r, "data": label, **rows[label][-1]}), flush=True)
    base = [x["link_kernel_ms"] for x in rows["missing=0.01"]]
    none = [x["link_kernel_ms"] for x in rows["missing=0.0"]]
    out = {"gpu": gpu, "sweeps_per_window": n, "kernel": engines["missing=0.01"][0].link_kernel("PCG-II"),
           "records_missing_a_non_constant_value": {k: round(v[1], 5) for k, v in engines.items()},
           "link_kernel_ms": {"missing=0.01": base, "missing=0.0": none},
           "difference_ms": round(min(base) - min(none), 3),
           "difference_share_of_kernel": round((min(base) - min(none)) / min(base), 4)}
    print(json.dumps(out), flush=True)
    for eng, _ in engines.values():
        eng.close()
    if args:
        with open(args[0], "w") as f:
            json.dump({"summary": out, "runs": rows}, f, indent=1)


if __name__ == "__main__":
    main()
