"""Time of linking new records to a chain (dbl_query_*): pass 1 (add_sample) and pass 2 (score_sample) per sample on
the device with device inputs, pass 1 once with host inputs, the read, and the numpy pass 1 on a few queries, scaled.
The chain is fabricated, not sampled: R records in clusters of random labels (0.6 R clusters), entity values drawn
uniformly, 10 attributes (5 Levenshtein over 2 000 random 4-8 letter names, 5 constant over 50 values).  Each query
cell copies an entity's value or draws a random one with probability 1/2.  Random names of that kind have almost no
Levenshtein neighbours, so the hit rows are short and the hashed hit masks rarely send the scan to a row search: the
pass-1 time is a best case against real name data, where rows of dozens of hits cost searches in global memory.
Reading the chain's files is not timed.  Prints the card and its power limit.

    PYTHONPATH=. python profiles/scripts/query_time.py [--records 1000000] [--queries 10000] [--samples 20]
"""
import argparse
import json
import subprocess
import time

import numpy as np


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--samples", type=int, default=20)
    ap.add_argument("--numpy-samples", type=int, default=1)
    ap.add_argument("--numpy-queries", type=int, default=200)
    a = ap.parse_args()
    import torch

    from dblink_b200 import analysis_arrays as aa, analysis_gpu
    from dblink_b200.engine import AttributeIndex

    rng = np.random.default_rng(1)
    letters = np.array(list("ABCDEFGHIJKLMNOPRSTUVWY"))
    names = sorted({"".join(rng.choice(letters, rng.integers(4, 9))) for _ in range(2500)})[:2000]
    idx = []
    for i in range(10):
        vals = names if i < 5 else [f"v{j}" for j in range(50)]
        w = {v: float(rng.integers(1, 50)) for v in vals}
        idx.append(AttributeIndex.build(w, "levenshtein" if i < 5 else "constant", 7.0, 10.0))
    tables = [ix.tables() for ix in idx]
    V = np.array([ix.num_values for ix in idx])
    R, Q, S = a.records, a.queries, a.samples
    K = int(R * 0.6)
    lab = np.r_[np.arange(K), rng.integers(0, K, R - K)].astype(np.int32)
    vals = (rng.random((K, 10)) * V).astype(np.int32)
    qx = np.where(rng.random((Q, 10)) < 0.5, vals[rng.integers(0, K, Q)], (rng.random((Q, 10)) * V).astype(np.int32))
    tab = aa.QueryTables(qx, np.zeros(Q, np.int32), tables, [i >= 5 for i in range(10)], 1)
    theta = rng.uniform(0.01, 0.1, (10, 1))
    dl, dv = torch.as_tensor(lab, device="cuda"), torch.as_tensor(vals, device="cuda")
    out = {}
    with analysis_gpu.Query(tab, R, R, 0.05) as qh:
        for name in ("add_sample", "score_sample"):
            t0 = time.perf_counter()
            for _ in range(S):
                getattr(qh, name)(dl.data_ptr(), (dv.data_ptr(), K), theta)
            out[f"{name}_ms_per_sample_device_inputs"] = (time.perf_counter() - t0) / S * 1e3
        t0 = time.perf_counter()
        res = qh.read()
        out["read_ms"] = (time.perf_counter() - t0) * 1e3
        out["candidates"] = int(len(res.sums))
    with analysis_gpu.Query(tab, R, R, 0.05) as qh:
        t0 = time.perf_counter()
        qh.add_sample(lab, vals, theta)
        out["add_sample_ms_host_inputs"] = (time.perf_counter() - t0) * 1e3
    small = aa.QueryTables(qx[:a.numpy_queries], np.zeros(a.numpy_queries, np.int32), tables,
                           [i >= 5 for i in range(10)], 1)
    qs = aa.QueryScores(small, R, R, 0.05)
    t0 = time.perf_counter()
    for _ in range(a.numpy_samples):
        qs.add_sample(lab, vals, theta)
    out["numpy_pass1_s_per_sample_scaled_to_all_queries"] = (time.perf_counter() - t0) / a.numpy_samples * Q / \
        a.numpy_queries
    out.update(records=R, clusters=K, queries=Q, samples=S, card=subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
        text=True).stdout.strip())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
