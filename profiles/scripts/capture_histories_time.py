"""Time of the capture histories of the 1M-record, 100-sample chain of smpc_time.py, with file ids drawn (seeded,
uniform) for F = 2, 4 and 12 files: dbl_capture_add_sample per sample with host labels and with device labels (CUDA
events around the device calls after a warm-up), the read, and the numpy path (analysis_arrays.CaptureCounts) per
sample on the first samples; the device checked equal to numpy on those.  Card name and power limit are read in the
same run.

    python profiles/scripts/capture_histories_time.py [--records 1000000] [--samples 100] [--numpy-samples 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag  # noqa: E402
from smpc_time import card, links  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--samples", type=int, default=100)
    ap.add_argument("--numpy-samples", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if _lib.load().dbl_device_count() < 1:
        raise SystemExit("no CUDA device: this script measures the GPU")
    R, S = args.records, args.samples
    link, _ = links(R, S, seed=1)
    labels = [np.unique(x, return_inverse=True)[1].astype(np.int32) for x in link]  # cluster positions in [0, R)
    dev = [torch.as_tensor(x, device="cuda") for x in labels]
    torch.cuda.synchronize()
    out = {"card": card(), "records": R, "samples": S, "files": {}}
    for F in (2, 4, 12):
        file = np.random.default_rng(F).integers(0, F, R).astype(np.int32)
        row = {}
        for where in ("host", "device"):
            with ag.Capture(file, F, S + 1) as cap:
                cap.add_sample(labels[0])  # warm-up
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t = time.perf_counter()
                start.record()
                for x, d in zip(labels, dev):
                    cap.add_sample(d.data_ptr() if where == "device" else x)
                stop.record()
                torch.cuda.synchronize()
                row[f"add_sample_ms_{where}_labels"] = start.elapsed_time(stop) / S
                row[f"add_sample_ms_{where}_labels_host_clock"] = 1e3 * (time.perf_counter() - t) / S
                t = time.perf_counter()
                H, L = cap.read()
                row["read_ms"] = 1e3 * (time.perf_counter() - t)
        n = args.numpy_samples
        cc = aa.CaptureCounts(file, F)
        t = time.perf_counter()
        for x in labels[:n]:
            cc.add_sample(x)
        row["numpy_ms_per_sample"] = 1e3 * (time.perf_counter() - t) / n
        with ag.Capture(file, F, n) as cap:
            for x in labels[:n]:
                cap.add_sample(x)
            gH, gL = cap.read()
        wH, wL = cc.read()
        row["device_equals_numpy"] = bool(np.array_equal(gH, wH) and np.array_equal(gL, wL))
        out["files"][F] = row
        print(F, json.dumps(row), flush=True)
    print(json.dumps(out))
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
