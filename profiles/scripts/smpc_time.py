"""Time of the shared most probable clusters (sMPC) of a 1 M-record chain: the chain read, the numpy sMPC
(analysis_arrays, S = 100 only: at S = 1 000 its signature matrix alone is 8 GB of host memory) and the GPU sMPC
(analysis_gpu), host clock around work that ends in a synchronise.

The chain is synthetic and seeded: R records, links to 3R/4 entities over 64 partitions, each sample moving 30 % of
the records (samples share most clusters, so modes repeat and tie).  The S = 100 chain is 100 such samples; the
S = 1 000 chain draws its samples (seeded) from those 100.  The read is timed on the first --read-samples samples
written to a linkage-chain.parquet in a temporary directory.

    python profiles/scripts/smpc_time.py [--records 1000000] [--read-samples 10]
"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402

from dblink_b200 import _lib, analysis_arrays as aa, analysis_gpu as ag, writers as w  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception as e:  # no nvidia-smi: the name alone
        import torch

        return f"{torch.cuda.get_device_name(0)}, power limit not reported ({type(e).__name__})"


def links(R, S, seed, partitions=64):
    rng = np.random.default_rng(seed)
    E = (3 * R) // 4
    blk = rng.integers(0, partitions, E).astype(np.int32)
    base = rng.integers(0, E, R).astype(np.int32)
    out = []
    for s in range(S):
        link = base.copy()
        move = rng.random(R) < 0.3
        link[move] = rng.integers(0, E, int(move.sum()))
        if s % 3 == 0:
            base = link
        out.append(link)
    return out, blk


def timed(fn, *a):
    t = time.perf_counter()
    r = fn(*a)
    return r, time.perf_counter() - t


def gpu_split(chain):
    """The GPU sMPC in its two halves: samples in (host labels + upload + signature kernels), then the sMPC."""
    R = chain.num_records
    post = ag.Posterior(R, len(chain.samples))
    try:
        t = time.perf_counter()
        for mem, off, _ in chain.samples:
            post.add_sample(ag.sample_clusters(R, mem, off))
        t_add = time.perf_counter() - t
        (labels, _), t_smpc = timed(post.smpc)
    finally:
        post.close()
    return labels, t_add, t_smpc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--records", type=int, default=1_000_000)
    ap.add_argument("--read-samples", type=int, default=10)
    args = ap.parse_args()
    R = args.records
    if _lib.load().dbl_device_count() == 0:
        sys.exit("no CUDA device")
    print("card:", card())
    print(f"host: {len(os.sched_getaffinity(0))} cpus visible")

    lk, blk = links(R, 100, seed=12345)
    ch100 = aa.ChainArrays(pa.array(["r%d" % i for i in range(R)]), np.arange(100, dtype=np.int64),
                           [aa.sample_from_links(l, blk) for l in lk])
    pool = np.random.default_rng(777).integers(0, 100, 1000)
    ch1000 = aa.ChainArrays(ch100.record_ids, np.arange(1000, dtype=np.int64), [ch100.samples[i] for i in pool])

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "linkage-chain.parquet")
        lw = w.LinkageChainWriter(path, write_buffer_size=2)
        for s in range(args.read_samples):
            lw.append(s, w.linkage_structure_arrow(lk[s], blk, ch100.record_ids))
        lw.close()
        read, t_read = timed(aa.read_chain_arrays, path)
    assert read.num_records == R and len(read.samples) == args.read_samples
    print(f"read_chain_arrays: {t_read / args.read_samples:.3f} s per sample ({args.read_samples} samples, "
          f"64 partitions, R = {R})")

    ag.shared_most_probable_clusters(aa.ChainArrays(np.arange(4), np.zeros(1, np.int64),
                                                    [aa.sample_from_links(np.arange(4, dtype=np.int32), blk)]))  # warm-up
    host, t_host = timed(aa.shared_most_probable_clusters, ch100)
    print(f"S = 100: numpy sMPC {t_host:.2f} s")
    dev, t_dev = timed(ag.shared_most_probable_clusters, ch100)
    assert np.array_equal(dev, host), "GPU labels differ from numpy labels"
    print(f"S = 100: GPU sMPC {t_dev:.2f} s end to end (labels equal numpy's)")
    for S, ch in ((100, ch100), (1000, ch1000)):
        labels, t_add, t_smpc = gpu_split(ch)
        if S == 100:
            assert np.array_equal(labels, host)
        print(f"S = {S}: GPU sMPC {t_add + t_smpc:.2f} s = {t_add:.2f} s adding samples "
              f"({t_add / S * 1e3:.1f} ms each) + {t_smpc:.2f} s dbl_posterior_smpc")


if __name__ == "__main__":
    main()
