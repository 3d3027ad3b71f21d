"""Chain outputs in the reference's formats.

  LinkageChainWriter  linkage-chain.parquet, hive-partitioned by partitionId, columns iteration:int64,
                      linkageStructure:list<list<string>> (package.scala:94-96, util/BufferedRDDWriter.scala:44-50)
  DiagnosticsWriter   diagnostics.csv with the header of DiagnosticsWriter.scala:39-45 and rows of :47-72
  save_cluster_size_distribution / save_partition_sizes   LinkageChain.scala:162-211
  save_pairwise_match_probabilities   pairwise-match-probabilities.csv: recordId1,recordId2,probability
  save_evaluation_samples   evaluation-samples.csv: every sample's counts and metrics against the ground truth
  save_binder_loss   binder-loss.csv: every sample's linked pairs and posterior expected Binder loss
  save_binder_search   binder-search.csv: every round of the Binder search from each start
  save_vi_loss   vi-loss.csv: every sample's number of clusters and posterior expected variation of information
"""
import os
import time

import numpy as np


def linkage_structure(link, block_of_entity, record_ids):
    """State.getLinkageStructure (State.scala:102-112): partition id -> list of clusters (lists of record ids);
    isolated entities carry no cluster."""
    order = np.argsort(link, kind="stable")
    sl = link[order]
    starts = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]])
    ends = np.r_[starts[1:], len(sl)]
    parts = {}
    for s, e in zip(starts, ends):
        ent = sl[s]
        parts.setdefault(int(block_of_entity[ent]), []).append([record_ids[i] for i in order[s:e]])
    return parts


def linkage_structure_arrow(link, block_of_entity, record_ids):
    """The same structure without Python loops over clusters: partition id -> pyarrow ListArray (list<string>), one
    entry per non-isolated entity, clusters in ascending entity id, records of a cluster in ascending record index.
    `record_ids` = a pyarrow string array (or anything pa.array accepts).  At 1M records this takes ~0.2 s where
    the list-of-lists form takes seconds, so a recorded sample costs about as much as the sweeps between samples."""
    import pyarrow as pa

    link = np.asarray(link)
    R = len(link)
    ids = record_ids if isinstance(record_ids, pa.Array) else pa.array([str(r) for r in record_ids], pa.string())
    rec_blk = np.asarray(block_of_entity)[link]
    order = np.lexsort((link, rec_blk))  # stable: by block, then entity, then record index
    sl, sb = link[order], rec_blk[order]
    cstart = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]]) if R else np.zeros(0, np.int64)
    cend = np.r_[cstart[1:], R]
    cblk = sb[cstart]
    values = ids.take(pa.array(order, pa.int64()))
    blocks, first = np.unique(cblk, return_index=True)
    last = np.r_[first[1:], len(cstart)]
    parts = {}
    for b, f, e in zip(blocks, first, last):  # one iteration per partition
        lo, hi = int(cstart[f]), int(cend[e - 1])
        offs = np.r_[cstart[f:e], hi] - lo
        parts[int(b)] = pa.ListArray.from_arrays(pa.array(offs, pa.int32()), values.slice(lo, hi - lo))
    # a partition that holds only isolated entities still has a row, with an empty linkage structure
    # (State.getLinkageStructure maps over every partition, State.scala:102-112)
    for b in np.unique(np.asarray(block_of_entity)):
        if int(b) not in parts:
            parts[int(b)] = pa.ListArray.from_arrays(pa.array([0], pa.int32()), pa.array([], pa.string()))
    return parts


class LinkageChainWriter:
    def __init__(self, path, write_buffer_size=10, append=False):
        import pyarrow as pa

        self.pa = pa
        self.path = path
        self.buf = []
        self.n = write_buffer_size
        self.file_no = 0
        self.schema = pa.schema([("iteration", pa.int64()), ("linkageStructure", pa.list_(pa.list_(pa.string())))])
        if os.path.exists(path) and not append:
            import shutil

            shutil.rmtree(path)
        os.makedirs(path, exist_ok=True)
        if append:
            self.file_no = sum(len(f) for _, _, f in os.walk(path))

    def append(self, iteration, parts):
        self.buf.append((iteration, parts))
        if len(self.buf) >= self.n:
            self.flush()

    def flush(self):
        import pyarrow.parquet as pq

        if not self.buf:
            return
        by_part = {}
        for it, parts in self.buf:
            for pid, clusters in parts.items():
                by_part.setdefault(pid, []).append((it, clusters))
        for pid, rows in by_part.items():
            d = os.path.join(self.path, f"partitionId={pid}")
            os.makedirs(d, exist_ok=True)
            pa = self.pa
            its = pa.array([r[0] for r in rows], pa.int64())
            if all(isinstance(r[1], pa.Array) for r in rows):  # linkage_structure_arrow: no Python lists at all
                offs = np.r_[0, np.cumsum([len(r[1]) for r in rows])]
                ls = pa.ListArray.from_arrays(pa.array(offs, pa.int32()), pa.concat_arrays([r[1] for r in rows]))
            else:
                ls = pa.array([r[1].to_pylist() if isinstance(r[1], pa.Array) else r[1] for r in rows],
                              pa.list_(pa.list_(pa.string())))
            tbl = pa.Table.from_arrays([its, ls], schema=self.schema)
            pq.write_table(tbl, os.path.join(d, f"part-{self.file_no:05d}.parquet"))
        self.file_no += 1
        self.buf = []

    close = flush


def read_linkage_chain(path, lower_iteration_cutoff=0):
    """LinkageChain.readLinkageChain (LinkageChain.scala:35-43) -> [(iteration, {partitionId: clusters})] sorted."""
    import pyarrow.parquet as pq

    samples = {}
    for d in sorted(os.listdir(path)):
        if not d.startswith("partitionId="):
            continue
        pid = int(d.split("=")[1])
        for f in sorted(os.listdir(os.path.join(path, d))):
            t = pq.ParquetFile(os.path.join(path, d, f)).read().to_pydict()
            for it, ls in zip(t["iteration"], t["linkageStructure"]):
                if it >= lower_iteration_cutoff:
                    samples.setdefault(it, {})[pid] = ls
    return sorted(samples.items())


class DiagnosticsWriter:
    def __init__(self, path, attribute_names, append=False):
        self.path = path
        self.names = list(attribute_names)
        new = not (append and os.path.exists(path))
        self.fh = open(path, "a" if append else "w")
        if new:
            agg = ",".join(f"aggDist-{n}" for n in self.names)
            rec = ",".join(f"recDistortion-{k}" for k in range(len(self.names) + 1))
            self.fh.write(f"iteration,systemTime-ms,numObservedEntities,logLikelihood,popSize,{agg},{rec}\n")

    def write_row(self, summary, pop_size):
        agg = summary["agg_dist"].sum(axis=1)  # summed over files (DiagnosticsWriter.scala:52-54)
        row = [str(summary["iteration"]), str(int(time.time() * 1000)), str(pop_size - summary["num_isolates"]),
               f"{summary['log_likelihood']:.9e}", str(pop_size)]
        row += [str(int(v)) for v in agg] + [str(int(v)) for v in summary["rec_dist"]]
        self.fh.write(",".join(row) + "\n")

    def close(self):
        self.fh.close()


def save_cluster_size_distribution(dist, path):
    """LinkageChain.saveClusterSizeDistribution (LinkageChain.scala:162-185)."""
    its = sorted(dist)
    mx = max((max(d) if d else 0) for d in dist.values()) if dist else 0
    with open(os.path.join(path, "cluster-size-distribution.csv"), "w") as fh:
        fh.write("iteration," + ",".join(str(k) for k in range(mx + 1)) + "\n")
        for it in its:
            fh.write(str(it) + "," + ",".join(str(dist[it].get(k, 0)) for k in range(mx + 1)) + "\n")


def save_partition_sizes(sizes, path):
    """LinkageChain.savePartitionSizes (LinkageChain.scala:193-211)."""
    its = sorted(sizes)
    pids = sorted({p for d in sizes.values() for p in d})
    with open(os.path.join(path, "partition-sizes.csv"), "w") as fh:
        fh.write("iteration," + ",".join(str(p) for p in pids) + "\n")
        for it in its:
            fh.write(str(it) + "," + ",".join(str(sizes[it].get(p, 0)) for p in pids) + "\n")


def save_pairwise_match_probabilities(first, second, count, num_samples, record_ids, threshold, path):
    """pairwise-match-probabilities.csv under `path`: header recordId1,recordId2,probability, then one row per pair
    with count / S >= threshold (float64; the row's text parses back to exactly count / S).  In a row recordId1 <
    recordId2 in code-point order; rows go by probability descending, then recordId1, then recordId2.  The R ids are
    ranked once and the rows sorted on integer ranks; the rows are joined by Arrow, not by a Python loop."""
    import pyarrow as pa
    import pyarrow.compute as pc

    from .analysis_arrays import min_match_count

    S = int(num_samples)
    with open(os.path.join(path, "pairwise-match-probabilities.csv"), "wb") as fh:
        fh.write(b"recordId1,recordId2,probability\n")
        if S == 0:
            return
        count = np.asarray(count, np.int64)
        keep = count >= min_match_count(threshold, S)
        first, second, count = np.asarray(first)[keep], np.asarray(second)[keep], count[keep]
        ids = record_ids if isinstance(record_ids, pa.Array) else pa.array([str(r) for r in record_ids], pa.string())
        ids = ids.cast(pa.large_string())
        rank = np.empty(len(ids), np.int64)
        rank[pc.sort_indices(ids).to_numpy()] = np.arange(len(ids))  # UTF-8 byte order = code-point order
        swap = rank[first] > rank[second]
        r1, r2 = np.where(swap, second, first), np.where(swap, first, second)
        order = np.lexsort((rank[r2], rank[r1], -count))
        r1, r2, count = r1[order], r2[order], count[order]
        # repr: the shortest text that parses back to the same float64; one per possible count
        text = pa.array([repr(c / S) + "\n" for c in range(S + 1)], pa.large_string())
        step = 1 << 20
        for lo in range(0, len(count), step):
            rows = pc.binary_join_element_wise(ids.take(r1[lo:lo + step]), ids.take(r2[lo:lo + step]),
                                               text.take(count[lo:lo + step]), pa.scalar(",", pa.large_string()))
            offs = np.frombuffer(rows.buffers()[1], np.int64)[rows.offset:rows.offset + len(rows) + 1]
            fh.write(memoryview(rows.buffers()[2])[offs[0]:offs[-1]])


EVALUATION_SAMPLES_HEADER = "iteration,numClusters,TP,FP,FN,precision,recall,f1score,adjRandIndex"


def save_evaluation_samples(iterations, rows, path):
    """evaluation-samples.csv under `path`: one row per sample (rows = analysis_arrays.sample_metrics, in iteration
    order); floats written with repr, so an undefined metric reads `nan`."""
    with open(os.path.join(path, "evaluation-samples.csv"), "w") as fh:
        fh.write(EVALUATION_SAMPLES_HEADER + "\n")
        for it, r in zip(iterations, rows):
            fh.write(f"{int(it)},{r['numClusters']},{r['TP']},{r['FP']},{r['FN']},{r['precision']!r},{r['recall']!r},"
                     f"{r['f1score']!r},{r['adjRandIndex']!r}\n")


BINDER_LOSS_HEADER = "chain,iteration,linkedPairs,expectedLoss"


def save_binder_loss(chains, iterations, linked_pairs, losses, path):
    """binder-loss.csv under `path`: one row per sample in pooled order (chain-major, then iteration), its record
    pairs linked and its expected loss (analysis_arrays.binder_losses), written with repr."""
    with open(os.path.join(path, "binder-loss.csv"), "w") as fh:
        fh.write(BINDER_LOSS_HEADER + "\n")
        for k, it, n, loss in zip(chains, iterations, linked_pairs, losses):
            fh.write(f"{int(k)},{int(it)},{int(n)},{float(loss)!r}\n")


BINDER_SEARCH_HEADER = "start,round,moves,linkedPairs,expectedLoss"


def save_binder_search(rows, path):
    """binder-search.csv under `path`: rows (start name, round, moves, linked pairs, expected loss) as
    project.binder_search_estimate gives them, round 0 being the start; the loss written with repr."""
    with open(os.path.join(path, "binder-search.csv"), "w") as fh:
        fh.write(BINDER_SEARCH_HEADER + "\n")
        for start, r, moves, n, loss in rows:
            fh.write(f"{start},{int(r)},{int(moves)},{int(n)},{float(loss)!r}\n")


VI_LOSS_HEADER = "chain,iteration,numClusters,expectedLoss"


def save_vi_loss(chains, iterations, num_clusters, losses, path):
    """vi-loss.csv under `path`: one row per sample in pooled order (chain-major, then iteration), its number of
    clusters and its expected variation of information (analysis_arrays.vi_losses), written with repr."""
    with open(os.path.join(path, "vi-loss.csv"), "w") as fh:
        fh.write(VI_LOSS_HEADER + "\n")
        for k, it, n, loss in zip(chains, iterations, num_clusters, losses):
            fh.write(f"{int(k)},{int(it)},{int(n)},{float(loss)!r}\n")
