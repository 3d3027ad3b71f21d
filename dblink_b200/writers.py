"""Chain outputs in the reference's formats.

  LinkageChainWriter  linkage-chain.parquet, hive-partitioned by partitionId, columns iteration:int64,
                      linkageStructure:list<list<string>> (package.scala:94-96, util/BufferedRDDWriter.scala:44-50)
  EntityValuesChainWriter   entity-values-chain.parquet: the value of every cluster's entity, aligned with the linkage
                      chain's rows and clusters
  DiagnosticsWriter   diagnostics.csv with the header of DiagnosticsWriter.scala:39-45 and rows of :47-72
  save_cluster_size_distribution / save_partition_sizes   LinkageChain.scala:162-211
  save_pairwise_match_probabilities   pairwise-match-probabilities.csv: recordId1,recordId2,probability
  save_evaluation_samples   evaluation-samples.csv: every sample's counts and metrics against the ground truth
  save_binder_loss   binder-loss.csv: every sample's linked pairs and posterior expected Binder loss
  save_binder_search   binder-search.csv: every round of the Binder search from each start
  save_vi_loss   vi-loss.csv: every sample's number of clusters and posterior expected variation of information
  save_entity_values   entity-values.csv: every cluster's most probable value of each attribute and its probability
  DistortionChainWriter   distortion-probabilities-chain.csv: every recorded sample's distortion probabilities
  save_query_links / save_query_summary   query-links.csv / query-summary.csv: new records linked to the chain
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


def cluster_layout(link, block_of_entity):
    """The order clusters are written in, shared by linkage-chain.parquet and entity-values-chain.parquet: records
    sorted by block, then entity, then record index.  Returns (order, cstart, cend, centity, parts): order = the
    records in that order, cluster k = order[cstart[k]:cend[k]] of entity centity[k], and parts = [(partition id,
    first cluster, end cluster)] over the partitions that hold clusters, in ascending partition id."""
    link = np.asarray(link)
    R = len(link)
    rec_blk = np.asarray(block_of_entity)[link]
    order = np.lexsort((link, rec_blk))  # stable: by block, then entity, then record index
    sl, sb = link[order], rec_blk[order]
    cstart = np.flatnonzero(np.r_[True, sl[1:] != sl[:-1]]) if R else np.zeros(0, np.int64)
    cend = np.r_[cstart[1:], R]
    blocks, first = np.unique(sb[cstart], return_index=True)
    last = np.r_[first[1:], len(cstart)]
    return order, cstart, cend, sl[cstart], [(int(b), int(f), int(e)) for b, f, e in zip(blocks, first, last)]


def _empty_partitions(parts, block_of_entity, empty):
    """A partition that holds only isolated entities still has a row, with an empty linkage structure
    (State.getLinkageStructure maps over every partition, State.scala:102-112)."""
    for b in np.unique(np.asarray(block_of_entity)):
        if int(b) not in parts:
            parts[int(b)] = empty()
    return parts


def linkage_structure_arrow(link, block_of_entity, record_ids, layout=None):
    """The same structure without Python loops over clusters: partition id -> pyarrow ListArray (list<string>), one
    entry per non-isolated entity, clusters in ascending entity id, records of a cluster in ascending record index.
    `record_ids` = a pyarrow string array (or anything pa.array accepts).  At 1M records this takes ~0.2 s where
    the list-of-lists form takes seconds, so a recorded sample costs about as much as the sweeps between samples.
    `layout` = cluster_layout(link, block_of_entity) when the caller already has it."""
    import pyarrow as pa

    ids = record_ids if isinstance(record_ids, pa.Array) else pa.array([str(r) for r in record_ids], pa.string())
    order, cstart, cend, _, parts_of = layout if layout is not None else cluster_layout(link, block_of_entity)
    values = ids.take(pa.array(order, pa.int64()))
    parts = {}
    for b, f, e in parts_of:  # one iteration per partition
        lo, hi = int(cstart[f]), int(cend[e - 1])
        offs = np.r_[cstart[f:e], hi] - lo
        parts[b] = pa.ListArray.from_arrays(pa.array(offs, pa.int32()), values.slice(lo, hi - lo))
    return _empty_partitions(parts, block_of_entity,
                             lambda: pa.ListArray.from_arrays(pa.array([0], pa.int32()), pa.array([], pa.string())))


def entity_values_arrow(link, block_of_entity, y, value_strings, layout=None):
    """Partition id -> [one pyarrow string array per matching attribute]: entry k of attribute a is the value of the
    entity of cluster k of the same partition in linkage_structure_arrow(link, block_of_entity, ...) -- non-isolated
    entities only, in the same order.  y = int32[E][A] entity value ids; value_strings[a] = attribute a's values in
    value-id order (a pyarrow string array or anything pa.array accepts).  `layout` = cluster_layout(link,
    block_of_entity) when the caller already has it: the sample step computes it once for both files."""
    import pyarrow as pa

    y = np.asarray(y)
    vals = [v if isinstance(v, pa.Array) else pa.array(list(v), pa.string()) for v in value_strings]
    _, _, _, centity, parts_of = layout if layout is not None else cluster_layout(link, block_of_entity)
    parts = {b: [vals[a].take(pa.array(y[centity[f:e], a], pa.int64())) for a in range(len(vals))]
             for b, f, e in parts_of}
    return _empty_partitions(parts, block_of_entity, lambda: [pa.array([], pa.string()) for _ in vals])


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


class EntityValuesChainWriter:
    """entity-values-chain.parquet, hive-partitioned by partitionId like linkage-chain.parquet, columns
    iteration:int64 and one list<string> per matching attribute, named after it (rows from entity_values_arrow).  It
    flushes in lockstep with the chain's LinkageChainWriter: the same buffer size, and file numbers starting at
    `file_no`, the linkage writer's, so the rows of one flush land in files of the same name in both."""

    def __init__(self, path, attribute_names, write_buffer_size, append, file_no):
        import pyarrow as pa

        self.pa = pa
        self.path = path
        self.names = list(attribute_names)
        self.buf = []
        self.n = write_buffer_size
        self.file_no = file_no
        self.schema = pa.schema([("iteration", pa.int64())] + [(a, pa.list_(pa.string())) for a in self.names])
        if os.path.exists(path) and not append:
            import shutil

            shutil.rmtree(path)
        os.makedirs(path, exist_ok=True)

    def append(self, iteration, parts):
        self.buf.append((iteration, parts))
        if len(self.buf) >= self.n:
            self.flush()

    def flush(self):
        import pyarrow.parquet as pq

        if not self.buf:
            return
        pa = self.pa
        by_part = {}
        for it, parts in self.buf:
            for pid, cols in parts.items():
                by_part.setdefault(pid, []).append((it, cols))
        for pid, rows in by_part.items():
            d = os.path.join(self.path, f"partitionId={pid}")
            os.makedirs(d, exist_ok=True)
            offs = pa.array(np.r_[0, np.cumsum([len(r[1][0]) if r[1] else 0 for r in rows])], pa.int32())
            cols = [pa.array([r[0] for r in rows], pa.int64())]
            for a in range(len(self.names)):
                cols.append(pa.ListArray.from_arrays(offs, pa.concat_arrays([r[1][a] for r in rows])))
            pq.write_table(pa.Table.from_arrays(cols, schema=self.schema),
                           os.path.join(d, f"part-{self.file_no:05d}.parquet"))
        self.file_no += 1
        self.buf = []

    close = flush


DISTORTION_CHAIN = "distortion-probabilities-chain.csv"


def distortion_columns(attribute_names, file_ids):
    """The theta columns of distortion-probabilities-chain.csv, attribute-major: <attribute>[<file id>]."""
    return [f"{a}[{f}]" for a in attribute_names for f in file_ids]


class DistortionChainWriter:
    """distortion-probabilities-chain.csv: header iteration,<attribute>[<file id>],... (distortion_columns), then one
    row per recorded sample, theta[A][F] attribute-major and written with repr, CSV-quoted where a name needs it.  A
    continued chain appends to the file (writing the header only when there is none)."""

    def __init__(self, path, columns, append=False):
        import csv

        new = not (append and os.path.exists(path))
        self.fh = open(path, "a" if not new else "w", newline="")
        self.out = csv.writer(self.fh, lineterminator="\n")
        if new:
            self.out.writerow(["iteration"] + list(columns))

    def write_row(self, iteration, theta):
        self.out.writerow([str(int(iteration))] + [repr(float(v)) for v in np.asarray(theta, np.float64).ravel()])

    def close(self):
        self.fh.close()


def save_distortion_probabilities(rows, path):
    """distortion-probabilities.csv under `path`: per attribute and file the pooled samples' mean, sd, 2.5 %, 50 % and
    97.5 % quantiles and their number S (analysis_arrays.distortion_summary), floats written with repr."""
    _save_csv(path, "distortion-probabilities.csv",
              ("attribute", "file", "mean", "sd", "q2.5", "q50", "q97.5", "samples"),
              [[a, f] + [repr(float(v)) for v in vals] + [s] for a, f, vals, s in rows])


QUERY_LINKS_HEADER = ("queryId", "recordId", "probability")
QUERY_SUMMARY_HEADER = ("queryId", "newEntityProbability", "bestRecordId", "bestProbability", "effectiveSamples",
                        "unseenAttributes")


def save_query_links(rows, path):
    """query-links.csv under `path`: (query id, record id, probability) rows as project.py orders them."""
    _save_csv(path, "query-links.csv", QUERY_LINKS_HEADER, [(q, r, repr(float(p))) for q, r, p in rows])


def save_query_summary(rows, path):
    """query-summary.csv under `path`: one row per query in query-file order."""
    _save_csv(path, "query-summary.csv", QUERY_SUMMARY_HEADER, rows)


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


def pair_row_order(first, second, count, record_ids):
    """The row order of pairwise-match-probabilities.csv: (ids as a large_string Arrow array, r1, r2, order), where
    r1[i] < r2[i] in record-id code-point order and `order` sorts the pairs by count descending, then r1, then r2
    (r1, r2 already in that order)."""
    import pyarrow as pa
    import pyarrow.compute as pc

    first, second, count = np.asarray(first), np.asarray(second), np.asarray(count, np.int64)
    ids = record_ids if isinstance(record_ids, pa.Array) else pa.array([str(r) for r in record_ids], pa.string())
    ids = ids.cast(pa.large_string())
    rank = np.empty(len(ids), np.int64)
    rank[pc.sort_indices(ids).to_numpy()] = np.arange(len(ids))  # UTF-8 byte order = code-point order
    swap = rank[first] > rank[second]
    r1, r2 = np.where(swap, second, first), np.where(swap, first, second)
    order = np.lexsort((rank[r2], rank[r1], -count))
    return ids, r1[order], r2[order], order


PAIRWISE_MATCH_DIAGNOSTICS_HEADER = ("recordId1,recordId2,probability,minChainProbability,maxChainProbability,splitRhat,"
                                     "ess,mcse")


def save_pairwise_match_diagnostics(first, second, count, num_samples, mix, mcse, record_ids, path):
    """pairwise-match-diagnostics.csv under `path`: the rows of pairwise-match-probabilities.csv (the same pairs,
    order and probability text, count / num_samples), each with its least and largest per-chain probability over the
    2N draws of a chain the diagnostics use, split-R̂, ESS and MCSE (mix = an analysis_arrays.MatchMixing), written
    with repr."""
    S = int(num_samples)
    with open(os.path.join(path, "pairwise-match-diagnostics.csv"), "w") as fh:
        fh.write(PAIRWISE_MATCH_DIAGNOSTICS_HEADER + "\n")
        if len(count) == 0:
            return
        ids, r1, r2, order = pair_row_order(first, second, count, record_ids)
        ids = ids.to_pylist()
        D = 2 * mix.N
        count = np.asarray(count, np.int64)[order]
        cols = [mix.chain_min[order], mix.chain_max[order], mix.rhat[order], mix.ess[order], np.asarray(mcse)[order]]
        step = 1 << 16
        for lo in range(0, len(order), step):
            fh.write("".join(f"{ids[a]},{ids[b]},{c / S!r},{lo_c / D!r},{hi_c / D!r},{float(rh)!r},{float(e)!r},"
                             f"{float(m)!r}\n"
                             for a, b, c, lo_c, hi_c, rh, e, m in zip(r1[lo:lo + step], r2[lo:lo + step],
                                                                     count[lo:lo + step].tolist(),
                                                                     *(x[lo:lo + step].tolist() for x in cols))))


def save_pairwise_match_diagnostics_summary(rows, path):
    """pairwise-match-diagnostics-summary.csv under `path`: (quantity, value) rows, floats written with repr."""
    with open(os.path.join(path, "pairwise-match-diagnostics-summary.csv"), "w") as fh:
        fh.write("quantity,value\n")
        for q, v in rows:
            fh.write(f"{q},{v!r}\n")


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
        ids, r1, r2, order = pair_row_order(np.asarray(first)[keep], np.asarray(second)[keep], count[keep], record_ids)
        count = count[keep][order]
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


VI_SEARCH_HEADER = "start,round,moves,numClusters,expectedLoss"


def save_vi_search(rows, path):
    """vi-search.csv under `path`: rows (start name, round, moves, clusters, quantised expected VI) as
    project.vi_search_estimate gives them, round 0 being the start; the loss written with repr."""
    with open(os.path.join(path, "vi-search.csv"), "w") as fh:
        fh.write(VI_SEARCH_HEADER + "\n")
        for start, r, moves, k, loss in rows:
            fh.write(f"{start},{int(r)},{int(moves)},{int(k)},{float(loss)!r}\n")


CREDIBLE_BALL_SAMPLES_HEADER = "chain,iteration,numClusters,viDistance,binderDistance"


def save_credible_ball_samples(chains, iterations, num_clusters, vi, binder, path):
    """credible-ball-samples.csv under `path`: one row per sample in pooled order (chain-major, then iteration), its
    number of clusters and its VI (written with repr) and Binder distance from the center of the ball."""
    with open(os.path.join(path, "credible-ball-samples.csv"), "w") as fh:
        fh.write(CREDIBLE_BALL_SAMPLES_HEADER + "\n")
        for k, it, n, v, b in zip(chains, iterations, num_clusters, vi, binder):
            fh.write(f"{int(k)},{int(it)},{int(n)},{float(v)!r},{int(b)}\n")


CREDIBLE_BALL_HEADER = ("distance,bound,center,level,radius,samplesInBall,samples,chain,iteration,numClusters,"
                        "distanceToCenter,ties")


def save_credible_ball(rows, path):
    """credible-ball.csv under `path`: rows (distance, bound, center, level, radius, samples in the ball, samples,
    chain, iteration, clusters, distance to the center, ties) as project.py gives them, one per distance and bound;
    floats written with repr."""
    with open(os.path.join(path, "credible-ball.csv"), "w") as fh:
        fh.write(CREDIBLE_BALL_HEADER + "\n")
        for row in rows:
            fh.write(",".join(repr(x) if isinstance(x, float) else str(x) for x in row) + "\n")


def save_entity_values(attribute_names, rows, path):
    """entity-values.csv under `path`: header cluster,size,<attr>,<attr>Probability,... (matching attributes in config
    order), then rows as analysis_arrays.entity_value_rows gives them, CSV-quoted where a value needs it."""
    import csv

    with open(os.path.join(path, "entity-values.csv"), "w", newline="") as fh:
        out = csv.writer(fh, lineterminator="\n")
        out.writerow(["cluster", "size"] + [x for a in attribute_names for x in (a, a + "Probability")])
        out.writerows(rows)


CLERICAL_REVIEW_HEADER = ("rank", "cluster", "size", "clusterProbability", "expectedFalseLinks", "expectedMissedLinks",
                          "expectedLoss", "weakestInternalLinkProbability", "strongestLinkInsideRecordId",
                          "strongestLinkOutsideRecordId", "strongestOutsideLinkProbability")
CLERICAL_REVIEW_RECORDS_HEADER = ("recordId", "cluster", "clusterProbability", "expectedFalseLinks",
                                  "expectedMissedLinks", "strongestOutsideRecordId", "strongestOutsideLinkProbability")
CLERICAL_REVIEW_EVALUATION_HEADER = ("rank", "cluster", "erroneous", "erroneousFound")


def _save_csv(path, name, header, rows):
    import csv

    with open(os.path.join(path, name), "w", newline="") as fh:
        out = csv.writer(fh, lineterminator="\n")
        out.writerow(header)
        out.writerows(rows)


def save_clerical_review(rows, path):
    """clerical-review.csv under `path`: one row per cluster of the point estimate in review order, as
    analysis_arrays.clerical_review_rows gives them, CSV-quoted where a record id needs it."""
    _save_csv(path, "clerical-review.csv", CLERICAL_REVIEW_HEADER, rows)


def save_clerical_review_records(rows, path):
    """clerical-review-records.csv under `path`: one row per record in chain record order, as
    analysis_arrays.clerical_review_record_rows gives them."""
    _save_csv(path, "clerical-review-records.csv", CLERICAL_REVIEW_RECORDS_HEADER, rows)


def save_clerical_review_evaluation(rows, path):
    """clerical-review-evaluation.csv under `path`: per position of the review queue its cluster, whether it is not
    exactly a true entity (1) and the erroneous clusters found up to it."""
    _save_csv(path, "clerical-review-evaluation.csv", CLERICAL_REVIEW_EVALUATION_HEADER, rows)


def _number(x):
    """An integer as itself, a float with repr."""
    return repr(float(x)) if isinstance(x, (float, np.floating)) else str(int(x))


def save_capture_histories(summary, chains, iterations, file_ids, path):
    """The capture-histories files under `path`, every number from an analysis_arrays.CaptureSummary over the pooled
    samples (chain-major), floats written with repr:
      capture-histories-samples.csv  chain, iteration, one 0/1 column per file id, entities: one row per sample and per
                                     history with a non-zero count, histories ascending
      capture-histories.csv          per history 1 .. 2^F - 1: its 0/1 columns, mean, sd and 2.5/50/97.5 % quantiles
                                     of its count
      population-size.csv            per quantity: mean, sd, quantiles over the samples where it is finite, and the
                                     number where it is infinite
      population-size-samples.csv    chain, iteration, one column per quantity"""
    fids = [str(f) for f in file_ids]
    H, hist = summary.H, summary.histories
    rows = []
    for k, it, row in zip(chains, iterations, H):
        for h in np.flatnonzero(row[1:]) + 1:
            rows.append([int(k), int(it)] + hist[h - 1].tolist() + [int(row[h])])
    _save_csv(path, "capture-histories-samples.csv", ["chain", "iteration"] + fids + ["entities"], rows)
    _save_csv(path, "capture-histories.csv", fids + ["mean", "sd", "q2.5", "q50", "q97.5"],
              [m.tolist() + [repr(v) for v in vals] for m, vals in zip(hist, summary.history_summary())])
    names = summary.quantity_names(fids)
    _save_csv(path, "population-size.csv", ("quantity", "mean", "sd", "q2.5", "q50", "q97.5", "infinite"),
              [[q] + [repr(v) for v in vals[:5]] + [vals[5]] for q, vals in zip(names, summary.quantity_summary())])
    _save_csv(path, "population-size-samples.csv", ["chain", "iteration"] + names,
              [[int(k), int(it)] + [_number(c[s]) for c in summary.columns]
               for s, (k, it) in enumerate(zip(chains, iterations))])


def save_file_links(record_ids, record_files, probabilities, file_ids, path):
    """file-links.csv under `path`: per record in data order its id, its file id and, per file id, the probability
    (written with repr) that its cluster holds another record of that file."""
    _save_csv(path, "file-links.csv", ["recordId", "fileId"] + [str(f) for f in file_ids],
              [[r, f] + [repr(float(p)) for p in row] for r, f, row in zip(record_ids, record_files, probabilities)])


def save_capture_histories_evaluation(rows, path):
    """capture-histories-evaluation.csv under `path`: rows (quantity, truth, posterior mean, 2.5 % and 97.5 %
    quantiles, 1 when the truth lies inside them), floats written with repr."""
    _save_csv(path, "capture-histories-evaluation.csv", ("quantity", "truth", "mean", "q2.5", "q97.5", "inside"),
              [[q, _number(t)] + [repr(float(v)) for v in vals] + [int(inside)] for q, t, *vals, inside in rows])
