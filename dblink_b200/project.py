"""Project: a dblink configuration bound to its data (Project.scala:32-230, ProjectSteps.scala:53-84).

Same HOCON surface as the reference (`dblink.data.*`, `dblink.partitioner`, `dblink.steps[*]`, ...); the sample
step runs on the GPU engine, summarize / evaluate read linkage-chain.parquet on the host and compute the shared most
probable clusters on the GPU when there is one.
"""
import os
import shutil

import numpy as np

from . import (_lib, analysis, analysis_arrays, analysis_gpu, config as hocon, convergence, sampler as chain, state_io,
               writers)
from .engine import GibbsEngine, KDTreePartitioner
from .records import (Attribute, RecordsCache, SimilarityFn, build_cache_from_columns, read_csv,  # noqa: F401
                      read_csv_columns)

SMPC_METRICS = ("pairwise", "cluster")  # ProjectStep.scala:36
# every sample at or after the cutoff against the ground truth: evaluation-samples.csv and a posterior summary
POSTERIOR_METRICS = ("posterior-pairwise", "posterior-cluster")
# the sample of least posterior expected Binder loss (falseLinkCost = the cost of a false link) against the ground truth
BINDER_METRICS = ("binder-pairwise", "binder-cluster")
# the least expected Binder loss found by single-record moves from the Binder sample and from the sMPC
BINDER_SEARCH_METRICS = ("binder-search-pairwise", "binder-search-cluster")
# the sample of least posterior expected variation of information against the ground truth
VI_METRICS = ("vi-pairwise", "vi-cluster")
# the least expected variation of information found by single-record moves from the VI sample and from the sMPC
VI_SEARCH_METRICS = ("vi-search-pairwise", "vi-search-cluster")
# whether the ground truth lies in the credible ball around a point estimate, in VI and in Binder distance
CREDIBLE_BALL_METRICS = ("credible-ball",)
# how well the clerical review queue of a point estimate finds its clusters that are not exactly a true entity
CLERICAL_REVIEW_METRICS = ("clerical-review",)
# the posterior capture histories, population sizes and file links against those of the ground truth
CAPTURE_HISTORY_METRICS = ("capture-histories",)
SUPPORTED_METRICS = (SMPC_METRICS + POSTERIOR_METRICS + BINDER_METRICS + BINDER_SEARCH_METRICS + VI_METRICS
                     + VI_SEARCH_METRICS + CREDIBLE_BALL_METRICS + CLERICAL_REVIEW_METRICS + CAPTURE_HISTORY_METRICS)
SUPPORTED_QUANTITIES = ("cluster-size-distribution", "partition-sizes", "shared-most-probable-clusters",  # :37
                        "pairwise-match-probabilities", "convergence-diagnostics", "binder-clusters",
                        "binder-search-clusters", "vi-clusters", "vi-search-clusters", "credible-ball",
                        "entity-values", "pairwise-match-diagnostics", "clerical-review", "distortion-probabilities",
                        "capture-histories")
# the point estimates a credible ball may be centred on
CREDIBLE_BALL_CENTERS = ("shared-most-probable-clusters", "binder-clusters", "binder-search-clusters", "vi-clusters",
                         "vi-search-clusters")


def shared_most_probable_clusters(chain):
    """sMPC labels of a ChainArrays: on the GPU when the platform has one (analysis_gpu), else on the host
    (analysis_arrays).  Both give identical labels, so the output files do not depend on the platform."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.shared_most_probable_clusters(chain)
    return analysis_arrays.shared_most_probable_clusters(chain)


def pairwise_match_counts(chain, min_count=1):
    """(first, second, count) of a ChainArrays, the pairs that share a cluster in at least min_count samples: on the
    GPU when the platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.pairwise_match_counts(chain, min_count=min_count)
    return analysis_arrays.pairwise_match_counts(chain, min_count=min_count)


def pairwise_match_diagnostics(chain, min_count=1):
    """(first, second, count, MatchMixing) of a ChainArrays, the pairs that share a cluster in at least min_count
    samples and their split-R̂ and ESS: on the GPU when the platform has one (analysis_gpu), else on the host
    (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.pairwise_match_diagnostics(chain, min_count=min_count)
    return analysis_arrays.pairwise_match_diagnostics(chain, min_count=min_count)


def posterior_metric_counts(chain, truth):
    """(tp, pred_pairs, num_clusters) of every sample of a ChainArrays against the ground truth: on the GPU when the
    platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.posterior_metric_counts(chain, truth)
    return analysis_arrays.posterior_metric_counts(chain, truth)


def binder_counts(chain):
    """(n, K) of every sample of a ChainArrays, the pairs it links and the sum of their match counts: on the GPU when
    the platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.binder_counts(chain)
    return analysis_arrays.binder_counts(chain)


def binder_estimate(chain, false_link_cost):
    """The sample of least posterior expected Binder loss of a ChainArrays: (its position, its labels, every sample's
    linked pairs and expected loss)."""
    if not chain.samples:
        raise ValueError("the Binder-loss estimate needs at least one sample at or after lowerIterationCutoff")
    n, K = binder_counts(chain)
    s = analysis_arrays.binder_estimate(n, K, false_link_cost)
    mem, off, _ = chain.samples[s]
    return (s, analysis_arrays.sample_labels(chain.num_records, mem, off), n,
            analysis_arrays.binder_losses(n, K, false_link_cost))


def binder_search(chain, false_link_cost, starts, max_rounds):
    """(chosen position, SearchRuns) of the single-record-move search from each start: on the GPU when the platform
    has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical results."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.binder_search(chain, false_link_cost, starts, max_rounds)
    return analysis_arrays.binder_search(chain, false_link_cost, starts, max_rounds)


def binder_search_estimate(chain, false_link_cost, max_rounds):
    """The search from the Binder sample and from the sMPC of a ChainArrays: (the chosen start's name, its SearchRun,
    the rows of binder-search.csv: per start and round its name, the round, the moves, the linked pairs and the
    expected loss at the given falseLinkCost; round 0 is the start)."""
    _, labels, n, _ = binder_estimate(chain, false_link_cost)
    best, runs = binder_search(chain, false_link_cost, [labels, shared_most_probable_clusters(chain)], max_rounds)
    C, S = int(n.sum()), len(n)
    rows = []
    for name, run in zip(analysis_arrays.SEARCH_STARTS, runs):
        linked = run.linked_pairs()
        losses = analysis_arrays.expected_losses(linked, run.count_sums(), C, S, false_link_cost)
        rows += [(name, r, m, k, loss) for r, (m, k, loss) in enumerate(zip(np.r_[0, run.moves], linked, losses))]
    return analysis_arrays.SEARCH_STARTS[best], runs[best], rows


def vi_cross_histograms(chain):
    """G of a ChainArrays, the cell histograms of every sample against the others: on the GPU when the platform has
    one (analysis_gpu), else on the host (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.vi_cross_histograms(chain)
    return analysis_arrays.vi_cross_histograms(chain)


def vi_estimate(chain):
    """The sample of least posterior expected variation of information of a ChainArrays: (its position, its labels,
    every sample's number of clusters and expected VI)."""
    if not chain.samples:
        raise ValueError("the VI estimate needs at least one sample at or after lowerIterationCutoff")
    G = vi_cross_histograms(chain)
    g = analysis_arrays.vi_cluster_histograms(chain, G.shape[1])
    losses = analysis_arrays.vi_losses(g, G, chain.num_records)
    s = analysis_arrays.vi_estimate(losses)
    mem, off, _ = chain.samples[s]
    return (s, analysis_arrays.sample_labels(chain.num_records, mem, off),
            np.array([len(off) - 1 for _, off, _ in chain.samples], np.int64), losses)


def vi_samples(chain):
    """Every sample of a ChainArrays held once for the VI search path: an analysis_gpu.VI handle when the platform has
    a device, else analysis_arrays.VISamples.  Both give identical results."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.vi_samples(chain)
    return analysis_arrays.VISamples(chain)


def vi_search_estimate(chain, max_rounds):
    """The VI search from the VI sample and from the sMPC of a ChainArrays, on one set of held samples that also gives
    the cross histograms and the scores: (the chosen start's name, its VISearchRun, the rows of vi-search.csv -- per
    start and round its name, the round, the moves, the clusters and the quantised expected VI E_q; round 0 is the
    start -- and the exact expected VI of [vi-sample start, smpc start, vi-sample result, smpc result])."""
    if not chain.samples:
        raise ValueError("the VI search needs at least one sample at or after lowerIterationCutoff")
    R, S = chain.num_records, len(chain.samples)
    width = analysis_arrays.vi_width(chain)
    analysis_arrays.check_vi_search_size(S, R)
    analysis_arrays.check_vi_search_squares(analysis_arrays.vi_sample_squares(chain))
    smpc = shared_most_probable_clusters(chain)
    table = analysis_arrays.vi_search_table(R)
    g = analysis_arrays.vi_cluster_histograms(chain, width)
    g_sum = g.sum(axis=0)
    with vi_samples(chain) as vi:
        s = analysis_arrays.vi_estimate(analysis_arrays.vi_losses(g, vi.cross(width), R))
        mem, off, _ = chain.samples[s]
        starts = [analysis_arrays.sample_labels(R, mem, off), smpc]
        runs = [vi.search(table, st, max_rounds) for st in starts]
        exact = [analysis_arrays.vi_label_loss(np.bincount(np.bincount(lab)), vi.score(lab, width), g_sum, S, R)
                 for lab in starts + [r.labels for r in runs]]
    best = analysis_arrays.vi_search_choice(runs)
    sample_sum = analysis_arrays.vi_sample_sum(chain, table)
    rows = []
    for name, st, run in zip(analysis_arrays.VI_SEARCH_STARTS, starts, runs):
        losses = analysis_arrays.vi_search_losses(run.objectives(), sample_sum, S, R)
        counts = [len(np.unique(st))] + run.clusters.tolist()
        rows += [(name, r, m, k, loss) for r, (m, k, loss) in enumerate(zip([0] + run.moves.tolist(), counts, losses))]
    return analysis_arrays.VI_SEARCH_STARTS[best], runs[best], rows, exact


def entity_value_modes(labels, value_samples, num_values):
    """(modes, counts, S) of the entity values of the clusters of labels over the samples of value_samples: on the
    GPU when the platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.entity_value_modes(labels, value_samples, num_values)
    return analysis_arrays.entity_value_modes(labels, value_samples, num_values)


def credible_ball_center(chain, center, false_link_cost, max_rounds):
    """The labels of the point estimate `center` (one of CREDIBLE_BALL_CENTERS) of a ChainArrays, computed as its own
    summarize quantity computes it."""
    if center == "shared-most-probable-clusters":
        return shared_most_probable_clusters(chain)
    if center == "binder-clusters":
        return binder_estimate(chain, false_link_cost)[1]
    if center == "binder-search-clusters":
        return binder_search_estimate(chain, false_link_cost, max_rounds)[1].labels
    if center == "vi-clusters":
        return vi_estimate(chain)[1]
    if center == "vi-search-clusters":
        return vi_search_estimate(chain, max_rounds)[1].labels
    raise ValueError(f"credibleBallCenter must be one of {CREDIBLE_BALL_CENTERS}.")


def record_links(chain, labels):
    """analysis_arrays.RecordLinks of the canonical labels[R] against the pair table of a ChainArrays: on the GPU when
    the platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give identical integers."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.record_links(chain, labels)
    first, second, count = analysis_arrays.pairwise_match_counts(chain)
    return analysis_arrays.record_links(first, second, count, labels, int(np.max(labels)) + 1)


def cluster_appearances(chain, labels):
    """A, int64[R]: the samples of a ChainArrays in which each record's cluster is its cluster in the canonical
    labels[R]: on the GPU when the platform has one (analysis_gpu), else on the host (analysis_arrays).  Both give
    identical integers."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.cluster_appearances(chain, labels)
    return analysis_arrays.cluster_appearances(chain, labels)


def clerical_review_estimate(chain, center, false_link_cost, max_rounds):
    """The analysis_arrays.ClericalReview of the point estimate `center` (one of CREDIBLE_BALL_CENTERS) of a
    ChainArrays, its clusters numbered canonically, ranked at falseLinkCost = false_link_cost."""
    if not chain.samples:
        raise ValueError("the clerical review needs at least one sample at or after lowerIterationCutoff")
    labels = analysis_arrays.canonical_clusters(credible_ball_center(chain, center, false_link_cost, max_rounds))
    return analysis_arrays.ClericalReview(record_links(chain, labels), cluster_appearances(chain, labels), labels,
                                          len(chain.samples), false_link_cost)


def credible_ball_estimate(chain, center, level, false_link_cost, max_rounds):
    """The credible ball of a ChainArrays around the estimate `center`: (its labels, every sample's number of clusters,
    {"vi" | "binder": (every sample's distance from the center, radius, in-ball mask, bounds)}), the bounds as
    analysis_arrays.credible_ball gives them.  The cells of the center with every sample come from one set of held
    samples (GPU or host)."""
    if not chain.samples:
        raise ValueError("the credible ball needs at least one sample at or after lowerIterationCutoff")
    R = chain.num_records
    labels = np.asarray(credible_ball_center(chain, center, false_link_cost, max_rounds), np.int64)
    width = analysis_arrays.vi_width(chain)
    g = analysis_arrays.vi_cluster_histograms(chain, width)
    with vi_samples(chain) as vi:
        G = vi.score_samples(labels, width)
    distances = analysis_arrays.credible_ball_distances(np.bincount(np.bincount(labels)), g, G, R)
    num_clusters = np.array([len(off) - 1 for _, off, _ in chain.samples], np.int64)
    balls = {name: (d,) + analysis_arrays.credible_ball(d, num_clusters, level)
             for name, d in zip(analysis_arrays.CREDIBLE_BALL_DISTANCES, distances)}
    return labels, num_clusters, balls


def credible_ball_truth(labels, truth):
    """(VI, Binder distance) of the ground truth from the labelling `labels`: one contingency table of the two, through
    analysis_arrays.credible_ball_distances."""
    labels, truth = np.asarray(labels, np.int64), np.unique(np.asarray(truth), return_inverse=True)[1].astype(np.int64)
    R = len(labels)
    _, n = np.unique(labels * max(R, 1) + truth, return_counts=True)
    sizes = np.bincount(np.bincount(truth))
    cells = np.bincount(n[n >= 2], minlength=len(sizes))
    vi, binder = analysis_arrays.credible_ball_distances(np.bincount(np.bincount(labels)), sizes[None, :],
                                                         cells[None, :], R)
    return float(vi[0]), int(binder[0])


def _credible_ball_rows(chain, center, level, balls):
    """The rows of credible-ball.csv: per distance and bound, (distance, bound, center, level, radius, samples in the
    ball, samples, chain, iteration, clusters, distance to the center, ties) of the bound's sample."""
    rows = []
    S = len(chain.samples)
    for name, (d, radius, inside, bounds) in balls.items():
        for bound in analysis_arrays.CREDIBLE_BALL_BOUNDS:
            s, ties = bounds[bound]
            rows.append((name, bound, center, level, radius, int(inside.sum()), S, int(chain.chains[s]),
                         int(chain.iterations[s]), len(chain.samples[s][1]) - 1, d[s].item(), ties))
    return rows


def _center_settings(prm, key, name):
    """The settings the point estimate prm[key] is computed with, for run.txt: `name`=center, then the settings that
    apply to it."""
    center = prm[key]
    out = f"{name}={center}"
    if center.startswith("binder"):
        out += f", falseLinkCost={prm['false_link_cost']}"
    if center.endswith("search-clusters"):
        out += f", maxSearchRounds={prm['max_search_rounds']}"
    return out


def _credible_ball_settings(prm):
    """The settings a credible ball's center is computed with, for run.txt."""
    return (_center_settings(prm, "credible_ball_center", "credibleBallCenter")
            + f", credibleLevel={prm['credible_level']}")


def _credible_ball_params(prm):
    center = prm.get("credibleBallCenter", "vi-search-clusters")
    if center not in CREDIBLE_BALL_CENTERS:
        raise ValueError(f"credibleBallCenter must be one of {CREDIBLE_BALL_CENTERS}.")
    level = prm.get("credibleLevel", 0.95)
    if isinstance(level, bool) or not isinstance(level, (int, float)) or not 0.0 < float(level) <= 1.0:
        raise ValueError("credibleLevel must be in (0, 1].")
    return dict(credible_ball_center=center, credible_level=float(level))


def _entity_values_center(prm):
    center = prm.get("entityValuesCenter", "shared-most-probable-clusters")
    if center not in CREDIBLE_BALL_CENTERS:
        raise ValueError(f"entityValuesCenter must be one of {CREDIBLE_BALL_CENTERS}.")
    return center


def _clerical_review_center(prm):
    center = prm.get("clericalReviewCenter", "shared-most-probable-clusters")
    if center not in CREDIBLE_BALL_CENTERS:
        raise ValueError(f"clericalReviewCenter must be one of {CREDIBLE_BALL_CENTERS}.")
    return center


def _clerical_review_settings(prm):
    """The settings a clerical review is computed with, for run.txt: its center's, then the cost of a false link the
    queue is ranked at."""
    return (_center_settings(prm, "clerical_review_center", "clericalReviewCenter")
            + f", ranked at falseLinkCost={prm['false_link_cost']}")


def _save_entity_values(prm):
    """{"save_entity_values": True} when the sample step records entity values, else nothing: a step without the
    option keeps the parameters it always had."""
    save = prm.get("saveEntityValues", False)
    if not isinstance(save, bool):
        raise ValueError("saveEntityValues must be a boolean.")
    return {"save_entity_values": True} if save else {}


def _save_distortion_probabilities(prm):
    """{"save_distortion_probabilities": True} when the sample step records theta, else nothing."""
    save = prm.get("saveDistortionProbabilities", False)
    if not isinstance(save, bool):
        raise ValueError("saveDistortionProbabilities must be a boolean.")
    return {"save_distortion_probabilities": True} if save else {}


def capture_histories(chain, file, num_files):
    """(H, L) of a ChainArrays whose record i is in file[i], the clusters of each sample per set of files and each
    record's links into every file: on the GPU when the platform has one (analysis_gpu), else on the host
    (analysis_arrays).  Both give identical arrays."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.capture_histories(chain, file, num_files)
    return analysis_arrays.capture_histories(chain, file, num_files)


def link_queries(tables, samples, num_records, population_size, min_link_probability):
    """analysis_arrays.QueryResult of the query records against the samples: on the GPU when the platform has one
    (analysis_gpu), else on the host (analysis_arrays).  Both give the same candidates and sums within rounding."""
    if _lib.load().dbl_device_count() > 0:
        return analysis_gpu.link_queries(tables, samples, num_records, population_size, min_link_probability)
    return analysis_arrays.link_queries(tables, samples, num_records, population_size, min_link_probability)


def _searched_cost(false_link_cost):
    a, b = analysis_arrays.search_cost(false_link_cost)
    return a / b


def _max_search_rounds(prm):
    m = prm.get("maxSearchRounds", 1000)
    if isinstance(m, bool) or not isinstance(m, int) or m < 1:
        raise ValueError("maxSearchRounds must be a positive integer.")
    return m


def _false_link_cost(prm):
    t = float(prm.get("falseLinkCost", 0.5))
    if not 0.0 <= t <= 1.0:
        raise ValueError("falseLinkCost must be in [0, 1].")
    return t


class Project:
    def __init__(self, cfg, base_dir="."):
        g = cfg.get
        self.cfg = cfg
        self.data_path = os.path.join(base_dir, cfg.get_string("dblink.data.path"))
        self.output_path = os.path.join(base_dir, cfg.get_string("dblink.outputPath"))
        self.rec_id_attribute = cfg.get_string("dblink.data.recordIdentifier")
        self.file_id_attribute = g("dblink.data.fileIdentifier", None)
        self.ent_id_attribute = g("dblink.data.entityIdentifier", None)
        self.null_value = cfg.get_string("dblink.data.nullValue")
        self.random_seed = cfg.get_int("dblink.randomSeed")
        # dblink.numChains: independent chains of the model swept together on one GPU, chain k keyed by randomSeed + k
        nc = g("dblink.numChains", 1)
        if isinstance(nc, bool) or not isinstance(nc, int) or nc < 1:
            raise ValueError("numChains must be a positive integer.")
        self.num_chains = nc
        self.population_size = g("dblink.populationSize", None)
        self.expected_max_cluster_size = int(g("dblink.expectedMaxClusterSize", 10))
        self.matching_attributes = []
        for c in cfg.get_list("dblink.data.matchingAttributes"):  # Project.parseMatchingAttributes, :201-216
            sf = c["similarityFunction"]
            if sf["name"] == "ConstantSimilarityFn":
                fn = SimilarityFn("ConstantSimilarityFn")
            elif sf["name"] in ("LevenshteinSimilarityFn", "JaroWinklerSimilarityFn"):
                fn = SimilarityFn(sf["name"], float(sf["parameters"]["threshold"]),
                                  float(sf["parameters"]["maxSimilarity"]))
            else:
                raise hocon.ConfigError("similarityFunction.name: unsupported value")
            self.matching_attributes.append(Attribute(c["name"], fn, float(c["distortionPrior"]["alpha"]),
                                                      float(c["distortionPrior"]["beta"])))
        p = cfg.get_config("dblink.partitioner")  # Project.parsePartitioner, :218-229
        if p.get_string("name") != "KDTreePartitioner":
            raise hocon.ConfigError("partitioner.name: unsupported value")
        names = [a.name for a in self.matching_attributes]
        self.num_levels = p.get_int("parameters.numLevels")
        self.partition_attribute_ids = [names.index(n) for n in p.get_list("parameters.matchingAttributes")]
        self._loaded = None

    @classmethod
    def from_file(cls, path):
        base = os.getcwd()
        return cls(hocon.parse_file(path), base)

    # ---- description (what Run.main writes to run.txt, Run.scala:38-43) ----------------------------
    def mk_string(self):
        """Project.mkString (Project.scala:58-96)."""
        def sim(fn):
            if fn.name == "ConstantSimilarityFn":
                return "ConstantSimilarityFn"
            return f"{fn.name}(threshold={fn.threshold}, maxSimilarity={fn.max_similarity})"

        L = ["Data settings", "-------------", f"  * Using data files located at '{self.data_path}'",
             f"  * The record identifier attribute is '{self.rec_id_attribute}'",
             f"  * The file identifier attribute is '{self.file_id_attribute}'" if self.file_id_attribute
             else "  * There is no file identifier",
             f"  * The entity identifier attribute is '{self.ent_id_attribute}'" if self.ent_id_attribute
             else "  * There is no entity identifier",
             "  * The matching attributes are " + ", ".join(f"'{a.name}'" for a in self.matching_attributes), "",
             "Hyperparameter settings", "-----------------------"]
        for i, a in enumerate(self.matching_attributes):
            L.append(f"  * '{a.name}' (id={i}) with {sim(a.similarity_fn)} and "
                     f"BetaShapeParameters(alpha={a.alpha}, beta={a.beta})")
        L += [f"  * Size of latent population is {self.population_size}", "",
              "Partition function settings", "---------------------------"]
        if self.num_levels == 0:
            L.append("  * KDTreePartitioner(numLevels=0)")
        else:
            L.append(f"  * KDTreePartitioner(numLevels={self.num_levels}, attributeIds="
                     f"[{','.join(str(i) for i in self.partition_attribute_ids)}])")
        L += ["", "Project settings", "----------------", f"  * Using randomSeed={self.random_seed}"]
        if self.num_chains > 1:
            L.append(f"  * Running numChains={self.num_chains} chains with seeds "
                     + ", ".join(str(s) for s in self.chain_seeds()) + " (one k-d tree, fitted on chain 0; chains "
                     "start from State.deterministic, not over-dispersed), outputs under chain-<k>/")
        L += [
              f"  * Using expectedMaxClusterSize={self.expected_max_cluster_size}",
              f"  * Saving Markov chain and complete final state to '{self.output_path}'",
              "  * Sweeps run on the CUDA device of this process (libdblink_b200); there are no Spark checkpoints"]
        return "\n".join(L) + "\n"

    def steps_mk_string(self):
        """ProjectSteps.mkString (ProjectSteps.scala:38-45) with the step descriptions of ProjectStep.scala."""
        L = ["Scheduled steps", "---------------"]
        braces = lambda xs: "{" + ", ".join(f"'{x}'" for x in xs) + "}"
        for name, prm in self.steps():
            if name == "sample":
                src = "saved state" if prm["resume"] else "new initial state"
                L.append(f"  * SampleStep: Evolving the chain from {src} with sampleSize={prm['sample_size']}, "
                         f"burninInterval={prm['burnin_interval']}, thinningInterval={prm['thinning_interval']} and "
                         f"sampler={prm['sampler']}"
                         + (", saving every sample's entity values (saveEntityValues=true)"
                            if prm.get("save_entity_values") else "")
                         + (", saving every sample's distortion probabilities (saveDistortionProbabilities=true)"
                            if prm.get("save_distortion_probabilities") else ""))
            elif name == "summarize":
                L.append(f"  * SummarizeStep: Calculating summary quantities {braces(prm['quantities'])} along the "
                         f"chain for iterations >= {prm['lower_iteration_cutoff']}")
                if "binder-clusters" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: binder-clusters is the sample of least posterior expected Binder "
                             f"loss with falseLinkCost={prm['false_link_cost']}")
                if "binder-search-clusters" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: binder-search-clusters is the least posterior expected Binder loss "
                             f"found by single-record moves from the Binder sample and the sMPC, with "
                             f"falseLinkCost={prm['false_link_cost']} (searched at "
                             f"{_searched_cost(prm['false_link_cost'])!r}) and "
                             f"maxSearchRounds={prm['max_search_rounds']}")
                if "vi-clusters" in prm["quantities"]:
                    L.append("  * SummarizeStep: vi-clusters is the sample of least posterior expected variation of "
                             "information")
                if "vi-search-clusters" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: vi-search-clusters is the least posterior expected variation of "
                             f"information found by single-record moves from the VI sample and the sMPC, with "
                             f"maxSearchRounds={prm['max_search_rounds']}")
                if "credible-ball" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: credible-ball is the smallest ball around a point estimate, in "
                             f"variation of information and in Binder distance, that holds a share of the samples, "
                             f"with {_credible_ball_settings(prm)}")
                if "pairwise-match-diagnostics" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: pairwise-match-diagnostics gives split-R̂, effective sample size and "
                             f"Monte Carlo standard error of every pair's link indicator, for the pairs of "
                             f"minMatchProbability={prm['min_match_probability']!r}")
                if "entity-values" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: entity-values is the most probable value of each attribute of the "
                             f"entity of each cluster of a point estimate, from the entity values saved with the "
                             f"samples, with {_center_settings(prm, 'entity_values_center', 'entityValuesCenter')}")
                if "distortion-probabilities" in prm["quantities"]:
                    L.append("  * SummarizeStep: distortion-probabilities summarises the distortion probabilities "
                             "saved with the samples, per attribute and file")
                if "clerical-review" in prm["quantities"]:
                    L.append(f"  * SummarizeStep: clerical-review ranks the clusters of a point estimate by their "
                             f"expected false and missed links, with {_clerical_review_settings(prm)}")
                if "capture-histories" in prm["quantities"]:
                    L.append("  * SummarizeStep: capture-histories counts every sample's clusters by the set of files "
                             "they hold, every record's links into each file, and population-size estimates from "
                             "those counts; their spread reflects linkage uncertainty only")
            elif name == "evaluate":
                smpc = [m for m in prm["metrics"] if m in SMPC_METRICS]
                post = [m for m in prm["metrics"] if m in POSTERIOR_METRICS]
                if smpc and prm["use_existing_smpc"]:
                    L.append(f"  * EvaluateStep: Evaluating saved sMPC clusters using {braces(smpc)} metrics")
                elif smpc:
                    L.append(f"  * EvaluateStep: Evaluating sMPC clusters (computed from the chain for iterations >= "
                             f"{prm['lower_iteration_cutoff']}) using {braces(smpc)} metrics")
                if post:
                    L.append(f"  * EvaluateStep: Evaluating every sample of the chain for iterations >= "
                             f"{prm['lower_iteration_cutoff']} using {braces(post)} metrics")
                binder = [m for m in prm["metrics"] if m in BINDER_METRICS]
                if binder:
                    L.append(f"  * EvaluateStep: Evaluating the sample of least posterior expected Binder loss "
                             f"(falseLinkCost={prm['false_link_cost']}, iterations >= {prm['lower_iteration_cutoff']}) "
                             f"using {braces(binder)} metrics")
                search = [m for m in prm["metrics"] if m in BINDER_SEARCH_METRICS]
                if search:
                    L.append(f"  * EvaluateStep: Evaluating the least posterior expected Binder loss found by "
                             f"single-record moves from the Binder sample and the sMPC (falseLinkCost="
                             f"{prm['false_link_cost']}, searched at {_searched_cost(prm['false_link_cost'])!r}, "
                             f"maxSearchRounds={prm['max_search_rounds']}, iterations >= "
                             f"{prm['lower_iteration_cutoff']}) using {braces(search)} metrics")
                vi = [m for m in prm["metrics"] if m in VI_METRICS]
                if vi:
                    L.append(f"  * EvaluateStep: Evaluating the sample of least posterior expected variation of "
                             f"information (iterations >= {prm['lower_iteration_cutoff']}) using {braces(vi)} metrics")
                vi_search = [m for m in prm["metrics"] if m in VI_SEARCH_METRICS]
                if vi_search:
                    L.append(f"  * EvaluateStep: Evaluating the least posterior expected variation of information "
                             f"found by single-record moves from the VI sample and the sMPC (maxSearchRounds="
                             f"{prm['max_search_rounds']}, iterations >= {prm['lower_iteration_cutoff']}) using "
                             f"{braces(vi_search)} metrics")
                ball = [m for m in prm["metrics"] if m in CREDIBLE_BALL_METRICS]
                if ball:
                    L.append(f"  * EvaluateStep: Evaluating whether the ground truth lies in the credible ball around a "
                             f"point estimate ({_credible_ball_settings(prm)}, iterations >= "
                             f"{prm['lower_iteration_cutoff']}) using {braces(ball)} metrics")
                review = [m for m in prm["metrics"] if m in CLERICAL_REVIEW_METRICS]
                if review:
                    L.append(f"  * EvaluateStep: Evaluating how soon the clerical review queue of a point estimate "
                             f"reaches its clusters that are not a true entity ({_clerical_review_settings(prm)}, "
                             f"iterations >= {prm['lower_iteration_cutoff']}) using {braces(review)} metrics")
                capture = [m for m in prm["metrics"] if m in CAPTURE_HISTORY_METRICS]
                if capture:
                    L.append(f"  * EvaluateStep: Evaluating the capture histories, population sizes and file links of "
                             f"every sample against those of the ground truth (iterations >= "
                             f"{prm['lower_iteration_cutoff']}) using {braces(capture)} metrics")
            elif name == "link-records":
                L.append(f"  * LinkRecordsStep: Linking the records of '{prm['query_path']}' to the chain for "
                         f"iterations >= {prm['lower_iteration_cutoff']}, reporting the records they share an entity "
                         f"with at minLinkProbability={prm['min_link_probability']!r}; each query is scored against "
                         f"the data alone: queries are not linked to each other and the chain is not updated")
            else:
                L.append("  * CopyFilesStep: Copying {" + ", ".join(prm["file_names"]) + "} to destination "
                         + prm["destination_path"])
        return "\n".join(L)

    def write_run_txt(self):
        """run.txt under outputPath: the project and its scheduled steps (Run.scala:38-43)."""
        os.makedirs(self.output_path, exist_ok=True)
        with open(os.path.join(self.output_path, "run.txt"), "w") as fh:
            fh.write(self.mk_string())
            fh.write("\n" + self.steps_mk_string())

    # ---- data ------------------------------------------------------------------------------------
    def load(self):
        if self._loaded is None:
            names = [a.name for a in self.matching_attributes]
            # columnar path (pyarrow): same cache / value ids as read_csv + RecordsCache.build + transform_records
            rec_ids, files, columns, ent_ids = read_csv_columns(self.data_path, self.rec_id_attribute, names,
                                                                self.file_id_attribute, self.ent_id_attribute,
                                                                self.null_value)
            cache, x, f = build_cache_from_columns(columns, files, self.matching_attributes,
                                                   self.expected_max_cluster_size)
            self._loaded = {"rec_ids": rec_ids.to_pylist(), "ent_ids": None if ent_ids is None else ent_ids.to_pylist(),
                            "cache": cache, "x": x, "file": f}
        return self._loaded

    def true_clusters(self):
        d = self.load()
        if d["ent_ids"] is None:
            return None
        return analysis.membership_to_clusters(d["rec_ids"], d["ent_ids"])

    def true_labels(self):
        """Ground truth as a function: record ids (pyarrow array, the chain's dictionary) -> int labels in that
        order; None when the data has no entity id column."""
        d = self.load()
        if d["ent_ids"] is None:
            return None

        def lookup(record_ids):
            import pyarrow as pa
            import pyarrow.compute as pc

            pos = pc.index_in(record_ids, value_set=pa.array([str(r) for r in d["rec_ids"]], pa.string()))
            if pos.null_count:
                raise ValueError("the chain mentions record ids that are not in the data")
            _, lab = np.unique(np.asarray([str(e) for e in d["ent_ids"]], dtype=object), return_inverse=True)
            return lab[pos.to_numpy(zero_copy_only=False)]

        return lookup

    def chain_seeds(self):
        return [self.random_seed + k for k in range(self.num_chains)]

    def chain_dirs(self):
        """Where each chain's linkage-chain.parquet / diagnostics.csv / state.npz live."""
        if self.num_chains == 1:
            return [self.output_path]
        return [os.path.join(self.output_path, f"chain-{k}") for k in range(self.num_chains)]

    def _new_engine(self):
        d = self.load()
        cache = d["cache"]
        return GibbsEngine(cache.indexes, [a.alpha for a in self.matching_attributes],
                           [a.beta for a in self.matching_attributes], None, self.random_seed, len(cache.file_ids))

    def fingerprint(self):
        d = self.load()
        return state_io.model_fingerprint(d["cache"].indexes, d["x"], d["file"],
                                          [a.alpha for a in self.matching_attributes],
                                          [a.beta for a in self.matching_attributes],
                                          extra=(int(self.random_seed), int(self.population_size or 0),
                                                 int(self.num_levels), tuple(self.partition_attribute_ids))
                                          + ((("numChains", self.num_chains),) if self.num_chains > 1 else ()))

    def generate_initial_state(self):
        """Project.generateInitialState (:130-145) -> a GibbsEngine at iteration 0."""
        d = self.load()
        eng = self._new_engine()
        if self.num_chains == 1:
            eng.init_state(d["x"], d["file"], int(self.population_size or 0))
            y0 = eng.download_state()["y"]
        else:  # one tree for every chain, fitted on chain 0's initial entity values
            eng.init_chains(d["x"], d["file"], int(self.population_size or 0), self.chain_seeds())
            y0 = eng.download_chains()[0]["y"]
        part = KDTreePartitioner(self.num_levels, self.partition_attribute_ids).fit(y0)
        eng.set_partitioner(part)
        eng._partitioner_keepalive = part
        return eng

    def saved_state(self):
        """Project.savedState (:113-128): the engine restored from `state.npz` under outputPath, or None.  The
        partition function is re-fitted on the deterministic initial entity values, exactly as the original run
        fitted it, so the resumed chain continues as if it had never stopped; the fingerprint covers the data, the
        tables, the priors, randomSeed, populationSize and the partitioner settings, so a state saved under a
        different configuration is refused instead of being continued with another key / partition function."""
        dirs = self.chain_dirs()
        if not all(state_io.saved_state_exists(p) for p in dirs):
            return None
        sts = [state_io.load_state(p, self.fingerprint()) for p in dirs]
        d = self.load()
        eng = self.generate_initial_state()
        if self.num_chains == 1:
            st = sts[0]
            eng.upload_state(d["x"], d["file"], st["z"], st["link"], st["y"], st["theta"], st["iteration"])
        else:
            if len({st["iteration"] for st in sts}) != 1:
                raise ValueError("the chains' saved states are at different iterations")
            eng.upload_chains(d["x"], d["file"], sts, self.chain_seeds(), sts[0]["iteration"])
        return eng

    def save_state(self, eng):
        if self.num_chains == 1:
            state_io.save_state(eng, self.output_path, self.fingerprint(), self.random_seed)
        else:
            state_io.save_chain_states(eng, self.chain_dirs(), self.fingerprint(), self.chain_seeds())

    # ---- steps (ProjectSteps.parseSteps) -------------------------------------------------------------
    def steps(self):
        out = []
        for st in self.cfg.get_list("dblink.steps"):
            prm = st.get("parameters", {})
            name = st["name"]
            if name == "sample":
                out.append(("sample", dict(sample_size=int(prm["sampleSize"]),
                                           burnin_interval=int(prm.get("burninInterval", 0)),
                                           thinning_interval=int(prm.get("thinningInterval", 1)),
                                           resume=bool(prm.get("resume", True)), sampler=prm.get("sampler", "PCG-I"),
                                           **_save_entity_values(prm), **_save_distortion_probabilities(prm))))
            elif name == "summarize":
                q = list(prm["quantities"])
                if not q or any(x not in SUPPORTED_QUANTITIES for x in q):
                    raise ValueError(f"quantities must be one of {SUPPORTED_QUANTITIES}.")
                if "capture-histories" in q:
                    analysis_arrays.check_capture_files(len(self.load()["cache"].file_ids))
                if "convergence-diagnostics" in q and self.num_chains < 2:
                    raise ValueError("convergence-diagnostics needs numChains >= 2.")
                # minMatchProbability: pairwise-match-probabilities.csv keeps the pairs at least this probable
                t = float(prm.get("minMatchProbability", 0.0))
                if not 0.0 <= t <= 1.0:
                    raise ValueError("minMatchProbability must be in [0, 1].")
                out.append(("summarize", dict(lower_iteration_cutoff=int(prm.get("lowerIterationCutoff", 0)),
                                              quantities=q, min_match_probability=t,
                                              false_link_cost=_false_link_cost(prm),
                                              max_search_rounds=_max_search_rounds(prm),
                                              entity_values_center=_entity_values_center(prm),
                                              clerical_review_center=_clerical_review_center(prm),
                                              **_credible_ball_params(prm))))
            elif name == "evaluate":
                m = list(prm["metrics"])
                if not m or any(x not in SUPPORTED_METRICS for x in m):
                    raise ValueError(f"metrics must be one of {SUPPORTED_METRICS}.")
                if any(x in CAPTURE_HISTORY_METRICS for x in m):
                    analysis_arrays.check_capture_files(len(self.load()["cache"].file_ids))
                out.append(("evaluate", dict(lower_iteration_cutoff=int(prm.get("lowerIterationCutoff", 0)), metrics=m,
                                             use_existing_smpc=bool(prm.get("useExistingSMPC", False)),
                                             false_link_cost=_false_link_cost(prm),
                                             max_search_rounds=_max_search_rounds(prm),
                                             clerical_review_center=_clerical_review_center(prm),
                                             **_credible_ball_params(prm))))
            elif name == "link-records":
                if "queryPath" not in prm:
                    raise ValueError("link-records needs queryPath.")
                out.append(("link-records", dict(
                    query_path=str(prm["queryPath"]), lower_iteration_cutoff=int(prm.get("lowerIterationCutoff", 0)),
                    min_link_probability=analysis_arrays._check_min_link_probability(
                        prm.get("minLinkProbability", 0.05)))))
            elif name == "copy-files":
                out.append(("copy-files", dict(file_names=list(prm["fileNames"]),
                                               destination_path=prm["destinationPath"],
                                               overwrite=bool(prm.get("overwrite", False)),
                                               delete_source=bool(prm.get("deleteSource", False)))))
            else:
                raise hocon.ConfigError("steps.name: unsupported step")
        return out

    def execute(self, log=print):
        eng = None
        results = {}
        for name, prm in self.steps():
            if name == "sample":
                if prm["resume"]:  # ProjectStep.scala:47-52
                    eng = eng or self.saved_state() or self.generate_initial_state()
                else:
                    eng = self.generate_initial_state()
                d = self.load()
                log(f"SampleStep: sampleSize={prm['sample_size']} burninInterval={prm['burnin_interval']} "
                    f"thinningInterval={prm['thinning_interval']} sampler={prm['sampler']}")
                chain.sample(eng, d["rec_ids"], [a.name for a in self.matching_attributes], prm["sample_size"],
                             self.output_path, prm["burnin_interval"], prm["thinning_interval"], sampler=prm["sampler"],
                             entity_values=self.attribute_values() if prm.get("save_entity_values") else None,
                             distortion_columns=self.distortion_columns()
                             if prm.get("save_distortion_probabilities") else None)
                self.save_state(eng)  # Sampler.scala:120
            elif name == "summarize":
                # array implementations (analysis_arrays): same quantities as analysis.py, no loop over clusters
                cut = prm["lower_iteration_cutoff"]
                ch = self.read_chain(cut)  # several chains: their samples pooled, chain-major
                for q in prm["quantities"]:
                    if q in ("cluster-size-distribution", "partition-sizes"):  # per chain
                        for dr in self.chain_dirs():
                            one = (ch if self.num_chains == 1 else
                                   analysis_arrays.read_chain_arrays(os.path.join(dr, "linkage-chain.parquet"), cut))
                            if q == "cluster-size-distribution":
                                writers.save_cluster_size_distribution(analysis_arrays.cluster_size_distribution(one),
                                                                       dr)
                            else:
                                writers.save_partition_sizes(analysis_arrays.partition_sizes(one), dr)
                    elif q == "convergence-diagnostics":
                        rows = convergence.convergence_diagnostics(
                            [os.path.join(dr, "diagnostics.csv") for dr in self.chain_dirs()], cut)
                        convergence.save_convergence_diagnostics(rows, self.output_path)
                    elif q == "pairwise-match-probabilities":
                        S, t = len(ch.samples), prm["min_match_probability"]
                        first, second, count = pairwise_match_counts(ch, min_count=analysis_arrays.min_match_count(t, S))
                        writers.save_pairwise_match_probabilities(first, second, count, S, ch.record_ids, t,
                                                                  self.output_path)
                    elif q == "pairwise-match-diagnostics":
                        S, t = len(ch.samples), prm["min_match_probability"]
                        first, second, count, mix = pairwise_match_diagnostics(
                            ch, min_count=analysis_arrays.min_match_count(t, S))
                        mcse = analysis_arrays.mcse(mix.count, mix.M * mix.N, mix.ess)
                        writers.save_pairwise_match_diagnostics(first, second, count, S, mix, mcse, ch.record_ids,
                                                                self.output_path)
                        writers.save_pairwise_match_diagnostics_summary(
                            analysis_arrays.match_diagnostics_summary(mix, mix.M // 2, mix.draws), self.output_path)
                    elif q == "binder-clusters":
                        s, labels, n, losses = binder_estimate(ch, prm["false_link_cost"])
                        self._save_smpc(analysis_arrays.labels_to_clusters(labels, ch.record_ids),
                                        "binder-clusters.csv")
                        writers.save_binder_loss(ch.chains, ch.iterations, n, losses, self.output_path)
                    elif q == "binder-search-clusters":
                        _, run, rows = binder_search_estimate(ch, prm["false_link_cost"], prm["max_search_rounds"])
                        self._save_smpc(analysis_arrays.labels_to_clusters(run.labels, ch.record_ids),
                                        "binder-search-clusters.csv")
                        writers.save_binder_search(rows, self.output_path)
                    elif q == "vi-clusters":
                        _, labels, num_clusters, losses = vi_estimate(ch)
                        self._save_smpc(analysis_arrays.labels_to_clusters(labels, ch.record_ids), "vi-clusters.csv")
                        writers.save_vi_loss(ch.chains, ch.iterations, num_clusters, losses, self.output_path)
                    elif q == "vi-search-clusters":
                        _, run, rows, _ = vi_search_estimate(ch, prm["max_search_rounds"])
                        self._save_smpc(analysis_arrays.labels_to_clusters(run.labels, ch.record_ids),
                                        "vi-search-clusters.csv")
                        writers.save_vi_search(rows, self.output_path)
                    elif q == "credible-ball":
                        center, level = prm["credible_ball_center"], prm["credible_level"]
                        _, num_clusters, balls = credible_ball_estimate(ch, center, level, prm["false_link_cost"],
                                                                        prm["max_search_rounds"])
                        writers.save_credible_ball_samples(ch.chains, ch.iterations, num_clusters, balls["vi"][0],
                                                           balls["binder"][0], self.output_path)
                        rows = _credible_ball_rows(ch, center, level, balls)
                        writers.save_credible_ball(rows, self.output_path)
                        for name, bound, *_ in rows:
                            mem, off, _ = ch.samples[balls[name][3][bound][0]]
                            self._save_smpc(analysis_arrays.labels_to_clusters(
                                analysis_arrays.sample_labels(ch.num_records, mem, off), ch.record_ids),
                                f"credible-ball-{name}-{bound}.csv")
                    elif q == "entity-values":
                        self._summarize_entity_values(ch, prm)
                    elif q == "distortion-probabilities":
                        A, F = len(self.matching_attributes), len(self.load()["cache"].file_ids)
                        theta = analysis_arrays.read_distortion_probabilities(self.chain_dirs(), ch, A, F)
                        cols = [(a.name, f) for a in self.matching_attributes for f in self.load()["cache"].file_ids]
                        writers.save_distortion_probabilities(
                            [(a, f, vals[:5], vals[5]) for (a, f), vals in
                             zip(cols, analysis_arrays.distortion_summary(theta))], self.output_path)
                    elif q == "capture-histories":
                        self._summarize_capture_histories(ch)
                    elif q == "clerical-review":
                        review = clerical_review_estimate(ch, prm["clerical_review_center"], prm["false_link_cost"],
                                                          prm["max_search_rounds"])
                        self._save_smpc(analysis_arrays.labels_to_clusters(review.labels, ch.record_ids),
                                        "clerical-review-clusters.csv")
                        writers.save_clerical_review(analysis_arrays.clerical_review_rows(review, ch.record_ids),
                                                     self.output_path)
                        writers.save_clerical_review_records(
                            analysis_arrays.clerical_review_record_rows(review, ch.record_ids), self.output_path)
                    else:
                        labels = shared_most_probable_clusters(ch)
                        self._save_smpc(analysis_arrays.labels_to_clusters(labels, ch.record_ids))
            elif name == "evaluate":
                true_labels = self.true_labels()
                if true_labels is None:
                    raise ValueError("Ground truth entity ids are required for evaluation")  # ProjectStep.scala:65
                cut = prm["lower_iteration_cutoff"]
                text, ch = [], None
                if any(m in SMPC_METRICS for m in prm["metrics"]):
                    ch = self.read_chain(cut)
                    smpc_path = os.path.join(self.output_path, "shared-most-probable-clusters.csv")
                    if prm["use_existing_smpc"] and os.path.exists(smpc_path):  # ProjectStep.scala EvaluateStep
                        labels = self._read_smpc_labels(smpc_path, ch.record_ids)
                    else:
                        labels = shared_most_probable_clusters(ch)
                        self._save_smpc(analysis_arrays.labels_to_clusters(labels, ch.record_ids))
                    truth = true_labels(ch.record_ids)
                    for m in prm["metrics"]:
                        if m == "pairwise":
                            results["pairwise"] = analysis_arrays.pairwise_metrics(labels, truth)
                            text.append(analysis.format_pairwise(results["pairwise"]))
                        elif m == "cluster":
                            results["cluster"] = analysis_arrays.adjusted_rand_index(labels, truth)
                            text.append(analysis.format_cluster(results["cluster"]))
                if any(m in POSTERIOR_METRICS for m in prm["metrics"]):
                    rows, true_clusters = self._evaluate_samples(cut, true_labels, ch)
                    summary = analysis_arrays.posterior_summary(rows)
                    for m in prm["metrics"]:
                        if m == "posterior-pairwise":
                            results[m] = {k: summary[k] for k in ("precision", "recall", "f1score")}
                            text.append(analysis.format_posterior_pairwise(summary, len(rows)))
                        elif m == "posterior-cluster":
                            results[m] = {k: summary[k] for k in ("adjRandIndex", "numClusters")}
                            results[m]["trueNumClusters"] = true_clusters
                            text.append(analysis.format_posterior_cluster(summary, len(rows), true_clusters))
                if any(m in BINDER_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    t = prm["false_link_cost"]
                    s, labels, _, _ = binder_estimate(ch, t)
                    truth = true_labels(ch.record_ids)
                    at = (int(ch.iterations[s]), int(ch.chains[s]), t)
                    for m in prm["metrics"]:
                        if m == "binder-pairwise":
                            results[m] = analysis_arrays.pairwise_metrics(labels, truth)
                            text.append(analysis.format_binder_pairwise(results[m], *at))
                        elif m == "binder-cluster":
                            results[m] = analysis_arrays.adjusted_rand_index(labels, truth)
                            text.append(analysis.format_binder_cluster(results[m], *at))
                if any(m in BINDER_SEARCH_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    t = prm["false_link_cost"]
                    start, run, _ = binder_search_estimate(ch, t, prm["max_search_rounds"])
                    truth = true_labels(ch.record_ids)
                    at = (start, run.rounds, run.converged, t, _searched_cost(t))
                    for m in prm["metrics"]:
                        if m == "binder-search-pairwise":
                            results[m] = analysis_arrays.pairwise_metrics(run.labels, truth)
                            text.append(analysis.format_binder_search_pairwise(results[m], *at))
                        elif m == "binder-search-cluster":
                            results[m] = analysis_arrays.adjusted_rand_index(run.labels, truth)
                            text.append(analysis.format_binder_search_cluster(results[m], *at))
                if any(m in VI_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    s, labels, _, losses = vi_estimate(ch)
                    truth = true_labels(ch.record_ids)
                    at = (int(ch.iterations[s]), int(ch.chains[s]), float(losses[s]))
                    for m in prm["metrics"]:
                        if m == "vi-pairwise":
                            results[m] = analysis_arrays.pairwise_metrics(labels, truth)
                            text.append(analysis.format_vi_pairwise(results[m], *at))
                        elif m == "vi-cluster":
                            results[m] = analysis_arrays.adjusted_rand_index(labels, truth)
                            text.append(analysis.format_vi_cluster(results[m], *at))
                if any(m in VI_SEARCH_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    start, run, _, exact = vi_search_estimate(ch, prm["max_search_rounds"])
                    truth = true_labels(ch.record_ids)
                    at = (start, run.rounds, run.converged, exact)
                    for m in prm["metrics"]:
                        if m == "vi-search-pairwise":
                            results[m] = analysis_arrays.pairwise_metrics(run.labels, truth)
                            text.append(analysis.format_vi_search_pairwise(results[m], *at))
                        elif m == "vi-search-cluster":
                            results[m] = analysis_arrays.adjusted_rand_index(run.labels, truth)
                            text.append(analysis.format_vi_search_cluster(results[m], *at))
                if any(m in CREDIBLE_BALL_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    center, level = prm["credible_ball_center"], prm["credible_level"]
                    labels, _, balls = credible_ball_estimate(ch, center, level, prm["false_link_cost"],
                                                              prm["max_search_rounds"])
                    truth = credible_ball_truth(labels, true_labels(ch.record_ids))
                    res = dict(center=center, level=level, samples=len(ch.samples))
                    for name, t in zip(analysis_arrays.CREDIBLE_BALL_DISTANCES, truth):
                        _, radius, inside, _ = balls[name]
                        res[name] = dict(truthDistance=t, radius=radius, truthInBall=t <= radius,
                                         samplesInBall=int(inside.sum()))
                    results["credible-ball"] = res
                    text.append(analysis.format_credible_ball(res))
                if any(m in CLERICAL_REVIEW_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    center = prm["clerical_review_center"]
                    review = clerical_review_estimate(ch, center, prm["false_link_cost"], prm["max_search_rounds"])
                    rows, res = analysis_arrays.clerical_review_evaluation(review, true_labels(ch.record_ids))
                    writers.save_clerical_review_evaluation(rows, self.output_path)
                    res["center"] = center
                    results["clerical-review"] = res
                    text.append(analysis.format_clerical_review(res))
                if any(m in CAPTURE_HISTORY_METRICS for m in prm["metrics"]):
                    ch = ch if ch is not None else self.read_chain(cut)
                    results["capture-histories"] = res = self._evaluate_capture_histories(ch, true_labels)
                    text.append(analysis.format_capture_histories(res, self.load()["cache"].file_ids))
                with open(os.path.join(self.output_path, "evaluation-results.txt"), "w") as fh:
                    fh.write("\n".join(text) + "\n")
            elif name == "link-records":
                self._link_records(prm)
            elif name == "copy-files":
                os.makedirs(prm["destination_path"], exist_ok=True)
                for fn in prm["file_names"]:
                    src = os.path.join(self.output_path, fn)
                    if os.path.exists(src):
                        dst = os.path.join(prm["destination_path"], os.path.basename(fn))
                        if os.path.exists(dst) and not prm["overwrite"]:
                            continue
                        (shutil.copytree if os.path.isdir(src) else shutil.copy)(src, dst)
                        if prm["delete_source"]:
                            (shutil.rmtree if os.path.isdir(src) else os.remove)(src)
        return results

    def read_chain(self, lower_iteration_cutoff=0):
        """The chain's samples at or after the cutoff; with several chains, all of them pooled chain-major."""
        paths = [os.path.join(dr, "linkage-chain.parquet") for dr in self.chain_dirs()]
        if self.num_chains == 1:
            return analysis_arrays.read_chain_arrays(paths[0], lower_iteration_cutoff)
        return analysis_arrays.read_pooled_chain_arrays(paths, lower_iteration_cutoff)

    def attribute_values(self):
        """Per matching attribute, the pyarrow string array of its values in value-id order (the strcmp order of the
        values, dbl_host.cpp)."""
        import pyarrow as pa

        return [pa.array([ix.value_of(v) for v in range(ix.num_values)], pa.string())
                for ix in self.load()["cache"].indexes]

    def distortion_columns(self):
        """The columns of distortion-probabilities-chain.csv: <attribute>[<file id>], attribute-major."""
        return writers.distortion_columns([a.name for a in self.matching_attributes], self.load()["cache"].file_ids)

    def read_queries(self, path):
        """(query ids, x int32[Q][A] with -1 for missing and unseen values, file int32[Q], unseen attribute names per
        query) of a query CSV with the data's record-id, matching-attribute and file-id columns."""
        import csv
        import gzip

        d = self.load()
        cache, names = d["cache"], [a.name for a in self.matching_attributes]
        wanted = [self.rec_id_attribute] + names + ([self.file_id_attribute] if self.file_id_attribute else [])
        with (gzip.open(path, "rt", newline="") if str(path).endswith(".gz") else open(path, newline="")) as fh:
            header = next(csv.reader(fh), [])
        missing = [c for c in wanted if c not in header]
        if missing:
            raise ValueError(f"the query file {path} lacks the column(s) {', '.join(missing)}")
        ids, files, cols, _ = read_csv_columns(path, self.rec_id_attribute, names, self.file_id_attribute, None,
                                               self.null_value)
        ids = [str(i) for i in ids.to_pylist()]
        if not ids:
            raise ValueError(f"the query file {path} has no records")
        if len(set(ids)) != len(ids):
            raise ValueError(f"the query file {path} has duplicate record ids")
        fpos = {f: i for i, f in enumerate(cache.file_ids)}
        file = []
        for f in files.to_pylist():
            if str(f) not in fpos:
                raise ValueError(f"the query file {path} has the file id {f!r}, which the data does not have")
            file.append(fpos[str(f)])
        Q = len(ids)
        x = np.full((Q, len(names)), -1, np.int32)
        unseen = [[] for _ in range(Q)]
        for a, (ix, col) in enumerate(zip(cache.indexes, cols)):
            for q, v in enumerate(col.to_pylist()):
                if v is None:
                    continue
                i = ix.value_idx_of(v)
                if i < 0:
                    unseen[q].append(names[a])
                else:
                    x[q, a] = i
        return ids, x, np.asarray(file, np.int32), unseen

    def _link_records(self, prm):
        """query-links.csv and query-summary.csv under outputPath: the query records of prm['query_path'] linked to
        the samples at or after the cutoff (project.link_queries)."""
        d = self.load()
        cache = d["cache"]
        ids, x, file, unseen = self.read_queries(prm["query_path"])
        t = prm["min_link_probability"]
        ch = self.read_chain(prm["lower_iteration_cutoff"])
        if not ch.samples:
            raise ValueError("link-records needs at least one sample at or after lowerIterationCutoff")
        names, values = [a.name for a in self.matching_attributes], self.attribute_values()
        A, F, R = len(names), len(cache.file_ids), ch.num_records
        theta = analysis_arrays.read_distortion_probabilities(self.chain_dirs(), ch, A, F)
        M = int(self.population_size or len(d["rec_ids"]))
        tables = analysis_arrays.QueryTables(x, file, [ix.tables() for ix in cache.indexes],
                                             [a.is_constant for a in self.matching_attributes], F)

        def samples():
            for s, v in enumerate(analysis_arrays.read_entity_values(self.chain_dirs(), ch, names, values)):
                mem, off, _ = ch.samples[s]
                yield analysis_arrays.query_sample_arrays(R, mem, off, v) + (theta[s],)

        res = link_queries(tables, samples, R, M, t)
        chain_ids = ch.record_ids.to_pylist()
        position = self._data_positions(ch)
        q, r, p = analysis_arrays.query_link_rows(res, t, position)
        writers.save_query_links([(ids[a], chain_ids[b], c) for a, b, c in zip(q.tolist(), r.tolist(), p.tolist())],
                                 self.output_path)
        first = {}
        for i, a in enumerate(q.tolist()):
            first.setdefault(a, i)  # rows go by probability descending, then data order: the first is the best
        rows = []
        for a in range(len(ids)):
            best = first.get(a)
            rows.append((ids[a], repr(float(res.new_entity_probability[a])),
                         "" if best is None else chain_ids[r[best]], "" if best is None else repr(float(p[best])),
                         repr(float(res.effective_samples[a])), ";".join(unseen[a])))
        writers.save_query_summary(rows, self.output_path)

    def _data_positions(self, ch):
        """int64[R]: the data row of each record of the chain."""
        data_pos = {r: i for i, r in enumerate(str(r) for r in self.load()["rec_ids"])}
        return np.array([data_pos[r] for r in ch.record_ids.to_pylist()], np.int64)

    def _capture_summary(self, ch, labels=None):
        """(CaptureSummary, data rows of the chain's records, their files) of the samples of ch, or of the one
        labelling labels[R] (chain record order) when given."""
        if not ch.samples:
            raise ValueError("capture-histories needs at least one sample at or after lowerIterationCutoff")
        d = self.load()
        F = len(d["cache"].file_ids)
        position = self._data_positions(ch)
        file = np.asarray(d["file"], np.int64)[position]
        if labels is None:
            H, L = capture_histories(ch, file, F)
        else:
            cc = analysis_arrays.CaptureCounts(file, F)
            cc.add_sample(analysis_arrays.canonical_clusters(labels))
            H, L = cc.read()
        return analysis_arrays.CaptureSummary(H, L, np.bincount(file, minlength=F)), position, file

    def _summarize_capture_histories(self, ch):
        """capture-histories-samples.csv, capture-histories.csv, population-size.csv, population-size-samples.csv and
        file-links.csv (records in data order) under outputPath."""
        summary, position, file = self._capture_summary(ch)
        file_ids = self.load()["cache"].file_ids
        writers.save_capture_histories(summary, ch.chains, ch.iterations, file_ids, self.output_path)
        order = np.argsort(position, kind="stable")
        ids = ch.record_ids.to_pylist()
        writers.save_file_links([ids[i] for i in order], [file_ids[f] for f in file[order]],
                                summary.link_probabilities()[order], file_ids, self.output_path)

    def _evaluate_capture_histories(self, ch, true_labels):
        """capture-histories-evaluation.csv under outputPath and the summary of analysis_arrays.capture_evaluation:
        the samples of ch against the ground truth, whose H and L are counted by the same code as one sample."""
        post, _, _ = self._capture_summary(ch)
        truth, _, _ = self._capture_summary(ch, true_labels(ch.record_ids))
        file_ids = [str(f) for f in self.load()["cache"].file_ids]
        rows_h, rows_q, res = analysis_arrays.capture_evaluation(post, truth)
        names = post.quantity_names(file_ids)
        rows = [("history[" + ",".join(f for f, b in zip(file_ids, post.histories[r[0] - 1]) if b) + "]", *r[1:])
                for r in rows_h]
        rows += [(names[r[0]], *r[1:]) for r in rows_q]
        writers.save_capture_histories_evaluation(rows, self.output_path)
        return res

    def _summarize_entity_values(self, ch, prm):
        """entity-values-clusters.csv (the center, line k = cluster k) and entity-values.csv (every cluster's most
        probable value of each attribute), from the entity values saved with the samples of ch."""
        labels = analysis_arrays.canonical_clusters(credible_ball_center(ch, prm["entity_values_center"],
                                                                         prm["false_link_cost"],
                                                                         prm["max_search_rounds"]))
        names, values = [a.name for a in self.matching_attributes], self.attribute_values()
        samples = analysis_arrays.read_entity_values(self.chain_dirs(), ch, names, values)
        modes, counts, S = entity_value_modes(labels, samples, [len(v) for v in values])
        self._save_smpc(analysis_arrays.labels_to_clusters(labels, ch.record_ids), "entity-values-clusters.csv")
        writers.save_entity_values(names, analysis_arrays.entity_value_rows(labels, modes, counts, S, values),
                                   self.output_path)

    def _evaluate_samples(self, lower_iteration_cutoff, true_labels, pooled=None):
        """Every sample at or after the cutoff against the ground truth: each chain's evaluation-samples.csv in its
        directory, and (the rows of all chains pooled chain-major, the true number of entities).  `pooled` is the
        chain already read by read_chain, reused when there is one chain."""
        rows, true_clusters = [], 0
        for dr in self.chain_dirs():
            ch = (pooled if pooled is not None and self.num_chains == 1 else
                  analysis_arrays.read_chain_arrays(os.path.join(dr, "linkage-chain.parquet"), lower_iteration_cutoff))
            truth = true_labels(ch.record_ids)
            one = analysis_arrays.sample_metrics(*posterior_metric_counts(ch, truth), truth)
            writers.save_evaluation_samples(ch.iterations, one, dr)
            rows += one
            true_clusters = len(np.unique(truth))
        return rows, true_clusters

    @staticmethod
    def _read_smpc_labels(path, record_ids):
        """Labels (aligned with record_ids) from a saved shared-most-probable-clusters.csv: one cluster per line."""
        pos = {r: i for i, r in enumerate(record_ids.to_pylist())}
        labels = np.full(len(pos), -1, np.int64)
        with open(path) as fh:
            for c, line in enumerate(fh):
                for rid in (t.strip() for t in line.split(",")):
                    if rid:
                        labels[pos[rid]] = c
        if (labels < 0).any():
            raise ValueError("shared-most-probable-clusters.csv does not cover every record of the chain")
        return labels

    def _save_smpc(self, clusters, file_name="shared-most-probable-clusters.csv"):
        """Clusters (lists of record ids) under outputPath, one per line, ids sorted and joined by ", "."""
        with open(os.path.join(self.output_path, file_name), "w") as fh:
            for c in clusters:
                fh.write(", ".join(sorted(c)) + "\n")
