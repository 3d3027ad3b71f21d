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
SUPPORTED_METRICS = SMPC_METRICS + POSTERIOR_METRICS + BINDER_METRICS + BINDER_SEARCH_METRICS + VI_METRICS
SUPPORTED_QUANTITIES = ("cluster-size-distribution", "partition-sizes", "shared-most-probable-clusters",  # :37
                        "pairwise-match-probabilities", "convergence-diagnostics", "binder-clusters",
                        "binder-search-clusters", "vi-clusters")


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
                         f"sampler={prm['sampler']}")
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
                                           resume=bool(prm.get("resume", True)), sampler=prm.get("sampler", "PCG-I"))))
            elif name == "summarize":
                q = list(prm["quantities"])
                if not q or any(x not in SUPPORTED_QUANTITIES for x in q):
                    raise ValueError(f"quantities must be one of {SUPPORTED_QUANTITIES}.")
                if "convergence-diagnostics" in q and self.num_chains < 2:
                    raise ValueError("convergence-diagnostics needs numChains >= 2.")
                # minMatchProbability: pairwise-match-probabilities.csv keeps the pairs at least this probable
                t = float(prm.get("minMatchProbability", 0.0))
                if not 0.0 <= t <= 1.0:
                    raise ValueError("minMatchProbability must be in [0, 1].")
                out.append(("summarize", dict(lower_iteration_cutoff=int(prm.get("lowerIterationCutoff", 0)),
                                              quantities=q, min_match_probability=t,
                                              false_link_cost=_false_link_cost(prm),
                                              max_search_rounds=_max_search_rounds(prm))))
            elif name == "evaluate":
                m = list(prm["metrics"])
                if not m or any(x not in SUPPORTED_METRICS for x in m):
                    raise ValueError(f"metrics must be one of {SUPPORTED_METRICS}.")
                out.append(("evaluate", dict(lower_iteration_cutoff=int(prm.get("lowerIterationCutoff", 0)), metrics=m,
                                             use_existing_smpc=bool(prm.get("useExistingSMPC", False)),
                                             false_link_cost=_false_link_cost(prm),
                                             max_search_rounds=_max_search_rounds(prm))))
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
                             self.output_path, prm["burnin_interval"], prm["thinning_interval"], sampler=prm["sampler"])
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
                with open(os.path.join(self.output_path, "evaluation-results.txt"), "w") as fh:
                    fh.write("\n".join(text) + "\n")
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
