/*
 * dblink_b200.h -- C ABI of the H100-native Gibbs-sweep engine for cleanzr/dblink's record-linkage model.
 *
 * The reference (Scala/Spark, no FFI of its own) has exactly one seam around the hot path; every entry
 * point below names the reference interface it replaces.  Paths are relative to
 * src/main/scala/com/github/cleanzr/dblink/ of cleanzr/dblink @ dc3dd0d; GU = GibbsUpdates.scala.
 *
 * Conventions (JNI/JCuda/ctypes friendly): opaque handles, plain pointers + sizes, int status
 * (0 = ok, negative = error; dbl_last_error() gives the text), no callbacks, no exceptions across the
 * boundary.  The caller owns every host buffer; the library owns every device buffer.  One context per
 * process/GPU; calls on one context are serialised by the caller.  All compute runs on the CUDA device
 * that is current when dbl_ctx_create() is called -- there is no CPU fallback.
 */
#ifndef DBLINK_B200_H
#define DBLINK_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DBL_OK 0
#define DBL_ERR_INVALID (-1)   /* bad argument (reference: require(...) -> IllegalArgumentException)            */
#define DBL_ERR_CUDA (-2)      /* CUDA runtime failure / no usable device                                       */
#define DBL_ERR_ZERO_MASS (-3) /* a categorical had zero/non-finite mass (random/IndexNonUniformDiscreteDist.scala:71-79) */
#define DBL_ERR_STATE (-4)     /* call sequence error (e.g. sweep before state upload)                          */

/* sampler = ProjectStep.scala:35,53-58 */
#define DBL_PCG_I 0            /* collapsedEntityIds=false, collapsedEntityValues=true  (default)               */
#define DBL_PCG_II 1           /* collapsedEntityIds=true,  collapsedEntityValues=true                          */
#define DBL_GIBBS 2            /* both false                                                                    */
#define DBL_GIBBS_SEQ 3        /* "Gibbs-Sequential": same conditionals as DBL_GIBBS (the reference's flag only
                                  disables its inverted index, GU:194-196)                                      */

#define DBL_MAX_ATTRS 32

/* similarity functions of an attribute (SimilarityFn.scala:50-107, plus Jaro-Winkler) */
#define DBL_SIM_CONSTANT 0     /* ConstantSimilarityFn                                                          */
#define DBL_SIM_LEVENSHTEIN 1  /* LevenshteinSimilarityFn: unit = 1 - 2 d / (|a| + |b| + d), lengths and edit
                                  distance in UTF-16 code units of the UTF-8 values, as String.length and
                                  getLevenshteinDistance count them; invalid UTF-8 is refused                  */
#define DBL_SIM_JARO_WINKLER 2 /* JaroWinklerSimilarityFn: Jaro-Winkler over bytes, prefix scale 0.1, common
                                  prefix capped at 4, no boost threshold; same truncation as Levenshtein         */

typedef struct dbl_index dbl_index;   /* AttributeIndex  (AttributeIndex.scala:39-104)                          */
typedef struct dbl_kdtree dbl_kdtree; /* KDTreePartitioner / MutableBST (partitioning/KDTreePartitioner.scala)  */
typedef struct dbl_ctx dbl_ctx;       /* State + broadcast RecordsCache/PartitionFunction (State.scala:56-68)   */

/* ---------------------------------------------------------------------------------------------------
 * Model tables.  Replaces AttributeIndex.apply (AttributeIndex.scala:107-127): value ids in sorted-string
 * order, empirical pmf, sparse exp(similarity) rows (computeSimValueIndex :219-231), normalisations
 * (computeSimNormalizations :234-245), cached base pmfs k=0..kmax (getSimNormDist :197-216,
 * RecordsCache.scala:112-113).  similarity: 0 = ConstantSimilarityFn, 1 = LevenshteinSimilarityFn
 * (SimilarityFn.scala:50-107), 2 = JaroWinklerSimilarityFn (DBL_SIM_*); any other value is DBL_ERR_INVALID.
 * For 1 and 2 a pair is in the sparse rows when exp(sim) > 1, sim = the truncation of SimilarityFn.scala:65-70
 * applied to the unit similarity.  `values` need not be sorted; `weights` are the value counts.  Values are UTF-8;
 * Levenshtein measures them in UTF-16 code units (a Java String's length and charAt), and with similarity 1 a value
 * that is not valid UTF-8 (RFC 3629: no overlong forms, no surrogates, nothing above U+10FFFF) is DBL_ERR_INVALID.
 * ------------------------------------------------------------------------------------------------- */
int dbl_index_build(dbl_index **out, const char *const *values, const double *weights, int32_t num_values,
                    int similarity, double threshold, double max_similarity, int32_t kmax);
/* Same object from pre-computed tables (phi = weight/total as in AttributeIndex.scala:114-115).  similarity 0 =
 * constant (no rows); 1 or 2 = non-constant, the rows given (both kinds give the same kind of tables); any other
 * value is DBL_ERR_INVALID. */
int dbl_index_from_tables(dbl_index **out, int32_t num_values, int similarity, const double *probs,
                          const int32_t *rowptr, const int32_t *col, const double *expsim, int32_t kmax);
void dbl_index_free(dbl_index *);
int32_t dbl_index_num_values(const dbl_index *);                 /* AttributeIndex.numValues                 */
int32_t dbl_index_nnz(const dbl_index *);
/* slots of the per-row perfect-hash tables the link kernel probes (32 = the fast instantiations; 0 = none: constant
 * attribute, or rows too long for a table) */
int32_t dbl_index_hash_slots(const dbl_index *);
/* slot codes of the 32-slot tables (num_values entries): a bijection of the value ids whose low five bits give each
 * value the same slot in every row's table; DBL_ERR_STATE when the index has none (other table sizes, or values that
 * did not colour) */
int dbl_index_slot_codes(const dbl_index *, int32_t *out);
/* 1 when dbl_index_build found the index's similarity pairs with the device kernel, 0 when the host loop did (or the
 * index is constant, or came from tables) */
int32_t dbl_index_pairs_on_device(const dbl_index *);
int32_t dbl_index_value_id(const dbl_index *, const char *value); /* valueIdxOf; -1 when absent              */
const char *dbl_index_value(const dbl_index *, int32_t value_id);
/* copies of the tables (arrays sized num_values, num_values+1, nnz, nnz); any pointer may be NULL */
int dbl_index_tables(const dbl_index *, double *phi /*probabilityOf*/, double *norm /*simNormalizationOf*/,
                     int32_t *rowptr, int32_t *col, double *expsim /*simValuesOf*/);
/* the derived tables: *kmax, then invnorm = 1/n(v), logphi, lognorm (num_values each) and the cached base pmfs pk and
 * their running sums cdf ((kmax+1) x num_values, row k = B_k); any pointer may be NULL */
int dbl_index_base_tables(const dbl_index *, int32_t *kmax, double *invnorm, double *logphi, double *lognorm, double *pk,
                          double *cdf);
double dbl_index_exp_sim(const dbl_index *, int32_t v1, int32_t v2); /* expSimOf; NaN when out of range        */
/* SimilarityFn.getSimilarity (SimilarityFn.scala:65-70, 84-96); similarity as in dbl_index_build (2 = Jaro-Winkler
 * unit similarity under the same truncation); NaN for an unknown similarity, and for similarity 1 when a or b is not
 * valid UTF-8 */
double dbl_similarity(int similarity, const char *a, const char *b, double threshold, double max_similarity);

/* ---------------------------------------------------------------------------------------------------
 * Partition function.  Replaces KDTreePartitioner.fit / getPartitionId
 * (partitioning/KDTreePartitioner.scala:37-62), MutableBST (MutableBST.scala:51-111) and the
 * DomainSplitters (DomainSplitter.scala:43-110).  y = E x A entity value ids, row-major.
 * ------------------------------------------------------------------------------------------------- */
int dbl_kdtree_fit(dbl_kdtree **out, const int32_t *y, int64_t num_entities, int32_t num_attrs,
                   int32_t num_levels, const int32_t *attr_ids, int32_t num_attr_ids);
int dbl_kdtree_from_arrays(dbl_kdtree **out, int32_t num_nodes, const int32_t *attr, const int32_t *kind,
                           const int32_t *split, const int32_t *set_ptr, const int32_t *set_val,
                           const int32_t *leaf_no);
void dbl_kdtree_free(dbl_kdtree *);
int32_t dbl_kdtree_num_nodes(const dbl_kdtree *);
int32_t dbl_kdtree_num_leaves(const dbl_kdtree *); /* PartitionFunction.numPartitions */
int32_t dbl_kdtree_set_len(const dbl_kdtree *);
int dbl_kdtree_export(const dbl_kdtree *, int32_t *attr, int32_t *kind, int32_t *split, int32_t *set_ptr,
                      int32_t *set_val, int32_t *leaf_no);
int32_t dbl_kdtree_partition_id(const dbl_kdtree *, const int32_t *entity_values); /* getPartitionId */

/* ---------------------------------------------------------------------------------------------------
 * Context = model (RecordsCache + PartitionFunction + Parameters broadcast once, State.scala:216-217,312)
 * ------------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t num_attrs;                 /* A <= DBL_MAX_ATTRS                                                */
  int32_t num_files;                 /* F (RecordsCache.fileSizes keys, sorted)                           */
  const dbl_index *const *indexes;   /* A attribute indexes                                               */
  const double *alpha;               /* A: distortionPrior alpha (BetaShapeParameters, package.scala:164) */
  const double *beta;                /* A                                                                 */
  const dbl_kdtree *tree;            /* NULL = a single block                                             */
  uint64_t seed;                     /* dblink.randomSeed                                                 */
  int32_t rank, world_size;          /* block shard owned by this context: blocks b with owner[b]==rank   */
} dbl_model_desc;

/* The CUDA device of the contexts the calling thread creates next (cudaSetDevice), and how many there are: for
 * hosts without CUDA bindings of their own (one JVM driving several GPUs, one thread per context). */
int dbl_set_device(int32_t device);
int32_t dbl_device_count(void);
int dbl_ctx_create(dbl_ctx **out, const dbl_model_desc *desc);
void dbl_ctx_destroy(dbl_ctx *);
const char *dbl_last_error(const dbl_ctx *); /* never NULL; "" when no error */

/* Install / replace the partition function (PartitionFunction.fit happens on the *initial entity values*,
 * State.scala:309-312, so the usual order is: create the context with tree = NULL, dbl_state_init,
 * dbl_state_download(y), dbl_kdtree_fit, dbl_set_partitioner).  The tree is copied to the device; the
 * caller keeps ownership.  NULL = a single block.  If a state is present it is re-partitioned. */
int dbl_set_partitioner(dbl_ctx *, const dbl_kdtree *tree);
int32_t dbl_num_partitions(const dbl_ctx *);

/* Deterministic initial state, State.deterministic (State.scala:205-334): one entity per record (or
 * population_size entities), values copied from the records, missing values drawn from phi, z = (x>=0 &
 * x!=y), theta = prior mean (DistortionProbs.scala:33-43).  x = R x A value ids (-1 missing,
 * RecordsCache.scala:127-130), file = R file ids in [0,F).  population_size <= 0 means R. */
int dbl_state_init(dbl_ctx *, int64_t num_records, const int32_t *x, const int32_t *file,
                   int64_t population_size);
/* Arbitrary state (resume; State.read, State.scala:160-193).  z = R x A bytes, link = R global entity ids,
 * y = E x A value ids, theta = A x F (host).  x, file, z, link, y may be host OR device pointers (unified
 * addressing decides): a multi-GPU caller can stage slices and all-gather them on the device first.
 * x = file = NULL keeps the records the context already holds (they never change along a chain: the reference
 * broadcasts its RecordsCache once); R and E must then be those of the state being replaced. */
int dbl_state_upload(dbl_ctx *, int64_t num_records, int64_t num_entities, const int32_t *x, const int32_t *file,
                     const uint8_t *z, const int32_t *link, const int32_t *y, const double *theta,
                     int64_t iteration);
/* Full state back to the host (State.save, State.scala:122-150); any pointer may be NULL. */
int dbl_state_download(dbl_ctx *, uint8_t *z, int32_t *link, int32_t *y, double *theta, int32_t *block_of_entity);
int64_t dbl_num_records(const dbl_ctx *);  /* of one chain */
int64_t dbl_num_entities(const dbl_ctx *); /* of one chain */
int64_t dbl_iteration(const dbl_ctx *);

/* ---------------------------------------------------------------------------------------------------
 * Batched chains: K >= 1 independent chains of the model in one context, swept together (one launch sequence per
 * sweep for all of them).  Chain k draws with Philox key seeds[k] and chain-local ids, so chain k is bit-equal to a
 * one-chain context created with seed seeds[k] and given the same partition function.  Layout is chain-major: chain k
 * owns records [kR, (k+1)R), entities [kE, (k+1)E), blocks [kB, (k+1)B) (B = leaves of the one tree all chains
 * share).  x and file are ONE copy of the records (R rows, host memory); the context replicates them.
 *   dbl_chains_init      State.deterministic for every chain (population_size <= 0 means R)
 *   dbl_chains_upload    resume: z (K R x A), link (K R, chain-LOCAL entity ids in [0, E)), y (K E x A), theta
 *                        (K x A x F), all chain-major, host memory
 *   dbl_chains_download  every chain at once, in the same layout; block_of_entity = leaf id in [0, B); any pointer
 *                        may be NULL
 *   dbl_chain_summary    dbl_summary of chain `chain` (agg_dist / theta A x F, rec_dist A + 1)
 * On a context holding K > 1 chains dbl_num_records / dbl_num_entities give one chain's R and E,
 * dbl_num_partitions gives K B, dbl_link_mass returns K R totals (chain-major); dbl_sweep, dbl_sweep_async, dbl_sync,
 * the link and graph modes and dbl_link_kernel work unchanged.  A zero-mass categorical in any chain abandons the
 * sweep for every chain (they share one iteration counter).  The calls that read or drive one chain
 * (dbl_state_download, dbl_links_download, dbl_summary, dbl_state_hash, the block-by-block API and the multi-GPU calls)
 * give DBL_ERR_STATE; dbl_state_init / dbl_state_upload turn the context back into a one-chain context.
 * DBL_ERR_INVALID: num_chains < 1, seeds NULL or not distinct, num_chains = 1 with seeds[0] other than the model's seed, a sharded context (world_size > 1), a file id outside
 * [0, F), a link outside its chain, K R or K E beyond 2^31 - 1.
 * ------------------------------------------------------------------------------------------------- */
int dbl_chains_init(dbl_ctx *, int32_t num_chains, const uint64_t *seeds, int64_t num_records, const int32_t *x,
                    const int32_t *file, int64_t population_size);
int dbl_chains_upload(dbl_ctx *, int32_t num_chains, const uint64_t *seeds, int64_t num_records,
                      int64_t num_entities, const int32_t *x, const int32_t *file, const uint8_t *z,
                      const int32_t *link, const int32_t *y, const double *theta, int64_t iteration);
int32_t dbl_num_chains(const dbl_ctx *);
int dbl_chains_download(dbl_ctx *, uint8_t *z, int32_t *link, int32_t *y, double *theta, int32_t *block_of_entity);

/* n_sweeps applications of the Markov transition operator State.nextState (State.scala:78-99):
 * updateDistProbs (GU:305-320) -> updatePartitions/updatePartition (GU:124-211: link draw per record
 * GU:363-466, entity values GU:731-755, distortions GU:324-359, new partition ids GU:206) ->
 * updateSummaryVariables (GU:219-301).  Everything runs on the device, the A x F Beta draws included; the host waits
 * once, at the end of the call.  Works on sharded contexts as well (after dbl_comm_import, see below). */
int dbl_sweep(dbl_ctx *, int sampler, int32_t n_sweeps);

/* The same transition one k-d-tree block at a time, mirroring the reference's per-partition task
 * GibbsUpdates.updatePartition (GU:156-211), for call-for-call comparison with a CPU chain:
 *   dbl_block_sweep_begin   updateDistProbs (GU:305-320): theta for the new iteration; block membership is frozen
 *   dbl_update_block        link draws, entity values, distortions and new partition ids of ONE block (each block
 *                           exactly once per sweep, in any order); rows of other blocks are not touched
 *   dbl_block_sweep_end     the shuffle by new partition id (GU:144) + updateSummaryVariables (GU:219-301)
 * begin + every block + end leaves exactly the state dbl_sweep(ctx, sampler, 1) leaves.  Unsharded contexts only. */
int dbl_block_sweep_begin(dbl_ctx *, int sampler);
int dbl_update_block(dbl_ctx *, int32_t block_id);
int dbl_block_sweep_end(dbl_ctx *);

/* Linkage structure for linkage-chain.parquet (State.getLinkageStructure, State.scala:102-112): record ->
 * entity links and each entity's current partition id. */
int dbl_links_download(dbl_ctx *, int32_t *link_out /*R*/, int32_t *block_of_entity_out /*E*/);

/* SummaryVars (package.scala:116-119) + what DiagnosticsWriter prints (DiagnosticsWriter.scala:39-72). */
typedef struct {
  int64_t iteration;
  int64_t num_isolates;
  double log_likelihood;
  int64_t pairs_scored; /* (record, candidate) pairs visited by link kernels since ctx creation: the block's entity
                           count per record in the dense kernels, the length of the posting list walked in the pruned one */
} dbl_summary_head;
int dbl_summary(dbl_ctx *, dbl_summary_head *head, int64_t *agg_dist /*A*F*/, int64_t *rec_dist /*A+1*/,
                double *theta /*A*F*/);
int dbl_chain_summary(dbl_ctx *, int32_t chain, dbl_summary_head *head, int64_t *agg_dist /*A*F*/,
                      int64_t *rec_dist /*A+1*/, double *theta /*A*F*/);

/* n sweeps enqueued on the context's stream without waiting for them (dbl_sweep = dbl_sweep_async + dbl_sync).
 * Nothing in a sweep needs the host: theta is drawn on the device, sizes are read from device memory, the exchange
 * of a sharded context is peer to peer.  dbl_sync waits, refreshes what dbl_summary / dbl_iteration report and
 * returns the status of the batch.  A sweep that meets a categorical without mass is ABANDONED: the state, theta
 * and the iteration are those before that sweep, later sweeps of the batch are skipped, DBL_ERR_ZERO_MASS is
 * returned (the reference fails the task and no new state exists, IndexNonUniformDiscreteDist.scala:78-79). */
int dbl_sweep_async(dbl_ctx *, int sampler, int32_t n_sweeps);
int dbl_sync(dbl_ctx *);

/* Order-independent fingerprint of the rows this context owns: hash_out[0] over (entity id, values), hash_out[1]
 * over (record id, link, distortion bits).  Sums over ranks (mod 2^64) identify the global state for any number of
 * ranks and any block placement. */
int dbl_state_hash(dbl_ctx *, uint64_t *hash_out /*2*/);

/* ---------------------------------------------------------------------------------------------------
 * Multi-GPU: one context per rank/GPU (dbl_model_desc.rank / world_size), blocks sharded over ranks.  Replaces
 * the one-task-per-partition fan-out (GU:137), the shuffle `.partitionBy(partitioner)` (GU:144), the broadcast of
 * theta (State.scala:84) and the summary accumulators (SummaryAccumulators.scala:54-63).  Every rank initialises
 * the same replicated state (dbl_state_init / dbl_state_upload, dbl_set_partitioner), then dbl_set_block_owners
 * carves out its shard.  Draws are keyed by global ids, so the chain is identical for any number of ranks.
 *
 * Data plane (a) -- peer to peer, inside the library, no host in the sweep:
 *   dbl_comm_export   allocates this rank's communication buffer and describes it in a DBL_COMM_BLOB_BYTES blob
 *                     (CUDA IPC handle); the host layer all-gathers the blobs with whatever it has (sockets, MPI,
 *                     torch.distributed, Spark's driver) -- this is the only thing it ever moves
 *   dbl_comm_import   maps every peer's buffer over NVLink / NVSwitch
 *   dbl_sweep / dbl_sweep_async then run the whole transition on the device: clusters whose new block belongs to
 *   another rank are written straight into that rank's receive buffer by the kernel that finds them, the partial
 *   summaries go into a slot of every peer, one flag barrier per sweep, theta is drawn redundantly on every rank.
 *   Block -> rank placement is re-evaluated on the device every `period` sweeps (dbl_set_rebalance) from the
 *   global block sizes with the LPT rule of partitioning/LPTScheduler.scala:57-76; re-placed blocks migrate as
 *   ordinary cluster messages.
 * Data plane (b) -- host-mediated (no peer access, several nodes): per sweep
 *   dbl_sweep_begin        theta | global summary, links, entity values, distortions of the owned shard; counts of
 *                          entity / record messages for every destination rank
 *   dbl_exchange_pack      messages into caller-provided DEVICE buffers, concatenated by destination rank:
 *                          entity message = 1 + A int32 words [e, y_0..y_{A-1}], record message = 3 words
 *                          [r, e, z bit mask]; the host moves them with one all-to-all (NCCL) each
 *   dbl_exchange_unpack    apply what was received
 *   dbl_partial_summary -> all-reduce on the host (with an error flag) -> dbl_sweep_end(global summary)
 * ------------------------------------------------------------------------------------------------- */
int dbl_set_block_owners(dbl_ctx *, const int32_t *owner_of_block /* numPartitions entries in [0, world); NULL =
                                                                      the table already on the device */);
int dbl_block_owners(dbl_ctx *, int32_t *owner_of_block_out);  /* current table (the device-side LPT may change it) */
#define DBL_COMM_BLOB_BYTES 192
int dbl_comm_export(dbl_ctx *, void *blob_out /* DBL_COMM_BLOB_BYTES */);
int dbl_comm_import(dbl_ctx *, const void *blobs /* world * DBL_COMM_BLOB_BYTES, in rank order */, int32_t world);
/* period = 0 switches the re-placement off; threshold = current makespan / LPT makespan above which the LPT table is
 * adopted (default: every 16 sweeps, 1.03) */
int dbl_set_rebalance(dbl_ctx *, int32_t period, double threshold);
/* cluster messages this rank sent in the last sweep collected by dbl_sync, placements adopted so far */
int dbl_last_exchange(dbl_ctx *, int64_t *ent_msgs, int64_t *rec_msgs, int64_t *replacements);
int dbl_sweep_begin(dbl_ctx *, int sampler, int64_t *ent_msgs_per_dest /*world*/, int64_t *rec_msgs_per_dest /*world*/);
int dbl_exchange_pack(dbl_ctx *, void *ent_buf_dev, void *rec_buf_dev);
int dbl_exchange_unpack(dbl_ctx *, const void *ent_buf_dev, int64_t n_ent_msgs, const void *rec_buf_dev,
                        int64_t n_rec_msgs);
int32_t dbl_summary_words(const dbl_ctx *); /* A*F + (A+1) + 2 */
int dbl_partial_summary(dbl_ctx *, int64_t *counts /*dbl_summary_words*/, double *loglik_without_prior);
int dbl_sweep_end(dbl_ctx *, const int64_t *global_counts, double global_loglik, int32_t failed_somewhere);
/* the rows this rank owns (zeros elsewhere) into caller-provided DEVICE buffers: y int32[E*A], block int32[E],
 * link int32[R], z uint8[R*A]; summing them over ranks (all-reduce) gives the full state on every rank */
int dbl_export_owned_dev(dbl_ctx *, void *y_dev, void *block_dev, void *link_dev, void *z_dev);
/* only the rows this rank owns, compacted, to the HOST: ids + rows (buffers sized for E / R rows); together the
 * ranks' rows are the state (State.save of a distributed state, State.scala:122-150) */
int dbl_download_owned(dbl_ctx *, int64_t *n_ent, int32_t *ent_ids, int32_t *y, int32_t *block_of_entity,
                       int64_t *n_rec, int32_t *rec_ids, int32_t *link, uint8_t *z);
/* which entities / records this rank currently owns (host byte arrays of E and R entries) */
int dbl_owned_masks(dbl_ctx *, uint8_t *ent_owned, uint8_t *rec_owned);

/* ---------------------------------------------------------------------------------------------------
 * Posterior summary.  Replaces LinkageChain.mostProbableClusters / sharedMostProbableClusters
 * (LinkageChain.scala:52-95): the shared most probable clusters (sMPC) of a chain, on the device that is current
 * when dbl_posterior_create() is called (dbl_set_device).  Samples are fed one at a time as cluster[R], an int32 in
 * [0, R) for every record (records with equal values share a cluster); the object keeps one 64-bit signature per
 * (record, sample) -- sig = mix64(wrapping sum of mix64(r) over the cluster ^ mix64(cluster size)), splitmix64's
 * finaliser -- in an R x max_samples device matrix.
 *   dbl_posterior_add_sample  cluster may be a host or a device pointer (ready when the call is made); a label
 *                             outside [0, R) or a sample beyond max_samples gives DBL_ERR_INVALID and adds nothing
 *   dbl_posterior_smpc        per record the signature it carries most often (ties: the one seen in the earliest
 *                             sample) and its frequency count / S (freq_out); records grouped by that signature, each
 *                             labelled by the smallest record index of its group (labels_out); either may be NULL;
 *                             DBL_ERR_STATE before the first sample
 * DBL_ERR_CUDA: no device, or the signature matrix (8 R max_samples bytes) does not fit on it.
 * ------------------------------------------------------------------------------------------------- */
typedef struct dbl_posterior dbl_posterior;
int dbl_posterior_create(dbl_posterior **out, int64_t num_records, int32_t max_samples);
void dbl_posterior_free(dbl_posterior *);
int dbl_posterior_add_sample(dbl_posterior *, const int32_t *cluster /* R, host or device */);
int32_t dbl_posterior_num_samples(const dbl_posterior *);
int dbl_posterior_smpc(dbl_posterior *, int32_t *labels_out /* R, may be NULL */, double *freq_out /* R, may be NULL */);

/* ---------------------------------------------------------------------------------------------------
 * Posterior pairwise match probabilities: for every unordered pair of records {a, b} that share a cluster in at least
 * one sample, count(a, b) = the number of samples in which they do (the probability is count / S), on the device that
 * is current when dbl_pairs_create() is called.  Samples are fed one at a time as cluster[R], as for dbl_posterior_*.
 * The object holds a sorted table of (first << 32 | second, int32 count) over the distinct pairs seen so far, at most
 * max_pairs of them (12 bytes each, twice: the table and the one the next sample merges into; the buffers grow on
 * demand, nothing is allocated up front for the cap).
 *   dbl_pairs_add_sample  cluster may be a host or a device pointer (ready when the call is made); the sample's pairs
 *                         (sum over its clusters of k(k-1)/2, counted in int64) are generated, radix-sorted and merged
 *                         into the table.  DBL_ERR_INVALID, adding nothing: a label outside [0, R); a sample whose pairs
 *                         alone exceed max_pairs (checked before anything is allocated for them); a sample whose pairs,
 *                         together with those already held, exceed max_pairs distinct pairs; S reaching INT32_MAX
 *   dbl_pairs_count       the number of held pairs with count >= min_count
 *   dbl_pairs_read        those pairs, in ascending (first, second) order, first < second (record indices), with
 *                         their counts; the three arrays (dbl_pairs_count entries) may be host or device pointers
 *   dbl_pairs_score_sample  any labelling cluster[R] (host or device pointer, as for add_sample) against the held
 *                         table: *num_pairs_out = n, the number of record pairs it puts together, and *count_sum_out =
 *                         K, the sum of count(a, b) over those pairs (a pair the table does not hold counts 0), both
 *                         int64.  The table and S do not change.  DBL_ERR_INVALID: a label outside [0, R), or n alone
 *                         exceeding max_pairs (checked before anything is allocated for the pairs).  With
 *                         t = the cost of a false link and 1 - t that of a missed link, the posterior expected Binder
 *                         loss of the labelling is ((1 - t) C + t S n - K) / S, C = sum of all held counts.
 *   dbl_pairs_binder_search  single-record moves from the labelling start[R] (host or device pointer, any labels in
 *                         [0, R)) while they lower J = a S n - b K, i.e. the expected Binder loss at t = a / b, against
 *                         the held table.  A round: every record's least (dJ, destination) over its partners' clusters
 *                         and, out of a cluster of two or more, a singleton (destination -1; a cluster counts as its
 *                         smallest record index), proposed if dJ < 0; a proposal is applied if it holds the least
 *                         (dJ, record) among the proposals touching each cluster it touches (its source, and its
 *                         destination unless a singleton).  The search stops when no record proposes (*converged_out
 *                         = 1) or after max_rounds rounds (0).  Per round moves / dn / dK (host, max_rounds entries
 *                         each, *rounds_out written): the moves applied and the sums of their changes of n and K.
 *                         labels_out (R, host or device): each record labelled by the smallest record index of its
 *                         cluster.  *n_out = sum over clusters of C(size, 2), *K_out = the sum of the held counts of the
 *                         pairs it links, so a result is never refused by max_pairs.  The table and S do not change.
 *                         DBL_ERR_INVALID: a NULL pointer, max_rounds < 1, not 0 <= a <= b <= 2^16, S R >= 2^44, a
 *                         start label outside [0, R).  Memory: 48 bytes per held pair and 56 per record, for the call.
 *   count / read / score_sample / binder_search before the first sample give DBL_ERR_STATE.
 * DBL_ERR_INVALID: num_records or max_pairs outside [1, 2^31 - 1].  DBL_ERR_CUDA: no device, or an allocation that
 * fails (the held table and the sample count stay as they were).
 * ------------------------------------------------------------------------------------------------- */
typedef struct dbl_pairs dbl_pairs;
int dbl_pairs_create(dbl_pairs **out, int64_t num_records, int64_t max_pairs);
void dbl_pairs_free(dbl_pairs *);
int dbl_pairs_add_sample(dbl_pairs *, const int32_t *cluster /* R, host or device */);
int32_t dbl_pairs_num_samples(const dbl_pairs *);
int dbl_pairs_count(dbl_pairs *, int32_t min_count, int64_t *n_out);
int dbl_pairs_read(dbl_pairs *, int32_t min_count, int32_t *first, int32_t *second, int32_t *count);
int dbl_pairs_score_sample(dbl_pairs *, const int32_t *cluster /* R, host or device */, int64_t *num_pairs_out,
                           int64_t *count_sum_out);
int dbl_pairs_binder_search(dbl_pairs *, int64_t a, int64_t b, const int32_t *start /* R, host or device */,
                            int32_t max_rounds, int32_t *labels_out /* R */, int32_t *rounds_out,
                            int32_t *converged_out, int64_t *moves, int64_t *dn, int64_t *dK /* max_rounds each, host */,
                            int64_t *n_out, int64_t *K_out);

/* ---------------------------------------------------------------------------------------------------
 * Every posterior sample against the ground truth: per sample, the integer counts its pairwise precision / recall /
 * F1 and adjusted Rand index are made of, on the device that is current when dbl_eval_create() is called.  truth is
 * one int32 label in [0, R) per record (records with equal labels are one true entity), host or device, uploaded once;
 * samples are fed one at a time as cluster[R], as for dbl_posterior_*.  Per sample, counted in int64:
 *   tp            sum over the cells (sample cluster, true entity) of C(n, 2): the pairs both put together
 *   pred_pairs    sum over the sample's clusters of C(size, 2)
 *   num_clusters  the number of distinct labels of the sample
 * The true pairs sum C(true size, 2) and C(R, 2) do not depend on the sample and are left to the caller.
 *   dbl_eval_add_sample  cluster may be a host or a device pointer (ready when the call is made); a label outside
 *                        [0, R) or a sample beyond max_samples gives DBL_ERR_INVALID and adds nothing
 *   dbl_eval_read        the S counts of each kind, in the order the samples were added, into host arrays;
 *                        DBL_ERR_STATE before the first sample
 * DBL_ERR_INVALID: num_records outside [1, 2^31 - 1], max_samples < 1, truth NULL or a true label outside [0, R) (no
 * object is created).  DBL_ERR_CUDA: no device, or an allocation that fails (24 bytes per record, and the
 * temporary storage of a radix sort of R 64-bit keys).
 * ------------------------------------------------------------------------------------------------- */
typedef struct dbl_eval dbl_eval;
int dbl_eval_create(dbl_eval **out, int64_t num_records, const int32_t *truth /* R, host or device */,
                    int32_t max_samples);
void dbl_eval_free(dbl_eval *);
int dbl_eval_add_sample(dbl_eval *, const int32_t *cluster /* R, host or device */);
int32_t dbl_eval_num_samples(const dbl_eval *);
int dbl_eval_read(dbl_eval *, int64_t *tp, int64_t *pred_pairs, int64_t *num_clusters /* S entries each, host */);

/* ---------------------------------------------------------------------------------------------------
 * Cell histograms for the posterior expected variation of information (VI) of every sample, on the device that is
 * current when dbl_vi_create() is called.  Samples are fed one at a time as cluster[R], as for dbl_posterior_*, and
 * held as an int32 [max_samples][R] device matrix allocated up front (4 R max_samples bytes).  For held samples
 * C_0 .. C_{S-1} and n >= 2:
 *   G[t][n] = sum over s != t of the number of cells (non-empty intersections of a cluster of C_t and one of C_s) of
 *             exactly n records, int64; G[t][0] = G[t][1] = 0.
 * With g_s[n] = the clusters of n records in sample s and D_t[n] = (S - 2) g_t[n] + sum_s g_s[n] - 2 G[t][n], the
 * expected VI of sample t against the S samples is sum over n of D_t[n] n log2 n / (R S); that sum is the caller's.
 *   dbl_vi_add_sample  cluster may be a host or a device pointer (ready when the call is made); a label outside
 *                      [0, R) or a sample beyond max_samples gives DBL_ERR_INVALID and adds nothing.  The handle
 *                      tracks M, the largest cluster of any held sample.
 *   dbl_vi_set_batch_keys  the keys one sort may hold (default 2^26; at least the records of one sample's clusters of
 *                      two or more are always taken together); DBL_ERR_INVALID below 1.  It bounds the memory of
 *                      dbl_vi_cross and does not change its result.
 *   dbl_vi_cross       G as S x width int64 (row-major, host or device pointer).  DBL_ERR_INVALID: width < M + 1 or
 *                      S width 8 bytes past INT64_MAX; DBL_ERR_STATE before the first sample.  Memory, the call's own
 *                      and freed on return: 8 S width bytes, 12 per record, and two buffers of 8 bytes per sorted key
 *                      (at most max(batch keys, R)) plus the sort's temporary storage.  The held samples do not
 *                      change, whatever the outcome.  The work is S (S - 1) / 2 sorts of the records in clusters of
 *                      two or more, batched over samples.
 * DBL_ERR_INVALID: num_records outside [1, 2^31 - 1] or max_samples < 1.  DBL_ERR_CUDA: no device, or the held label
 * matrix (or a buffer of dbl_vi_cross) does not fit on it.
 * ------------------------------------------------------------------------------------------------- */
typedef struct dbl_vi dbl_vi;
int dbl_vi_create(dbl_vi **out, int64_t num_records, int32_t max_samples);
void dbl_vi_free(dbl_vi *);
int dbl_vi_add_sample(dbl_vi *, const int32_t *cluster /* R, host or device */);
int32_t dbl_vi_num_samples(const dbl_vi *);
int dbl_vi_set_batch_keys(dbl_vi *, int64_t max_keys);
int dbl_vi_cross(dbl_vi *, int64_t width, int64_t *G_out /* S x width */);

/* The protocol functions of the theta draw (DESIGN.md 4.5), exposed so that they can be checked without a GPU:
 * log / exp built from individually rounded binary64 operations, and updateDistProbs (GU:305-320) itself. */
double dbl_det_log(double x);
double dbl_det_exp(double x);
int dbl_draw_theta(int32_t num_attrs, int32_t num_files, const double *alpha, const double *beta, uint64_t seed,
                   const int64_t *agg_dist /*A*F*/, const int64_t *file_sizes /*F*/, int64_t iteration,
                   double *theta_out /*A*F*/);

/* count of kernels launched by this context since creation (bench.py's gpu_launches) */
int64_t dbl_kernel_launches(const dbl_ctx *);
/* Link-kernel selection: 0 = automatic (PCG-II: TMA-staged dense kernel; PCG-I/Gibbs: scoring pruned through a
 * per-sweep inverted index), 1 = always the generic fallback kernel, 2 = dense TMA kernels for every sampler.
 * All produce identical draws; this exists so tests can cover every kernel. */
int dbl_set_link_mode(dbl_ctx *, int mode);
/* which link kernel a sweep with this sampler launches: 0 generic fallback, 1 dense must-match kernel, 2 index-pruned
 * kernel, 3 k_link_pcg2 (+4: byte-packed constants, +8: 32-slot tables known at compile time) and, for k_link_pcg2
 * only, the tile format it reads (+16: 16-bit non-constant values, +32: slot codes instead of value ids, +64: the two
 * records of a warp share paired key tables, +128: two records per warp).  A model that falls back to the generic
 * kernel runs an order of magnitude slower: benches and tests assert what they expect. */
int dbl_link_kernel(const dbl_ctx *, int sampler);
/* Link-mass capture (checking only; off by default, free when off): with on != 0 every link kernel stores the total
 * mass of each record's categorical -- the sum of its protocol weights over the block, the number the draw tests for
 * zero / non-finite -- into a device array of R entries, from the link phase of the sweep that ran last.  Toggling
 * drops captured sweep graphs.  dbl_link_mass copies the R totals (record order) to the host; DBL_ERR_STATE before a
 * sweep with the capture on.  Both return DBL_ERR_STATE on a sharded context. */
int dbl_set_link_mass_capture(dbl_ctx *, int on);
int dbl_link_mass(dbl_ctx *, double *mass_out /*R*/);
/* How dbl_sweep / dbl_sweep_async enqueue several sweeps: 0 = automatic (problems small enough to be bound by kernel
 * launches, and the index-pruned samplers at every size, replay a captured CUDA graph of one sweep), 1 = every sweep
 * enqueued kernel by kernel (and timed phase by phase, dbl_link_kernel_ms / dbl_phase_ms), 2 = graphs whenever
 * possible.  Same chain either way. */
int dbl_set_graph_mode(dbl_ctx *, int mode);
/* CUDA-event time (ms) of the last dbl_sweep call, first operation to last operation on the context's stream */
double dbl_last_sweep_ms(const dbl_ctx *);
/* CUDA-event time (ms) spent in the link-scoring kernel since the last call; resets the accumulator */
double dbl_link_kernel_ms(dbl_ctx *, int64_t *launches);
/* CUDA-event time (ms) of the eagerly enqueued sweeps since the last call, by phase: out4 = {link update GU:186-199,
 * entity values + distortions + partial summary GU:201-210, exchange of moved clusters + summary reduction GU:144 (0
 * on one rank), re-layout by block}; returns the number of sweeps summed; resets the accumulators */
int64_t dbl_phase_ms(dbl_ctx *, double *out4);
const char *dbl_version(void);

#ifdef __cplusplus
}
#endif
#endif
