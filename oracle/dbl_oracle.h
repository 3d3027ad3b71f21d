/*
 * dbl_oracle.h -- CPU ORACLE for the dblink Gibbs-sweep hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This directory is a from-scratch CPU restatement of the algorithm in the reference
 * (cleanzr/dblink @ dc3dd0d, paths relative to src/main/scala/com/github/cleanzr/dblink/).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * import, link or execute anything in here.  The product (dblink_b200/) never does.
 *
 * PARITY STATUS
 *   - table level (similarity fn, value ids, phi, sparse expSim rows, normalisations, theta init):
 *     PINNED by the reference's own golden vectors (SimilarityFnTest.scala:46-74,
 *     AttributeIndexTest.scala:38-99, DistortionProbsTest.scala:30-33) -- see tests/test_oracle_golden.py.
 *   - the sweep itself (every update* in GibbsUpdates.scala): "parity unpinned" by the reference --
 *     it has no sampler test, its RNG is commons-math3 MersenneTwister + alias tables + Scala HashMap
 *     iteration order + Spark shuffle order, and no JVM exists in this environment.  The oracle
 *     therefore (i) restates each conditional literally (orc_ref_* functions, citing GU lines), and
 *     (ii) defines the counter-based draw protocol (Philox4x32-10 + fixed-order inverse-CDF draws)
 *     that the CUDA path must reproduce bit-for-bit; tests check (ii) against (i) distributionally
 *     and against brute-force posterior enumeration.
 */
#ifndef DBL_ORACLE_H
#define DBL_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum { ORC_PCG_I = 0, ORC_PCG_II = 1, ORC_GIBBS = 2, ORC_GIBBS_SEQ = 3 };
enum { ORC_PHASE_INIT = 0, ORC_PHASE_THETA = 1, ORC_PHASE_LINK = 2, ORC_PHASE_VALUE = 3, ORC_PHASE_DIST = 4 };

typedef struct orc_index orc_index;
typedef struct orc_kdtree orc_kdtree;
typedef struct orc_model orc_model;
typedef struct orc_state orc_state;

/* ---- RNG protocol ---- */
void orc_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]);
void orc_uniform2(uint64_t seed, uint32_t phase, uint32_t iter, uint32_t id, uint32_t sub, double u[2]);

/* ---- similarity function (SimilarityFn.scala:61-98) ----
   UTF-8 values measured in UTF-16 code units, as the reference's Java Strings are; -1 / NaN when a value is not
   valid UTF-8 */
int orc_levenshtein(const char *a, const char *b);
double orc_lev_similarity(const char *a, const char *b, double threshold, double max_sim);

/* ---- attribute index (AttributeIndex.scala:107-245); NULL when a non-constant index has invalid UTF-8 ---- */
orc_index *orc_index_build(const char *const *values, const double *weights, int V, int is_const,
                           double threshold, double max_sim, int kmax);
void orc_index_free(orc_index *);
int orc_index_num_values(const orc_index *);
int orc_index_is_const(const orc_index *);
int orc_index_value_id(const orc_index *, const char *value); /* -1 when absent */
const char *orc_index_value(const orc_index *, int v);
const double *orc_index_phi(const orc_index *);
const double *orc_index_norm(const orc_index *);
const double *orc_index_invnorm(const orc_index *);
const int32_t *orc_index_rowptr(const orc_index *);
const int32_t *orc_index_col(const orc_index *);
const double *orc_index_expsim(const orc_index *);
int orc_index_nnz(const orc_index *);
int orc_index_kmax(const orc_index *);
const double *orc_index_pk(const orc_index *);  /* (kmax+1) x V normalised base pmfs */
const double *orc_index_cdf(const orc_index *); /* (kmax+1) x V cumulative */
double orc_index_exp_sim_of(const orc_index *, int v1, int v2);
/* build directly from tables (for synthetic models whose tables were made elsewhere) */
orc_index *orc_index_from_tables(int V, int is_const, const double *phi, const int32_t *rowptr,
                                 const int32_t *col, const double *expsim, int kmax);

/* ---- k-d tree partition function (partitioning/ dir) ---- */
orc_kdtree *orc_kdtree_fit(const int32_t *y, int64_t E, int A, int num_levels, const int32_t *attr_ids,
                           int n_attr_ids);
orc_kdtree *orc_kdtree_from_arrays(int n_nodes, const int32_t *attr, const int32_t *kind,
                                   const int32_t *split, const int32_t *set_ptr, const int32_t *set_val,
                                   const int32_t *leaf_no);
void orc_kdtree_free(orc_kdtree *);
int orc_kdtree_num_nodes(const orc_kdtree *);
int orc_kdtree_num_leaves(const orc_kdtree *);
int orc_kdtree_set_len(const orc_kdtree *);
void orc_kdtree_export(const orc_kdtree *, int32_t *attr, int32_t *kind, int32_t *split, int32_t *set_ptr,
                       int32_t *set_val, int32_t *leaf_no);
int orc_kdtree_leaf(const orc_kdtree *, const int32_t *yrow);

/* ---- model + state ---- */
orc_model *orc_model_create(int A, int F, orc_index *const *idx, const double *alpha, const double *beta,
                            const orc_kdtree *tree, uint64_t seed);
void orc_model_free(orc_model *);

/* deterministic initial state (State.scala:205-334) */
orc_state *orc_state_init(const orc_model *, int64_t R, const int32_t *x, const int32_t *file, int64_t pop_size);
/* arbitrary state */
orc_state *orc_state_from_arrays(const orc_model *, int64_t R, int64_t E, const int32_t *x, const int32_t *file,
                                 const uint8_t *z, const int32_t *link, const int32_t *y, const double *theta,
                                 int64_t iteration);
void orc_state_free(orc_state *);
int64_t orc_state_R(const orc_state *);
int64_t orc_state_E(const orc_state *);
int64_t orc_state_iteration(const orc_state *);
const int32_t *orc_state_y(const orc_state *);
const int32_t *orc_state_link(const orc_state *);
const uint8_t *orc_state_z(const orc_state *);
const int32_t *orc_state_block(const orc_state *);
const double *orc_state_theta(const orc_state *);
/* R entries: the total mass of each record's link categorical (the sum orc_draw_index tests for zero / non-finite)
   in the link phase of the last sweep; zeros before the first sweep */
const double *orc_state_last_link_mass(const orc_state *);
/* summary (GibbsUpdates.scala:219-301) -- recomputed on demand */
typedef struct {
  int64_t iteration;
  int64_t num_isolates;
  double log_likelihood;
} orc_summary_head;
void orc_state_summary(const orc_state *, orc_summary_head *head, int64_t *agg_dist /*A*F*/, int64_t *rec_dist /*A+1*/);

/* one sweep: theta -> links -> values -> distortions -> blocks (State.scala:78-99). 0 on success. */
int orc_state_sweep(orc_state *, int sampler);
/* bench only: phases (3)-(5) and the summary pass of one sweep from the current links on nthreads threads;
   sec[0..3] = wall seconds of values / distortions / re-route / summary */
void orc_rest_of_sweep_timed(orc_state *, int sampler, int nthreads, double *sec);
/* protocol log / exp of the theta draw (DESIGN.md 4.5) */
double orc_det_log(double x);
double orc_det_exp(double x);
/* only the theta draw for the next iteration (GU:305-320) */
void orc_draw_theta(const orc_model *, const int64_t *agg_dist, const int64_t *file_sizes, uint32_t iter,
                    double *theta_out);

/* ---- protocol primitives exposed for unit tests ---- */
int orc_draw_index(const double *w, int64_t n, double u, int *status, double *total_out);
int orc_invcdf(const double *cdf, int V, double u);
/* literal restatements of the reference's per-record link weights (GU:363-466) for distribution tests */
void orc_ref_link_weights(const orc_state *, int64_t r, int sampler, const int32_t *cand, int64_t n_cand,
                          double *w_out);
/* protocol link weights for the same candidates (differ from the literal ones by a record-constant factor) */
void orc_link_weights(const orc_state *, int64_t r, int sampler, const int32_t *cand, int64_t n_cand,
                      double *w_out);
/* literal restatement of the collapsed / non-collapsed entity-value conditional over the whole domain
   (GU:576-599 + 534-570, GU:605-646 + 702-727, GU:652-698): pmf_out has V_a entries, normalised. */
void orc_ref_value_pmf(const orc_state *, int64_t e, int a, int sampler, double *pmf_out);
/* protocol draw of one entity value given explicit uniforms */
int orc_value_draw(const orc_state *, int64_t e, int a, int sampler, double u0, double u1);
/* literal distortion probability (GU:324-359): P(z=1) */
double orc_ref_dist_prob(const orc_state *, int64_t r, int a);

/* alias sampler (random/AliasSampler.scala:49-118): returns 0 ok, -1 invalid weight, -2 zero mass */
int orc_alias_build(const double *w, int n, double *prob_out, int32_t *alias_out);
int orc_alias_sample(const double *prob, const int32_t *alias, int n, double u);

#ifdef __cplusplus
}
#endif
#endif
