/* private layouts shared by dbl_oracle.c and dbl_refsweep.c (oracle = test infrastructure only) */
#ifndef DBL_ORACLE_PRIV_H
#define DBL_ORACLE_PRIV_H
#include "dbl_oracle.h"

struct orc_index {
  int V, is_const, kmax;
  char **values;   /* sorted */
  double *probs;   /* weight/total (AttributeIndex.scala:114-115)                  */
  double *phi;     /* probabilityOf: probs renormalised by DiscreteDist (:122,:136) */
  double *norm;    /* simNormalizationOf = 1/sum (:234-245)                         */
  double *invnorm; /* the sum itself                                                */
  int32_t *rowptr, *col;
  double *expsim;
  double *pk, *cdf; /* (kmax+1) x V */
};

struct orc_kdtree {
  int n_nodes, n_leaves;
  int32_t *attr;    /* -1: leaf or absent */
  int32_t *kind;    /* 0 range (right iff value > split), 1 set (right iff value in set) */
  int32_t *split;
  int32_t *set_ptr; /* n_nodes + 1 */
  int32_t *set_val; /* sorted ascending per node */
  int32_t *leaf_no; /* MutableBST node.value; -1 for absent nodes */
  int set_len, set_cap;
};

struct orc_model {
  int A, F;
  orc_index **idx; /* borrowed */
  double *alpha, *beta;
  const orc_kdtree *tree; /* borrowed */
  uint64_t seed;
};

struct orc_state {
  const orc_model *m;
  int64_t R, E, iteration;
  int32_t *x, *file, *link, *y, *blk;
  uint8_t *z;
  double *theta;       /* A x F */
  double *mass;        /* R: total mass of each record's link categorical in the last sweep (0 before any) */
  int64_t *file_sizes; /* F */
};

#endif
