// Device half of libdblink_b200: the Gibbs sweep of dblink's record-linkage model on one H100.
//
// Reference (cleanzr/dblink @ dc3dd0d, src/main/scala/com/github/cleanzr/dblink/, GU = GibbsUpdates.scala):
//   State.nextState State.scala:78-99 -> updatePartition GU:156-211
//     link draw per record        GU:363-395 (PCG-II), GU:399-466 (PCG-I / Gibbs, dense form)   -> k_link
//     entity values per (e, attr) GU:534-599, 605-646, 702-755                                   -> k_values
//     distortions per (r, attr)   GU:324-359                                                     -> k_dist
//     new partition id            GU:206, partitioning/MutableBST.scala:61-79                    -> k_entity_post
//   updateSummaryVariables GU:219-301                                   -> k_entity_post / k_dist accumulators
//   the shuffle GU:144                                                  -> relayout() (sort by block id)
//
// Numerics: all likelihood arithmetic is IEEE binary64 with no FMA contraction (-fmad=false) so that the
// CPU oracle (oracle/dbl_oracle.c, -ffp-contract=off) reproduces every draw bit for bit.  Draw protocol:
// DESIGN.md section 4.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cub/cub.cuh>
#include <map>
#include <optional>
#include <string>
#include <vector>

#include "dbl_internal.h"
#define DBL_ENGINE_TU 1
#include "dbl_link.cuh"
#include "dbl_link_pcg2.cuh"
#include "dbl_scale.h"

#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      ctx->set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                       \
      return DBL_ERR_CUDA;                                                                      \
    }                                                                                           \
  } while (0)

// ---------------------------------------------------------------------------------------------------
// device-side model
// ---------------------------------------------------------------------------------------------------
struct TreeDev {
  int n_nodes;
  const int *attr, *kind, *split, *set_ptr, *set_val, *leaf_no;
};

// ---------------------------------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ int invcdf(const double *cdf, int V, double u) {
  int lo = 0, hi = V;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] > u) hi = mid; else lo = mid + 1;
  }
  return lo < V ? lo : V - 1;
}

__device__ __forceinline__ int tree_leaf(const TreeDev &t, const int *yrow) {
  int node = 0;
  while (node < t.n_nodes && t.attr[node] >= 0) {
    const int v = yrow[t.attr[node]];
    bool right;
    if (t.kind[node]) {
      int lo = t.set_ptr[node], hi = t.set_ptr[node + 1] - 1;
      right = false;
      while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const int s = t.set_val[mid];
        if (s == v) { right = true; break; }
        if (s < v) lo = mid + 1; else hi = mid - 1;
      }
    } else {
      right = v > t.split[node];
    }
    node = right ? 2 * node + 2 : 2 * node + 1;
  }
  return t.leaf_no[node];
}

// ---------------------------------------------------------------------------------------------------
// Row kernels run in one of two modes:
//   prefix mode (inside a sweep): rows = the first ctl[CTL_OWNED_*] entries of ent_sorted / rec_sorted, i.e. exactly
//     the entities / records of the blocks this rank owns, counted on the DEVICE (no host round trip); grid-stride,
//     so the launch does not depend on the count; the kernel returns at once when the sweep was abandoned;
//   mask mode (state set-up): every row whose ownership byte is set.
// ---------------------------------------------------------------------------------------------------
struct RowSet {
  const long long *ctl;         // control block
  const int *sorted;            // ent_sorted / rec_sorted (prefix mode) or nullptr (mask mode)
  const unsigned char *owned;   // ownership bytes (mask mode)
  int64_t n_all;                // E or R
  int count_word;               // CTL_OWNED_ENT / CTL_OWNED_REC
  __device__ __forceinline__ int64_t count() const { return sorted ? (int64_t)ctl[count_word] : n_all; }
  __device__ __forceinline__ int64_t row(int64_t i) const {
    if (sorted) return sorted[i];
    return owned[i] ? i : -1;
  }
  __device__ __forceinline__ bool dead() const { return sorted && sweep_dead(ctl); }
};
#define GRID_STRIDE(i, n) \
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (n); i += (int64_t)gridDim.x * blockDim.x)

// one atomic per distinct key among the active lanes of the warp
__device__ __forceinline__ void warp_hist_add(unsigned long long *bins, int key) {
  const unsigned peers = __match_any_sync(__activemask(), key);
  if ((__ffs(peers) - 1) == (int)(threadIdx.x & 31)) atomicAdd(&bins[key], (unsigned long long)__popc(peers));
}

// ---------------------------------------------------------------------------------------------------
// k_entity_post: per entity N(e) = prod_{non-const a} n_a(y_a); new block id (GU:206); entity part of the
// summary: isolates (GU:267-269) and sum_a log phi_a(y_a) (GU:234-237, 271-274); sizes of the new blocks (the
// input of the block -> rank placement, partitioning/LPTScheduler.scala:57-76).
// part = partial summary words of this rank: [A*F] aggDist, [A+1] recDist, isolates, log-likelihood (f64 bits),
// [P] entities per block, [P] records per block.
// ---------------------------------------------------------------------------------------------------
struct EntPostParams {
  RowSet rows;
  ChainMap cm;  // batched chains: block k * blocks + leaf; summary words of chain k at iso_slot + k / ll_slot + k
  int A;
  const int *y;
  const AttrDev *attrs;
  TreeDev tree;
  double *entN;
  int *blk;
  const int *ent_rec_ptr;  // nullptr: no summary
  unsigned long long *part;
  int iso_slot, ll_slot, blk_slot;  // blk_slot < 0: no block histogram
};
// batched chains: a thread's rows come in chain order (rows are sorted by block, blocks are chain-major), so it adds
// its sums into the chain's words whenever the chain changes, and once at the end
__device__ __forceinline__ void flush_chain_sums(unsigned long long *part, int iso_slot, int ll_slot, int &iso,
                                                 double &ll) {
  if (ll != 0.0) atomicAdd(reinterpret_cast<double *>(&part[ll_slot]), ll);
  if (iso) atomicAdd(&part[iso_slot], (unsigned long long)iso);
  ll = 0.0;
  iso = 0;
}
__device__ __forceinline__ void flush_chain_ll(unsigned long long *part, int ll_slot, double &ll) {
  if (ll != 0.0) atomicAdd(reinterpret_cast<double *>(&part[ll_slot]), ll);
  ll = 0.0;
}
__global__ void __launch_bounds__(256) k_entity_post(EntPostParams p) {
  if (p.rows.dead()) return;
  const int64_t n = p.rows.count();
  double ll = 0.0;
  int iso = 0, ck = 0;  // ck: the chain ll / iso belong to (batched chains)
  GRID_STRIDE(i, n) {
    const int64_t e = p.rows.row(i);
    if (e < 0) continue;
    int kb = 0;  // first block of the entity's chain
    if (p.cm.K > 1) {
      const int k = (int)e / p.cm.ents;
      if (k != ck && p.ent_rec_ptr) flush_chain_sums(p.part, p.iso_slot + ck, p.ll_slot + ck, iso, ll);
      ck = k;
      kb = k * p.cm.blocks;
    }
    const int *ye = p.y + e * p.A;
    double nn = 1.0;
    for (int a = 0; a < p.A; ++a) {
      const AttrDev &at = p.attrs[a];
      const int v = ye[a];
      if (!at.is_const) nn = nn * at.norm[v];
      ll += at.logphi[v];
    }
    p.entN[e] = nn;
    const int b = kb + (p.tree.n_nodes > 0 ? tree_leaf(p.tree, ye) : 0);
    p.blk[e] = b;
    if (p.ent_rec_ptr) {
      iso += (p.ent_rec_ptr[e] == p.ent_rec_ptr[e + 1]);
      if (p.blk_slot >= 0) warp_hist_add(p.part + p.blk_slot, b);
    }
  }
  if (p.ent_rec_ptr && p.cm.K > 1) {
    flush_chain_sums(p.part, p.iso_slot + ck, p.ll_slot + ck, iso, ll);
  } else if (p.ent_rec_ptr) {
    typedef cub::BlockReduce<double, 256> BR;
    typedef cub::BlockReduce<int, 256> BRI;
    __shared__ typename BR::TempStorage t1;
    __shared__ typename BRI::TempStorage t2;
    const double s = BR(t1).Sum(ll);
    const int c = BRI(t2).Sum(iso);
    if (threadIdx.x == 0) {
      if (s != 0.0) atomicAdd(reinterpret_cast<double *>(&p.part[p.ll_slot]), s);
      if (c) atomicAdd(&p.part[p.iso_slot], (unsigned long long)c);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// layout ("re-partitioning", replaces the shuffle GU:144): entities and records grouped by block
// ---------------------------------------------------------------------------------------------------
__global__ void k_iota(int64_t n, int *out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (int)i;
}
__global__ void k_hist(int64_t n, const int *__restrict__ key, int *__restrict__ cnt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) atomicAdd(&cnt[key[i]], 1);
}
// sort keys; entities / records this rank does not own go to the dummy slot (block P, entity E)
// Records are grouped by block and, within a block, by a static cost class, so that the records sharing a CTA of
// the link kernel (and its tile ring) advance at the same pace.  The order of records inside a block has no effect
// on the draws (every record has its own counter-based stream).
constexpr int REC_CLASS_BITS = 8;
// cost class of a record (x is static), from hq = the expected number of similar-but-different candidate values per
// 32-candidate step (how often the warp takes the rare multiply: equal or similar value), from the empirical value
// frequencies, in 0..63: a record without a missing non-constant value has class hq; one with a missing non-constant
// value 64 + 4 lo + hq / 16, lo = the first non-constant attribute it misses (0..15, in attribute order), so that
// records missing the same attribute share work items of k_link_pcg2 (whose producer stages the 1/n(y) columns the
// work item's records miss, and whose warps skip the probes of an attribute both their records miss).
__global__ void k_rec_class(int64_t R, int A, const AttrDev *__restrict__ attrs, const int *__restrict__ x,
                            unsigned char *__restrict__ cls) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int lo = -1;
  double h = 0.0;
  for (int a = 0, q = 0; a < A; ++a) {
    const AttrDev &at = attrs[a];
    if (at.is_const) continue;
    const int xv = x[r * A + a];
    if (xv < 0) { if (lo < 0) lo = q; ++q; continue; }
    ++q;
    h += at.probs[xv];  // an equal value takes the same path as a similar one (one table, see k_link_pcg2)
    for (int i = at.rowptr[xv]; i < at.rowptr[xv + 1]; ++i)
      if (at.col[i] != xv) h += at.probs[at.col[i]];
  }
  const int hq = min(63, (int)(h * 32.0 * 8.0));
  cls[r] = (unsigned char)(lo < 0 ? hq : 64 | (min(lo, 15) << 2) | (hq >> 4));
}
// block sort keys of the entities and of the records in one launch
__global__ void k_block_keys(int64_t E, int64_t R, const int *__restrict__ blk, const int *__restrict__ link,
                             const unsigned char *__restrict__ ent_owned, const unsigned char *__restrict__ rec_owned,
                             const unsigned char *__restrict__ rec_class, int P, int *__restrict__ ent_key,
                             int *__restrict__ rec_key) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < E) ent_key[i] = ent_owned[i] ? blk[i] : P;
  if (i < R)  // not owned: behind every owned key, spread over the class bits (see sentinel_spread)
    rec_key[i] = rec_owned[i] ? ((blk[link[i]] << REC_CLASS_BITS) | rec_class[i])
                              : ((P << REC_CLASS_BITS) | (int)(i & ((1 << REC_CLASS_BITS) - 1)));
}
__global__ void k_rec_link_keys(int64_t R, const int *__restrict__ link, const unsigned char *__restrict__ rec_owned,
                                int E, int spread, int *__restrict__ key) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < R) key[r] = rec_owned[r] ? link[r] : E + (int)(r % spread);  // see sentinel_spread
}
// the same inside a sweep, fused with the commit of the link draws: the link kernels wrote them to newlink; they
// become the state only if no categorical of the sweep was without mass (the reference fails the task and no new
// state exists, IndexNonUniformDiscreteDist.scala:78-79)
__global__ void k_commit_link_keys(int64_t R, const long long *__restrict__ ctl, const int *__restrict__ newlink,
                                   int *__restrict__ link, const unsigned char *__restrict__ rec_owned, int E,
                                   int spread, int *__restrict__ key) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int l = link[r];
  const bool own = rec_owned[r];
  if (own && !sweep_dead(ctl)) {
    l = newlink[r];
    link[r] = l;
  }
  key[r] = own ? l : E + (int)(r % spread);  // see sentinel_spread
}
// offsets from sorted keys: ptr[k] = first position whose key is >= k, for k = 0..n_keys (keys beyond the data
// point at n).  One pass over the sorted array; replaces an atomic histogram + scan.
__device__ __forceinline__ void segment_ptr_at(int64_t i, int64_t n, int n_keys, const int *__restrict__ sorted_key,
                                               int *__restrict__ ptr, int shift) {
  if (i > n) return;
  const int cur = (i < n) ? min(sorted_key[i] >> shift, n_keys) : n_keys;
  const int prev = (i > 0) ? min(sorted_key[i - 1] >> shift, n_keys) : -1;
  for (int k = prev + 1; k <= cur; ++k) ptr[k] = (int)i;
}
__global__ void k_segment_ptr(int64_t n, int n_keys, const int *__restrict__ sorted_key, int *__restrict__ ptr,
                              int shift = 0) {
  segment_ptr_at((int64_t)blockIdx.x * blockDim.x + threadIdx.x, n, n_keys, sorted_key, ptr, shift);
}
// block offsets of the sorted entities and of the sorted records in one launch
__global__ void k_block_ptrs(int64_t E, int64_t R, int P, const int *__restrict__ blk_sorted, int *__restrict__ ent_ptr,
                             const int *__restrict__ rec_key_sorted, int *__restrict__ rec_ptr) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  segment_ptr_at(i, E, P, blk_sorted, ent_ptr, 0);
  segment_ptr_at(i, R, P, rec_key_sorted, rec_ptr, REC_CLASS_BITS);
}
// prefix sums over the P blocks (P is 2^numLevels: small); publishes the owned counts (everything before the dummy
// block) in the control block -- they size the prefix-mode row kernels of the next sweep.  As the last kernel of a
// sweep it also adopts the partial summary as the global one (single rank: adopt_nw > 0) and counts the sweep
// (finish), unless the sweep was abandoned.
__global__ void k_block_scan(int P, const int *__restrict__ ent_ptr, const int *__restrict__ rec_ptr,
                             int *__restrict__ tile_ptr, int *__restrict__ cta_ptr, int warps_per_cta,
                             int *__restrict__ cta_ptr2, int warps_per_cta2, int *__restrict__ cta_ptr3,
                             int recs_per_item3, long long *__restrict__ ctl,
                             int adopt_nw, const unsigned long long *__restrict__ part, long long *__restrict__ glob,
                             int finish) {
  const bool dead = sweep_dead(ctl);
  if (adopt_nw > 0 && !dead)
    for (int i = threadIdx.x; i < adopt_nw; i += blockDim.x) glob[i] = (long long)part[i];
  if (threadIdx.x == 0) {
    int t = 0, c = 0, c2 = 0, c3 = 0;
    for (int b = 0; b < P; ++b) {
      tile_ptr[b] = t; cta_ptr[b] = c; cta_ptr2[b] = c2; cta_ptr3[b] = c3;
      t += (ent_ptr[b + 1] - ent_ptr[b] + TE - 1) / TE;
      const int nr = rec_ptr[b + 1] - rec_ptr[b];
      c += (nr + warps_per_cta - 1) / warps_per_cta;
      c2 += (nr + warps_per_cta2 - 1) / warps_per_cta2;
      c3 += (nr + recs_per_item3 - 1) / recs_per_item3;
    }
    tile_ptr[P] = t; cta_ptr[P] = c; cta_ptr2[P] = c2; cta_ptr3[P] = c3;
    ctl[CTL_OWNED_ENT] = ent_ptr[P];
    ctl[CTL_OWNED_REC] = rec_ptr[P];
    if (finish && !dead) ctl[CTL_ITER] += 1;
  }
}
// The tiled, block-sorted copy of the entity table, one thread per tile slot (padding slots of a block's last tile are
// zeroed here: no memset of the whole table).
struct TileSrc {
  int64_t n_slots;
  int A, P;
  const int *y, *ent_sorted, *ent_ptr, *tile_ptr, *perm;
  const double *entN;
  // tile T and slot of thread i, its entity's values (nullptr: padding) and N; false past the last tile
  __device__ bool at(int64_t i, int &T, int &slot, const int *&yrow, double &N) const {
    T = (int)(i / TE);
    slot = (int)(i % TE);
    if (i >= n_slots || T >= tile_ptr[P]) return false;
    int lo = 0, hi = P;  // block of tile T: last b with tile_ptr[b] <= T
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (tile_ptr[mid] <= T) lo = mid; else hi = mid;
    }
    const int j = (T - tile_ptr[lo]) * TE + slot;
    const int64_t e = j < ent_ptr[lo + 1] - ent_ptr[lo] ? ent_sorted[ent_ptr[lo] + j] : -1;
    yrow = e >= 0 ? y + e * A : nullptr;
    N = e >= 0 ? entN[e] : 0.0;
    return true;
  }
};
// tiles of format f, NS non-constant attributes; invn (k_link_pcg2, may be null): the 1/n(y) columns of every tile,
// [tile][q][slot] (LinkParams::tile_invn), the invnorm of the entity's value of kernel-order attribute A - NS + q
// (= scinvnorm of its slot code: the columns do not depend on the format)
__global__ void k_build_entity_tiles(TileSrc s, Pcg2Format f, int NS, const AttrDev *__restrict__ attrs,
                                     int *__restrict__ tiles, double *__restrict__ invn) {
  int T, slot;
  const int *yrow;
  double N;
  if (!s.at((int64_t)blockIdx.x * blockDim.x + threadIdx.x, T, slot, yrow, N)) return;
  pcg2_store(f, s.A, NS, yrow, s.perm, attrs, tiles + (size_t)T * f.layout(s.A, NS).words(), slot, N);
  if (invn)
    for (int q = 0; q < NS; ++q) {
      const int a = s.perm[s.A - NS + q];
      invn[((size_t)T * NS + q) * TE + slot] = yrow ? attrs[a].invnorm[yrow[a]] : 0.0;
    }
}

// ---------------------------------------------------------------------------------------------------
// sweep bookkeeping on the device (the host only enqueues): theta draw, link commit, end of sweep
// ---------------------------------------------------------------------------------------------------
// updateDistProbs GU:305-320: theta[a,f] ~ Beta(alpha_a + aggDist[a,f], beta_a + N_f - aggDist[a,f]) from the GLOBAL
// summary of the previous state.  Every rank draws the same values from the same counter-based stream (replaces
// the broadcast, State.scala:84).  theta_prev keeps the old values: an abandoned sweep restores them.
// Batched chains: column f belongs to chain f / files_per_chain, which draws with its own key and its own id a * F1 + f1.
__global__ void k_theta(int A, int F, uint64_t seed, const uint64_t *__restrict__ seeds, int files_per_chain,
                        long long *__restrict__ ctl, const long long *__restrict__ glob,
                        const double *__restrict__ alpha, const double *__restrict__ beta,
                        const double *__restrict__ file_size, double *__restrict__ theta,
                        double *__restrict__ theta_prev, unsigned long long *__restrict__ part, int nw) {
  if (sweep_dead(ctl)) return;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) part[i] = 0ull;  // the partial summary of the sweep starts empty
  const uint32_t it = (uint32_t)(ctl[CTL_ITER] + 1);
  for (int i = threadIdx.x; i < A * F; i += blockDim.x) {
    const int a = i / F, f = i % F;
    theta_prev[i] = theta[i];
    uint64_t s = seed;
    uint32_t id = (uint32_t)i;
    if (seeds) {
      const int k = f / files_per_chain;
      s = seeds[k];
      id = (uint32_t)(a * files_per_chain + (f - k * files_per_chain));
    }
    theta[i] = draw_theta_one(s, it, id, alpha[a], beta[a], (double)glob[i], file_size[f]);
  }
  if (threadIdx.x == 0) { ctl[CTL_MOVED_ENT] = 0; ctl[CTL_MOVED_REC] = 0; ctl[CTL_WORK] = 0; ctl[CTL_HEAVY] = 0; }
}
// single rank: the partial summary is the global one
__global__ void k_reduce_local(int nw, const long long *__restrict__ ctl, const unsigned long long *__restrict__ part,
                               long long *__restrict__ glob) {
  if (sweep_dead(ctl)) return;
  for (int i = threadIdx.x; i < nw; i += blockDim.x) glob[i] = (long long)part[i];
}
__global__ void k_finish(long long *__restrict__ ctl) {
  if (threadIdx.x == 0 && !sweep_dead(ctl)) ctl[CTL_ITER] += 1;
}

// ---------------------------------------------------------------------------------------------------
// k_values: one thread per (entity, attribute).  updateEntityValueCollapsed GU:576-599 +
// perturbedDistYCollapsed GU:534-570 (PCG-I/II); updateEntityValue GU:605-646 + perturbedDistY GU:702-727.
// ---------------------------------------------------------------------------------------------------
// batched loads of k_values on sizes that fill the GPU (see value_update): pairs (2) beat none (1) and four at a time
// (64 registers either way: with four the spills grow)
constexpr int VALUES_UB_LARGE = 2;
struct ValParams {
  int A, F, sampler;
  uint64_t seed;
  ChainMap cm;
  RowSet rows;  // owned entities
  const AttrDev *attrs;
  const int *x, *file;
  const unsigned *zmask;
  const double *theta;
  const int *ent_rec_ptr, *rec_by_ent;
  int *y;
  long long *far_list;  // (entity, attribute) rows e * A + a whose draw k_values_rescaled makes; count in ctl[CTL_FAR]
};

struct BaseDist {
  const AttrDev *at;
  int k, sc, ez;  // sc: the uncached weights are rescaled, zk = Z_k * 2^(-512 ez)
  const double *pk, *cdf;
  double zk;
};
__device__ __forceinline__ double base_weight(const AttrDev &at, int k, int v) {
  double w = at.probs[v];
  if (!at.is_const)
    for (int i = 0; i < k; ++i) w = w * at.norm[v];
  return w;
}
// RS: the uncached weights may need rescaling (DESIGN.md section 4.7).  Never for k <= 1 (Z_0 = 1, Z_1 >= min n(v)),
// so the draws of isolated entities and single-record clusters compile without it
template <bool RS>
__device__ void base_init(BaseDist &b, const AttrDev &at, int k) {
  b.at = &at;
  if (at.is_const) k = 0;
  b.k = k;
  b.sc = 0;
  if (k <= at.kmax) {
    b.pk = at.pk + (size_t)k * at.V;
    b.cdf = at.cdf + (size_t)k * at.V;
    b.zk = 0.0;
  } else {  // beyond the cached powers (getSimNormDist cache miss, AttributeIndex.scala:199-205)
    b.pk = nullptr; b.cdf = nullptr;
    double z = 0.0;
    for (int v = 0; v < at.V; ++v) z += base_weight(at, k, v);
    if (RS) {
      b.sc = !(z >= BASE_Z_MIN);  // as base_row: the weights underflow, rescale them
      if (b.sc) z = base_z_sc(at.V, at.probs, at.norm, at.is_const, k, b.ez);
    }
    b.zk = z;
  }
}
// uncached weight of v at the scale of zk
template <bool RS>
__device__ __forceinline__ double base_w(const BaseDist &b, int v) {
  if (RS && b.sc) {
    int e;
    const double w = base_weight_sc(b.at->probs, b.at->norm, b.at->is_const, b.k, v, e);
    return sc_down(w, e - b.ez);
  }
  return base_weight(*b.at, b.k, v);
}
template <bool RS>
__device__ __forceinline__ double base_prob(const BaseDist &b, int v) {
  return b.pk ? b.pk[v] : base_w<RS>(b, v) / b.zk;
}
template <bool RS>
__device__ int base_draw(const BaseDist &b, double u) {
  if (b.cdf) return invcdf(b.cdf, b.at->V, u);
  double c = 0.0;
  for (int v = 0; v < b.at->V; ++v) {
    c += base_w<RS>(b, v) / b.zk;
    if (c > u) return v;
  }
  return b.at->V - 1;
}

// factor contributed by record r to candidate value v; false when v is outside the record's support
__device__ __forceinline__ bool g_factor(const ValParams &p, const AttrDev &at, int a, int r, bool collapsed, int v,
                                         double &g) {
  const int xr = p.x[(int64_t)r * p.A + a];
  if (at.is_const) {
    if (v != xr || !collapsed) return false;
    const double th = p.theta[a * p.F + p.file[r]];
    g = 1.0 + (1.0 / th - 1.0) / at.phi[xr];  // GU:553
    return true;
  }
  double e;
  if (!row_find(at, xr, v, e)) return false;
  if (collapsed && v == xr) {
    const double th = p.theta[a * p.F + p.file[r]];
    g = e + (1.0 / th - 1.0) / (at.phi[xr] * at.norm[xr]);  // GU:557,560
  } else {
    g = e;
  }
  return true;
}
__device__ __forceinline__ bool in_support(const ValParams &p, const AttrDev &at, int a, int r, int v) {
  const int xr = p.x[(int64_t)r * p.A + a];
  if (at.is_const) return v == xr;
  double e;
  return row_find(at, xr, v, e);
}

// the value draw of an entity with two or more linked records (first-appearance enumeration of the support, two
// passes).  Plain weights W(v) = B_k(v) (G(v) - 1); SC: every weight carried as W * 2^(512 e) (DESIGN.md section
// 4.7): t(v) = B_k(v) Z_k (G(v) - 1), the walk in units of the largest scale E, Z_k only in the mixture test.  The
// plain form returns VALUE_FAR when the total leaves the double range (G overflows for clusters of about 709 / ln g
// agreeing records, and 0 * inf is NaN where B_k(v) underflowed as well); k_values_rescaled then draws with SC.
// RS: the base distribution may be rescaled (base_init<RS>).
constexpr int VALUE_FAR = -2;
template <bool SC, bool RS>
__device__ __forceinline__ int cluster_draw(const ValParams &p, const AttrDev &at, int a, int lo, int hi, bool collapsed,
                                            const BaseDist &b, U2 u) {
  const int *rec = p.rec_by_ent;
  double total = 0.0, target = 0.0, cum = 0.0;
  int picked = -1, last_pos = -1, E = INT_MIN;
  for (int pass = 0; pass < 2; ++pass) {
    for (int i = lo; i < hi; ++i) {
      const int r = rec[i];
      const int xr = p.x[(int64_t)r * p.A + a];
      if (xr < 0) continue;
      // an earlier record with the same value has already introduced every value of this record's similarity row
      // (the usual case inside a cluster: duplicates agree): nothing new to add, and no pairwise searches
      bool repeated = false;
      for (int j = lo; j < i && !repeated; ++j) repeated = (p.x[(int64_t)rec[j] * p.A + a] == xr);
      if (repeated) continue;
      const int nv = at.is_const ? 1 : (at.rowptr[xr + 1] - at.rowptr[xr]);
      const int *vals = at.is_const ? nullptr : (at.col + at.rowptr[xr]);
      for (int q = 0; q < nv; ++q) {
        const int v = at.is_const ? xr : vals[q];
        bool seen = false;
        for (int j = lo; j < i && !seen; ++j) {
          const int rj = rec[j];
          if (p.x[(int64_t)rj * p.A + a] < 0) continue;
          seen = in_support(p, at, a, rj, v);
        }
        if (seen) continue;
        double G = 1.0;
        int eg = 0;
        for (int j = i; j < hi; ++j) {
          const int rj = rec[j];
          const int xj = p.x[(int64_t)rj * p.A + a];
          if (xj < 0) continue;
          double g;
          if (!at.is_const && xj == xr) {
            // a record observing the same value as record i (record i itself; duplicates that agree): v sits at
            // position q of that value's row, so the search of g_factor would return exactly this element
            const double ex = at.expsim[at.rowptr[xr] + q];
            if (collapsed && v == xr) {
              const double th = p.theta[a * p.F + p.file[rj]];
              g = ex + (1.0 / th - 1.0) / (at.phi[xr] * at.norm[xr]);  // GU:557,560
            } else {
              g = ex;
            }
            G = G * g;
          } else if (g_factor(p, at, a, rj, collapsed, v, g)) {
            G = G * g;
          } else {
            continue;
          }
          if (SC && G > SC_UP) { G = G * SC_DN; ++eg; }
        }
        double W;
        int ew = 0;
        if (!SC) {
          W = base_prob<RS>(b, v) * (G - 1.0);  // GU:567 / 724
        } else {  // G - 1 == G at eg > 0: 2^-512 is below half an ulp of G >= 1
          int eb;
          W = base_weight_sc(at.probs, at.norm, at.is_const, b.k, v, eb) * (eg ? G : G - 1.0);
          ew = eb + eg;
          if (pass == 1) W = sc_down(W, ew - E);
        }
        if (pass == 0) {
          if (!SC) {
            total += W;
          } else if (W > 0.0) {
            if (E == INT_MIN) E = ew;
            if (ew > E) { total = sc_down(total, E - ew); E = ew; }
            total += sc_down(W, ew - E);
          }
        } else {
          cum += W;
          if (W > 0.0) last_pos = v;
          if (picked < 0 && cum > target) picked = v;
        }
      }
    }
    if (pass == 0) {
      if (!SC && !(total <= DBL_MAX)) return VALUE_FAR;
      double mix = total;  // the plain total of the mixture test GU:593-594
      if (SC && E != INT_MIN) {
        int ez;
        mix = total / base_z_sc(at.V, at.probs, at.norm, at.is_const, b.k, ez);
        for (int d = E - ez; d > 0; --d) mix = mix * SC_UP;
        mix = sc_down(mix, E - ez);
      }
      if (u.u0 < 1.0 / (1.0 + mix)) return base_draw<RS>(b, u.u1);  // GU:593-594
      target = u.u1 * total;
    }
  }
  if (picked < 0) picked = last_pos;
  if (picked < 0) picked = base_draw<RS>(b, u.u1);
  return picked;
}

// new value of attribute a of entity e.  UB > 1: the loop over the similarity row of a single linked record fetches
// UB candidates at a time (independent loads, same sums in the same order): for problems too small to fill the GPU
// the kernel's time is the longest dependent-load chain of one thread, not throughput
template <int UB>
__device__ int value_update(const ValParams &p, uint32_t iter, int64_t e, int a) {
  const AttrDev &at = p.attrs[a];
  const bool collapsed = (p.sampler == DBL_PCG_I || p.sampler == DBL_PCG_II);
  const U2 u = chain_uniform2(p.seed, p.cm.seeds, p.cm.ents, PH_VALUE, iter, e, (uint32_t)a);
  const int lo = p.ent_rec_ptr[e], hi = p.ent_rec_ptr[e + 1];
  const int *rec = p.rec_by_ent;

  int k = 0;
  for (int i = lo; i < hi; ++i) k += (p.x[(int64_t)rec[i] * p.A + a] >= 0);
  BaseDist b;
  if (k == 0) {  // GU:588-589
    base_init<false>(b, at, 0);
    return base_draw<false>(b, u.u1);
  }
  if (!collapsed) {
    for (int i = lo; i < hi; ++i) {  // GU:619-630
      const int r = rec[i];
      const int xr = p.x[(int64_t)r * p.A + a];
      if (xr >= 0 && !((p.zmask[r] >> a) & 1u)) return xr;
    }
    if (at.is_const) {  // GU:633-634
      base_init<false>(b, at, 0);
      return base_draw<false>(b, u.u1);
    }
  }
  double total = 0.0, target = 0.0, cum = 0.0;
  int picked = -1, last_pos = -1;
  if (hi - lo == 1) {
    base_init<false>(b, at, k);  // GU:584-586
    // one linked record (most entities): the candidate values are the record's own similarity row, so the factors
    // come straight from that row (no searches, no first-appearance check); same operations as the general path
    const int r = rec[lo];
    const int xr = p.x[(int64_t)r * p.A + a];  // observed (k == 1)
    const int q0 = at.is_const ? 0 : at.rowptr[xr];
    const int nv = at.is_const ? 1 : (at.rowptr[xr + 1] - q0);
    double extra = 0.0;  // what the collapsed update adds to the factor of v == x (GU:553,557,560)
    if (collapsed) {
      const double th = p.theta[a * p.F + p.file[r]];
      extra = at.is_const ? (1.0 / th - 1.0) / at.phi[xr] : (1.0 / th - 1.0) / (at.phi[xr] * at.norm[xr]);
    }
    auto weight = [&](int q, int &v) -> double {
      double G = 1.0;
      if (at.is_const) {
        v = xr;
        if (collapsed) G = G * (1.0 + extra);
      } else {
        v = at.col[q0 + q];
        const double ex = at.expsim[q0 + q];
        G = G * ((collapsed && v == xr) ? ex + extra : ex);
      }
      return base_prob<false>(b, v) * (G - 1.0);  // GU:567 / 724
    };
    if constexpr (UB > 1) {
      // same weights, same order of the sums; the loads of UB consecutive candidates are issued together
      auto batch = [&](int q, int (&v)[UB], double (&W)[UB]) {
        double ex[UB], bp[UB];
#pragma unroll
        for (int i = 0; i < UB; ++i) {
          const int qq = min(q + i, nv - 1);
          v[i] = at.is_const ? xr : at.col[q0 + qq];
          ex[i] = at.is_const ? 0.0 : at.expsim[q0 + qq];
        }
#pragma unroll
        for (int i = 0; i < UB; ++i) bp[i] = base_prob<false>(b, v[i]);
#pragma unroll
        for (int i = 0; i < UB; ++i) {
          double G = 1.0;
          if (at.is_const) { if (collapsed) G = G * (1.0 + extra); }
          else G = G * ((collapsed && v[i] == xr) ? ex[i] + extra : ex[i]);
          W[i] = bp[i] * (G - 1.0);
        }
      };
      for (int q = 0; q < nv; q += UB) {
        int v[UB];
        double W[UB];
        batch(q, v, W);
#pragma unroll
        for (int i = 0; i < UB; ++i)
          if (q + i < nv) total += W[i];
      }
      if (u.u0 < 1.0 / (1.0 + total)) return base_draw<false>(b, u.u1);  // GU:593-594
      target = u.u1 * total;
      for (int q = 0; q < nv && picked < 0; q += UB) {
        int v[UB];
        double W[UB];
        batch(q, v, W);
#pragma unroll
        for (int i = 0; i < UB; ++i)
          if (q + i < nv && picked < 0) {
            cum += W[i];
            if (W[i] > 0.0) last_pos = v[i];
            if (cum > target) picked = v[i];
          }
      }
    } else {
      for (int q = 0; q < nv; ++q) {
        int v;
        total += weight(q, v);
      }
      if (u.u0 < 1.0 / (1.0 + total)) return base_draw<false>(b, u.u1);  // GU:593-594
      target = u.u1 * total;
      for (int q = 0; q < nv && picked < 0; ++q) {
        int v;
        const double W = weight(q, v);
        cum += W;
        if (W > 0.0) last_pos = v;
        if (cum > target) picked = v;
      }
    }
    if (picked < 0) picked = last_pos;
    if (picked < 0) picked = base_draw<false>(b, u.u1);
    return picked;
  }
  base_init<false>(b, at, k);  // GU:584-586
  if (!b.pk && !(b.zk >= BASE_Z_MIN)) return VALUE_FAR;  // the uncached weights underflow: k_values_rescaled draws
  return cluster_draw<false, false>(p, at, a, lo, hi, collapsed, b, u);  // VALUE_FAR: k_values_rescaled draws
}

template <int UB>
__global__ void __launch_bounds__(128) k_values(ValParams p) {
  if (p.rows.dead()) return;
  const uint32_t iter = (uint32_t)(p.rows.ctl[CTL_ITER] + 1);
  const int64_t n = p.rows.count() * p.A;
  GRID_STRIDE(t, n) {  // entity-major: the attributes of an entity share its record list (an attribute-major mapping,
                       // one code path per warp, was measured slower at 1M)
    const int64_t e = p.rows.row(t / p.A);
    if (e < 0) continue;
    const int a = (int)(t % p.A);
    const int v = value_update<UB>(p, iter, e, a);
    if (v != VALUE_FAR) p.y[e * p.A + a] = v;
    else p.far_list[atomicAdd(reinterpret_cast<unsigned long long *>(const_cast<long long *>(p.rows.ctl) + CTL_FAR), 1ull)] = e * p.A + a;
  }
}
// the draws k_values left because their weights leave the double range, as the oracle makes them: rescaled base
// weights, then rescaled perturbation weights when the plain total still leaves the range.  A kernel of
// its own: inlined into k_values the rare rescaled draw costs every common draw registers.  One CTA: usually there
// are none, and the kernel reads the count, zeroes it and returns.
__global__ void __launch_bounds__(128) k_values_rescaled(ValParams p) {
  long long *cnt = const_cast<long long *>(p.rows.ctl) + CTL_FAR;
  const int64_t n = *cnt;
  if (!p.rows.dead()) {
    const uint32_t iter = (uint32_t)(p.rows.ctl[CTL_ITER] + 1);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const int64_t e = p.far_list[i] / p.A;
      const int a = (int)(p.far_list[i] % p.A);
      const AttrDev &at = p.attrs[a];
      const U2 u = chain_uniform2(p.seed, p.cm.seeds, p.cm.ents, PH_VALUE, iter, e, (uint32_t)a);
      const int lo = p.ent_rec_ptr[e], hi = p.ent_rec_ptr[e + 1];
      int k = 0;
      for (int j = lo; j < hi; ++j) k += (p.x[(int64_t)p.rec_by_ent[j] * p.A + a] >= 0);
      const bool collapsed = (p.sampler == DBL_PCG_I || p.sampler == DBL_PCG_II);
      BaseDist b;
      base_init<true>(b, at, k);
      const int v = cluster_draw<false, true>(p, at, a, lo, hi, collapsed, b, u);
      p.y[e * p.A + a] = v != VALUE_FAR ? v : cluster_draw<true, true>(p, at, a, lo, hi, collapsed, b, u);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *cnt = 0;
}

// ---------------------------------------------------------------------------------------------------
// k_dist: one thread per record.  updateDistortions GU:324-359 with the new y, fused with the record part
// of updateSummaryVariables GU:239-266.  draw = 0 only accumulates the summary of the current state.
// ---------------------------------------------------------------------------------------------------
struct DistParams {
  int A, F, draw;
  uint64_t seed;
  ChainMap cm;  // batched chains: recDist of chain k at [A*F + k(A+1)], log-likelihood at ll_slot + k
  RowSet rows;  // owned records
  const AttrDev *attrs;
  const int *x, *file, *link, *y, *blk;
  unsigned *zmask;
  const double *theta;
  unsigned long long *part;  // [A*F] aggDist, then [A+1] recDist, ...
  int ll_slot, blk_slot;     // blk_slot < 0: no block histogram
};

__global__ void __launch_bounds__(256) k_dist(DistParams p) {
  if (p.rows.dead()) return;
  const uint32_t iter = (uint32_t)(p.rows.ctl[CTL_ITER] + 1);
  const int64_t n = p.rows.count();
  double ll = 0.0;
  int ck = 0;  // the chain ll belongs to (batched chains)
  GRID_STRIDE(i, n) {
    const int64_t r = p.rows.row(i);
    if (r < 0) continue;
    int rd = 0;  // first recDist word of the record's chain
    if (p.cm.K > 1) {
      const int k = (int)r / p.cm.recs;
      if (k != ck) flush_chain_ll(p.part, p.ll_slot + ck, ll);
      ck = k;
      rd = k * (p.A + 1);
    }
    const int f = p.file[r];
    const int e = p.link[r];
    const int *ye = p.y + (int64_t)e * p.A;
    unsigned zm = p.zmask[r];
    int nd = 0;
    for (int a = 0; a < p.A; ++a) {
      const AttrDev &at = p.attrs[a];
      const int xv = p.x[r * p.A + a];
      const int yv = ye[a];
      bool z;
      if (p.draw) {
        const double th = p.theta[a * p.F + f];
        if (xv < 0) {
          const U2 u = chain_uniform2(p.seed, p.cm.seeds, p.cm.recs, PH_DIST, iter, r, (uint32_t)a);
          z = u.u0 < th;  // GU:331-334
        } else if (xv != yv) {
          z = true;  // GU:352-354
        } else {
          const U2 u = chain_uniform2(p.seed, p.cm.seeds, p.cm.recs, PH_DIST, iter, r, (uint32_t)a);
          double pr1 = th * at.phi[xv];
          if (!at.is_const) {
            pr1 = pr1 * at.norm[xv];
            pr1 = pr1 * at.diag[xv];
          }
          const double pr0 = 1.0 - th;
          const double den = pr1 + pr0;
          const double pz = (den != 0.0) ? pr1 / den : 0.0;  // GU:349-350
          z = u.u0 < pz;
        }
        zm = z ? (zm | (1u << a)) : (zm & ~(1u << a));
      } else {
        z = (zm >> a) & 1u;
      }
      if (z) {
        ++nd;
        atomicAdd(&p.part[a * p.F + f], 1ull);  // GU:246
        if (xv >= 0) {                          // GU:248-258
          ll += at.logphi[xv];
          if (!at.is_const) {
            ll += at.lognorm[yv];
            double ex;
            if (row_find(at, xv, yv, ex)) ll += log(ex);
          }
        }
      }
    }
    if (p.draw) p.zmask[r] = zm;
    warp_hist_add(p.part + p.A * p.F, rd + nd);  // GU:265
    if (p.blk_slot >= 0) warp_hist_add(p.part + p.blk_slot, p.blk[e]);
  }
  if (p.cm.K > 1) {
    flush_chain_ll(p.part, p.ll_slot + ck, ll);
    return;
  }
  typedef cub::BlockReduce<double, 256> BR;
  __shared__ typename BR::TempStorage tmp;
  const double s = BR(tmp).Sum(ll);
  if (threadIdx.x == 0 && s != 0.0) atomicAdd(reinterpret_cast<double *>(&p.part[p.ll_slot]), s);
}

// ---------------------------------------------------------------------------------------------------
// k_init_state: State.deterministic (State.scala:253-301) -- entity e copies record e (if any), missing
// values drawn from phi; record r links to entity r mod E; z = (x>=0 && x!=y).
// ---------------------------------------------------------------------------------------------------
// batched chains: entity e of chain k copies record e of chain k
__global__ void k_init_entities(int64_t E, int64_t R, int A, uint64_t seed, ChainMap cm, const AttrDev *__restrict__ attrs,
                                const int *__restrict__ x, int *__restrict__ y) {
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid >= E * A) return;
  const int64_t e = tid / A;
  const int a = (int)(tid % A);
  int64_t el = e, rec = e, rc = R;  // chain-local entity id, the record it copies, records of its chain
  if (cm.K > 1) {
    const int64_t k = e / cm.ents;
    el = e - k * cm.ents;
    rec = k * cm.recs + el;
    rc = cm.recs;
  }
  int v = (el < rc) ? x[rec * A + a] : -1;
  if (v < 0) {
    const U2 u = chain_uniform2(seed, cm.seeds, cm.ents, PH_INIT, 0u, e, (uint32_t)a);
    v = invcdf(attrs[a].cdf, attrs[a].V, u.u1);
  }
  y[tid] = v;
}
__global__ void k_init_records(int64_t E, int64_t R, int A, ChainMap cm, const int *__restrict__ x,
                               const int *__restrict__ y, int *__restrict__ link, unsigned *__restrict__ zmask) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int64_t e = r % E;
  if (cm.K > 1) {  // record r of chain k links to entity (r mod E1) of chain k
    const int64_t k = r / cm.recs;
    e = k * cm.ents + (r - k * cm.recs) % cm.ents;
  }
  link[r] = (int)e;
  unsigned zm = 0;
  for (int a = 0; a < A; ++a) {
    const int xv = x[r * A + a];
    if (xv >= 0 && xv != y[e * A + a]) zm |= 1u << a;
  }
  zmask[r] = zm;
}
// range checks of an uploaded state (the reference would fail with ArrayIndexOutOfBounds / require):
// bit 0 record value id, bit 1 file id, bit 2 link, bit 3 entity value id
__global__ void k_validate(int64_t R, int64_t E, int A, int F, const AttrDev *__restrict__ attrs,
                           const int *__restrict__ x, const int *__restrict__ file, const int *__restrict__ link,
                           const int *__restrict__ y, int *__restrict__ flag) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int bad = 0;
  if (i < R) {
    for (int a = 0; a < A; ++a) {
      const int v = x[i * A + a];
      if (v < -1 || v >= attrs[a].V) bad |= 1;
    }
    if (file[i] < 0 || file[i] >= F) bad |= 2;
    if (link && (link[i] < 0 || link[i] >= E)) bad |= 4;
  }
  if (y && i < E)
    for (int a = 0; a < A; ++a) {
      const int v = y[i * A + a];
      if (v < 0 || v >= attrs[a].V) bad |= 8;
    }
  if (i < R)  // not an error: bit 4 = the record misses a non-constant value (k_link_pcg2 needs the 1/n(y) columns)
    for (int a = 0; a < A; ++a)
      if (!attrs[a].is_const && x[i * A + a] == -1) bad |= 16;
  bad = __reduce_or_sync(FULL, bad);  // one atomic per warp (blocks of 256 threads: whole warps)
  if (bad && (threadIdx.x & 31) == 0) atomicOr(flag, bad);
}
__global__ void k_pack_z(int64_t R, int A, const uint8_t *__restrict__ z, unsigned *__restrict__ zmask) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  unsigned zm = 0;
  for (int a = 0; a < A; ++a) zm |= (z[r * A + a] ? 1u : 0u) << a;
  zmask[r] = zm;
}
__global__ void k_unpack_z(int64_t R, int A, const unsigned *__restrict__ zmask, uint8_t *__restrict__ z) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const unsigned zm = zmask[r];
  for (int a = 0; a < A; ++a) z[r * A + a] = (zm >> a) & 1u;
}

// ---------------------------------------------------------------------------------------------------
// multi-GPU: ownership and the exchange of clusters whose new block belongs to another rank (replaces the
// shuffle `.partitionBy(partitioner)`, GU:144).  Messages: entity = [e, y_0..y_{A-1}], record = [r, e, zmask].
// ---------------------------------------------------------------------------------------------------
__global__ void k_mark_ent_owned(int64_t E, const int *__restrict__ blk, const int *__restrict__ owner, int rank,
                                 unsigned char *__restrict__ ent_owned) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < E) ent_owned[e] = (owner[blk[e]] == rank);
}
__global__ void k_mark_ent_block(int64_t E, const int *__restrict__ blk, int block, unsigned char *__restrict__ ent_owned) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e < E) ent_owned[e] = (blk[e] == block);
}
__global__ void k_mark_rec_owned(int64_t R, const int *__restrict__ link, const unsigned char *__restrict__ ent_owned,
                                 unsigned char *__restrict__ rec_owned) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < R) rec_owned[r] = ent_owned[link[r]];
}

// ---- the cluster messages of a sharded sweep -------------------------------------------------------------------
// One set of kernels writes and applies the messages for both transports; they differ only in where the messages go
// (MsgOut) and where the received ones are (MsgIn), two tables indexed by barrier parity:
// * peer to peer (dbl_sweep on a connected context): every rank owns one communication buffer (cudaMalloc, exported
//   with cudaIpc, mapped by every peer over NVLink/NVSwitch).  k_move_* write the messages STRAIGHT into the
//   destination rank's receive buffer (slot from a system-scope atomic on the destination's cursor), the partial
//   summary goes into a slot of every peer, one flag barrier follows, then every rank unpacks what it received and
//   reduces the summary slots in rank order.  No host round trip.  Receive buffers have room for EVERY entity and
//   record (an entity moves at most once per sweep), and everything is double buffered by barrier parity, so a fast
//   rank can run ahead by one sweep without overwriting what a slow one still reads.  dbl_comm_import fills the
//   tables once; the parity is picked on the device, so captured sweeps replay.
// * host-mediated (dbl_sweep_begin / dbl_exchange_pack / dbl_exchange_unpack / dbl_sweep_end): k_move_* write into
//   the caller's send buffers, rank d's messages at the offset of the counts before d, with cursors of this context;
//   k_unpack_* read the caller's receive buffers.  Both parities point at the same buffers.
constexpr int MAX_WORLD = 16;
struct CommDev {
  int rank, world, A, nws;  // nws = summary words per slot (partial summary + status)
  long long cap_e, cap_r;
  unsigned char *base[MAX_WORLD];  // communication buffer of every rank (own buffer at [rank])
  size_t off_cursor, off_slots, off_ent, off_rec;
  __device__ __forceinline__ unsigned long long *arrive(int d) const { return reinterpret_cast<unsigned long long *>(base[d]); }
  __host__ __device__ __forceinline__ unsigned long long *cursor(int d, int par) const {
    return reinterpret_cast<unsigned long long *>(base[d] + off_cursor) + 2 * par;
  }
  __device__ __forceinline__ long long *slot(int d, int par, int src) const {
    return reinterpret_cast<long long *>(base[d] + off_slots) + ((size_t)par * world + src) * nws;
  }
  int *recv_ent(int d, int par) const { return reinterpret_cast<int *>(base[d] + off_ent) + (size_t)par * cap_e * (A + 1); }
  int *recv_rec(int d, int par) const { return reinterpret_cast<int *>(base[d] + off_rec) + (size_t)par * cap_r * 3; }
};
__device__ __forceinline__ int comm_parity(const long long *ctl) { return (int)((ctl[CTL_EPOCH] + 1) & 1); }

// where the messages for destination rank d go, by parity
struct MsgOut {
  int *ent[MAX_WORLD][2], *rec[MAX_WORLD][2];
  unsigned long long *cursor[MAX_WORLD][2];  // cursor pair: [0] entities, [1] records
};
// where the messages this rank received are, by parity
struct MsgIn {
  const int *ent[2], *rec[2];
  const unsigned long long *count[2];  // count pair: [0] entities, [1] records
};

// slot in rank d's area for every lane that has a message for d: one system-scope atomic per destination and warp.
// Every lane of the warp calls it (d < 0: nothing to send).
__device__ __forceinline__ long long dest_slot(const MsgOut &o, int par, int which, int d) {
  const int lane = threadIdx.x & 31;
  const unsigned grp = __match_any_sync(FULL, d);
  const int leader = __ffs(grp) - 1;
  unsigned long long basev = 0;
  if (d >= 0 && lane == leader) basev = atomicAdd_system(o.cursor[d][par] + which, (unsigned long long)__popc(grp));
  basev = __shfl_sync(FULL, basev, leader);
  return (long long)basev + __popc(grp & ((1u << lane) - 1u));
}

struct MoveParams {
  int rank;
  MsgOut out;
  long long *ctl;
  int A;
  const int *ent_sorted, *rec_sorted;
  const int *blk, *owner, *link, *y;
  const unsigned *zmask;
  int *ent_dest;
  unsigned char *ent_owned, *rec_owned;
};
__global__ void __launch_bounds__(256) k_move_ent(MoveParams p) {
  if (sweep_dead(p.ctl)) return;
  const int64_t n = p.ctl[CTL_OWNED_ENT];
  const int64_t n32 = (n + 31) & ~(int64_t)31;  // whole warps stay in the loop together
  const int par = comm_parity(p.ctl);
  int sent = 0;
  GRID_STRIDE(i, n32) {
    int d = -1;
    int64_t e = -1;
    if (i < n) {
      e = p.ent_sorted[i];
      const int o = p.owner[p.blk[e]];
      if (o != p.rank) d = o;
      p.ent_dest[e] = d;
    }
    const long long slot = dest_slot(p.out, par, 0, d);
    if (d >= 0) {
      int *m = p.out.ent[d][par] + slot * (p.A + 1);
      m[0] = (int)e;
      for (int a = 0; a < p.A; ++a) m[1 + a] = p.y[e * p.A + a];
      p.ent_owned[e] = 0;
      ++sent;
    }
  }
  if (sent) atomicAdd(reinterpret_cast<unsigned long long *>(&p.ctl[CTL_MOVED_ENT]), (unsigned long long)sent);
}
__global__ void __launch_bounds__(256) k_move_rec(MoveParams p) {
  if (sweep_dead(p.ctl)) return;
  const int64_t n = p.ctl[CTL_OWNED_REC];
  const int64_t n32 = (n + 31) & ~(int64_t)31;
  const int par = comm_parity(p.ctl);
  int sent = 0;
  GRID_STRIDE(i, n32) {
    int d = -1;
    int64_t r = -1;
    if (i < n) {
      r = p.rec_sorted[i];
      d = p.ent_dest[p.link[r]];
    }
    const long long slot = dest_slot(p.out, par, 1, d);
    if (d >= 0) {
      int *m = p.out.rec[d][par] + slot * 3;
      m[0] = (int)r; m[1] = p.link[r]; m[2] = (int)p.zmask[r];
      p.rec_owned[r] = 0;
      ++sent;
    }
  }
  if (sent) atomicAdd(reinterpret_cast<unsigned long long *>(&p.ctl[CTL_MOVED_REC]), (unsigned long long)sent);
}
// partial summary (+ status) into a slot of every rank, then the barrier: rank r stores the new epoch into
// arrive[r] of every peer (release, system scope) and waits until its own arrive[] shows every peer (acquire).
// Never skipped, even when the sweep was abandoned locally: the peers are waiting.  A peer that does not show up
// within timeout_cycles sets ST_PEER_TIMEOUT instead of hanging the GPU.
__global__ void __launch_bounds__(256) k_publish_barrier(CommDev c, long long *ctl, const unsigned long long *part, int nw,
                                                         long long timeout_cycles) {
  const long long epoch = ctl[CTL_EPOCH] + 1;
  const int par = (int)(epoch & 1);
  __shared__ int s_timeout;
  if (threadIdx.x == 0) s_timeout = 0;
  for (int i = threadIdx.x; i < c.nws; i += blockDim.x) {
    const long long v = (i < nw) ? (long long)part[i] : ctl[CTL_STATUS];
    for (int d = 0; d < c.world; ++d) c.slot(d, par, c.rank)[i] = v;
  }
  __syncthreads();
  if ((int)threadIdx.x < c.world) {
    const int d = threadIdx.x;
    __threadfence_system();
    unsigned long long *flag = c.arrive(d) + c.rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(flag), "l"((unsigned long long)epoch) : "memory");
    const unsigned long long *mine = c.arrive(c.rank) + d;
    const long long t0 = clock64();
    for (;;) {
      unsigned long long v;
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory");
      if (v >= (unsigned long long)epoch) break;
      if (clock64() - t0 > timeout_cycles) { s_timeout = 1; break; }
      __nanosleep(200);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    ctl[CTL_EPOCH] = epoch;
    if (s_timeout) ctl[CTL_STATUS] |= ST_PEER_TIMEOUT;
  }
}
// what the peers wrote for this rank (parity of the barrier just passed)
__device__ __forceinline__ int done_parity(const long long *ctl) { return (int)(ctl[CTL_EPOCH] & 1); }
struct UnpackParams {
  MsgIn in;
  const long long *ctl;
  int A;
  const AttrDev *attrs;
  TreeDev tree;
  int *y, *blk, *link;
  double *entN;
  unsigned *zmask;
  unsigned char *ent_owned, *rec_owned;
};
__global__ void __launch_bounds__(256) k_unpack_ent(UnpackParams p) {
  if (p.ctl[CTL_STATUS] & ST_PEER_TIMEOUT) return;
  const int par = done_parity(p.ctl);
  const int64_t n = (int64_t) * reinterpret_cast<const volatile unsigned long long *>(p.in.count[par]);
  const int *buf = p.in.ent[par];
  GRID_STRIDE(i, n) {
    const int *m = buf + i * (p.A + 1);
    const int64_t e = m[0];
    double nn = 1.0;
    for (int a = 0; a < p.A; ++a) {
      const int v = m[1 + a];
      p.y[e * p.A + a] = v;
      if (!p.attrs[a].is_const) nn = nn * p.attrs[a].norm[v];
    }
    p.entN[e] = nn;
    p.blk[e] = p.tree.n_nodes > 0 ? tree_leaf(p.tree, m + 1) : 0;
    p.ent_owned[e] = 1;
  }
}
__global__ void __launch_bounds__(256) k_unpack_rec(UnpackParams p) {
  if (p.ctl[CTL_STATUS] & ST_PEER_TIMEOUT) return;
  const int par = done_parity(p.ctl);
  const int64_t n = (int64_t) * reinterpret_cast<const volatile unsigned long long *>(p.in.count[par] + 1);
  const int *buf = p.in.rec[par];
  GRID_STRIDE(i, n) {
    const int *m = buf + i * 3;
    const int64_t r = m[0];
    p.link[r] = m[1];
    p.zmask[r] = (unsigned)m[2];
    p.rec_owned[r] = 1;
  }
}
// global summary = sum of the slots in rank order (SummaryAccumulators.scala:54-63; integer words exact, the
// log-likelihood word is an f64 sum in a fixed order, so every rank gets identical bits); a peer's status makes the
// sweep fail here as well; the cursors of this parity are cleared for their next use two barriers from now
__global__ void __launch_bounds__(256) k_reduce_peers(CommDev c, long long *ctl, int nw, int ll_slot,
                                                      long long *__restrict__ glob) {
  const int par = done_parity(ctl);
  __shared__ long long s_status;
  if (threadIdx.x == 0) s_status = 0;
  __syncthreads();
  const bool timed_out = (ctl[CTL_STATUS] & ST_PEER_TIMEOUT) != 0;
  for (int i = threadIdx.x; i < c.nws && !timed_out; i += blockDim.x) {
    if (i == nw) {  // status word
      long long st = 0;
      for (int s = 0; s < c.world; ++s) st |= c.slot(c.rank, par, s)[i];
      if (st) atomicOr(reinterpret_cast<unsigned long long *>(&s_status), (unsigned long long)st);
    } else if (i == ll_slot) {
      double sum = 0.0;
      for (int s = 0; s < c.world; ++s) sum += __longlong_as_double(c.slot(c.rank, par, s)[i]);
      glob[i] = __double_as_longlong(sum);
    } else {
      long long sum = 0;
      for (int s = 0; s < c.world; ++s) sum += c.slot(c.rank, par, s)[i];
      glob[i] = sum;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_status && !ctl[CTL_STATUS]) ctl[CTL_STATUS] = (s_status & ST_ZERO_MASS) ? (ST_ZERO_MASS | ST_PEER_ERROR) : ST_PEER_ERROR;
    unsigned long long *cur = c.cursor(c.rank, par);
    cur[0] = 0; cur[1] = 0;
  }
}
// Block -> rank placement on the device (partitioning/LPTScheduler.scala:57-76: longest processing time first, cost
// of a block = records x entities), re-evaluated from the GLOBAL block sizes of the state just produced, so every
// rank computes the same table.  The new table only re-routes: blocks migrate with the next exchange as ordinary
// cluster messages.  Adopted only when the current table is more than `threshold` above the LPT makespan.
__global__ void k_lpt(int P, int world, int ent_slot, int rec_slot, const long long *__restrict__ glob,
                      long long *__restrict__ ctl, int period, double threshold, int *__restrict__ owner,
                      int *__restrict__ scratch /* 2*P ints */, double *__restrict__ dscratch /* P + world doubles */) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (sweep_dead(ctl) || period <= 0 || ((ctl[CTL_ITER] + 1) % period) != 0) return;
  int *order = scratch, *cand = scratch + P;
  double *cost = dscratch, *load = dscratch + P;
  double total = 0.0;
  for (int b = 0; b < P; ++b) {
    cost[b] = (double)glob[ent_slot + b] * (double)glob[rec_slot + b];
    total += cost[b];
    order[b] = b;
  }
  if (!(total > 0.0)) return;
  for (int i = 1; i < P; ++i) {  // insertion sort by (-cost, block id)
    const int b = order[i];
    int j = i - 1;
    while (j >= 0 && (cost[order[j]] < cost[b] || (cost[order[j]] == cost[b] && order[j] > b))) { order[j + 1] = order[j]; --j; }
    order[j + 1] = b;
  }
  for (int r = 0; r < world; ++r) load[r] = 0.0;
  for (int i = 0; i < P; ++i) {
    const int b = order[i];
    int best = 0;
    for (int r = 1; r < world; ++r) if (load[r] < load[best]) best = r;
    cand[b] = best;
    load[best] += cost[b];
  }
  double lpt_max = 0.0;
  for (int r = 0; r < world; ++r) lpt_max = fmax(lpt_max, load[r]);
  for (int r = 0; r < world; ++r) load[r] = 0.0;
  for (int b = 0; b < P; ++b) load[owner[b]] += cost[b];
  double cur_max = 0.0;
  for (int r = 0; r < world; ++r) cur_max = fmax(cur_max, load[r]);
  if (cur_max > threshold * lpt_max) {
    for (int b = 0; b < P; ++b) owner[b] = cand[b];
    ctl[CTL_REPLACED] += 1;
  }
}

// ---- read-out of a sharded state --------------------------------------------------------------------------
// owned rows of the state into caller-provided device buffers, zeros elsewhere (summing over ranks = full state)
__global__ void k_export_ent(int64_t E, int A, const unsigned char *__restrict__ owned, const int *__restrict__ y,
                             const int *__restrict__ blk, int *__restrict__ y_out, int *__restrict__ blk_out) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const bool o = owned[e];
  for (int a = 0; a < A; ++a) y_out[e * A + a] = o ? y[e * A + a] : 0;
  blk_out[e] = o ? blk[e] : 0;
}
__global__ void k_export_rec(int64_t R, int A, const unsigned char *__restrict__ owned, const int *__restrict__ link,
                             const unsigned *__restrict__ zmask, int *__restrict__ link_out,
                             unsigned char *__restrict__ z_out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const bool o = owned[r];
  link_out[r] = o ? link[r] : 0;
  const unsigned zm = o ? zmask[r] : 0u;
  for (int a = 0; a < A; ++a) z_out[r * A + a] = (zm >> a) & 1u;
}
// owned rows only, compacted in the order of ent_sorted / rec_sorted (block-major): ids + rows
__global__ void k_gather_ent(int64_t n, int A, const int *__restrict__ ent_sorted, const int *__restrict__ y,
                             const int *__restrict__ blk, int *__restrict__ ids, int *__restrict__ y_out,
                             int *__restrict__ blk_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t e = ent_sorted[i];
  ids[i] = (int)e;
  for (int a = 0; a < A; ++a) y_out[i * A + a] = y[e * A + a];
  blk_out[i] = blk[e];
}
__global__ void k_gather_rec(int64_t n, int A, const int *__restrict__ rec_sorted, const int *__restrict__ link,
                             const unsigned *__restrict__ zmask, int *__restrict__ ids, int *__restrict__ link_out,
                             unsigned char *__restrict__ z_out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int64_t r = rec_sorted[i];
  ids[i] = (int)r;
  link_out[i] = link[r];
  const unsigned zm = zmask[r];
  for (int a = 0; a < A; ++a) z_out[i * A + a] = (zm >> a) & 1u;
}
// Order-independent 64-bit fingerprint of the owned rows: sum over rows of a mixed hash of (row id, row contents).
// Sums of the per-rank values (mod 2^64) are the same for every rank count and placement.
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__global__ void __launch_bounds__(256) k_state_hash(RowSet ents, RowSet recs, int A, const int *__restrict__ y,
                                                    const int *__restrict__ link, const unsigned *__restrict__ zmask,
                                                    unsigned long long *__restrict__ out /*2*/) {
  unsigned long long he = 0, hr = 0;
  const int64_t ne = ents.count(), nr = recs.count();
  GRID_STRIDE(i, ne) {
    const int64_t e = ents.row(i);
    if (e < 0) continue;
    unsigned long long h = mix64(0xE000000000000000ull ^ (unsigned long long)e);
    for (int a = 0; a < A; ++a) h = mix64(h ^ (unsigned long long)(unsigned)y[e * A + a]);
    he += h;
  }
  GRID_STRIDE(i, nr) {
    const int64_t r = recs.row(i);
    if (r < 0) continue;
    unsigned long long h = mix64(0xA000000000000000ull ^ (unsigned long long)r);
    h = mix64(h ^ (unsigned long long)(unsigned)link[r]);
    h = mix64(h ^ (unsigned long long)zmask[r]);
    hr += h;
  }
  typedef cub::BlockReduce<unsigned long long, 256> BR;
  __shared__ typename BR::TempStorage t1, t2;
  const unsigned long long se = BR(t1).Sum(he), sr = BR(t2).Sum(hr);
  if (threadIdx.x == 0) { atomicAdd(&out[0], se); atomicAdd(&out[1], sr); }
}

// ---------------------------------------------------------------------------------------------------
// host-side context
// ---------------------------------------------------------------------------------------------------
// cudaFree synchronises the whole device.  Several ranks may share one device, and while a sharded sweep is being
// enqueued (the first one after a state of another size reallocates buffers) a peer's k_publish_barrier may already
// spin, waiting for kernels this rank has not launched yet: the free would wait for the barrier and the barrier for
// the free until it times out.  dbl_sweep_async of a sharded context parks the buffers it replaces here instead; the
// context frees them when it enqueues no sweep (state upload, dbl_comm_export, destruction).
static thread_local std::vector<void *> *t_deferred_free = nullptr;

template <typename T>
struct DevBuf {
  T *p = nullptr;
  size_t n = 0;
  cudaError_t alloc(size_t count) {
    release();
    n = count;
    return cudaMalloc((void **)&p, std::max<size_t>(count, 1) * sizeof(T));
  }
  void release() {
    if (p) {
      if (t_deferred_free) t_deferred_free->push_back(p);
      else cudaFree(p);
    }
    p = nullptr; n = 0;
  }
  ~DevBuf() { release(); }
};

// what dbl_comm_export hands to the peers (DBL_COMM_BLOB_BYTES)
struct CommBlob {
  uint32_t magic;
  int32_t rank, world, device;
  int64_t pid;
  uint64_t ptr;  // address in the exporting process (used when the importer IS that process)
  uint64_t bytes;
  int64_t E, R;
  int32_t A, nws;
  cudaIpcMemHandle_t handle;
  char pad[DBL_COMM_BLOB_BYTES - 4 - 12 - 8 - 8 - 8 - 16 - 8 - (int)sizeof(cudaIpcMemHandle_t)];
};
static_assert(sizeof(CommBlob) == DBL_COMM_BLOB_BYTES, "blob layout");
constexpr uint32_t COMM_MAGIC = 0xDB1B2002u;

struct dbl_ctx {
  int A = 0, F = 0, P = 1, device = 0;
  uint64_t seed = 0;
  int rank = 0, world = 1;
  std::vector<double> alpha, beta;
  std::string err;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;

  // model (device)
  std::vector<DevBuf<double>> dtab;  // per-attr double tables
  std::vector<DevBuf<int>> itab;
  DevBuf<AttrDev> attrs;
  DevBuf<int> perm_dev;
  int perm[DBL_MAX_ATTRS] = {0};
  int n_str = 0;       // non-constant attributes
  int hslots = 32, hshift = 27;  // common hash-table size of the non-constant attributes; hslots = 0: none
  Pcg2Format pcg2_fmt{};         // tile format of k_link_pcg2 (pcg2_format; quad: pcg2_quad in alloc_blocks)
  std::vector<AttrDev> h_attrs;
  DevBuf<int> tree_buf;
  TreeDev tree{};
  DevBuf<double> prior;  // alpha[A], beta[A], file sizes[F] (k_theta)

  // batched chains (dbl_chains_*): K chains of the model, chain-major; F, P, R, E count all of them (F = K F1,
  // P = K B), so every kernel indexes exactly as for one chain
  int K = 1, F1 = 0, B = 1;
  DevBuf<uint64_t> chain_seeds;  // K keys (K > 1 only)
  ChainMap chain_map() const {
    ChainMap m;
    m.K = K; m.recs = (int)(R / K); m.ents = (int)(E / K); m.files = F1; m.blocks = B;
    m.seeds = K > 1 ? chain_seeds.p : nullptr;
    return m;
  }

  // state
  int64_t R = 0, E = 0, iteration = 0;
  bool has_state = false;
  DevBuf<int> x, file, link, newlink, y, blk;
  DevBuf<uint8_t> zbytes;  // staging for the byte-per-flag host format of z
  DevBuf<int> vflag, file_cnt;
  DevBuf<unsigned> zmask;
  DevBuf<double> entN;
  std::vector<double> h_theta, h_file_sizes_d;
  std::vector<int64_t> file_sizes;
  long long h_head[2] = {0, 0};  // staging of (iteration, status) for a new state

  // control block (one allocation, mirrored in pinned host memory by snapshot()):
  //   [CTL_WORDS] ctl | [nw] partial summary | [nw] global summary | [A*F] theta | [A*F] theta_prev | [2] hash
  DevBuf<long long> cb;
  long long *h_cb = nullptr;  // pinned
  size_t cb_words = 0;
  int nw = 0;  // summary words: A*F + K(A+1) + 2K + 2*P
  long long *ctl() const { return cb.p; }
  unsigned long long *part() const { return reinterpret_cast<unsigned long long *>(cb.p + CTL_WORDS); }
  long long *glob() const { return cb.p + CTL_WORDS + nw; }
  double *theta() const { return reinterpret_cast<double *>(cb.p + CTL_WORDS + 2 * (size_t)nw); }
  double *theta_prev() const { return theta() + (size_t)A * F; }
  unsigned long long *hash_words() const { return reinterpret_cast<unsigned long long *>(theta_prev() + (size_t)A * F); }
  const long long *h_ctl() const { return h_cb; }
  const long long *h_part() const { return h_cb + CTL_WORDS; }
  const long long *h_glob() const { return h_cb + CTL_WORDS + nw; }
  const double *h_theta_dev() const { return reinterpret_cast<const double *>(h_cb + CTL_WORDS + 2 * (size_t)nw); }
  // [A*F] aggDist, [K(A+1)] recDist of every chain, [K] isolates, [K] log-likelihood (f64 bits); one chain: the words
  // a host-mediated all-reduce carries
  int n_counts() const { return A * F + K * (A + 1) + 2 * K; }
  int iso_slot() const { return A * F + K * (A + 1); }  // chain k: + k
  int ll_slot() const { return A * F + K * (A + 1) + K; }
  int blk_ent_slot() const { return n_counts(); }
  int blk_rec_slot() const { return n_counts() + P; }

  // ownership (multi-GPU sharding by block)
  std::vector<int> owner_h;  // P entries; default: everything owned by this rank
  DevBuf<int> owner, ent_dest, ent_key, link_key;
  DevBuf<unsigned char> ent_owned, rec_owned;
  // host-mediated exchange: [world] cursor pairs of the sent messages, then the pair of received counts
  DevBuf<unsigned long long> move_cnt;
  std::vector<int64_t> h_move_ent, h_move_rec;  // messages per destination, from the block histograms
  bool in_sweep = false, in_block_sweep = false;
  int block_sampler = 0;
  std::vector<char> block_done;
  DevBuf<int> blk_frozen;
  bool all_owned = true;  // no shard has been carved out of the replicated state yet

  // peer-to-peer exchange
  DevBuf<unsigned char> comm_buf;
  size_t comm_bytes = 0;
  CommDev comm{};
  MsgOut p2p_out{};  // the mapped receive buffers and cursors (dbl_comm_import)
  MsgIn p2p_in{};
  bool comm_ready = false;
  std::vector<void *> ipc_opened;
  DevBuf<int> lpt_scratch;
  DevBuf<double> lpt_dscratch;
  int rebalance_period = 16;
  double rebalance_threshold = 1.03;
  long long barrier_timeout_cycles = 120000000000LL;  // ~60 s at 1.9 GHz: ranks may reach their first sweep far apart

  // layout
  DevBuf<int> iota, blk_sorted, ent_sorted, rec_key, rec_key_sorted, rec_sorted;
  DevBuf<int> ent_ptr, tile_ptr, rec_ptr, cta_ptr, cta_ptr2, cta_ptr3, tiles;
  DevBuf<double> lane_sums;  // k_link_pcg2 scratch: pass-1 lane sums per chunk of every resident warp
  std::optional<Pcg2Format> tiles_fmt;  // the format `tiles` holds for the current layout; none: not built
  // k_link_pcg2's 1/n(y) columns beside the tiles (LinkParams::tile_invn), allocated only when some record misses a
  // non-constant value (rec_missing, found by k_validate at upload); tiles_invn: built with the current tiles
  DevBuf<double> tile_invn;
  bool rec_missing = false, tiles_invn = false;
  // inverted index of the block tables for the pruned PCG-I link kernel (built on demand, once per sweep): E * A ids,
  // unsigned or (inv_ids64) unsigned long long, with their candidate positions
  DevBuf<unsigned char> inv_ids_in, inv_ids;
  bool inv_ids64 = false;
  DevBuf<int> inv_pos_in, inv_pos, inv_vptr, heavy_list;
  DevBuf<long long> far_list;  // k_values -> k_values_rescaled
  InvDense inv_dense;
  bool inv_use_dense = false;  // inv_vptr holds the dense pointer table
  DevBuf<unsigned char> inv_tmp;
  size_t inv_tmp_bytes = 0;
  bool inv_valid = false;
  DevBuf<int> link_sorted, rec_by_ent, ent_rec_ptr;
  DevBuf<unsigned char> rec_class;  // static cost class of a record (k_rec_class)
  DevBuf<unsigned char> cub_tmp;
  size_t cub_bytes = 0;
  int max_ctas = 0;
  DevBuf<int> gather_i;  // staging of dbl_download_owned
  DevBuf<unsigned char> gather_b;

  // host copies refreshed by snapshot()
  int64_t h_pairs = 0;
  int64_t h_owned_ent = -1, h_owned_rec = -1;  // -1 = not known on the host since the last re-partitioning

  int64_t launches = 0;
  double link_ms = 0.0;
  int link_mode = 0;  // 0 auto, 1 generic kernel everywhere, 2 dense TMA kernels everywhere (no pruning)
  bool link_mass_on = false;   // dbl_set_link_mass_capture: the link kernels store every record's total mass
  DevBuf<double> link_mass;    // R entries, allocated by the first sweep with the capture on
  double last_sweep_ms = 0.0;
  int64_t link_launches = 0;
  // eager sweeps are timed phase by phase: events before / after the link kernel, after the value / distortion /
  // summary kernels, after the exchange, after the re-layout
  struct PhaseEvents { cudaEvent_t e[5]; };
  std::vector<PhaseEvents> pending_events, event_pool;
  PhaseEvents cur_events{};
  bool cur_timed = false;
  double phase_ms[4] = {0, 0, 0, 0};
  int64_t phase_sweeps = 0;
  size_t pcg2_smem_cfg = 0, match_smem_cfg = 0;  // dynamic shared memory opted in on THIS device
  int sm_count = 132;                           // replaced by the device's count in dbl_ctx_create
  int pcg2_grid = 0;                            // persistent CTAs of k_link_pcg2 (set by alloc_blocks)
  int pcg2_recs = LINK_WARPS;                   // records per work item of k_link_pcg2
  bool async_open = false;  // sweeps enqueued by dbl_sweep_async, not yet collected by dbl_sync
  // CUDA graphs of one sweep (launch-bound problem sizes): key = sampler * 4 + link mode
  struct SweepGraph { cudaGraph_t graph = nullptr; cudaGraphExec_t exec = nullptr; int64_t launches = 0; };
  std::map<int, SweepGraph> graphs;
  std::map<int, bool> graph_warm;  // one eager sweep of that kind has run (lazy allocations, shared-memory opt-ins)
  int graph_mode = 0;              // 0 auto (small problems), 1 never, 2 always
  bool capturing = false;
  void drop_graphs() {
    for (auto &kv : graphs) {
      if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
      if (kv.second.graph) cudaGraphDestroy(kv.second.graph);
    }
    graphs.clear();
    graph_warm.clear();
  }
  std::vector<void *> deferred_free;  // buffers a sharded sweep replaced (t_deferred_free)
  void free_deferred() {
    for (void *q : deferred_free) cudaFree(q);
    deferred_free.clear();
  }

  void set_error(const std::string &s) { err = s; }
};

static inline int grid_for(int64_t n, int bs) { return (int)std::max<int64_t>(1, (n + bs - 1) / bs); }
// grid of a grid-stride kernel over at most n rows: one wave of resident CTAs on this device
static inline int grid_rows(const dbl_ctx *ctx, int64_t n, int bs) {
  return (int)std::min<int64_t>((int64_t)ctx->sm_count * (2048 / bs), std::max<int64_t>(1, (n + bs - 1) / bs));
}

static RowSet rows_prefix(dbl_ctx *ctx, bool ents) {
  RowSet r;
  r.ctl = ctx->ctl();
  r.sorted = ents ? ctx->ent_sorted.p : ctx->rec_sorted.p;
  r.owned = nullptr;
  r.n_all = ents ? ctx->E : ctx->R;
  r.count_word = ents ? CTL_OWNED_ENT : CTL_OWNED_REC;
  return r;
}
static RowSet rows_masked(dbl_ctx *ctx, bool ents) {
  RowSet r;
  r.ctl = ctx->ctl();
  r.sorted = nullptr;
  r.owned = ents ? ctx->ent_owned.p : ctx->rec_owned.p;
  r.n_all = ents ? ctx->E : ctx->R;
  r.count_word = ents ? CTL_OWNED_ENT : CTL_OWNED_REC;
  return r;
}

static int upload_tree(dbl_ctx *ctx, const dbl_kdtree *t) {
  if (t) {
    const int n = t->n_nodes;
    std::vector<int> pack;
    pack.insert(pack.end(), t->attr.begin(), t->attr.end());
    pack.insert(pack.end(), t->kind.begin(), t->kind.end());
    pack.insert(pack.end(), t->split.begin(), t->split.end());
    pack.insert(pack.end(), t->set_ptr.begin(), t->set_ptr.end());
    pack.insert(pack.end(), t->leaf_no.begin(), t->leaf_no.end());
    pack.insert(pack.end(), t->set_val.begin(), t->set_val.end());
    for (int i = 0; i < n; ++i)
      if (t->attr[i] >= ctx->A) { ctx->set_error("partitioner attribute id out of range"); return DBL_ERR_INVALID; }
    CUDA_TRY(ctx->tree_buf.alloc(pack.size()));
    CUDA_TRY(cudaMemcpy(ctx->tree_buf.p, pack.data(), pack.size() * sizeof(int), cudaMemcpyHostToDevice));
    int *base = ctx->tree_buf.p;
    ctx->tree.n_nodes = n;
    ctx->tree.attr = base;
    ctx->tree.kind = base + n;
    ctx->tree.split = base + 2 * n;
    ctx->tree.set_ptr = base + 3 * n;
    ctx->tree.leaf_no = base + 3 * n + (n + 1);
    ctx->tree.set_val = base + 4 * n + (n + 1);
    ctx->B = t->n_leaves;
  } else {
    ctx->tree.n_nodes = 0;
    ctx->B = 1;
  }
  ctx->P = ctx->K * ctx->B;  // every chain has the blocks of the one tree
  return DBL_OK;
}

static int upload_model(dbl_ctx *ctx, const dbl_model_desc *d) {
  const int A = d->num_attrs;
  ctx->h_attrs.resize(A);
  ctx->dtab.resize((size_t)A * 13);
  ctx->itab.resize((size_t)A * 6);
  auto up_d = [&](DevBuf<double> &b, const std::vector<double> &v) -> cudaError_t {
    cudaError_t e = b.alloc(v.size());
    if (e != cudaSuccess) return e;
    if (v.empty()) return cudaSuccess;
    return cudaMemcpy(b.p, v.data(), v.size() * sizeof(double), cudaMemcpyHostToDevice);
  };
  auto up_i = [&](DevBuf<int> &b, const std::vector<int32_t> &v) -> cudaError_t {
    cudaError_t e = b.alloc(v.size());
    if (e != cudaSuccess) return e;
    if (v.empty()) return cudaSuccess;
    return cudaMemcpy(b.p, v.data(), v.size() * sizeof(int), cudaMemcpyHostToDevice);
  };
  // one hash-table size for the whole model: re-hash the smaller tables to the largest
  int Hmax = 32;
  bool hash_ok = true;
  for (int a = 0; a < A; ++a) {
    if (d->indexes[a]->is_const) continue;
    if (d->indexes[a]->hsize <= 0) hash_ok = false;
    Hmax = std::max(Hmax, d->indexes[a]->hsize);
  }
  std::vector<dbl_index> rehashed(A);
  for (int a = 0; a < A; ++a) {
    const dbl_index *ix = d->indexes[a];
    if (hash_ok && !ix->is_const && ix->hsize != Hmax) {
      rehashed[a] = *ix;
      rehashed[a].build_hash(Hmax);
      if (rehashed[a].hsize != Hmax) hash_ok = false;
      ix = &rehashed[a];
    }
    DevBuf<double> *t = &ctx->dtab[(size_t)a * 13];
    DevBuf<int> *ti = &ctx->itab[(size_t)a * 6];
    CUDA_TRY(up_d(t[0], ix->phi));
    CUDA_TRY(up_d(t[1], ix->probs));
    CUDA_TRY(up_d(t[2], ix->norm));
    CUDA_TRY(up_d(t[3], ix->invnorm));
    CUDA_TRY(up_d(t[4], ix->pk));
    CUDA_TRY(up_d(t[5], ix->cdf));
    CUDA_TRY(up_d(t[6], ix->logphi));
    CUDA_TRY(up_d(t[7], ix->lognorm));
    CUDA_TRY(up_d(t[8], ix->expsim));
    CUDA_TRY(up_i(ti[0], ix->rowptr));
    CUDA_TRY(up_i(ti[1], ix->col));
    CUDA_TRY(up_d(t[9], ix->hvals));
    {
      std::vector<double> diag(ix->V, 1.0);  // E(v, v) (AttributeIndex.expSimOf(v, v)); 1 when the row has no entry
      for (int v = 0; v < ix->V && !ix->is_const; ++v)
        for (int q = ix->rowptr[v]; q < ix->rowptr[v + 1]; ++q)
          if (ix->col[q] == v) diag[v] = ix->expsim[q];
      CUDA_TRY(up_d(t[10], diag));
    }
    CUDA_TRY(up_i(ti[2], ix->hkeys));
    {
      std::vector<int32_t> hm(ix->hmult.begin(), ix->hmult.end());
      CUDA_TRY(up_i(ti[3], hm));
    }
    const bool sc = !ix->pcode.empty();
    if (sc) {
      CUDA_TRY(up_i(ti[4], ix->pcode));
      CUDA_TRY(up_i(ti[5], ix->sckeys));
      CUDA_TRY(up_d(t[11], ix->scvals));
      // 1/n(y) of the missing-value records, indexed by the code the tiles carry (codes no value has: 1)
      const int cmax = *std::max_element(ix->pcode.begin(), ix->pcode.end());
      std::vector<double> inv((size_t)cmax + 1, 1.0);
      for (int v = 0; v < ix->V; ++v) inv[ix->pcode[v]] = ix->invnorm[v];
      CUDA_TRY(up_d(t[12], inv));
    }
    AttrDev &h = ctx->h_attrs[a];
    h.pcode = sc ? ti[4].p : nullptr; h.sckeys = sc ? ti[5].p : nullptr;
    h.scvals = sc ? t[11].p : nullptr; h.scinvnorm = sc ? t[12].p : nullptr;
    h.V = ix->V; h.is_const = ix->is_const ? 1 : 0; h.kmax = ix->kmax; h.hsize = ix->hsize;
    h.hshift = ix->hshift; h.pad0 = h.pad1 = h.pad2 = 0;
    h.hvals = t[9].p; h.hkeys = ti[2].p; h.hmult = reinterpret_cast<const unsigned *>(ti[3].p);
    h.phi = t[0].p; h.probs = t[1].p; h.norm = t[2].p; h.invnorm = t[3].p; h.pk = t[4].p; h.cdf = t[5].p;
    h.logphi = t[6].p; h.lognorm = t[7].p; h.expsim = t[8].p; h.diag = t[10].p;
    h.rowptr = ti[0].p; h.col = ti[1].p;
  }
  CUDA_TRY(ctx->attrs.alloc(A));
  CUDA_TRY(cudaMemcpy(ctx->attrs.p, ctx->h_attrs.data(), sizeof(AttrDev) * A, cudaMemcpyHostToDevice));
  {
    int k = 0;
    for (int a = 0; a < A; ++a) if (ctx->h_attrs[a].is_const) ctx->perm[k++] = a;
    ctx->n_str = A - k;
    for (int a = 0; a < A; ++a) if (!ctx->h_attrs[a].is_const) ctx->perm[k++] = a;
    ctx->hslots = hash_ok ? Hmax : 0;
    ctx->hshift = 32;
    for (int h2 = 1; h2 < Hmax; h2 <<= 1) ctx->hshift -= 1;
    CUDA_TRY(ctx->perm_dev.alloc(A));
    CUDA_TRY(cudaMemcpy(ctx->perm_dev.p, ctx->perm, sizeof(int) * A, cudaMemcpyHostToDevice));
  }
  ctx->pcg2_fmt = pcg2_format(d, ctx->hslots);
  return upload_tree(ctx, d->tree);
}

// (re)allocate the control block for the current number of blocks; the global summary and theta survive
static int alloc_control(dbl_ctx *ctx) {
  const int A = ctx->A, F = ctx->F;
  const int nw = ctx->n_counts() + 2 * ctx->P;
  const size_t words = CTL_WORDS + 2 * (size_t)nw + 2 * (size_t)A * F + 2;
  if (ctx->cb.p && ctx->nw == nw) return DBL_OK;
  std::vector<long long> keep_ctl(CTL_WORDS, 0), keep_glob(ctx->n_counts(), 0);
  std::vector<double> keep_theta(2 * (size_t)A * F, 0.0);
  const bool had = ctx->cb.p != nullptr;
  if (had) {
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    CUDA_TRY(cudaMemcpy(keep_ctl.data(), ctx->ctl(), sizeof(long long) * CTL_WORDS, cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(keep_glob.data(), ctx->glob(), sizeof(long long) * ctx->n_counts(), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(keep_theta.data(), ctx->theta(), sizeof(double) * 2 * A * F, cudaMemcpyDeviceToHost));
  }
  CUDA_TRY(ctx->cb.alloc(words));
  ctx->cb_words = words;
  ctx->nw = nw;
  if (ctx->h_cb) cudaFreeHost(ctx->h_cb);
  CUDA_TRY(cudaMallocHost((void **)&ctx->h_cb, words * sizeof(long long)));
  memset(ctx->h_cb, 0, words * sizeof(long long));
  CUDA_TRY(cudaMemset(ctx->cb.p, 0, words * sizeof(long long)));
  if (had) {
    CUDA_TRY(cudaMemcpy(ctx->ctl(), keep_ctl.data(), sizeof(long long) * CTL_WORDS, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(ctx->glob(), keep_glob.data(), sizeof(long long) * ctx->n_counts(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(ctx->theta(), keep_theta.data(), sizeof(double) * 2 * A * F, cudaMemcpyHostToDevice));
  }
  return DBL_OK;
}

// for hosts without CUDA bindings of their own (a JVM through JNI): the device of the contexts this thread creates
extern "C" int dbl_set_device(int32_t device) { return cudaSetDevice(device) == cudaSuccess ? DBL_OK : DBL_ERR_CUDA; }
extern "C" int32_t dbl_device_count(void) {
  int n = 0;
  return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0;
}

extern "C" int dbl_ctx_create(dbl_ctx **out, const dbl_model_desc *d) {
  if (!out || !d || d->num_attrs <= 0 || d->num_attrs > DBL_MAX_ATTRS || d->num_files <= 0 || !d->indexes ||
      !d->alpha || !d->beta)
    return DBL_ERR_INVALID;
  for (int a = 0; a < d->num_attrs; ++a)
    if (!d->indexes[a] || !(d->alpha[a] > 0.0) || !(d->beta[a] > 0.0)) return DBL_ERR_INVALID;  // package.scala:165
  if (d->world_size > MAX_WORLD || d->rank < 0 || (d->world_size > 0 && d->rank >= d->world_size)) return DBL_ERR_INVALID;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return DBL_ERR_CUDA;  // no CPU fallback
  auto *ctx = new dbl_ctx();
  ctx->A = d->num_attrs;
  ctx->F = d->num_files;
  ctx->F1 = d->num_files;
  ctx->seed = d->seed;
  ctx->rank = d->rank;
  ctx->world = d->world_size > 0 ? d->world_size : 1;
  ctx->alpha.assign(d->alpha, d->alpha + ctx->A);
  ctx->beta.assign(d->beta, d->beta + ctx->A);
  cudaGetDevice(&ctx->device);
  {
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device) == cudaSuccess && sms > 0)
      ctx->sm_count = sms;
  }
  *out = ctx;
  CUDA_TRY(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreate(&ctx->ev0));
  CUDA_TRY(cudaEventCreate(&ctx->ev1));
  int rc = upload_model(ctx, d);
  if (rc != DBL_OK) return rc;
  rc = alloc_control(ctx);
  if (rc != DBL_OK) return rc;
  CUDA_TRY(ctx->prior.alloc(2 * (size_t)ctx->A + ctx->F));
  {
    std::vector<double> pr(2 * (size_t)ctx->A + ctx->F, 0.0);
    std::copy(ctx->alpha.begin(), ctx->alpha.end(), pr.begin());
    std::copy(ctx->beta.begin(), ctx->beta.end(), pr.begin() + ctx->A);
    CUDA_TRY(cudaMemcpy(ctx->prior.p, pr.data(), pr.size() * sizeof(double), cudaMemcpyHostToDevice));
  }
  ctx->h_theta.assign((size_t)ctx->A * ctx->F, 0.0);
  return DBL_OK;
}

static void comm_close(dbl_ctx *ctx) {
  for (void *p : ctx->ipc_opened) cudaIpcCloseMemHandle(p);
  ctx->ipc_opened.clear();
  ctx->comm_ready = false;
}

extern "C" void dbl_ctx_destroy(dbl_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  comm_close(ctx);
  ctx->drop_graphs();
  ctx->free_deferred();
  for (auto &pe : ctx->pending_events) for (cudaEvent_t e : pe.e) cudaEventDestroy(e);
  for (auto &pe : ctx->event_pool) for (cudaEvent_t e : pe.e) cudaEventDestroy(e);
  if (ctx->ev0) cudaEventDestroy(ctx->ev0);
  if (ctx->ev1) cudaEventDestroy(ctx->ev1);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->h_cb) cudaFreeHost(ctx->h_cb);
  delete ctx;
}
extern "C" const char *dbl_last_error(const dbl_ctx *ctx) { return ctx ? ctx->err.c_str() : "null context"; }
extern "C" int64_t dbl_num_records(const dbl_ctx *ctx) { return ctx ? ctx->R / ctx->K : 0; }  // of one chain
extern "C" int64_t dbl_num_entities(const dbl_ctx *ctx) { return ctx ? ctx->E / ctx->K : 0; }
extern "C" int32_t dbl_num_chains(const dbl_ctx *ctx) { return ctx ? ctx->K : 0; }
extern "C" int64_t dbl_iteration(const dbl_ctx *ctx) { return ctx ? ctx->iteration : 0; }
extern "C" int64_t dbl_kernel_launches(const dbl_ctx *ctx) { return ctx ? ctx->launches : 0; }
extern "C" const char *dbl_version(void) { return "dblink_b200 0.2 (sm_90a)"; }

// the 1/n(y) columns of k_link_pcg2, as many tiles as `tiles` holds: only while some record misses a non-constant
// value (48 MB at 1 M entities and 6 non-constant attributes)
static int alloc_tile_invn(dbl_ctx *ctx) {
  const size_t n = (ctx->rec_missing && ctx->n_str > 0 && ctx->P > 0)
                       ? ((size_t)(ctx->E / TE) + (size_t)ctx->P + 1) * ctx->n_str * TE : 0;
  if (n == ctx->tile_invn.n) return DBL_OK;
  ctx->drop_graphs();  // captured sweeps hold the link parameters by value
  ctx->tiles_fmt.reset();
  if (n == 0) ctx->tile_invn.release();
  else CUDA_TRY(ctx->tile_invn.alloc(n));
  return DBL_OK;
}

static int alloc_blocks(dbl_ctx *ctx) {
  const int P = ctx->P;
  ctx->drop_graphs();  // captured sweeps hold the old buffers / tree
  if ((int)ctx->owner_h.size() != P) ctx->owner_h.assign(P, ctx->rank);
  CUDA_TRY(ctx->owner.alloc(P));
  CUDA_TRY(cudaMemcpy(ctx->owner.p, ctx->owner_h.data(), sizeof(int) * P, cudaMemcpyHostToDevice));
  CUDA_TRY(ctx->ent_ptr.alloc(P + 1));
  CUDA_TRY(ctx->tile_ptr.alloc(P + 1));
  CUDA_TRY(ctx->rec_ptr.alloc(P + 1));
  CUDA_TRY(ctx->cta_ptr.alloc(P + 1));
  CUDA_TRY(ctx->cta_ptr2.alloc(P + 1));
  CUDA_TRY(ctx->cta_ptr3.alloc(P + 1));
  CUDA_TRY(ctx->lpt_scratch.alloc(2 * (size_t)P));
  CUDA_TRY(ctx->lpt_dscratch.alloc((size_t)P + MAX_WORLD));
  // sized for the unpacked format: a packed one needs a constant attribute, so it has no more words per entity
  const size_t max_tiles = (size_t)(ctx->E / TE) + (size_t)P + 1;
  CUDA_TRY(ctx->tiles.alloc(max_tiles * TileLayout::of(ctx->A).words()));
  if (int rc = alloc_tile_invn(ctx)) return rc;
  // work item and grid of the persistent PCG-II kernel for this model shape and size (see Pcg2Format::rpw)
  const Pcg2Format f = pcg2_quad(ctx->pcg2_fmt, ctx->n_str, ctx->R / ctx->world, ctx->sm_count);
  if (f.quad != ctx->pcg2_fmt.quad) ctx->pcg2_smem_cfg = 0;  // another instantiation: opt in to its shared memory
  ctx->pcg2_fmt = f;
  ctx->pcg2_recs = LINK_WARPS * ctx->pcg2_fmt.rpw(ctx->n_str);
  ctx->pcg2_grid = ctx->sm_count * ctx->pcg2_fmt.ctas_per_sm(ctx->n_str);
  const size_t need = (size_t)ctx->pcg2_grid * ctx->pcg2_recs * 1024;
  if (ctx->lane_sums.n < need) CUDA_TRY(ctx->lane_sums.alloc(need));
  ctx->max_ctas = (int)((ctx->R + LINK_WARPS - 1) / LINK_WARPS) + P;
  return alloc_control(ctx);
}

static int alloc_state(dbl_ctx *ctx, int64_t R, int64_t E) {
  const int A = ctx->A;
  if (R <= 0 || E <= 0 || R > 0x7fffffff || E > 0x7fffffff) { ctx->set_error("bad R/E"); return DBL_ERR_INVALID; }
  ctx->all_owned = true;
  if (ctx->R == R && ctx->E == E && ctx->x.p && ctx->tiles.p) {  // same shape as the previous state: reuse buffers
    CUDA_TRY(cudaMemsetAsync(ctx->ent_owned.p, 1, E, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(ctx->rec_owned.p, 1, R, ctx->stream));
    return DBL_OK;
  }
  if (ctx->comm_ready || ctx->comm_buf.p) {  // the communication buffers were sized for the old state
    comm_close(ctx);
    ctx->comm_buf.release();
  }
  ctx->R = R; ctx->E = E;
  ctx->drop_graphs();
  CUDA_TRY(ctx->zbytes.alloc((size_t)R * A));
  CUDA_TRY(ctx->vflag.alloc(1));
  CUDA_TRY(ctx->file_cnt.alloc(ctx->F));
  CUDA_TRY(ctx->x.alloc((size_t)R * A));
  CUDA_TRY(ctx->file.alloc(R));
  CUDA_TRY(ctx->link.alloc(R));
  CUDA_TRY(ctx->newlink.alloc(R));
  CUDA_TRY(ctx->zmask.alloc(R));
  CUDA_TRY(ctx->y.alloc((size_t)E * A));
  CUDA_TRY(ctx->blk.alloc(E));
  CUDA_TRY(ctx->entN.alloc(E));
  CUDA_TRY(ctx->ent_owned.alloc(E));
  CUDA_TRY(ctx->rec_owned.alloc(R));
  CUDA_TRY(ctx->rec_class.alloc(R));
  CUDA_TRY(cudaMemsetAsync(ctx->ent_owned.p, 1, E, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(ctx->rec_owned.p, 1, R, ctx->stream));
  CUDA_TRY(ctx->ent_dest.alloc(E));
  CUDA_TRY(ctx->ent_key.alloc(E));
  CUDA_TRY(ctx->link_key.alloc(R));
  CUDA_TRY(ctx->move_cnt.alloc(2 * (size_t)ctx->world + 2));
  const int64_t M = std::max(R, E);
  CUDA_TRY(ctx->iota.alloc(M));
  k_iota<<<grid_for(M, 256), 256, 0, ctx->stream>>>(M, ctx->iota.p);
  CUDA_TRY(ctx->blk_sorted.alloc(E));
  CUDA_TRY(ctx->ent_sorted.alloc(E));
  CUDA_TRY(ctx->rec_key.alloc(R));
  CUDA_TRY(ctx->rec_key_sorted.alloc(R));
  CUDA_TRY(ctx->rec_sorted.alloc(R));
  { int rc = alloc_blocks(ctx); if (rc) return rc; }
  CUDA_TRY(ctx->link_sorted.alloc(R));
  CUDA_TRY(ctx->rec_by_ent.alloc(R));
  CUDA_TRY(ctx->ent_rec_ptr.alloc(E + 1));
  size_t b1 = 0, b2 = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b1, (const int *)nullptr, (int *)nullptr, (const int *)nullptr,
                                  (int *)nullptr, (int)M, 0, 32, ctx->stream);
  cub::DeviceScan::ExclusiveSum(nullptr, b2, (const int *)nullptr, (int *)nullptr, (int)(E + 1), ctx->stream);
  ctx->cub_bytes = std::max(b1, b2) + 256;
  CUDA_TRY(ctx->cub_tmp.alloc(ctx->cub_bytes));
  return DBL_OK;
}

static int bits_for(int64_t n) {
  int b = 1;
  while (((int64_t)1 << b) < n) ++b;
  return b;
}

// Sort keys of rows a shard does not own must sort behind every real key.  One sentinel value would put 7/8 of the
// items of an 8-rank shard into the same radix bin, and a radix sort serialises on a bin that takes everything; so
// they are spread over the unused top of the key range: `spread` values above n_keys, in a key of `bits` bits.
static void sentinel_spread(int64_t n_keys, int world, int *bits, long long *spread) {
  int b = bits_for(n_keys + 1);
  long long sp = ((long long)1 << b) - n_keys;
  if (world > 1 && sp < 256) { ++b; sp = ((long long)1 << b) - n_keys; }
  *bits = b;
  *spread = world > 1 ? sp : 1;
}

// CSR entity -> linked records in ascending record id (LinksIndex, GU:84-119)
static int build_links_csr(dbl_ctx *ctx, bool commit_newlinks = false) {
  const int64_t R = ctx->R, E = ctx->E;
  size_t tb = ctx->cub_bytes;
  int bits;
  long long spread;
  sentinel_spread(E, ctx->world, &bits, &spread);
  if (commit_newlinks)  // inside a sweep: the draws of the link kernel become the links (unless the sweep was abandoned)
    k_commit_link_keys<<<grid_for(R, 256), 256, 0, ctx->stream>>>(R, ctx->ctl(), ctx->newlink.p, ctx->link.p,
                                                                 ctx->rec_owned.p, (int)E, (int)spread, ctx->link_key.p);
  else
    k_rec_link_keys<<<grid_for(R, 256), 256, 0, ctx->stream>>>(R, ctx->link.p, ctx->rec_owned.p, (int)E, (int)spread,
                                                              ctx->link_key.p);
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const int *)ctx->link_key.p, ctx->link_sorted.p,
                                           (const int *)ctx->iota.p, ctx->rec_by_ent.p, (int)R, 0, bits, ctx->stream));
  k_segment_ptr<<<grid_for(R + 1, 256), 256, 0, ctx->stream>>>(R, (int)E, ctx->link_sorted.p, ctx->ent_rec_ptr.p);
  ctx->launches += 3;
  return DBL_OK;
}

// group entities and records by block (replaces the shuffle, GU:144); the tiled copy of the entity table is built
// on demand by ensure_tiles().  end_of_sweep: this is the last step of a sweep -- the scan kernel also adopts the
// partial summary as the global one (single rank) and counts the sweep.
static int relayout(dbl_ctx *ctx, bool end_of_sweep = false) {
  const int64_t R = ctx->R, E = ctx->E;
  const int P = ctx->P;
  const int pb = bits_for(P + 1);
  size_t tb = ctx->cub_bytes;
  k_block_keys<<<grid_for(std::max(E, R), 256), 256, 0, ctx->stream>>>(E, R, ctx->blk.p, ctx->link.p, ctx->ent_owned.p,
                                                                        ctx->rec_owned.p, ctx->rec_class.p, P,
                                                                        ctx->ent_key.p, ctx->rec_key.p);
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const int *)ctx->ent_key.p, ctx->blk_sorted.p,
                                           (const int *)ctx->iota.p, ctx->ent_sorted.p, (int)E, 0, pb, ctx->stream));
  tb = ctx->cub_bytes;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(ctx->cub_tmp.p, tb, (const int *)ctx->rec_key.p, ctx->rec_key_sorted.p,
                                           (const int *)ctx->iota.p, ctx->rec_sorted.p, (int)R, 0,
                                           pb + REC_CLASS_BITS, ctx->stream));
  k_block_ptrs<<<grid_for(std::max(E, R) + 1, 256), 256, 0, ctx->stream>>>(E, R, P, ctx->blk_sorted.p, ctx->ent_ptr.p,
                                                                            ctx->rec_key_sorted.p, ctx->rec_ptr.p);
  k_block_scan<<<1, 128, 0, ctx->stream>>>(P, ctx->ent_ptr.p, ctx->rec_ptr.p, ctx->tile_ptr.p, ctx->cta_ptr.p,
                                           LINK_WARPS, ctx->cta_ptr2.p, MATCH_WARPS, ctx->cta_ptr3.p, ctx->pcg2_recs, ctx->ctl(),
                                           (end_of_sweep && ctx->world <= 1) ? ctx->nw : 0, ctx->part(), ctx->glob(),
                                           end_of_sweep ? 1 : 0);
  ctx->launches += 9;
  ctx->inv_valid = false;
  ctx->tiles_fmt.reset();
  ctx->h_owned_ent = ctx->h_owned_rec = -1;  // changed on the device; snapshot() brings them back
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

// tiled copy of the block-sorted entity table in format f, the one the coming link kernel reads; one buffer for
// every format, rebuilt when it holds another.  invn: with k_link_pcg2's 1/n(y) columns (when allocated)
static int ensure_tiles(dbl_ctx *ctx, Pcg2Format f, bool invn = false) {
  invn = invn && ctx->tile_invn.p;
  if (ctx->tiles_fmt == f && ctx->tiles_invn == invn) return DBL_OK;
  const int64_t n_slots = (int64_t)((size_t)(ctx->E / TE) + (size_t)ctx->P + 1) * TE;
  const TileSrc s{n_slots, ctx->A, ctx->P, ctx->y.p, ctx->ent_sorted.p, ctx->ent_ptr.p, ctx->tile_ptr.p,
                  ctx->perm_dev.p, ctx->entN.p};
  k_build_entity_tiles<<<grid_for(n_slots, 256), 256, 0, ctx->stream>>>(s, f, ctx->n_str, ctx->attrs.p, ctx->tiles.p,
                                                                         invn ? ctx->tile_invn.p : nullptr);
  ctx->launches += 1;
  ctx->tiles_fmt = f;
  ctx->tiles_invn = invn;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

// entity N / block ids / partial summary of the owned rows; in_sweep: prefix mode + distortion draws (GU:324-359)
static int refresh_summary(dbl_ctx *ctx, bool in_sweep) {
  const int A = ctx->A, F = ctx->F;
  if (!in_sweep) CUDA_TRY(cudaMemsetAsync(ctx->part(), 0, sizeof(long long) * ctx->nw, ctx->stream));  // else: k_theta
  EntPostParams ep;
  ep.rows = in_sweep ? rows_prefix(ctx, true) : rows_masked(ctx, true);
  ep.cm = ctx->chain_map();
  ep.A = A; ep.y = ctx->y.p; ep.attrs = ctx->attrs.p; ep.tree = ctx->tree; ep.entN = ctx->entN.p; ep.blk = ctx->blk.p;
  ep.ent_rec_ptr = ctx->ent_rec_ptr.p; ep.part = ctx->part(); ep.iso_slot = ctx->iso_slot(); ep.ll_slot = ctx->ll_slot();
  ep.blk_slot = ctx->world > 1 ? ctx->blk_ent_slot() : -1;
  k_entity_post<<<grid_rows(ctx, ctx->E, 256), 256, 0, ctx->stream>>>(ep);
  DistParams dp;
  dp.A = A; dp.F = F; dp.draw = in_sweep ? 1 : 0; dp.seed = ctx->seed; dp.cm = ctx->chain_map();
  dp.rows = in_sweep ? rows_prefix(ctx, false) : rows_masked(ctx, false);
  dp.attrs = ctx->attrs.p; dp.x = ctx->x.p; dp.file = ctx->file.p; dp.link = ctx->link.p;
  dp.y = ctx->y.p; dp.blk = ctx->blk.p; dp.zmask = ctx->zmask.p; dp.theta = ctx->theta(); dp.part = ctx->part();
  dp.ll_slot = ctx->ll_slot();
  dp.blk_slot = ctx->world > 1 ? ctx->blk_rec_slot() : -1;
  k_dist<<<grid_rows(ctx, ctx->R, 256), 256, 0, ctx->stream>>>(dp);
  ctx->launches += 3;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

// the partial summary of a context that owns everything IS the global one
static int adopt_local_summary(dbl_ctx *ctx) {
  k_reduce_local<<<1, 256, 0, ctx->stream>>>(ctx->nw, ctx->ctl(), ctx->part(), ctx->glob());
  ctx->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

static void recycle_events(dbl_ctx *ctx) {
  for (auto &pe : ctx->pending_events) {
    float ms[4] = {0.f, 0.f, 0.f, 0.f};
    bool ok = true;
    for (int i = 0; i < 4; ++i) ok = ok && cudaEventElapsedTime(&ms[i], pe.e[i], pe.e[i + 1]) == cudaSuccess;
    if (ok) {
      ctx->link_ms += ms[0];
      ctx->link_launches += 1;
      for (int i = 0; i < 4; ++i) ctx->phase_ms[i] += ms[i];
      ctx->phase_sweeps += 1;
    }
    ctx->event_pool.push_back(pe);
  }
  ctx->pending_events.clear();
}

// One device -> host copy of the control block, one synchronisation: iteration, status, owned counts, global
// summary, theta.  This is the only point where the host waits for the device.
static int snapshot(dbl_ctx *ctx) {
  CUDA_TRY(cudaMemcpyAsync(ctx->h_cb, ctx->cb.p, ctx->cb_words * sizeof(long long), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  recycle_events(ctx);
  const long long *c = ctx->h_ctl();
  ctx->iteration = c[CTL_ITER];
  ctx->h_pairs = c[CTL_PAIRS];
  ctx->h_owned_ent = c[CTL_OWNED_ENT];
  ctx->h_owned_rec = c[CTL_OWNED_REC];
  const long long st = c[CTL_STATUS];
  if (st) {
    const bool sharded = !ctx->all_owned;
    if (!sharded && st == ST_ZERO_MASS) {
      // the abandoned sweep changed nothing but theta: put the previous values back, the state is the one before it
      std::copy(ctx->h_theta_dev() + (size_t)ctx->A * ctx->F, ctx->h_theta_dev() + 2 * (size_t)ctx->A * ctx->F, ctx->h_theta.begin());
      CUDA_TRY(cudaMemcpyAsync(ctx->theta(), ctx->theta_prev(), sizeof(double) * ctx->A * ctx->F, cudaMemcpyDeviceToDevice,
                               ctx->stream));
    } else {
      ctx->has_state = false;  // shards are no longer at the same iteration: the caller has to upload a state again
    }
    CUDA_TRY(cudaMemsetAsync(ctx->ctl() + CTL_STATUS, 0, sizeof(long long), ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (st & ST_PEER_TIMEOUT) { ctx->set_error("a peer rank did not reach the exchange barrier (time-out)"); return DBL_ERR_CUDA; }
    ctx->set_error((st & ST_PEER_ERROR) && !(st & ST_ZERO_MASS) ? "the sweep failed on a peer rank"
                                                                : "zero probability mass in a link draw");
    return (st & ST_ZERO_MASS) ? DBL_ERR_ZERO_MASS : DBL_ERR_CUDA;
  }
  std::copy(ctx->h_theta_dev(), ctx->h_theta_dev() + (size_t)ctx->A * ctx->F, ctx->h_theta.begin());
  return DBL_OK;
}

static int finish_new_state(dbl_ctx *ctx, bool check_state, bool new_records) {
  // range checks on the device, then file sizes (RecordsCache.fileSizes)
  CUDA_TRY(cudaMemsetAsync(ctx->vflag.p, 0, sizeof(int), ctx->stream));
  k_validate<<<grid_for(std::max(ctx->R, ctx->E), 256), 256, 0, ctx->stream>>>(
      ctx->R, ctx->E, ctx->A, ctx->F, ctx->attrs.p, ctx->x.p, ctx->file.p, check_state ? ctx->link.p : nullptr,
      check_state ? ctx->y.p : nullptr, ctx->vflag.p);
  int bad = 0;
  CUDA_TRY(cudaMemcpyAsync(&bad, ctx->vflag.p, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
  std::vector<int> hc(ctx->F);
  if (new_records) {
    CUDA_TRY(cudaMemsetAsync(ctx->file_cnt.p, 0, sizeof(int) * ctx->F, ctx->stream));
    k_hist<<<grid_for(ctx->R, 256), 256, 0, ctx->stream>>>(ctx->R, ctx->file.p, ctx->file_cnt.p);
    CUDA_TRY(cudaMemcpyAsync(hc.data(), ctx->file_cnt.p, sizeof(int) * ctx->F, cudaMemcpyDeviceToHost, ctx->stream));
  }
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // nothing below may run on out-of-range ids
  ctx->rec_missing = (bad & 16) != 0;
  bad &= 15;
  if (int rc = alloc_tile_invn(ctx)) return rc;
  if (bad) {
    ctx->has_state = false;
    ctx->set_error(bad & 1 ? "record value id out of range" : bad & 2 ? "file id out of range"
                   : bad & 4 ? "link out of range" : "entity value id out of range");
    return DBL_ERR_INVALID;
  }
  if (new_records) {
    ctx->file_sizes.assign(hc.begin(), hc.end());
    ctx->h_file_sizes_d.assign(hc.begin(), hc.end());
    CUDA_TRY(cudaMemcpyAsync(ctx->prior.p + 2 * ctx->A, ctx->h_file_sizes_d.data(), sizeof(double) * ctx->F,
                             cudaMemcpyHostToDevice, ctx->stream));
  }
  ctx->launches += 2;
  // iteration / status of the new state
  ctx->h_head[0] = ctx->iteration; ctx->h_head[1] = 0;
  CUDA_TRY(cudaMemcpyAsync(ctx->ctl(), ctx->h_head, sizeof(ctx->h_head), cudaMemcpyHostToDevice, ctx->stream));
  int rc = build_links_csr(ctx);
  if (rc) return rc;
  rc = refresh_summary(ctx, false);
  if (rc) return rc;
  rc = adopt_local_summary(ctx);
  if (rc) return rc;
  // a sharded context is carved up by dbl_set_block_owners next, which lays the shard out; until then nothing reads
  // the layout (dbl_set_partitioner builds its own)
  if (ctx->world <= 1) {
    rc = relayout(ctx);
    if (rc) return rc;
  }
  rc = snapshot(ctx);
  if (rc) return rc;
  ctx->has_state = true;
  return DBL_OK;
}

extern "C" int dbl_set_partitioner(dbl_ctx *ctx, const dbl_kdtree *tree) {
  if (!ctx) return DBL_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (ctx->has_state && !ctx->all_owned) { ctx->set_error("dbl_set_partitioner after dbl_set_block_owners"); return DBL_ERR_STATE; }
  ctx->drop_graphs();
  int rc = upload_tree(ctx, tree);
  if (rc) return rc;
  if (!ctx->has_state) return alloc_control(ctx);
  rc = alloc_blocks(ctx);
  if (rc) return rc;
  rc = refresh_summary(ctx, false);  // recomputes block ids (and the unchanged summary)
  if (rc) return rc;
  rc = adopt_local_summary(ctx);
  if (rc) return rc;
  rc = relayout(ctx);
  if (rc) return rc;
  return snapshot(ctx);
}
extern "C" int32_t dbl_num_partitions(const dbl_ctx *ctx) { return ctx ? ctx->P : 0; }

static int upload_theta(dbl_ctx *ctx) {
  const size_t n = (size_t)ctx->A * ctx->F;
  CUDA_TRY(cudaMemcpyAsync(ctx->theta(), ctx->h_theta.data(), sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(ctx->theta_prev(), ctx->h_theta.data(), sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
  return DBL_OK;  // h_theta is next written by snapshot(), i.e. after the stream has drained
}

// Number of chains and their keys.  Changing K re-shapes everything sized by F, P or the summary: the state that
// follows (dbl_state_init / _upload, dbl_chains_init / _upload) is allocated afresh.
static int set_chains(dbl_ctx *ctx, int K, const uint64_t *seeds) {
  if (K == 1 && ctx->K == 1) return DBL_OK;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  ctx->drop_graphs();  // captured sweeps hold the key table and the shapes
  if (K > 1) {
    if (ctx->chain_seeds.n != (size_t)K) CUDA_TRY(ctx->chain_seeds.alloc(K));
    CUDA_TRY(cudaMemcpy(ctx->chain_seeds.p, seeds, sizeof(uint64_t) * K, cudaMemcpyHostToDevice));
  } else {
    ctx->chain_seeds.release();
  }
  if (K == ctx->K) return DBL_OK;
  const int A = ctx->A;
  ctx->K = K;
  ctx->F = K * ctx->F1;
  ctx->P = K * ctx->B;
  ctx->has_state = false;
  ctx->R = ctx->E = 0;  // alloc_state sizes every buffer for the new shape
  CUDA_TRY(ctx->prior.alloc(2 * (size_t)A + ctx->F));
  CUDA_TRY(cudaMemcpy(ctx->prior.p, ctx->alpha.data(), sizeof(double) * A, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(ctx->prior.p + A, ctx->beta.data(), sizeof(double) * A, cudaMemcpyHostToDevice));
  ctx->h_theta.assign((size_t)A * ctx->F, 0.0);
  ctx->file_sizes.clear();
  // a control block of the new shape; the counters of the context (pairs scored, ...) carry over
  long long keep[CTL_WORDS];
  CUDA_TRY(cudaMemcpy(keep, ctx->ctl(), sizeof(keep), cudaMemcpyDeviceToHost));
  ctx->cb.release();
  int rc = alloc_control(ctx);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpy(ctx->ctl(), keep, sizeof(keep), cudaMemcpyHostToDevice));
  return DBL_OK;
}

static int state_init(dbl_ctx *ctx, int64_t R, const int32_t *x, const int32_t *file, int64_t pop) {
  CUDA_TRY(cudaSetDevice(ctx->device));
  const int64_t E = pop > 0 ? pop : R;
  int rc = alloc_state(ctx, R, E);
  if (rc) return rc;
  const int A = ctx->A;
  CUDA_TRY(cudaMemcpyAsync(ctx->x.p, x, sizeof(int) * R * A, cudaMemcpyHostToDevice, ctx->stream));
  k_rec_class<<<grid_for(R, 256), 256, 0, ctx->stream>>>(R, A, ctx->attrs.p, ctx->x.p, ctx->rec_class.p);
  CUDA_TRY(cudaMemcpyAsync(ctx->file.p, file, sizeof(int) * R, cudaMemcpyHostToDevice, ctx->stream));
  k_init_entities<<<grid_for(E * A, 256), 256, 0, ctx->stream>>>(E, R, A, ctx->seed, ctx->chain_map(), ctx->attrs.p,
                                                                  ctx->x.p, ctx->y.p);
  k_init_records<<<grid_for(R, 256), 256, 0, ctx->stream>>>(E, R, A, ctx->chain_map(), ctx->x.p, ctx->y.p, ctx->link.p,
                                                            ctx->zmask.p);
  ctx->launches += 3;
  for (int a = 0; a < A; ++a)
    for (int f = 0; f < ctx->F; ++f)
      ctx->h_theta[a * ctx->F + f] = ctx->alpha[a] / (ctx->alpha[a] + ctx->beta[a]);  // DistortionProbs.scala:38-40
  rc = upload_theta(ctx);
  if (rc) return rc;
  ctx->iteration = 0;
  return finish_new_state(ctx, false, true);
}

extern "C" int dbl_state_init(dbl_ctx *ctx, int64_t R, const int32_t *x, const int32_t *file, int64_t pop) {
  if (!ctx || !x || !file) return DBL_ERR_INVALID;
  CUDA_TRY(cudaSetDevice(ctx->device));
  ctx->free_deferred();
  int rc = set_chains(ctx, 1, nullptr);
  if (rc) return rc;
  return state_init(ctx, R, x, file, pop);
}

static int state_upload(dbl_ctx *ctx, int64_t R, int64_t E, const int32_t *x, const int32_t *file, const uint8_t *z,
                        const int32_t *link, const int32_t *y, const double *theta, int64_t iteration) {
  const bool new_records = (x != nullptr);
  if (!new_records && (!ctx->x.p || ctx->R != R || ctx->E != E)) {
    ctx->set_error("dbl_state_upload without records: the context holds no records / state of that shape");
    return DBL_ERR_STATE;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  int rc = alloc_state(ctx, R, E);
  if (rc) return rc;
  const int A = ctx->A;
  DevBuf<uint8_t> &zb = ctx->zbytes;
  if (new_records) {
    CUDA_TRY(cudaMemcpyAsync(ctx->x.p, x, sizeof(int) * R * A, cudaMemcpyDefault, ctx->stream));
    k_rec_class<<<grid_for(R, 256), 256, 0, ctx->stream>>>(R, A, ctx->attrs.p, ctx->x.p, ctx->rec_class.p);
    CUDA_TRY(cudaMemcpyAsync(ctx->file.p, file, sizeof(int) * R, cudaMemcpyDefault, ctx->stream));
  }
  CUDA_TRY(cudaMemcpyAsync(zb.p, z, (size_t)R * A, cudaMemcpyDefault, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(ctx->link.p, link, sizeof(int) * R, cudaMemcpyDefault, ctx->stream));
  CUDA_TRY(cudaMemcpyAsync(ctx->y.p, y, sizeof(int) * E * A, cudaMemcpyDefault, ctx->stream));
  k_pack_z<<<grid_for(R, 256), 256, 0, ctx->stream>>>(R, A, zb.p, ctx->zmask.p);
  ctx->launches += 2;
  std::copy(theta, theta + (size_t)A * ctx->F, ctx->h_theta.begin());
  rc = upload_theta(ctx);
  if (rc) return rc;
  ctx->iteration = iteration;
  return finish_new_state(ctx, true, new_records);
}

extern "C" int dbl_state_upload(dbl_ctx *ctx, int64_t R, int64_t E, const int32_t *x, const int32_t *file,
                                const uint8_t *z, const int32_t *link, const int32_t *y, const double *theta,
                                int64_t iteration) {
  if (!ctx || !z || !link || !y || !theta || ((x == nullptr) != (file == nullptr))) return DBL_ERR_INVALID;
  if (!x && ctx->K > 1) {
    ctx->set_error("dbl_state_upload without records: the context holds the records of several chains");
    return DBL_ERR_STATE;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  ctx->free_deferred();
  int rc = set_chains(ctx, 1, nullptr);
  if (rc) return rc;
  return state_upload(ctx, R, E, x, file, z, link, y, theta, iteration);
}

// the calls that read or drive ONE chain refuse a context holding several
static int one_chain_only(dbl_ctx *ctx, const char *what) {
  if (ctx->K == 1) return DBL_OK;
  ctx->set_error(std::string(what) + " needs a context holding one chain (dbl_chains_download / dbl_chain_summary "
                 "read batched chains)");
  return DBL_ERR_STATE;
}

static int state_download(dbl_ctx *ctx, uint8_t *z, int32_t *link, int32_t *y, double *theta, int32_t *block_of_entity) {
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  const int A = ctx->A;
  DevBuf<uint8_t> &zb = ctx->zbytes;
  if (z) {
    k_unpack_z<<<grid_for(ctx->R, 256), 256, 0, ctx->stream>>>(ctx->R, A, ctx->zmask.p, zb.p);
    ctx->launches += 1;
    CUDA_TRY(cudaMemcpyAsync(z, zb.p, (size_t)ctx->R * A, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (link) CUDA_TRY(cudaMemcpyAsync(link, ctx->link.p, sizeof(int) * ctx->R, cudaMemcpyDeviceToHost, ctx->stream));
  if (y) CUDA_TRY(cudaMemcpyAsync(y, ctx->y.p, sizeof(int) * ctx->E * A, cudaMemcpyDeviceToHost, ctx->stream));
  if (block_of_entity)
    CUDA_TRY(cudaMemcpyAsync(block_of_entity, ctx->blk.p, sizeof(int) * ctx->E, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  if (theta) std::copy(ctx->h_theta.begin(), ctx->h_theta.end(), theta);
  return DBL_OK;
}

extern "C" int dbl_state_download(dbl_ctx *ctx, uint8_t *z, int32_t *link, int32_t *y, double *theta,
                                  int32_t *block_of_entity) {
  if (!ctx) return DBL_ERR_INVALID;
  int rc = one_chain_only(ctx, "dbl_state_download");
  if (rc) return rc;
  return state_download(ctx, z, link, y, theta, block_of_entity);
}

extern "C" int dbl_links_download(dbl_ctx *ctx, int32_t *link_out, int32_t *block_out) {
  return dbl_state_download(ctx, nullptr, link_out, nullptr, nullptr, block_out);
}

// ---------------------------------------------------------------------------------------------------
// batched chains: K chains of the model in one context (DESIGN.md 4.6)
// ---------------------------------------------------------------------------------------------------
static int check_chains(dbl_ctx *ctx, int32_t K, const uint64_t *seeds, int64_t R, int64_t E) {
  if (ctx->world > 1) { ctx->set_error("batched chains need an unsharded context"); return DBL_ERR_INVALID; }
  if (K < 1 || !seeds) { ctx->set_error("num_chains must be >= 1, with one seed per chain"); return DBL_ERR_INVALID; }
  std::vector<uint64_t> s(seeds, seeds + K);
  std::sort(s.begin(), s.end());
  if (std::adjacent_find(s.begin(), s.end()) != s.end()) { ctx->set_error("chain seeds must be distinct"); return DBL_ERR_INVALID; }
  // one chain is the one-chain context, keyed by the model's seed: a different key would be silently ignored
  if (K == 1 && seeds[0] != ctx->seed) {
    ctx->set_error("one chain draws with the model's seed: seeds[0] must equal dbl_model_desc.seed");
    return DBL_ERR_INVALID;
  }
  if (R <= 0 || E <= 0 || (int64_t)K * R > 0x7fffffff || (int64_t)K * E > 0x7fffffff) {
    ctx->set_error("bad R/E for this number of chains");
    return DBL_ERR_INVALID;
  }
  if (ctx->in_sweep || ctx->async_open) { ctx->set_error("a sweep is open"); return DBL_ERR_STATE; }
  return DBL_OK;
}
// the records of one chain -> K chain-major copies; chain k reads files [k F1, (k+1) F1)
static int replicate_records(dbl_ctx *ctx, int K, int64_t R, const int32_t *x, const int32_t *file,
                             std::vector<int32_t> &xk, std::vector<int32_t> &fk) {
  const int A = ctx->A;
  for (int64_t r = 0; r < R; ++r)
    if (file[r] < 0 || file[r] >= ctx->F1) { ctx->set_error("file id out of range"); return DBL_ERR_INVALID; }
  xk.resize((size_t)K * R * A);
  fk.resize((size_t)K * R);
  for (int k = 0; k < K; ++k) {
    std::copy(x, x + R * A, xk.begin() + (size_t)k * R * A);
    for (int64_t r = 0; r < R; ++r) fk[(size_t)k * R + r] = k * ctx->F1 + file[r];
  }
  return DBL_OK;
}

extern "C" int dbl_chains_init(dbl_ctx *ctx, int32_t K, const uint64_t *seeds, int64_t R, const int32_t *x,
                               const int32_t *file, int64_t pop) {
  if (!ctx || !x || !file) return DBL_ERR_INVALID;
  const int64_t E = pop > 0 ? pop : R;
  int rc = check_chains(ctx, K, seeds, R, E);
  if (rc) return rc;
  std::vector<int32_t> xk, fk;
  rc = replicate_records(ctx, K, R, x, file, xk, fk);
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  rc = set_chains(ctx, K, seeds);
  if (rc) return rc;
  return state_init(ctx, K * R, xk.data(), fk.data(), K * E);
}

extern "C" int dbl_chains_upload(dbl_ctx *ctx, int32_t K, const uint64_t *seeds, int64_t R, int64_t E,
                                 const int32_t *x, const int32_t *file, const uint8_t *z, const int32_t *link,
                                 const int32_t *y, const double *theta, int64_t iteration) {
  if (!ctx || !x || !file || !z || !link || !y || !theta) return DBL_ERR_INVALID;
  int rc = check_chains(ctx, K, seeds, R, E);
  if (rc) return rc;
  std::vector<int32_t> xk, fk;
  rc = replicate_records(ctx, K, R, x, file, xk, fk);
  if (rc) return rc;
  const int A = ctx->A, F1 = ctx->F1;
  std::vector<int32_t> lk((size_t)K * R);  // chain-local links -> global entity ids
  for (int64_t i = 0; i < (int64_t)K * R; ++i) {
    if (link[i] < 0 || link[i] >= E) { ctx->set_error("link outside its chain"); return DBL_ERR_INVALID; }
    lk[i] = (int32_t)((i / R) * E + link[i]);
  }
  std::vector<double> th((size_t)A * K * F1);  // K x A x F1 -> A x (K F1)
  for (int k = 0; k < K; ++k)
    for (int a = 0; a < A; ++a)
      for (int f = 0; f < F1; ++f) th[((size_t)a * K + k) * F1 + f] = theta[((size_t)k * A + a) * F1 + f];
  CUDA_TRY(cudaSetDevice(ctx->device));
  rc = set_chains(ctx, K, seeds);
  if (rc) return rc;
  return state_upload(ctx, K * R, K * E, xk.data(), fk.data(), z, lk.data(), y, th.data(), iteration);
}

extern "C" int dbl_chains_download(dbl_ctx *ctx, uint8_t *z, int32_t *link, int32_t *y, double *theta,
                                   int32_t *block_of_entity) {
  if (!ctx) return DBL_ERR_INVALID;
  int rc = state_download(ctx, z, link, y, nullptr, block_of_entity);
  if (rc) return rc;
  const int K = ctx->K, A = ctx->A, F1 = ctx->F1;
  const int64_t R1 = ctx->R / K, E1 = ctx->E / K;
  if (link) for (int64_t i = 0; i < ctx->R; ++i) link[i] -= (int32_t)((i / R1) * E1);
  if (block_of_entity) for (int64_t e = 0; e < ctx->E; ++e) block_of_entity[e] -= (int32_t)((e / E1) * ctx->B);
  if (theta)
    for (int k = 0; k < K; ++k)
      for (int a = 0; a < A; ++a)
        for (int f = 0; f < F1; ++f) theta[((size_t)k * A + a) * F1 + f] = ctx->h_theta[((size_t)a * K + k) * F1 + f];
  return DBL_OK;
}

// ---------------------------------------------------------------------------------------------------
// link kernel dispatch
// ---------------------------------------------------------------------------------------------------
#define DBL_DECL(N) Pcg2Kernel dbl_pcg2_kernel_a##N(int ns, Pcg2Format f);
DBL_DECL(1) DBL_DECL(2) DBL_DECL(3) DBL_DECL(4) DBL_DECL(5) DBL_DECL(6) DBL_DECL(7) DBL_DECL(8)
DBL_DECL(9) DBL_DECL(10) DBL_DECL(11) DBL_DECL(12) DBL_DECL(13) DBL_DECL(14) DBL_DECL(15) DBL_DECL(16)
#undef DBL_DECL

// The (block, attribute, value) ids of every slot of the block-sorted entity table, sorted with the candidate
// positions as payload: a stable radix sort on the significant bits only, so positions stay ascending inside an id.
template <class K>
static int sort_inverted_index(dbl_ctx *ctx, long long n_ids, long long spread, int bits) {
  const int64_t cap = ctx->E * ctx->A;
  // the slot count (inv_pos) and the key bytes together identify (cap, key width); the byte size alone does not
  if (ctx->inv_pos.n != (size_t)cap || ctx->inv_ids.n != (size_t)cap * sizeof(K)) {
    CUDA_TRY(ctx->inv_ids_in.alloc((size_t)cap * sizeof(K)));
    CUDA_TRY(ctx->inv_ids.alloc((size_t)cap * sizeof(K)));
    CUDA_TRY(ctx->inv_pos_in.alloc(cap));
    CUDA_TRY(ctx->inv_pos.alloc(cap));
    size_t tb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, (const K *)nullptr, (K *)nullptr, (const int *)nullptr, (int *)nullptr,
                                    (int)cap, 0, 8 * (int)sizeof(K), ctx->stream);
    if (ctx->inv_tmp_bytes < tb + 256) { ctx->inv_tmp_bytes = tb + 256; CUDA_TRY(ctx->inv_tmp.alloc(ctx->inv_tmp_bytes)); }
  }
  K *ids_in = reinterpret_cast<K *>(ctx->inv_ids_in.p), *ids = reinterpret_cast<K *>(ctx->inv_ids.p);
  k_inv_ids<<<grid_for(cap, 256), 256, 0, ctx->stream>>>(ctx->E, ctx->A, ctx->P, ctx->inv_dense, n_ids, spread, ctx->y.p,
                                                       ctx->blk_sorted.p, ctx->ent_sorted.p, ctx->ent_ptr.p,
                                                       ctx->perm_dev.p, ids_in, ctx->inv_pos_in.p);
  size_t tb = ctx->inv_tmp_bytes;
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(ctx->inv_tmp.p, tb, (const K *)ids_in, ids, (const int *)ctx->inv_pos_in.p,
                                           ctx->inv_pos.p, (int)cap, 0, bits, ctx->stream));
  ctx->launches += 4;
  return DBL_OK;
}

// (block, attribute, value) -> candidate positions, for k_link_pruned.  One index whatever the sizes: 32-bit ids when
// the id space and the sentinel spread fit, 64-bit otherwise.  When the dense pointer table is small enough (P * sum
// of vocabulary sizes entries) a record finds its posting list with two loads; otherwise with two binary searches in
// its block's range of the sorted ids.  No size depends on the shard: nothing is read back.
static int ensure_inverted_index(dbl_ctx *ctx) {
  if (ctx->inv_valid) return DBL_OK;
  const int64_t cap = ctx->E * ctx->A;
  if (cap > 0x7fffffff) { ctx->set_error("inverted index too large"); return DBL_ERR_INVALID; }
  InvDense &dn = ctx->inv_dense;
  dn.A = ctx->A; dn.sumV = 0;
  for (int k = 0; k < ctx->A; ++k) { dn.voff[k] = dn.sumV; dn.sumV += ctx->h_attrs[ctx->perm[k]].V; }
  const long long n_ids = (long long)ctx->P * dn.sumV;
  int bits;
  long long spread;
  sentinel_spread(n_ids, ctx->world, &bits, &spread);
  ctx->inv_ids64 = bits > 32;
  int rc = ctx->inv_ids64 ? sort_inverted_index<unsigned long long>(ctx, n_ids, spread, bits)
                          : sort_inverted_index<unsigned>(ctx, n_ids, spread, bits);
  if (rc) return rc;
  long long dense_max = 1ll << 25;  // entries; DBL_INV_DENSE_MAX overrides (tests force the binary-search path with 0)
  if (const char *ev = getenv("DBL_INV_DENSE_MAX")) dense_max = atoll(ev);
  ctx->inv_use_dense = !ctx->inv_ids64 && n_ids <= dense_max;  // 64-bit ids: a table of more than 2^32 entries
  if (ctx->inv_use_dense) {
    if (ctx->inv_vptr.n != (size_t)n_ids + 1) CUDA_TRY(ctx->inv_vptr.alloc((size_t)n_ids + 1));
    k_inv_value_ptr32<<<grid_for(cap + 1, 256), 256, 0, ctx->stream>>>(cap, n_ids, (long long)dn.sumV,
                                                                       (const unsigned *)ctx->inv_ids.p, ctx->inv_vptr.p);
    ctx->launches += 1;
  }
  ctx->inv_valid = true;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

static bool pcg2_kernel_fits(const dbl_ctx *ctx) {
  return ctx->hslots > 0 && ctx->A <= LINK_MAX_UNROLL_A &&
         pcg2_smem_bytes(ctx->pcg2_fmt, ctx->A, ctx->n_str, ctx->hslots, false) <= 100 * 1024;
}
static int dispatch_pcg2(dbl_ctx *ctx, const LinkParams *lp, int grid = 0) {
  Pcg2Kernel k = nullptr;
  switch (ctx->A) {
#define DBL_CASE(N) case N: k = dbl_pcg2_kernel_a##N(ctx->n_str, ctx->pcg2_fmt); break;
    DBL_CASE(1) DBL_CASE(2) DBL_CASE(3) DBL_CASE(4) DBL_CASE(5) DBL_CASE(6) DBL_CASE(7) DBL_CASE(8)
    DBL_CASE(9) DBL_CASE(10) DBL_CASE(11) DBL_CASE(12) DBL_CASE(13) DBL_CASE(14) DBL_CASE(15) DBL_CASE(16)
#undef DBL_CASE
  }
  const size_t smem = pcg2_smem_bytes(ctx->pcg2_fmt, ctx->A, ctx->n_str, ctx->hslots, ctx->tile_invn.p != nullptr);
  const int rc = pcg2_launch(k, smem, lp, grid, ctx->stream, &ctx->pcg2_smem_cfg);
  if (rc != 0) { ctx->set_error(std::string("k_link_pcg2 launch: ") + cudaGetErrorString((cudaError_t)rc)); return DBL_ERR_CUDA; }
  return DBL_OK;
}

// the link kernel a sweep with this sampler launches, numbered as dbl_link_kernel reports it
enum LinkKernel { LINK_GENERIC = 0, LINK_MATCH = 1, LINK_PRUNED = 2, LINK_PCG2 = 3 };
static LinkKernel link_kernel(const dbl_ctx *ctx, int sampler) {
  const int mode = ctx->link_mode;  // 0 auto, 1 force generic, 2 dense kernels for every sampler
  if (mode != 1 && sampler == DBL_PCG_II && pcg2_kernel_fits(ctx)) return LINK_PCG2;
  if (mode == 0 && sampler != DBL_PCG_II) return LINK_PRUNED;
  if (mode != 1 && sampler != DBL_PCG_II) return LINK_MATCH;
  return LINK_GENERIC;
}

static int launch_link(dbl_ctx *ctx, int sampler) {
  const int A = ctx->A;
  LinkParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.A = A; lp.F = ctx->F; lp.P = ctx->P; lp.sampler = sampler; lp.seed = ctx->seed; lp.ctl = ctx->ctl();
  lp.attrs = ctx->attrs.p; lp.x = ctx->x.p; lp.file = ctx->file.p; lp.link = ctx->link.p; lp.zmask = ctx->zmask.p;
  lp.theta = ctx->theta(); lp.ent_ptr = ctx->ent_ptr.p; lp.tile_ptr = ctx->tile_ptr.p; lp.rec_ptr = ctx->rec_ptr.p;
  lp.cta_ptr = ctx->cta_ptr.p; lp.ent_sorted = ctx->ent_sorted.p; lp.rec_sorted = ctx->rec_sorted.p;
  lp.tiles = ctx->tiles.p; lp.newlink = ctx->newlink.p;
  lp.work = reinterpret_cast<unsigned long long *>(ctx->ctl() + CTL_WORK);
  lp.lane_sums = ctx->lane_sums.p;
  lp.status = reinterpret_cast<unsigned long long *>(ctx->ctl() + CTL_STATUS);
  lp.pairs = reinterpret_cast<unsigned long long *>(ctx->ctl() + CTL_PAIRS);
  for (int k = 0; k < A; ++k) lp.perm[k] = ctx->perm[k];
  lp.chain_seeds = ctx->chain_map().seeds;
  lp.chain_recs = ctx->chain_map().recs;
  if (ctx->link_mass_on) {
    if (ctx->link_mass.n != (size_t)ctx->R) {  // the first sweep of a kind runs eagerly: never inside a graph capture
      CUDA_TRY(ctx->link_mass.alloc((size_t)ctx->R));
      CUDA_TRY(cudaMemsetAsync(ctx->link_mass.p, 0, sizeof(double) * (size_t)ctx->R, ctx->stream));
    }
    // a shard scores only the records it owns; every other entry keeps the all-ones pattern, a NaN no kernel stores
    if (ctx->world > 1)
      CUDA_TRY(cudaMemsetAsync(ctx->link_mass.p, 0xFF, sizeof(double) * (size_t)ctx->R, ctx->stream));
    lp.link_mass = ctx->link_mass.p;
  }
  lp.hslots = ctx->hslots; lp.hshift = ctx->hshift;
  const LinkKernel kernel = link_kernel(ctx, sampler);
  if (kernel == LINK_PCG2) {
    // persistent CTAs: a few per SM, each takes groups of LINK_WARPS records from the work counter until none is left
    // (k_theta zeroed the counter; the block-level API launches the kernel once per block after one k_theta)
    if (ctx->in_block_sweep) CUDA_TRY(cudaMemsetAsync(lp.work, 0, sizeof(unsigned long long), ctx->stream));
    int rc = ensure_tiles(ctx, ctx->pcg2_fmt, true);
    if (rc) return rc;
    lp.tile_invn = ctx->tile_invn.p;
    lp.cta_ptr = ctx->cta_ptr3.p;  // work items of PCG2_RECS records
    return dispatch_pcg2(ctx, &lp, std::min(ctx->max_ctas, ctx->pcg2_grid));
  }
  {
    int rc = ensure_tiles(ctx, Pcg2Format{});  // every other link kernel reads the unpacked format
    if (rc) return rc;
  }
  if (kernel == LINK_PRUNED) {  // pruned scoring through the inverted index
    int rc = ensure_inverted_index(ctx);
    if (rc) return rc;
    PrunedParams pp;
    pp.lp = lp;
    pp.inv_pos = ctx->inv_pos.p;
    pp.rec_key_sorted = ctx->rec_key_sorted.p;
    pp.rec_key_shift = REC_CLASS_BITS;
    pp.inv_vptr = ctx->inv_use_dense ? ctx->inv_vptr.p : nullptr;
    pp.inv_key32 = ctx->inv_ids64 ? nullptr : reinterpret_cast<const unsigned *>(ctx->inv_ids.p);
    pp.inv_key64 = ctx->inv_ids64 ? reinterpret_cast<const unsigned long long *>(ctx->inv_ids.p) : nullptr;
    pp.sumV = ctx->inv_dense.sumV;
    for (int k = 0; k < A; ++k) pp.voff[k] = ctx->inv_dense.voff[k];
    if (ctx->heavy_list.n != (size_t)ctx->R) CUDA_TRY(ctx->heavy_list.alloc((size_t)ctx->R));
    pp.heavy_list = ctx->heavy_list.p;
    if (ctx->in_block_sweep)  // the block-level API launches once per block after one k_theta
      CUDA_TRY(cudaMemsetAsync(ctx->ctl() + CTL_HEAVY, 0, sizeof(long long), ctx->stream));
    k_link_pruned<<<(int)std::min<int64_t>(grid_for(ctx->R, LINK_WARPS), (int64_t)ctx->sm_count * 16), LINK_WARPS * 32, 0,
                    ctx->stream>>>(pp);
    // records whose whole block has to be scored (no must-match attribute), a CTA each; usually none: the kernel
    // reads the count and returns
    k_link_heavy<<<ctx->sm_count * 2, HEAVY_WARPS * 32, 0, ctx->stream>>>(pp);
    ctx->launches += 1;
    return DBL_OK;
  }
  if (kernel == LINK_MATCH) {
    const size_t ring = (size_t)LINK_STAGES * TileLayout::of(A).words() * 4 + 128;  // the tile ring of k_link_match
    if (ctx->match_smem_cfg < ring) {
      CUDA_TRY(cudaFuncSetAttribute(k_link_match, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ring));
      ctx->match_smem_cfg = ring;
    }
    lp.cta_ptr = ctx->cta_ptr2.p;  // MATCH_WARPS records per CTA
    const int grid = (int)((ctx->R + MATCH_WARPS - 1) / MATCH_WARPS) + ctx->P;
    k_link_match<<<grid, (MATCH_WARPS + 1) * 32, ring, ctx->stream>>>(lp);
    return DBL_OK;
  }
  k_link_generic<<<ctx->max_ctas, LINK_WARPS * 32, 0, ctx->stream>>>(lp);
  return DBL_OK;
}

// ---------------------------------------------------------------------------------------------------
// one application of State.nextState (State.scala:78-99), enqueued on the context's stream without any host
// synchronisation
// ---------------------------------------------------------------------------------------------------
// (1) theta | summary of the previous state (State.scala:83, GU:305-320)
static int enqueue_theta(dbl_ctx *ctx) {
  k_theta<<<1, 128, 0, ctx->stream>>>(ctx->A, ctx->F, ctx->seed, ctx->chain_map().seeds, ctx->F1, ctx->ctl(), ctx->glob(),
                                       ctx->prior.p,
                                       ctx->prior.p + ctx->A, ctx->prior.p + 2 * ctx->A, ctx->theta(), ctx->theta_prev(),
                                       ctx->part(), ctx->nw);
  ctx->launches += 1;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

// (2)-(4) for the owned entities / records (all of them on an unsharded context): updatePartition, GU:156-211
static int update_owned(dbl_ctx *ctx, int sampler) {
  const int A = ctx->A, F = ctx->F;
  // (2) links
  const bool timed = ctx->cur_timed;
  if (timed) CUDA_TRY(cudaEventRecord(ctx->cur_events.e[0], ctx->stream));
  {
    int rc = launch_link(ctx, sampler);
    if (rc) return rc;
  }
  if (timed) CUDA_TRY(cudaEventRecord(ctx->cur_events.e[1], ctx->stream));
  ctx->launches += 1;
  CUDA_TRY(cudaGetLastError());
  // (3) entity values (the links are committed by the first kernel of the CSR build)
  int rc = build_links_csr(ctx, true);
  if (rc) return rc;
  ValParams vp;
  vp.A = A; vp.F = F; vp.sampler = sampler; vp.seed = ctx->seed; vp.cm = ctx->chain_map(); vp.rows = rows_prefix(ctx, true);
  vp.attrs = ctx->attrs.p; vp.x = ctx->x.p; vp.file = ctx->file.p; vp.zmask = ctx->zmask.p; vp.theta = ctx->theta();
  vp.ent_rec_ptr = ctx->ent_rec_ptr.p; vp.rec_by_ent = ctx->rec_by_ent.p; vp.y = ctx->y.p;
  if (ctx->far_list.n != (size_t)(ctx->E * A)) CUDA_TRY(ctx->far_list.alloc((size_t)(ctx->E * A)));
  vp.far_list = ctx->far_list.p;
  // latency-bound sizes (the grid does not fill the GPU a few times over): the variant with batched loads
  if (ctx->E * A <= (int64_t)ctx->sm_count * 2048 * 4) k_values<8><<<grid_rows(ctx, ctx->E * A, 128), 128, 0, ctx->stream>>>(vp);
  else k_values<VALUES_UB_LARGE><<<grid_rows(ctx, ctx->E * A, 128), 128, 0, ctx->stream>>>(vp);
  k_values_rescaled<<<1, 128, 0, ctx->stream>>>(vp);
  ctx->launches += 2;
  // (4) N(e), new block ids, distortions, partial summary
  return refresh_summary(ctx, true);
}

// the messages of the clusters whose new block belongs to another rank, written through `out` by the rank that owned
// them and applied from `in` by the one that receives them (either transport).  max_*: the most messages `in` can hold.
static void launch_move(dbl_ctx *ctx, const MsgOut &out) {
  MoveParams mp;
  mp.rank = ctx->rank; mp.out = out; mp.ctl = ctx->ctl(); mp.A = ctx->A;
  mp.ent_sorted = ctx->ent_sorted.p; mp.rec_sorted = ctx->rec_sorted.p;
  mp.blk = ctx->blk.p; mp.owner = ctx->owner.p; mp.link = ctx->link.p; mp.y = ctx->y.p; mp.zmask = ctx->zmask.p;
  mp.ent_dest = ctx->ent_dest.p; mp.ent_owned = ctx->ent_owned.p; mp.rec_owned = ctx->rec_owned.p;
  k_move_ent<<<grid_rows(ctx, ctx->E, 256), 256, 0, ctx->stream>>>(mp);
  k_move_rec<<<grid_rows(ctx, ctx->R, 256), 256, 0, ctx->stream>>>(mp);
  ctx->launches += 2;
}
static void launch_unpack(dbl_ctx *ctx, const MsgIn &in, int64_t max_ent, int64_t max_rec) {
  UnpackParams up;
  up.in = in; up.ctl = ctx->ctl(); up.A = ctx->A; up.attrs = ctx->attrs.p; up.tree = ctx->tree; up.y = ctx->y.p;
  up.blk = ctx->blk.p; up.link = ctx->link.p; up.entN = ctx->entN.p; up.zmask = ctx->zmask.p;
  up.ent_owned = ctx->ent_owned.p; up.rec_owned = ctx->rec_owned.p;
  k_unpack_ent<<<grid_rows(ctx, max_ent, 256), 256, 0, ctx->stream>>>(up);
  k_unpack_rec<<<grid_rows(ctx, max_rec, 256), 256, 0, ctx->stream>>>(up);
  ctx->launches += 2;
}

// (5) the shuffle (GU:144) + the global summary (SummaryAccumulators.scala:54-63), peer to peer
static int exchange_p2p(dbl_ctx *ctx) {
  launch_move(ctx, ctx->p2p_out);
  k_publish_barrier<<<1, 256, 0, ctx->stream>>>(ctx->comm, ctx->ctl(), ctx->part(), ctx->nw, ctx->barrier_timeout_cycles);
  launch_unpack(ctx, ctx->p2p_in, ctx->E, ctx->R);
  k_reduce_peers<<<1, 256, 0, ctx->stream>>>(ctx->comm, ctx->ctl(), ctx->nw, ctx->ll_slot(), ctx->glob());
  ctx->launches += 2;
  if (ctx->rebalance_period > 0 && ctx->P <= 1024) {
    k_lpt<<<1, 32, 0, ctx->stream>>>(ctx->P, ctx->world, ctx->blk_ent_slot(), ctx->blk_rec_slot(), ctx->glob(), ctx->ctl(),
                                     ctx->rebalance_period, ctx->rebalance_threshold, ctx->owner.p, ctx->lpt_scratch.p,
                                     ctx->lpt_dscratch.p);
    ctx->launches += 1;
  }
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

static int enqueue_sweep_phases(dbl_ctx *ctx, int sampler) {
  const bool timed = ctx->cur_timed;
  int rc = enqueue_theta(ctx);
  if (rc) return rc;
  rc = update_owned(ctx, sampler);
  if (rc) return rc;
  if (timed) CUDA_TRY(cudaEventRecord(ctx->cur_events.e[2], ctx->stream));
  if (ctx->world > 1) {
    rc = exchange_p2p(ctx);
    if (rc) return rc;
  }
  if (timed) CUDA_TRY(cudaEventRecord(ctx->cur_events.e[3], ctx->stream));
  rc = relayout(ctx, true);  // + global summary of a single rank, + iteration count
  if (rc) return rc;
  if (timed) CUDA_TRY(cudaEventRecord(ctx->cur_events.e[4], ctx->stream));
  return DBL_OK;
}

static int enqueue_sweep(dbl_ctx *ctx, int sampler) {
  ctx->cur_timed = !ctx->capturing && ctx->pending_events.size() < 256;  // per-phase timing (eager sweeps only)
  if (ctx->cur_timed) {
    if (!ctx->event_pool.empty()) { ctx->cur_events = ctx->event_pool.back(); ctx->event_pool.pop_back(); }
    else for (cudaEvent_t &e : ctx->cur_events.e) CUDA_TRY(cudaEventCreate(&e));
  }
  const int rc = enqueue_sweep_phases(ctx, sampler);
  if (ctx->cur_timed) (rc ? ctx->event_pool : ctx->pending_events).push_back(ctx->cur_events);
  ctx->cur_timed = false;
  return rc;
}

static int check_sweep_args(dbl_ctx *ctx, int sampler, int32_t n_sweeps) {
  if (sampler < 0 || sampler > 3 || n_sweeps < 0) { ctx->set_error("bad sampler / n_sweeps"); return DBL_ERR_INVALID; }
  if (!ctx->has_state) { ctx->set_error("dbl_sweep before dbl_state_init/upload"); return DBL_ERR_STATE; }
  if (ctx->world > 1 && !ctx->comm_ready) {
    ctx->set_error("dbl_sweep on a sharded context needs dbl_comm_export / dbl_comm_import first "
                   "(or drive the host-mediated exchange: dbl_sweep_begin / dbl_exchange_* / dbl_sweep_end)");
    return DBL_ERR_STATE;
  }
  if (ctx->world > 1 && ctx->all_owned) { ctx->set_error("dbl_sweep on a sharded context before dbl_set_block_owners"); return DBL_ERR_STATE; }
  if (ctx->in_sweep) { ctx->set_error("dbl_sweep inside an open sweep"); return DBL_ERR_STATE; }
  return DBL_OK;
}

// Launch-bound sizes (RLdata-sized problems: a sweep is ~50 tiny kernels) replay one captured sweep instead of
// enqueueing it again: nothing in a sweep depends on the host, every varying quantity is read from device memory.
static bool graph_allowed(const dbl_ctx *ctx, int sampler) {
  if (ctx->graph_mode == 1) return false;
  if (ctx->graph_mode == 2) return true;
  // PCG-II at large sizes: tens of milliseconds of GPU time per sweep hide the ~35 launches.  The pruned samplers
  // do not: their sweep is ~3 ms of GPU time at 1 M records and shrinks with the rank count while the host's share
  // (launches, CUB set-up) does not: with 8 processes on a 16-CPU quota the eager sweeps on 8 GPUs were host-bound.
  return ctx->R + ctx->E <= 400000 || sampler != DBL_PCG_II;
}

static int run_sweeps(dbl_ctx *ctx, int sampler, int32_t n_sweeps) {
  int s = 0;
  if (n_sweeps >= 2 && graph_allowed(ctx, sampler)) {
    const int key = sampler * 4 + ctx->link_mode;
    if (!ctx->graph_warm[key]) {  // first sweep of this kind eagerly: allocations and opt-ins happen outside a capture
      int rc = enqueue_sweep(ctx, sampler);
      if (rc) return rc;
      ctx->graph_warm[key] = true;
      s = 1;
    }
    auto it = ctx->graphs.find(key);
    if (it == ctx->graphs.end() && n_sweeps - s >= 2) {
      dbl_ctx::SweepGraph g;
      const int64_t before = ctx->launches;
      CUDA_TRY(cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal));
      ctx->capturing = true;
      int rc = enqueue_sweep(ctx, sampler);
      ctx->capturing = false;
      cudaError_t e = cudaStreamEndCapture(ctx->stream, &g.graph);
      g.launches = ctx->launches - before;
      ctx->launches = before;
      if (rc) { if (g.graph) cudaGraphDestroy(g.graph); return rc; }
      if (e != cudaSuccess) { ctx->set_error(std::string("graph capture: ") + cudaGetErrorString(e)); return DBL_ERR_CUDA; }
      CUDA_TRY(cudaGraphInstantiate(&g.exec, g.graph, 0));
      it = ctx->graphs.emplace(key, g).first;
    }
    if (it != ctx->graphs.end())
      for (; s < n_sweeps; ++s) {
        CUDA_TRY(cudaGraphLaunch(it->second.exec, ctx->stream));
        ctx->launches += it->second.launches;
      }
  }
  for (; s < n_sweeps; ++s) {
    int rc = enqueue_sweep(ctx, sampler);
    if (rc) return rc;
  }
  return DBL_OK;
}

extern "C" int dbl_sweep_async(dbl_ctx *ctx, int sampler, int32_t n_sweeps) {
  if (!ctx) return DBL_ERR_INVALID;
  int rc = check_sweep_args(ctx, sampler, n_sweeps);
  if (rc) return rc;
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (!ctx->async_open) CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
  ctx->async_open = true;
  t_deferred_free = ctx->world > 1 ? &ctx->deferred_free : nullptr;
  rc = run_sweeps(ctx, sampler, n_sweeps);
  t_deferred_free = nullptr;
  return rc;
}

extern "C" int dbl_set_graph_mode(dbl_ctx *ctx, int mode) {
  if (!ctx || mode < 0 || mode > 2) return DBL_ERR_INVALID;
  ctx->graph_mode = mode;
  return DBL_OK;
}

extern "C" int dbl_sync(dbl_ctx *ctx) {
  if (!ctx) return DBL_ERR_INVALID;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  const bool timed = ctx->async_open;
  if (timed) CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
  ctx->async_open = false;
  int rc = snapshot(ctx);
  if (timed) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_sweep_ms = ms;
  }
  return rc;
}

extern "C" int dbl_sweep(dbl_ctx *ctx, int sampler, int32_t n_sweeps) {
  if (!ctx) return DBL_ERR_INVALID;
  if (ctx->async_open) { ctx->set_error("dbl_sweep with asynchronous sweeps pending: call dbl_sync first"); return DBL_ERR_STATE; }
  int rc = dbl_sweep_async(ctx, sampler, n_sweeps);
  if (rc) { ctx->async_open = false; return rc; }
  return dbl_sync(ctx);
}

// ---------------------------------------------------------------------------------------------------
// block-level entry points: one call per k-d-tree block, mirroring GibbsUpdates.updatePartition (GU:156-211)
// ---------------------------------------------------------------------------------------------------
extern "C" int dbl_block_sweep_begin(dbl_ctx *ctx, int sampler) {
  if (!ctx) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_block_sweep_begin")) return rc1;
  if (sampler < 0 || sampler > 3) { ctx->set_error("bad sampler"); return DBL_ERR_INVALID; }
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  if (ctx->world > 1) { ctx->set_error("block-level sweeps need an unsharded context"); return DBL_ERR_STATE; }
  if (ctx->in_sweep || ctx->async_open) { ctx->set_error("a sweep is already open"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
  int rc = enqueue_theta(ctx);
  if (rc) return rc;
  // block membership is fixed for the whole sweep (the shuffle happens after every partition was updated, GU:144)
  CUDA_TRY(ctx->blk_frozen.alloc(ctx->E));
  CUDA_TRY(cudaMemcpyAsync(ctx->blk_frozen.p, ctx->blk.p, sizeof(int) * ctx->E, cudaMemcpyDeviceToDevice, ctx->stream));
  ctx->block_done.assign(ctx->P, 0);
  ctx->block_sampler = sampler;
  ctx->in_sweep = true;
  ctx->in_block_sweep = true;
  return DBL_OK;
}

extern "C" int dbl_update_block(dbl_ctx *ctx, int32_t block_id) {
  if (!ctx) return DBL_ERR_INVALID;
  if (!ctx->in_block_sweep) { ctx->set_error("dbl_update_block outside dbl_block_sweep_begin/end"); return DBL_ERR_STATE; }
  if (block_id < 0 || block_id >= ctx->P) { ctx->set_error("block id out of range"); return DBL_ERR_INVALID; }
  if (ctx->block_done[block_id]) { ctx->set_error("block already updated in this sweep"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  k_mark_ent_block<<<grid_for(ctx->E, 256), 256, 0, ctx->stream>>>(ctx->E, ctx->blk_frozen.p, block_id, ctx->ent_owned.p);
  k_mark_rec_owned<<<grid_for(ctx->R, 256), 256, 0, ctx->stream>>>(ctx->R, ctx->link.p, ctx->ent_owned.p,
                                                                  ctx->rec_owned.p);
  ctx->launches += 2;
  int rc = relayout(ctx);  // tiles of this block only (everything else sorts into the dummy block)
  if (rc) return rc;
  rc = update_owned(ctx, ctx->block_sampler);
  if (rc) return rc;
  ctx->block_done[block_id] = 1;
  return DBL_OK;
}

extern "C" int dbl_block_sweep_end(dbl_ctx *ctx) {
  if (!ctx) return DBL_ERR_INVALID;
  if (!ctx->in_block_sweep) { ctx->set_error("dbl_block_sweep_end without dbl_block_sweep_begin"); return DBL_ERR_STATE; }
  for (int b = 0; b < ctx->P; ++b)
    if (!ctx->block_done[b]) { ctx->set_error("dbl_block_sweep_end: not every block was updated"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  ctx->in_sweep = ctx->in_block_sweep = false;
  CUDA_TRY(cudaMemsetAsync(ctx->ent_owned.p, 1, ctx->E, ctx->stream));
  CUDA_TRY(cudaMemsetAsync(ctx->rec_owned.p, 1, ctx->R, ctx->stream));
  int rc = build_links_csr(ctx);
  if (rc) return rc;
  rc = refresh_summary(ctx, false);  // summary of the whole state (updateSummaryVariables, GU:219-301)
  if (rc) return rc;
  rc = adopt_local_summary(ctx);
  if (rc) return rc;
  rc = relayout(ctx);  // the shuffle: regroup by the new block ids
  if (rc) return rc;
  k_finish<<<1, 32, 0, ctx->stream>>>(ctx->ctl());
  ctx->launches += 1;
  CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
  rc = snapshot(ctx);
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_sweep_ms = ms;
  return rc;
}

// ---------------------------------------------------------------------------------------------------
// multi-GPU entry points: blocks are sharded over ranks; one exchange of moved clusters per sweep
// ---------------------------------------------------------------------------------------------------
static int apply_ownership(dbl_ctx *ctx) {
  k_mark_ent_owned<<<grid_for(ctx->E, 256), 256, 0, ctx->stream>>>(ctx->E, ctx->blk.p, ctx->owner.p, ctx->rank,
                                                                  ctx->ent_owned.p);
  k_mark_rec_owned<<<grid_for(ctx->R, 256), 256, 0, ctx->stream>>>(ctx->R, ctx->link.p, ctx->ent_owned.p,
                                                                  ctx->rec_owned.p);
  ctx->launches += 2;
  CUDA_TRY(cudaGetLastError());
  return DBL_OK;
}

extern "C" int dbl_set_block_owners(dbl_ctx *ctx, const int32_t *owner_of_block) {
  if (!ctx) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_set_block_owners")) return rc1;
  if (!ctx->has_state) { ctx->set_error("set_block_owners needs a (replicated) state"); return DBL_ERR_STATE; }
  if (!ctx->all_owned) { ctx->set_error("set_block_owners needs the replicated state: upload / init it again first"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (owner_of_block) {  // NULL = the table the context already holds on the device (the device-side LPT may have changed it)
    for (int b = 0; b < ctx->P; ++b)
      if (owner_of_block[b] < 0 || owner_of_block[b] >= ctx->world) { ctx->set_error("owner out of range"); return DBL_ERR_INVALID; }
    ctx->owner_h.assign(owner_of_block, owner_of_block + ctx->P);
    CUDA_TRY(cudaMemcpyAsync(ctx->owner.p, ctx->owner_h.data(), sizeof(int) * ctx->P, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  }
  int rc = apply_ownership(ctx);
  if (rc) return rc;
  ctx->all_owned = (ctx->world <= 1);
  rc = build_links_csr(ctx);  // of the shard; the global summary (of the replicated state) stays
  if (rc) return rc;
  rc = relayout(ctx);
  if (rc) return rc;
  return snapshot(ctx);
}

extern "C" int dbl_block_owners(dbl_ctx *ctx, int32_t *owner_out) {
  if (!ctx || !owner_out) return DBL_ERR_INVALID;
  if (!ctx->owner.p) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaMemcpyAsync(owner_out, ctx->owner.p, sizeof(int) * ctx->P, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

extern "C" int dbl_set_rebalance(dbl_ctx *ctx, int32_t period, double threshold) {
  if (!ctx || period < 0 || !(threshold >= 1.0)) return DBL_ERR_INVALID;
  ctx->drop_graphs();
  ctx->rebalance_period = period;
  ctx->rebalance_threshold = threshold;
  return DBL_OK;
}

// With lazy module loading (the CUDA default) the FIRST launch of a kernel may synchronise the whole context.  Inside a
// sharded sweep that is fatal when several ranks share one device (the tests do): rank A waits in the exchange barrier
// for rank B, whose next launch waits for A's barrier kernel to finish.  So every kernel a sweep can launch is loaded
// here, before the first sharded sweep (and before any graph capture): by attribute query for our own kernels, by
// running the (idempotent) layout / index builds once for the CUB kernels they use.
static int preload_kernels(dbl_ctx *ctx) {
  cudaFuncAttributes fa;
#define DBL_LOAD(k) CUDA_TRY(cudaFuncGetAttributes(&fa, k))
  DBL_LOAD(k_theta); DBL_LOAD(k_link_heavy); DBL_LOAD(k_commit_link_keys); DBL_LOAD(k_build_entity_tiles); DBL_LOAD(k_values<VALUES_UB_LARGE>); DBL_LOAD(k_values<8>); DBL_LOAD(k_values_rescaled); DBL_LOAD(k_entity_post); DBL_LOAD(k_dist);
  DBL_LOAD(k_reduce_local); DBL_LOAD(k_finish); DBL_LOAD(k_move_ent); DBL_LOAD(k_move_rec); DBL_LOAD(k_publish_barrier);
  DBL_LOAD(k_unpack_ent); DBL_LOAD(k_unpack_rec); DBL_LOAD(k_reduce_peers); DBL_LOAD(k_lpt);
  DBL_LOAD(k_link_generic); DBL_LOAD(k_link_match); DBL_LOAD(k_link_pruned); DBL_LOAD(k_state_hash);
  DBL_LOAD(k_gather_ent); DBL_LOAD(k_gather_rec); DBL_LOAD(k_export_ent); DBL_LOAD(k_export_rec);
  DBL_LOAD(k_inv_ids<unsigned>); DBL_LOAD(k_inv_ids<unsigned long long>); DBL_LOAD(k_inv_value_ptr32);
#undef DBL_LOAD
  if (pcg2_kernel_fits(ctx)) {
    int rc = dispatch_pcg2(ctx, nullptr);
    if (rc) return rc;
  }
  int rc = build_links_csr(ctx);
  if (rc) return rc;
  ctx->inv_valid = false;
  rc = ensure_inverted_index(ctx);
  if (rc) return rc;
  rc = relayout(ctx);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

// ---- peer-to-peer communicator ------------------------------------------------------------------------------
static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

extern "C" int dbl_comm_export(dbl_ctx *ctx, void *blob_out) {
  if (!ctx || !blob_out) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_comm_export")) return rc1;
  if (!ctx->has_state) { ctx->set_error("dbl_comm_export needs a state (the buffers are sized by it)"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  comm_close(ctx);
  ctx->drop_graphs();
  ctx->free_deferred();
  CommDev &c = ctx->comm;
  memset(&c, 0, sizeof(c));
  c.rank = ctx->rank; c.world = ctx->world; c.A = ctx->A; c.nws = ctx->nw + 1;
  c.cap_e = ctx->E; c.cap_r = ctx->R;
  c.off_cursor = 256;
  c.off_slots = 512;
  c.off_ent = align_up(c.off_slots + 2 * (size_t)c.world * c.nws * 8, 256);
  c.off_rec = align_up(c.off_ent + 2 * (size_t)c.cap_e * (c.A + 1) * 4, 256);
  const size_t bytes = align_up(c.off_rec + 2 * (size_t)c.cap_r * 3 * 4, 256);
  if (ctx->comm_bytes != bytes || !ctx->comm_buf.p) {
    CUDA_TRY(ctx->comm_buf.alloc(bytes));
    ctx->comm_bytes = bytes;
  }
  CUDA_TRY(cudaMemset(ctx->comm_buf.p, 0, 512 + 2 * (size_t)c.world * c.nws * 8));
  long long zero = 0;  // barrier epochs restart with the buffers
  CUDA_TRY(cudaMemcpy(ctx->ctl() + CTL_EPOCH, &zero, sizeof(zero), cudaMemcpyHostToDevice));
  CommBlob b;
  memset(&b, 0, sizeof(b));
  b.magic = COMM_MAGIC; b.rank = ctx->rank; b.world = ctx->world; b.device = ctx->device;
  b.pid = (int64_t)getpid();
  b.ptr = (uint64_t)(uintptr_t)ctx->comm_buf.p;
  b.bytes = bytes; b.E = ctx->E; b.R = ctx->R; b.A = ctx->A; b.nws = c.nws;
  if (ctx->world > 1 && cudaIpcGetMemHandle(&b.handle, ctx->comm_buf.p) != cudaSuccess) {
    // no IPC on this system: ranks living in this process still reach the buffer through b.ptr; a rank in another
    // process will fail in dbl_comm_import and the host layer falls back to the host-mediated exchange
    cudaGetLastError();
    memset(&b.handle, 0, sizeof(b.handle));
  }
  memcpy(blob_out, &b, sizeof(b));
  return DBL_OK;
}

extern "C" int dbl_comm_import(dbl_ctx *ctx, const void *blobs, int32_t world) {
  if (!ctx || !blobs) return DBL_ERR_INVALID;
  if (world != ctx->world) { ctx->set_error("dbl_comm_import: world size differs from the context's"); return DBL_ERR_INVALID; }
  if (!ctx->comm_buf.p) { ctx->set_error("dbl_comm_import before dbl_comm_export"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  const CommBlob *bl = static_cast<const CommBlob *>(blobs);
  for (int r = 0; r < world; ++r) {
    CommBlob b;
    memcpy(&b, &bl[r], sizeof(b));
    if (b.magic != COMM_MAGIC || b.rank != r || b.world != world || b.E != ctx->E || b.R != ctx->R || b.A != ctx->A ||
        b.nws != ctx->comm.nws || b.bytes != ctx->comm_bytes) {
      ctx->set_error("dbl_comm_import: blob " + std::to_string(r) + " does not describe a matching rank");
      return DBL_ERR_INVALID;
    }
    if (r == ctx->rank) {
      ctx->comm.base[r] = ctx->comm_buf.p;
    } else if (b.pid == (int64_t)getpid()) {  // several ranks in one process (tests): plain pointers
      if (b.device != ctx->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { ctx->set_error("no peer access between the devices"); return DBL_ERR_CUDA; }
        cudaGetLastError();
      }
      ctx->comm.base[r] = reinterpret_cast<unsigned char *>((uintptr_t)b.ptr);
    } else {
      void *p = nullptr;
      cudaError_t e = cudaIpcOpenMemHandle(&p, b.handle, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        ctx->set_error(std::string("cudaIpcOpenMemHandle (rank ") + std::to_string(r) + "): " + cudaGetErrorString(e));
        comm_close(ctx);
        return DBL_ERR_CUDA;
      }
      ctx->ipc_opened.push_back(p);
      ctx->comm.base[r] = static_cast<unsigned char *>(p);
    }
  }
  const CommDev &c = ctx->comm;
  for (int par = 0; par < 2; ++par) {
    for (int d = 0; d < world; ++d) {
      ctx->p2p_out.ent[d][par] = c.recv_ent(d, par);
      ctx->p2p_out.rec[d][par] = c.recv_rec(d, par);
      ctx->p2p_out.cursor[d][par] = c.cursor(d, par);
    }
    ctx->p2p_in.ent[par] = c.recv_ent(ctx->rank, par);
    ctx->p2p_in.rec[par] = c.recv_rec(ctx->rank, par);
    ctx->p2p_in.count[par] = c.cursor(ctx->rank, par);
  }
  ctx->drop_graphs();
  if (ctx->has_state) { int rc = preload_kernels(ctx); if (rc) return rc; }
  ctx->comm_ready = true;
  return DBL_OK;
}

extern "C" int dbl_last_exchange(dbl_ctx *ctx, int64_t *ent_msgs, int64_t *rec_msgs, int64_t *replacements) {
  if (!ctx || !ctx->h_cb) return DBL_ERR_INVALID;
  if (ent_msgs) *ent_msgs = ctx->h_ctl()[CTL_MOVED_ENT];
  if (rec_msgs) *rec_msgs = ctx->h_ctl()[CTL_MOVED_REC];
  if (replacements) *replacements = ctx->h_ctl()[CTL_REPLACED];
  return DBL_OK;
}

// ---- host-mediated exchange ---------------------------------------------------------------------------------
extern "C" int dbl_sweep_begin(dbl_ctx *ctx, int sampler, int64_t *ent_counts, int64_t *rec_counts) {
  if (!ctx || !ent_counts || !rec_counts) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_sweep_begin")) return rc1;
  if (sampler < 0 || sampler > 3) { ctx->set_error("bad sampler"); return DBL_ERR_INVALID; }
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  if (ctx->in_sweep || ctx->async_open) { ctx->set_error("dbl_sweep_begin twice"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
  int rc = enqueue_theta(ctx);
  if (rc) return rc;
  rc = update_owned(ctx, sampler);
  if (rc) return rc;
  const int W = ctx->world;
  std::vector<int> owner(ctx->P);  // the device's table: dbl_set_block_owners(ctx, NULL) does not update owner_h
  CUDA_TRY(cudaMemcpyAsync(owner.data(), ctx->owner.p, sizeof(int) * ctx->P, cudaMemcpyDeviceToHost, ctx->stream));
  rc = snapshot(ctx);  // also the partial summary of the shard (dbl_partial_summary) and the sweep's status
  // messages to rank d = the owned entities / records whose new block d owns: the block histograms of the summary.
  // An abandoned sweep sends nothing, but the caller still runs the collective calls of the sweep.
  ctx->h_move_ent.assign(W, 0);
  ctx->h_move_rec.assign(W, 0);
  if (!rc) {
    for (int b = 0; b < ctx->P; ++b) {
      const int d = owner[b];
      if (d == ctx->rank) continue;
      ctx->h_move_ent[d] += ctx->h_part()[ctx->blk_ent_slot() + b];
      ctx->h_move_rec[d] += ctx->h_part()[ctx->blk_rec_slot() + b];
    }
  }
  for (int d = 0; d < W; ++d) { ent_counts[d] = ctx->h_move_ent[d]; rec_counts[d] = ctx->h_move_rec[d]; }
  ctx->in_sweep = true;
  return rc;
}

extern "C" int dbl_exchange_pack(dbl_ctx *ctx, void *ent_buf_dev, void *rec_buf_dev) {
  if (!ctx) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_exchange_pack")) return rc1;
  if (!ctx->in_sweep) { ctx->set_error("dbl_exchange_pack outside a sweep"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  const int W = ctx->world;
  int64_t oe = 0, orc = 0;
  for (int d = 0; d < W; ++d) { oe += ctx->h_move_ent[d]; orc += ctx->h_move_rec[d]; }
  if ((oe > 0 && !ent_buf_dev) || (orc > 0 && !rec_buf_dev)) return DBL_ERR_INVALID;
  if (oe + orc == 0) return DBL_OK;  // also every abandoned sweep: nothing may leave this rank
  // rank d's messages follow those of the ranks before it; the cursors are this context's
  MsgOut out{};
  oe = orc = 0;
  for (int d = 0; d < W; ++d) {
    for (int par = 0; par < 2; ++par) {
      out.ent[d][par] = static_cast<int *>(ent_buf_dev) + oe * (ctx->A + 1);
      out.rec[d][par] = static_cast<int *>(rec_buf_dev) + orc * 3;
      out.cursor[d][par] = ctx->move_cnt.p + 2 * d;
    }
    oe += ctx->h_move_ent[d];
    orc += ctx->h_move_rec[d];
  }
  CUDA_TRY(cudaMemsetAsync(ctx->move_cnt.p, 0, sizeof(unsigned long long) * 2 * W, ctx->stream));
  launch_move(ctx, out);
  CUDA_TRY(cudaGetLastError());
  std::vector<unsigned long long> cur(2 * W);
  CUDA_TRY(cudaMemcpyAsync(cur.data(), ctx->move_cnt.p, sizeof(unsigned long long) * 2 * W, cudaMemcpyDeviceToHost,
                           ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // the host moves the buffers with NCCL on its own stream
  // the buffers were sized by the counts of dbl_sweep_begin: the messages written must be exactly those
  for (int d = 0; d < W; ++d)
    if ((int64_t)cur[2 * d] != ctx->h_move_ent[d] || (int64_t)cur[2 * d + 1] != ctx->h_move_rec[d]) {
      ctx->has_state = false;
      ctx->set_error("dbl_exchange_pack: " + std::to_string(cur[2 * d]) + " entity / " + std::to_string(cur[2 * d + 1]) +
                     " record messages for rank " + std::to_string(d) + ", but dbl_sweep_begin counted " +
                     std::to_string(ctx->h_move_ent[d]) + " / " + std::to_string(ctx->h_move_rec[d]));
      return DBL_ERR_STATE;
    }
  return DBL_OK;
}

extern "C" int dbl_exchange_unpack(dbl_ctx *ctx, const void *ent_buf_dev, int64_t n_ent, const void *rec_buf_dev,
                                   int64_t n_rec) {
  if (!ctx || n_ent < 0 || n_rec < 0) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_exchange_unpack")) return rc1;
  if (!ctx->in_sweep) { ctx->set_error("dbl_exchange_unpack outside a sweep"); return DBL_ERR_STATE; }
  if ((n_ent > 0 && !ent_buf_dev) || (n_rec > 0 && !rec_buf_dev)) return DBL_ERR_INVALID;
  if (n_ent + n_rec == 0) return DBL_OK;
  CUDA_TRY(cudaSetDevice(ctx->device));
  unsigned long long *count = ctx->move_cnt.p + 2 * ctx->world;
  const unsigned long long n[2] = {(unsigned long long)n_ent, (unsigned long long)n_rec};  // staging: alive until the sync
  CUDA_TRY(cudaMemcpyAsync(count, n, sizeof(n), cudaMemcpyHostToDevice, ctx->stream));
  const MsgIn in{{static_cast<const int *>(ent_buf_dev), static_cast<const int *>(ent_buf_dev)},
                 {static_cast<const int *>(rec_buf_dev), static_cast<const int *>(rec_buf_dev)},
                 {count, count}};
  launch_unpack(ctx, in, n_ent, n_rec);
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

// global_counts = the all-reduced words of dbl_partial_summary (drives the next theta draw); failed != 0: some rank
// reported an error for this sweep, so it is abandoned on every rank
extern "C" int dbl_sweep_end(dbl_ctx *ctx, const int64_t *global_counts, double global_loglik, int32_t failed) {
  if (!ctx || !global_counts) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_sweep_end")) return rc1;
  if (!ctx->in_sweep) { ctx->set_error("dbl_sweep_end without dbl_sweep_begin"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  ctx->in_sweep = false;
  if (failed) {
    ctx->has_state = false;
    ctx->set_error("the sweep failed on a peer rank");
    return DBL_ERR_CUDA;
  }
  std::vector<long long> g(ctx->n_counts());
  for (int i = 0; i < ctx->n_counts(); ++i) g[i] = global_counts[i];
  memcpy(&g[ctx->ll_slot()], &global_loglik, sizeof(double));
  CUDA_TRY(cudaMemcpyAsync(ctx->glob(), g.data(), sizeof(long long) * ctx->n_counts(), cudaMemcpyHostToDevice, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  int rc = relayout(ctx);
  if (rc) return rc;
  k_finish<<<1, 32, 0, ctx->stream>>>(ctx->ctl());
  ctx->launches += 1;
  CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
  rc = snapshot(ctx);
  float ms = 0.f;
  if (cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_sweep_ms = ms;
  return rc;
}

// partial summary of the shard after dbl_sweep_begin / dbl_set_block_owners (host copy, no device work)
extern "C" int dbl_partial_summary(dbl_ctx *ctx, int64_t *counts, double *loglik) {
  if (!ctx || !counts || !loglik) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_partial_summary")) return rc1;
  for (int i = 0; i < ctx->n_counts(); ++i) counts[i] = ctx->h_part()[i];
  counts[ctx->ll_slot()] = 0;
  memcpy(loglik, &ctx->h_part()[ctx->ll_slot()], sizeof(double));
  return DBL_OK;
}
extern "C" int32_t dbl_summary_words(const dbl_ctx *ctx) { return ctx ? ctx->n_counts() : 0; }

extern "C" int dbl_export_owned_dev(dbl_ctx *ctx, void *y_dev, void *blk_dev, void *link_dev, void *z_dev) {
  if (!ctx || !y_dev || !blk_dev || !link_dev || !z_dev) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_export_owned_dev")) return rc1;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  k_export_ent<<<grid_for(ctx->E, 256), 256, 0, ctx->stream>>>(ctx->E, ctx->A, ctx->ent_owned.p, ctx->y.p, ctx->blk.p,
                                                              (int *)y_dev, (int *)blk_dev);
  k_export_rec<<<grid_for(ctx->R, 256), 256, 0, ctx->stream>>>(ctx->R, ctx->A, ctx->rec_owned.p, ctx->link.p,
                                                              ctx->zmask.p, (int *)link_dev, (unsigned char *)z_dev);
  ctx->launches += 2;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

// the rows this rank owns, compacted (block-major order): ids + rows.  Host buffers sized for E / R rows.
extern "C" int dbl_download_owned(dbl_ctx *ctx, int64_t *n_ent, int32_t *ent_ids, int32_t *y, int32_t *block,
                                  int64_t *n_rec, int32_t *rec_ids, int32_t *link, uint8_t *z) {
  if (!ctx || !n_ent || !n_rec) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_download_owned")) return rc1;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  if (ctx->world > 1 && ctx->all_owned) { ctx->set_error("dbl_download_owned before dbl_set_block_owners"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (ctx->h_owned_ent < 0 || ctx->h_owned_rec < 0) { int rc = snapshot(ctx); if (rc) return rc; }
  const int64_t ne = ctx->h_owned_ent, nr = ctx->h_owned_rec;
  const int A = ctx->A;
  *n_ent = ne; *n_rec = nr;
  if (!(ent_ids && y && block) && !(rec_ids && link && z)) return DBL_OK;  // counts only
  const size_t need_i = (size_t)(ne * (A + 2) + nr * 2) + 1;
  if (ctx->gather_i.n < need_i) CUDA_TRY(ctx->gather_i.alloc(need_i));
  if (ctx->gather_b.n < (size_t)nr * A + 1) CUDA_TRY(ctx->gather_b.alloc((size_t)nr * A + 1));
  int *eids = ctx->gather_i.p, *yo = eids + ne, *bo = yo + ne * A, *rids = bo + ne, *lo = rids + nr;
  if (ne > 0 && ent_ids && y && block) {
    k_gather_ent<<<grid_for(ne, 256), 256, 0, ctx->stream>>>(ne, A, ctx->ent_sorted.p, ctx->y.p, ctx->blk.p, eids, yo, bo);
    CUDA_TRY(cudaMemcpyAsync(ent_ids, eids, sizeof(int) * ne, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(y, yo, sizeof(int) * ne * A, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(block, bo, sizeof(int) * ne, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (nr > 0 && rec_ids && link && z) {
    k_gather_rec<<<grid_for(nr, 256), 256, 0, ctx->stream>>>(nr, A, ctx->rec_sorted.p, ctx->link.p, ctx->zmask.p, rids, lo,
                                                            ctx->gather_b.p);
    CUDA_TRY(cudaMemcpyAsync(rec_ids, rids, sizeof(int) * nr, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(link, lo, sizeof(int) * nr, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(z, ctx->gather_b.p, (size_t)nr * A, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ctx->launches += 2;
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

extern "C" int dbl_owned_masks(dbl_ctx *ctx, uint8_t *ent_owned, uint8_t *rec_owned) {
  if (!ctx) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_owned_masks")) return rc1;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  if (ent_owned) CUDA_TRY(cudaMemcpyAsync(ent_owned, ctx->ent_owned.p, ctx->E, cudaMemcpyDeviceToHost, ctx->stream));
  if (rec_owned) CUDA_TRY(cudaMemcpyAsync(rec_owned, ctx->rec_owned.p, ctx->R, cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

// fingerprint of the rows this rank owns: hash[0] entities (id, values), hash[1] records (id, link, distortion bits);
// the sums over ranks mod 2^64 identify the global state whatever the number of ranks or the placement
extern "C" int dbl_state_hash(dbl_ctx *ctx, uint64_t *hash_out) {
  if (!ctx || !hash_out) return DBL_ERR_INVALID;
  if (int rc1 = one_chain_only(ctx, "dbl_state_hash")) return rc1;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaMemsetAsync(ctx->hash_words(), 0, 2 * sizeof(unsigned long long), ctx->stream));
  k_state_hash<<<grid_rows(ctx, std::max(ctx->E, ctx->R), 256), 256, 0, ctx->stream>>>(
      rows_masked(ctx, true), rows_masked(ctx, false), ctx->A, ctx->y.p, ctx->link.p, ctx->zmask.p, ctx->hash_words());
  ctx->launches += 1;
  unsigned long long h[2] = {0, 0};
  CUDA_TRY(cudaMemcpyAsync(h, ctx->hash_words(), sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  hash_out[0] = h[0]; hash_out[1] = h[1];
  return DBL_OK;
}

// which link kernel a sweep with this sampler launches: 0 k_link_generic, 1 k_link_match, 2 k_link_pruned,
// 3 k_link_pcg2 plus the bits of the model's tile format (Pcg2Format::bits, decided by pcg2_format at model upload)
// and +256 when the 1/n(y) columns travel with the tiles (some record misses a non-constant value)
extern "C" int dbl_link_kernel(const dbl_ctx *ctx, int sampler) {
  if (!ctx || sampler < 0 || sampler > 3) return DBL_ERR_INVALID;
  const LinkKernel kernel = link_kernel(ctx, sampler);
  if (kernel != LINK_PCG2) return kernel;
  return LINK_PCG2 + ctx->pcg2_fmt.bits(ctx->n_str) + (ctx->tile_invn.p ? 256 : 0);
}

extern "C" int dbl_set_link_mode(dbl_ctx *ctx, int mode) {
  if (!ctx || mode < 0 || mode > 2) return DBL_ERR_INVALID;
  ctx->drop_graphs();
  ctx->link_mode = mode;
  return DBL_OK;
}

extern "C" int dbl_set_link_mass_capture(dbl_ctx *ctx, int on) {
  if (!ctx) return DBL_ERR_INVALID;
  ctx->drop_graphs();  // captured sweeps hold the link parameters by value
  ctx->link_mass_on = on != 0;
  if (!ctx->link_mass_on) ctx->link_mass.release();
  return DBL_OK;
}

extern "C" int dbl_link_mass(dbl_ctx *ctx, double *mass_out) {
  if (!ctx || !mass_out) return DBL_ERR_INVALID;
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  if (!ctx->link_mass_on || ctx->link_mass.n != (size_t)ctx->R) {
    ctx->set_error("dbl_link_mass: no sweep has run with the capture on (dbl_set_link_mass_capture)");
    return DBL_ERR_STATE;
  }
  CUDA_TRY(cudaSetDevice(ctx->device));
  CUDA_TRY(cudaMemcpyAsync(mass_out, ctx->link_mass.p, sizeof(double) * (size_t)ctx->R, cudaMemcpyDeviceToHost,
                           ctx->stream));
  CUDA_TRY(cudaStreamSynchronize(ctx->stream));
  return DBL_OK;
}

extern "C" double dbl_last_sweep_ms(const dbl_ctx *ctx) { return ctx ? ctx->last_sweep_ms : 0.0; }

extern "C" double dbl_link_kernel_ms(dbl_ctx *ctx, int64_t *launches) {
  if (!ctx) return 0.0;
  const double ms = ctx->link_ms;
  if (launches) *launches = ctx->link_launches;
  ctx->link_ms = 0.0;
  ctx->link_launches = 0;
  return ms;
}

extern "C" int64_t dbl_phase_ms(dbl_ctx *ctx, double *out4) {
  if (!ctx || !out4) return 0;
  const int64_t n = ctx->phase_sweeps;
  for (int i = 0; i < 4; ++i) { out4[i] = ctx->phase_ms[i]; ctx->phase_ms[i] = 0.0; }
  ctx->phase_sweeps = 0;
  return n;
}

// summary of chain k: its files are the columns [k F1, (k+1) F1) of aggDist / theta
static int chain_summary(dbl_ctx *ctx, int k, dbl_summary_head *head, int64_t *agg_dist, int64_t *rec_dist,
                         double *theta) {
  if (!ctx->has_state) { ctx->set_error("no state"); return DBL_ERR_STATE; }
  const int A = ctx->A, F = ctx->F, F1 = ctx->F1, f0 = k * F1;
  const long long *g = ctx->h_glob();
  if (head) {
    head->iteration = ctx->iteration;
    head->num_isolates = g[ctx->iso_slot() + k];
    double ll;
    memcpy(&ll, &g[ctx->ll_slot() + k], sizeof(double));
    for (int a = 0; a < A; ++a)
      for (int f = f0; f < f0 + F1; ++f) {  // GU:286-293
        const double th = ctx->h_theta[a * F + f];
        const double nd = (double)g[a * F + f];
        ll += (ctx->alpha[a] + nd - 1.0) * std::log(th) +
              (ctx->beta[a] + (double)ctx->file_sizes[f] - nd - 1.0) * std::log(1.0 - th);
      }
    head->log_likelihood = ll;
    head->pairs_scored = ctx->h_pairs;
  }
  for (int a = 0; a < A; ++a)
    for (int f = 0; f < F1; ++f) {
      if (agg_dist) agg_dist[a * F1 + f] = g[a * F + f0 + f];
      if (theta) theta[a * F1 + f] = ctx->h_theta[a * F + f0 + f];
    }
  if (rec_dist) for (int i = 0; i <= A; ++i) rec_dist[i] = g[A * F + k * (A + 1) + i];
  return DBL_OK;
}

extern "C" int dbl_summary(dbl_ctx *ctx, dbl_summary_head *head, int64_t *agg_dist, int64_t *rec_dist, double *theta) {
  if (!ctx) return DBL_ERR_INVALID;
  int rc = one_chain_only(ctx, "dbl_summary");
  if (rc) return rc;
  return chain_summary(ctx, 0, head, agg_dist, rec_dist, theta);
}

extern "C" int dbl_chain_summary(dbl_ctx *ctx, int32_t chain, dbl_summary_head *head, int64_t *agg_dist,
                                 int64_t *rec_dist, double *theta) {
  if (!ctx) return DBL_ERR_INVALID;
  if (chain < 0 || chain >= ctx->K) { ctx->set_error("chain out of range"); return DBL_ERR_INVALID; }
  return chain_summary(ctx, chain, head, agg_dist, rec_dist, theta);
}
