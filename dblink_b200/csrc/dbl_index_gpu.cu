// AttributeIndex construction on the GPU (the step before the sweep; AttributeIndex.scala:107-245):
//   * all-pairs thresholded Levenshtein or Jaro-Winkler (computeSimValueIndex, :219-231: V^2 pairs, keep
//     exp(sim) > 1);
//   * the similarity normalisations n_a(v) (computeSimNormalizations, :234-245) and the base pmfs / cdfs
//     B_k, k = 0..kmax (getSimNormDist, :197-216).
//
// Everything stays bit-identical to the host loops: the device computes only INTEGERS -- the edit distance, or the
// Jaro-Winkler counts (m, h, l) -- of the pairs that can possibly have a positive truncated similarity (the host
// turns (integers, lengths) into sim and exp(sim) with the same double arithmetic as the host-only path), and the
// normalisation / pmf kernels run the host's sequential sums unchanged, one independent sum per thread (this TU is
// compiled with -fmad=false like the rest).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "dbl_internal.h"
#include "dbl_scale.h"

namespace {
constexpr int MAXL = 64;        // longest string the bit-parallel kernel takes (one 64-bit word per column)
constexpr int LEV_WARPS = 8;    // warps per CTA; every warp scores its own texts against the CTA's 32 patterns
constexpr int LEV_TEXTS = 256;  // texts per CTA (32 per warp)

// Myers / Hyyro bit-parallel edit distance, one PATTERN per lane, one TEXT per warp iteration:
//   the CTA owns patterns i0 .. i0+31 (lane = pattern) and texts j0 .. j0+LEV_TEXTS-1;
//   Peq[c][lane] (shared memory, 256 x 32 x 8 bytes) = positions of byte c in the lane's pattern: a warp reads
//   Peq[c][0..31] for ONE byte c of the current text -- 32 consecutive 8-byte words, no bank conflict;
//   a column of the DP matrix is two 64-bit words (Pv, Mv) per lane: ~16 integer operations per text byte instead
//   of 5 per DP cell.
// Only pairs j > i are produced (the matrix is symmetric), and only those whose distance can give a positive
// truncated similarity: sim > 0  <=>  d < (|a| + |b|) (1 - t) / (1 + t), t = threshold / maxSimilarity.
// Peq[c][lane] = bit set of the positions of byte c in pattern i0 + lane (all zero for lanes past V)
__device__ __forceinline__ void load_patterns(unsigned long long *peq, int V, const unsigned char *__restrict__ strs,
                                              int i, int m) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = threadIdx.x; k < 256 * 32; k += blockDim.x) peq[k] = 0ull;
  __syncthreads();
  if (warp == 0 && i < V)
    for (int q = 0; q < m; ++q) peq[(int)strs[(size_t)i * MAXL + q] * 32 + lane] |= 1ull << q;
  __syncthreads();
}

__global__ void __launch_bounds__(LEV_WARPS * 32) k_lev_tiles(int V, const unsigned char *__restrict__ strs,
                                                              const int *__restrict__ lens, double ratio,
                                                              unsigned long long cap,
                                                              unsigned long long *__restrict__ count,
                                                              int4 *__restrict__ out) {
  extern __shared__ unsigned long long peq[];  // [256][32]
  const int i0 = blockIdx.y * 32;
  const int j0 = blockIdx.x * LEV_TEXTS;
  if (j0 + LEV_TEXTS <= i0) return;  // whole text tile at or below the diagonal
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = i0 + lane;
  const int m = (i < V) ? lens[i] : 0;
  load_patterns(peq, V, strs, i, m);
  const unsigned long long top = m > 0 ? 1ull << (m - 1) : 0ull;
  for (int jj = warp; jj < LEV_TEXTS; jj += LEV_WARPS) {
    const int j = j0 + jj;
    if (j >= V) break;
    const int n = lens[j];
    // texts are short: every lane reads the same bytes (broadcast from L1)
    unsigned long long Pv = ~0ull, Mv = 0ull;
    int score = m;
    for (int q = 0; q < n; ++q) {
      const unsigned long long Eq = peq[(int)strs[(size_t)j * MAXL + q] * 32 + lane];
      const unsigned long long Xv = Eq | Mv;
      const unsigned long long Xh = (((Eq & Pv) + Pv) ^ Pv) | Eq;
      unsigned long long Ph = Mv | ~(Xh | Pv);
      unsigned long long Mh = Pv & Xh;
      if (Ph & top) ++score;
      else if (Mh & top) --score;
      Ph = (Ph << 1) | 1ull;
      Mh = Mh << 1;
      Pv = Mh | ~(Xv | Ph);
      Mv = Ph & Xv;
    }
    const int d = (m == 0) ? n : score;
    if (i < V && j > i) {
      const int maxd = (int)((double)(m + n) * ratio) + 1;  // +1 keeps the filter conservative
      if (d <= maxd) {
        const unsigned long long slot = atomicAdd(count, 1ull);
        if (slot < cap) out[slot] = make_int4(i, j, d, 0);
      }
    }
  }
}

// Slack of the device's Jaro-Winkler filters against t = threshold / maxSimilarity: the host keeps a pair only when
// maxSimilarity * unit > threshold, and the device's double estimates are within a few ulps of the host's, so a pair
// the filters drop has unit < t - 1e-9 and a truncated similarity of exactly 0.
constexpr double JW_SLACK = 1e-9;

// Jaro-Winkler counts in the k_lev_tiles layout (lane = pattern a = string i, one text b = string j per warp
// iteration, Peq in shared memory).  The greedy scan runs over the TEXT: each byte b[q] takes the lowest unmatched
// pattern position in the window [q - w, q + w] holding the same byte (Peq & window & ~flagP); flagT records the
// matched text positions.  This is the host's scan with a and b swapped; the counts (m, h) are symmetric in (a, b),
// so they are the host's counts of (i, j) and (j, i) alike.  h pairs the k-th set bits of flagP and flagT: pattern
// position ip holds b[jp] iff bit ip of Peq[b[jp]] is set.  l = the first q < 4 where bit q of Peq[b[q]] is clear.
// The pair is skipped before the scan when even m = min(la, lb), h = 0, l = 4 cannot pass t (jaro <= (2 + min/max)/3),
// and after it when its own estimate cannot; the host recomputes the exact double from (m, h, l).
__global__ void __launch_bounds__(LEV_WARPS * 32) k_jw_tiles(int V, const unsigned char *__restrict__ strs,
                                                             const int *__restrict__ lens, double t,
                                                             unsigned long long cap,
                                                             unsigned long long *__restrict__ count,
                                                             int4 *__restrict__ out) {
  extern __shared__ unsigned long long peq[];  // [256][32]
  const int i0 = blockIdx.y * 32;
  const int j0 = blockIdx.x * LEV_TEXTS;
  if (j0 + LEV_TEXTS <= i0) return;  // whole text tile at or below the diagonal
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = i0 + lane;
  const int la = (i < V) ? lens[i] : 0;
  load_patterns(peq, V, strs, i, la);
  const double cut = t - JW_SLACK;
  for (int jj = warp; jj < LEV_TEXTS; jj += LEV_WARPS) {
    const int j = j0 + jj;
    if (j >= V) break;
    if (i >= V || j <= i) continue;
    const int lb = lens[j];
    const unsigned char *T = strs + (size_t)j * MAXL;  // every lane reads the same bytes (broadcast from L1)
    const int lo = min(la, lb), hi = max(la, lb);
    if (hi > 0) {
      const double jb = (2.0 + (double)lo / hi) / 3.0;
      if (jb + 0.4 * (1.0 - jb) < cut) continue;
    }
    const int w = max(0, hi / 2 - 1);
    unsigned long long fp = 0ull, ft = 0ull;
    int l = 0;
    bool prefix = true;
    for (int q = 0; q < lb; ++q) {
      const unsigned long long Eq = peq[(int)T[q] * 32 + lane];
      if (q < 4 && prefix) {
        if ((Eq >> q) & 1ull) ++l;
        else prefix = false;
      }
      const unsigned long long win = (~0ull << max(0, q - w)) & ((2ull << min(q + w, 63)) - 1ull);
      const unsigned long long cand = Eq & win & ~fp;
      if (cand) {
        fp |= cand & (0ull - cand);
        ft |= 1ull << q;
      }
    }
    const int m = __popcll(fp);
    if (m == 0 && hi > 0) continue;  // unit 0; two empty strings (unit 1) leave with code 0
    int h = 0;
    for (unsigned long long p = fp, s = ft; p; p &= p - 1, s &= s - 1) {
      const int ip = __ffsll((long long)p) - 1, jp = __ffsll((long long)s) - 1;
      h += (int)(~(peq[(int)T[jp] * 32 + lane] >> ip) & 1ull);
    }
    if (m > 0) {
      const double jaro = ((double)m / la + (double)m / lb + ((double)m - 0.5 * h) / m) / 3.0;
      if (jaro + 0.1 * l * (1.0 - jaro) < cut) continue;
    }
    const unsigned long long slot = atomicAdd(count, 1ull);
    if (slot < cap) out[slot] = make_int4(i, j, m | h << 8 | l << 16, 0);
  }
}

// computeSimNormalizations (AttributeIndex.scala:234-245): n(v) = 1 / sum_w probs(w) * E(v, w), the sum taken over
// ALL values in ascending id with E = 1 outside the sparse row -- the host loop, one value per thread
__global__ void k_sim_norms(int V, const double *__restrict__ probs, const int *__restrict__ rowptr,
                            const int *__restrict__ col, const double *__restrict__ expsim, double *__restrict__ norm,
                            double *__restrict__ invnorm) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  double acc = 0.0;
  int p = rowptr[v];
  const int pe = rowptr[v + 1];
  int next = p < pe ? col[p] : V;
  for (int w = 0; w < V; ++w) {
    double e = 1.0;
    if (w == next) {
      e = expsim[p++];
      next = p < pe ? col[p] : V;
    }
    acc += probs[w] * e;
  }
  invnorm[v] = acc;
  norm[v] = 1.0 / acc;
}

// getSimNormDist (AttributeIndex.scala:197-216): B_k(v) = probs(v) n(v)^k / Z_k for k = 0..kmax, and the running sums
// the inverse-cdf draws use; sequential sums as on the host (base_row), one k per thread
__global__ void k_base_pmfs(int V, int kmax, int is_const, const double *__restrict__ probs,
                            const double *__restrict__ norm, double *__restrict__ pk, double *__restrict__ cdf) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > kmax) return;
  base_row(V, probs, norm, is_const != 0, k, pk + (size_t)k * V, cdf + (size_t)k * V);
}

struct Dev {
  void *p = nullptr;
  bool alloc(size_t bytes) { return cudaMalloc(&p, std::max<size_t>(bytes, 16)) == cudaSuccess; }
  ~Dev() { if (p) cudaFree(p); }
};
}  // namespace

// Fills (oi, oj, oc) with (i, j>i, code) for every pair that may have a positive similarity: code = the edit distance
// (similarity 1, k_lev_tiles) or m | h << 8 | l << 16 (similarity 2, k_jw_tiles).  Returns false when the GPU path is
// not applicable (no device, strings too long) -- the caller then uses the host loop.
bool gpu_similarity_candidates(int similarity, const std::vector<std::string> &values, double threshold,
                               double max_sim, std::vector<int> &oi, std::vector<int> &oj, std::vector<int> &oc) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return false; }
  const int V = (int)values.size();
  for (auto &s : values)
    if ((int)s.size() > MAXL) return false;
  std::vector<unsigned char> h_strs((size_t)V * MAXL, 0);
  std::vector<int> h_lens(V);
  for (int v = 0; v < V; ++v) {
    h_lens[v] = (int)values[v].size();
    std::memcpy(&h_strs[(size_t)v * MAXL], values[v].data(), values[v].size());
  }
  const double t = threshold / max_sim;
  // both kernels take one double: Levenshtein the distance ratio of its length bound, Jaro-Winkler t itself
  const bool jw = similarity == DBL_SIM_JARO_WINKLER;
  const auto kernel = jw ? k_jw_tiles : k_lev_tiles;
  const double param = jw ? t : (1.0 - t) / (1.0 + t);
  Dev d_strs, d_lens, d_count;
  if (!d_strs.alloc(h_strs.size()) || !d_lens.alloc(sizeof(int) * V) || !d_count.alloc(sizeof(unsigned long long))) {
    cudaGetLastError();
    return false;
  }
  cudaMemcpy(d_strs.p, h_strs.data(), h_strs.size(), cudaMemcpyHostToDevice);
  cudaMemcpy(d_lens.p, h_lens.data(), sizeof(int) * V, cudaMemcpyHostToDevice);
  const size_t smem = 256 * 32 * sizeof(unsigned long long);
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  unsigned long long cap = std::max<unsigned long long>((unsigned long long)V * 64ull, 1ull << 20);
  for (int attempt = 0; attempt < 3; ++attempt) {
    Dev d_out;
    if (!d_out.alloc(sizeof(int4) * cap)) break;
    cudaMemset(d_count.p, 0, sizeof(unsigned long long));
    // 2-D grid of tiles: x = text tiles (no 65 535 limit on this axis), y = pattern tiles of 32 (V <= 2 097 120)
    const dim3 grid((unsigned)((V + LEV_TEXTS - 1) / LEV_TEXTS), (unsigned)((V + 31) / 32));
    if (grid.y > 65535u) break;
    kernel<<<grid, LEV_WARPS * 32, smem>>>(V, (const unsigned char *)d_strs.p, (const int *)d_lens.p, param, cap,
                                           (unsigned long long *)d_count.p, (int4 *)d_out.p);
    unsigned long long n = 0;
    if (cudaMemcpy(&n, d_count.p, sizeof(n), cudaMemcpyDeviceToHost) != cudaSuccess) break;
    if (n <= cap) {
      std::vector<int4> h((size_t)n);
      if (n) cudaMemcpy(h.data(), d_out.p, sizeof(int4) * n, cudaMemcpyDeviceToHost);
      // the order in which pairs were appended depends on scheduling; the caller sorts the rows
      oi.resize(n); oj.resize(n); oc.resize(n);
      for (size_t k = 0; k < n; ++k) { oi[k] = h[k].x; oj[k] = h[k].y; oc[k] = h[k].z; }
      return true;
    }
    cap = n + 1024;
  }
  cudaGetLastError();
  return false;
}

// norm / invnorm / pk / cdf of an index from its probs and sparse rows, on the device.  Same values as
// dbl_index::finish()'s host loops.  Returns false when no device is usable.
bool gpu_index_tables(int V, int kmax, bool is_const, const std::vector<double> &probs,
                      const std::vector<int32_t> &rowptr, const std::vector<int32_t> &col,
                      const std::vector<double> &expsim, std::vector<double> &norm, std::vector<double> &invnorm,
                      std::vector<double> &pk, std::vector<double> &cdf) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return false; }
  Dev d_probs, d_rowptr, d_col, d_exp, d_norm, d_inv, d_pk, d_cdf;
  const size_t nnz = col.size(), nk = (size_t)(kmax + 1) * V;
  if (!d_probs.alloc(sizeof(double) * V) || !d_rowptr.alloc(sizeof(int) * (V + 1)) || !d_col.alloc(sizeof(int) * nnz) ||
      !d_exp.alloc(sizeof(double) * nnz) || !d_norm.alloc(sizeof(double) * V) || !d_inv.alloc(sizeof(double) * V) ||
      !d_pk.alloc(sizeof(double) * nk) || !d_cdf.alloc(sizeof(double) * nk)) {
    cudaGetLastError();
    return false;
  }
  cudaMemcpy(d_probs.p, probs.data(), sizeof(double) * V, cudaMemcpyHostToDevice);
  cudaMemcpy(d_rowptr.p, rowptr.data(), sizeof(int) * (V + 1), cudaMemcpyHostToDevice);
  if (nnz) {
    cudaMemcpy(d_col.p, col.data(), sizeof(int) * nnz, cudaMemcpyHostToDevice);
    cudaMemcpy(d_exp.p, expsim.data(), sizeof(double) * nnz, cudaMemcpyHostToDevice);
  }
  norm.assign(V, 1.0);
  invnorm.assign(V, 1.0);
  if (!is_const) {
    k_sim_norms<<<(V + 127) / 128, 128>>>(V, (const double *)d_probs.p, (const int *)d_rowptr.p, (const int *)d_col.p,
                                          (const double *)d_exp.p, (double *)d_norm.p, (double *)d_inv.p);
    cudaMemcpy(norm.data(), d_norm.p, sizeof(double) * V, cudaMemcpyDeviceToHost);
    cudaMemcpy(invnorm.data(), d_inv.p, sizeof(double) * V, cudaMemcpyDeviceToHost);
  } else {
    cudaMemcpy(d_norm.p, norm.data(), sizeof(double) * V, cudaMemcpyHostToDevice);
  }
  k_base_pmfs<<<(kmax + 1 + 31) / 32, 32>>>(V, kmax, is_const ? 1 : 0, (const double *)d_probs.p, (const double *)d_norm.p,
                                            (double *)d_pk.p, (double *)d_cdf.p);
  pk.assign(nk, 0.0);
  cdf.assign(nk, 0.0);
  cudaMemcpy(pk.data(), d_pk.p, sizeof(double) * nk, cudaMemcpyDeviceToHost);
  cudaMemcpy(cdf.data(), d_cdf.p, sizeof(double) * nk, cudaMemcpyDeviceToHost);
  if (cudaGetLastError() != cudaSuccess) return false;
  return true;
}
