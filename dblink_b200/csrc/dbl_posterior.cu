// Shared most probable clusters (sMPC) of a linkage chain on the GPU (LinkageChain.scala:52-95): for every record the
// cluster it belongs to most often along the chain, then records grouped by that cluster.
//
// Same quantities, bit for bit, as dblink_b200/analysis_arrays.py (cluster_signatures, most_probable_signature,
// shared_most_probable_clusters):
//   * a cluster of a sample is identified by a 64-bit signature of its SET of records: the wrapping sum of mix64(r)
//     over its members, mixed with its size -- sig = mix64(sum ^ mix64(size)); sums are order independent, so the
//     per-cluster accumulation may use atomics;
//   * a record's most probable signature is the one it carries in most samples, ties going to the signature seen in
//     the earliest sample; its frequency is count / S;
//   * the sMPC label of a record is the smallest record index among the records with the same best signature.
// Signatures live in a record-major device matrix [R][max_samples]; the mode runs over blocks of records, each a
// stable segmented radix sort of (signature, sample index) pairs followed by one scan per record.
//
// Posterior pairwise match counts (dbl_pairs_*, same numbers as analysis_arrays.pairwise_match_counts): for every
// unordered pair of records the number of samples in which they share a cluster.  The handle holds a sorted table of
// (first << 32 | second, count) over the pairs seen so far; each sample's pairs are generated, sorted and merged into
// it -- see dbl_pairs_add_sample.  dbl_pairs_score_sample generates the pairs of any labelling the same way and sums
// their held counts (the Binder-loss estimate of analysis_arrays.binder_counts).
//
// Every sample against the ground truth (dbl_eval_*, same numbers as analysis_arrays.posterior_metric_counts): per
// sample the pair counts the pairwise metrics and the adjusted Rand index are made of -- tp = sum over the cells
// (sample cluster, true entity) of C(n, 2), pred_pairs = sum over sample clusters of C(size, 2) -- and the number of
// clusters, all in int64.  Each record becomes one key, sample label above true label; the keys are radix-sorted on
// their 2 ceil(log2 R) bits, so cells and clusters are runs of the sorted keys -- see dbl_eval_add_sample.
//
// Cell histograms of every pair of held samples (dbl_vi_*, same numbers as analysis_arrays.vi_cross_histograms): for
// every sample t and cell size n >= 2, the number of cells of n records in C_t ^ C_s summed over the other samples s,
// in int64 -- the integers the posterior expected variation of information is made of.  Cells are runs of radix-sorted
// (s, label in C_t, label in C_s) keys over the records in C_t's clusters of two or more -- see dbl_vi_cross.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cub/cub.cuh>

#include "dbl_internal.h"

namespace {
// (signature, sample) pairs sorted per record block: bounds the block's temporaries (~2 GB) whatever R and S are
constexpr int64_t PAIR_BLOCK = int64_t(1) << 26;
constexpr int THREADS = 256;

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {  // splitmix64 finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

int grid_for(int64_t n) { return (int)std::min<int64_t>((n + THREADS - 1) / THREADS, 4096); }

// any label outside [0, R) raises the flag; runs before anything indexes by label
__global__ void k_check_labels(int64_t R, const int32_t *__restrict__ cluster, int *__restrict__ bad) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    if (cluster[r] < 0 || (int64_t)cluster[r] >= R) *bad = 1;
}

__global__ void k_accumulate(int64_t R, const int32_t *__restrict__ cluster, unsigned long long *__restrict__ sum,
                             unsigned int *__restrict__ size) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = cluster[r];
    atomicAdd(&sum[c], mix64((unsigned long long)r));
    atomicAdd(&size[c], 1u);
  }
}

// column s of the record-major signature matrix
__global__ void k_signatures(int64_t R, int32_t stride, int32_t s, const int32_t *__restrict__ cluster,
                             const unsigned long long *__restrict__ sum, const unsigned int *__restrict__ size,
                             unsigned long long *__restrict__ sig) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = cluster[r];
    sig[r * stride + s] = mix64(sum[c] ^ mix64((unsigned long long)size[c]));
  }
}

// the S signatures of records lo .. lo+nb-1, packed [nb][S], each with its sample index
__global__ void k_gather(const unsigned long long *__restrict__ sig, int32_t stride, int64_t lo, int64_t nb, int32_t S,
                         unsigned long long *__restrict__ keys, int32_t *__restrict__ samples) {
  const int64_t n = nb * S;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = j / S;
    const int32_t s = (int32_t)(j - i * S);
    keys[j] = sig[(lo + i) * stride + s];
    samples[j] = s;
  }
}

__global__ void k_segment_offsets(int64_t nb, int32_t S, int32_t *__restrict__ off) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= nb; i += (int64_t)gridDim.x * blockDim.x)
    off[i] = (int32_t)(i * S);
}

// one record per thread over its S sorted pairs: runs of equal signatures; the longest run wins, ties going to the
// run whose first sample is earliest (the sort is stable, so a run's first element carries its earliest sample)
__global__ void k_mode(const unsigned long long *__restrict__ keys, const int32_t *__restrict__ samples, int64_t nb,
                       int32_t S, int64_t lo, unsigned long long *__restrict__ best, double *__restrict__ freq) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nb; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long *k = keys + i * S;
    const int32_t *v = samples + i * S;
    unsigned long long run_key = k[0], best_key = k[0];
    int32_t run_start = 0, best_count = 0, best_first = INT_MAX;
    for (int32_t j = 1; j <= S; ++j) {
      const unsigned long long kj = j < S ? k[j] : 0ull;
      if (j == S || kj != run_key) {
        const int32_t count = j - run_start, first = v[run_start];
        if (count > best_count || (count == best_count && first < best_first)) {
          best_count = count;
          best_first = first;
          best_key = run_key;
        }
        run_start = j;
        run_key = kj;
      }
    }
    best[lo + i] = best_key;
    if (freq) freq[lo + i] = (double)best_count / (double)S;
  }
}

__global__ void k_iota(int64_t n, int32_t *__restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (int32_t)i;
}

// position of every run head of sorted keys, 0 elsewhere (a max-scan then gives each position its run's start)
template <class T>
__global__ void k_run_heads(int64_t n, const T *__restrict__ keys, int32_t *__restrict__ head) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? (int32_t)i : 0;
}

// records are sorted stably by best signature, so the record at a run's head is the smallest index of its group
__global__ void k_scatter_labels(int64_t n, const int32_t *__restrict__ record, const int32_t *__restrict__ head,
                                 int32_t *__restrict__ labels) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    labels[record[i]] = record[head[i]];
}

struct MaxOp {
  __device__ __forceinline__ int32_t operator()(int32_t a, int32_t b) const { return a > b ? a : b; }
};

// A device buffer.  alloc() takes exactly what it is asked for; reserve() only grows: to at least twice its size, at
// most `limit` bytes unless more is needed, and a new allocation replaces the old one only once it has succeeded.
struct Buf {
  void *p = nullptr;
  size_t cap = 0;
  ~Buf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) {
    const cudaError_t e = cudaMalloc(&p, std::max<size_t>(bytes, 16));
    if (e == cudaSuccess) cap = bytes;
    return e;
  }
  cudaError_t reserve(size_t need, size_t limit = SIZE_MAX) {
    if (need <= cap) return cudaSuccess;
    Buf nb;
    const cudaError_t e = nb.alloc(std::max(need, std::min(limit, cap > SIZE_MAX / 2 ? SIZE_MAX : 2 * cap)));
    if (e != cudaSuccess) return e;
    std::swap(p, nb.p);  // nb now frees the old buffer
    std::swap(cap, nb.cap);
    return cudaSuccess;
  }
  template <class T> T *as() const { return (T *)p; }
};

// the object's device is current for the duration of a call; the caller's is restored afterwards
struct DeviceScope {
  int prev = -1, dev;
  explicit DeviceScope(int d) : dev(d) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceScope() { if (prev >= 0 && prev != dev) cudaSetDevice(prev); }
};

#define POST_TRY(expr)                   \
  do {                                   \
    if ((expr) != cudaSuccess) {         \
      cudaGetLastError();                \
      return DBL_ERR_CUDA;               \
    }                                    \
  } while (0)

// What every handle holds: its device, R, the number of samples added, its stream, the labels of the sample being
// added and the label check flag.
struct Handle {
  int device = 0;
  int64_t R = 0;
  int32_t S = 0;
  cudaStream_t stream = nullptr;
  Buf cluster, bad;

  // R labels, host or device (unified addressing picks the copy direction), into dst, then the range check:
  // DBL_ERR_INVALID when one is outside [0, R)
  int take_labels(const int32_t *labels, Buf &dst) {
    POST_TRY(cudaMemcpyAsync(dst.p, labels, sizeof(int32_t) * R, cudaMemcpyDefault, stream));
    POST_TRY(cudaMemsetAsync(bad.p, 0, sizeof(int), stream));
    k_check_labels<<<grid_for(R), THREADS, 0, stream>>>(R, dst.as<int32_t>(), bad.as<int>());
    int flag = 0;
    POST_TRY(cudaMemcpyAsync(&flag, bad.p, sizeof(int), cudaMemcpyDeviceToHost, stream));
    POST_TRY(cudaStreamSynchronize(stream));
    return flag ? DBL_ERR_INVALID : DBL_OK;
  }
};

template <class H>
void free_handle(H *p) {
  if (!p) return;
  DeviceScope ds(p->device);
  if (p->stream) {
    cudaStreamSynchronize(p->stream);
    cudaStreamDestroy(p->stream);
  }
  delete p;  // Buf destructors free the device memory
}

// A create, once its own arguments are checked: a device must exist; the handle lives on the current one, with its
// stream, sample labels and check flag, then init(p) allocates the rest.  On failure the half-built handle is freed.
template <class H, class Init>
int open_handle(H **out, int64_t num_records, Init init) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return DBL_ERR_CUDA;
  }
  auto *p = new H();
  p->R = num_records;
  int rc = DBL_ERR_CUDA;
  if (cudaGetDevice(&p->device) == cudaSuccess &&
      cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) == cudaSuccess &&
      p->cluster.alloc(sizeof(int32_t) * (size_t)num_records) == cudaSuccess && p->bad.alloc(sizeof(int)) == cudaSuccess)
    rc = init(p);
  if (rc != DBL_OK) {
    cudaGetLastError();
    free_handle(p);
    return rc;
  }
  *out = p;
  return DBL_OK;
}

// Records grouped by key: a stable radix sort of (key, record) over bits [0, end_bit), then every sorted position's
// run start, an inclusive max-scan of the run heads.  The sort is stable, so a run keeps its records in their order in
// rec.  key_s, rec_s and start receive the n sorted keys, sorted records and run starts; head is n entries of scratch;
// tmp grows to the temporary storage of the sort and the scan.
template <class T>
int group_by_key(int64_t n, int end_bit, const T *key, const int32_t *rec, T *key_s, int32_t *rec_s, int32_t *head,
                 int32_t *start, Buf &tmp, cudaStream_t st) {
  size_t tb_sort = 0, tb_scan = 0;
  POST_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, key, key_s, rec, rec_s, n, 0, end_bit, st));
  POST_TRY(cub::DeviceScan::InclusiveScan(nullptr, tb_scan, head, start, MaxOp(), n, st));
  POST_TRY(tmp.reserve(std::max(tb_sort, tb_scan)));
  size_t tb = tmp.cap;
  POST_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tb, key, key_s, rec, rec_s, n, 0, end_bit, st));
  k_run_heads<<<grid_for(n), THREADS, 0, st>>>(n, key_s, head);
  tb = tmp.cap;
  POST_TRY(cub::DeviceScan::InclusiveScan(tmp.p, tb, head, start, MaxOp(), n, st));
  return DBL_OK;
}
}  // namespace

struct dbl_posterior : Handle {
  int32_t max_samples = 0;
  Buf sig;   // [R][max_samples] signatures
  Buf sum;   // R wrapping sums of mix64(record) per cluster
  Buf size;  // R cluster sizes
};

extern "C" int dbl_posterior_create(dbl_posterior **out, int64_t num_records, int32_t max_samples) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  // a record's S samples are sorted in one block, so max_samples <= PAIR_BLOCK
  if (num_records <= 0 || num_records > INT32_MAX || max_samples <= 0 || max_samples > PAIR_BLOCK)
    return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_posterior *p) {
    p->max_samples = max_samples;
    if (p->sig.alloc(sizeof(unsigned long long) * (size_t)num_records * (size_t)max_samples) != cudaSuccess ||
        p->sum.alloc(sizeof(unsigned long long) * (size_t)num_records) != cudaSuccess ||
        p->size.alloc(sizeof(unsigned int) * (size_t)num_records) != cudaSuccess)
      return DBL_ERR_CUDA;  // the signature matrix does not fit
    return DBL_OK;
  });
}

extern "C" void dbl_posterior_free(dbl_posterior *p) { free_handle(p); }

extern "C" int32_t dbl_posterior_num_samples(const dbl_posterior *p) { return p ? p->S : 0; }

extern "C" int dbl_posterior_add_sample(dbl_posterior *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  const int32_t *c = p->cluster.as<int32_t>();
  POST_TRY(cudaMemsetAsync(p->sum.p, 0, sizeof(unsigned long long) * R, st));
  POST_TRY(cudaMemsetAsync(p->size.p, 0, sizeof(unsigned int) * R, st));
  k_accumulate<<<grid_for(R), THREADS, 0, st>>>(R, c, p->sum.as<unsigned long long>(), p->size.as<unsigned int>());
  k_signatures<<<grid_for(R), THREADS, 0, st>>>(R, p->max_samples, p->S, c, p->sum.as<unsigned long long>(),
                                                p->size.as<unsigned int>(), p->sig.as<unsigned long long>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  ++p->S;
  return DBL_OK;
}

extern "C" int dbl_posterior_smpc(dbl_posterior *p, int32_t *labels_out, double *freq_out) {
  if (!p) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  const int64_t R = p->R;
  const int32_t S = p->S;
  cudaStream_t st = p->stream;
  Buf best, freq;
  POST_TRY(best.alloc(sizeof(unsigned long long) * R));
  if (freq_out) POST_TRY(freq.alloc(sizeof(double) * R));
  {
    // most probable signature per record, one block of records at a time
    const int64_t nb_max = std::min<int64_t>(R, std::max<int64_t>(1, PAIR_BLOCK / S));
    const int64_t np = nb_max * S;
    Buf keys_in, keys_out, samp_in, samp_out, off, tmp;
    POST_TRY(keys_in.alloc(sizeof(unsigned long long) * np));
    POST_TRY(keys_out.alloc(sizeof(unsigned long long) * np));
    POST_TRY(samp_in.alloc(sizeof(int32_t) * np));
    POST_TRY(samp_out.alloc(sizeof(int32_t) * np));
    POST_TRY(off.alloc(sizeof(int32_t) * (nb_max + 1)));
    size_t tb = 0;
    POST_TRY(cub::DeviceSegmentedRadixSort::SortPairs(
        nullptr, tb, (const unsigned long long *)nullptr, (unsigned long long *)nullptr, (const int32_t *)nullptr,
        (int32_t *)nullptr, (int)np, (int)nb_max, (const int32_t *)nullptr, (const int32_t *)nullptr, 0, 64, st));
    POST_TRY(tmp.alloc(tb));
    k_segment_offsets<<<grid_for(nb_max + 1), THREADS, 0, st>>>(nb_max, S, off.as<int32_t>());
    for (int64_t lo = 0; lo < R; lo += nb_max) {
      const int64_t nb = std::min<int64_t>(nb_max, R - lo);
      size_t tbb = tb;
      k_gather<<<grid_for(nb * S), THREADS, 0, st>>>(p->sig.as<unsigned long long>(), p->max_samples, lo, nb, S,
                                                     keys_in.as<unsigned long long>(), samp_in.as<int32_t>());
      POST_TRY(cub::DeviceSegmentedRadixSort::SortPairs(
          tmp.p, tbb, keys_in.as<unsigned long long>(), keys_out.as<unsigned long long>(), samp_in.as<int32_t>(),
          samp_out.as<int32_t>(), (int)(nb * S), (int)nb, off.as<int32_t>(), off.as<int32_t>() + 1, 0, 64, st));
      k_mode<<<grid_for(nb), THREADS, 0, st>>>(keys_out.as<unsigned long long>(), samp_out.as<int32_t>(), nb, S, lo,
                                               best.as<unsigned long long>(), freq_out ? freq.as<double>() : nullptr);
    }
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));  // the block buffers are freed here
  }
  if (freq_out) POST_TRY(cudaMemcpy(freq_out, freq.p, sizeof(double) * R, cudaMemcpyDeviceToHost));
  if (!labels_out) return DBL_OK;
  // group records by best signature, then scatter each group's smallest record index to its records
  Buf rec_in, keys_s, rec_s, head, start, labels, tmp;
  POST_TRY(rec_in.alloc(sizeof(int32_t) * R));
  POST_TRY(keys_s.alloc(sizeof(unsigned long long) * R));
  POST_TRY(rec_s.alloc(sizeof(int32_t) * R));
  POST_TRY(head.alloc(sizeof(int32_t) * R));
  POST_TRY(start.alloc(sizeof(int32_t) * R));
  POST_TRY(labels.alloc(sizeof(int32_t) * R));
  k_iota<<<grid_for(R), THREADS, 0, st>>>(R, rec_in.as<int32_t>());
  const int rc = group_by_key(R, 64, best.as<unsigned long long>(), rec_in.as<int32_t>(),
                              keys_s.as<unsigned long long>(), rec_s.as<int32_t>(), head.as<int32_t>(),
                              start.as<int32_t>(), tmp, st);
  if (rc != DBL_OK) return rc;
  k_scatter_labels<<<grid_for(R), THREADS, 0, st>>>(R, rec_s.as<int32_t>(), start.as<int32_t>(), labels.as<int32_t>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaMemcpyAsync(labels_out, labels.p, sizeof(int32_t) * R, cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// ---- posterior pairwise match counts -------------------------------------------------------------------------------
namespace {
constexpr int WARPS_PER_BLOCK = THREADS / 32;

// bits needed to hold every value in [0, n)
int bits_for(int64_t n) {
  int b = 1;
  while (b < 62 && (int64_t(1) << b) < n) ++b;
  return b;
}

__device__ __forceinline__ int64_t lower_bound_u64(const unsigned long long *__restrict__ a, int64_t n,
                                                   unsigned long long key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// the last position of each cluster writes the cluster's size at its first position
__global__ void k_cluster_sizes(int64_t R, const int32_t *__restrict__ lab, const int32_t *__restrict__ start,
                                int32_t *__restrict__ size_at_start) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x)
    if (i == R - 1 || lab[i] != lab[i + 1]) size_at_start[start[i]] = (int32_t)(i - start[i] + 1);
}

// row length of every sorted position: its partners are the later positions of its cluster; entry R is 0, so an
// exclusive scan over R + 1 entries ends with the sample's pair count
__global__ void k_row_lengths(int64_t R, const int32_t *__restrict__ start, const int32_t *__restrict__ size_at_start,
                              long long *__restrict__ row) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= R; i += (int64_t)gridDim.x * blockDim.x)
    row[i] = i < R ? (long long)start[i] + size_at_start[start[i]] - 1 - i : 0;
}

// one warp per sorted position writes that record's row of partners at its int64 offset: a cluster of k records is
// spread over k warps, whatever k is.  Members of a cluster are in ascending record index (the label sort is
// stable), so first < second.
__global__ void k_emit_pairs(int64_t R, const int32_t *__restrict__ rec, const long long *__restrict__ off,
                             unsigned long long *__restrict__ keys) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t w = blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5); w < R; w += nwarps) {
    const long long o = off[w], n = off[w + 1] - o;
    if (n == 0) continue;
    const unsigned long long hi = (unsigned long long)(uint32_t)rec[w] << 32;
    for (long long j = lane; j < n; j += 32) keys[o + j] = hi | (uint32_t)rec[w + 1 + j];
  }
}

// 1 for a sample key the held table does not have yet; entry n is 0, so an exclusive scan gives every new key its
// rank among the new ones and ends with their number
__global__ void k_probe_new(int64_t n, const unsigned long long *__restrict__ keys, int64_t H,
                            const unsigned long long *__restrict__ held, int32_t *__restrict__ is_new) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j <= n; j += (int64_t)gridDim.x * blockDim.x) {
    if (j == n) {
      is_new[j] = 0;
      continue;
    }
    const unsigned long long k = keys[j];
    const int64_t b = lower_bound_u64(held, H, k);
    is_new[j] = !(b < H && held[b] == k);
  }
}

// merge, held side: an entry moves up by the number of new keys below it, and counts one more if the sample has it
__global__ void k_merge_held(int64_t H, const unsigned long long *__restrict__ held, const int32_t *__restrict__ hcnt,
                             int64_t n, const unsigned long long *__restrict__ keys, const int32_t *__restrict__ rank,
                             unsigned long long *__restrict__ out_key, int32_t *__restrict__ out_cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < H; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = held[i];
    const int64_t lb = lower_bound_u64(keys, n, k);
    const int64_t pos = i + rank[lb];
    out_key[pos] = k;
    out_cnt[pos] = hcnt[i] + (lb < n && keys[lb] == k);
  }
}

// merge, sample side: a new key lands after the held entries below it and the new keys before it, with count 1
__global__ void k_merge_new(int64_t n, const unsigned long long *__restrict__ keys, const int32_t *__restrict__ is_new,
                            const int32_t *__restrict__ rank, int64_t H, const unsigned long long *__restrict__ held,
                            unsigned long long *__restrict__ out_key, int32_t *__restrict__ out_cnt) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    if (!is_new[j]) continue;
    const unsigned long long k = keys[j];
    const int64_t pos = lower_bound_u64(held, H, k) + rank[j];
    out_key[pos] = k;
    out_cnt[pos] = 1;
  }
}

// the keys of one sample (in any order) looked up in the held table: the sum of the counts of those it holds, a key it
// does not hold adding 0; summed per warp in uint64 and added with one atomic per warp, so the total is exact and
// does not depend on the order
__global__ void k_score_pairs(int64_t n, const unsigned long long *__restrict__ keys, int64_t H,
                              const unsigned long long *__restrict__ held, const int32_t *__restrict__ hcnt,
                              unsigned long long *__restrict__ sum) {
  unsigned long long acc = 0;
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[j];
    const int64_t b = lower_bound_u64(held, H, k);
    if (b < H && held[b] == k) acc += (uint32_t)hcnt[b];
  }
  acc = warp_sum_u64(acc);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(sum, acc);
}

__global__ void k_flag_min_count(int64_t H, const int32_t *__restrict__ cnt, int32_t min_count,
                                 int32_t *__restrict__ flag) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= H; i += (int64_t)gridDim.x * blockDim.x)
    flag[i] = i < H && cnt[i] >= min_count;
}

__global__ void k_scatter_pairs(int64_t H, const unsigned long long *__restrict__ key, const int32_t *__restrict__ cnt,
                                const int32_t *__restrict__ flag, const int32_t *__restrict__ pos,
                                int32_t *__restrict__ first, int32_t *__restrict__ second, int32_t *__restrict__ count) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < H; i += (int64_t)gridDim.x * blockDim.x) {
    if (!flag[i]) continue;
    const int32_t p = pos[i];
    first[p] = (int32_t)(key[i] >> 32);
    second[p] = (int32_t)(key[i] & 0xffffffffull);
    count[p] = cnt[i];
  }
}
}  // namespace

struct dbl_pairs : Handle {
  int64_t max_pairs = 0, H = 0;         // H = distinct pairs held
  int lab_bits = 1, key_bits = 33;      // radix sort end bits of the labels and of the pair keys
  Buf iota, lab_s, rec_s;               // record indices; labels and records sorted by label
  Buf head, start, size;                // run heads, cluster start per position, cluster size at its start
  Buf row, off;                         // int64 row lengths and their exclusive scan, R + 1 each
  Buf key_in, key_s, is_new, rank;      // grown on demand: the sample's pair keys (unsorted, sorted), merge ranks
  Buf tab_key[2], tab_cnt[2];           // grown on demand: held table (index cur), the one the next sample merges into
  int cur = 0;
  Buf tmp;                              // CUB temporary storage, grown on demand
  Buf score;                            // the uint64 count sum of dbl_pairs_score_sample
};

extern "C" int dbl_pairs_create(dbl_pairs **out, int64_t num_records, int64_t max_pairs) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || max_pairs <= 0 || max_pairs > INT32_MAX) return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_pairs *p) {
    const int64_t R = num_records;
    p->max_pairs = max_pairs;
    p->lab_bits = bits_for(R);
    p->key_bits = 32 + bits_for(R);
    const size_t r4 = sizeof(int32_t) * (size_t)R, r8 = sizeof(long long) * (size_t)(R + 1);
    if (p->iota.alloc(r4) != cudaSuccess || p->lab_s.alloc(r4) != cudaSuccess || p->rec_s.alloc(r4) != cudaSuccess ||
        p->head.alloc(r4) != cudaSuccess || p->start.alloc(r4) != cudaSuccess || p->size.alloc(r4) != cudaSuccess ||
        p->row.alloc(r8) != cudaSuccess || p->off.alloc(r8) != cudaSuccess ||
        p->score.alloc(sizeof(unsigned long long)) != cudaSuccess)
      return DBL_ERR_CUDA;
    k_iota<<<grid_for(R), THREADS, 0, p->stream>>>(R, p->iota.as<int32_t>());
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(p->stream));
    return DBL_OK;
  });
}

extern "C" void dbl_pairs_free(dbl_pairs *p) { free_handle(p); }

extern "C" int32_t dbl_pairs_num_samples(const dbl_pairs *p) { return p ? p->S : 0; }

// One sample's pair keys, unsorted, into key_in: check the labels; stable radix sort of (label, record); cluster
// starts and sizes; every position's row of partners and its int64 offset, whose total *n_out is the sample's pair
// count sum k(k-1)/2; refuse (DBL_ERR_INVALID) before allocating anything for the pairs if that count alone exceeds
// max_pairs; emit the keys.  Neither the held table nor S changes.
static int pairs_emit_sample(dbl_pairs *p, const int32_t *cluster, long long *n_out) {
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;

  // records grouped by label, ascending record index within a cluster; tmp is grown before anything uses it
  size_t tb = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, p->row.as<long long>(), p->off.as<long long>(), R + 1, st));
  POST_TRY(p->tmp.reserve(tb));
  const int rc = group_by_key(R, p->lab_bits, p->cluster.as<int32_t>(), p->iota.as<int32_t>(), p->lab_s.as<int32_t>(),
                              p->rec_s.as<int32_t>(), p->head.as<int32_t>(), p->start.as<int32_t>(), p->tmp, st);
  if (rc != DBL_OK) return rc;
  k_cluster_sizes<<<grid_for(R), THREADS, 0, st>>>(R, p->lab_s.as<int32_t>(), p->start.as<int32_t>(),
                                                   p->size.as<int32_t>());
  k_row_lengths<<<grid_for(R + 1), THREADS, 0, st>>>(R, p->start.as<int32_t>(), p->size.as<int32_t>(),
                                                     p->row.as<long long>());
  tb = p->tmp.cap;
  POST_TRY(cub::DeviceScan::ExclusiveSum(p->tmp.p, tb, p->row.as<long long>(), p->off.as<long long>(), R + 1, st));
  long long n = 0;
  POST_TRY(cudaMemcpyAsync(&n, p->off.as<long long>() + R, sizeof(long long), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  if (n > p->max_pairs) return DBL_ERR_INVALID;  // this sample alone: nothing allocated for its pairs

  const size_t cap8 = sizeof(unsigned long long) * (size_t)p->max_pairs;
  POST_TRY(p->key_in.reserve(sizeof(unsigned long long) * (size_t)n, cap8));
  if (n > 0)
    k_emit_pairs<<<(int)std::min<int64_t>((R + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 8192), THREADS, 0, st>>>(
        R, p->rec_s.as<int32_t>(), p->off.as<long long>(), p->key_in.as<unsigned long long>());
  *n_out = n;
  return DBL_OK;
}

// One sample: its pair keys (pairs_emit_sample); radix-sort them; merge them into the spare table (a binary search per
// key on either side gives its place); commit by swapping tables only if the union fits max_pairs.  A refusal or
// failure leaves the held table and S as they were.
extern "C" int dbl_pairs_add_sample(dbl_pairs *p, const int32_t *cluster) {
  if (!p || !cluster || p->S == INT32_MAX) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  long long n = 0;
  if (const int rc = pairs_emit_sample(p, cluster, &n); rc != DBL_OK) return rc;
  const int64_t H = p->H;
  cudaStream_t st = p->stream;

  // the sample's keys, sorted
  const size_t cap8 = sizeof(unsigned long long) * (size_t)p->max_pairs, cap4 = sizeof(int32_t) * (size_t)(p->max_pairs + 1);
  POST_TRY(p->key_s.reserve(sizeof(unsigned long long) * (size_t)n, cap8));
  POST_TRY(p->is_new.reserve(sizeof(int32_t) * (size_t)(n + 1), cap4));
  POST_TRY(p->rank.reserve(sizeof(int32_t) * (size_t)(n + 1), cap4));
  const unsigned long long *keys = p->key_s.as<unsigned long long>();
  if (n > 0) {
    size_t tbk = 0;
    POST_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tbk, (const unsigned long long *)nullptr,
                                            (unsigned long long *)nullptr, (int64_t)n, 0, p->key_bits, st));
    POST_TRY(p->tmp.reserve(tbk));
    tbk = p->tmp.cap;
    POST_TRY(cub::DeviceRadixSort::SortKeys(p->tmp.p, tbk, p->key_in.as<unsigned long long>(),
                                            p->key_s.as<unsigned long long>(), (int64_t)n, 0, p->key_bits, st));
  }

  // which keys are new, and their ranks among the new ones
  const unsigned long long *held = p->tab_key[p->cur].as<unsigned long long>();
  const int32_t *hcnt = p->tab_cnt[p->cur].as<int32_t>();
  k_probe_new<<<grid_for(n + 1), THREADS, 0, st>>>(n, keys, H, held, p->is_new.as<int32_t>());
  size_t tbr = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tbr, (const int32_t *)nullptr, (int32_t *)nullptr, (int64_t)n + 1,
                                         st));
  POST_TRY(p->tmp.reserve(tbr));
  tbr = p->tmp.cap;
  POST_TRY(cub::DeviceScan::ExclusiveSum(p->tmp.p, tbr, p->is_new.as<int32_t>(), p->rank.as<int32_t>(),
                                         (int64_t)n + 1, st));
  int32_t fresh = 0;
  POST_TRY(cudaMemcpyAsync(&fresh, p->rank.as<int32_t>() + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  const int64_t H2 = H + fresh;
  if (H2 > p->max_pairs) return DBL_ERR_INVALID;  // the union does not fit: the held table stays as it is

  // merge into the spare table, then commit
  const int nxt = p->cur ^ 1;
  POST_TRY(p->tab_key[nxt].reserve(sizeof(unsigned long long) * (size_t)H2, cap8));
  POST_TRY(p->tab_cnt[nxt].reserve(sizeof(int32_t) * (size_t)H2, sizeof(int32_t) * (size_t)p->max_pairs));
  unsigned long long *ok = p->tab_key[nxt].as<unsigned long long>();
  int32_t *oc = p->tab_cnt[nxt].as<int32_t>();
  if (H > 0)
    k_merge_held<<<grid_for(H), THREADS, 0, st>>>(H, held, hcnt, n, keys, p->rank.as<int32_t>(), ok, oc);
  if (n > 0)
    k_merge_new<<<grid_for(n), THREADS, 0, st>>>(n, keys, p->is_new.as<int32_t>(), p->rank.as<int32_t>(), H, held, ok,
                                                 oc);
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  p->cur = nxt;
  p->H = H2;
  ++p->S;
  return DBL_OK;
}

// One labelling scored against the held table: its pair keys (pairs_emit_sample), unsorted, each looked up in the
// table by k_score_pairs.  n = its pair count, K = the sum of the held counts of its pairs.
extern "C" int dbl_pairs_score_sample(dbl_pairs *p, const int32_t *cluster, int64_t *num_pairs_out,
                                      int64_t *count_sum_out) {
  if (!p || !cluster || !num_pairs_out || !count_sum_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  long long n = 0;
  if (const int rc = pairs_emit_sample(p, cluster, &n); rc != DBL_OK) return rc;
  const int64_t H = p->H;
  cudaStream_t st = p->stream;
  unsigned long long *sum = p->score.as<unsigned long long>(), K = 0;
  POST_TRY(cudaMemsetAsync(sum, 0, sizeof(unsigned long long), st));
  if (n > 0 && H > 0)
    k_score_pairs<<<grid_for(n), THREADS, 0, st>>>(n, p->key_in.as<unsigned long long>(), H,
                                                   p->tab_key[p->cur].as<unsigned long long>(),
                                                   p->tab_cnt[p->cur].as<int32_t>(), sum);
  POST_TRY(cudaMemcpyAsync(&K, sum, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  *num_pairs_out = n;
  *count_sum_out = (int64_t)K;
  return DBL_OK;
}

// the held pairs with count >= min_count, in table (ascending key) order: into device arrays when first != NULL
static int pairs_select(dbl_pairs *p, int32_t min_count, int64_t *n_out, int32_t *first, int32_t *second,
                        int32_t *count) {
  if (!p || !n_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  const int64_t H = p->H;
  cudaStream_t st = p->stream;
  Buf flag, pos, tmp;
  POST_TRY(flag.alloc(sizeof(int32_t) * (H + 1)));
  POST_TRY(pos.alloc(sizeof(int32_t) * (H + 1)));
  size_t tb = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int32_t *)nullptr, (int32_t *)nullptr, H + 1, st));
  POST_TRY(tmp.alloc(tb));
  const int32_t *cnt = p->tab_cnt[p->cur].as<int32_t>();
  k_flag_min_count<<<grid_for(H + 1), THREADS, 0, st>>>(H, cnt, min_count, flag.as<int32_t>());
  POST_TRY(cub::DeviceScan::ExclusiveSum(tmp.p, tb, flag.as<int32_t>(), pos.as<int32_t>(), H + 1, st));
  int32_t n = 0;
  POST_TRY(cudaMemcpyAsync(&n, pos.as<int32_t>() + H, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  *n_out = n;
  if (!first || n == 0 || H == 0) return DBL_OK;
  k_scatter_pairs<<<grid_for(H), THREADS, 0, st>>>(H, p->tab_key[p->cur].as<unsigned long long>(), cnt,
                                                   flag.as<int32_t>(), pos.as<int32_t>(), first, second, count);
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

extern "C" int dbl_pairs_count(dbl_pairs *p, int32_t min_count, int64_t *n_out) {
  return pairs_select(p, min_count, n_out, nullptr, nullptr, nullptr);
}

extern "C" int dbl_pairs_read(dbl_pairs *p, int32_t min_count, int32_t *first, int32_t *second, int32_t *count) {
  if (!p || !first || !second || !count) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  int64_t n = 0;
  int rc = dbl_pairs_count(p, min_count, &n);
  if (rc != DBL_OK || n == 0) return rc;
  Buf f, s, c;
  POST_TRY(f.alloc(sizeof(int32_t) * n));
  POST_TRY(s.alloc(sizeof(int32_t) * n));
  POST_TRY(c.alloc(sizeof(int32_t) * n));
  rc = pairs_select(p, min_count, &n, f.as<int32_t>(), s.as<int32_t>(), c.as<int32_t>());
  if (rc != DBL_OK) return rc;
  // host or device outputs: unified addressing picks the copy direction
  POST_TRY(cudaMemcpy(first, f.p, sizeof(int32_t) * n, cudaMemcpyDefault));
  POST_TRY(cudaMemcpy(second, s.p, sizeof(int32_t) * n, cudaMemcpyDefault));
  POST_TRY(cudaMemcpy(count, c.p, sizeof(int32_t) * n, cudaMemcpyDefault));
  return DBL_OK;
}

// ---- the Binder search: parallel single-record moves against the held table ----------------------------------------
namespace {
constexpr long long NO_MOVE = LLONG_MAX;

__global__ void k_widen_labels(int64_t R, const int32_t *__restrict__ in, unsigned long long *__restrict__ out) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    out[r] = (uint32_t)in[r];
}

__global__ void k_label_sizes(int64_t R, const int32_t *__restrict__ lab, int32_t *__restrict__ size) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(&size[lab[r]], 1);
}

// every held pair twice, once from each of its records: key = record << lab_bits | the partner's label, value = the
// pair's count.  Sorted, a record's entries are one segment, grouped by partner label.
__global__ void k_partner_keys(int64_t H, int lab_bits, const unsigned long long *__restrict__ held,
                               const int32_t *__restrict__ hcnt, const int32_t *__restrict__ lab,
                               unsigned long long *__restrict__ key, int32_t *__restrict__ val) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < 2 * H; e += (int64_t)gridDim.x * blockDim.x) {
    const bool from_first = e < H;
    const int64_t t = from_first ? e : e - H;
    const unsigned long long k = held[t];
    const uint32_t f = (uint32_t)(k >> 32), s = (uint32_t)(k & 0xffffffffull);
    key[e] = (unsigned long long)(from_first ? f : s) << lab_bits | (uint32_t)lab[from_first ? s : f];
    val[e] = hcnt[t];
  }
}

// One record per thread over its segment of the sorted entries (found by binary search): w_A = the counts of its
// partners in its own cluster A, then per partner cluster X (runs of equal labels, ascending) w_X and
// dJ = aS (|X| - |A| + 1) - b (w_X - w_A); a singleton (|A| > 1) is dJ = aS (1 - |A|) + b w_A and is tried first as
// destination -1, so a strict < keeps the least (dJ, destination).  A record with dJ < 0 proposes its move and claims
// its source and destination clusters with atomicMin on dJ; proposals are counted into *num_props.
__global__ void k_best_move(int64_t R, int lab_bits, int64_t n, const unsigned long long *__restrict__ key,
                            const int32_t *__restrict__ val, const int32_t *__restrict__ lab,
                            const int32_t *__restrict__ size, long long aS, long long b, long long *__restrict__ prop_dJ,
                            int32_t *__restrict__ prop_dest, long long *__restrict__ prop_dK,
                            long long *__restrict__ claim_dJ, unsigned long long *__restrict__ num_props) {
  const unsigned long long mask = (1ull << lab_bits) - 1;
  unsigned long long props = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t lo = lower_bound_u64(key, n, (unsigned long long)r << lab_bits);
    const int64_t hi = lower_bound_u64(key, n, (unsigned long long)(r + 1) << lab_bits);
    const int32_t A = lab[r];
    const long long sA = size[A];
    long long wA = 0;
    for (int64_t k = lo; k < hi; ++k)
      if ((key[k] & mask) == (unsigned long long)A) wA += val[k];
    long long best = NO_MOVE, best_dK = 0;
    int32_t dest = INT_MAX;
    if (sA > 1) {
      best = aS * (1 - sA) + b * wA;
      best_dK = -wA;
      dest = -1;
    }
    long long w = 0;
    for (int64_t k = lo; k < hi; ++k) {
      const unsigned long long X = key[k] & mask;
      w += val[k];
      if (k + 1 == hi || (key[k + 1] & mask) != X) {
        if (X != (unsigned long long)A) {
          const long long dK = w - wA, dJ = aS * (size[X] - sA + 1) - b * dK;
          if (dJ < best) {
            best = dJ;
            best_dK = dK;
            dest = (int32_t)X;
          }
        }
        w = 0;
      }
    }
    const bool propose = best < 0;
    prop_dJ[r] = propose ? best : NO_MOVE;
    prop_dest[r] = dest;
    prop_dK[r] = best_dK;
    if (propose) {
      atomicMin(&claim_dJ[A], best);
      if (dest >= 0) atomicMin(&claim_dJ[dest], best);
      ++props;
    }
  }
  props = warp_sum_u64(props);
  if ((threadIdx.x & 31) == 0 && props) atomicAdd(num_props, props);
}

// second stage of the claims: among the proposals of least dJ on a cluster, the least record index
__global__ void k_claim_record(int64_t R, const int32_t *__restrict__ lab, const long long *__restrict__ prop_dJ,
                               const int32_t *__restrict__ prop_dest, const long long *__restrict__ claim_dJ,
                               unsigned int *__restrict__ claim_i) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const long long dJ = prop_dJ[r];
    if (dJ == NO_MOVE) continue;
    const int32_t A = lab[r], X = prop_dest[r];
    if (claim_dJ[A] == dJ) atomicMin(&claim_i[A], (unsigned int)r);
    if (X >= 0 && claim_dJ[X] == dJ) atomicMin(&claim_i[X], (unsigned int)r);
  }
}

// A proposal that holds the claim of every cluster it touches moves its record: the record's group key becomes its
// destination's label, or R + r for a singleton (a key no cluster has); every other record keeps its label.  The
// round's moves, sum of dn = |X| - |A| + 1 and sum of dK go to stats[0..2], summed exactly in uint64.
__global__ void k_apply_moves(int64_t R, const int32_t *__restrict__ lab, const int32_t *__restrict__ size,
                              const long long *__restrict__ prop_dJ, const int32_t *__restrict__ prop_dest,
                              const long long *__restrict__ prop_dK, const long long *__restrict__ claim_dJ,
                              const unsigned int *__restrict__ claim_i, unsigned long long *__restrict__ gkey,
                              unsigned long long *__restrict__ stats) {
  unsigned long long moves = 0, dn = 0, dK = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t A = lab[r];
    unsigned long long k = (uint32_t)A;
    const long long dJ = prop_dJ[r];
    if (dJ != NO_MOVE) {
      const int32_t X = prop_dest[r];
      const bool win = claim_dJ[A] == dJ && claim_i[A] == (unsigned int)r &&
                       (X < 0 || (claim_dJ[X] == dJ && claim_i[X] == (unsigned int)r));
      if (win) {
        k = X >= 0 ? (unsigned long long)X : (unsigned long long)(R + r);
        ++moves;
        dn += (unsigned long long)((X >= 0 ? (long long)size[X] : 0ll) - size[A] + 1);
        dK += (unsigned long long)prop_dK[r];
      }
    }
    gkey[r] = k;
  }
  moves = warp_sum_u64(moves);
  dn = warp_sum_u64(dn);
  dK = warp_sum_u64(dK);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&stats[0], moves);
    atomicAdd(&stats[1], dn);
    atomicAdd(&stats[2], dK);
  }
}

// n = sum over clusters of C(size, 2), K = the counts of the held pairs whose records share a label: out[0], out[1]
__global__ void k_search_counts(int64_t R, const int32_t *__restrict__ size, int64_t H,
                                const unsigned long long *__restrict__ held, const int32_t *__restrict__ hcnt,
                                const int32_t *__restrict__ lab, unsigned long long *__restrict__ out) {
  unsigned long long n = 0, K = 0;
  const int64_t m = R > H ? R : H;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < R) n += (unsigned long long)size[i] * (unsigned long long)(size[i] - 1) / 2;
    if (i < H) {
      const unsigned long long k = held[i];
      if (lab[k >> 32] == lab[k & 0xffffffffull]) K += (uint32_t)hcnt[i];
    }
  }
  n = warp_sum_u64(n);
  K = warp_sum_u64(K);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], n);
    atomicAdd(&out[1], K);
  }
}
}  // namespace

// The search: check the start labels (into the handle's sample-label buffer) and group them canonically; then rounds of
// sizes, partner keys, their radix sort (2 lab_bits bits, double-buffered), best moves, the two-stage claims, the
// moves, and the canonical relabel by group_by_key, until no record proposes or max_rounds rounds are done.  Every
// buffer is the call's own (48 bytes per held pair and 56 per record, plus the handle's scratch and sort storage), so
// the table and S never change, whatever the outcome.
extern "C" int dbl_pairs_binder_search(dbl_pairs *p, int64_t a, int64_t b, const int32_t *start, int32_t max_rounds,
                                       int32_t *labels_out, int32_t *rounds_out, int32_t *converged_out,
                                       int64_t *moves, int64_t *dn, int64_t *dK, int64_t *n_out, int64_t *K_out) {
  if (!p || !start || !labels_out || !rounds_out || !converged_out || !moves || !dn || !dK || !n_out || !K_out ||
      max_rounds < 1 || b < 1 || b > (int64_t(1) << 16) || a < 0 || a > b)
    return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  if ((int64_t)p->S * p->R >= (int64_t(1) << 44)) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(start, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R, H = p->H, E = 2 * H;
  const int bits = p->lab_bits, gbits = bits_for(2 * R);
  cudaStream_t st = p->stream;
  const unsigned long long *held = p->tab_key[p->cur].as<unsigned long long>();
  const int32_t *hcnt = p->tab_cnt[p->cur].as<int32_t>();

  const size_t e8 = sizeof(unsigned long long) * (size_t)E, e4 = sizeof(int32_t) * (size_t)E;
  const size_t r4 = sizeof(int32_t) * (size_t)R, r8 = sizeof(long long) * (size_t)R;
  Buf key[2], val[2], lab, size, gkey, gkey_s, prop_dJ, prop_dest, prop_dK, claim_dJ, claim_i, stats;
  POST_TRY(key[0].alloc(e8));
  POST_TRY(key[1].alloc(e8));
  POST_TRY(val[0].alloc(e4));
  POST_TRY(val[1].alloc(e4));
  POST_TRY(lab.alloc(r4));
  POST_TRY(size.alloc(r4));
  POST_TRY(gkey.alloc(r8));
  POST_TRY(gkey_s.alloc(r8));
  POST_TRY(prop_dJ.alloc(r8));
  POST_TRY(prop_dest.alloc(r4));
  POST_TRY(prop_dK.alloc(r8));
  POST_TRY(claim_dJ.alloc(r8));
  POST_TRY(claim_i.alloc(r4));
  POST_TRY(stats.alloc(4 * sizeof(unsigned long long)));
  cub::DoubleBuffer<unsigned long long> kb(key[0].as<unsigned long long>(), key[1].as<unsigned long long>());
  cub::DoubleBuffer<int32_t> vb(val[0].as<int32_t>(), val[1].as<int32_t>());
  size_t tb = 0;
  if (E > 0) {
    POST_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, kb, vb, E, 0, 2 * bits, st));
    POST_TRY(p->tmp.reserve(tb));
  }
  unsigned long long *st4 = stats.as<unsigned long long>();
  int32_t *L = lab.as<int32_t>(), *Z = size.as<int32_t>();

  // the labels of gkey, grouped; each record labelled by its group's smallest record index
  auto relabel = [&]() {
    const int rc = group_by_key(R, gbits, gkey.as<unsigned long long>(), p->iota.as<int32_t>(),
                                gkey_s.as<unsigned long long>(), p->rec_s.as<int32_t>(), p->head.as<int32_t>(),
                                p->start.as<int32_t>(), p->tmp, st);
    if (rc == DBL_OK)
      k_scatter_labels<<<grid_for(R), THREADS, 0, st>>>(R, p->rec_s.as<int32_t>(), p->start.as<int32_t>(), L);
    return rc;
  };
  auto sizes = [&]() {
    POST_TRY(cudaMemsetAsync(Z, 0, r4, st));
    k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, L, Z);
    return DBL_OK;
  };
  k_widen_labels<<<grid_for(R), THREADS, 0, st>>>(R, p->cluster.as<int32_t>(), gkey.as<unsigned long long>());
  if (const int rc = relabel(); rc != DBL_OK) return rc;

  const long long aS = (long long)a * p->S;
  int32_t rounds = 0, converged = 0;
  for (;;) {
    if (const int rc = sizes(); rc != DBL_OK) return rc;
    if (E > 0) {
      k_partner_keys<<<grid_for(E), THREADS, 0, st>>>(H, bits, held, hcnt, L, kb.Current(), vb.Current());
      size_t tbs = p->tmp.cap;
      POST_TRY(cub::DeviceRadixSort::SortPairs(p->tmp.p, tbs, kb, vb, E, 0, 2 * bits, st));
    }
    POST_TRY(cudaMemsetAsync(claim_dJ.p, 0x7f, r8, st));  // above every dJ < 0
    POST_TRY(cudaMemsetAsync(claim_i.p, 0xff, r4, st));   // above every record index
    POST_TRY(cudaMemsetAsync(st4, 0, 4 * sizeof(unsigned long long), st));
    k_best_move<<<grid_for(R), THREADS, 0, st>>>(R, bits, E, kb.Current(), vb.Current(), L, Z, aS, b,
                                                 prop_dJ.as<long long>(), prop_dest.as<int32_t>(),
                                                 prop_dK.as<long long>(), claim_dJ.as<long long>(), st4 + 3);
    k_claim_record<<<grid_for(R), THREADS, 0, st>>>(R, L, prop_dJ.as<long long>(), prop_dest.as<int32_t>(),
                                                    claim_dJ.as<long long>(), claim_i.as<unsigned int>());
    unsigned long long props = 0;
    POST_TRY(cudaMemcpyAsync(&props, st4 + 3, sizeof(props), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    if (props == 0) {
      converged = 1;
      break;
    }
    if (rounds == max_rounds) break;
    k_apply_moves<<<grid_for(R), THREADS, 0, st>>>(R, L, Z, prop_dJ.as<long long>(), prop_dest.as<int32_t>(),
                                                   prop_dK.as<long long>(), claim_dJ.as<long long>(),
                                                   claim_i.as<unsigned int>(), gkey.as<unsigned long long>(), st4);
    if (const int rc = relabel(); rc != DBL_OK) return rc;
    unsigned long long log[3];
    POST_TRY(cudaMemcpyAsync(log, st4, sizeof(log), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    moves[rounds] = (int64_t)log[0];
    dn[rounds] = (int64_t)log[1];
    dK[rounds] = (int64_t)log[2];
    ++rounds;
  }

  // n and K of the result, from its sizes and one pass over the held table
  if (const int rc = sizes(); rc != DBL_OK) return rc;
  POST_TRY(cudaMemsetAsync(st4, 0, 2 * sizeof(unsigned long long), st));
  k_search_counts<<<grid_for(std::max(R, H)), THREADS, 0, st>>>(R, Z, H, held, hcnt, L, st4);
  unsigned long long nk[2];
  POST_TRY(cudaMemcpyAsync(nk, st4, sizeof(nk), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaMemcpyAsync(labels_out, L, r4, cudaMemcpyDefault, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  *rounds_out = rounds;
  *converged_out = converged;
  *n_out = (int64_t)nk[0];
  *K_out = (int64_t)nk[1];
  return DBL_OK;
}

// ---- every sample against the ground truth -------------------------------------------------------------------------
namespace {
// one key per record: its sample label above its true label, each in lab_bits bits
__global__ void k_pack_labels(int64_t R, int lab_bits, const int32_t *__restrict__ cluster,
                              const int32_t *__restrict__ truth, unsigned long long *__restrict__ key) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    key[r] = (unsigned long long)(uint32_t)cluster[r] << lab_bits | (uint32_t)truth[r];
}

// Over the sorted keys: the last position of each run of equal keys (one cell of the contingency table) and of each
// run of equal sample labels (one predicted cluster) finds its run's first position by binary search and adds
// C(run length, 2); cluster runs are counted.  out = {tp, pred_pairs, num_clusters}, summed exactly in uint64.
__global__ void k_eval_counts(int64_t R, int lab_bits, const unsigned long long *__restrict__ key,
                              unsigned long long *__restrict__ tp, unsigned long long *__restrict__ pred_pairs,
                              unsigned long long *__restrict__ num_clusters) {
  unsigned long long cell = 0, pred = 0, clusters = 0;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = key[i];
    const bool last = i == R - 1;
    if (last || key[i + 1] != k) {
      const unsigned long long n = (unsigned long long)(i + 1 - lower_bound_u64(key, i + 1, k));
      cell += n * (n - 1) / 2;
    }
    const unsigned long long hi = k >> lab_bits;
    if (last || (key[i + 1] >> lab_bits) != hi) {
      const unsigned long long n = (unsigned long long)(i + 1 - lower_bound_u64(key, i + 1, hi << lab_bits));
      pred += n * (n - 1) / 2;
      ++clusters;
    }
  }
  cell = warp_sum_u64(cell);
  pred = warp_sum_u64(pred);
  clusters = warp_sum_u64(clusters);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(tp, cell);
    atomicAdd(pred_pairs, pred);
    atomicAdd(num_clusters, clusters);
  }
}
}  // namespace

struct dbl_eval : Handle {
  int32_t max_samples = 0;
  int lab_bits = 1;                // bits of a label in [0, R)
  Buf truth;                       // true labels
  Buf key_in, key_s;               // packed (sample label, true label) per record, unsorted and sorted
  Buf tmp;                         // CUB temporary storage of the key sort
  Buf counts;                      // [3][max_samples] uint64: tp, pred_pairs, num_clusters per sample
};

extern "C" int dbl_eval_create(dbl_eval **out, int64_t num_records, const int32_t *truth, int32_t max_samples) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || !truth || max_samples <= 0) return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_eval *p) {
    const int64_t R = num_records;
    p->max_samples = max_samples;
    p->lab_bits = bits_for(R);
    const size_t r4 = sizeof(int32_t) * (size_t)R, r8 = sizeof(unsigned long long) * (size_t)R;
    size_t tb = 0;
    if (p->truth.alloc(r4) != cudaSuccess || p->key_in.alloc(r8) != cudaSuccess || p->key_s.alloc(r8) != cudaSuccess ||
        p->counts.alloc(3 * sizeof(unsigned long long) * (size_t)max_samples) != cudaSuccess ||
        cub::DeviceRadixSort::SortKeys(nullptr, tb, p->key_in.as<unsigned long long>(),
                                       p->key_s.as<unsigned long long>(), R, 0, 2 * p->lab_bits,
                                       p->stream) != cudaSuccess ||
        p->tmp.alloc(tb) != cudaSuccess)
      return DBL_ERR_CUDA;
    return p->take_labels(truth, p->truth);
  });
}

extern "C" void dbl_eval_free(dbl_eval *p) { free_handle(p); }

extern "C" int32_t dbl_eval_num_samples(const dbl_eval *p) { return p ? p->S : 0; }

// One sample: check the labels; pack (label, true label) per record into 2 lab_bits bits; radix-sort on those bits;
// one pass over the sorted keys writes the sample's three counts into column S.  S moves only on success.
extern "C" int dbl_eval_add_sample(dbl_eval *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  k_pack_labels<<<grid_for(R), THREADS, 0, st>>>(R, p->lab_bits, p->cluster.as<int32_t>(), p->truth.as<int32_t>(),
                                                 p->key_in.as<unsigned long long>());
  size_t tb = p->tmp.cap;
  POST_TRY(cub::DeviceRadixSort::SortKeys(p->tmp.p, tb, p->key_in.as<unsigned long long>(),
                                          p->key_s.as<unsigned long long>(), R, 0, 2 * p->lab_bits, st));
  unsigned long long *c = p->counts.as<unsigned long long>() + p->S;
  const int32_t M = p->max_samples;
  for (int j = 0; j < 3; ++j) POST_TRY(cudaMemsetAsync(c + (size_t)j * M, 0, sizeof(unsigned long long), st));
  k_eval_counts<<<grid_for(R), THREADS, 0, st>>>(R, p->lab_bits, p->key_s.as<unsigned long long>(), c, c + M,
                                                 c + 2 * (size_t)M);
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  ++p->S;
  return DBL_OK;
}

extern "C" int dbl_eval_read(dbl_eval *p, int64_t *tp, int64_t *pred_pairs, int64_t *num_clusters) {
  if (!p || !tp || !pred_pairs || !num_clusters) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  const unsigned long long *c = p->counts.as<unsigned long long>();
  const size_t M = (size_t)p->max_samples, bytes = sizeof(int64_t) * (size_t)p->S;
  POST_TRY(cudaMemcpyAsync(tp, c, bytes, cudaMemcpyDeviceToHost, p->stream));
  POST_TRY(cudaMemcpyAsync(pred_pairs, c + M, bytes, cudaMemcpyDeviceToHost, p->stream));
  POST_TRY(cudaMemcpyAsync(num_clusters, c + 2 * M, bytes, cudaMemcpyDeviceToHost, p->stream));
  POST_TRY(cudaStreamSynchronize(p->stream));
  return DBL_OK;
}

// ---- the variation-of-information estimate: cell histograms of every pair of held samples -------------------------
namespace {
constexpr int VI_SMEM_BINS = 64;  // cell sizes below this are summed per block in shared memory for row t

// every record's cluster size, then the largest into *max_size
__global__ void k_max_size(int64_t R, const int32_t *__restrict__ size, int32_t *__restrict__ max_size) {
  int32_t m = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    m = max(m, size[r]);
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(max_size, m);
}

// 1 for a record in a cluster of two or more of C_t (only those can be in a cell of two or more); entry R is 0, so an
// exclusive scan gives every flagged record its place and ends with their number
__global__ void k_flag_big(int64_t R, const int32_t *__restrict__ lab, const int32_t *__restrict__ size,
                           int32_t *__restrict__ flag) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r <= R; r += (int64_t)gridDim.x * blockDim.x)
    flag[r] = r < R && size[lab[r]] >= 2;
}

__global__ void k_scatter_flagged(int64_t R, const int32_t *__restrict__ flag, const int32_t *__restrict__ pos,
                                  int32_t *__restrict__ sel) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    if (flag[r]) sel[pos[r]] = (int32_t)r;
}

// one key per (sample s0 + i, selected record): i << 2 lab_bits | label in C_t << lab_bits | label in C_s; the
// selected records are in ascending index, so a sample's labels are read in order
__global__ void k_vi_keys(int64_t nsel, int32_t B, int lab_bits, int64_t R, const int32_t *__restrict__ sel,
                          const int32_t *__restrict__ lab_t, const int32_t *__restrict__ rows,
                          unsigned long long *__restrict__ key) {
  for (int32_t i = blockIdx.y; i < B; i += gridDim.y) {
    const int32_t *lab_s = rows + (int64_t)i * R;
    const unsigned long long hi = (unsigned long long)i << (2 * lab_bits);
    for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nsel; k += (int64_t)gridDim.x * blockDim.x) {
      const int32_t r = sel[k];
      key[(int64_t)i * nsel + k] = hi | (unsigned long long)(uint32_t)lab_t[r] << lab_bits | (uint32_t)lab_s[r];
    }
  }
}

// the length of the run of sorted keys that ends at i (key[i] == k): gallop back from i, then a binary search
__device__ __forceinline__ int64_t run_length(const unsigned long long *__restrict__ key, int64_t i,
                                              unsigned long long k) {
  int64_t known = i, step = 1, lo = 0;  // key[known] == k
  for (;;) {
    const int64_t j = i - step;
    if (j < 0) break;
    if (key[j] != k) {
      lo = j + 1;
      break;
    }
    known = j;
    step <<= 1;
  }
  return i + 1 - (lo + lower_bound_u64(key + lo, known - lo, k));
}

// Over the sorted keys of one batch: the last position of each run of n >= 2 equal keys (a cell of C_t ^ C_s) adds 1
// to G[t][n] and to G[s][n].  A warp's lanes take 32 consecutive positions; lanes with equal (s, n), or equal n for
// row t, are summed by __match_any_sync and add once, row t's small n into a shared-memory histogram first.
__global__ void k_vi_cells(int64_t n, int hi_shift, const unsigned long long *__restrict__ key, int32_t s0, int32_t t,
                           int64_t width, unsigned long long *__restrict__ G) {
  __shared__ unsigned long long hist[VI_SMEM_BINS];
  for (int j = threadIdx.x; j < VI_SMEM_BINS; j += blockDim.x) hist[j] = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  unsigned long long *Gt = G + (int64_t)t * width;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < n;
       base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = base + lane;
    int64_t len = 0;
    unsigned long long k = 0;
    if (i < n) {
      k = key[i];
      if (i > 0 && key[i - 1] == k && (i == n - 1 || key[i + 1] != k)) len = run_length(key, i, k);
    }
    const unsigned emit = __ballot_sync(0xffffffffu, len >= 2);
    if (len >= 2) {
      const int64_t s = s0 + (int64_t)(k >> hi_shift);
      const unsigned by_s = __match_any_sync(emit, (unsigned long long)s << 32 | (unsigned long long)len);
      if (lane == __ffs(by_s) - 1) atomicAdd(&G[s * width + len], (unsigned long long)__popc(by_s));
      const unsigned by_n = __match_any_sync(emit, (unsigned long long)len);
      if (lane == __ffs(by_n) - 1) {
        if (len < VI_SMEM_BINS) atomicAdd(&hist[len], (unsigned long long)__popc(by_n));
        else atomicAdd(&Gt[len], (unsigned long long)__popc(by_n));
      }
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < VI_SMEM_BINS && j < width; j += blockDim.x)
    if (hist[j]) atomicAdd(&Gt[j], hist[j]);
}
}  // namespace

struct dbl_vi : Handle {
  int32_t max_samples = 0;
  int lab_bits = 1;                       // bits of a label in [0, R)
  int32_t max_size = 0;                   // M, the largest cluster of any held sample
  int64_t batch_keys = PAIR_BLOCK;        // keys of one batch of samples s (at least the selected records of one)
  Buf rows;                               // [max_samples][R] held labels
  Buf size, peak;                         // cluster sizes of one sample; its largest (int32)
};

extern "C" int dbl_vi_create(dbl_vi **out, int64_t num_records, int32_t max_samples) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || max_samples <= 0) return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_vi *p) {
    const int64_t R = num_records;
    p->max_samples = max_samples;
    p->lab_bits = bits_for(R);
    const size_t r4 = sizeof(int32_t) * (size_t)R;
    if (p->rows.alloc(r4 * (size_t)max_samples) != cudaSuccess || p->size.alloc(r4) != cudaSuccess ||
        p->peak.alloc(sizeof(int32_t)) != cudaSuccess)
      return DBL_ERR_CUDA;  // the held label matrix does not fit
    return DBL_OK;
  });
}

extern "C" void dbl_vi_free(dbl_vi *p) { free_handle(p); }

extern "C" int32_t dbl_vi_num_samples(const dbl_vi *p) { return p ? p->S : 0; }

extern "C" int dbl_vi_set_batch_keys(dbl_vi *p, int64_t max_keys) {
  if (!p || max_keys < 1) return DBL_ERR_INVALID;
  p->batch_keys = max_keys;
  return DBL_OK;
}

// One sample: check the labels; its largest cluster; append it as row S.  S and M move only on success.
extern "C" int dbl_vi_add_sample(dbl_vi *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  int32_t *Z = p->size.as<int32_t>();
  POST_TRY(cudaMemsetAsync(Z, 0, sizeof(int32_t) * R, st));
  POST_TRY(cudaMemsetAsync(p->peak.p, 0, sizeof(int32_t), st));
  k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, p->cluster.as<int32_t>(), Z);
  k_max_size<<<grid_for(R), THREADS, 0, st>>>(R, Z, p->peak.as<int32_t>());
  POST_TRY(cudaMemcpyAsync(p->rows.as<int32_t>() + (size_t)p->S * R, p->cluster.p, sizeof(int32_t) * R,
                           cudaMemcpyDeviceToDevice, st));
  int32_t m = 0;
  POST_TRY(cudaMemcpyAsync(&m, p->peak.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  p->max_size = std::max(p->max_size, m);
  ++p->S;
  return DBL_OK;
}

// G[t][n] = sum over s != t of the cells of n >= 2 records in C_t ^ C_s, each unordered pair {t, s} counted once and
// added to both rows.  For every t: the sizes of C_t and its n_t records in clusters of two or more, in ascending index
// (flags, an exclusive scan, a scatter); then the samples s > t in batches of B, B n_t <= max(batch_keys, n_t) keys
// that fit 64 bits; per batch the keys (k_vi_keys), one radix sort over their 2 lab_bits + bits_for(B) bits, and one
// pass (k_vi_cells) over the sorted keys.  The held samples never change.
extern "C" int dbl_vi_cross(dbl_vi *p, int64_t width, int64_t *G_out) {
  if (!p || !G_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  if (width < (int64_t)p->max_size + 1 || width > INT64_MAX / 8 / p->S) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  const int64_t R = p->R;
  const int32_t S = p->S;
  const int b = p->lab_bits;
  cudaStream_t st = p->stream;
  const size_t gbytes = sizeof(unsigned long long) * (size_t)S * (size_t)width;
  Buf G, flag, pos, sel, key[2], tmp;
  POST_TRY(G.alloc(gbytes));
  POST_TRY(cudaMemsetAsync(G.p, 0, gbytes, st));
  if (S > 1) {
    POST_TRY(flag.alloc(sizeof(int32_t) * (size_t)(R + 1)));
    POST_TRY(pos.alloc(sizeof(int32_t) * (size_t)(R + 1)));
    POST_TRY(sel.alloc(sizeof(int32_t) * (size_t)R));
    const int32_t *rows = p->rows.as<int32_t>();
    int32_t *Z = p->size.as<int32_t>();
    size_t tb_scan = 0;
    POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb_scan, (const int32_t *)nullptr, (int32_t *)nullptr, R + 1, st));
    // the batch width in samples allowed by 64-bit keys: bits_for(B) <= 64 - 2 b
    const int64_t B_bits = (64 - 2 * b) >= 31 ? INT32_MAX : (int64_t(1) << (64 - 2 * b));
    // the key buffers grow on demand, never past the largest batch this call can make
    const int64_t most_keys = std::min<int64_t>(std::max<int64_t>(p->batch_keys, R), R * (int64_t)(S - 1));
    const size_t key_limit = sizeof(unsigned long long) * (size_t)most_keys;
    for (int32_t t = 0; t + 1 < S; ++t) {
      const int32_t *lab_t = rows + (size_t)t * R;
      POST_TRY(cudaMemsetAsync(Z, 0, sizeof(int32_t) * R, st));
      k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, lab_t, Z);
      k_flag_big<<<grid_for(R + 1), THREADS, 0, st>>>(R, lab_t, Z, flag.as<int32_t>());
      POST_TRY(tmp.reserve(tb_scan));
      size_t tb = tmp.cap;
      POST_TRY(cub::DeviceScan::ExclusiveSum(tmp.p, tb, flag.as<int32_t>(), pos.as<int32_t>(), R + 1, st));
      k_scatter_flagged<<<grid_for(R), THREADS, 0, st>>>(R, flag.as<int32_t>(), pos.as<int32_t>(), sel.as<int32_t>());
      int32_t nsel = 0;
      POST_TRY(cudaMemcpyAsync(&nsel, pos.as<int32_t>() + R, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      POST_TRY(cudaGetLastError());
      POST_TRY(cudaStreamSynchronize(st));
      if (nsel == 0) continue;  // C_t is all singletons: every cell with it is a singleton
      const int64_t B_max = std::min<int64_t>({(int64_t)S - 1 - t, std::max<int64_t>(1, p->batch_keys / nsel),
                                               B_bits});
      for (int32_t s0 = t + 1; s0 < S; s0 += (int32_t)B_max) {
        const int32_t B = (int32_t)std::min<int64_t>(B_max, S - s0);
        const int64_t n = (int64_t)B * nsel;
        const int end_bit = 2 * b + bits_for(B);
        POST_TRY(key[0].reserve(sizeof(unsigned long long) * (size_t)n, key_limit));
        POST_TRY(key[1].reserve(sizeof(unsigned long long) * (size_t)n, key_limit));
        cub::DoubleBuffer<unsigned long long> kb(key[0].as<unsigned long long>(), key[1].as<unsigned long long>());
        const dim3 grid((unsigned)std::min<int64_t>((nsel + THREADS - 1) / THREADS, 1024),
                        (unsigned)std::min<int32_t>(B, 65535));
        k_vi_keys<<<grid, THREADS, 0, st>>>(nsel, B, b, R, sel.as<int32_t>(), lab_t, rows + (size_t)s0 * R,
                                            kb.Current());
        size_t tbs = 0;
        POST_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tbs, kb, n, 0, end_bit, st));
        POST_TRY(tmp.reserve(tbs));
        tbs = tmp.cap;
        POST_TRY(cub::DeviceRadixSort::SortKeys(tmp.p, tbs, kb, n, 0, end_bit, st));
        k_vi_cells<<<grid_for(n), THREADS, 0, st>>>(n, 2 * b, kb.Current(), s0, t, width,
                                                    G.as<unsigned long long>());
        POST_TRY(cudaGetLastError());
      }
    }
  }
  // host or device output: unified addressing picks the copy direction
  POST_TRY(cudaMemcpyAsync(G_out, G.p, gbytes, cudaMemcpyDefault, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}
