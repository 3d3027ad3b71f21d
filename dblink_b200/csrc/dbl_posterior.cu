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
// On the same handle, the VI search (dbl_vi_search, same numbers as analysis_arrays.vi_search_rounds) and the cells of
// any labelling with every held sample (dbl_vi_score, as analysis_arrays.vi_label_cells) share one cell pass over
// radix-sorted (s, label in C_s, label in c) keys -- see vi_cell_batches; dbl_vi_score_samples keeps the cells of
// each sample apart (as analysis_arrays.vi_sample_cells), for the credible ball around a point estimate.
//
// Entity values per cluster of a point estimate (dbl_values_*, same numbers as analysis_arrays.EntityValueCounts): for
// one attribute, count(c, v) = the (sample, record of c) pairs whose entity has value v, in int64.  The handle holds a
// sorted table of (c << bits(V) | v, count); each sample's keys are radix-sorted, run-length encoded and merged into
// it by the merge kernels of dbl_pairs, with the run lengths as counts -- see dbl_values_add_sample.  The modes are a
// segmented arg-max over the table (dbl_values_modes).
//
// Clerical review of a point estimate (same integers as analysis_arrays.record_links / cluster_appearances): per
// record W, I and its strongest partner outside its cluster, per cluster its held internal pairs and their least
// count, by one pass over the held pair table (dbl_pairs_record_links); per record the samples holding its cluster of
// the estimate, by comparing its row of the sMPC signature matrix with the estimate's own signatures
// (dbl_posterior_cluster_counts).
//
// Capture histories (dbl_capture_*, same integers as analysis_arrays.capture_histories): per sample the number of
// clusters holding records of exactly each set of files, and per record the samples in which its cluster holds another
// record of each file.  Per sample, every record ORs its file bit into its cluster's history word (and, when the bit
// was already set, into its duplicate word), then one pass over the labels histograms the history words -- see
// dbl_capture_add_sample.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <cub/cub.cuh>
#include <new>
#include <vector>

#include "dbl_internal.h"

namespace {
// (signature, sample) pairs sorted per record block: bounds the block's temporaries (~2 GB) whatever R and S are
constexpr int64_t PAIR_BLOCK = int64_t(1) << 26;
constexpr int THREADS = 256;
constexpr int WARPS_PER_BLOCK = THREADS / 32;

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {  // splitmix64 finaliser
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

int grid_for(int64_t n) { return (int)std::min<int64_t>((n + THREADS - 1) / THREADS, 4096); }

// any of the R labels outside [0, bound) raises the flag; runs before anything indexes by label
__global__ void k_check_labels(int64_t R, int64_t bound, const int32_t *__restrict__ cluster, int *__restrict__ bad) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    if (cluster[r] < 0 || (int64_t)cluster[r] >= bound) *bad = 1;
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
  // reserve() that keeps the first `keep` bytes: copied on st, synchronised before the old buffer is freed
  cudaError_t reserve_keep(size_t need, size_t keep, cudaStream_t st) {
    if (need <= cap) return cudaSuccess;
    Buf nb;
    cudaError_t e = nb.alloc(std::max(need, cap > SIZE_MAX / 2 ? SIZE_MAX : 2 * cap));
    if (e == cudaSuccess && keep) e = cudaMemcpyAsync(nb.p, p, keep, cudaMemcpyDeviceToDevice, st);
    if (e == cudaSuccess && keep) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return e;
    std::swap(p, nb.p);
    std::swap(cap, nb.cap);
    return cudaSuccess;
  }
  void reset() {
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
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
  // DBL_ERR_INVALID when one is outside [0, bound), bound = R unless given
  int take_labels(const int32_t *labels, Buf &dst, int64_t bound = -1) {
    POST_TRY(cudaMemcpyAsync(dst.p, labels, sizeof(int32_t) * R, cudaMemcpyDefault, stream));
    POST_TRY(cudaMemsetAsync(bad.p, 0, sizeof(int), stream));
    k_check_labels<<<grid_for(R), THREADS, 0, stream>>>(R, bound < 0 ? R : bound, dst.as<int32_t>(), bad.as<int>());
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

// ---- how often each cluster of a labelling appears in the samples -------------------------------------------------
namespace {
// any of the C clusters without a record raises the flag (the labels are then not canonical for C)
template <class T>
__global__ void k_flag_empty(int64_t C, const T *__restrict__ size, int *__restrict__ bad) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < C; k += (int64_t)gridDim.x * blockDim.x)
    if (size[k] == 0) *bad = 1;
}

// one warp per record: the samples whose signature of the record equals the center's, over its row of the
// record-major signature matrix (32 consecutive samples per load)
__global__ void k_match_center(int64_t R, int32_t stride, int32_t S, const unsigned long long *__restrict__ sig,
                               const unsigned long long *__restrict__ center, int32_t *__restrict__ count) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t r = blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5); r < R; r += nwarps) {
    const unsigned long long c = center[r], *row = sig + r * stride;
    int32_t n = 0;
    for (int32_t s = lane; s - lane < S; s += 32) n += __popc(__ballot_sync(0xffffffffu, s < S && row[s] == c));
    if (lane == 0) count[r] = n;
  }
}
}  // namespace

// The labels (canonical for C) into the handle's label buffer and their cluster sizes by k_accumulate, which refuse
// a label outside [0, C) and an empty cluster; the center's signatures by k_signatures as one column of an R x 1
// matrix; then every record's row of the signature matrix against them.
extern "C" int dbl_posterior_cluster_counts(dbl_posterior *p, const int32_t *labels, int32_t num_clusters,
                                            int32_t *count_out) {
  if (!p || !labels || !count_out || num_clusters < 1 || num_clusters > p->R) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(labels, p->cluster, num_clusters); rc != DBL_OK) return rc;
  const int64_t R = p->R, C = num_clusters;
  cudaStream_t st = p->stream;
  const int32_t *c = p->cluster.as<int32_t>();
  unsigned long long *sum = p->sum.as<unsigned long long>();
  unsigned int *size = p->size.as<unsigned int>();
  POST_TRY(cudaMemsetAsync(sum, 0, sizeof(unsigned long long) * R, st));
  POST_TRY(cudaMemsetAsync(size, 0, sizeof(unsigned int) * R, st));
  k_accumulate<<<grid_for(R), THREADS, 0, st>>>(R, c, sum, size);
  k_flag_empty<<<grid_for(C), THREADS, 0, st>>>(C, size, p->bad.as<int>());  // bad is 0 after take_labels
  int flag = 0;
  POST_TRY(cudaMemcpyAsync(&flag, p->bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  if (flag) return DBL_ERR_INVALID;
  Buf center, count;
  POST_TRY(center.alloc(sizeof(unsigned long long) * R));
  POST_TRY(count.alloc(sizeof(int32_t) * R));
  k_signatures<<<grid_for(R), THREADS, 0, st>>>(R, 1, 0, c, sum, size, center.as<unsigned long long>());
  k_match_center<<<(int)std::min<int64_t>((R + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 8192), THREADS, 0, st>>>(
      R, p->max_samples, p->S, p->sig.as<unsigned long long>(), center.as<unsigned long long>(), count.as<int32_t>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaMemcpyAsync(count_out, count.p, sizeof(int32_t) * R, cudaMemcpyDefault, st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// ---- posterior pairwise match counts -------------------------------------------------------------------------------
namespace {
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

// merge, held side: an entry moves up by the number of new keys below it, and counts add[lb] more (1 when add is
// null) if the sample has it.  Cnt is int32 for the pairs table, int64 for the entity-value table.
template <class Cnt>
__global__ void k_merge_held(int64_t H, const unsigned long long *__restrict__ held, const Cnt *__restrict__ hcnt,
                             int64_t n, const unsigned long long *__restrict__ keys, const int32_t *__restrict__ add,
                             const int32_t *__restrict__ rank, unsigned long long *__restrict__ out_key,
                             Cnt *__restrict__ out_cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < H; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = held[i];
    const int64_t lb = lower_bound_u64(keys, n, k);
    const int64_t pos = i + rank[lb];
    out_key[pos] = k;
    out_cnt[pos] = hcnt[i] + (lb < n && keys[lb] == k ? (add ? (Cnt)add[lb] : (Cnt)1) : (Cnt)0);
  }
}

// merge, sample side: a new key lands after the held entries below it and the new keys before it, with count add[j]
// (1 when add is null)
template <class Cnt>
__global__ void k_merge_new(int64_t n, const unsigned long long *__restrict__ keys, const int32_t *__restrict__ add,
                            const int32_t *__restrict__ is_new, const int32_t *__restrict__ rank, int64_t H,
                            const unsigned long long *__restrict__ held, unsigned long long *__restrict__ out_key,
                            Cnt *__restrict__ out_cnt) {
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    if (!is_new[j]) continue;
    const unsigned long long k = keys[j];
    const int64_t pos = lower_bound_u64(held, H, k) + rank[j];
    out_key[pos] = k;
    out_cnt[pos] = add ? (Cnt)add[j] : (Cnt)1;
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

// The n sorted distinct keys of a sample against a held sorted table of H keys: is_new[j] = 1 for a key the table
// lacks, rank = the exclusive scan of is_new over n + 1 entries, *fresh_out = the number of new keys.  is_new and rank
// must hold n + 1 entries; tmp grows to the scan's temporary storage.
int probe_new_keys(int64_t n, const unsigned long long *keys, int64_t H, const unsigned long long *held, Buf &is_new,
                   Buf &rank, Buf &tmp, cudaStream_t st, int64_t *fresh_out) {
  k_probe_new<<<grid_for(n + 1), THREADS, 0, st>>>(n, keys, H, held, is_new.as<int32_t>());
  size_t tbr = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tbr, (const int32_t *)nullptr, (int32_t *)nullptr, (int64_t)n + 1,
                                         st));
  POST_TRY(tmp.reserve(tbr));
  tbr = tmp.cap;
  POST_TRY(cub::DeviceScan::ExclusiveSum(tmp.p, tbr, is_new.as<int32_t>(), rank.as<int32_t>(), (int64_t)n + 1, st));
  int32_t fresh = 0;
  POST_TRY(cudaMemcpyAsync(&fresh, rank.as<int32_t>() + n, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  *fresh_out = fresh;
  return DBL_OK;
}

// The union of the held table (held, hcnt; H entries) and the probed sample keys (probe_new_keys), each sample key
// counting add[j] (1 when add is null), into (out_key, out_cnt), H + fresh entries; synchronised.
template <class Cnt>
int merge_keys(int64_t H, const unsigned long long *held, const Cnt *hcnt, int64_t n, const unsigned long long *keys,
               const int32_t *add, const Buf &is_new, const Buf &rank, unsigned long long *out_key, Cnt *out_cnt,
               cudaStream_t st) {
  if (H > 0)
    k_merge_held<Cnt><<<grid_for(H), THREADS, 0, st>>>(H, held, hcnt, n, keys, add, rank.as<int32_t>(), out_key,
                                                       out_cnt);
  if (n > 0)
    k_merge_new<Cnt><<<grid_for(n), THREADS, 0, st>>>(n, keys, add, is_new.as<int32_t>(), rank.as<int32_t>(), H, held,
                                                      out_key, out_cnt);
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
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
  Buf trace;                            // dbl_pairs_trace_begin: [ceil(P / 32)][H] uint32 bits, word-major
  int32_t trace_P = 0;                  // its positions P; 0 = no trace
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
  int64_t fresh = 0;
  if (const int rc = probe_new_keys(n, keys, H, held, p->is_new, p->rank, p->tmp, st, &fresh); rc != DBL_OK) return rc;
  const int64_t H2 = H + fresh;
  if (H2 > p->max_pairs) return DBL_ERR_INVALID;  // the union does not fit: the held table stays as it is

  // merge into the spare table, then commit
  const int nxt = p->cur ^ 1;
  POST_TRY(p->tab_key[nxt].reserve(sizeof(unsigned long long) * (size_t)H2, cap8));
  POST_TRY(p->tab_cnt[nxt].reserve(sizeof(int32_t) * (size_t)H2, sizeof(int32_t) * (size_t)p->max_pairs));
  if (const int rc = merge_keys<int32_t>(H, held, hcnt, n, keys, nullptr, p->is_new, p->rank,
                                         p->tab_key[nxt].as<unsigned long long>(), p->tab_cnt[nxt].as<int32_t>(), st);
      rc != DBL_OK)
    return rc;
  p->cur = nxt;
  p->H = H2;
  ++p->S;
  p->trace.reset();  // its rows were the old table's pairs
  p->trace_P = 0;
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

// ---- per-pair MCMC diagnostics: split-R̂ and effective sample size of every held pair's link indicator -------------
// A bit trace holds x_s(pair) = 1[the pair shares a cluster in sample s] for every held pair and pooled position s,
// word-major ([ceil(P / 32)][H] uint32), filled one sample at a time by looking its pair keys up in the held table.
// dbl_pairs_mixing splits each of K chains (n draws from a start position) into two halves of N = n / 2 draws and
// computes, per pair, in int64 (see analysis_arrays.pairwise_match_diagnostics for the definitions):
//   L_m[tau] = sum_{t < N - tau} x_t x_{t + tau},  h_m[tau] = sum_{t < N - tau} x_t,  g_m[tau] = sum_{t >= tau} x_t,
//   Q_m[tau] = N^2 L - N c_m (h + g) + (N - tau) c_m^2  (N^3 x the half's biased autocovariance),  A = sum_m Q_m,
//   V = (M - 1)(N - 1) A[0] + N (N - 1) (M sum c_m^2 - (sum c_m)^2),  Wn = (M - 1) N A[0],
//   u[0] = 2 V,  u[tau] = 2 (V - Wn + (M - 1)(N - 1) A[tau]),
// R̂ = sqrt(V / Wn), and Geyer's initial positive and monotone sequences over the lag pairs of u, streamed: the
// monotone sequence makes each pair sum the running minimum of those before it.  Every integer fits int64 when
// M N^2 < 2^30 (so M^2 N^4 < 2^60).
namespace {
constexpr int64_t MAX_TRACE_WORDS = int64_t(1) << 31;
constexpr int64_t MIXING_SIZE_BOUND = int64_t(1) << 30;  // M N^2 below this

// every key of one sample found in the held table sets bit `pos` of that pair's row; keys it does not hold are ignored
__global__ void k_mark_pairs(int64_t n, const unsigned long long *__restrict__ keys, int64_t H,
                             const unsigned long long *__restrict__ held, int32_t pos, uint32_t *__restrict__ trace) {
  uint32_t *row = trace + (int64_t)(pos >> 5) * H;
  const uint32_t bit = 1u << (pos & 31);
  for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < n; j += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[j];
    const int64_t b = lower_bound_u64(held, H, k);
    if (b < H && held[b] == k) atomicOr(row + b, bit);
  }
}

// the low `k` bits set (none for k <= 0, all for k >= 32)
__device__ __forceinline__ uint32_t low_bits(int64_t k) {
  return k <= 0 ? 0u : k >= 32 ? 0xffffffffu : (1u << k) - 1u;
}

// bits s .. s + 31 of pair h's row (positions at or past the trace's end read 0)
__device__ __forceinline__ uint32_t trace_bits(const uint32_t *__restrict__ trace, int64_t H, int64_t W, int64_t h,
                                               int64_t s) {
  const int64_t w = s >> 5;
  const uint32_t lo = w < W ? trace[w * H + h] : 0u, hi = w + 1 < W ? trace[(w + 1) * H + h] : 0u;
  return __funnelshift_r(lo, hi, (uint32_t)(s & 31));
}

// One warp per held pair with count >= min_count, written at out[pos[h]].  The lanes take 32 lags at a time; each lane
// walks the 2K halves once per batch, so the halves' counts come with every batch.  The Geyer pass runs on every lane
// (the lag values are shuffled to all), and the warp stops as soon as the sequence truncates.
__global__ void k_pair_mixing(int64_t H, const int32_t *__restrict__ flag, const int32_t *__restrict__ pos,
                              const uint32_t *__restrict__ trace, int64_t W, int32_t K,
                              const int32_t *__restrict__ starts, int32_t n, double ess_floor,
                              int32_t *__restrict__ c_out, int32_t *__restrict__ cmin_out,
                              int32_t *__restrict__ cmax_out, int32_t *__restrict__ maxt_out,
                              double *__restrict__ rhat_out, double *__restrict__ ess_out) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  const int64_t N = n / 2, M = 2 * (int64_t)K, nw = (N + 31) / 32;
  for (int64_t h = blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5); h < H; h += nwarps) {
    if (!flag[h]) continue;
    long long V = 0, Wn = 0, acc_even = 0, run_min = 0, cur = 0, sum_c = 0;
    int32_t cmin = INT32_MAX, cmax = 0;
    int64_t t = 0;
    double acc = 0.0;
    bool stop = false;
    for (int64_t base = 0; !stop; base += 32) {
      const int64_t tau = base + lane;
      long long A = 0, S1 = 0, S2 = 0;
      for (int32_t k = 0; k < K; ++k) {
        int32_t chain_c = 0;
        for (int half = 0; half < 2; ++half) {
          const int64_t s0 = (int64_t)starts[k] + (half ? n - N : 0);
          long long L = 0, hh = 0, gg = 0, c = 0;
          for (int64_t i = 0; i < nw; ++i) {
            const uint32_t x = trace_bits(trace, H, W, h, s0 + 32 * i) & low_bits(N - 32 * i);
            const uint32_t y = trace_bits(trace, H, W, h, s0 + tau + 32 * i);
            const uint32_t mk = low_bits(N - tau - 32 * i);
            L += __popc(x & y & mk);
            hh += __popc(x & mk);
            gg += __popc(y & mk);
            c += __popc(x);
          }
          A += N * N * L - N * c * (hh + gg) + (N - tau) * c * c;
          S1 += c;
          S2 += c * c;
          chain_c += (int32_t)c;
        }
        cmin = min(cmin, chain_c);
        cmax = max(cmax, chain_c);
      }
      if (base == 0) {
        const long long A0 = __shfl_sync(0xffffffffu, A, 0);
        V = (M - 1) * (N - 1) * A0 + N * (N - 1) * (M * S2 - S1 * S1);
        Wn = (M - 1) * N * A0;
        sum_c = S1;
        if (V == 0) break;
      }
      const long long u = tau == 0 ? 2 * V : 2 * (V - Wn + (M - 1) * (N - 1) * A);
      // the lag pairs of this batch, in order, until the sequence truncates
      for (int j = 0; j < 32 && !stop; j += 2) {
        const long long even = __shfl_sync(0xffffffffu, u, j), odd = __shfl_sync(0xffffffffu, u, j + 1);
        const long long P = even + odd;
        if (base + j == 0) {
          run_min = cur = P;
        } else {
          acc = __dadd_rn(acc, __ll2double_rn(cur));  // the previous pair lies before max_t
          t = base + j;
          cur = min(P, run_min);
          run_min = cur;
        }
        if (!(t < N - 5 && P > 0)) {
          stop = true;
          acc_even = (P >= 0 || even > 0) ? even : 0;
        }
      }
    }
    if (lane == 0) {
      const int64_t o = pos[h];
      c_out[o] = (int32_t)sum_c;
      cmin_out[o] = cmin;
      cmax_out[o] = cmax;
      if (V == 0) {
        maxt_out[o] = 0;
        rhat_out[o] = __longlong_as_double(0x7ff8000000000000ll);  // NaN
        ess_out[o] = __longlong_as_double(0x7ff8000000000000ll);
      } else {
        maxt_out[o] = (int32_t)t;
        rhat_out[o] = Wn > 0 ? __dsqrt_rn(__ddiv_rn(__ll2double_rn(V), __ll2double_rn(Wn)))
                             : __longlong_as_double(0x7ff0000000000000ll);  // +inf
        const double num = __dadd_rn(__dadd_rn(acc, acc), __ll2double_rn(acc_even));
        const double tau_hat = __dadd_rn(-1.0, __ddiv_rn(num, __ll2double_rn(2 * V)));
        ess_out[o] = __ddiv_rn(__ll2double_rn(M * N), tau_hat > ess_floor ? tau_hat : ess_floor);
      }
    }
  }
}
}  // namespace

// A zeroed trace of num_positions bits per held pair; replaces any earlier one.
extern "C" int dbl_pairs_trace_begin(dbl_pairs *p, int32_t num_positions) {
  if (!p || num_positions < 1) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  const int64_t W = ((int64_t)num_positions + 31) / 32;
  if (p->H > 0 && W > MAX_TRACE_WORDS / p->H) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  p->trace.reset();
  p->trace_P = 0;
  const size_t bytes = sizeof(uint32_t) * (size_t)(W * p->H);
  POST_TRY(p->trace.alloc(bytes));
  POST_TRY(cudaMemsetAsync(p->trace.p, 0, bytes, p->stream));
  POST_TRY(cudaStreamSynchronize(p->stream));
  p->trace_P = num_positions;
  return DBL_OK;
}

// One labelling's pairs (pairs_emit_sample) set bit `position` of the held pairs among them.
extern "C" int dbl_pairs_trace_sample(dbl_pairs *p, const int32_t *cluster, int32_t position) {
  if (!p || !cluster) return DBL_ERR_INVALID;
  if (p->trace_P == 0) return DBL_ERR_STATE;
  if (position < 0 || position >= p->trace_P) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  long long n = 0;
  if (const int rc = pairs_emit_sample(p, cluster, &n); rc != DBL_OK) return rc;
  cudaStream_t st = p->stream;
  if (n > 0 && p->H > 0)
    k_mark_pairs<<<grid_for(n), THREADS, 0, st>>>(n, p->key_in.as<unsigned long long>(), p->H,
                                                  p->tab_key[p->cur].as<unsigned long long>(), position,
                                                  p->trace.as<uint32_t>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// split-R̂ and ESS of every held pair with count >= min_count, in dbl_pairs_read order.
extern "C" int dbl_pairs_mixing(dbl_pairs *p, int32_t min_count, int32_t num_chains, const int32_t *chain_starts,
                                int32_t draws, double ess_floor, int32_t *count_out, int32_t *chain_min_out,
                                int32_t *chain_max_out, int32_t *max_t_out, double *rhat_out, double *ess_out) {
  if (!p || !chain_starts || !count_out || !chain_min_out || !chain_max_out || !max_t_out || !rhat_out || !ess_out)
    return DBL_ERR_INVALID;
  if (p->trace_P == 0) return DBL_ERR_STATE;
  const int64_t N = draws / 2, M = 2 * (int64_t)num_chains;
  // N <= 2^15 keeps M N^2 inside int64 for any K
  if (num_chains < 1 || N < 2 || N > 32768 || M * N * N >= MIXING_SIZE_BOUND) return DBL_ERR_INVALID;
  for (int32_t k = 0; k < num_chains; ++k)
    if (chain_starts[k] < 0 || (int64_t)chain_starts[k] + draws > p->trace_P) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  const int64_t H = p->H, W = ((int64_t)p->trace_P + 31) / 32;
  cudaStream_t st = p->stream;
  Buf flag, pos, tmp, starts;
  POST_TRY(flag.alloc(sizeof(int32_t) * (H + 1)));
  POST_TRY(pos.alloc(sizeof(int32_t) * (H + 1)));
  POST_TRY(starts.alloc(sizeof(int32_t) * num_chains));
  POST_TRY(cudaMemcpyAsync(starts.p, chain_starts, sizeof(int32_t) * num_chains, cudaMemcpyHostToDevice, st));
  size_t tb = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int32_t *)nullptr, (int32_t *)nullptr, H + 1, st));
  POST_TRY(tmp.alloc(tb));
  k_flag_min_count<<<grid_for(H + 1), THREADS, 0, st>>>(H, p->tab_cnt[p->cur].as<int32_t>(), min_count,
                                                        flag.as<int32_t>());
  POST_TRY(cub::DeviceScan::ExclusiveSum(tmp.p, tb, flag.as<int32_t>(), pos.as<int32_t>(), H + 1, st));
  int32_t sel = 0;
  POST_TRY(cudaMemcpyAsync(&sel, pos.as<int32_t>() + H, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  if (sel == 0) return DBL_OK;
  Buf out4[4], out8[2];
  for (Buf &b : out4) POST_TRY(b.alloc(sizeof(int32_t) * (size_t)sel));
  for (Buf &b : out8) POST_TRY(b.alloc(sizeof(double) * (size_t)sel));
  k_pair_mixing<<<(int)std::min<int64_t>((H + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 8192), THREADS, 0, st>>>(
      H, flag.as<int32_t>(), pos.as<int32_t>(), p->trace.as<uint32_t>(), W, num_chains, starts.as<int32_t>(), draws,
      ess_floor, out4[0].as<int32_t>(), out4[1].as<int32_t>(), out4[2].as<int32_t>(), out4[3].as<int32_t>(),
      out8[0].as<double>(), out8[1].as<double>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  // host or device outputs: unified addressing picks the copy direction
  int32_t *o4[4] = {count_out, chain_min_out, chain_max_out, max_t_out};
  double *o8[2] = {rhat_out, ess_out};
  for (int i = 0; i < 4; ++i) POST_TRY(cudaMemcpy(o4[i], out4[i].p, sizeof(int32_t) * (size_t)sel, cudaMemcpyDefault));
  for (int i = 0; i < 2; ++i) POST_TRY(cudaMemcpy(o8[i], out8[i].p, sizeof(double) * (size_t)sel, cudaMemcpyDefault));
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
// round's moves, sum of dn = |X| - |A| + 1 and sum of the proposals' int64 payloads (the Binder search's dK, the VI
// search's dJ) go to stats[0..2], summed exactly in uint64.
__global__ void k_apply_moves(int64_t R, const int32_t *__restrict__ lab, const int32_t *__restrict__ size,
                              const long long *__restrict__ prop_dJ, const int32_t *__restrict__ prop_dest,
                              const long long *__restrict__ payload, const long long *__restrict__ claim_dJ,
                              const unsigned int *__restrict__ claim_i, unsigned long long *__restrict__ gkey,
                              unsigned long long *__restrict__ stats) {
  unsigned long long moves = 0, dn = 0, sum = 0;
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
        sum += (unsigned long long)payload[r];
      }
    }
    gkey[r] = k;
  }
  moves = warp_sum_u64(moves);
  dn = warp_sum_u64(dn);
  sum = warp_sum_u64(sum);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&stats[0], moves);
    atomicAdd(&stats[1], dn);
    atomicAdd(&stats[2], sum);
  }
}

// The labels after a round's moves: records grouped by their group key gkey (gbits bits), each labelled by its group's
// smallest record index into L.  gkey_s, rec_s, head and start are R entries of scratch each; tmp grows as the sort
// and scan need.
int canonical_relabel(int64_t R, int gbits, const unsigned long long *gkey, const int32_t *iota,
                      unsigned long long *gkey_s, int32_t *rec_s, int32_t *head, int32_t *start, int32_t *L, Buf &tmp,
                      cudaStream_t st) {
  const int rc = group_by_key(R, gbits, gkey, iota, gkey_s, rec_s, head, start, tmp, st);
  if (rc == DBL_OK) k_scatter_labels<<<grid_for(R), THREADS, 0, st>>>(R, rec_s, start, L);
  return rc;
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
    return canonical_relabel(R, gbits, gkey.as<unsigned long long>(), p->iota.as<int32_t>(),
                             gkey_s.as<unsigned long long>(), p->rec_s.as<int32_t>(), p->head.as<int32_t>(),
                             p->start.as<int32_t>(), L, p->tmp, st);
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

// ---- every record's links against a labelling, for clerical review ------------------------------------------------
namespace {
// Per held pair (f, s, n), f < s: W of both records += n; when lab[f] == lab[s], I of both += n and the cluster gets
// one more held internal pair and min= n as its least count; otherwise each record's strongest outside partner
// max= n << 32 | (0xFFFFFFFF - partner), so ties go to the smaller partner.  The table is sorted by f, so the lanes
// of a warp mostly share f: f's updates are reduced over each run of equal f in the warp (a segmented shuffle
// reduction) and applied once by the run's first lane; s's go straight to atomics.  Every update is an integer
// atomic, so the result does not depend on their order.
__global__ void k_record_links(int64_t H, const unsigned long long *__restrict__ held, const int32_t *__restrict__ hcnt,
                               const int32_t *__restrict__ lab, unsigned long long *__restrict__ W,
                               unsigned long long *__restrict__ I, unsigned long long *__restrict__ best,
                               unsigned long long *__restrict__ inner, unsigned int *__restrict__ least) {
  const int lane = threadIdx.x & 31;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < H;
       base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = base + lane;
    uint32_t f = 0xffffffffu;  // no record: R <= 2^31 - 1
    int32_t L = 0;
    unsigned long long w = 0, in = 0, top = 0, pairs = 0;
    unsigned int lo = 0xffffffffu;
    if (e < H) {
      const unsigned long long k = held[e];
      f = (uint32_t)(k >> 32);
      const uint32_t s = (uint32_t)(k & 0xffffffffull), n = (uint32_t)hcnt[e];
      L = lab[f];
      w = n;
      atomicAdd(&W[s], w);
      if (L == lab[s]) {
        in = n;
        pairs = 1;
        lo = n;
        atomicAdd(&I[s], in);
      } else {
        top = (unsigned long long)n << 32 | (0xffffffffu - s);
        atomicMax(&best[s], (unsigned long long)n << 32 | (0xffffffffu - f));
      }
    }
    const uint32_t prev = __shfl_up_sync(0xffffffffu, f, 1);
    const bool head = lane == 0 || prev != f;
    const unsigned later = __ballot_sync(0xffffffffu, head) & ~((2u << lane) - 1u);  // lane 31: 2u << 31 == 0
    const int end = later ? __ffs(later) - 1 : 32;  // one past the last lane of this lane's run
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long w2 = __shfl_down_sync(0xffffffffu, w, o), in2 = __shfl_down_sync(0xffffffffu, in, o);
      const unsigned long long top2 = __shfl_down_sync(0xffffffffu, top, o);
      const unsigned long long pairs2 = __shfl_down_sync(0xffffffffu, pairs, o);
      const unsigned int lo2 = __shfl_down_sync(0xffffffffu, lo, o);
      if (lane + o < end) {
        w += w2;
        in += in2;
        top = top2 > top ? top2 : top;
        pairs += pairs2;
        lo = lo2 < lo ? lo2 : lo;
      }
    }
    if (head && e < H) {
      atomicAdd(&W[f], w);
      if (in) atomicAdd(&I[f], in);
      if (top) atomicMax(&best[f], top);
      if (pairs) {
        atomicAdd(&inner[L], pairs);
        atomicMin(&least[L], lo);
      }
    }
  }
}

// the packed partners as (partner, count), -1 and 0 for none; the least internal count, 0 for a cluster without one
__global__ void k_links_out(int64_t R, int64_t C, const unsigned long long *__restrict__ best,
                            const unsigned long long *__restrict__ inner, const unsigned int *__restrict__ least,
                            int32_t *__restrict__ partner, int32_t *__restrict__ partner_count,
                            int32_t *__restrict__ least_out) {
  const int64_t m = R > C ? R : C;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    if (i < R) {
      const unsigned long long b = best[i];
      partner[i] = b ? (int32_t)(0xffffffffu - (uint32_t)(b & 0xffffffffull)) : -1;
      partner_count[i] = (int32_t)(b >> 32);
    }
    if (i < C) least_out[i] = inner[i] ? (int32_t)least[i] : 0;
  }
}
}  // namespace

// The labels (canonical for C) into the handle's label buffer, checked for range and for an empty cluster before
// anything else; then one pass of k_record_links over the held table.  The table and S do not change.
extern "C" int dbl_pairs_record_links(dbl_pairs *p, const int32_t *labels, int32_t num_clusters, int64_t *W_out,
                                      int64_t *I_out, int32_t *partner_out, int32_t *partner_count_out,
                                      int64_t *inner_out, int32_t *least_out) {
  if (!p || !labels || !W_out || !I_out || !partner_out || !partner_count_out || !inner_out || !least_out ||
      num_clusters < 1 || num_clusters > p->R)
    return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(labels, p->cluster, num_clusters); rc != DBL_OK) return rc;
  const int64_t R = p->R, C = num_clusters, H = p->H;
  cudaStream_t st = p->stream;
  const int32_t *L = p->cluster.as<int32_t>();
  int32_t *size = p->size.as<int32_t>();
  POST_TRY(cudaMemsetAsync(size, 0, sizeof(int32_t) * C, st));
  k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, L, size);
  k_flag_empty<<<grid_for(C), THREADS, 0, st>>>(C, size, p->bad.as<int>());  // bad is 0 after take_labels
  int flag = 0;
  POST_TRY(cudaMemcpyAsync(&flag, p->bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  if (flag) return DBL_ERR_INVALID;

  const size_t r8 = sizeof(unsigned long long) * (size_t)R, r4 = sizeof(int32_t) * (size_t)R;
  const size_t c8 = sizeof(unsigned long long) * (size_t)C, c4 = sizeof(int32_t) * (size_t)C;
  Buf W, I, best, inner, least, partner, pcount, lout;
  POST_TRY(W.alloc(r8));
  POST_TRY(I.alloc(r8));
  POST_TRY(best.alloc(r8));
  POST_TRY(inner.alloc(c8));
  POST_TRY(least.alloc(c4));
  POST_TRY(partner.alloc(r4));
  POST_TRY(pcount.alloc(r4));
  POST_TRY(lout.alloc(c4));
  POST_TRY(cudaMemsetAsync(W.p, 0, r8, st));
  POST_TRY(cudaMemsetAsync(I.p, 0, r8, st));
  POST_TRY(cudaMemsetAsync(best.p, 0, r8, st));
  POST_TRY(cudaMemsetAsync(inner.p, 0, c8, st));
  POST_TRY(cudaMemsetAsync(least.p, 0xff, c4, st));
  if (H > 0)
    k_record_links<<<grid_for(H), THREADS, 0, st>>>(H, p->tab_key[p->cur].as<unsigned long long>(),
                                                    p->tab_cnt[p->cur].as<int32_t>(), L,
                                                    W.as<unsigned long long>(), I.as<unsigned long long>(),
                                                    best.as<unsigned long long>(), inner.as<unsigned long long>(),
                                                    least.as<unsigned int>());
  k_links_out<<<grid_for(std::max(R, C)), THREADS, 0, st>>>(R, C, best.as<unsigned long long>(),
                                                          inner.as<unsigned long long>(), least.as<unsigned int>(),
                                                          partner.as<int32_t>(), pcount.as<int32_t>(),
                                                          lout.as<int32_t>());
  POST_TRY(cudaGetLastError());
  // host or device outputs: unified addressing picks the copy direction
  POST_TRY(cudaMemcpyAsync(W_out, W.p, r8, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(I_out, I.p, r8, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(partner_out, partner.p, r4, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(partner_count_out, pcount.p, r4, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(inner_out, inner.p, c8, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(least_out, lout.p, c4, cudaMemcpyDefault, st));
  POST_TRY(cudaStreamSynchronize(st));
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

namespace {
// out[0] = the sum over the clusters of a sample of |K|^2 (= sum over records of their cluster's size), out[1] = its
// records in clusters of two or more (the keys it gives a cell pass)
__global__ void k_sample_stats(int64_t R, const int32_t *__restrict__ lab, const int32_t *__restrict__ size,
                               unsigned long long *__restrict__ out) {
  unsigned long long q = 0, big = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int32_t k = size[lab[r]];
    q += (unsigned long long)k;
    big += k >= 2;
  }
  q = warp_sum_u64(q);
  big = warp_sum_u64(big);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], q);
    atomicAdd(&out[1], big);
  }
}

struct SampleStats {
  int64_t squares;  // sum over the sample's clusters of |K|^2: bounds its contributions to a round of the VI search
  int64_t keys;     // its records in clusters of two or more: its keys in a cell pass
};
}  // namespace

struct dbl_vi : Handle {
  int32_t max_samples = 0;
  int lab_bits = 1;                       // bits of a label in [0, R)
  int32_t max_size = 0;                   // M, the largest cluster of any held sample
  int64_t batch_keys = PAIR_BLOCK;        // keys of one batch of samples s (at least the selected records of one)
  Buf rows;                               // [max_samples][R] held labels
  Buf size, peak, sq;                     // cluster sizes of one sample; its largest (int32); its SampleStats
  std::vector<SampleStats> stats;         // per held sample
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
        p->peak.alloc(sizeof(int32_t)) != cudaSuccess || p->sq.alloc(2 * sizeof(unsigned long long)) != cudaSuccess)
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

// One sample: check the labels; its largest cluster, its sum of squared cluster sizes and its records in clusters of two
// or more; append it as row S.  S, M and the per-sample counts move only on success.
extern "C" int dbl_vi_add_sample(dbl_vi *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  int32_t *Z = p->size.as<int32_t>();
  POST_TRY(cudaMemsetAsync(Z, 0, sizeof(int32_t) * R, st));
  POST_TRY(cudaMemsetAsync(p->peak.p, 0, sizeof(int32_t), st));
  POST_TRY(cudaMemsetAsync(p->sq.p, 0, 2 * sizeof(unsigned long long), st));
  k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, p->cluster.as<int32_t>(), Z);
  k_max_size<<<grid_for(R), THREADS, 0, st>>>(R, Z, p->peak.as<int32_t>());
  k_sample_stats<<<grid_for(R), THREADS, 0, st>>>(R, p->cluster.as<int32_t>(), Z, p->sq.as<unsigned long long>());
  POST_TRY(cudaMemcpyAsync(p->rows.as<int32_t>() + (size_t)p->S * R, p->cluster.p, sizeof(int32_t) * R,
                           cudaMemcpyDeviceToDevice, st));
  int32_t m = 0;
  unsigned long long q[2] = {0, 0};
  POST_TRY(cudaMemcpyAsync(&m, p->peak.p, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaMemcpyAsync(q, p->sq.p, sizeof(q), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  try {
    p->stats.push_back({(int64_t)q[0], (int64_t)q[1]});
  } catch (const std::bad_alloc &) {
    return DBL_ERR_CUDA;  // nothing has moved
  }
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

// ---- the VI search and the expected VI of any labelling: cells of c ^ C_s over every held sample --------------------
namespace {
constexpr int64_t VI_MAX_SQUARES = int64_t(1) << 28;  // a sample's sum over clusters of |K|^2 the search accepts

// one key per selected record r of sample s0 + sl: sl << 2 lab_bits | label in C_s << lab_bits | label in c, with r
__global__ void k_vis_keys(int64_t nsel, const int32_t *__restrict__ sel, const int32_t *__restrict__ lab_s,
                           const int32_t *__restrict__ L, int32_t sl, int lab_bits, unsigned long long *__restrict__ key,
                           int32_t *__restrict__ rec) {
  const unsigned long long hi = (unsigned long long)sl << (2 * lab_bits);
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < nsel; k += (int64_t)gridDim.x * blockDim.x) {
    const int32_t r = sel[k];
    key[k] = hi | (unsigned long long)(uint32_t)lab_s[r] << lab_bits | (uint32_t)L[r];
    rec[k] = r;
  }
}

__global__ void k_cell_heads(int64_t n, const unsigned long long *__restrict__ key, int32_t *__restrict__ head) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    head[i] = i == 0 || key[i] != key[i - 1];
}

// cell c (0-based, in sorted order) starts at cpos[c]; cpos[number of cells] = n
__global__ void k_cell_pos(int64_t n, const int32_t *__restrict__ head, const int32_t *__restrict__ crank,
                           int32_t *__restrict__ cpos) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (head[i]) cpos[crank[i] - 1] = (int32_t)i;
    if (i == n - 1) cpos[crank[i]] = (int32_t)n;
  }
}

// cells of n >= 2 records counted into G[n] (n < width, as every cell is inside a cluster of at most M records)
__global__ void k_cell_hist(int64_t ncell, const int32_t *__restrict__ cpos, unsigned long long *__restrict__ G) {
  for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < ncell; c += (int64_t)gridDim.x * blockDim.x) {
    const int32_t m = cpos[c + 1] - cpos[c];
    if (m >= 2) atomicAdd(&G[m], 1ull);
  }
}

// Per sample: each cell of n >= 2 records counted into G[s][n], s = s0 + (its first key >> hi_shift).  Cells are in key
// order, sample then cluster, so a warp's cells mostly share a row and a small n; lanes with equal (s, n) are summed by
// __match_any_sync and add once.
__global__ void k_cell_rows(int64_t ncell, int hi_shift, const unsigned long long *__restrict__ key,
                            const int32_t *__restrict__ cpos, int32_t s0, int64_t width,
                            unsigned long long *__restrict__ G) {
  const int lane = threadIdx.x & 31;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < ncell;
       base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t c = base + lane;
    int32_t m = 0;
    int64_t s = 0;
    if (c < ncell) {
      const int32_t first = cpos[c];
      m = cpos[c + 1] - first;
      s = s0 + (int64_t)(key[first] >> hi_shift);
    }
    const unsigned emit = __ballot_sync(0xffffffffu, m >= 2);
    if (m >= 2) {
      const unsigned same = __match_any_sync(emit, (unsigned long long)s << 32 | (unsigned long long)(uint32_t)m);
      if (lane == __ffs(same) - 1) atomicAdd(&G[s * width + m], (unsigned long long)__popc(same));
    }
  }
}

// sum over cells of F_q(n) into *out
__global__ void k_cell_F(int64_t ncell, const int32_t *__restrict__ cpos, const long long *__restrict__ F,
                         unsigned long long *__restrict__ out) {
  unsigned long long acc = 0;
  for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < ncell; c += (int64_t)gridDim.x * blockDim.x)
    acc += (unsigned long long)F[cpos[c + 1] - cpos[c]];
  acc = warp_sum_u64(acc);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, acc);
}

// sum over clusters of F_q(|X|), and the number of clusters: out[0], out[1]
__global__ void k_size_stats(int64_t R, const int32_t *__restrict__ size, const long long *__restrict__ F,
                             unsigned long long *__restrict__ out) {
  unsigned long long f = 0, k = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    f += (unsigned long long)F[size[r]];
    k += size[r] > 0;
  }
  f = warp_sum_u64(f);
  k = warp_sum_u64(k);
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], f);
    atomicAdd(&out[1], k);
  }
}

// the cells of the sample cluster K holding sorted position i: [first cell, its number of cells)
__device__ __forceinline__ void cluster_cells(const unsigned long long *__restrict__ key, int64_t n, int lab_bits,
                                              const int32_t *__restrict__ crank, int64_t i, int32_t *first,
                                              int32_t *count) {
  const unsigned long long K = key[i] >> lab_bits;
  const int64_t lo = lower_bound_u64(key, n, K << lab_bits), hi = lower_bound_u64(key, n, (K + 1) << lab_bits);
  *first = crank[lo] - 1;
  *count = crank[hi - 1] - crank[lo] + 1;
}

// per sorted position, the number of cells of its sample cluster (its contributions); entry n is 0
__global__ void k_vis_count(int64_t n, int lab_bits, const unsigned long long *__restrict__ key,
                            const int32_t *__restrict__ crank, long long *__restrict__ cnt) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t first = 0, count = 0;
    if (i < n) cluster_cells(key, n, lab_bits, crank, i, &first, &count);
    cnt[i] = count;
  }
}

// One warp per sorted position (record i, in sample cluster K) writes, at its int64 offset, one contribution per cell
// (K, B) of m records: key i << lab_bits | B, value D_q[m] for B != c(i), D_q[m - 1] for i's own cell.
__global__ void k_vis_emit(int64_t n, int lab_bits, const unsigned long long *__restrict__ key,
                           const int32_t *__restrict__ rec, const int32_t *__restrict__ crank,
                           const int32_t *__restrict__ cpos, const long long *__restrict__ off,
                           const int32_t *__restrict__ L, const long long *__restrict__ Dq,
                           unsigned long long *__restrict__ ckey, long long *__restrict__ cval) {
  const int lane = threadIdx.x & 31;
  const unsigned long long mask = (1ull << lab_bits) - 1;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t w = blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5); w < n; w += nwarps) {
    int32_t first = 0, count = 0;
    cluster_cells(key, n, lab_bits, crank, w, &first, &count);
    const int32_t i = rec[w];
    const unsigned long long A = (uint32_t)L[i], hi = (unsigned long long)(uint32_t)i << lab_bits;
    const long long o = off[w];
    for (int32_t j = lane; j < count; j += 32) {
      const int32_t s = cpos[first + j], m = cpos[first + j + 1] - s;
      const unsigned long long B = key[s] & mask;
      ckey[o + j] = hi | B;
      cval[o + j] = Dq[B == A ? m - 1 : m];
    }
  }
}

// One record per thread over its segment of the reduced (record << lab_bits | cluster, w) table: w_A of its own
// cluster A, then per cluster B (ascending) dJ = S (D_q[|B|] - D_q[a - 1]) - 2 (w_B - w_A); the singleton (a > 1) is
// dJ = -S D_q[a - 1] + 2 w_A and is tried first as destination -1, so a strict < keeps the least (dJ, destination).
// A record with dJ < 0 proposes its move and claims its source and destination with atomicMin on dJ.
__global__ void k_vis_best_move(int64_t R, int lab_bits, int64_t n, const unsigned long long *__restrict__ key,
                                const long long *__restrict__ w, const int32_t *__restrict__ lab,
                                const int32_t *__restrict__ size, const long long *__restrict__ Dq, long long S,
                                long long *__restrict__ prop_dJ, int32_t *__restrict__ prop_dest,
                                long long *__restrict__ claim_dJ, unsigned long long *__restrict__ num_props) {
  const unsigned long long mask = (1ull << lab_bits) - 1;
  unsigned long long props = 0;
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x) {
    const int64_t lo = lower_bound_u64(key, n, (unsigned long long)r << lab_bits);
    const int64_t hi = lower_bound_u64(key, n, (unsigned long long)(r + 1) << lab_bits);
    const int32_t A = lab[r];
    const long long a = size[A], dA = Dq[a - 1];
    long long wA = 0;
    for (int64_t k = lo; k < hi; ++k)
      if ((key[k] & mask) == (unsigned long long)A) wA = w[k];
    long long best = NO_MOVE;
    int32_t dest = INT_MAX;
    if (a > 1) {
      best = -S * dA + 2 * wA;
      dest = -1;
    }
    for (int64_t k = lo; k < hi; ++k) {
      const unsigned long long X = key[k] & mask;
      if (X == (unsigned long long)A) continue;
      const long long dJ = S * (Dq[size[X]] - dA) - 2 * (w[k] - wA);
      if (dJ < best) {
        best = dJ;
        dest = (int32_t)X;
      }
    }
    const bool propose = best < 0;
    prop_dJ[r] = propose ? best : NO_MOVE;
    prop_dest[r] = dest;
    if (propose) {
      atomicMin(&claim_dJ[A], best);
      if (dest >= 0) atomicMin(&claim_dJ[dest], best);
      ++props;
    }
  }
  props = warp_sum_u64(props);
  if ((threadIdx.x & 31) == 0 && props) atomicAdd(num_props, props);
}

// The cells of a labelling L (int32 [R], device, labels in [0, R)) with every held sample, batch by batch.  Each sample
// has a weight, its keys (the score) or its sum of |K|^2 (the search, which bounds its contributions); a batch takes
// samples while their weights stay within max(batch_keys, that of its first sample), their keys within INT32_MAX and
// its key bits within 63.  Per sample the records in its clusters of two or more (flags, an exclusive scan, a scatter)
// give one key each (k_vis_keys), so the key buffers hold the batch's keys and no more; the batch's (key, record) pairs
// are radix-sorted, and the cells are their runs of equal keys: cell ranks (an inclusive scan of the heads) and cell
// starts.  on_batch(s0, n, ncell) sees the batch's first sample s0, the sorted keys in key.Current(), their records in
// rec.Current(), the ranks in crank and the starts in cpos.
struct CellPass {
  Buf key[2], rec[2], head, crank, cpos, flag, pos, sel, tmp;
  cub::DoubleBuffer<unsigned long long> kb;
  cub::DoubleBuffer<int32_t> rb;
};

template <class OnBatch>
int vi_cell_batches(dbl_vi *p, const int32_t *L, int64_t SampleStats::*weight, CellPass &c, OnBatch on_batch) {
  const int64_t R = p->R;
  const int32_t S = p->S;
  const int b = p->lab_bits;
  cudaStream_t st = p->stream;
  const int32_t *rows = p->rows.as<int32_t>();
  int32_t *Z = p->size.as<int32_t>();
  POST_TRY(c.flag.reserve(sizeof(int32_t) * (size_t)(R + 1)));
  POST_TRY(c.pos.reserve(sizeof(int32_t) * (size_t)(R + 1)));
  POST_TRY(c.sel.reserve(sizeof(int32_t) * (size_t)R));
  size_t tb_scan = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb_scan, (const int32_t *)nullptr, (int32_t *)nullptr, R + 1, st));
  for (int32_t s0 = 0; s0 < S;) {
    const std::vector<SampleStats> &ss = p->stats;
    const int64_t limit = std::max(p->batch_keys, ss[s0].*weight);
    int32_t s1 = s0 + 1;
    int64_t w = ss[s0].*weight, keys = ss[s0].keys;  // keys <= R <= INT32_MAX
    while (s1 < S && w + ss[s1].*weight <= limit && keys + ss[s1].keys <= INT32_MAX &&
           2 * b + bits_for((int64_t)s1 - s0 + 1) <= 63) {
      w += ss[s1].*weight;
      keys += ss[s1++].keys;
    }
    const int32_t B = s1 - s0;
    POST_TRY(c.key[0].reserve(sizeof(unsigned long long) * (size_t)keys));
    POST_TRY(c.key[1].reserve(sizeof(unsigned long long) * (size_t)keys));
    POST_TRY(c.rec[0].reserve(sizeof(int32_t) * (size_t)keys));
    POST_TRY(c.rec[1].reserve(sizeof(int32_t) * (size_t)keys));
    c.kb = cub::DoubleBuffer<unsigned long long>(c.key[0].as<unsigned long long>(), c.key[1].as<unsigned long long>());
    c.rb = cub::DoubleBuffer<int32_t>(c.rec[0].as<int32_t>(), c.rec[1].as<int32_t>());
    int64_t n = 0;
    for (int32_t s = s0; s < s1; ++s) {
      const int32_t *lab_s = rows + (size_t)s * R;
      POST_TRY(cudaMemsetAsync(Z, 0, sizeof(int32_t) * R, st));
      k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, lab_s, Z);
      k_flag_big<<<grid_for(R + 1), THREADS, 0, st>>>(R, lab_s, Z, c.flag.as<int32_t>());
      POST_TRY(c.tmp.reserve(tb_scan));
      size_t tb = c.tmp.cap;
      POST_TRY(cub::DeviceScan::ExclusiveSum(c.tmp.p, tb, c.flag.as<int32_t>(), c.pos.as<int32_t>(), R + 1, st));
      k_scatter_flagged<<<grid_for(R), THREADS, 0, st>>>(R, c.flag.as<int32_t>(), c.pos.as<int32_t>(),
                                                         c.sel.as<int32_t>());
      const int64_t nsel = ss[s].keys;  // what the scan selects, counted when the sample was added
      if (nsel > 0)
        k_vis_keys<<<grid_for(nsel), THREADS, 0, st>>>(nsel, c.sel.as<int32_t>(), lab_s, L, s - s0, b,
                                                       c.kb.Current() + n, c.rb.Current() + n);
      n += nsel;
    }
    POST_TRY(cudaGetLastError());
    const int32_t first = s0;
    s0 = s1;
    if (n == 0) continue;  // every sample of the batch is all singletons: every cell with them is a singleton
    const int end_bit = 2 * b + bits_for(B);
    POST_TRY(c.head.reserve(sizeof(int32_t) * (size_t)n));
    POST_TRY(c.crank.reserve(sizeof(int32_t) * (size_t)n));
    POST_TRY(c.cpos.reserve(sizeof(int32_t) * (size_t)(n + 1)));
    size_t tbs = 0, tbc = 0;
    POST_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tbs, c.kb, c.rb, n, 0, end_bit, st));
    POST_TRY(cub::DeviceScan::InclusiveSum(nullptr, tbc, (const int32_t *)nullptr, (int32_t *)nullptr, n, st));
    POST_TRY(c.tmp.reserve(std::max(tbs, tbc)));
    tbs = c.tmp.cap;
    POST_TRY(cub::DeviceRadixSort::SortPairs(c.tmp.p, tbs, c.kb, c.rb, n, 0, end_bit, st));
    k_cell_heads<<<grid_for(n), THREADS, 0, st>>>(n, c.kb.Current(), c.head.as<int32_t>());
    tbc = c.tmp.cap;
    POST_TRY(cub::DeviceScan::InclusiveSum(c.tmp.p, tbc, c.head.as<int32_t>(), c.crank.as<int32_t>(), n, st));
    k_cell_pos<<<grid_for(n), THREADS, 0, st>>>(n, c.head.as<int32_t>(), c.crank.as<int32_t>(), c.cpos.as<int32_t>());
    int32_t ncell = 0;
    POST_TRY(cudaMemcpyAsync(&ncell, c.crank.as<int32_t>() + n - 1, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    if (const int rc = on_batch(first, n, (int64_t)ncell); rc != DBL_OK) return rc;
  }
  return DBL_OK;
}
}  // namespace

// G[n] = the cells of n >= 2 records of labels ^ C_s summed over the held samples s, from the cell pass of the search.
extern "C" int dbl_vi_score(dbl_vi *p, const int32_t *labels, int64_t width, int64_t *G_out) {
  if (!p || !labels || !G_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  if (width < (int64_t)p->max_size + 1 || width > INT64_MAX / 8) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(labels, p->cluster); rc != DBL_OK) return rc;
  cudaStream_t st = p->stream;
  const size_t gbytes = sizeof(unsigned long long) * (size_t)width;
  Buf G;
  CellPass c;
  POST_TRY(G.alloc(gbytes));
  POST_TRY(cudaMemsetAsync(G.p, 0, gbytes, st));
  const int rc = vi_cell_batches(p, p->cluster.as<int32_t>(), &SampleStats::keys, c, [&](int32_t, int64_t, int64_t ncell) {
    k_cell_hist<<<grid_for(ncell), THREADS, 0, st>>>(ncell, c.cpos.as<int32_t>(), G.as<unsigned long long>());
    return DBL_OK;
  });
  if (rc != DBL_OK) return rc;
  POST_TRY(cudaMemcpyAsync(G_out, G.p, gbytes, cudaMemcpyDefault, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// G[s][n] = the cells of n >= 2 records of labels ^ C_s, one row per held sample: the score's cell pass, each batch's
// cells counted into the rows of their samples (k_cell_rows).
extern "C" int dbl_vi_score_samples(dbl_vi *p, const int32_t *labels, int64_t width, int64_t *G_out) {
  if (!p || !labels || !G_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  if (width < (int64_t)p->max_size + 1 || width > INT64_MAX / 8 / p->S) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(labels, p->cluster); rc != DBL_OK) return rc;
  cudaStream_t st = p->stream;
  const int hi_shift = 2 * p->lab_bits;
  const size_t gbytes = sizeof(unsigned long long) * (size_t)p->S * (size_t)width;
  Buf G;
  CellPass c;
  POST_TRY(G.alloc(gbytes));
  POST_TRY(cudaMemsetAsync(G.p, 0, gbytes, st));
  const int rc = vi_cell_batches(p, p->cluster.as<int32_t>(), &SampleStats::keys, c,
                                 [&](int32_t s0, int64_t, int64_t ncell) {
                                   k_cell_rows<<<grid_for(ncell), THREADS, 0, st>>>(
                                       ncell, hi_shift, c.kb.Current(), c.cpos.as<int32_t>(), s0, width,
                                       G.as<unsigned long long>());
                                   return DBL_OK;
                                 });
  if (rc != DBL_OK) return rc;
  POST_TRY(cudaMemcpyAsync(G_out, G.p, gbytes, cudaMemcpyDefault, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// The search: check the table and the bounds; take and canonically group the start; then rounds of sizes, the cell
// pass with every sample's contributions (k_vis_count, an int64 scan, k_vis_emit), each batch's contributions sorted
// with the running table and reduced by key into it, best moves, the two-stage claims, the moves and the canonical
// relabel of the Binder search, until no record proposes or max_rounds rounds are done.  The first round's cell pass
// also sums F_q over the cells, which with the sizes gives J_q of the start.  Every buffer is the call's own.
extern "C" int dbl_vi_search(dbl_vi *p, const int64_t *step, const int32_t *start, int32_t max_rounds,
                             int32_t *labels_out, int32_t *rounds_out, int32_t *converged_out, int64_t *moves,
                             int64_t *clusters, int64_t *dJ, int64_t *J0_out) {
  if (!p || !step || !start || !labels_out || !rounds_out || !converged_out || !moves || !clusters || !dJ || !J0_out ||
      max_rounds < 1)
    return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  const int64_t R = p->R;
  const int32_t S = p->S;
  if (step[0] != 0) return DBL_ERR_INVALID;
  for (int64_t m = 1; m < R; ++m)
    if (step[m] < step[m - 1]) return DBL_ERR_INVALID;
  // every J_q, dJ and round sum is within 4 S R D_q[R - 1] in magnitude
  if ((unsigned __int128)S * (unsigned __int128)R * (unsigned __int128)step[R - 1] >= ((unsigned __int128)1 << 61))
    return DBL_ERR_INVALID;
  for (int32_t s = 0; s < S; ++s)
    if (p->stats[s].squares > VI_MAX_SQUARES) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(start, p->cluster); rc != DBL_OK) return rc;
  const int b = p->lab_bits, gbits = bits_for(2 * R);
  cudaStream_t st = p->stream;

  const size_t r4 = sizeof(int32_t) * (size_t)R, r8 = sizeof(long long) * (size_t)R;
  Buf Dq, F, iota, lab, size, gkey, gkey_s, rec_s, head, start_b, prop_dJ, prop_dest, claim_dJ, claim_i, stats;
  Buf cnt, off, ck[2], cv[2], nruns;
  CellPass c;
  POST_TRY(Dq.alloc(r8));
  POST_TRY(F.alloc(sizeof(long long) * (size_t)(R + 1)));
  POST_TRY(iota.alloc(r4));
  POST_TRY(lab.alloc(r4));
  POST_TRY(size.alloc(r4));
  POST_TRY(gkey.alloc(r8));
  POST_TRY(gkey_s.alloc(r8));
  POST_TRY(rec_s.alloc(r4));
  POST_TRY(head.alloc(r4));
  POST_TRY(start_b.alloc(r4));
  POST_TRY(prop_dJ.alloc(r8));
  POST_TRY(prop_dest.alloc(r4));
  POST_TRY(claim_dJ.alloc(r8));
  POST_TRY(claim_i.alloc(r4));
  POST_TRY(stats.alloc(8 * sizeof(unsigned long long)));
  POST_TRY(nruns.alloc(sizeof(long long)));
  {
    // F_q(n) = sum over m < n of D_q[m], exact in int64 by the bound above
    std::vector<long long> f;
    try {
      f.resize((size_t)R + 1);
    } catch (const std::bad_alloc &) {
      return DBL_ERR_CUDA;
    }
    f[0] = 0;
    for (int64_t m = 0; m < R; ++m) f[m + 1] = f[m] + step[m];
    POST_TRY(cudaMemcpyAsync(Dq.p, step, r8, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(F.p, f.data(), sizeof(long long) * (size_t)(R + 1), cudaMemcpyHostToDevice, st));
    POST_TRY(cudaStreamSynchronize(st));
  }
  unsigned long long *st8 = stats.as<unsigned long long>();
  int32_t *L = lab.as<int32_t>(), *Z = size.as<int32_t>();
  const long long *dq = Dq.as<long long>();
  k_iota<<<grid_for(R), THREADS, 0, st>>>(R, iota.as<int32_t>());
  auto relabel = [&]() {
    return canonical_relabel(R, gbits, gkey.as<unsigned long long>(), iota.as<int32_t>(),
                             gkey_s.as<unsigned long long>(), rec_s.as<int32_t>(), head.as<int32_t>(),
                             start_b.as<int32_t>(), L, c.tmp, st);
  };
  // sizes of L, then sum of F_q over its clusters and its number of clusters into st8[4], st8[5]
  auto sizes = [&]() {
    POST_TRY(cudaMemsetAsync(Z, 0, r4, st));
    POST_TRY(cudaMemsetAsync(st8 + 4, 0, 2 * sizeof(unsigned long long), st));
    k_label_sizes<<<grid_for(R), THREADS, 0, st>>>(R, L, Z);
    k_size_stats<<<grid_for(R), THREADS, 0, st>>>(R, Z, F.as<long long>(), st8 + 4);
    return DBL_OK;
  };
  k_widen_labels<<<grid_for(R), THREADS, 0, st>>>(R, p->cluster.as<int32_t>(), gkey.as<unsigned long long>());
  if (const int rc = relabel(); rc != DBL_OK) return rc;
  if (const int rc = sizes(); rc != DBL_OK) return rc;
  POST_TRY(cudaMemsetAsync(st8 + 6, 0, sizeof(unsigned long long), st));  // sum of F_q over the start's cells

  int32_t rounds = 0, converged = 0;
  long long J0 = 0;
  for (;;) {
    // every sample's contributions, reduced into (record << b | cluster, w) in ck/cv[cur], acc_n entries
    int cur = 0;
    int64_t acc_n = 0;
    const bool first_round = rounds == 0;
    const int rc = vi_cell_batches(p, L, &SampleStats::squares, c, [&](int32_t, int64_t n, int64_t ncell) {
      if (first_round)
        k_cell_F<<<grid_for(ncell), THREADS, 0, st>>>(ncell, c.cpos.as<int32_t>(), F.as<long long>(), st8 + 6);
      POST_TRY(cnt.reserve(sizeof(long long) * (size_t)(n + 1)));
      POST_TRY(off.reserve(sizeof(long long) * (size_t)(n + 1)));
      k_vis_count<<<grid_for(n + 1), THREADS, 0, st>>>(n, b, c.kb.Current(), c.crank.as<int32_t>(),
                                                        cnt.as<long long>());
      size_t tb = 0;
      POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt.as<long long>(), off.as<long long>(), n + 1, st));
      POST_TRY(c.tmp.reserve(tb));
      tb = c.tmp.cap;
      POST_TRY(cub::DeviceScan::ExclusiveSum(c.tmp.p, tb, cnt.as<long long>(), off.as<long long>(), n + 1, st));
      long long nc = 0;
      POST_TRY(cudaMemcpyAsync(&nc, off.as<long long>() + n, sizeof(long long), cudaMemcpyDeviceToHost, st));
      POST_TRY(cudaStreamSynchronize(st));
      const int64_t total = acc_n + nc;
      // both sides hold the running table and the batch's contributions; side cur keeps its running table
      const size_t need = sizeof(long long) * (size_t)total, keep = sizeof(long long) * (size_t)acc_n;
      POST_TRY(ck[cur].reserve_keep(need, keep, st));
      POST_TRY(cv[cur].reserve_keep(need, keep, st));
      POST_TRY(ck[cur ^ 1].reserve(need));
      POST_TRY(cv[cur ^ 1].reserve(need));
      k_vis_emit<<<(int)std::min<int64_t>((n + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 8192), THREADS, 0, st>>>(
          n, b, c.kb.Current(), c.rb.Current(), c.crank.as<int32_t>(), c.cpos.as<int32_t>(), off.as<long long>(), L,
          dq, ck[cur].as<unsigned long long>() + acc_n, cv[cur].as<long long>() + acc_n);
      // the running table and the batch's contributions, sorted and reduced by key into the other side
      cub::DoubleBuffer<unsigned long long> kk(ck[cur].as<unsigned long long>(), ck[cur ^ 1].as<unsigned long long>());
      cub::DoubleBuffer<long long> vv(cv[cur].as<long long>(), cv[cur ^ 1].as<long long>());
      size_t tbs = 0, tbr = 0;
      POST_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tbs, kk, vv, total, 0, 2 * b, st));
      POST_TRY(c.tmp.reserve(tbs));
      tbs = c.tmp.cap;
      POST_TRY(cub::DeviceRadixSort::SortPairs(c.tmp.p, tbs, kk, vv, total, 0, 2 * b, st));
      const int sorted = kk.Current() == ck[cur].as<unsigned long long>() ? cur : cur ^ 1;
      const int other = sorted ^ 1;
      POST_TRY(cub::DeviceReduce::ReduceByKey(nullptr, tbr, ck[sorted].as<unsigned long long>(),
                                              ck[other].as<unsigned long long>(), cv[sorted].as<long long>(),
                                              cv[other].as<long long>(), nruns.as<long long>(), cub::Sum(), total,
                                              st));
      POST_TRY(c.tmp.reserve(tbr));
      tbr = c.tmp.cap;
      POST_TRY(cub::DeviceReduce::ReduceByKey(c.tmp.p, tbr, ck[sorted].as<unsigned long long>(),
                                              ck[other].as<unsigned long long>(), cv[sorted].as<long long>(),
                                              cv[other].as<long long>(), nruns.as<long long>(), cub::Sum(), total,
                                              st));
      long long runs = 0;
      POST_TRY(cudaMemcpyAsync(&runs, nruns.p, sizeof(long long), cudaMemcpyDeviceToHost, st));
      POST_TRY(cudaGetLastError());
      POST_TRY(cudaStreamSynchronize(st));
      cur = other;
      acc_n = runs;
      return DBL_OK;
    });
    if (rc != DBL_OK) return rc;
    if (first_round) {
      unsigned long long f[3];
      POST_TRY(cudaMemcpyAsync(f, st8 + 4, sizeof(f), cudaMemcpyDeviceToHost, st));
      POST_TRY(cudaStreamSynchronize(st));
      J0 = (long long)S * (long long)f[0] - 2 * (long long)f[2];
    }
    POST_TRY(cudaMemsetAsync(claim_dJ.p, 0x7f, r8, st));  // above every dJ < 0
    POST_TRY(cudaMemsetAsync(claim_i.p, 0xff, r4, st));   // above every record index
    POST_TRY(cudaMemsetAsync(st8, 0, 4 * sizeof(unsigned long long), st));
    k_vis_best_move<<<grid_for(R), THREADS, 0, st>>>(R, b, acc_n, ck[cur].as<unsigned long long>(),
                                                     cv[cur].as<long long>(), L, Z, dq, S, prop_dJ.as<long long>(),
                                                     prop_dest.as<int32_t>(), claim_dJ.as<long long>(), st8 + 3);
    k_claim_record<<<grid_for(R), THREADS, 0, st>>>(R, L, prop_dJ.as<long long>(), prop_dest.as<int32_t>(),
                                                    claim_dJ.as<long long>(), claim_i.as<unsigned int>());
    unsigned long long props = 0;
    POST_TRY(cudaMemcpyAsync(&props, st8 + 3, sizeof(props), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    if (props == 0) {
      converged = 1;
      break;
    }
    if (rounds == max_rounds) break;
    k_apply_moves<<<grid_for(R), THREADS, 0, st>>>(R, L, Z, prop_dJ.as<long long>(), prop_dest.as<int32_t>(),
                                                   prop_dJ.as<long long>(), claim_dJ.as<long long>(),
                                                   claim_i.as<unsigned int>(), gkey.as<unsigned long long>(), st8);
    if (const int rc2 = relabel(); rc2 != DBL_OK) return rc2;
    if (const int rc2 = sizes(); rc2 != DBL_OK) return rc2;
    unsigned long long log[6];
    POST_TRY(cudaMemcpyAsync(log, st8, sizeof(log), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    moves[rounds] = (int64_t)log[0];
    dJ[rounds] = (int64_t)log[2];
    clusters[rounds] = (int64_t)log[5];
    ++rounds;
  }
  POST_TRY(cudaMemcpyAsync(labels_out, L, r4, cudaMemcpyDefault, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  *rounds_out = rounds;
  *converged_out = converged;
  *J0_out = (int64_t)J0;
  return DBL_OK;
}

// ---- entity values per cluster of a point estimate -----------------------------------------------------------------
namespace {
// one key per record: its cluster label above the value of the entity it links to in this sample
__global__ void k_value_keys(int64_t R, int val_bits, const int32_t *__restrict__ label,
                             const int32_t *__restrict__ value, unsigned long long *__restrict__ key) {
  for (int64_t r = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; r < R; r += (int64_t)gridDim.x * blockDim.x)
    key[r] = (unsigned long long)(uint32_t)label[r] << val_bits | (uint32_t)value[r];
}

// Segmented arg-max over the held table, pass 1: best[c] = the largest count of label c.  The table is sorted by key,
// so the entries of a label are contiguous and a warp's lanes hold runs of equal labels: a segmented shuffle reduction
// leaves each run's largest count at its first lane, which adds one atomic.  A label of many entries costs one atomic
// per warp it spans.
__global__ void k_mode_count(int64_t H, int val_bits, const unsigned long long *__restrict__ key,
                             const long long *__restrict__ cnt, unsigned long long *__restrict__ best) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t base = (blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5)) * 32; base < H; base += nwarps * 32) {
    const int64_t i = base + lane;
    const bool valid = i < H;
    const long long lab = valid ? (long long)(key[i] >> val_bits) : -1 - lane;  // a tail lane matches no one
    long long c = valid ? cnt[i] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const long long ol = __shfl_down_sync(0xffffffffu, lab, o), oc = __shfl_down_sync(0xffffffffu, c, o);
      if (lane + o < 32 && ol == lab && oc > c) c = oc;
    }
    const long long prev = __shfl_up_sync(0xffffffffu, lab, 1);
    if (valid && (lane == 0 || prev != lab)) atomicMax(&best[lab], (unsigned long long)c);
  }
}

// pass 2: first[c] = the first table position of label c whose count is best[c], i.e. its smallest such value; the
// lanes of a warp with equal labels and the best count elect their lowest lane, which adds one atomic
__global__ void k_mode_first(int64_t H, int val_bits, const unsigned long long *__restrict__ key,
                             const long long *__restrict__ cnt, const unsigned long long *__restrict__ best,
                             unsigned long long *__restrict__ first) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t base = (blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5)) * 32; base < H; base += nwarps * 32) {
    const int64_t i = base + lane;
    const unsigned long long lab = i < H ? key[i] >> val_bits : 0ull;
    const bool hit = i < H && (unsigned long long)cnt[i] == best[lab];
    const unsigned peers = __match_any_sync(0xffffffffu, hit ? lab : ~0ull);
    if (hit && lane == __ffs(peers) - 1) atomicMin(&first[lab], (unsigned long long)i);
  }
}

// per label its mode (the value of its first best position, -1 when the label has no record) and the mode's count
__global__ void k_mode_out(int64_t C, unsigned long long mask, const unsigned long long *__restrict__ key,
                           const unsigned long long *__restrict__ best, const unsigned long long *__restrict__ first,
                           int32_t *__restrict__ mode, long long *__restrict__ count) {
  for (int64_t c = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; c < C; c += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long f = first[c];
    mode[c] = f == ~0ull ? -1 : (int32_t)(key[f] & mask);
    count[c] = (long long)best[c];
  }
}
}  // namespace

struct dbl_values : Handle {
  int32_t C = 0, V = 0;
  int val_bits = 1, key_bits = 2;       // bits of a value in [0, V); radix sort end bit of the keys
  int64_t H = 0;                        // distinct (label, value) keys held
  Buf labels;                           // R labels in [0, C); Handle::cluster receives each sample's values
  Buf key_in, key_s, uniq;              // R keys each: unsorted, sorted, distinct
  Buf runs, nruns;                      // R int32 run lengths of the distinct keys; their number
  Buf is_new, rank;                     // R + 1 each: merge flags and ranks
  Buf tab_key[2], tab_cnt[2];           // grown on demand: held table (index cur), the one the next sample merges into
  int cur = 0;
  Buf tmp;                              // CUB temporary storage, grown on demand
};

extern "C" int dbl_values_create(dbl_values **out, int64_t num_records, const int32_t *labels, int32_t num_clusters,
                                 int32_t num_values) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || !labels || num_clusters <= 0 || num_values <= 0)
    return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_values *p) {
    const int64_t R = num_records;
    p->C = num_clusters;
    p->V = num_values;
    p->val_bits = bits_for(num_values);
    p->key_bits = bits_for(num_clusters) + p->val_bits;
    const size_t r4 = sizeof(int32_t) * (size_t)R, r8 = sizeof(unsigned long long) * (size_t)R;
    if (p->labels.alloc(r4) != cudaSuccess || p->key_in.alloc(r8) != cudaSuccess || p->key_s.alloc(r8) != cudaSuccess ||
        p->uniq.alloc(r8) != cudaSuccess || p->runs.alloc(r4) != cudaSuccess ||
        p->nruns.alloc(sizeof(int64_t)) != cudaSuccess || p->is_new.alloc(r4 + sizeof(int32_t)) != cudaSuccess ||
        p->rank.alloc(r4 + sizeof(int32_t)) != cudaSuccess)
      return DBL_ERR_CUDA;
    return p->take_labels(labels, p->labels, num_clusters);
  });
}

extern "C" void dbl_values_free(dbl_values *p) { free_handle(p); }

extern "C" int32_t dbl_values_num_samples(const dbl_values *p) { return p ? p->S : 0; }

// One sample: check the values; key (label << val_bits | value) per record; radix-sort on key_bits bits; run-length
// encode into (distinct key, records); merge those into the spare table with their run lengths as counts, then commit
// by swapping tables.  A refusal or failure leaves the held table and S as they were.
extern "C" int dbl_values_add_sample(dbl_values *p, const int32_t *values) {
  if (!p || !values || p->S == INT32_MAX) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(values, p->cluster, p->V); rc != DBL_OK) return rc;
  const int64_t R = p->R, H = p->H;
  cudaStream_t st = p->stream;
  k_value_keys<<<grid_for(R), THREADS, 0, st>>>(R, p->val_bits, p->labels.as<int32_t>(), p->cluster.as<int32_t>(),
                                                p->key_in.as<unsigned long long>());
  size_t tb_sort = 0, tb_rle = 0;
  unsigned long long *ks = p->key_s.as<unsigned long long>(), *uniq = p->uniq.as<unsigned long long>();
  POST_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tb_sort, p->key_in.as<unsigned long long>(), ks, R, 0, p->key_bits,
                                          st));
  POST_TRY(cub::DeviceRunLengthEncode::Encode(nullptr, tb_rle, ks, uniq, p->runs.as<int32_t>(),
                                              p->nruns.as<int64_t>(), R, st));
  POST_TRY(p->tmp.reserve(std::max(tb_sort, tb_rle)));
  size_t tb = p->tmp.cap;
  POST_TRY(cub::DeviceRadixSort::SortKeys(p->tmp.p, tb, p->key_in.as<unsigned long long>(), ks, R, 0, p->key_bits,
                                          st));
  tb = p->tmp.cap;
  POST_TRY(cub::DeviceRunLengthEncode::Encode(p->tmp.p, tb, ks, uniq, p->runs.as<int32_t>(), p->nruns.as<int64_t>(),
                                              R, st));
  int64_t n = 0;
  POST_TRY(cudaMemcpyAsync(&n, p->nruns.p, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));

  const unsigned long long *held = p->tab_key[p->cur].as<unsigned long long>();
  const long long *hcnt = p->tab_cnt[p->cur].as<long long>();
  int64_t fresh = 0;
  if (const int rc = probe_new_keys(n, uniq, H, held, p->is_new, p->rank, p->tmp, st, &fresh); rc != DBL_OK) return rc;
  const int64_t H2 = H + fresh;
  const int nxt = p->cur ^ 1;
  POST_TRY(p->tab_key[nxt].reserve(sizeof(unsigned long long) * (size_t)H2));
  POST_TRY(p->tab_cnt[nxt].reserve(sizeof(long long) * (size_t)H2));
  if (const int rc = merge_keys<long long>(H, held, hcnt, n, uniq, p->runs.as<int32_t>(), p->is_new, p->rank,
                                           p->tab_key[nxt].as<unsigned long long>(), p->tab_cnt[nxt].as<long long>(),
                                           st);
      rc != DBL_OK)
    return rc;
  p->cur = nxt;
  p->H = H2;
  ++p->S;
  return DBL_OK;
}

// Per label the value of largest count, ties to the smallest value: k_mode_count, then k_mode_first, over the held
// table; a label without records gets mode -1 and count 0.  The table and S do not change.
extern "C" int dbl_values_modes(dbl_values *p, int32_t *mode_out, int64_t *count_out) {
  if (!p || !mode_out || !count_out) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  const int64_t C = p->C, H = p->H;
  cudaStream_t st = p->stream;
  Buf best, first, mode, count;
  POST_TRY(best.alloc(sizeof(unsigned long long) * C));
  POST_TRY(first.alloc(sizeof(unsigned long long) * C));
  POST_TRY(mode.alloc(sizeof(int32_t) * C));
  POST_TRY(count.alloc(sizeof(long long) * C));
  POST_TRY(cudaMemsetAsync(best.p, 0, sizeof(unsigned long long) * C, st));
  POST_TRY(cudaMemsetAsync(first.p, 0xff, sizeof(unsigned long long) * C, st));
  const unsigned long long *key = p->tab_key[p->cur].as<unsigned long long>();
  const long long *cnt = p->tab_cnt[p->cur].as<long long>();
  const int warp_grid = (int)std::min<int64_t>((H + THREADS - 1) / THREADS, 8192);
  k_mode_count<<<warp_grid, THREADS, 0, st>>>(H, p->val_bits, key, cnt, best.as<unsigned long long>());
  k_mode_first<<<warp_grid, THREADS, 0, st>>>(H, p->val_bits, key, cnt, best.as<unsigned long long>(),
                                              first.as<unsigned long long>());
  k_mode_out<<<grid_for(C), THREADS, 0, st>>>(C, (1ull << p->val_bits) - 1, key, best.as<unsigned long long>(),
                                              first.as<unsigned long long>(), mode.as<int32_t>(),
                                              count.as<long long>());
  POST_TRY(cudaGetLastError());
  // host or device outputs: unified addressing picks the copy direction
  POST_TRY(cudaMemcpyAsync(mode_out, mode.p, sizeof(int32_t) * C, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(count_out, count.p, sizeof(int64_t) * C, cudaMemcpyDefault, st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// ---- new records linked to a finished chain: the posterior predictive of each query record's entity --------------
// For query q (value ids x_qa, -1 = missing, file f(q)) and a sample with clusters k of entity values y_ka and
// distortion probabilities theta_af, the collapsed PCG-II link weight against cluster k is w(q, k) = prod over the
// observed a of g_qa(y_ka), g = (1 - theta) [x = y] + theta psi(x) norm(y) expsim(x, y), and the expected weight of an
// entity no record links to is m(q) = prod over the observed a of h_qa, h = psi(x) ((1 - theta) + theta sigma(x)).
// Every weight is carried relative to m: rho(q, k) = prod_a r_qa(y), r = g / h = c0 [x = y] + c1 norm(y) expsim(x, y)
// with c0 = (1 - theta) / h and c1 = theta psi(x) / h, so a product of 32 factors stays in range whatever the
// attributes' probabilities.  log Z(q) = log m(q) + log(sum_k rho(q, k) + M - K).
//   pass 1 (dbl_query_add_sample): k_query_scan sums rho over a chunk of clusters per query -- a block holds 128
//     queries' coefficients and hit masks in shared memory and streams tiles of the clusters' value rows and norms;
//     the chunks' partial sums are added in chunk order (k_query_logz), so the bits do not depend on the schedule.  A
//     second scan emits the clusters with rho >= t (sum rho + M - K), i.e. w >= t Z; their records become candidate
//     keys q << 32 | r, merged into the held sorted set by the merge kernels of dbl_pairs.
//   pass 2 (dbl_query_score_sample): one thread per held candidate adds exp(log w - L_q), L_q = max_s log Z_s(q).
// A query's hits for attribute a are the sparse row of x (the value ids y with expsim(x, y) != 1), sorted; a 64-bit
// mask of hashed hit ids in shared memory skips the search of the row for almost every y that is not a hit.
namespace {
constexpr int QUERY_THREADS = 128;  // queries per scan block
constexpr int QUERY_TILE = 64;      // clusters per shared-memory tile

__device__ __forceinline__ unsigned long long hit_bit(int32_t y) {
  return 1ull << ((uint32_t)y * 0x9E3779B1u >> 26);
}

// expsim(x, y) of a query attribute: its sorted hit row [lo, hi), 1 off the row
__device__ __forceinline__ double hit_value(const int32_t *__restrict__ col, const double *__restrict__ val,
                                            long long lo, long long hi, int32_t y) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const int32_t c = col[mid];
    if (c == y) return val[mid];
    if (c < y) lo = mid + 1;
    else hi = mid;
  }
  return 1.0;
}

// one sample's coefficients, one thread per query: c0, c1 per observed attribute, log m(q)
__global__ void k_query_coef(int32_t Q, int32_t A, int32_t F, const int32_t *__restrict__ file,
                             const int32_t *__restrict__ x, const double *__restrict__ psi,
                             const double *__restrict__ sigma, const double *__restrict__ theta, double *__restrict__ c0,
                             double *__restrict__ c1, double *__restrict__ logm) {
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < Q; q += (int64_t)gridDim.x * blockDim.x) {
    double lm = 0.0;
    for (int a = 0; a < A; ++a) {
      const int64_t i = q * A + a;
      if (x[i] < 0) {
        c0[i] = 0.0;
        c1[i] = 0.0;
        continue;
      }
      const double th = theta[a * F + file[q]];
      const double h = psi[i] * ((1.0 - th) + th * sigma[i]);
      c0[i] = (1.0 - th) / h;
      c1[i] = th * psi[i] / h;
      lm += log(h);
    }
    logm[q] = lm;
  }
}

// value ids of the K clusters in [0, V_a)
__global__ void k_query_check_values(int64_t n, int32_t A, const int32_t *__restrict__ y,
                                     const int32_t *__restrict__ nv, int *__restrict__ bad) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t v = y[i];
    if (v < 0 || v >= nv[i % A]) *bad = 1;
  }
}

// rho = prod_a r_qa(y_a) over the observed attributes, in attribute order
__device__ __forceinline__ double query_rho(int32_t A, const int32_t *ys, const double *nrm, const int32_t *sx,
                                            const double *sc0, const double *sc1, const unsigned long long *smask,
                                            int stride, int64_t qa0, const long long *__restrict__ hoff,
                                            const int32_t *__restrict__ hcol, const double *__restrict__ hval) {
  double rho = 1.0;
  for (int a = 0; a < A; ++a) {
    const int32_t xv = sx[a * stride];
    if (xv < 0) continue;
    const int32_t y = ys[a];
    double t = sc1[a * stride] * nrm[a];
    if (smask[a * stride] & hit_bit(y)) t = t * hit_value(hcol, hval, hoff[qa0 + a], hoff[qa0 + a + 1], y);
    rho = rho * ((y == xv ? sc0[a * stride] : 0.0) + t);
  }
  return rho;
}

// Pass-1 scan of clusters [chunk lo, hi) for the block's 128 queries.  EMIT = false: partial[chunk][q] = the sum of
// rho in cluster order.  EMIT = true: every (q, k) with rho >= thr[q] is appended to out (q << 32 | k) while it fits.
template <bool EMIT>
__global__ void __launch_bounds__(QUERY_THREADS) k_query_scan(
    int32_t Q, int32_t A, int64_t K, int64_t chunk, const int32_t *__restrict__ y, const int32_t *__restrict__ voff,
    const double *__restrict__ norm, const int32_t *__restrict__ x, const double *__restrict__ c0,
    const double *__restrict__ c1, const unsigned long long *__restrict__ mask, const long long *__restrict__ hoff,
    const int32_t *__restrict__ hcol, const double *__restrict__ hval, double *__restrict__ partial,
    const double *__restrict__ thr, unsigned long long *__restrict__ out, unsigned long long *__restrict__ count,
    unsigned long long cap) {
  extern __shared__ double smem[];
  double *sc0 = smem, *sc1 = sc0 + A * QUERY_THREADS;
  unsigned long long *smask = (unsigned long long *)(sc1 + A * QUERY_THREADS);
  double *tnrm = (double *)(smask + A * QUERY_THREADS);
  int32_t *sx = (int32_t *)(tnrm + A * QUERY_TILE), *ty = sx + A * QUERY_THREADS;
  const int tx = threadIdx.x;
  const int64_t q = (int64_t)blockIdx.x * QUERY_THREADS + tx;
  const bool live = q < Q;
  for (int a = 0; a < A; ++a) {
    const int64_t i = q * A + a;
    sx[a * QUERY_THREADS + tx] = live ? x[i] : -1;
    sc0[a * QUERY_THREADS + tx] = live ? c0[i] : 0.0;
    sc1[a * QUERY_THREADS + tx] = live ? c1[i] : 0.0;
    smask[a * QUERY_THREADS + tx] = live ? mask[i] : 0ull;
  }
  const int64_t lo = (int64_t)blockIdx.y * chunk, hi = K < lo + chunk ? K : lo + chunk;
  const double t_q = EMIT && live ? thr[q] : 0.0;
  double sum = 0.0;
  for (int64_t k0 = lo; k0 < hi; k0 += QUERY_TILE) {
    const int n = (int)(hi - k0 < QUERY_TILE ? hi - k0 : QUERY_TILE);
    __syncthreads();
    for (int j = tx; j < n * A; j += QUERY_THREADS) {
      const int a = j % A;
      const int32_t v = y[k0 * A + j];
      ty[j] = v;
      tnrm[j] = norm[voff[a] + v];
    }
    __syncthreads();
    if (!live) continue;
    for (int j = 0; j < n; ++j) {
      const double rho = query_rho(A, ty + j * A, tnrm + j * A, sx + tx, sc0 + tx, sc1 + tx, smask + tx,
                                   QUERY_THREADS, q * A, hoff, hcol, hval);
      if (EMIT) {
        if (rho >= t_q) {
          const unsigned long long at = atomicAdd(count, 1ull);
          if (at < cap) out[at] = (unsigned long long)q << 32 | (unsigned long long)(k0 + j);
        }
      } else {
        sum += rho;
      }
    }
  }
  if (!EMIT && live) partial[(int64_t)blockIdx.y * Q + q] = sum;
}

// per query: the chunks' sums in chunk order, log Z = log m + log(sum + M - K), and the emission threshold
__global__ void k_query_logz(int32_t Q, int32_t chunks, const double *__restrict__ partial, double extra,
                             const double *__restrict__ logm, double t, double *__restrict__ logz,
                             double *__restrict__ thr) {
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < Q; q += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int32_t c = 0; c < chunks; ++c) s += partial[(int64_t)c * Q + q];
    s += extra;
    logz[q] = logm[q] + log(s);
    thr[q] = t * s;
  }
}

// per cluster: its first position among the records sorted by label (then k_query_cluster_sizes: its size)
__global__ void k_query_cluster_bounds(int64_t R, const int32_t *__restrict__ lab_s, int32_t *__restrict__ cstart) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = lab_s[i];
    if (i == 0 || lab_s[i - 1] != c) cstart[c] = (int32_t)i;
  }
}

__global__ void k_query_cluster_sizes(int64_t R, const int32_t *__restrict__ lab_s, const int32_t *__restrict__ cstart,
                                      int32_t *__restrict__ csize) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x) {
    const int32_t c = lab_s[i];
    if (i == R - 1 || lab_s[i + 1] != c) csize[c] = (int32_t)(i - cstart[c] + 1);
  }
}

__global__ void k_query_flag_empty(int64_t K, const int32_t *__restrict__ csize, int *__restrict__ bad) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < K; k += (int64_t)gridDim.x * blockDim.x)
    if (csize[k] <= 0) *bad = 1;
}

// entry n is 0, so an exclusive scan over n + 1 entries ends with the number of candidate keys
__global__ void k_query_emit_sizes(int64_t n, const unsigned long long *__restrict__ qk,
                                   const int32_t *__restrict__ csize, long long *__restrict__ len) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i <= n; i += (int64_t)gridDim.x * blockDim.x)
    len[i] = i < n ? csize[(uint32_t)(qk[i] & 0xffffffffull)] : 0;
}

// one warp per emitted (q, k): the keys q << 32 | r of the records of cluster k
__global__ void k_query_emit_keys(int64_t n, const unsigned long long *__restrict__ qk,
                                  const int32_t *__restrict__ cstart, const int32_t *__restrict__ rec_s,
                                  const long long *__restrict__ off, unsigned long long *__restrict__ keys) {
  const int lane = threadIdx.x & 31;
  const int64_t nwarps = (int64_t)gridDim.x * WARPS_PER_BLOCK;
  for (int64_t w = blockIdx.x * (int64_t)WARPS_PER_BLOCK + (threadIdx.x >> 5); w < n; w += nwarps) {
    const unsigned long long hi = qk[w] & 0xffffffff00000000ull;
    const int32_t k = (int32_t)(qk[w] & 0xffffffffull);
    const long long o = off[w], m = off[w + 1] - o;
    const int32_t *rec = rec_s + cstart[k];
    for (long long j = lane; j < m; j += 32) keys[o + j] = hi | (uint32_t)rec[j];
  }
}

// per query the largest log Z over the pass-1 samples
__global__ void k_query_scale(int32_t Q, int32_t S, const double *__restrict__ logz, double *__restrict__ scale) {
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < Q; q += (int64_t)gridDim.x * blockDim.x) {
    double m = -INFINITY;
    for (int32_t s = 0; s < S; ++s) m = fmax(m, logz[(int64_t)s * Q + q]);
    scale[q] = m;
  }
}

// pass 2, one thread per candidate: sum += exp(log m + log rho - L_q) of the record's cluster in this sample
__global__ void k_query_score(int64_t H, int32_t A, const unsigned long long *__restrict__ key,
                              const int32_t *__restrict__ label, const int32_t *__restrict__ y,
                              const int32_t *__restrict__ voff, const double *__restrict__ norm,
                              const int32_t *__restrict__ x, const double *__restrict__ c0,
                              const double *__restrict__ c1, const unsigned long long *__restrict__ mask,
                              const long long *__restrict__ hoff, const int32_t *__restrict__ hcol,
                              const double *__restrict__ hval, const double *__restrict__ logm,
                              const double *__restrict__ scale, double *__restrict__ sum) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < H; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = (int64_t)(key[i] >> 32);
    const int32_t r = (int32_t)(key[i] & 0xffffffffull);
    const int32_t *ys = y + (int64_t)label[r] * A;
    const int64_t qa0 = q * A;
    double rho = 1.0;
    for (int a = 0; a < A; ++a) {
      const int32_t xv = x[qa0 + a];
      if (xv < 0) continue;
      const int32_t v = ys[a];
      double t = c1[qa0 + a] * norm[voff[a] + v];
      if (mask[qa0 + a] & hit_bit(v)) t = t * hit_value(hcol, hval, hoff[qa0 + a], hoff[qa0 + a + 1], v);
      rho = rho * ((v == xv ? c0[qa0 + a] : 0.0) + t);
    }
    sum[i] += exp(logm[q] + log(rho) - scale[q]);
  }
}

__global__ void k_query_split(int64_t H, const unsigned long long *__restrict__ key, int32_t *__restrict__ query,
                              int32_t *__restrict__ record) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < H; i += (int64_t)gridDim.x * blockDim.x) {
    query[i] = (int32_t)(key[i] >> 32);
    record[i] = (int32_t)(key[i] & 0xffffffffull);
  }
}

// per query, in sample order: sum Z~, sum Z~^2 and the new-entity sum, Z~ = exp(log Z - L_q)
__global__ void k_query_totals(int32_t Q, int32_t S, const double *__restrict__ logz, const double *__restrict__ logm,
                               const long long *__restrict__ kcount, int64_t M, const double *__restrict__ scale,
                               double *__restrict__ zsum, double *__restrict__ zsq, double *__restrict__ fresh) {
  for (int64_t q = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; q < Q; q += (int64_t)gridDim.x * blockDim.x) {
    double a = 0.0, b = 0.0, c = 0.0;
    for (int32_t s = 0; s < S; ++s) {
      const double z = exp(logz[(int64_t)s * Q + q] - scale[q]);
      a += z;
      b += z * z;
      const long long un = M - kcount[s];
      if (un > 0) c += exp(log((double)un) + logm[(int64_t)s * Q + q] - scale[q]);
    }
    zsum[q] = a;
    zsq[q] = b;
    fresh[q] = c;
  }
}
}  // namespace

struct dbl_query : Handle {
  int32_t Q = 0, A = 0, F = 0;
  int64_t M = 0, max_candidates = 0;
  double t = 0.0;
  int64_t emit_cap = 0;                 // (q, k) pairs one sample may emit: Q (floor(1 / t) + 2), max_candidates
  int q_bits = 1;                       // bits of a query index
  Buf voff, nvals, norm;                // per attribute: offset into norm, V_a; norm(y) of every attribute
  Buf file, x, psi, sigma, mask;        // per query / (query, attribute)
  Buf hoff, hcol, hval;                 // hit rows: (Q A + 1) int64 offsets, their value ids and expsim
  Buf c0, c1, logm1, thr, theta;        // one sample's coefficients, log m, emission thresholds and theta
  Buf y;                                // one sample's cluster values [K][A]
  Buf partial;                          // [chunks][Q] pass-1 sums
  Buf logz, logm, kcount;               // per pass-1 sample: [S][Q] log Z, [S][Q] log m, K_s
  int32_t S2 = 0;                       // pass-2 samples scored
  Buf scale, sums;                      // L_q; per held candidate the pass-2 sum
  Buf iota, lab_s, rec_s, head, start;  // records grouped by label
  Buf cstart, csize;                    // per cluster
  Buf emit, emit_n, len, off;           // emitted (q, k), their count, key counts and offsets
  Buf key_in, key_s, is_new, rank;      // candidate keys of a sample, merge flags and ranks
  Buf tab_key[2], tab_cnt[2];           // held candidate set (index cur) and the spare one
  int cur = 0;
  int64_t H = 0;
  Buf tmp;
};

namespace {
size_t query_smem(int32_t A) {
  return (size_t)A * QUERY_THREADS * (3 * sizeof(double) + sizeof(int32_t)) +
         (size_t)A * QUERY_TILE * (sizeof(double) + sizeof(int32_t));
}

// One sample's common steps: labels in [0, K), value ids in range, theta in [0, 1]; theta and the values uploaded;
// the coefficients and log m of every query (into c0, c1, logm_out)
int query_take_sample(dbl_query *p, const int32_t *labels, int32_t K, const int32_t *values, const double *theta,
                      double *logm_out) {
  if (K <= 0 || K > p->M || K > p->R) return DBL_ERR_INVALID;
  const int A = p->A, F = p->F;
  for (int i = 0; i < A * F; ++i)
    if (!(theta[i] >= 0.0 && theta[i] <= 1.0)) return DBL_ERR_INVALID;
  if (const int rc = p->take_labels(labels, p->cluster, K); rc != DBL_OK) return rc;
  cudaStream_t st = p->stream;
  const int64_t n = (int64_t)K * A;
  POST_TRY(p->y.reserve(sizeof(int32_t) * (size_t)n));
  POST_TRY(cudaMemcpyAsync(p->y.p, values, sizeof(int32_t) * n, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(p->theta.p, theta, sizeof(double) * A * F, cudaMemcpyHostToDevice, st));
  POST_TRY(cudaMemsetAsync(p->bad.p, 0, sizeof(int), st));
  k_query_check_values<<<grid_for(n), THREADS, 0, st>>>(n, A, p->y.as<int32_t>(), p->nvals.as<int32_t>(),
                                                        p->bad.as<int>());
  int flag = 0;
  POST_TRY(cudaMemcpyAsync(&flag, p->bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaStreamSynchronize(st));
  if (flag) return DBL_ERR_INVALID;
  k_query_coef<<<grid_for(p->Q), THREADS, 0, st>>>(p->Q, A, F, p->file.as<int32_t>(), p->x.as<int32_t>(),
                                                   p->psi.as<double>(), p->sigma.as<double>(), p->theta.as<double>(),
                                                   p->c0.as<double>(), p->c1.as<double>(), logm_out);
  POST_TRY(cudaGetLastError());
  return DBL_OK;
}
}  // namespace

extern "C" int dbl_query_create(dbl_query **out, int64_t num_records, int64_t population_size, int32_t num_queries,
                                int32_t num_attrs, int32_t num_files, const int32_t *num_values, const double *norm,
                                const int32_t *file, const int32_t *x, const double *psi, const double *sigma,
                                const int64_t *hit_offsets, const int32_t *hit_values, const double *hit_expsim,
                                double min_link_probability, int64_t max_candidates) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || population_size < 1 || num_queries <= 0 || num_attrs <= 0 ||
      num_attrs > 32 || num_files <= 0 || !num_values || !norm || !file || !x || !psi || !sigma || !hit_offsets ||
      !(min_link_probability > 0.0 && min_link_probability <= 1.0) || max_candidates <= 0 ||
      max_candidates > INT32_MAX)
    return DBL_ERR_INVALID;
  const int64_t Q = num_queries, A = num_attrs, QA = Q * A, nh = hit_offsets[QA];
  if (hit_offsets[0] != 0 || nh < 0 || (nh > 0 && (!hit_values || !hit_expsim))) return DBL_ERR_INVALID;
  std::vector<int32_t> voff(A);
  int64_t nv_total = 0;
  for (int a = 0; a < A; ++a) {
    if (num_values[a] <= 0) return DBL_ERR_INVALID;
    voff[a] = (int32_t)nv_total;
    nv_total += num_values[a];
  }
  if (nv_total > INT32_MAX) return DBL_ERR_INVALID;
  for (int64_t q = 0; q < Q; ++q)
    if (file[q] < 0 || file[q] >= num_files) return DBL_ERR_INVALID;
  for (int64_t i = 0; i < QA; ++i) {
    const int a = (int)(i % A);
    if (x[i] < -1 || x[i] >= num_values[a] || hit_offsets[i] > hit_offsets[i + 1]) return DBL_ERR_INVALID;
  }
  std::vector<unsigned long long> mask(QA, 0ull);
  for (int64_t i = 0; i < QA; ++i)
    for (int64_t j = hit_offsets[i]; j < hit_offsets[i + 1]; ++j) {
      const int32_t v = hit_values[j];
      if (v < 0 || v >= num_values[i % A] || (j > hit_offsets[i] && hit_values[j - 1] >= v)) return DBL_ERR_INVALID;
      mask[i] |= 1ull << ((uint32_t)v * 0x9E3779B1u >> 26);
    }
  return open_handle(out, num_records, [&](dbl_query *p) {
    p->Q = num_queries;
    p->A = num_attrs;
    p->F = num_files;
    p->M = population_size;
    p->t = min_link_probability;
    p->max_candidates = max_candidates;
    // every emitted (q, k) adds at least one candidate key, so more than max_candidates is a refusal anyway
    // clamped before the product: at most max_candidates (< 2^31) per query, so Q times it fits int64
    const int64_t per_query = (int64_t)std::min(std::floor(1.0 / min_link_probability) + 2.0, (double)max_candidates);
    p->emit_cap = std::min<int64_t>(Q * per_query, max_candidates);
    p->q_bits = bits_for(Q);
    const int64_t R = num_records;
    const size_t r4 = sizeof(int32_t) * (size_t)R, qa8 = sizeof(double) * (size_t)QA;
    if (p->voff.alloc(sizeof(int32_t) * A) != cudaSuccess || p->nvals.alloc(sizeof(int32_t) * A) != cudaSuccess ||
        p->norm.alloc(sizeof(double) * nv_total) != cudaSuccess || p->file.alloc(sizeof(int32_t) * Q) != cudaSuccess ||
        p->x.alloc(sizeof(int32_t) * QA) != cudaSuccess || p->psi.alloc(qa8) != cudaSuccess ||
        p->sigma.alloc(qa8) != cudaSuccess || p->mask.alloc(qa8) != cudaSuccess ||
        p->hoff.alloc(sizeof(long long) * (QA + 1)) != cudaSuccess ||
        p->hcol.alloc(sizeof(int32_t) * std::max<int64_t>(nh, 1)) != cudaSuccess ||
        p->hval.alloc(sizeof(double) * std::max<int64_t>(nh, 1)) != cudaSuccess || p->c0.alloc(qa8) != cudaSuccess ||
        p->c1.alloc(qa8) != cudaSuccess || p->logm1.alloc(sizeof(double) * Q) != cudaSuccess ||
        p->thr.alloc(sizeof(double) * Q) != cudaSuccess || p->theta.alloc(sizeof(double) * A * num_files) != cudaSuccess ||
        p->scale.alloc(sizeof(double) * Q) != cudaSuccess || p->iota.alloc(r4) != cudaSuccess ||
        p->lab_s.alloc(r4) != cudaSuccess || p->rec_s.alloc(r4) != cudaSuccess || p->head.alloc(r4) != cudaSuccess ||
        p->start.alloc(r4) != cudaSuccess || p->cstart.alloc(r4) != cudaSuccess || p->csize.alloc(r4) != cudaSuccess ||
        p->emit.alloc(sizeof(unsigned long long) * std::min<int64_t>(p->emit_cap, 4 * Q + 1024)) != cudaSuccess ||
        p->emit_n.alloc(sizeof(unsigned long long)) != cudaSuccess)
      return DBL_ERR_CUDA;
    cudaStream_t st = p->stream;
    POST_TRY(cudaMemcpyAsync(p->voff.p, voff.data(), sizeof(int32_t) * A, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->nvals.p, num_values, sizeof(int32_t) * A, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->norm.p, norm, sizeof(double) * nv_total, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->file.p, file, sizeof(int32_t) * Q, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->x.p, x, sizeof(int32_t) * QA, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->psi.p, psi, qa8, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->sigma.p, sigma, qa8, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->mask.p, mask.data(), qa8, cudaMemcpyHostToDevice, st));
    POST_TRY(cudaMemcpyAsync(p->hoff.p, hit_offsets, sizeof(long long) * (QA + 1), cudaMemcpyHostToDevice, st));
    if (nh > 0) {
      POST_TRY(cudaMemcpyAsync(p->hcol.p, hit_values, sizeof(int32_t) * nh, cudaMemcpyHostToDevice, st));
      POST_TRY(cudaMemcpyAsync(p->hval.p, hit_expsim, sizeof(double) * nh, cudaMemcpyHostToDevice, st));
    }
    // the largest any handle needs (32 attributes): a later handle with fewer attributes must not lower the limit an
    // earlier one launches under
    const int smem = (int)query_smem(32);
    POST_TRY(cudaFuncSetAttribute(k_query_scan<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    POST_TRY(cudaFuncSetAttribute(k_query_scan<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    k_iota<<<grid_for(R), THREADS, 0, st>>>(R, p->iota.as<int32_t>());
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaStreamSynchronize(st));
    return DBL_OK;
  });
}

extern "C" void dbl_query_free(dbl_query *p) { free_handle(p); }

extern "C" int32_t dbl_query_num_samples(const dbl_query *p) { return p ? p->S : 0; }

// Pass 1, one sample: coefficients; the scan's sums and log Z; the emitting scan; the emitted clusters' records as
// candidate keys, radix-sorted and merged into the spare set; commit (set swap, log Z / log m / K kept, S + 1) only when
// the union fits max_candidates.  A refusal or failure leaves the handle as it was.
extern "C" int dbl_query_add_sample(dbl_query *p, const int32_t *labels, int32_t num_clusters, const int32_t *values,
                                    const double *theta) {
  if (!p || !labels || !values || !theta || p->S == INT32_MAX) return DBL_ERR_INVALID;
  if (p->S2 > 0) return DBL_ERR_STATE;  // pass 2 has begun
  DeviceScope ds(p->device);
  const int64_t Q = p->Q, A = p->A, R = p->R, K = num_clusters, S = p->S;
  cudaStream_t st = p->stream;
  POST_TRY(p->logz.reserve_keep(sizeof(double) * Q * (S + 1), sizeof(double) * Q * S, st));
  POST_TRY(p->logm.reserve_keep(sizeof(double) * Q * (S + 1), sizeof(double) * Q * S, st));
  POST_TRY(p->kcount.reserve_keep(sizeof(long long) * (S + 1), sizeof(long long) * S, st));
  double *logz_s = p->logz.as<double>() + Q * S, *logm_s = p->logm.as<double>() + Q * S;
  if (const int rc = query_take_sample(p, labels, num_clusters, values, theta, logm_s); rc != DBL_OK) return rc;

  // records grouped by cluster; every cluster must hold one
  const int rc_g = group_by_key(R, bits_for(K), p->cluster.as<int32_t>(), p->iota.as<int32_t>(),
                                p->lab_s.as<int32_t>(), p->rec_s.as<int32_t>(), p->head.as<int32_t>(),
                                p->start.as<int32_t>(), p->tmp, st);
  if (rc_g != DBL_OK) return rc_g;
  POST_TRY(cudaMemsetAsync(p->csize.p, 0, sizeof(int32_t) * K, st));
  k_query_cluster_bounds<<<grid_for(R), THREADS, 0, st>>>(R, p->lab_s.as<int32_t>(), p->cstart.as<int32_t>());
  k_query_cluster_sizes<<<grid_for(R), THREADS, 0, st>>>(R, p->lab_s.as<int32_t>(), p->cstart.as<int32_t>(),
                                                         p->csize.as<int32_t>());
  POST_TRY(cudaMemsetAsync(p->bad.p, 0, sizeof(int), st));
  k_query_flag_empty<<<grid_for(K), THREADS, 0, st>>>(K, p->csize.as<int32_t>(), p->bad.as<int>());

  // the scan: sums per chunk, then log Z and thresholds, then the emitting scan
  const int64_t qtiles = (Q + QUERY_THREADS - 1) / QUERY_THREADS;
  const int64_t tiles = (K + QUERY_TILE - 1) / QUERY_TILE;
  const int64_t chunks = std::max<int64_t>(1, std::min<int64_t>(tiles, (2048 + qtiles - 1) / qtiles));
  const int64_t chunk = ((tiles + chunks - 1) / chunks) * QUERY_TILE;
  const int64_t used = (K + chunk - 1) / chunk;
  POST_TRY(p->partial.reserve(sizeof(double) * Q * used));
  const dim3 grid((unsigned)qtiles, (unsigned)used);
  const size_t smem = query_smem((int32_t)A);
  k_query_scan<false><<<grid, QUERY_THREADS, smem, st>>>(
      (int32_t)Q, (int32_t)A, K, chunk, p->y.as<int32_t>(), p->voff.as<int32_t>(), p->norm.as<double>(),
      p->x.as<int32_t>(), p->c0.as<double>(), p->c1.as<double>(), p->mask.as<unsigned long long>(),
      p->hoff.as<long long>(), p->hcol.as<int32_t>(), p->hval.as<double>(), p->partial.as<double>(), nullptr, nullptr,
      nullptr, 0);
  k_query_logz<<<grid_for(Q), THREADS, 0, st>>>((int32_t)Q, (int32_t)used, p->partial.as<double>(),
                                                (double)(p->M - K), logm_s, p->t, logz_s, p->thr.as<double>());
  // the emitting scan; run again with a larger buffer when the first one overflowed it
  unsigned long long n_emit = 0;
  int flag = 0;
  for (int pass = 0; pass < 2; ++pass) {
    const unsigned long long room = p->emit.cap / sizeof(unsigned long long);
    POST_TRY(cudaMemsetAsync(p->emit_n.p, 0, sizeof(unsigned long long), st));
    k_query_scan<true><<<grid, QUERY_THREADS, smem, st>>>(
        (int32_t)Q, (int32_t)A, K, chunk, p->y.as<int32_t>(), p->voff.as<int32_t>(), p->norm.as<double>(),
        p->x.as<int32_t>(), p->c0.as<double>(), p->c1.as<double>(), p->mask.as<unsigned long long>(),
        p->hoff.as<long long>(), p->hcol.as<int32_t>(), p->hval.as<double>(), nullptr, p->thr.as<double>(),
        p->emit.as<unsigned long long>(), p->emit_n.as<unsigned long long>(), room);
    POST_TRY(cudaGetLastError());
    POST_TRY(cudaMemcpyAsync(&n_emit, p->emit_n.p, sizeof(n_emit), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaMemcpyAsync(&flag, p->bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    POST_TRY(cudaStreamSynchronize(st));
    if (flag || n_emit > (unsigned long long)p->emit_cap) return DBL_ERR_INVALID;
    if (n_emit <= room) break;
    POST_TRY(p->emit.reserve(sizeof(unsigned long long) * n_emit));
  }
  POST_TRY(p->len.reserve(sizeof(long long) * (n_emit + 1)));
  POST_TRY(p->off.reserve(sizeof(long long) * (n_emit + 1)));

  // the emitted clusters' records as keys q << 32 | r
  const int64_t ne = (int64_t)n_emit;
  size_t tb = 0;
  POST_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, p->len.as<long long>(), p->off.as<long long>(), ne + 1, st));
  POST_TRY(p->tmp.reserve(tb));
  k_query_emit_sizes<<<grid_for(ne + 1), THREADS, 0, st>>>(ne, p->emit.as<unsigned long long>(),
                                                           p->csize.as<int32_t>(), p->len.as<long long>());
  tb = p->tmp.cap;
  POST_TRY(cub::DeviceScan::ExclusiveSum(p->tmp.p, tb, p->len.as<long long>(), p->off.as<long long>(), ne + 1, st));
  long long n = 0;
  POST_TRY(cudaMemcpyAsync(&n, p->off.as<long long>() + ne, sizeof(long long), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  if (n > p->max_candidates) return DBL_ERR_INVALID;  // this sample alone does not fit
  const size_t cap8 = sizeof(unsigned long long) * (size_t)p->max_candidates;
  const size_t cap4 = sizeof(int32_t) * (size_t)(p->max_candidates + 1);
  POST_TRY(p->key_in.reserve(sizeof(unsigned long long) * (size_t)n, cap8));
  POST_TRY(p->key_s.reserve(sizeof(unsigned long long) * (size_t)n, cap8));
  POST_TRY(p->is_new.reserve(sizeof(int32_t) * (size_t)(n + 1), cap4));
  POST_TRY(p->rank.reserve(sizeof(int32_t) * (size_t)(n + 1), cap4));
  if (n > 0) {
    k_query_emit_keys<<<(int)std::min<int64_t>((ne + WARPS_PER_BLOCK - 1) / WARPS_PER_BLOCK, 8192), THREADS, 0, st>>>(
        ne, p->emit.as<unsigned long long>(), p->cstart.as<int32_t>(), p->rec_s.as<int32_t>(), p->off.as<long long>(),
        p->key_in.as<unsigned long long>());
    size_t tbk = 0;
    POST_TRY(cub::DeviceRadixSort::SortKeys(nullptr, tbk, (const unsigned long long *)nullptr,
                                            (unsigned long long *)nullptr, (int64_t)n, 0, 32 + p->q_bits, st));
    POST_TRY(p->tmp.reserve(tbk));
    tbk = p->tmp.cap;
    POST_TRY(cub::DeviceRadixSort::SortKeys(p->tmp.p, tbk, p->key_in.as<unsigned long long>(),
                                            p->key_s.as<unsigned long long>(), (int64_t)n, 0, 32 + p->q_bits, st));
  }

  // merge into the spare set, then commit
  const unsigned long long *keys = p->key_s.as<unsigned long long>();
  const unsigned long long *held = p->tab_key[p->cur].as<unsigned long long>();
  const int32_t *hcnt = p->tab_cnt[p->cur].as<int32_t>();
  const int64_t H = p->H;
  int64_t fresh = 0;
  if (const int rc = probe_new_keys(n, keys, H, held, p->is_new, p->rank, p->tmp, st, &fresh); rc != DBL_OK) return rc;
  const int64_t H2 = H + fresh;
  if (H2 > p->max_candidates) return DBL_ERR_INVALID;  // the union does not fit: the held set stays as it is
  const int nxt = p->cur ^ 1;
  POST_TRY(p->tab_key[nxt].reserve(sizeof(unsigned long long) * (size_t)H2, cap8));
  POST_TRY(p->tab_cnt[nxt].reserve(sizeof(int32_t) * (size_t)H2, sizeof(int32_t) * (size_t)p->max_candidates));
  if (const int rc = merge_keys<int32_t>(H, held, hcnt, n, keys, nullptr, p->is_new, p->rank,
                                         p->tab_key[nxt].as<unsigned long long>(), p->tab_cnt[nxt].as<int32_t>(), st);
      rc != DBL_OK)
    return rc;
  const long long kc = K;
  POST_TRY(cudaMemcpyAsync(p->kcount.as<long long>() + S, &kc, sizeof(long long), cudaMemcpyHostToDevice, st));
  POST_TRY(cudaStreamSynchronize(st));
  p->cur = nxt;
  p->H = H2;
  ++p->S;
  return DBL_OK;
}

// Pass 2, one sample, in pass-1 order: the same checks and coefficients, then one thread per held candidate.  The
// first call fixes L_q and zeroes the sums.  A refusal leaves the sums as they were.
extern "C" int dbl_query_score_sample(dbl_query *p, const int32_t *labels, int32_t num_clusters, const int32_t *values,
                                      const double *theta) {
  if (!p || !labels || !values || !theta) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  if (p->S2 >= p->S) return DBL_ERR_INVALID;  // more pass-2 samples than pass-1 samples
  DeviceScope ds(p->device);
  const int64_t Q = p->Q, H = p->H, s = p->S2;
  cudaStream_t st = p->stream;
  long long kc = 0;
  POST_TRY(cudaMemcpy(&kc, p->kcount.as<long long>() + s, sizeof(long long), cudaMemcpyDeviceToHost));
  if (kc != num_clusters) return DBL_ERR_INVALID;  // not the pass-1 sample at this position
  if (const int rc = query_take_sample(p, labels, num_clusters, values, theta, p->logm1.as<double>()); rc != DBL_OK)
    return rc;
  if (s == 0) {
    POST_TRY(p->sums.reserve(sizeof(double) * (size_t)std::max<int64_t>(H, 1)));
    POST_TRY(cudaMemsetAsync(p->sums.p, 0, sizeof(double) * (size_t)std::max<int64_t>(H, 1), st));
    k_query_scale<<<grid_for(Q), THREADS, 0, st>>>((int32_t)Q, p->S, p->logz.as<double>(), p->scale.as<double>());
  }
  if (H > 0)
    k_query_score<<<grid_for(H), THREADS, 0, st>>>(
        H, p->A, p->tab_key[p->cur].as<unsigned long long>(), p->cluster.as<int32_t>(), p->y.as<int32_t>(),
        p->voff.as<int32_t>(), p->norm.as<double>(), p->x.as<int32_t>(), p->c0.as<double>(), p->c1.as<double>(),
        p->mask.as<unsigned long long>(), p->hoff.as<long long>(), p->hcol.as<int32_t>(), p->hval.as<double>(),
        p->logm1.as<double>(), p->scale.as<double>(), p->sums.as<double>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  ++p->S2;
  return DBL_OK;
}

extern "C" int dbl_query_num_candidates(const dbl_query *p, int64_t *n_out) {
  if (!p || !n_out) return DBL_ERR_INVALID;
  *n_out = p->H;
  return DBL_OK;
}

// The held candidates in (query, record) order with their pass-2 sums, and per query L_q, sum Z~, sum Z~^2, the
// new-entity sum and every pass-1 sample's log Z ([S][Q]).  Host or device outputs.
extern "C" int dbl_query_read(dbl_query *p, int32_t *query, int32_t *record, double *sum, double *scale, double *zsum,
                              double *zsq, double *fresh, double *logz) {
  if (!p || (p->H > 0 && (!query || !record || !sum)) || !scale || !zsum || !zsq || !fresh || !logz)
    return DBL_ERR_INVALID;
  if (p->S == 0 || p->S2 != p->S) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  const int64_t Q = p->Q, H = p->H, S = p->S;
  cudaStream_t st = p->stream;
  Buf f, r, a, b, c;
  POST_TRY(f.alloc(sizeof(int32_t) * std::max<int64_t>(H, 1)));
  POST_TRY(r.alloc(sizeof(int32_t) * std::max<int64_t>(H, 1)));
  POST_TRY(a.alloc(sizeof(double) * Q));
  POST_TRY(b.alloc(sizeof(double) * Q));
  POST_TRY(c.alloc(sizeof(double) * Q));
  if (H > 0)
    k_query_split<<<grid_for(H), THREADS, 0, st>>>(H, p->tab_key[p->cur].as<unsigned long long>(), f.as<int32_t>(),
                                                   r.as<int32_t>());
  k_query_totals<<<grid_for(Q), THREADS, 0, st>>>((int32_t)Q, (int32_t)S, p->logz.as<double>(), p->logm.as<double>(),
                                                  p->kcount.as<long long>(), p->M, p->scale.as<double>(), a.as<double>(),
                                                  b.as<double>(), c.as<double>());
  POST_TRY(cudaGetLastError());
  // host or device outputs: unified addressing picks the copy direction
  if (H > 0) {
    POST_TRY(cudaMemcpyAsync(query, f.p, sizeof(int32_t) * H, cudaMemcpyDefault, st));
    POST_TRY(cudaMemcpyAsync(record, r.p, sizeof(int32_t) * H, cudaMemcpyDefault, st));
    POST_TRY(cudaMemcpyAsync(sum, p->sums.p, sizeof(double) * H, cudaMemcpyDefault, st));
  }
  POST_TRY(cudaMemcpyAsync(scale, p->scale.p, sizeof(double) * Q, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(zsum, a.p, sizeof(double) * Q, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(zsq, b.p, sizeof(double) * Q, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(fresh, c.p, sizeof(double) * Q, cudaMemcpyDefault, st));
  POST_TRY(cudaMemcpyAsync(logz, p->logz.p, sizeof(double) * Q * S, cudaMemcpyDefault, st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}

// ---- capture histories: which files each cluster of each sample holds ----------------------------------------------
namespace {
constexpr int CAPTURE_MAX_FILES = 12;  // 2^12 int32 histogram cells: 16 KB of shared memory per block

// One pass over the records: hist[c] |= the file bit of every record of cluster c, and dup[c] gets the bits of the
// files with two or more records in c.  A record whose atomicOr finds its bit already set is not its file's first in c;
// only the first record of a file in c sees the bit clear, so the words are exact in any order.  The lanes of a warp
// sharing a label OR their bits together first (and mark the files two of them share), so one update per label and
// warp reaches memory: a cluster of thousands of records does not serialise on one word.
__global__ void k_capture_or(int64_t R, const int32_t *__restrict__ cluster, const int32_t *__restrict__ file,
                             unsigned *__restrict__ hist, unsigned *__restrict__ dup) {
  const int lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x + (threadIdx.x & ~31); base < R; base += stride) {
    const int64_t r = base + lane;
    const unsigned live = __ballot_sync(0xffffffffu, r < R);
    if (r >= R) continue;
    const int32_t c = cluster[r];
    const unsigned bit = 1u << file[r];
    const unsigned peers = __match_any_sync(live, (unsigned long long)(uint32_t)c);
    const unsigned same_file = __match_any_sync(live, (unsigned long long)(uint32_t)c << 32 | bit);
    const unsigned word = __reduce_or_sync(peers, bit);
    const unsigned twice = __reduce_or_sync(peers, __popc(same_file) > 1 ? bit : 0u);
    if (lane == __ffs(peers) - 1) {
      const unsigned old = atomicOr(&hist[c], word);
      const unsigned d = (old & word) | twice;
      if (d) atomicOr(&dup[c], d);
    }
  }
}

// One pass over [0, R): label i's history word, when non-zero, counts into a shared-memory histogram of the 2^F words,
// flushed into row Hrow with 64-bit atomics; record i adds its cluster's bits to its own row of L -- the other files'
// bits of the history and its own file's bit of the duplicate word (a thread owns its record's row: no atomics).
__global__ void k_capture_count(int64_t R, int32_t F, const int32_t *__restrict__ cluster,
                                const int32_t *__restrict__ file, const unsigned *__restrict__ hist,
                                const unsigned *__restrict__ dup, unsigned long long *__restrict__ Hrow,
                                int32_t *__restrict__ L) {
  extern __shared__ int32_t cells[];
  const int ncell = 1 << F;
  for (int j = threadIdx.x; j < ncell; j += blockDim.x) cells[j] = 0;
  __syncthreads();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < R; i += (int64_t)gridDim.x * blockDim.x) {
    const unsigned w = hist[i];
    if (w) atomicAdd(&cells[w], 1);
    const int32_t c = cluster[i];
    const unsigned own = 1u << file[i];
    unsigned bits = (hist[c] & ~own) | (dup[c] & own);
    int32_t *row = L + i * F;
    while (bits) {
      const int g = __ffs(bits) - 1;
      bits &= bits - 1;
      row[g] += 1;
    }
  }
  __syncthreads();
  for (int j = threadIdx.x; j < ncell; j += blockDim.x)
    if (cells[j]) atomicAdd(&Hrow[j], (unsigned long long)cells[j]);
}
}  // namespace

struct dbl_capture : Handle {
  int32_t F = 1, max_samples = 0;
  Buf file;       // R file numbers in [0, F)
  Buf hist, dup;  // R history words and R duplicate words of the sample being added
  Buf H;          // [max_samples][2^F] int64 cluster counts per history
  Buf L;          // [R][F] int32 record links
};

extern "C" int dbl_capture_create(dbl_capture **out, int64_t num_records, const int32_t *file, int32_t num_files,
                                  int32_t max_samples) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  if (num_records <= 0 || num_records > INT32_MAX || !file || num_files < 1 || num_files > CAPTURE_MAX_FILES ||
      max_samples < 1)
    return DBL_ERR_INVALID;
  return open_handle(out, num_records, [&](dbl_capture *p) {
    const size_t R = (size_t)num_records, cells = (size_t)1 << num_files;
    p->F = num_files;
    p->max_samples = max_samples;
    if (p->file.alloc(sizeof(int32_t) * R) != cudaSuccess || p->hist.alloc(sizeof(unsigned) * R) != cudaSuccess ||
        p->dup.alloc(sizeof(unsigned) * R) != cudaSuccess ||
        p->H.alloc(sizeof(unsigned long long) * cells * (size_t)max_samples) != cudaSuccess ||
        p->L.alloc(sizeof(int32_t) * R * (size_t)num_files) != cudaSuccess)
      return DBL_ERR_CUDA;
    if (const int rc = p->take_labels(file, p->file, num_files); rc != DBL_OK) return rc;
    POST_TRY(cudaMemsetAsync(p->H.p, 0, sizeof(unsigned long long) * cells * (size_t)max_samples, p->stream));
    POST_TRY(cudaMemsetAsync(p->L.p, 0, sizeof(int32_t) * R * (size_t)num_files, p->stream));
    POST_TRY(cudaStreamSynchronize(p->stream));
    return DBL_OK;
  });
}

extern "C" void dbl_capture_free(dbl_capture *p) { free_handle(p); }

extern "C" int32_t dbl_capture_num_samples(const dbl_capture *p) { return p ? p->S : 0; }

// One sample: check the labels; clear the words; OR every record's file bit into its cluster's words; count the
// history words into row S of H and every record's links into L.  S, H and L move only when the labels pass.
extern "C" int dbl_capture_add_sample(dbl_capture *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  if (const int rc = p->take_labels(cluster, p->cluster); rc != DBL_OK) return rc;
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  const int32_t *c = p->cluster.as<int32_t>(), *f = p->file.as<int32_t>();
  POST_TRY(cudaMemsetAsync(p->hist.p, 0, sizeof(unsigned) * R, st));
  POST_TRY(cudaMemsetAsync(p->dup.p, 0, sizeof(unsigned) * R, st));
  k_capture_or<<<grid_for(R), THREADS, 0, st>>>(R, c, f, p->hist.as<unsigned>(), p->dup.as<unsigned>());
  const size_t cells = (size_t)1 << p->F;
  k_capture_count<<<grid_for(R), THREADS, sizeof(int32_t) * cells, st>>>(
      R, p->F, c, f, p->hist.as<unsigned>(), p->dup.as<unsigned>(), p->H.as<unsigned long long>() + cells * p->S,
      p->L.as<int32_t>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaStreamSynchronize(st));
  ++p->S;
  return DBL_OK;
}

extern "C" int dbl_capture_read(dbl_capture *p, int64_t *histories, int32_t *record_links) {
  if (!p || !histories) return DBL_ERR_INVALID;
  if (p->S == 0) return DBL_ERR_STATE;
  DeviceScope ds(p->device);
  cudaStream_t st = p->stream;
  POST_TRY(cudaMemcpyAsync(histories, p->H.p, sizeof(int64_t) * ((size_t)1 << p->F) * (size_t)p->S,
                           cudaMemcpyDeviceToHost, st));
  if (record_links)  // host or device: unified addressing picks the copy direction
    POST_TRY(cudaMemcpyAsync(record_links, p->L.p, sizeof(int32_t) * (size_t)p->R * (size_t)p->F, cudaMemcpyDefault,
                             st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}
