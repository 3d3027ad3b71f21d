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

// position of every run head of the sorted best signatures, 0 elsewhere (a max-scan then gives each element its head)
__global__ void k_run_heads(int64_t n, const unsigned long long *__restrict__ keys, int32_t *__restrict__ head) {
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

struct Buf {
  void *p = nullptr;
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, std::max<size_t>(bytes, 16)); }
  ~Buf() { if (p) cudaFree(p); }
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
}  // namespace

struct dbl_posterior {
  int device = 0;
  int64_t R = 0;
  int32_t max_samples = 0, S = 0;
  cudaStream_t stream = nullptr;
  Buf sig;      // [R][max_samples] signatures
  Buf cluster;  // R labels of the sample being added
  Buf sum;      // R wrapping sums of mix64(record) per cluster
  Buf size;     // R cluster sizes
  Buf bad;      // label check flag
};

#define POST_TRY(expr)                   \
  do {                                   \
    if ((expr) != cudaSuccess) {         \
      cudaGetLastError();                \
      return DBL_ERR_CUDA;               \
    }                                    \
  } while (0)

extern "C" int dbl_posterior_create(dbl_posterior **out, int64_t num_records, int32_t max_samples) {
  if (!out) return DBL_ERR_INVALID;
  *out = nullptr;
  // a record's S samples are sorted in one block, so max_samples <= PAIR_BLOCK
  if (num_records <= 0 || num_records > INT32_MAX || max_samples <= 0 || max_samples > PAIR_BLOCK)
    return DBL_ERR_INVALID;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { cudaGetLastError(); return DBL_ERR_CUDA; }
  auto *p = new dbl_posterior();
  p->R = num_records;
  p->max_samples = max_samples;
  int rc = DBL_OK;
  if (cudaGetDevice(&p->device) != cudaSuccess || cudaStreamCreateWithFlags(&p->stream, cudaStreamNonBlocking) != cudaSuccess ||
      p->sig.alloc(sizeof(unsigned long long) * (size_t)num_records * (size_t)max_samples) != cudaSuccess ||
      p->cluster.alloc(sizeof(int32_t) * (size_t)num_records) != cudaSuccess ||
      p->sum.alloc(sizeof(unsigned long long) * (size_t)num_records) != cudaSuccess ||
      p->size.alloc(sizeof(unsigned int) * (size_t)num_records) != cudaSuccess || p->bad.alloc(sizeof(int)) != cudaSuccess)
    rc = DBL_ERR_CUDA;  // no device, or the signature matrix does not fit
  if (rc != DBL_OK) {
    cudaGetLastError();
    dbl_posterior_free(p);
    return rc;
  }
  *out = p;
  return DBL_OK;
}

extern "C" void dbl_posterior_free(dbl_posterior *p) {
  if (!p) return;
  DeviceScope ds(p->device);
  if (p->stream) {
    cudaStreamSynchronize(p->stream);
    cudaStreamDestroy(p->stream);
  }
  delete p;  // Buf destructors free the device memory
}

extern "C" int32_t dbl_posterior_num_samples(const dbl_posterior *p) { return p ? p->S : 0; }

extern "C" int dbl_posterior_add_sample(dbl_posterior *p, const int32_t *cluster) {
  if (!p || !cluster || p->S >= p->max_samples) return DBL_ERR_INVALID;
  DeviceScope ds(p->device);
  const int64_t R = p->R;
  cudaStream_t st = p->stream;
  const int32_t *c = p->cluster.as<int32_t>();
  // host or device labels: unified addressing picks the copy direction
  POST_TRY(cudaMemcpyAsync(p->cluster.p, cluster, sizeof(int32_t) * R, cudaMemcpyDefault, st));
  POST_TRY(cudaMemsetAsync(p->bad.p, 0, sizeof(int), st));
  k_check_labels<<<grid_for(R), THREADS, 0, st>>>(R, c, p->bad.as<int>());
  int bad = 0;
  POST_TRY(cudaMemcpyAsync(&bad, p->bad.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaStreamSynchronize(st));
  if (bad) return DBL_ERR_INVALID;
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
  // group records by best signature: stable sort of (signature, record), run heads, max-scan, scatter
  Buf rec_in, keys_s, rec_s, head, head_scan, labels, tmp;
  POST_TRY(rec_in.alloc(sizeof(int32_t) * R));
  POST_TRY(keys_s.alloc(sizeof(unsigned long long) * R));
  POST_TRY(rec_s.alloc(sizeof(int32_t) * R));
  POST_TRY(head.alloc(sizeof(int32_t) * R));
  POST_TRY(head_scan.alloc(sizeof(int32_t) * R));
  POST_TRY(labels.alloc(sizeof(int32_t) * R));
  size_t tb_sort = 0, tb_scan = 0;
  POST_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, (const unsigned long long *)nullptr,
                                           (unsigned long long *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
                                           (int)R, 0, 64, st));
  POST_TRY(cub::DeviceScan::InclusiveScan(nullptr, tb_scan, (const int32_t *)nullptr, (int32_t *)nullptr, MaxOp(),
                                          (int)R, st));
  POST_TRY(tmp.alloc(std::max(tb_sort, tb_scan)));
  k_iota<<<grid_for(R), THREADS, 0, st>>>(R, rec_in.as<int32_t>());
  POST_TRY(cub::DeviceRadixSort::SortPairs(tmp.p, tb_sort, best.as<unsigned long long>(),
                                           keys_s.as<unsigned long long>(), rec_in.as<int32_t>(), rec_s.as<int32_t>(),
                                           (int)R, 0, 64, st));
  k_run_heads<<<grid_for(R), THREADS, 0, st>>>(R, keys_s.as<unsigned long long>(), head.as<int32_t>());
  POST_TRY(cub::DeviceScan::InclusiveScan(tmp.p, tb_scan, head.as<int32_t>(), head_scan.as<int32_t>(), MaxOp(), (int)R,
                                          st));
  k_scatter_labels<<<grid_for(R), THREADS, 0, st>>>(R, rec_s.as<int32_t>(), head_scan.as<int32_t>(),
                                                    labels.as<int32_t>());
  POST_TRY(cudaGetLastError());
  POST_TRY(cudaMemcpyAsync(labels_out, labels.p, sizeof(int32_t) * R, cudaMemcpyDeviceToHost, st));
  POST_TRY(cudaStreamSynchronize(st));
  return DBL_OK;
}
