// Internal declarations shared by the host (.cpp) and device (.cu) halves of libdblink_b200.
#pragma once
#include <cmath>
#include <cstdint>
#include <string>
#include <vector>

#include "dblink_b200.h"

// ---- RNG protocol (DESIGN.md "Draw protocol"): Philox4x32-10, counter = (id, sub, iteration, phase),
// key = 64-bit seed; the same function cuRAND ships as curand_Philox4x32_10.
#if defined(__CUDACC__)
#define DBL_HD __host__ __device__ __forceinline__
#else
#define DBL_HD inline
#endif

enum : uint32_t { PH_INIT = 0, PH_THETA = 1, PH_LINK = 2, PH_VALUE = 3, PH_DIST = 4 };

struct Philox4 {
  uint32_t v[4];
};

DBL_HD Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0;
    const uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
    const uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1;
    c3 = (uint32_t)p0;
    c0 = n0;
    c2 = n2;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  Philox4 r;
  r.v[0] = c0; r.v[1] = c1; r.v[2] = c2; r.v[3] = c3;
  return r;
}

// uniform in the open interval (0,1) from 64 random bits: ((bits >> 12) + 0.5) * 2^-52 (exact in binary64)
DBL_HD double unit_from_bits(uint32_t lo, uint32_t hi) {
  const uint64_t x = ((uint64_t)hi << 32) | lo;
  return ((double)(x >> 12) + 0.5) * 2.220446049250313080847263336181640625e-16;
}

struct U2 {
  double u0, u1;
};
DBL_HD U2 uniform2(uint64_t seed, uint32_t phase, uint32_t iter, uint32_t id, uint32_t sub) {
  const Philox4 p = philox4x32_10(id, sub, iter, phase, (uint32_t)seed, (uint32_t)(seed >> 32));
  U2 r;
  r.u0 = unit_from_bits(p.v[0], p.v[1]);
  r.u1 = unit_from_bits(p.v[2], p.v[3]);
  return r;
}

// ---- deterministic elementary functions for the theta draw (DESIGN.md 4.5) --------------------------------
// The Beta draws of updateDistProbs (GU:305-320) need log / exp; libm differs between glibc and CUDA in the last
// bit, and the theta draw runs on the DEVICE here (no host round trip per sweep), so the protocol defines both
// functions through individually rounded binary64 + - * / only (no FMA: -fmad=false / -ffp-contract=off), which
// every IEEE-754 implementation evaluates identically.  The CPU oracle carries its own restatement of the same
// recipe (oracle/dbl_oracle.c); the parity tests compare theta bit for bit.
//   log x = k ln2 + 2s + s R(s^2), x = 2^k m, m in (sqrt(1/2), sqrt(2)], s = (m-1)/(m+1), R = sum_{i=1..11} 2/(2i+1) z^i
//   exp x = 2^k sum_{n=0..14} r^n/n!,  k = floor(x/ln2 + 1/2), r = x - k ln2  (ln2 split hi + lo)
DBL_HD double dbl_bits_to_double(uint64_t b) {
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long)b);
#else
  double d;
  __builtin_memcpy(&d, &b, 8);
  return d;
#endif
}
DBL_HD uint64_t dbl_double_to_bits(double d) {
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double_as_longlong(d);
#else
  uint64_t b;
  __builtin_memcpy(&b, &d, 8);
  return b;
#endif
}
constexpr double DET_LN2_HI = 0x1.62e4200000000p-1, DET_LN2_LO = 0x1.fdf473de6af28p-22;

DBL_HD double det_log(double x) {  // x > 0, finite
  int k = 0;
  uint64_t b = dbl_double_to_bits(x);
  if (((b >> 52) & 0x7ffu) == 0) {  // subnormal: scale by 2^54 (exact)
    x = x * 18014398509481984.0;
    k = -54;
    b = dbl_double_to_bits(x);
  }
  k += (int)((b >> 52) & 0x7ffu) - 1023;
  double m = dbl_bits_to_double((b & 0x000fffffffffffffull) | 0x3ff0000000000000ull);
  if (m > 0x1.6a09e667f3bcdp+0) { m = m * 0.5; k += 1; }
  const double f = m - 1.0;
  const double s = f / (2.0 + f);
  const double z = s * s;
  double R = 0x1.642c8590b2164p-4;
  R = R * z; R = R + 0x1.8618618618618p-4;
  R = R * z; R = R + 0x1.af286bca1af28p-4;
  R = R * z; R = R + 0x1.e1e1e1e1e1e1ep-4;
  R = R * z; R = R + 0x1.1111111111111p-3;
  R = R * z; R = R + 0x1.3b13b13b13b14p-3;
  R = R * z; R = R + 0x1.745d1745d1746p-3;
  R = R * z; R = R + 0x1.c71c71c71c71cp-3;
  R = R * z; R = R + 0x1.2492492492492p-2;
  R = R * z; R = R + 0x1.999999999999ap-2;
  R = R * z; R = R + 0x1.5555555555555p-1;
  R = R * z;
  const double dk = (double)k;
  double t = s * R;
  t = 2.0 * s + t;
  t = t + dk * DET_LN2_LO;
  return dk * DET_LN2_HI + t;
}

DBL_HD double det_exp(double x) {  // finite x
  if (x > 709.0) return dbl_bits_to_double(0x7ff0000000000000ull);
  if (x < -745.0) return 0.0;
  const double t = x * 0x1.71547652b82fep+0 + 0.5;
  long long ki = (long long)t;
  if ((double)ki > t) ki -= 1;  // floor
  const double kf = (double)ki;
  double r = x - kf * DET_LN2_HI;
  r = r - kf * DET_LN2_LO;
  double p = 0x1.93974a8c07c9dp-37;
  p = p * r; p = p + 0x1.6124613a86d09p-33;
  p = p * r; p = p + 0x1.1eed8eff8d898p-29;
  p = p * r; p = p + 0x1.ae64567f544e4p-26;
  p = p * r; p = p + 0x1.27e4fb7789f5cp-22;
  p = p * r; p = p + 0x1.71de3a556c734p-19;
  p = p * r; p = p + 0x1.a01a01a01a01ap-16;
  p = p * r; p = p + 0x1.a01a01a01a01ap-13;
  p = p * r; p = p + 0x1.6c16c16c16c17p-10;
  p = p * r; p = p + 0x1.1111111111111p-7;
  p = p * r; p = p + 0x1.5555555555555p-5;
  p = p * r; p = p + 0x1.5555555555555p-3;
  p = p * r; p = p + 0.5;
  p = p * r; p = p + 1.0;
  p = p * r; p = p + 1.0;
  if (ki < -1000) {  // towards the subnormals: two exact-power-of-two factors
    p = p * dbl_bits_to_double((uint64_t)(1023 - 1000) << 52);
    ki += 1000;
  }
  return p * dbl_bits_to_double((uint64_t)(1023 + ki) << 52);
}

// Theta stream (GU:305-320): Beta(a,b) = X/(X+Y), X, Y ~ Gamma by Marsaglia & Tsang (2000), normals by the polar
// method, uniforms from Philox (phase THETA, id = attr*F + file, sub = call counter).
struct ThetaStream {
  uint64_t seed;
  uint32_t iter, id, calls;
  DBL_HD U2 next() { return uniform2(seed, PH_THETA, iter, id, calls++); }
  DBL_HD double unif() { return next().u0; }
  DBL_HD double normal() {
    for (;;) {
      const U2 u = next();
      const double v1 = 2.0 * u.u0 - 1.0, v2 = 2.0 * u.u1 - 1.0;
      double s = v1 * v1;
      s = s + v2 * v2;
      if (s >= 1.0 || s == 0.0) continue;
      double q = -2.0 * det_log(s);
      q = q / s;
      return v1 * sqrt(q);
    }
  }
  DBL_HD double gamma_ge1(double shape) {
    const double d = shape - 1.0 / 3.0;
    const double c = 1.0 / sqrt(9.0 * d);
    for (;;) {
      const double xn = normal();
      double v = 1.0 + c * xn;
      if (v <= 0.0) continue;
      v = v * v * v;
      const double u = unif();
      const double lhs = det_log(u);
      double t1 = 0.5 * xn;
      t1 = t1 * xn;
      double rhs = t1 + d;
      rhs = rhs - d * v;
      rhs = rhs + d * det_log(v);
      if (lhs < rhs) return d * v;
    }
  }
  DBL_HD double gamma(double shape) {
    if (shape < 1.0) {  // boost: Gamma(a) = Gamma(a+1) U^(1/a)
      const double g = gamma_ge1(shape + 1.0);
      const double u = unif();
      return g * det_exp(det_log(u) / shape);
    }
    return gamma_ge1(shape);
  }
};
DBL_HD double draw_theta_one(uint64_t seed, uint32_t iter, uint32_t id, double alpha, double beta, double n_dist,
                             double file_size) {
  const double s1 = n_dist + alpha;              // GU:312
  const double s2 = file_size - n_dist + beta;   // GU:313
  ThetaStream ts{seed, iter, id, 0};
  const double gx = ts.gamma(s1);
  const double gy = ts.gamma(s2);
  return gx / (gx + gy);
}

// ---- host-side model objects ------------------------------------------------------------------------
struct dbl_index {
  int32_t V = 0;
  bool is_const = true;
  int32_t kmax = 0;
  std::vector<std::string> values;  // sorted
  std::vector<double> probs;        // weight / total
  std::vector<double> phi;          // probabilityOf (renormalised)
  std::vector<double> norm, invnorm;
  std::vector<int32_t> rowptr, col;
  std::vector<double> expsim;
  std::vector<double> pk, cdf;      // (kmax+1) x V
  std::vector<double> logphi, lognorm;
  // per-row perfect hash of the off-diagonal similar values (link kernel): slot = (uint32(v) * hmult[x]) >> hshift
  int32_t hsize = 0, hshift = 32;  // hsize == 0: no table (constant attribute, or rows too long)
  std::vector<uint32_t> hmult;     // V
  std::vector<int32_t> hkeys;      // V x hsize, -1 = empty
  std::vector<double> hvals;       // V x hsize
  // slot codes (hsize == 32 only; empty when the values do not colour): pcode[v] & 31 is the slot of v in EVERY row's
  // table, so a candidate is hashed once for all records; the code-keyed tables lay each row out by those slots
  std::vector<int32_t> pcode;      // V, a bijection onto a subset of [0, 32 * (largest colour class))
  std::vector<int32_t> sckeys;     // V x 32, key = pcode of the entry's value, -1 = empty
  std::vector<double> scvals;      // V x 32
  void finish();
  void build_hash(int min_slots = 32);
  void build_slot_codes();
};

struct dbl_kdtree {
  int32_t n_nodes = 1, n_leaves = 1;
  std::vector<int32_t> attr, kind, split, set_ptr, set_val, leaf_no;
  int32_t leaf_node(const int32_t *yrow) const;
};

// theta draw (GU:305-320) -- host, libm
void host_draw_theta(int A, int F, const double *alpha, const double *beta, uint64_t seed, const int64_t *agg_dist,
                     const int64_t *file_sizes, uint32_t iter, double *theta_out);
int host_levenshtein(const char *a, int la, const char *b, int lb);
void host_jaro_winkler_counts(const char *a, int la, const char *b, int lb, int &m, int &h, int &l);
// GPU all-pairs candidates for the attribute index (dbl_index_gpu.cu): (i, j > i, code) with code = the edit
// distance (similarity 1) or m | h << 8 | l << 16 (similarity 2, Jaro-Winkler counts); false = not applicable
bool gpu_similarity_candidates(int similarity, const std::vector<std::string> &values, double threshold,
                               double max_sim, std::vector<int> &oi, std::vector<int> &oj, std::vector<int> &oc);
// norm / invnorm / pk / cdf on the device (dbl_index_gpu.cu), same values as the host loops; false = not applicable
bool gpu_index_tables(int V, int kmax, bool is_const, const std::vector<double> &probs,
                      const std::vector<int32_t> &rowptr, const std::vector<int32_t> &col,
                      const std::vector<double> &expsim, std::vector<double> &norm, std::vector<double> &invnorm,
                      std::vector<double> &pk, std::vector<double> &cdf);
// unit similarities and the truncation of SimilarityFn.scala:65-70 (dbl_host.cpp, compiled without FP contraction)
double host_levenshtein_unit(int dist, int la, int lb);
double host_jaro_winkler_unit(int m, int h, int l, int la, int lb);
double host_similarity_from_unit(double unit, double threshold, double max_sim);
