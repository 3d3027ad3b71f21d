// Exact power-of-two rescaling of the entity-value weights (DESIGN.md section 4.7), shared by the host and device
// builds of the base pmfs and by the value update.  A weight that may leave the double range is carried as
// w * 2^(512 e): w stays normal and every step is one of the plain arithmetic's roundings or an exact scaling, so
// while the plain arithmetic stays normal both give the same bits.
#pragma once

#ifdef __CUDACC__
#define DBL_HD __host__ __device__ __forceinline__
#else
#define DBL_HD inline
#endif

constexpr double SC_UP = 0x1p512, SC_DN = 0x1p-512;
constexpr double BASE_Z_MIN = 0x1p-969;  // DBL_MIN * 2^53: a base row whose plain Z_k falls below it is rescaled

// probs(v) n(v)^k as w * 2^(512 e): the k multiplications of the plain weight, w brought back above 2^-512 after
// each (n(v) > 2^-510 keeps the product normal)
DBL_HD double base_weight_sc(const double *probs, const double *norm, bool is_const, int k, int v, int &e) {
  double w = probs[v];
  e = 0;
  if (!is_const)
    for (int i = 0; i < k; ++i) {
      w = w * norm[v];
      if (w < SC_DN) { w = w * SC_UP; --e; }
    }
  return w;
}
// w * 2^(512 d) for d <= 0
DBL_HD double sc_down(double w, int d) {
  for (; d < 0 && w != 0.0; ++d) w = w * SC_DN;
  return w;
}
// Z_k = sum_v probs(v) n(v)^k as z * 2^(512 ez): id order, the sum kept at the scale of the largest weight so far
DBL_HD double base_z_sc(int V, const double *probs, const double *norm, bool is_const, int k, int &ez) {
  double z = base_weight_sc(probs, norm, is_const, k, 0, ez);
  for (int v = 1; v < V; ++v) {
    int e;
    const double w = base_weight_sc(probs, norm, is_const, k, v, e);
    if (e > ez) { z = sc_down(z, ez - e); ez = e; }
    z += sc_down(w, e - ez);
  }
  return z;
}
// row k of the base pmfs B_k(v) = probs(v) n(v)^k / Z_k (k successive multiplications, normalised like DiscreteDist,
// random/IndexNonUniformDiscreteDist.scala:66-88) and its running sums; the weights are rescaled when they underflow
DBL_HD void base_row(int V, const double *probs, const double *norm, bool is_const, int k, double *p, double *c) {
  double z = 0.0;
  for (int v = 0; v < V; ++v) {
    double w = probs[v];
    if (!is_const)
      for (int i = 0; i < k; ++i) w = w * norm[v];
    p[v] = w;
    z += w;
  }
  if (!(z >= BASE_Z_MIN)) {
    int E;
    z = base_z_sc(V, probs, norm, is_const, k, E);
    for (int v = 0; v < V; ++v) {
      int e;
      const double w = base_weight_sc(probs, norm, is_const, k, v, e);
      p[v] = sc_down(w, e - E);
    }
  }
  double run = 0.0;
  for (int v = 0; v < V; ++v) {
    p[v] = p[v] / z;
    run += p[v];
    c[v] = run;
  }
}
