// Host half of libdblink_b200: model-table construction, k-d tree, the A x F Beta draws of theta.
// These are the driver-side pieces of the reference (they run once, or once per sweep on A*F scalars);
// everything that scales with records/entities is in dbl_engine.cu.
//
// Reference paths: src/main/scala/com/github/cleanzr/dblink/ ; GU = GibbsUpdates.scala.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <map>
#include <numeric>
#include <queue>
#include <thread>
#include <tuple>

#include "dbl_internal.h"
#include "dbl_scale.h"

// ---------------------------------------------------------------------------------------------------
// SimilarityFn.scala:61-98
// ---------------------------------------------------------------------------------------------------
// Strict UTF-8 (RFC 3629) to UTF-16 code units, the units a Java String holds: no overlong forms, no encoded
// surrogates, nothing above U+10FFFF, no stray or missing continuation bytes.  The units are appended to out.
// false = not valid UTF-8.
bool host_utf8_to_utf16(const char *s, size_t n, std::u16string &out) {
  const unsigned char *p = (const unsigned char *)s, *e = p + n;
  while (p < e) {
    uint32_t c = *p++;
    int extra;
    uint32_t lowest;
    if (c < 0x80) { out.push_back((char16_t)c); continue; }
    if (c >= 0xC2 && c <= 0xDF) { extra = 1; c &= 0x1F; lowest = 0x80; }
    else if (c >= 0xE0 && c <= 0xEF) { extra = 2; c &= 0x0F; lowest = 0x800; }
    else if (c >= 0xF0 && c <= 0xF4) { extra = 3; c &= 0x07; lowest = 0x10000; }
    else return false;  // a continuation byte, C0 / C1 (always overlong) or F5..FF
    if (e - p < extra) return false;
    for (int k = 0; k < extra; ++k, ++p) {
      if ((*p & 0xC0) != 0x80) return false;
      c = c << 6 | (*p & 0x3F);
    }
    if (c < lowest || c > 0x10FFFF || (c >= 0xD800 && c <= 0xDFFF)) return false;
    if (c < 0x10000) {
      out.push_back((char16_t)c);
    } else {
      c -= 0x10000;
      out.push_back((char16_t)(0xD800 + (c >> 10)));
      out.push_back((char16_t)(0xDC00 + (c & 0x3FF)));
    }
  }
  return true;
}

// commons-lang3 getLevenshteinDistance over UTF-16 code units (SimilarityFn.scala:95 compares with charAt)
int host_levenshtein(const char16_t *a, int la, const char16_t *b, int lb) {
  if (la == 0) return lb;
  if (lb == 0) return la;
  // two-row DP on the shorter string
  if (lb > la) { std::swap(a, b); std::swap(la, lb); }
  int buf[2][256];
  std::vector<int> big;
  int *prev = buf[0], *cur = buf[1];
  if (lb + 1 > 256) { big.resize(2 * (size_t)(lb + 1)); prev = big.data(); cur = big.data() + lb + 1; }
  for (int j = 0; j <= lb; ++j) prev[j] = j;
  for (int i = 1; i <= la; ++i) {
    cur[0] = i;
    const char16_t ca = a[i - 1];
    for (int j = 1; j <= lb; ++j) {
      const int sub = prev[j - 1] + (ca != b[j - 1] ? 1 : 0);
      const int del = prev[j] + 1, ins = cur[j - 1] + 1;
      cur[j] = std::min(sub, std::min(del, ins));
    }
    std::swap(prev, cur);
  }
  return prev[lb];
}

double host_levenshtein_unit(int dist, int la, int lb) {
  const int total = la + lb;
  double unit = 1.0;                        // SimilarityFn.scala:86-90
  if (total > 0) {
    const double d = (double)dist;
    unit = 1.0 - 2.0 * d / ((double)total + d);
  }
  return unit;
}

// Jaro-Winkler counts by the greedy scan: each a[i], left to right, takes the first unmatched b[j] with
// |i - j| <= w = max(0, max(la, lb) / 2 - 1) and a[i] == b[j] (m matches); h = matched positions k whose k-th matched
// bytes of a and b differ; l = common prefix, at most 4.  (m, h) are symmetric in (a, b), which the GPU path relies on.
void host_jaro_winkler_counts(const char *a, int la, const char *b, int lb, int &m, int &h, int &l) {
  m = h = l = 0;
  if (la == 0 || lb == 0) return;
  const int w = std::max(0, std::max(la, lb) / 2 - 1);
  char buf[2][256];
  std::vector<char> big;
  char *ma = buf[0], *mb = buf[1];
  if (la > 256 || lb > 256) { big.resize((size_t)la + lb); ma = big.data(); mb = big.data() + la; }
  std::memset(ma, 0, la);
  std::memset(mb, 0, lb);
  for (int i = 0; i < la; ++i)
    for (int j = std::max(0, i - w); j < std::min(lb, i + w + 1); ++j)
      if (!mb[j] && a[i] == b[j]) { ma[i] = mb[j] = 1; ++m; break; }
  for (int i = 0, j = 0; i < la; ++i) {
    if (!ma[i]) continue;
    while (!mb[j]) ++j;
    if (a[i] != b[j]) ++h;
    ++j;
  }
  while (l < 4 && l < la && l < lb && a[l] == b[l]) ++l;
}

double host_jaro_winkler_unit(int m, int h, int l, int la, int lb) {
  if (la == 0 && lb == 0) return 1.0;
  if (m == 0) return 0.0;
  const double jaro = ((double)m / la + (double)m / lb + ((double)m - 0.5 * h) / m) / 3.0;
  return jaro + (0.1 * l) * (1.0 - jaro);  // this TU is compiled with -ffp-contract=off: no FMA here
}

double host_similarity_from_unit(double unit, double threshold, double max_sim) {
  const double factor = max_sim / (max_sim - threshold);  // SimilarityFn.scala:63
  const double s = factor * (max_sim * unit - threshold);  // :66
  return s > 0.0 ? s : 0.0;
}

// unit similarities of a pair: Levenshtein over UTF-16 code units, Jaro-Winkler over UTF-8 bytes
static double host_levenshtein_unit_of(const char16_t *a, int la, const char16_t *b, int lb) {
  return host_levenshtein_unit(host_levenshtein(a, la, b, lb), la, lb);
}
static double host_jaro_winkler_unit_of(const std::string &a, const std::string &b) {
  int m, h, l;
  host_jaro_winkler_counts(a.data(), (int)a.size(), b.data(), (int)b.size(), m, h, l);
  return host_jaro_winkler_unit(m, h, l, (int)a.size(), (int)b.size());
}

// The vocabulary's code units as byte symbols for the device kernel, which indexes its match masks by byte.  The edit
// distance only asks whether two units are equal, so any one-to-one map keeps every distance: the identity when every
// unit is below 256, otherwise a dense table of the distinct units.  false = more than 256 distinct units.
static bool lev_byte_symbols(const std::u16string &units, const std::vector<size_t> &off,
                             std::vector<std::string> &out) {
  std::vector<uint8_t> seen(65536, 0), sym(65536, 0);
  for (char16_t c : units) seen[c] = 1;
  if (std::count(seen.begin() + 256, seen.end(), 1) == 0) {
    for (int c = 0; c < 256; ++c) sym[c] = (uint8_t)c;
  } else {
    int n = 0;
    for (int c = 0; c < 65536; ++c)
      if (seen[c]) {
        if (n == 256) return false;
        sym[c] = (uint8_t)n++;
      }
  }
  out.resize(off.size() - 1);
  for (size_t v = 0; v + 1 < off.size(); ++v) {
    out[v].resize(off[v + 1] - off[v]);
    for (size_t q = off[v]; q < off[v + 1]; ++q) out[v][q - off[v]] = (char)sym[units[q]];
  }
  return true;
}

// unit similarity from the integer a device kernel reports for a pair: the edit distance, or m | h << 8 | l << 16
static double host_unit_from_code(int similarity, int code, int la, int lb) {
  if (similarity == DBL_SIM_JARO_WINKLER)
    return host_jaro_winkler_unit(code & 255, (code >> 8) & 255, code >> 16, la, lb);
  return host_levenshtein_unit(code, la, lb);
}

// ---------------------------------------------------------------------------------------------------
// AttributeIndex.scala:107-245
// ---------------------------------------------------------------------------------------------------
void dbl_index::finish() {
  // DBL_INDEX_GPU: "0" = host loops, "1" = GPU whenever there is one, unset = GPU for vocabularies where the O(V^2)
  // normalisation loop matters.  Both give the same tables (same sums in the same order).
  const char *env = std::getenv("DBL_INDEX_GPU");
  const bool want_gpu = env ? (env[0] == '1') : (V >= 2048);
  if (want_gpu && gpu_index_tables(V, kmax, is_const, probs, rowptr, col, expsim, norm, invnorm, pk, cdf)) {
    // tables built on the device
  } else {
    norm.assign(V, 1.0);
    invnorm.assign(V, 1.0);
    if (!is_const) {
      for (int v = 0; v < V; ++v) {  // computeSimNormalizations, :234-245
        double acc = 0.0;
        int p = rowptr[v];
        const int pe = rowptr[v + 1];
        for (int w = 0; w < V; ++w) {
          double e = 1.0;
          if (p < pe && col[p] == w) e = expsim[p++];
          acc += probs[w] * e;
        }
        invnorm[v] = acc;
        norm[v] = 1.0 / acc;
      }
    }
    pk.assign((size_t)(kmax + 1) * V, 0.0);
    cdf.assign((size_t)(kmax + 1) * V, 0.0);
    for (int k = 0; k <= kmax; ++k)
      base_row(V, probs.data(), norm.data(), is_const, k, pk.data() + (size_t)k * V, cdf.data() + (size_t)k * V);
  }
  phi.assign(pk.begin(), pk.begin() + V);
  logphi.resize(V);
  lognorm.resize(V);
  for (int v = 0; v < V; ++v) {
    logphi[v] = std::log(phi[v]);
    lognorm[v] = std::log(norm[v]);
  }
  build_hash();
}

// Per-row perfect hash tables for expSimOf(x, y) (AttributeIndex.scala:183-186), the row's own value x included: the
// link kernel answers "is y equal or similar to x, and what is the factor" with one shared-memory probe (the entry of
// x itself is replaced per record by the exact-match multiplier).  All rows of an attribute share the table size (a
// power of two <= 256); each row has its own multiplier found by search.
void dbl_index::build_hash(int min_slots) {
  hsize = 0;
  hshift = 32;
  hmult.clear(); hkeys.clear(); hvals.clear();
  pcode.clear(); sckeys.clear(); scvals.clear();
  if (is_const) return;
  int maxlen = 0;
  for (int v = 0; v < V; ++v) maxlen = std::max(maxlen, rowptr[v + 1] - rowptr[v] + 1);
  int H = std::max(32, min_slots);
  while (H < maxlen) H <<= 1;  // a perfect hash needs H >= row length; the multiplier search below decides the rest
  for (; H <= 256; H <<= 1) {
    int lg = 0;
    while ((1 << lg) < H) ++lg;
    const int shift = 32 - lg;
    std::vector<uint32_t> mult(V, 0);
    std::vector<int32_t> keys((size_t)V * H, -1);
    std::vector<double> vals((size_t)V * H, 1.0);
    bool ok = true;
    std::vector<int> used(H);
    for (int v = 0; v < V && ok; ++v) {
      bool found = false;
      for (uint32_t k = 0; k < 2048 && !found; ++k) {
        const uint32_t m = 2654435761u * (2 * k + 1);
        std::fill(used.begin(), used.end(), 0);
        bool clash = false;
        used[((uint32_t)v * m) >> shift] = 1;  // the row's own value always has an entry
        for (int p = rowptr[v]; p < rowptr[v + 1] && !clash; ++p) {
          if (col[p] == v) continue;
          const uint32_t s = ((uint32_t)col[p] * m) >> shift;
          if (used[s]) clash = true;
          used[s] = 1;
        }
        if (!clash) { mult[v] = m; found = true; }
      }
      if (!found) { ok = false; break; }
      keys[(size_t)v * H + (((uint32_t)v * mult[v]) >> shift)] = v;  // value: the diagonal exp sim (1 when absent)
      for (int p = rowptr[v]; p < rowptr[v + 1]; ++p) {
        const uint32_t s = ((uint32_t)col[p] * mult[v]) >> shift;
        keys[(size_t)v * H + s] = col[p];
        vals[(size_t)v * H + s] = expsim[p];
      }
    }
    if (ok) {
      hsize = H; hshift = shift;
      hmult.swap(mult); hkeys.swap(keys); hvals.swap(vals);
      build_slot_codes();
      return;
    }
  }
}

// Slot codes for the 32-slot tables: colour the values with 32 colours so that the values of every row's table
// T(x) = {x} + row(x) get distinct colours; then pcode(v) = colour(v) + 32 k, k numbering the values of v's colour in
// ascending id order, is a bijection whose low five bits are the slot of v in every table that holds v.  The link
// kernel stores pcode(y) in its tiles and hashes a candidate once for all the records it scores.  Greedy colouring
// (DSatur order: the value with the most distinct colours among its conflicts first, then the most conflicts), each
// value taking the allowed colour used least so far, which keeps the code range close to V.  No table is built when
// some value runs out of colours.
void dbl_index::build_slot_codes() {
  pcode.clear(); sckeys.clear(); scvals.clear();
  if (is_const || hsize != 32) return;
  constexpr int H = 32;
  // T(x) without a duplicate of x (a row may hold its own diagonal), and its transpose: the x with v in T(x)
  std::vector<int32_t> tptr(V + 1, 0), tval;
  tval.reserve((size_t)V + rowptr[V]);
  for (int x = 0; x < V; ++x) {
    tval.push_back(x);
    for (int p = rowptr[x]; p < rowptr[x + 1]; ++p)
      if (col[p] != x) tval.push_back(col[p]);
    tptr[x + 1] = (int32_t)tval.size();
  }
  std::vector<int32_t> iptr(V + 1, 0), ival(tval.size());
  for (int32_t v : tval) ++iptr[v + 1];
  for (int v = 0; v < V; ++v) iptr[v + 1] += iptr[v];
  {
    std::vector<int32_t> fill(iptr.begin(), iptr.end() - 1);
    for (int x = 0; x < V; ++x)
      for (int i = tptr[x]; i < tptr[x + 1]; ++i) ival[fill[tval[i]]++] = x;
  }
  std::vector<int64_t> deg(V, 0);  // conflicts counted with multiplicity: an ordering key only
  for (int v = 0; v < V; ++v)
    for (int i = iptr[v]; i < iptr[v + 1]; ++i) deg[v] += tptr[ival[i] + 1] - tptr[ival[i]] - 1;
  std::vector<int> colour(V, -1);
  std::vector<uint32_t> forbid(V, 0u);
  int64_t used[H] = {};
  using Key = std::tuple<int, int64_t, int>;  // (distinct forbidden colours, conflicts, -value): max-heap
  std::priority_queue<Key> heap;
  for (int v = 0; v < V; ++v) heap.emplace(0, deg[v], -v);
  while (!heap.empty()) {
    const auto [sat, dg, nv] = heap.top();
    heap.pop();
    const int v = -nv;
    if (colour[v] >= 0 || sat != __builtin_popcount(forbid[v])) continue;  // stale entry
    const uint32_t allowed = ~forbid[v];
    if (!allowed) return;  // 32 colours are not enough: the kernel keeps the per-row multipliers
    int c = -1;
    for (int k = 0; k < H; ++k)
      if (((allowed >> k) & 1u) && (c < 0 || used[k] < used[c])) c = k;
    colour[v] = c;
    ++used[c];
    for (int i = iptr[v]; i < iptr[v + 1]; ++i) {
      const int x = ival[i];
      for (int j = tptr[x]; j < tptr[x + 1]; ++j) {
        const int u = tval[j];
        if (colour[u] >= 0 || ((forbid[u] >> c) & 1u)) continue;
        forbid[u] |= 1u << c;
        heap.emplace(__builtin_popcount(forbid[u]), deg[u], -u);
      }
    }
  }
  std::vector<int32_t> code(V);
  int64_t seen[H] = {};
  for (int v = 0; v < V; ++v) code[v] = colour[v] + H * (int32_t)seen[colour[v]]++;
  std::vector<int32_t> keys((size_t)V * H, -1);
  std::vector<double> vals((size_t)V * H, 1.0);
  for (int x = 0; x < V; ++x) {
    keys[(size_t)x * H + colour[x]] = code[x];  // value: the diagonal exp sim (1 when absent), as in build_hash
    for (int p = rowptr[x]; p < rowptr[x + 1]; ++p) {
      keys[(size_t)x * H + colour[col[p]]] = code[col[p]];
      vals[(size_t)x * H + colour[col[p]]] = expsim[p];
    }
  }
  pcode.swap(code); sckeys.swap(keys); scvals.swap(vals);
}

extern "C" int dbl_index_build(dbl_index **out, const char *const *values, const double *weights, int32_t V,
                               int similarity, double threshold, double max_sim, int32_t kmax) {
  if (!out || !values || !weights || V <= 0 || kmax < 0) return DBL_ERR_INVALID;  // "index cannot be empty" :111
  if (similarity < DBL_SIM_CONSTANT || similarity > DBL_SIM_JARO_WINKLER) return DBL_ERR_INVALID;
  if (similarity != DBL_SIM_CONSTANT && !(max_sim > 0.0 && threshold >= 0.0 && threshold < max_sim))
    return DBL_ERR_INVALID;  // SimilarityFn.scala:59-61
  auto *ix = new dbl_index();
  ix->V = V;
  ix->is_const = (similarity == DBL_SIM_CONSTANT);
  ix->kmax = kmax;
  std::vector<int> order(V);
  std::iota(order.begin(), order.end(), 0);
  std::sort(order.begin(), order.end(), [&](int a, int b) { return std::strcmp(values[a], values[b]) < 0; });
  ix->values.resize(V);
  ix->probs.resize(V);
  double total = 0.0;
  for (int i = 0; i < V; ++i) total += weights[order[i]];
  for (int i = 0; i < V; ++i) {
    ix->values[i] = values[order[i]];
    ix->probs[i] = weights[order[i]] / total;
  }
  ix->rowptr.assign(V + 1, 0);
  if (!ix->is_const) {
    // all-pairs thresholded similarity (computeSimValueIndex, :219-231)
    const bool lev = similarity == DBL_SIM_LEVENSHTEIN;
    std::u16string units;               // Levenshtein: every value decoded once, value v = units[off[v] .. off[v+1])
    std::vector<size_t> off(V + 1, 0);
    bool ascii = true;                  // every value ASCII: its code units are its bytes
    if (lev) {
      size_t bytes = 0;
      for (int i = 0; i < V; ++i) bytes += ix->values[i].size();
      units.reserve(bytes);
      for (int i = 0; i < V; ++i) {
        if (!host_utf8_to_utf16(ix->values[i].data(), ix->values[i].size(), units)) {
          delete ix;
          return DBL_ERR_INVALID;
        }
        off[i + 1] = units.size();
        ascii = ascii && off[i + 1] - off[i] == ix->values[i].size();
      }
    }
    std::vector<std::vector<std::pair<int32_t, double>>> rows(V);
    std::vector<int> len(V);  // Levenshtein: code units (String.length); Jaro-Winkler: bytes
    for (int i = 0; i < V; ++i) len[i] = lev ? (int)(off[i + 1] - off[i]) : (int)ix->values[i].size();
    bool done = false;
    const char *env = std::getenv("DBL_INDEX_GPU");  // "0" = host only, "1" = GPU whenever possible
    const bool want_gpu = env ? (env[0] == '1') : (V >= 2048);
    if (want_gpu) {
      // integer codes of the candidate pairs on the GPU (edit distance, or Jaro-Winkler counts), identical double
      // arithmetic afterwards.  Levenshtein hands the kernel one byte symbol per code unit (an ASCII vocabulary: its
      // own bytes).
      const bool mapped = lev && !ascii;
      std::vector<std::string> symbols;
      std::vector<int> ci, cj, cc;
      if ((!mapped || lev_byte_symbols(units, off, symbols)) &&
          gpu_similarity_candidates(similarity, mapped ? symbols : ix->values, threshold, max_sim, ci, cj, cc)) {
        for (int r = 0; r < V; ++r) {  // the diagonal: distance 0; m = |v|, h = 0, l = min(4, |v|)
          const int code = similarity == DBL_SIM_JARO_WINKLER ? len[r] | std::min(4, len[r]) << 16 : 0;
          const double e =
              std::exp(host_similarity_from_unit(host_unit_from_code(similarity, code, len[r], len[r]), threshold, max_sim));
          if (e > 1.0) rows[r].emplace_back(r, e);
        }
        for (size_t k = 0; k < ci.size(); ++k) {
          const int i = ci[k], j = cj[k];
          const double e =
              std::exp(host_similarity_from_unit(host_unit_from_code(similarity, cc[k], len[i], len[j]), threshold, max_sim));
          if (e > 1.0) { rows[i].emplace_back(j, e); rows[j].emplace_back(i, e); }
        }
        for (int r = 0; r < V; ++r) std::sort(rows[r].begin(), rows[r].end());
        done = true;
        ix->pairs_on_device = true;
      }
    }
    if (!done) {
      std::atomic<int> next{0};
      auto work = [&]() {
        for (;;) {
          const int i = next.fetch_add(16);
          if (i >= V) break;
          for (int r = i; r < std::min(V, i + 16); ++r) {
            auto &row = rows[r];
            for (int c = 0; c < V; ++c) {
              const double u = lev ? host_levenshtein_unit_of(&units[off[r]], len[r], &units[off[c]], len[c])
                                   : host_jaro_winkler_unit_of(ix->values[r], ix->values[c]);
              const double e = std::exp(host_similarity_from_unit(u, threshold, max_sim));
              if (e > 1.0) row.emplace_back(c, e);
            }
          }
        }
      };
      unsigned nt = std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
      if (V < 512) nt = 1;
      std::vector<std::thread> th;
      for (unsigned t = 1; t < nt; ++t) th.emplace_back(work);
      work();
      for (auto &t : th) t.join();
    }
    for (int r = 0; r < V; ++r) ix->rowptr[r + 1] = ix->rowptr[r] + (int32_t)rows[r].size();
    ix->col.resize(ix->rowptr[V]);
    ix->expsim.resize(ix->rowptr[V]);
    for (int r = 0; r < V; ++r) {
      int p = ix->rowptr[r];
      for (auto &ce : rows[r]) { ix->col[p] = ce.first; ix->expsim[p] = ce.second; ++p; }
    }
  }
  ix->finish();
  *out = ix;
  return DBL_OK;
}

extern "C" int dbl_index_from_tables(dbl_index **out, int32_t V, int similarity, const double *probs,
                                     const int32_t *rowptr, const int32_t *col, const double *expsim, int32_t kmax) {
  if (!out || !probs || V <= 0 || kmax < 0) return DBL_ERR_INVALID;
  if (similarity < DBL_SIM_CONSTANT || similarity > DBL_SIM_JARO_WINKLER) return DBL_ERR_INVALID;
  auto *ix = new dbl_index();
  ix->V = V;
  ix->is_const = (similarity == DBL_SIM_CONSTANT);
  ix->kmax = kmax;
  ix->probs.assign(probs, probs + V);
  ix->rowptr.assign(V + 1, 0);
  if (!ix->is_const) {
    if (!rowptr || !col || !expsim) { delete ix; return DBL_ERR_INVALID; }
    ix->rowptr.assign(rowptr, rowptr + V + 1);
    ix->col.assign(col, col + rowptr[V]);
    ix->expsim.assign(expsim, expsim + rowptr[V]);
  }
  ix->finish();
  *out = ix;
  return DBL_OK;
}

extern "C" void dbl_index_free(dbl_index *ix) { delete ix; }
extern "C" int32_t dbl_index_num_values(const dbl_index *ix) { return ix ? ix->V : 0; }
extern "C" int32_t dbl_index_nnz(const dbl_index *ix) { return ix ? ix->rowptr[ix->V] : 0; }
extern "C" int32_t dbl_index_pairs_on_device(const dbl_index *ix) { return ix && ix->pairs_on_device ? 1 : 0; }
extern "C" int32_t dbl_index_value_id(const dbl_index *ix, const char *value) {
  if (!ix || !value || ix->values.empty()) return -1;
  auto it = std::lower_bound(ix->values.begin(), ix->values.end(), std::string(value));
  if (it == ix->values.end() || *it != value) return -1;
  return (int32_t)(it - ix->values.begin());
}
extern "C" const char *dbl_index_value(const dbl_index *ix, int32_t v) {
  if (!ix || v < 0 || v >= (int32_t)ix->values.size()) return nullptr;
  return ix->values[v].c_str();
}
extern "C" int dbl_index_tables(const dbl_index *ix, double *phi, double *norm, int32_t *rowptr, int32_t *col,
                                double *expsim) {
  if (!ix) return DBL_ERR_INVALID;
  if (phi) std::copy(ix->phi.begin(), ix->phi.end(), phi);
  if (norm) std::copy(ix->norm.begin(), ix->norm.end(), norm);
  if (rowptr) std::copy(ix->rowptr.begin(), ix->rowptr.end(), rowptr);
  if (col) std::copy(ix->col.begin(), ix->col.end(), col);
  if (expsim) std::copy(ix->expsim.begin(), ix->expsim.end(), expsim);
  return DBL_OK;
}
extern "C" int dbl_index_base_tables(const dbl_index *ix, int32_t *kmax, double *invnorm, double *logphi,
                                     double *lognorm, double *pk, double *cdf) {
  if (!ix) return DBL_ERR_INVALID;
  if (kmax) *kmax = ix->kmax;
  if (invnorm) std::copy(ix->invnorm.begin(), ix->invnorm.end(), invnorm);
  if (logphi) std::copy(ix->logphi.begin(), ix->logphi.end(), logphi);
  if (lognorm) std::copy(ix->lognorm.begin(), ix->lognorm.end(), lognorm);
  if (pk) std::copy(ix->pk.begin(), ix->pk.end(), pk);
  if (cdf) std::copy(ix->cdf.begin(), ix->cdf.end(), cdf);
  return DBL_OK;
}
extern "C" double dbl_index_exp_sim(const dbl_index *ix, int32_t v1, int32_t v2) {
  if (!ix || v1 < 0 || v2 < 0 || v1 >= ix->V || v2 >= ix->V)
    return std::numeric_limits<double>::quiet_NaN();  // reference: require(...) throws, AttributeIndex.scala:184
  if (ix->is_const) return 1.0;
  const auto b = ix->col.begin() + ix->rowptr[v1], e = ix->col.begin() + ix->rowptr[v1 + 1];
  const auto it = std::lower_bound(b, e, v2);
  return (it != e && *it == v2) ? ix->expsim[it - ix->col.begin()] : 1.0;  // getOrElse(valueId2, 1.0), :185
}
extern "C" double dbl_similarity(int similarity, const char *a, const char *b, double threshold, double max_sim) {
  if (similarity < DBL_SIM_CONSTANT || similarity > DBL_SIM_JARO_WINKLER) return std::numeric_limits<double>::quiet_NaN();
  if (similarity == DBL_SIM_CONSTANT) return 0.0;  // ConstantSimilarityFn, SimilarityFn.scala:50
  const std::string sa(a), sb(b);
  double unit;
  if (similarity == DBL_SIM_LEVENSHTEIN) {
    std::u16string ua, ub;
    if (!host_utf8_to_utf16(sa.data(), sa.size(), ua) || !host_utf8_to_utf16(sb.data(), sb.size(), ub))
      return std::numeric_limits<double>::quiet_NaN();
    unit = host_levenshtein_unit_of(ua.data(), (int)ua.size(), ub.data(), (int)ub.size());
  } else {
    unit = host_jaro_winkler_unit_of(sa, sb);
  }
  return host_similarity_from_unit(unit, threshold, max_sim);
}

// ---------------------------------------------------------------------------------------------------
// partitioning/KDTreePartitioner.scala:37-62,80-105; MutableBST.scala:51-111; DomainSplitter.scala:43-110
// ---------------------------------------------------------------------------------------------------
int32_t dbl_kdtree::leaf_node(const int32_t *yrow) const {
  int32_t node = 0;
  while (node < n_nodes && attr[node] >= 0) {
    const int32_t v = yrow[attr[node]];
    bool right;
    if (kind[node]) right = std::binary_search(set_val.begin() + set_ptr[node], set_val.begin() + set_ptr[node + 1], v);
    else right = v > split[node];
    node = right ? 2 * node + 2 : 2 * node + 1;
  }
  return node;
}

extern "C" int dbl_kdtree_fit(dbl_kdtree **out, const int32_t *y, int64_t E, int32_t A, int32_t num_levels,
                              const int32_t *attr_ids, int32_t n_attr_ids) {
  if (!out || num_levels < 0 || num_levels > 20 || A <= 0) return DBL_ERR_INVALID;
  if (num_levels > 0 && (!attr_ids || n_attr_ids <= 0 || !y)) return DBL_ERR_INVALID;  // KDTreePartitioner.scala:31
  for (int i = 0; i < n_attr_ids; ++i)
    if (attr_ids[i] < 0 || attr_ids[i] >= A) return DBL_ERR_INVALID;
  auto *t = new dbl_kdtree();
  const int n = (1 << (num_levels + 1)) - 1;
  t->n_nodes = n;
  t->attr.assign(n, -1);
  t->kind.assign(n, 0);
  t->split.assign(n, 0);
  t->leaf_no.assign(n, -1);
  t->leaf_no[0] = 0;
  t->n_leaves = 1;
  std::vector<std::vector<int32_t>> sets(n);
  std::vector<int32_t> node_of((size_t)std::max<int64_t>(E, 1));
  for (int level = 0; level < num_levels; ++level) {
    const int attr = attr_ids[level % n_attr_ids];  // cycle, KDTreePartitioner.scala:45-49
    // value histogram per frontier node (getNewSplits, :80-105)
    std::map<int32_t, std::map<int32_t, double>> dom;
    auto leaf_during_fit = [&](const int32_t *yrow) {  // set_ptr/set_val are only assembled after the last level
      int32_t node = 0;
      while (node < n && t->attr[node] >= 0) {
        const int32_t v = yrow[t->attr[node]];
        const bool right = t->kind[node] ? std::binary_search(sets[node].begin(), sets[node].end(), v)
                                         : (v > t->split[node]);
        node = right ? 2 * node + 2 : 2 * node + 1;
      }
      return node;
    };
    for (int64_t e = 0; e < E; ++e) dom[leaf_during_fit(y + e * A)][y[e * A + attr]] += 1.0;
    for (auto &nd : dom) {  // ascending node id (the reference's Map order is unspecified)
      const int32_t node = nd.first;
      std::vector<std::pair<int32_t, double>> d(nd.second.begin(), nd.second.end());  // ascending value
      double half = 0.0;
      for (auto &vw : d) half += vw.second;
      half = half / 2.0;
      if (d.size() <= 30) {  // LPTDomainSplitter, DomainSplitter.scala:86-110
        std::stable_sort(d.begin(), d.end(), [](auto &p, auto &q) { return p.second > q.second; });
        double left = 0.0, right = 0.0;
        for (auto &vw : d) {
          if (left >= right) { sets[node].push_back(vw.first); right += vw.second; }
          else left += vw.second;
        }
        std::sort(sets[node].begin(), sets[node].end());
        t->kind[node] = 1;
      } else {  // RanDomainSplitter, DomainSplitter.scala:57-75
        double cum = 0.0;
        size_t i = 0;
        while (cum <= half && i < d.size() - 1) { cum += d[i].second; ++i; }
        t->kind[node] = 0;
        t->split[node] = d[i].first;
      }
      t->attr[node] = attr;  // MutableBST.splitNode, MutableBST.scala:87-111
      t->leaf_no[2 * node + 1] = t->leaf_no[node];
      t->leaf_no[2 * node + 2] = t->n_leaves++;
    }
  }
  t->set_ptr.assign(n + 1, 0);
  for (int i = 0; i < n; ++i) {
    t->set_ptr[i + 1] = t->set_ptr[i] + (int32_t)sets[i].size();
    t->set_val.insert(t->set_val.end(), sets[i].begin(), sets[i].end());
  }
  *out = t;
  return DBL_OK;
}

extern "C" int dbl_kdtree_from_arrays(dbl_kdtree **out, int32_t n, const int32_t *attr, const int32_t *kind,
                                      const int32_t *split, const int32_t *set_ptr, const int32_t *set_val,
                                      const int32_t *leaf_no) {
  if (!out || n <= 0 || !attr || !kind || !split || !set_ptr || !leaf_no) return DBL_ERR_INVALID;
  auto *t = new dbl_kdtree();
  t->n_nodes = n;
  t->attr.assign(attr, attr + n);
  t->kind.assign(kind, kind + n);
  t->split.assign(split, split + n);
  t->set_ptr.assign(set_ptr, set_ptr + n + 1);
  if (set_ptr[n] > 0) t->set_val.assign(set_val, set_val + set_ptr[n]);
  t->leaf_no.assign(leaf_no, leaf_no + n);
  int nl = 0;
  for (int i = 0; i < n; ++i)
    if (attr[i] < 0 && leaf_no[i] + 1 > nl) nl = leaf_no[i] + 1;
  t->n_leaves = nl;
  *out = t;
  return DBL_OK;
}
extern "C" void dbl_kdtree_free(dbl_kdtree *t) { delete t; }
extern "C" int32_t dbl_kdtree_num_nodes(const dbl_kdtree *t) { return t ? t->n_nodes : 0; }
extern "C" int32_t dbl_kdtree_num_leaves(const dbl_kdtree *t) { return t ? t->n_leaves : 1; }
extern "C" int32_t dbl_kdtree_set_len(const dbl_kdtree *t) { return t ? (int32_t)t->set_val.size() : 0; }
extern "C" int dbl_kdtree_export(const dbl_kdtree *t, int32_t *attr, int32_t *kind, int32_t *split, int32_t *set_ptr,
                                 int32_t *set_val, int32_t *leaf_no) {
  if (!t) return DBL_ERR_INVALID;
  if (attr) std::copy(t->attr.begin(), t->attr.end(), attr);
  if (kind) std::copy(t->kind.begin(), t->kind.end(), kind);
  if (split) std::copy(t->split.begin(), t->split.end(), split);
  if (set_ptr) std::copy(t->set_ptr.begin(), t->set_ptr.end(), set_ptr);
  if (set_val) std::copy(t->set_val.begin(), t->set_val.end(), set_val);
  if (leaf_no) std::copy(t->leaf_no.begin(), t->leaf_no.end(), leaf_no);
  return DBL_OK;
}
extern "C" int32_t dbl_kdtree_partition_id(const dbl_kdtree *t, const int32_t *yrow) {
  if (!t) return 0;
  return t->leaf_no[t->leaf_node(yrow)];  // MutableBST.getLeafNumber, MutableBST.scala:51-54
}

// ---------------------------------------------------------------------------------------------------
// updateDistProbs, GU:305-320 on the host (used by the host-mediated exchange path and by tests); the sweep itself
// draws theta on the device with the same function (draw_theta_one, dbl_internal.h).
// ---------------------------------------------------------------------------------------------------
void host_draw_theta(int A, int F, const double *alpha, const double *beta, uint64_t seed, const int64_t *agg_dist,
                     const int64_t *file_sizes, uint32_t iter, double *theta_out) {
  for (int a = 0; a < A; ++a)
    for (int f = 0; f < F; ++f)
      theta_out[a * F + f] = draw_theta_one(seed, iter, (uint32_t)(a * F + f), alpha[a], beta[a],
                                            (double)agg_dist[a * F + f], (double)file_sizes[f]);
}

extern "C" double dbl_det_log(double x) { return det_log(x); }
extern "C" double dbl_det_exp(double x) { return det_exp(x); }
extern "C" int dbl_draw_theta(int32_t A, int32_t F, const double *alpha, const double *beta, uint64_t seed,
                              const int64_t *agg_dist, const int64_t *file_sizes, int64_t iteration, double *theta_out) {
  if (A <= 0 || F <= 0 || !alpha || !beta || !agg_dist || !file_sizes || !theta_out) return DBL_ERR_INVALID;
  host_draw_theta(A, F, alpha, beta, seed, agg_dist, file_sizes, (uint32_t)iteration, theta_out);
  return DBL_OK;
}

extern "C" int32_t dbl_index_hash_slots(const dbl_index *ix) { return ix ? ix->hsize : 0; }
extern "C" int dbl_index_slot_codes(const dbl_index *ix, int32_t *out) {
  if (!ix || !out) return DBL_ERR_INVALID;
  if (ix->pcode.empty()) return DBL_ERR_STATE;
  std::copy(ix->pcode.begin(), ix->pcode.end(), out);
  return DBL_OK;
}
