// k_link_pcg2<A, NS, HC, PK>: the PCG-II link update (updateEntityIdCollapsed, GU:363-395) with everything about
// the model shape known at compile time: A attributes in kernel order, the last NS of them non-constant; HC = 32
// when the hash tables have 32 slots (else the size is a run-time parameter); PK = the constant attributes arrive
// byte-packed.
//
//  * persistent CTAs: the grid is a few CTAs per SM; each takes the next group of LINK_WARPS records of some block
//    from a device-side counter until none is left (no empty CTAs on a shard that owns 1/8 of the records, no tail);
//  * the block's entity table streams through shared memory in TE-entity "quad tiles" moved by TMA bulk copies
//    (cp.async.bulk.shared::cluster.global + mbarrier ring, one producer warp per CTA); a quad tile keeps the words
//    of one entity in groups of four, so a lane fetches everything it needs about its candidate with QW/4 128-bit
//    shared-memory loads (3 for 6 non-constant attributes + packed constants + N) instead of one load per word;
//  * each consumer warp owns one record; its constants (value ids, hash multipliers) are registers;
//  * constant attributes: the product of the exact-match multipliers comes from a 16-entry per-record table indexed
//    by the byte-wise match mask of the packed values (PK), else from per-attribute compares;
//  * non-constant attributes: ONE probe per (candidate, attribute) of a 32-slot perfect-hash table in shared memory
//    (one key word per bank = one conflict-free wavefront) that holds the record's similarity row INCLUDING the
//    record's own value, whose entry carries the exact-match multiplier of protocol 4.1 -- so "equal" and "similar"
//    are the same look-up and the multiply is skipped warp-wide by one vote per step when nobody hit (the usual case);
//  * lane l scores candidate 32*step + l; lane sums / chunk totals / draw as in DESIGN.md section 4.
#pragma once
#include <type_traits>

#include "dbl_link.cuh"

// Per (record, non-constant attribute): H key words then H f64 values, H = p.hslots (a power of two >= 32, the same
// for every attribute of the model; 32 = one key per bank = conflict-free probes).
__device__ __host__ __forceinline__ int pcg2_tab_bytes(int H) { return H * 12; }

// w *= r when y == x (shapes without the packed-constant table; ptxas turns any predicated form into DMUL + 2 FSEL)
__device__ __forceinline__ void mul_if_eq(double &w, int y, int x, double r) {
  if (y == x) w = w * r;
}

template <int A, int NS>
struct Pcg2Rec {
  int x[A];                      // record value id; -1 = missing (never equals an entity value)
  double rm[A];                  // multiplier on an exact match
  unsigned hm[NS > 0 ? NS : 1];  // hash multipliers of the non-constant attributes
  unsigned mmask;                // missing non-constant attributes (bit = kernel position)
  unsigned xpack;                // PK: the record's constant-attribute values, one byte each (0xFF = cannot match)
};

// PK kernels: index into the record's table of constant-attribute products from the byte-packed values of a
// candidate: bit k of the index = (byte k of ypack == byte k of xpack)
__device__ __forceinline__ unsigned pcg2_const_index(unsigned ypack, unsigned xpack) {
  const unsigned d = ypack ^ xpack;
  const unsigned nz = ((d & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | d;  // bit 7 of a byte set <=> the byte of d is non-zero
  const unsigned eq = (~nz & 0x80808080u) >> 7;               // bit 8k set <=> byte k equal
  return (eq * 0x01020408u) >> 24;                            // gathers bits 0, 8, 16, 24 into bits 0..3
}

// one candidate out of a quad tile: values in kernel order (PK: only the non-constant ones + the packed word), N
template <int A, int NS, bool PK>
struct Pcg2Cand {
  int y[A];
  unsigned ypack;
  double N;
};
template <int A, int NS, bool PK>
__device__ __forceinline__ void pcg2_load(Pcg2Cand<A, NS, PK> &c, const int *tile, int slot) {
  constexpr int NV = qtile_nv(A, NS, PK), NG = qtile_groups(NV);
  int v[NG * 4];
  const int4 *q = reinterpret_cast<const int4 *>(tile);
#pragma unroll
  for (int g = 0; g < NG; ++g) {
    const int4 t = q[g * TE + slot];
    v[4 * g] = t.x; v[4 * g + 1] = t.y; v[4 * g + 2] = t.z; v[4 * g + 3] = t.w;
  }
  if constexpr (PK) {
#pragma unroll
    for (int q2 = 0; q2 < NS; ++q2) c.y[A - NS + q2] = v[q2];
    c.ypack = (unsigned)v[NS];
  } else {
#pragma unroll
    for (int k = 0; k < A; ++k) c.y[k] = v[k];
    c.ypack = 0u;
  }
  c.N = reinterpret_cast<const double *>(tile + NG * 4 * TE)[slot];
}

// With skewed (Zipf-like) value frequencies some lane of the warp finds an equal or similar value on almost every
// step (96 % at BASELINE's 1M configuration), so a warp-wide vote that skips the multiplies does not pay: the
// multiplies are predicated per lane and the compiler is free to overlap them with the next step's loads.
// DBL_PCG2_VOTE=1 brings the vote back (CONVERGED = every lane of the warp executes the call, i.e. the main loop).
#ifndef DBL_PCG2_VOTE
#define DBL_PCG2_VOTE 0
#endif
// PK kernels: 1 = the product of the matching constant attributes comes from the record's 16-entry table in shared
// memory (index from a SWAR byte compare), 0 = predicated multiplies
#ifndef DBL_PCG2_CTAB
#define DBL_PCG2_CTAB 1
#endif
template <int A, int NS, int HC, bool CONVERGED, bool PK, bool MISSING = true>
__device__ __forceinline__ double pcg2_weight(const Pcg2Rec<A, NS> &rc, const LinkParams &p, const char *tab,
                                              const double *ctab, const Pcg2Cand<A, NS, PK> &cd) {
  const int hslots = HC ? HC : p.hslots;
  const int hshift = HC ? 27 : p.hshift;
  const int tabb = pcg2_tab_bytes(hslots);
  const int *y = cd.y;
  double w = cd.N;
  if constexpr (NS < A) {  // protocol 4.1: the constant attributes form their own product c; w = N * c
    double c = 1.0;
    if constexpr (PK) {
#if DBL_PCG2_CTAB
      c = ctab[pcg2_const_index(cd.ypack, rc.xpack)];
#else
      // the same product, multiplied out: byte k of d is zero <=> constant attribute k matches (a missing record
      // value is 0xFF and matches nothing); no table look-up, i.e. two shared-memory wavefronts less per candidate
      const unsigned d = cd.ypack ^ rc.xpack;
#pragma unroll
      for (int k = 0; k < A - NS; ++k)
        if ((d & (0xFFu << (8 * k))) == 0u) c = c * rc.rm[k];
#endif
    } else {
#pragma unroll
      for (int k = 0; k < A - NS; ++k) mul_if_eq(c, y[k], rc.x[k], rc.rm[k]);
    }
    w = w * c;
  }
  // protocol 4.1: non-constant attributes in kernel order, each contributes at most one factor: the exact-match
  // multiplier when y == x, exp(similarity) when y is similar to x -- both sit in the record's hash table
  if (CONVERGED && DBL_PCG2_VOTE) {
    bool hit[NS > 0 ? NS : 1];
    bool any = false;
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int yv = y[A - NS + q];
      const unsigned slot = ((unsigned)yv * rc.hm[q]) >> hshift;
      hit[q] = (reinterpret_cast<const int *>(tab + q * tabb)[slot] == yv);
      any = any || hit[q];
    }
    if (NS > 0 && __any_sync(FULL, any)) {
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        if (hit[q]) {
          const unsigned slot = ((unsigned)y[A - NS + q] * rc.hm[q]) >> hshift;
          w = w * reinterpret_cast<const double *>(tab + q * tabb + hslots * 4)[slot];
        }
      }
    }
  } else {
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int yv = y[A - NS + q];
      const unsigned slot = ((unsigned)yv * rc.hm[q]) >> hshift;
      if (reinterpret_cast<const int *>(tab + q * tabb)[slot] == yv)
        w = w * reinterpret_cast<const double *>(tab + q * tabb + hslots * 4)[slot];
    }
  }
  if (MISSING && rc.mmask) {
#pragma unroll
    for (int q = 0; q < NS; ++q)
      if ((rc.mmask >> (A - NS + q)) & 1u) w = w * p.attrs[p.perm[A - NS + q]].invnorm[y[A - NS + q]];
  }
  return w;
}

#ifndef DBL_PCG2_CTAS_PER_SM
#define DBL_PCG2_CTAS_PER_SM 3
#endif

// Records per consumer warp.  With 2, a lane fetches its candidate once and scores it for both records: half the
// tile loads and half the tile traffic through shared memory per (record, candidate) pair, two independent
// dependency chains per warp; the price is registers (96 instead of 72: 2 CTAs per SM instead of 3) and twice the
// per-record tables in shared memory -- so it is used for the 32-slot instantiations with up to 8 non-constant
// attributes (faster at A = 10, NS = 6; three records per warp spill).
#ifndef DBL_PCG2_RPW_MAX
#define DBL_PCG2_RPW_MAX 2
#endif
__host__ __device__ constexpr int pcg2_rpw(int HC, int NS) { return (HC == 32 && NS >= 1 && NS <= 8) ? DBL_PCG2_RPW_MAX : 1; }
// Consumer warps per CTA of the two-record shapes.  Every 32-byte sector a bulk copy lands in shared memory costs
// the L1 data pipe about two wavefronts, so more records per staged tile should help -- but ONE CTA of 16 consumer
// warps per SM was slower than two CTAs of 8 (one ring per SM: every warp waits for the slowest at each stage), so 8
// it stays.
#ifndef DBL_PCG2_WARPS2
#define DBL_PCG2_WARPS2 8
#endif
__host__ __device__ constexpr int pcg2_warps(int HC, int NS) { return pcg2_rpw(HC, NS) >= 2 ? DBL_PCG2_WARPS2 : LINK_WARPS; }
// 3 CTAs per SM (72 registers) only where one record per warp fits them: few non-constant attributes
__host__ __device__ constexpr int pcg2_ctas_per_sm(int HC, int NS) {
#ifdef DBL_PCG2_CTAS2
  return pcg2_rpw(HC, NS) >= 2 ? DBL_PCG2_CTAS2 : (NS > 6 ? 2 : DBL_PCG2_CTAS_PER_SM);
#else
  return pcg2_rpw(HC, NS) >= 2 ? (pcg2_warps(HC, NS) > 8 ? 1 : 2) : (NS > 6 ? 2 : DBL_PCG2_CTAS_PER_SM);
#endif
}

template <int A, int NS, int HC, bool PK>
__global__ void __launch_bounds__((pcg2_warps(HC, NS) + 1) * 32, pcg2_ctas_per_sm(HC, NS)) k_link_pcg2(LinkParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ int s_cta;
  if (sweep_dead(p.ctl)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr int NV = qtile_nv(A, NS, PK);
  constexpr int TW = qtile_words(NV) * TE;
  constexpr int NC = A - NS;
  constexpr int RPW = pcg2_rpw(HC, NS);
  constexpr int WARPS = pcg2_warps(HC, NS);   // consumer warps; warp WARPS is the producer
  constexpr int PCG2_RECS = WARPS * RPW;      // records per work item (= per "CTA" of cta_ptr)
  TileRing rg;
  rg.tiles = reinterpret_cast<int *>(smem);
  rg.full = reinterpret_cast<uint64_t *>(smem + (size_t)LINK_STAGES * TW * 4);
  rg.empty = rg.full + LINK_STAGES;
  rg.tw = TW;
  static_assert(2 * LINK_STAGES * 8 <= 128, "barrier area");
  const int tabrec = (NS > 0 ? NS : 1) * pcg2_tab_bytes(HC ? HC : p.hslots);  // bytes of one record's hash tables
  char *tab0 = reinterpret_cast<char *>(smem) + (size_t)LINK_STAGES * TW * 4 + 128 + (size_t)warp * RPW * tabrec;
  // PK: products of the matching constant attributes, by match mask, 16 entries per record
  double *ctab0 = reinterpret_cast<double *>(reinterpret_cast<char *>(smem) + (size_t)LINK_STAGES * TW * 4 + 128 +
                                            (size_t)PCG2_RECS * tabrec) + warp * RPW * 16;
#ifndef DBL_PCG2_LDGSTS
#define DBL_PCG2_LDGSTS 0
#endif
  ring_init(rg, WARPS, DBL_PCG2_LDGSTS ? 32 : 1);
  const int total_ctas = p.cta_ptr[p.P];
  int tbase = 0;  // tiles this CTA has streamed so far: stage and phase of the ring continue across work items

  for (;;) {
    if (threadIdx.x == 0) s_cta = (int)atomicAdd(p.work, 1ull);
    __syncthreads();
    const int cta = s_cta;
    __syncthreads();
    if (cta >= total_ctas) break;
    const int b = find_block(p, cta);
    const int n = p.ent_ptr[b + 1] - p.ent_ptr[b];
    const int ntiles = p.tile_ptr[b + 1] - p.tile_ptr[b];
    const int *gtiles = p.qtiles + (size_t)p.tile_ptr[b] * TW;

    if (warp == WARPS) {  // producer warp
#if DBL_PCG2_LDGSTS
      ring_produce_ldgsts(rg, gtiles, ntiles, tbase, lane);
#else
      if (lane == 0) ring_produce<true>(rg, gtiles, ntiles, tbase);
#endif
      tbase += ntiles;
      continue;
    }

    // ---- per-record constants: lane k prepares kernel-order attribute k, then everything is broadcast
    Pcg2Rec<A, NS> rc[RPW];
    int rr[RPW];
    bool act[RPW];
#pragma unroll
    for (int ri = 0; ri < RPW; ++ri) {
      const int ridx = p.rec_ptr[b] + (cta - p.cta_ptr[b]) * PCG2_RECS + warp * RPW + ri;
      act[ri] = ridx < p.rec_ptr[b + 1];
      rr[ri] = act[ri] ? p.rec_sorted[ridx] : -1;
      const int r = rr[ri];
      char *tab = tab0 + ri * tabrec;
      double *ctab = ctab0 + ri * 16;
      int xv = -1;
      double rmv = 1.0;
      unsigned hmv = 0;
      bool is_m = false;
      if (act[ri] && lane < A) {
        const int a = p.perm[lane];
        const AttrDev &at = p.attrs[a];
        xv = p.x[(int64_t)r * A + a];
        if (xv < 0) {
          is_m = !at.is_const;
        } else {
          const double th = p.theta[a * p.F + p.file[r]];
          double d = th * at.phi[xv];
          if (at.is_const) {
            rmv = 1.0 + (1.0 - th) / d;
          } else {
            d = d * at.norm[xv];
            rmv = at.diag[xv] + (1.0 - th) / d;
            hmv = at.hmult[xv];
          }
        }
      }
      rmv = (rmv - 1.0) + 1.0;  // protocol: the multiplier is defined through (r - 1) (identity below ~2^53)
      rc[ri].mmask = __ballot_sync(FULL, is_m);
#pragma unroll
      for (int k = 0; k < A; ++k) {
        rc[ri].x[k] = __shfl_sync(FULL, xv, k);
        rc[ri].rm[k] = shfl_d(rmv, k);
      }
#pragma unroll
      for (int q = 0; q < NS; ++q) rc[ri].hm[q] = __shfl_sync(FULL, hmv, A - NS + q);
      // hash tables of the record's similarity rows -> shared memory (all-empty table when the value is missing);
      // the entry of the record's own value gets the exact-match multiplier (it depends on theta of the record's file)
      const int H = HC ? HC : p.hslots;
      const int hshift = HC ? 27 : p.hshift;
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const AttrDev &at = p.attrs[p.perm[A - NS + q]];
        int *kd = reinterpret_cast<int *>(tab + q * pcg2_tab_bytes(H));
        double *vd = reinterpret_cast<double *>(tab + q * pcg2_tab_bytes(H) + H * 4);
        const int xq = rc[ri].x[A - NS + q];
        const unsigned own = (xq >= 0) ? (((unsigned)xq * rc[ri].hm[q]) >> hshift) : 0xFFFFFFFFu;
        for (int i = lane; i < H; i += 32) {
          kd[i] = (xq >= 0) ? at.hkeys[(size_t)xq * H + i] : -1;
          vd[i] = ((unsigned)i == own) ? rc[ri].rm[A - NS + q] : ((xq >= 0) ? at.hvals[(size_t)xq * H + i] : 1.0);
        }
      }
      rc[ri].xpack = 0xFFFFFFFFu;
      if constexpr (PK) {
        static_assert(!PK || (NC >= 1 && NC <= 4), "PK packs 1..4 constant attributes");
#pragma unroll
        for (int k = 0; k < NC; ++k)
          rc[ri].xpack = (rc[ri].xpack & ~(0xFFu << (8 * k))) |
                         ((unsigned)(rc[ri].x[k] < 0 ? 0xFF : rc[ri].x[k]) << (8 * k));
        if (lane < 16) {
          double c = 1.0;
#pragma unroll
          for (int k = 0; k < NC; ++k)
            if ((lane >> k) & 1) c = c * rc[ri].rm[k];
          ctab[lane] = c;
        }
      }
    }
    __syncwarp();

    const int nsteps = ntiles * (TE / 32);          // steps beyond the last candidate add zeros
    const int tpc = max(1, (ntiles + 31) >> 5);     // a chunk is a whole number of tiles
    const int spc = (TE / 32) * tpc;
    const int nchunks = (nsteps + spc - 1) / spc;

    // ---- pass 1 over the TMA-staged tiles.  Records without a missing non-constant attribute (most of them) take a
    // loop body without the gather of 1/n(y): straight-line code the compiler can overlap across the steps of a tile
    double run[RPW], Q[RPW], acc[RPW];
    unsigned any_missing = 0;
#pragma unroll
    for (int ri = 0; ri < RPW; ++ri) { run[ri] = 0.0; Q[ri] = 0.0; acc[ri] = 0.0; any_missing |= rc[ri].mmask; }
    int chunk = 0, tile_in_chunk = 0;
    double *my_sums = p.lane_sums + ((size_t)blockIdx.x * WARPS + warp) * RPW * 1024;  // [record][chunk][lane]
    auto pass1 = [&](auto missing_tag) {
      constexpr bool MISSING = decltype(missing_tag)::value;
      for (int t = 0; t < ntiles; ++t) {
        const int g = tbase + t;
        const int s = g % LINK_STAGES;
        mbar_wait(&rg.full[s], (g / LINK_STAGES) & 1);
        if (act[0]) {  // (the second record of a warp is only there when the first is)
          const int *tile = rg.tiles + (size_t)s * TW;
#pragma unroll
          for (int q = 0; q < TE / 32; ++q) {
            Pcg2Cand<A, NS, PK> cd;
            pcg2_load<A, NS, PK>(cd, tile, q * 32 + lane);
#pragma unroll
            for (int ri = 0; ri < RPW; ++ri)
              acc[ri] = acc[ri] + pcg2_weight<A, NS, HC, true, PK, MISSING>(rc[ri], p, tab0 + ri * tabrec,
                                                                          ctab0 + ri * 16, cd);
          }
          if (++tile_in_chunk == tpc || t + 1 == ntiles) {
#pragma unroll
            for (int ri = 0; ri < RPW; ++ri) {
              my_sums[ri * 1024 + chunk * 32 + lane] = acc[ri];  // pass 2 reads the chosen chunk's sums back
              run[ri] = run[ri] + butterfly_sum(acc[ri]);
              if (lane == chunk) Q[ri] = run[ri];
              acc[ri] = 0.0;
            }
            ++chunk;
            tile_in_chunk = 0;
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&rg.empty[s]);
      }
    };
    if (any_missing) pass1(std::true_type{}); else pass1(std::false_type{});
    tbase += ntiles;

    // ---- pass 2 from the L2-resident copy of the tiles, one record after the other
#pragma unroll
    for (int ri = 0; ri < RPW; ++ri) {
      if (!act[ri]) continue;
      const int r = rr[ri];
      store_mass(p, lane, r, run[ri]);
      if (!(run[ri] > 0.0) || isinf(run[ri])) { fail_link(p, lane, r); continue; }
      auto wf = [&](int j) -> double {
        if (j >= n) return 0.0;
        Pcg2Cand<A, NS, PK> cd;
        pcg2_load<A, NS, PK>(cd, gtiles + (size_t)(j / TE) * TW, j % TE);
        return pcg2_weight<A, NS, HC, false, PK>(rc[ri], p, tab0 + ri * tabrec, ctab0 + ri * 16, cd);
      };
      const U2 u = uniform2(p.seed, PH_LINK, link_iter(p), (uint32_t)r, 0u);
      const int j = finish_draw(lane, n, nsteps, spc, nchunks, Q[ri], run[ri], u.u0, wf, my_sums + ri * 1024);
      store_link(p, lane, r, b, n, j);
    }
  }
}

inline size_t pcg2_smem_bytes(int A, int NS, int H, bool PK) {
  const size_t recs = (size_t)pcg2_warps(H == 32 ? 32 : 0, NS) * pcg2_rpw(H == 32 ? 32 : 0, NS);
  return (size_t)LINK_STAGES * qtile_words(qtile_nv(A, NS, PK)) * TE * 4 + 128 +
         recs * (NS > 0 ? NS : 1) * pcg2_tab_bytes(H) + recs * 16 * sizeof(double);
}

// launch k_link_pcg2<A, NS, HC> for a runtime NS in [0, A]; HC = 32 (compile-time table size) when the model's
// tables have 32 slots, else 0 (size read from the parameters); returns cudaError_t as int
template <int A, int NS, int HC, bool PK>
int pcg2_launch_one(int grid, cudaStream_t stream, const LinkParams &lp, size_t *configured) {
  const size_t smem = pcg2_smem_bytes(A, NS, lp.hslots, PK);
  // the opt-in is per device: the cache belongs to the context (one model shape = one instantiation per context)
  if (*configured < smem) {
    cudaError_t e = cudaFuncSetAttribute(k_link_pcg2<A, NS, HC, PK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    *configured = smem;
  }
  if (grid <= 0) {  // load the kernel without running it (see preload_kernels in dbl_engine.cu)
    cudaFuncAttributes fa;
    return (int)cudaFuncGetAttributes(&fa, k_link_pcg2<A, NS, HC, PK>);
  }
  k_link_pcg2<A, NS, HC, PK><<<grid, (pcg2_warps(HC, NS) + 1) * 32, smem, stream>>>(lp);
  return (int)cudaGetLastError();
}

template <int A, int NS>
struct Pcg2Launch {
  static int go(int ns, int grid, cudaStream_t stream, const LinkParams &lp, size_t *cfg) {
    if (ns == NS) {
      // byte-packed constant attributes: 1..4 of them, every vocabulary <= 255, 32-slot tables (lp.qtile_pk)
      if constexpr (A - NS >= 1 && A - NS <= 4) {
        if (lp.qtile_pk) return pcg2_launch_one<A, NS, 32, true>(grid, stream, lp, cfg);
      }
      return lp.hslots == 32 ? pcg2_launch_one<A, NS, 32, false>(grid, stream, lp, cfg)
                             : pcg2_launch_one<A, NS, 0, false>(grid, stream, lp, cfg);
    }
    if constexpr (NS > 0) return Pcg2Launch<A, NS - 1>::go(ns, grid, stream, lp, cfg);
    return (int)cudaErrorInvalidValue;
  }
};
