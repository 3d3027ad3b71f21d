// k_link_pcg2<A, NS, HC, PK, ID16, SC>: the PCG-II link update (updateEntityIdCollapsed, GU:363-395) with everything
// about the model shape known at compile time: A attributes in kernel order, the last NS of them non-constant; HC = 32
// when the hash tables have 32 slots (else the size is a run-time parameter); PK = the constant attributes arrive
// byte-packed; ID16 (PK only) = the non-constant values arrive as 16-bit halves, two per word (every non-constant
// value, or SC code, is < 65536); SC (PK only) = those values are slot codes (AttrDev::pcode, dbl_index::
// build_slot_codes) whose low five bits are the value's slot in every record's table.  HC, PK, ID16 and SC are one
// Pcg2Format, which pcg2_format decides once per model; the tiles, the launch and dbl_link_kernel's report follow it.
//
//  * persistent CTAs: the grid is a few CTAs per SM; each takes the next group of LINK_WARPS records of some block
//    from a device-side counter until none is left (no empty CTAs on a shard that owns 1/8 of the records, no tail);
//  * the block's entity table streams through shared memory in TE-entity "quad tiles" moved by TMA bulk copies
//    (cp.async.bulk.shared::cluster.global + mbarrier ring, one producer warp per CTA); a quad tile keeps the words
//    of one entity in groups of four, so a lane fetches everything it needs about its candidate with 128-bit
//    shared-memory loads instead of one load per word: at 6 non-constant attributes + packed constants, ONE LDS.128
//    (ID16: 3 words of values + the packed word) and the LDS.64 of N = 6 wavefronts per warp-step, against two
//    LDS.128 + N = 10 with 32-bit values; the unpacking costs one LOP3 or SHF per value (6 per candidate, shared by
//    the warp's two records; one PRMT per value with paired tables);
//  * each consumer warp owns one record (two in the 32-slot shapes); its constants (value ids, hash multipliers
//    unless SC) are registers;
//  * constant attributes: the product of the exact-match multipliers comes from a 16-entry per-record table indexed
//    by the byte-wise match mask of the packed values (PK), else from per-attribute compares;
//  * non-constant attributes: ONE probe per (candidate, attribute) of a 32-slot perfect-hash table in shared memory
//    (one key word per bank = one conflict-free wavefront) that holds the record's similarity row INCLUDING the
//    record's own value, whose entry carries the exact-match multiplier of protocol 4.1 -- so "equal" and "similar"
//    are the same look-up, and a lane multiplies only where it hit (predicated, no warp vote); with SC the slot is
//    code & 31, computed once per (candidate, attribute) for both records of the warp (no per-record multiplier);
//    with ID16 and SC the two records' tables are paired (PAIR_KEYS): one key word holds both records' 16-bit keys
//    of a slot, so one key load and one value address serve both records;
//  * records with a missing non-constant value multiply by 1/n(y) of that attribute (their probe never hits): the
//    1/n(y) of
//    every tile entity travel with the tiles (LinkParams::tile_invn, one f64 column of TE per non-constant
//    attribute), and the producer stages the columns its work item's records miss in the same ring stage as the
//    tile, so that no pass-1 loop reads global memory;
//  * lane l scores candidate 32*step + l; lane sums / chunk totals / draw as in DESIGN.md section 4.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "dbl_link.cuh"

// The tile format {HC, PK, ID16, SC} of k_link_pcg2 and what follows from it (A attributes, NS non-constant)
struct Pcg2Format {
  int hc;              // 32: the model's hash tables have 32 slots, a compile-time size; 0: p.hslots
  __host__ __device__ static constexpr int hc_of(int hslots) { return hslots == 32 ? 32 : 0; }
  bool pk, id16, sc;   // byte-packed constants; 16-bit non-constant values; slot codes in place of value ids
  // Words of an entity in the tiles (TileLayout): pk: the NS non-constant values then the byte-packed constants;
  // else all A values in kernel order.  id16: the NS values are 16-bit, two per word (value 2i in the low half of
  // word i), so A = 10 with 6 non-constant attributes needs one group instead of two.  pcg2_store writes them,
  // pcg2_load reads them.
  __host__ __device__ constexpr int nv(int A, int NS) const { return pk ? (id16 ? (NS + 1) / 2 : NS) + 1 : A; }
  __host__ __device__ constexpr TileLayout layout(int A, int NS) const { return TileLayout::of(nv(A, NS)); }
  __host__ __device__ constexpr bool operator==(Pcg2Format o) const {
    return hc == o.hc && pk == o.pk && id16 == o.id16 && sc == o.sc;
  }
  // Records per consumer warp.  With 2, a lane fetches its candidate once and scores it for both records: half the
  // tile loads and half the tile traffic through shared memory per (record, candidate) pair, two independent
  // dependency chains per warp; the price is registers (96 instead of 72: 2 CTAs per SM instead of 3) and twice the
  // per-record tables in shared memory -- so it is used for the 32-slot instantiations with up to 8 non-constant
  // attributes (faster at A = 10, NS = 6; three records per warp spill).  Every shape has LINK_WARPS consumer warps:
  // ONE CTA of 16 consumer warps per SM was slower than two CTAs of 8 (one ring per SM: every warp waits for the
  // slowest at each stage).
  __host__ __device__ constexpr int rpw(int NS) const { return (hc == 32 && NS >= 1 && NS <= 8) ? 2 : 1; }
  // 3 CTAs per SM (72 registers) only where one record per warp fits them: few non-constant attributes
  __host__ __device__ constexpr int ctas_per_sm(int NS) const { return (rpw(NS) >= 2 || NS > 6) ? 2 : 3; }
  // the two records of a warp share paired key tables (PAIR_KEYS) when every code fits 16 bits
  __host__ __device__ constexpr bool paired(int NS) const { return id16 && sc && rpw(NS) == 2; }
  // as dbl_link_kernel reports it: +4 pk, +8 hc = 32, +16 id16, +32 sc, +64 paired, +128 two records per warp
  constexpr int bits(int NS) const {
    return (pk ? 4 : 0) + (hc == 32 ? 8 : 0) + (id16 ? 16 : 0) + (sc ? 32 : 0) + (paired(NS) ? 64 : 0) +
           (rpw(NS) == 2 ? 128 : 0);
  }
};

// The tile format of a model, the one place its rules live.  hslots: the model's common hash-table size (0: none).
// DBL_NO_PACK, DBL_NO_SC and DBL_NO_ID16 (tests) withhold a format from a model that would get it.
inline Pcg2Format pcg2_format(const dbl_model_desc *d, int hslots) {
  int nc = 0, code_max = 0;
  bool const_bytes = true, ids16 = true, codes = true;
  for (int a = 0; a < d->num_attrs; ++a) {
    const dbl_index &ix = *d->indexes[a];
    if (ix.is_const) {
      ++nc;
      const_bytes = const_bytes && ix.V <= 255;
      continue;
    }
    ids16 = ids16 && ix.V <= 65536;
    codes = codes && !ix.pcode.empty();
    if (codes) code_max = std::max(code_max, *std::max_element(ix.pcode.begin(), ix.pcode.end()));
  }
  Pcg2Format f{Pcg2Format::hc_of(hslots), false, false, false};
  // byte-packed constants: 1..4 of them, every vocabulary <= 255, 32-slot tables
  f.pk = nc >= 1 && nc <= 4 && const_bytes && f.hc == 32 && !getenv("DBL_NO_PACK");
  // slot codes: packed tiles, and every non-constant attribute has them
  f.sc = f.pk && nc < d->num_attrs && codes && !getenv("DBL_NO_SC");
  // 16-bit values: packed tiles, every non-constant vocabulary fits, and so does every code (codes may exceed the ids)
  f.id16 = f.pk && ids16 && !(f.sc && code_max > 65535) && !getenv("DBL_NO_ID16");
  return f;
}

// Per (record, non-constant attribute): H key words then H f64 values, H = p.hslots (a power of two >= 32, the same
// for every attribute of the model; 32 = one key per bank = conflict-free probes).
__device__ __host__ __forceinline__ int pcg2_tab_bytes(int H) { return H * 12; }

// Paired tables (16-bit slot codes, two records per warp: Pcg2Format::paired): per (warp, non-constant attribute) 32
// key words, word s = the key of record 0 at slot s in the low half and record 1's in the high half (one word per
// bank: one conflict-free probe serves both records), then record 0's 32 f64 values, then record 1's, PAIR_VALS bytes
// further: both value loads of a probe share one address.  An empty half at slot s holds s ^ 1, which no code with
// code & 31 == s equals.
constexpr int PAIR_KEYS = 32 * 4, PAIR_VALS = 32 * 8, PAIR_ATTR_BYTES = PAIR_KEYS + 2 * PAIR_VALS;

// w *= r when y == x (shapes without the packed-constant table; ptxas turns any predicated form into DMUL + 2 FSEL)
__device__ __forceinline__ void mul_if_eq(double &w, int y, int x, double r) {
  if (y == x) w = w * r;
}

template <int A, int NS, bool SC>
struct Pcg2Rec {
  int x[A];                                // record value id; -1 = missing (never equals an entity value)
  double rm[A];                            // multiplier on an exact match
  unsigned hm[(NS > 0 && !SC) ? NS : 1];  // hash multipliers of the non-constant attributes (SC: none)
  unsigned mmask;                // missing non-constant attributes (bit = kernel position)
  unsigned xpack;                // PK: the record's constant-attribute values, one byte each (0xFF = cannot match)
};

// PK kernels: BYTE offset into the record's table of constant-attribute products (8-byte entries) from the
// byte-packed values of a candidate: bit k of the entry index = (byte k of ypack == byte k of xpack)
__device__ __forceinline__ unsigned pcg2_const_offset(unsigned ypack, unsigned xpack) {
  const unsigned d = ypack ^ xpack;
  const unsigned nz = ((d & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | d;  // bit 7 of a byte set <=> the byte of d is non-zero
  const unsigned eq = ~nz & 0x80808080u;                      // bit 8k+7 set <=> byte k equal
  // the partial product of bit 8k+7 and bit 7j of the multiplier lands on bit 8k+7j+7: j = 3-k puts bit 8k+7 on bit
  // 28+k, and no two of the 16 partial products share a bit (no carries), so bits 28..31 are the four flags and
  // bits 25..27 are zero: the shift by 25 yields 8 * index, which ptxas adds to the table base in one LEA.HI
  return (eq * 0x00204081u) >> 25;
}

// One entity into slot `slot` of a tile of format f (pcg2_load reads it back).  y: the entity's values by attribute
// id, nullptr for a padding slot (all zero); perm: kernel order.  Packed tiles: the non-constant values (f.sc: their
// slot codes, AttrDev::pcode) at 32 or (f.id16) 16 bits, then the constants, one byte each.
__device__ __forceinline__ void pcg2_store(Pcg2Format f, int A, int NS, const int *y, const int *perm,
                                           const AttrDev *attrs, int *tile, int slot, double N) {
  const TileLayout tl = f.layout(A, NS);
  const int nid = f.id16 ? (NS + 1) / 2 : NS;  // words of non-constant values (packed tiles)
  auto ns_val = [&](int k) -> unsigned {       // value or slot code of kernel-order attribute k
    const int yv = y[perm[k]];
    return (unsigned)(f.sc ? attrs[perm[k]].pcode[yv] : yv);
  };
  for (int g = 0; g < tl.ng; ++g) {
    unsigned v[4] = {0u, 0u, 0u, 0u};
    for (int c = 0, w = 4 * g; c < 4 && y; ++c, ++w) {
      if (!f.pk) v[c] = w < A ? (unsigned)y[perm[w]] : 0u;
      else if (w < nid && f.id16)  // values 2w (low half) and 2w + 1 (high half)
        v[c] = (ns_val(A - NS + 2 * w) & 0xFFFFu) | (2 * w + 1 < NS ? ns_val(A - NS + 2 * w + 1) << 16 : 0u);
      else if (w < nid) v[c] = ns_val(A - NS + w);
      else if (w == nid)
        for (int k = 0; k < A - NS; ++k) v[c] |= ((unsigned)y[perm[k]] & 0xFFu) << (8 * k);
    }
    reinterpret_cast<int4 *>(tile)[TileLayout::group(g, slot)] = make_int4(v[0], v[1], v[2], v[3]);
  }
  reinterpret_cast<double *>(tile + tl.n_word())[slot] = N;
}

// one candidate out of a tile: values in kernel order (PK: only the non-constant ones + the packed word), N
template <int A, int NS, bool PK>
struct Pcg2Cand {
  int y[A];
  unsigned y16[(NS + 1) / 2 > 0 ? (NS + 1) / 2 : 1];  // ID16: the words of 16-bit values as loaded
  unsigned ypack;
  double N;
};
template <int A, int NS, bool PK, bool ID16>
__device__ __forceinline__ void pcg2_load(Pcg2Cand<A, NS, PK> &c, const int *tile, int slot) {
  static_assert(PK || !ID16, "16-bit values only in the packed tiles");
  constexpr TileLayout TL = Pcg2Format{0, PK, ID16, false}.layout(A, NS);  // the layout depends on PK and ID16 only
  int v[TL.ng * 4];
  const int4 *q = reinterpret_cast<const int4 *>(tile);
#pragma unroll
  for (int g = 0; g < TL.ng; ++g) {
    const int4 t = q[TileLayout::group(g, slot)];
    v[4 * g] = t.x; v[4 * g + 1] = t.y; v[4 * g + 2] = t.z; v[4 * g + 3] = t.w;
  }
  if constexpr (PK && ID16) {
#pragma unroll
    for (int q2 = 0; q2 < (NS + 1) / 2; ++q2) c.y16[q2] = (unsigned)v[q2];
#pragma unroll
    for (int q2 = 0; q2 < NS; ++q2) c.y[A - NS + q2] = (int)(q2 & 1 ? (unsigned)v[q2 >> 1] >> 16 : v[q2 >> 1] & 0xFFFF);
    c.ypack = (unsigned)v[(NS + 1) / 2];
  } else if constexpr (PK) {
#pragma unroll
    for (int q2 = 0; q2 < NS; ++q2) c.y[A - NS + q2] = v[q2];
    c.ypack = (unsigned)v[NS];
  } else {
#pragma unroll
    for (int k = 0; k < A; ++k) c.y[k] = v[k];
    c.ypack = 0u;
  }
  c.N = reinterpret_cast<const double *>(tile + TL.n_word())[slot];
}

// With skewed (Zipf-like) value frequencies some lane of the warp finds an equal or similar value on almost every
// step (96 % at BASELINE's 1M configuration), so a warp-wide vote that skips the multiplies does not pay: the
// multiplies are predicated per lane and the compiler is free to overlap them with the next step's loads.
// SC: the non-constant values are slot codes (AttrDev::pcode), whose low five bits are the slot in every record's
// table: the slot of a probe does not depend on the record, so it is computed once for the warp's records, which need
// no multipliers.
// inv: the candidate's entry of its tile's first 1/n(y) column (LinkParams::tile_invn), column q at inv[q * TE]: in
// pass 1 the column staged in shared memory with the tile, in pass 2 the one in global memory; read only for the
// attributes the record misses.  Their probes stay: the record's table of such an attribute is empty, so the probe
// never hits, and a warp-uniform skip per attribute cost more instructions per tile than the probes it saves (569
// against 630 at A = 10, NS = 6, paired).
template <int A, int NS, int HC, bool PK, bool SC, bool MISSING = true>
__device__ __forceinline__ double pcg2_weight(const Pcg2Rec<A, NS, SC> &rc, const LinkParams &p, const char *tab,
                                              const double *ctab, const Pcg2Cand<A, NS, PK> &cd, const double *inv) {
  static_assert(!SC || (PK && HC == 32), "slot codes only in the packed 32-slot tiles");
  const int hslots = HC ? HC : p.hslots;
  const int hshift = HC ? 27 : p.hshift;
  const int tabb = pcg2_tab_bytes(hslots);
  const int *y = cd.y;
  double w = cd.N;
  if constexpr (NS < A) {  // protocol 4.1: the constant attributes form their own product c; w = N * c
    double c = 1.0;
    if constexpr (PK) {
      // the record's 16-entry table of products, indexed by a SWAR byte compare of the packed values
      c = *reinterpret_cast<const double *>(reinterpret_cast<const char *>(ctab) + pcg2_const_offset(cd.ypack, rc.xpack));
    } else {
#pragma unroll
      for (int k = 0; k < A - NS; ++k) mul_if_eq(c, y[k], rc.x[k], rc.rm[k]);
    }
    w = w * c;
  }
  // protocol 4.1: non-constant attributes in kernel order, each contributes at most one factor: the exact-match
  // multiplier when y == x, exp(similarity) when y is similar to x -- both sit in the record's hash table
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const int yv = y[A - NS + q];
    unsigned slot;
    // SC: the AND is opaque to the compiler, which would otherwise fold it into (y << 2) & 0x7C and (y << 3) & 0xF8
    // (two more instructions per probe); kept as an AND, each table address is one multiply-add of the slot
    if constexpr (SC) asm("and.b32 %0, %1, 31;" : "=r"(slot) : "r"(yv));
    else slot = ((unsigned)yv * rc.hm[q]) >> hshift;
    if (reinterpret_cast<const int *>(tab + q * tabb)[slot] == yv)
      w = w * reinterpret_cast<const double *>(tab + q * tabb + hslots * 4)[slot];
  }
  if (MISSING && rc.mmask) {
#pragma unroll
    for (int q = 0; q < NS; ++q)
      if ((rc.mmask >> (A - NS + q)) & 1u) w = w * inv[q * TE];
  }
  return w;
}

// Paired tables: whether half H (0 low, 1 high) of k ^ c2 is zero, as one 3-input lop3, (k ^ c2) & mask, which ptxas
// turns into one LOP3 that writes the predicate.  Written in C, the compiler computes the XOR once for both halves
// and tests each with a LOP3 of its own (and the low half as a sign-extended 16-bit compare unless the AND is opaque).
template <int H>
__device__ __forceinline__ bool pcg2_half_hit(unsigned k, unsigned c2) {
  unsigned hit;
  asm("{\n\t.reg .pred p;\n\t.reg .b32 t;\n\tlop3.b32 t, %1, %2, %3, 0x28;\n\tsetp.eq.u32 p, t, 0;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(hit)
      : "r"(k), "r"(c2), "n"(H ? 0xFFFF0000u : 0xFFFFu));
  return hit != 0;
}

// Paired tables (Pcg2Format::paired): the weights of one candidate for the warp's records whose bit is set in `recs`, in w[0]
// and w[1]; each is the product pcg2_weight forms, factor for factor in the same order.  Per (candidate, attribute):
// one PRMT spreads the 16-bit code over both halves of a word, c2 = {code, code}; ONE key load at slot code & 31
// serves both records, whose hits are the halves of k ^ c2 that are zero (pcg2_half_hit); one value address serves
// both predicated value loads (record 1's values are PAIR_VALS bytes past record 0's).  inv: as in pcg2_weight.
template <int A, int NS, bool MISSING = true>
__device__ __forceinline__ void pcg2_weight_pair(const Pcg2Rec<A, NS, true> (&rc)[2], unsigned recs,
                                                 const char *tab, const double *ctab, const Pcg2Cand<A, NS, true> &cd,
                                                 double (&w)[2], const double *inv) {
  static_assert(NS >= 1 && NS < A, "paired tables: packed constants and at least one non-constant attribute");
#pragma unroll
  for (int ri = 0; ri < 2; ++ri)  // protocol 4.1: w = N * (product of the constant attributes' multipliers)
    w[ri] = cd.N * *reinterpret_cast<const double *>(reinterpret_cast<const char *>(ctab + ri * 16) +
                                                     pcg2_const_offset(cd.ypack, rc[ri].xpack));
#pragma unroll
  for (int q = 0; q < NS; ++q) {
    const unsigned c2 = __byte_perm(cd.y16[q >> 1], 0u, (q & 1) ? 0x3232 : 0x1010);
    unsigned slot;  // opaque AND, as in pcg2_weight
    asm("and.b32 %0, %1, 31;" : "=r"(slot) : "r"(c2));
    const unsigned k = reinterpret_cast<const unsigned *>(tab + q * PAIR_ATTR_BYTES)[slot];
    const double *v = reinterpret_cast<const double *>(tab + q * PAIR_ATTR_BYTES + PAIR_KEYS) + slot;
    if ((recs & 1u) && pcg2_half_hit<0>(k, c2)) w[0] = w[0] * v[0];
    if ((recs & 2u) && pcg2_half_hit<1>(k, c2)) w[1] = w[1] * v[PAIR_VALS / 8];
  }
  if (MISSING) {
#pragma unroll
    for (int ri = 0; ri < 2; ++ri) {
      if (!((recs >> ri) & 1u) || !rc[ri].mmask) continue;
#pragma unroll
      for (int q = 0; q < NS; ++q)
        if ((rc[ri].mmask >> (A - NS + q)) & 1u) w[ri] = w[ri] * inv[q * TE];
    }
  }
}

// bytes of one consumer warp's hash tables (H = the table size of the model)
__host__ __device__ inline int pcg2_warp_tab_bytes(Pcg2Format f, int NS, int H) {
  return f.paired(NS) ? NS * PAIR_ATTR_BYTES : f.rpw(NS) * (NS > 0 ? NS : 1) * pcg2_tab_bytes(H);
}

template <int A, int NS, int HC, bool PK, bool ID16, bool SC>
__global__ void __launch_bounds__((LINK_WARPS + 1) * 32, Pcg2Format{HC, PK, ID16, SC}.ctas_per_sm(NS)) k_link_pcg2(LinkParams p) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ int s_cta;
  if (sweep_dead(p.ctl)) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  constexpr Pcg2Format FMT{HC, PK, ID16, SC};
  constexpr int TW = FMT.layout(A, NS).words();
  constexpr int NC = A - NS;
  constexpr int RPW = FMT.rpw(NS);
  constexpr int WARPS = LINK_WARPS;           // consumer warps; warp WARPS is the producer
  constexpr int PCG2_RECS = WARPS * RPW;      // records per work item (= per "CTA" of cta_ptr)
  TileRing rg;
  rg.tiles = reinterpret_cast<int *>(smem);
  rg.full = reinterpret_cast<uint64_t *>(smem + (size_t)LINK_STAGES * TW * 4);
  rg.empty = rg.full + LINK_STAGES;
  rg.tw = TW;
  static_assert(2 * LINK_STAGES * 8 <= 128, "barrier area");
  constexpr bool PAIR = FMT.paired(NS);
  const int tabrec = (NS > 0 ? NS : 1) * pcg2_tab_bytes(HC ? HC : p.hslots);  // bytes of one record's hash tables
  // ... of one warp's.  HC = 0: the records per warp of this stride come from p.hslots at run time (1 in every launch);
  // a compile-time 1 moves ptxas's spills and cost 1.2 % at A = 11, NS = 5 (H100 SXM, 700 W)
  const int wtab = pcg2_warp_tab_bytes(HC ? FMT : Pcg2Format{Pcg2Format::hc_of(p.hslots)}, NS, HC ? HC : p.hslots);
  char *tab0 = reinterpret_cast<char *>(smem) + (size_t)LINK_STAGES * TW * 4 + 128 + (size_t)warp * wtab;
  // PK: products of the matching constant attributes, by match mask, 16 entries per record
  double *ctab0 = reinterpret_cast<double *>(reinterpret_cast<char *>(smem) + (size_t)LINK_STAGES * TW * 4 + 128 +
                                            (size_t)WARPS * wtab) + warp * RPW * 16;
  // the 1/n(y) columns of the staged tiles (only when p.tile_invn: see pcg2_smem_bytes)
  rg.cols = reinterpret_cast<double *>(reinterpret_cast<char *>(smem) + (size_t)LINK_STAGES * TW * 4 + 128 +
                                       (size_t)WARPS * wtab) + WARPS * RPW * 16;
  rg.ncols = NS;
  ring_init(rg, WARPS);
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
    const int *gtiles = p.tiles + (size_t)p.tile_ptr[b] * TW;
    const double *gcols = p.tile_invn ? p.tile_invn + (size_t)p.tile_ptr[b] * NS * TE : nullptr;
    const int rec0 = p.rec_ptr[b] + (cta - p.cta_ptr[b]) * PCG2_RECS;  // first record of the work item

    if (warp == WARPS) {  // producer warp
      // the columns to stage: the non-constant attributes that some record of the work item misses
      unsigned cmask = 0u;
      if (gcols && lane < PCG2_RECS && rec0 + lane < p.rec_ptr[b + 1]) {
        const int r = p.rec_sorted[rec0 + lane];
#pragma unroll
        for (int q = 0; q < NS; ++q)
          if (p.x[(int64_t)r * A + p.perm[A - NS + q]] < 0) cmask |= 1u << q;
      }
      cmask = __reduce_or_sync(FULL, cmask);
      if (lane == 0) ring_produce<true>(rg, gtiles, ntiles, tbase, gcols, cmask);
      tbase += ntiles;
      continue;
    }

    // ---- per-record constants: lane k prepares kernel-order attribute k, then everything is broadcast
    Pcg2Rec<A, NS, SC> rc[RPW];
    int rr[RPW];
    bool act[RPW];
#pragma unroll
    for (int ri = 0; ri < RPW; ++ri) {
      const int ridx = rec0 + warp * RPW + ri;
      act[ri] = ridx < p.rec_ptr[b + 1];
      rr[ri] = act[ri] ? p.rec_sorted[ridx] : -1;
      const int r = rr[ri];
      char *tab = PAIR ? tab0 : tab0 + ri * tabrec;
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
            if constexpr (!SC) hmv = at.hmult[xv];
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
      if constexpr (!SC) {
#pragma unroll
        for (int q = 0; q < NS; ++q) rc[ri].hm[q] = __shfl_sync(FULL, hmv, A - NS + q);
      }
      // hash tables of the record's similarity rows -> shared memory (all-empty table when the value is missing);
      // the entry of the record's own value gets the exact-match multiplier (it depends on theta of the record's file)
      const int H = HC ? HC : p.hslots;
      const int hshift = HC ? 27 : p.hshift;
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const AttrDev &at = p.attrs[p.perm[A - NS + q]];
        char *tq = tab + q * (PAIR ? PAIR_ATTR_BYTES : pcg2_tab_bytes(H));
        int *kd = reinterpret_cast<int *>(tq);
        double *vd = reinterpret_cast<double *>(tq + (PAIR ? PAIR_KEYS + ri * PAIR_VALS : H * 4));
        const int xq = rc[ri].x[A - NS + q];
        // SC: the code-keyed tables, each value at the slot its code names
        const int *hkeys = SC ? at.sckeys : at.hkeys;
        const double *hvals = SC ? at.scvals : at.hvals;
        unsigned own;
        if constexpr (SC) own = (xq >= 0) ? ((unsigned)at.pcode[xq] & 31u) : 0xFFFFFFFFu;
        else own = (xq >= 0) ? (((unsigned)xq * rc[ri].hm[q]) >> hshift) : 0xFFFFFFFFu;
        for (int i = lane; i < H; i += 32) {
          const int key = (xq >= 0) ? hkeys[(size_t)xq * H + i] : -1;
          if constexpr (PAIR)  // the record's half of the paired key word; empty: i ^ 1
            reinterpret_cast<unsigned short *>(kd)[2 * i + ri] = (unsigned short)(key >= 0 ? key : i ^ 1);
          else
            kd[i] = key;
          vd[i] = ((unsigned)i == own) ? rc[ri].rm[A - NS + q] : ((xq >= 0) ? hvals[(size_t)xq * H + i] : 1.0);
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

    const DrawGeom geo = draw_geom(ntiles);

    // ---- pass 1 over the TMA-staged tiles.  Records without a missing non-constant attribute (most of them) take a
    // loop body without the gather of 1/n(y): straight-line code the compiler can overlap across the steps of a tile
    double run[RPW], Q[RPW], acc[RPW];  // run, Q: each record's Checkpoints, with `chunk` shared by the records
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
          const double *cols = rg.cols + (size_t)s * NS * TE + lane;  // the staged 1/n(y) columns (MISSING)
#pragma unroll
          for (int q = 0; q < TE / 32; ++q) {
            Pcg2Cand<A, NS, PK> cd;
            pcg2_load<A, NS, PK, ID16>(cd, tile, q * 32 + lane);
            if constexpr (PAIR) {
              double w[2];
              pcg2_weight_pair<A, NS, MISSING>(rc, 3u, tab0, ctab0, cd, w, cols + q * 32);
              acc[0] = acc[0] + w[0];
              acc[1] = acc[1] + w[1];
            } else {
#pragma unroll
              for (int ri = 0; ri < RPW; ++ri)
                acc[ri] = acc[ri] + pcg2_weight<A, NS, HC, PK, SC, MISSING>(rc[ri], p, tab0 + ri * tabrec,
                                                                          ctab0 + ri * 16, cd, cols + q * 32);
            }
          }
          if (++tile_in_chunk == geo.tpc || t + 1 == ntiles) {
#pragma unroll
            for (int ri = 0; ri < RPW; ++ri) {
              my_sums[ri * 1024 + chunk * 32 + lane] = acc[ri];  // pass 2 reads the chosen chunk's sums back
              close_chunk(lane, chunk, acc[ri], run[ri], Q[ri]);
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
      if (!check_mass(p, lane, r, run[ri])) continue;
      auto wf = [&](int j) -> double {
        if (j >= n) return 0.0;
        Pcg2Cand<A, NS, PK> cd;
        pcg2_load<A, NS, PK, ID16>(cd, gtiles + (size_t)(j / TE) * TW, j % TE);
        // the candidate's 1/n(y) in global memory (read only when the record misses a value: then gcols is set)
        const double *inv = gcols + (size_t)(j / TE) * NS * TE + j % TE;
        if constexpr (PAIR) {  // record ri's half of the paired tables
          double w[2];
          pcg2_weight_pair<A, NS>(rc, 1u << ri, tab0, ctab0, cd, w, inv);
          return ri ? w[1] : w[0];
        } else {
          return pcg2_weight<A, NS, HC, PK, SC>(rc[ri], p, tab0 + ri * tabrec, ctab0 + ri * 16, cd, inv);
        }
      };
      const U2 u = link_uniform(p, r);
      const int j = finish_draw(lane, n, geo, Q[ri], run[ri], u.u0, wf, my_sums + ri * 1024);
      store_link(p, lane, r, b, n, j);
    }
  }
}

// dynamic shared memory of one CTA (H = the table size of the model); invn: with the ring's 1/n(y) columns, NS per
// stage (LinkParams::tile_invn set: some record misses a non-constant value)
inline size_t pcg2_smem_bytes(Pcg2Format f, int A, int NS, int H, bool invn) {
  return (size_t)LINK_STAGES * f.layout(A, NS).words() * 4 + 128 + (size_t)LINK_WARPS * pcg2_warp_tab_bytes(f, NS, H) +
         (size_t)LINK_WARPS * f.rpw(NS) * 16 * sizeof(double) + (invn ? (size_t)LINK_STAGES * NS * TE * sizeof(double) : 0);
}

// k_link_pcg2<A, NS, ...> of format f for a runtime NS in [0, A] (nullptr: none); the `if constexpr` guards only keep
// out the formats pcg2_format never gives this shape (packed constants need 1..4 of them, slot codes NS >= 1)
using Pcg2Kernel = void (*)(LinkParams);
template <int A, int NS>
Pcg2Kernel pcg2_kernel(int ns, Pcg2Format f) {
  if (ns != NS) {
    if constexpr (NS > 0) return pcg2_kernel<A, NS - 1>(ns, f);
    return nullptr;
  }
  if constexpr (A - NS >= 1 && A - NS <= 4) {
    if constexpr (NS >= 1) {
      if (f.sc) return f.id16 ? k_link_pcg2<A, NS, 32, true, true, true> : k_link_pcg2<A, NS, 32, true, false, true>;
    }
    if (f.pk) return f.id16 ? k_link_pcg2<A, NS, 32, true, true, false> : k_link_pcg2<A, NS, 32, true, false, false>;
  }
  return f.hc ? k_link_pcg2<A, NS, 32, false, false, false> : k_link_pcg2<A, NS, 0, false, false, false>;
}

// launch kernel k on `grid` CTAs with `smem` bytes of dynamic shared memory; lp == nullptr: load the kernel without
// running it (see preload_kernels in dbl_engine.cu); returns cudaError_t as int
inline int pcg2_launch(Pcg2Kernel k, size_t smem, const LinkParams *lp, int grid, cudaStream_t stream,
                       size_t *configured) {
  if (!k) return (int)cudaErrorInvalidValue;
  // the opt-in is per device: the cache belongs to the context (one model shape = one instantiation per context)
  if (*configured < smem) {
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    *configured = smem;
  }
  cudaFuncAttributes fa;
  if (!lp) return (int)cudaFuncGetAttributes(&fa, k);
  k<<<grid, (LINK_WARPS + 1) * 32, smem, stream>>>(*lp);
  return (int)cudaGetLastError();
}
