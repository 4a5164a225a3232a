// Host build of the limb-level arithmetic in field.cuh / curve.cuh (same code path as the device,
// PTX carry-chain primitives replaced by their emulation).  TEST INFRASTRUCTURE: loaded only by
// tests/test_host_arith.py through ctypes; never linked into libplonk_b200.so.  It also exports the proof layout
// (proof_layout.cuh) for tests/test_proof_layout.py, the prover's memory plan (memory_plan.cuh) for
// tests/test_sliced_prover.py and the permutation's label body (permutation.cuh) for tests/test_wiring_host.py.
#include "field.cuh"
#include "curve.cuh"
#include "msm_digits.cuh"
#include "modinv.cuh"
#include "msm_bucket.cuh"
#include "msm_sort.cuh"
#include "ntt_shard.cuh"
#include "proof_layout.cuh"
#include "memory_plan.cuh"
#include "permutation.cuh"
#include "solve.cuh"
#include <unordered_map>
#include <algorithm>
#include <vector>
#include <cstring>
using namespace pb200;

template <class F> static F ld(const uint32_t* p) { F r; memcpy(r.v, p, 32); return r; }
template <class F> static void st(uint32_t* p, const F& a) { memcpy(p, a.v, 32); }

extern "C" {
// op: 0 add, 1 sub, 2 mul, 3 neg, 4 inv, 5 to_mont, 6 from_mont, 7 dbl, 8 sqr, 9 inv by safegcd (Montgomery
// contract of op 4), 10 plain-integer inverse by safegcd ; field: 0 Fr, 1 Fq
int hs_field_op(int field, int op, const uint32_t* a, const uint32_t* b, uint32_t* out) {
#define RUN(F)                                                   \
  {                                                              \
    F x = ld<F>(a), y = ld<F>(b), r;                             \
    switch (op) {                                                \
      case 0: r = fp_add(x, y); break;                           \
      case 1: r = fp_sub(x, y); break;                           \
      case 2: r = fp_mul(x, y); break;                           \
      case 3: r = fp_neg(x); break;                              \
      case 4: r = fp_inv(x); break;                              \
      case 5: r = fp_to_mont(x); break;                          \
      case 6: r = fp_from_mont(x); break;                        \
      case 7: r = fp_dbl(x); break;                              \
      case 8: r = fp_sqr(x); break;                              \
      case 9: r = fp_inv_gcd(x); break;                          \
      case 10: r = fp_inv_plain_gcd(x); break;                   \
      case 11: r = fp_mul_lazy(x, y); break;                     \
      case 12: r = fp_sqr_lazy(x); break;                        \
      case 13: r = fp_sub_lazy(x, y); break;                     \
      case 14: r = fp_neg_lazy(x); break;                        \
      case 15: r = fp_is_zero_lazy(x) ? F::one() : F::zero(); break; \
      default: return -1;                                        \
    }                                                            \
    st(out, r);                                                  \
  }
  if (field == 0) RUN(Fr) else RUN(Fq)
#undef RUN
  return 0;
}

// redc(a b + c d) without the final subtraction (fp_mul2_lazy)
int hs_field_mul2(int field, const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* d, uint32_t* out) {
  if (field == 0) st(out, fp_mul2_lazy(ld<Fr>(a), ld<Fr>(b), ld<Fr>(c), ld<Fr>(d)));
  else st(out, fp_mul2_lazy(ld<Fq>(a), ld<Fq>(b), ld<Fq>(c), ld<Fq>(d)));
  return 0;
}
}  // extern "C"

// The group law as it was written before the lazily reduced primitives (canonical products, fp_sqr = fp_mul(a, a),
// two reductions for Y3): the reference the shipped formulas must match limb for limb, since both keep every
// coordinate they return canonical.
static Fq ref_sqr(const Fq& a) { return fp_mul(a, a); }
static void ref_double(G1XYZZ& a) {
  if (a.is_inf()) return;
  Fq U = fp_dbl(a.Y), V = ref_sqr(U), W = fp_mul(U, V), S = fp_mul(a.X, V), M = ref_sqr(a.X);
  M = fp_add(fp_dbl(M), M);
  Fq X3 = fp_sub(ref_sqr(M), fp_dbl(S));
  a.Y = fp_sub(fp_mul(M, fp_sub(S, X3)), fp_mul(W, a.Y));
  a.X = X3;
  a.ZZ = fp_mul(V, a.ZZ);
  a.ZZZ = fp_mul(W, a.ZZZ);
}
static void ref_add_mixed(G1XYZZ& acc, const G1Affine& p) {
  if (acc.is_inf()) { acc = g1_from_affine(p); return; }
  Fq U2 = fp_mul(p.x, acc.ZZ), S2 = fp_mul(p.y, acc.ZZZ), Pd = fp_sub(U2, acc.X), Rd = fp_sub(S2, acc.Y);
  if (Pd.is_zero()) {
    if (Rd.is_zero()) { acc = g1_from_affine(p); ref_double(acc); }
    else acc = G1XYZZ::identity();
    return;
  }
  Fq PP = ref_sqr(Pd), PPP = fp_mul(Pd, PP), Q = fp_mul(acc.X, PP);
  Fq X3 = fp_sub(fp_sub(ref_sqr(Rd), PPP), fp_dbl(Q));
  acc.Y = fp_sub(fp_mul(Rd, fp_sub(Q, X3)), fp_mul(acc.Y, PPP));
  acc.X = X3;
  acc.ZZ = fp_mul(acc.ZZ, PP);
  acc.ZZZ = fp_mul(acc.ZZZ, PPP);
}
static void ref_add(G1XYZZ& acc, const G1XYZZ& q) {
  if (q.is_inf()) return;
  if (acc.is_inf()) { acc = q; return; }
  Fq U1 = fp_mul(acc.X, q.ZZ), U2 = fp_mul(q.X, acc.ZZ), S1 = fp_mul(acc.Y, q.ZZZ), S2 = fp_mul(q.Y, acc.ZZZ);
  Fq Pd = fp_sub(U2, U1), Rd = fp_sub(S2, S1);
  if (Pd.is_zero()) {
    if (Rd.is_zero()) ref_double(acc);
    else acc = G1XYZZ::identity();
    return;
  }
  Fq PP = ref_sqr(Pd), PPP = fp_mul(Pd, PP), Q = fp_mul(U1, PP);
  Fq X3 = fp_sub(fp_sub(ref_sqr(Rd), PPP), fp_dbl(Q));
  acc.Y = fp_sub(fp_mul(Rd, fp_sub(Q, X3)), fp_mul(S1, PPP));
  acc.X = X3;
  acc.ZZ = fp_mul(fp_mul(acc.ZZ, q.ZZ), PP);
  acc.ZZZ = fp_mul(fp_mul(acc.ZZZ, q.ZZZ), PPP);
}

extern "C" {
// hs_curve_op's ops 0, 1, 2, 4, 5 by the reference formulas above (4 and 5 are the same sums as 0 and 1)
int hs_curve_op_ref(int op, const uint32_t* acc_in, const uint32_t* other, int other_inf, uint32_t* out) {
  G1XYZZ acc;
  memcpy(&acc, acc_in, sizeof(acc));
  if (op == 0 || op == 4) {
    G1Affine p;
    memcpy(&p.x, other, 32);
    memcpy(&p.y, other + 8, 32);
    if (!other_inf) ref_add_mixed(acc, p);
  } else if (op == 1 || op == 5) {
    G1XYZZ q;
    memcpy(&q, other, sizeof(q));
    ref_add(acc, q);
  } else if (op == 2) {
    ref_double(acc);
  } else {
    return -1;
  }
  memcpy(out, &acc, sizeof(acc));
  return 0;
}

// The join of the slab-sharded NTT (ntt_shard.cuh): out[k] = sum_r x[r] w^(r k) for G = 2^log_g elements in Montgomery
// form, tw = w^0 .. w^(G/2 - 1) (Montgomery).  x, out: G x 8 limbs; tw: 4 x 8 limbs.
int hs_small_dft(int log_g, const uint32_t* x, const uint32_t* tw, uint32_t* out) {
  DftTw t;
  for (int k = 0; k < 4; k++) t.w[k] = ld<Fr>(tw + 8 * k);
#define RUN_DFT(LG)                                                     \
  {                                                                     \
    Fr v[1 << LG];                                                      \
    for (int i = 0; i < (1 << LG); i++) v[i] = ld<Fr>(x + 8 * i);       \
    small_dft<LG>(v, t);                                                \
    for (int i = 0; i < (1 << LG); i++) st(out + 8 * i, v[i]);          \
  }
  switch (log_g) {
    case 1: RUN_DFT(1) break;
    case 2: RUN_DFT(2) break;
    case 3: RUN_DFT(3) break;
    default: return -1;
  }
#undef RUN_DFT
  return 0;
}

// signed digits of a canonical scalar for window size c: writes W = ceil(256 / c) digits (sign * magnitude) and
// returns the carry left after the last window (must be 0 for scalars < r)
int hs_msm_digits(const uint32_t* scalar, uint32_t c, int32_t* digits, uint32_t* n_windows) {
  MsmGeom g;
  g.c = c;
  g.W = (256 + c - 1) / c;
  g.half = 1u << (c - 1);
  g.fixed_base = 0;
  g.point_stride = 0;
  g.batch = 1;
  g.lo = 0;
  g.nloc = g.half;
  g.own_log = 0;
  g.own_rank = 0;
  g.sets = g.W;
  g.nb = g.half * g.W;
  Fr s = ld<Fr>(scalar);
  DigitWalk dw(&s, 0, 0);
  for (uint32_t w = 0; w < g.W; w++) {
    uint32_t neg, d = dw.next(w, g, neg);
    digits[w] = neg ? -(int32_t)d : (int32_t)d;
  }
  *n_windows = g.W;
  return (int)dw.carry;
}

// G1 ops on Montgomery-form coordinates.  xyzz: 4x8 limbs (X, Y, ZZ, ZZZ); affine: 2x8 limbs + inf flag.
// op: 0 xyzz += affine, 1 xyzz += xyzz, 2 double, 3 to_affine
int hs_curve_op(int op, const uint32_t* acc_in, const uint32_t* other, int other_inf, uint32_t* out) {
  G1XYZZ acc;
  memcpy(&acc, acc_in, sizeof(acc));
  switch (op) {
    case 0: {
      G1Affine p;
      memcpy(&p.x, other, 32);
      memcpy(&p.y, other + 8, 32);
      if (!other_inf) g1_add_mixed(acc, p);
      break;
    }
    case 4: {
      G1Affine p;
      memcpy(&p.x, other, 32);
      memcpy(&p.y, other + 8, 32);
      if (!other_inf) g1_add_mixed_uniform(acc, p);
      break;
    }
    case 1: {
      G1XYZZ q;
      memcpy(&q, other, sizeof(q));
      g1_add(acc, q);
      break;
    }
    case 2: g1_double(acc); break;
    case 5: {
      G1XYZZ q;
      memcpy(&q, other, sizeof(q));
      g1_add_uniform(acc, q);
      break;
    }
    case 3: {
      G1Affine p;
      bool inf = g1_to_affine(acc, p);
      memcpy(out, &p.x, 32);
      memcpy(out + 8, &p.y, 32);
      return inf ? 1 : 0;
    }
    default: return -1;
  }
  memcpy(out, &acc, sizeof(acc));
  return 0;
}

}  // extern "C"

// MSM geometry of a call.  [lo, hi): the bucket magnitudes this "rank" owns; hi = 0xffffffff - log_g (log_g < 16)
// instead selects the strided shard of rank lo out of 2^log_g.  false on bad input.
static bool msm_geom(uint32_t n, uint32_t batch, uint32_t c, int fixed_base, uint32_t lo, uint32_t hi, MsmGeom& g) {
  g.c = c;
  g.W = (256 + c - 1) / c;
  g.half = 1u << (c - 1);
  g.fixed_base = fixed_base ? 1 : 0;
  g.point_stride = fixed_base ? n : 0;
  g.batch = batch;
  g.own_log = 0;
  g.own_rank = 0;
  if (hi >= 0xfffffff0u && hi != 0xffffffffu) {  // strided shard: 2^(0xffffffff - hi) ranks, rank = lo
    g.own_log = 0xffffffffu - hi;
    g.own_rank = lo;
    g.lo = 0;
    g.nloc = g.half >> g.own_log;
    if (!g.nloc || lo >= (1u << g.own_log)) return false;
  } else {
    if (hi > g.half) hi = g.half;
    if (lo >= hi) return false;
    g.lo = lo;
    g.nloc = hi - lo;
  }
  g.sets = fixed_base ? batch : g.W;
  g.nb = g.sets * g.nloc;
  return true;
}

// k_scan_tile_sums + k_scan_tiles + k_scan_apply of msm.cu: off = exclusive prefix of the (padded) counts, counts
// zeroed; *max_out = the largest raw count
static void host_scan(uint32_t* cnt, uint32_t len, uint32_t pad, uint32_t* off, uint32_t* max_out) {
  uint32_t run = 0, m = 0;
  for (uint32_t b = 0; b < len; b++) {
    off[b] = run;
    run += (cnt[b] + pad) & ~pad;
    m = std::max(m, cnt[b]);
    cnt[b] = 0;
  }
  off[len] = run;
  if (max_out) *max_out = m;
}

// The sort of msm_run_batch (msm_sort.cuh) on the CPU: every kernel's blocks one after the other, each block as a
// loop over its phases, each phase as a loop over the block's nt threads.  Out: counts (nb raw counts + the max),
// off (nb + 1), sorted (off[nb] + 2 positions, unused ones PB_MSM_PAD).
static void host_msm_sort(const MsmGeom& g, const std::vector<Fr>& sc, uint32_t n, uint32_t pad, uint32_t lb,
                          uint32_t T, uint32_t spb, uint32_t bin_nt, uint32_t chunk_nt, std::vector<uint32_t>& counts,
                          std::vector<uint32_t>& off, std::vector<uint32_t>& sorted) {
  const uint32_t nbins = ((g.nb - 1) >> lb) + 1;
  const uint32_t batch = g.fixed_base ? g.batch : 1;
  std::vector<uint32_t> bin_cnt(nbins, 0), bin_off(nbins + 1), chunk_first(nbins + 1);
  std::vector<SortEntry> binned((size_t)n * g.W * batch);
  counts.assign(g.nb + 1, 0);
  off.assign(g.nb + 1, 0);
  SortArgs a;
  for (uint32_t k = 0; k < 4; k++) a.sb.p[k] = k < batch ? sc.data() + (size_t)k * n : nullptr;
  a.n = n;
  a.from_mont = 0;
  a.g = g;
  a.lb = lb;
  a.nbins = nbins;
  a.T = T;
  a.bin_cnt = bin_cnt.data();
  a.bin_off = bin_off.data();
  a.binned = binned.data();
  a.chunk_first = chunk_first.data();
  a.counts = counts.data();
  a.offsets = off.data();
  a.sorted = nullptr;
  a.spb = spb;
  std::vector<uint32_t> sh_cnt(std::max(nbins, 1u << lb)), sh_loc(sh_cnt.size()), sh_base(sh_cnt.size()), runs;
  std::vector<SortEntry> bin_stage_buf((size_t)spb * g.W);
  std::vector<uint32_t> chunk_stage_buf(T);
  // the block scan of the placement kernels: runs[t] = exclusive prefix of the threads' scan_part_sum; the total
  auto block_scan = [&](uint32_t len, uint32_t nt) {
    runs.assign(nt, 0);
    uint32_t run = 0;
    for (uint32_t t = 0; t < nt; t++) { runs[t] = run; run += scan_part_sum(sh_cnt.data(), len, t, nt); }
    return run;
  };
  const uint32_t bin_blocks = (n + spb - 1) / spb;
  // k_msm_bin_count
  for (uint32_t k = 0; k < batch; k++)
    for (uint32_t bx = 0; bx < bin_blocks; bx++) {
      for (uint32_t t = 0; t < bin_nt; t++) sort_zero(sh_cnt.data(), nbins, t, bin_nt);
      for (uint32_t t = 0; t < bin_nt; t++) bin_hist(a, bx, k, t, bin_nt, sh_cnt.data());
      for (uint32_t t = 0; t < bin_nt; t++) bin_flush(a, t, bin_nt, sh_cnt.data());
    }
  host_scan(bin_cnt.data(), nbins, 0, bin_off.data(), nullptr);
  // k_msm_bin_scatter; blocks in reverse order, so the bins' ranges are not filled in walk order
  for (uint32_t k = batch; k-- > 0;)
    for (uint32_t bx = bin_blocks; bx-- > 0;) {
      for (uint32_t t = 0; t < bin_nt; t++) sort_zero(sh_cnt.data(), nbins, t, bin_nt);
      for (uint32_t t = 0; t < bin_nt; t++) bin_hist(a, bx, k, t, bin_nt, sh_cnt.data());
      const uint32_t total = block_scan(nbins, bin_nt);
      for (uint32_t t = 0; t < bin_nt; t++)
        bin_reserve(a, t, bin_nt, runs[t], sh_cnt.data(), sh_loc.data(), sh_base.data());
      for (uint32_t t = 0; t < bin_nt; t++) bin_stage(a, bx, k, t, bin_nt, sh_cnt.data(), sh_loc.data(), bin_stage_buf.data());
      for (uint32_t t = 0; t < bin_nt; t++)
        bin_copy_out(a, t, bin_nt, total, sh_loc.data(), sh_base.data(), bin_stage_buf.data());
    }
  // k_msm_chunk_map
  {
    std::vector<uint32_t> sums(256);
    for (uint32_t t = 0; t < 256; t++) sums[t] = chunk_map_sum(a, t);
    uint32_t run = 0;
    for (uint32_t t = 0; t < 256; t++) { const uint32_t s = sums[t]; sums[t] = run; run += s; }
    for (uint32_t t = 0; t < 256; t++) chunk_map_write(a, t, sums[t], run);
  }
  // the chunk kernels, with a grid of `grid` blocks walking the chunks grid-stride
  const uint32_t grid = 3;
  SortChunk ch;
  for (uint32_t bx = 0; bx < grid; bx++)
    for (uint32_t c = bx; chunk_locate(a, c, ch); c += grid) {
      for (uint32_t t = 0; t < chunk_nt; t++) sort_zero(sh_cnt.data(), ch.nkeys, t, chunk_nt);
      for (uint32_t t = 0; t < chunk_nt; t++) chunk_hist(a, ch, t, chunk_nt, sh_cnt.data());
      for (uint32_t t = 0; t < chunk_nt; t++) chunk_flush(a, ch, t, chunk_nt, sh_cnt.data());
    }
  host_scan(counts.data(), g.nb, pad, off.data(), &counts[g.nb]);
  sorted.assign(off[g.nb] + 2, PB_MSM_PAD);
  a.sorted = sorted.data();
  for (uint32_t bx = grid; bx-- > 0;)
    for (uint32_t c = bx; chunk_locate(a, c, ch); c += grid) {
      for (uint32_t t = 0; t < chunk_nt; t++) sort_zero(sh_cnt.data(), ch.nkeys, t, chunk_nt);
      for (uint32_t t = 0; t < chunk_nt; t++) chunk_hist(a, ch, t, chunk_nt, sh_cnt.data());
      const uint32_t total = block_scan(ch.nkeys, chunk_nt);
      for (uint32_t t = 0; t < chunk_nt; t++)
        chunk_reserve(a, ch, t, chunk_nt, runs[t], sh_cnt.data(), sh_loc.data(), sh_base.data());
      for (uint32_t t = 0; t < chunk_nt; t++) chunk_stage(a, ch, t, chunk_nt, sh_cnt.data(), sh_loc.data(), chunk_stage_buf.data());
      for (uint32_t t = 0; t < chunk_nt; t++)
        chunk_copy_out(a, ch, t, chunk_nt, sh_loc.data(), sh_base.data(), chunk_stage_buf.data());
      if (total != ch.hi - ch.lo) abort();
    }
}

extern "C" {
// The sort alone: scalars: batch * n canonical scalars; geometry as hs_msm_pipeline; lb: key bits per bin
// (0xffffffff: what msm.cu picks), T: entries per chunk, spb: scalars per bin-kernel block (0: what msm.cu picks),
// bin_nt / chunk_nt: threads per block of the bin / chunk kernels.  Writes counts (nb + 1: raw counts, then the
// max), off (nb + 1) and sorted[0 .. off[nb]) (at most cap words).  Returns nb, -1 on bad input.
int hs_msm_sort(const uint32_t* scalars, uint32_t n, uint32_t batch, uint32_t c, int fixed_base, uint32_t lo,
                uint32_t hi, uint32_t pad, uint32_t lb, uint32_t T, uint32_t spb, uint32_t bin_nt, uint32_t chunk_nt,
                uint32_t* counts_out, uint32_t* off_out, uint32_t* sorted_out, uint32_t cap) {
  if (!n || !batch || batch > 4 || (!fixed_base && batch != 1) || c < 1 || c > 16 || !T || !bin_nt || !chunk_nt)
    return -1;
  MsmGeom g;
  if (!msm_geom(n, batch, c, fixed_base, lo, hi, g)) return -1;
  if (lb == 0xffffffffu) lb = sort_default_lb(g.nb);
  if (((g.nb - 1) >> lb) >= PB_SORT_MAX_BINS || (1u << lb) > PB_SORT_MAX_BIN_KEYS) return -1;
  if (!spb) spb = PB_SORT_BIN_STAGE / g.W;
  std::vector<Fr> sc((size_t)batch * n);
  for (size_t i = 0; i < sc.size(); i++) sc[i] = ld<Fr>(scalars + 8 * i);
  std::vector<uint32_t> counts, off, sorted;
  host_msm_sort(g, sc, n, pad ? 1 : 0, lb, T, spb, bin_nt, chunk_nt, counts, off, sorted);
  if (off[g.nb] > cap) return -1;
  memcpy(counts_out, counts.data(), counts.size() * 4);
  memcpy(off_out, off.data(), off.size() * 4);
  memcpy(sorted_out, sorted.data(), (size_t)off[g.nb] * 4);
  return (int)g.nb;
}

// The whole bucket pipeline of msm.cu on the CPU, every thread body run in a loop: signed-digit slicing, the
// two-level counting sort, rounds of batched affine additions (msm_bucket.cuh), recursive bucket reduction,
// bucket-range offset and window Horner.  points: n canonical affine points (16 words each); scalars: batch * n
// canonical scalars; fixed_base != 0 builds the window table 2^(c w) P_i first (batch <= 4 scalar vectors share it).
// [lo, hi): the bucket magnitudes this "rank" owns.  out: one canonical affine point (+ identity flag) per scalar
// vector: the rank's partial sum.  Returns the number of accumulation rounds that did work, -1 on bad input.
int hs_msm_pipeline(const uint32_t* points, uint32_t n, const uint32_t* scalars, uint32_t batch, uint32_t c,
                    int fixed_base, uint32_t lo, uint32_t hi, uint32_t B, uint32_t g0, uint32_t* out, uint8_t* out_inf) {
  if (!n || !batch || batch > 4 || (!fixed_base && batch != 1) || c < 1 || c > 16 || B < 2 || B > PB_AFF_BMAX) return -1;
  if (g0 < 2 || (g0 & (g0 - 1))) return -1;
  MsmGeom g;
  if (!msm_geom(n, batch, c, fixed_base, lo, hi, g)) return -1;
  // point table
  std::vector<G1Affine> tab(fixed_base ? (size_t)g.W * n : n);
  for (uint32_t i = 0; i < n; i++) {
    tab[i].x = fp_to_mont(ld<Fq>(points + 16 * i));
    tab[i].y = fp_to_mont(ld<Fq>(points + 16 * i + 8));
  }
  if (fixed_base)
    for (uint32_t w = 1; w < g.W; w++)
      for (uint32_t i = 0; i < n; i++) {
        G1XYZZ a;
        g1_double_affine(a, tab[(size_t)(w - 1) * n + i]);
        for (uint32_t k = 1; k < c; k++) g1_double(a);
        g1_to_affine(a, tab[(size_t)w * n + i]);
      }
  std::vector<Fr> sc((size_t)batch * n);
  for (size_t i = 0; i < sc.size(); i++) sc[i] = ld<Fr>(scalars + 8 * i);
  // the two-level counting sort of msm.cu, padded, with the launch's bin width, chunk size and block sizes
  std::vector<uint32_t> counts, off, sorted;
  host_msm_sort(g, sc, n, 1, sort_default_lb(g.nb), PB_SORT_CHUNK, PB_SORT_BIN_STAGE / g.W, PB_SORT_BIN_THREADS,
                PB_SORT_CHUNK_THREADS, counts, off, sorted);
  const uint32_t maxc = counts[g.nb];
  // accumulation rounds
  const uint64_t positions = (uint64_t)n * g.W * batch + g.nb, s_bound = positions / 2;
  std::vector<G1Affine> pts(s_bound + 1);
  AffAcc a;
  a.table = tab.data();
  a.sorted = sorted.data();
  a.pts = pts.data();
  a.off = off.data();
  a.cnt = counts.data();
  a.max_cnt = counts.data() + g.nb;
  a.nbl = g.nb;
  a.B = B;
  Fq pref[PB_AFF_BMAX];
  uint32_t desc[PB_AFF_BMAX];
  int rounds = 0;
  for (uint32_t r = 0; r < 32; r++) {
    a.r = r;
    if (r > 0 && maxc > (1u << r)) rounds = r + 1;
    if (r == 0) rounds = 1;
    const uint64_t T = aff_round_threads(s_bound, B, r) + 40;  // spare threads must do nothing
    // descending thread order: a right-hand slot read late must still be intact (it is never written in its round)
    for (uint64_t t = T; t-- > 0;) {
      if (r == 0) aff_round0_thread(a, t, pref, desc);
      else aff_round_thread(a, t, pref, desc);
    }
  }
  // reduction
  ReduceArgs ra;
  ra.pts = pts.data(); ra.off = off.data(); ra.cnt = counts.data(); ra.xb = nullptr;
  ra.sets = g.sets; ra.m = g.nloc; ra.g = g0;
  std::vector<SR> cur((size_t)g.sets * reduce_groups(ra.m, ra.g)), nxt;
  ra.out = cur.data();
  for (uint64_t t = 0; t < cur.size() + 3; t++) reduce_level0_thread(ra, t);
  uint32_t m = reduce_groups(ra.m, ra.g), log_G = 0;
  while ((1u << log_G) < g0) log_G++;
  while (m > 8) {
    // the block-wide level (k_reduce_block in msm.cu), its phases run thread by thread
    const uint32_t chunks = reduce_chunks(m);
    nxt.assign((size_t)g.sets * chunks, SR());
    BlockLevelArgs ba;
    ba.in = cur.data(); ba.out = nxt.data(); ba.sets = g.sets; ba.m = m; ba.log_G = log_G;
    for (uint32_t set = 0; set < g.sets; set++)
      for (uint32_t chunk = 0; chunk < chunks; chunk++) {
        const uint32_t NT = PB_REDUCE_THREADS;
        std::vector<G1XYZZ> sh(NT), xs(NT), tmp(NT);
        for (uint32_t t = 0; t < NT; t++) blk_local(ba, set, chunk, t, sh[t], xs[t]);
        for (uint32_t d = 1; d < NT; d <<= 1) {
          for (uint32_t t = 0; t < NT; t++) tmp[t] = blk_scan_step(sh.data(), t, d);
          sh = tmp;
        }
        const G1XYZZ s_total = sh[0];
        for (uint32_t t = 0; t < NT; t++) tmp[t] = blk_weight(ba, t, xs[t], sh[t]);
        sh = tmp;
        for (uint32_t d = NT / 2; d > 0; d >>= 1)
          for (uint32_t t = 0; t < NT; t++) blk_tree_step(sh.data(), t, d);
        nxt[(size_t)set * chunks + chunk].S = s_total;
        nxt[(size_t)set * chunks + chunk].R = sh[0];
      }
    m = chunks;
    log_G += 9;
    cur.swap(nxt);
  }
  {  // the last <= 8 elements of every set: folded by the host code of msm.cu
    std::vector<SR> fin(g.sets);
    for (uint32_t s = 0; s < g.sets; s++) fin[s] = reduce_fold_final(cur.data() + (size_t)s * m, m, log_G);
    cur.swap(fin);
  }
  std::vector<G1XYZZ> ws(g.sets);
  for (uint32_t s = 0; s < g.sets; s++) {
    if (g.own_log) {  // strided shard: sum_k (G k + r + 1) B_k = G R + (r + 1 - G) S
      std::vector<SR> one(1, cur[s]);
      // a one-rank "join" with the rank's own coefficient: reuse the library's formula through its pieces
      G1XYZZ gr = cur[s].R;
      for (uint32_t k = 0; k < g.own_log; k++) g1_double(gr);
      G1XYZZ ms = G1XYZZ::identity();
      const uint32_t coef = (1u << g.own_log) - 1 - g.own_rank;  // subtract (G - 1 - r) S
      for (int i = 31; i >= 0; i--) { g1_double(ms); if ((coef >> i) & 1) g1_add(ms, cur[s].S); }
      ms.Y = fp_neg(ms.Y);
      g1_add(gr, ms);
      ws[s] = gr;
      continue;
    }
    ws[s] = cur[s].R;
    G1XYZZ ml = G1XYZZ::identity();
    for (int i = 31; i >= 0; i--) { g1_double(ml); if ((g.lo >> i) & 1) g1_add(ml, cur[s].S); }
    g1_add(ws[s], ml);
  }
  auto emit = [&](const G1XYZZ& r, uint32_t k) {
    G1Affine p;
    bool inf = g1_to_affine(r, p);
    out_inf[k] = inf ? 1 : 0;
    Fq x = fp_from_mont(p.x), y = fp_from_mont(p.y);
    st(out + 16 * k, x);
    st(out + 16 * k + 8, y);
  };
  if (fixed_base) {
    for (uint32_t k = 0; k < batch; k++) emit(ws[k], k);
  } else {
    G1XYZZ r = G1XYZZ::identity();
    for (int w = (int)g.W - 1; w >= 0; w--) {
      if (w != (int)g.W - 1) for (uint32_t k = 0; k < c; k++) g1_double(r);
      g1_add(r, ws[w]);
    }
    emit(r, 0);
  }
  return rounds;
}
}

extern "C" {
// field k of the proof layout: its label, -> is_point, step, block; null past the last field
const char* hs_proof_field(int k, int* is_point, int* step, int* block) {
  if (k < 0 || k >= PROOF_FIELDS) return nullptr;
  *is_point = PROOF_LAYOUT[k].is_point;
  *step = PROOF_LAYOUT[k].step;
  *block = (int)PROOF_LAYOUT[k].block;
  return PROOF_LAYOUT[k].label;
}
// challenge k: its label, -> step, block; null past the last challenge
const char* hs_proof_challenge(int k, int* step, int* block) {
  if (k < 0 || k >= PROOF_CHALLENGES) return nullptr;
  *step = CHALLENGE_LAYOUT[k].step;
  *block = (int)CHALLENGE_LAYOUT[k].block;
  return CHALLENGE_LAYOUT[k].label;
}
}

extern "C" {
// the prover's device bytes by count (memory_plan.cuh): out[0..3] = full circuit, proof, ntt, msm; out[4..7] = the same
// sliced.  Returns plan_choose for free_bytes: 0 full, 1 sliced, -1 neither fits.
int hs_prover_memory(int log_n, int n_custom, uint32_t msm_c, uint32_t msm_batch, uint64_t msm_now, uint64_t free_bytes,
                     int force_sliced, uint64_t* out) {
  const ProverMemory m = prover_memory(log_n, n_custom, msm_c, msm_batch, msm_now);
  const MemoryCount* c[2] = {&m.full, &m.sliced};
  for (int k = 0; k < 2; k++) {
    out[4 * k] = c[k]->circuit;
    out[4 * k + 1] = c[k]->proof;
    out[4 * k + 2] = c[k]->ntt;
    out[4 * k + 3] = c[k]->msm;
  }
  return plan_choose(m, free_bytes, force_sliced != 0);
}
}

extern "C" {
// The permutation of permutation.cu on the CPU: the same id check and keys, std::sort in place of the radix sort, the
// label body run for every sorted position.  ids: 3n ids, row-major L R O; omega: the n-th root of unity, canonical
// (8 words); out: S1 | S2 | S3, 3n canonical values.  Returns -1, or the index of the first bad id (nothing written).
int64_t hs_permutation(const int64_t* ids, int log_n, const uint32_t* omega, uint32_t* out) {
  const uint64_t n = (uint64_t)1 << log_n, m = 3 * n;
  const int cb = perm_cell_bits(log_n);
  int64_t max_id = -1;
  const int64_t bad = perm_check_ids(ids, m, &max_id);
  if (bad >= 0) return bad;
  std::vector<uint64_t> keys(m);
  for (uint64_t k = 0; k < m; k++) keys[k] = perm_key(ids[k], k, cb);
  std::sort(keys.begin(), keys.end());
  if (perm_sort_bits(log_n, max_id) < 64 && keys.back() >> perm_sort_bits(log_n, max_id)) abort();  // bits unused
  std::vector<Fr> wpow(n);
  const Fr w = fp_to_mont(ld<Fr>(omega));
  Fr cur = Fr::one();
  for (uint64_t i = 0; i < n; i++) { wpow[i] = fp_from_mont(cur); cur = fp_mul(cur, w); }
  std::vector<Fr> S(m);
  PermArgs a;
  a.keys = keys.data();
  a.wpow = wpow.data();
  a.S = S.data();
  a.n = n;
  a.m = m;
  a.cb = cb;
  for (uint64_t k = 0; k < m; k++) perm_label(a, k);
  for (uint64_t k = 0; k < m; k++) st(out + 8 * k, S[k]);
  return -1;
}
}

extern "C" {
// The wire solver of solve.cu on the CPU: the rows in row order, each defining row through the same solve_gate body.
// ids: 3n ids, row-major L R O, rows from m on unused; sel: QL QR QM QO QC (n canonical values each, 8 words a value);
// exps: six exponents per custom term, custom: their selectors; inputs: n_in ids and canonical values.  out: A | B | C.
// Returns 0, or 1 when a cell has no value (unset, or read by a defining row before its variable is defined).
int hs_solve(const int64_t* ids, int log_n, uint64_t m, const uint32_t* sel, int n_custom, const uint8_t* exps,
             const uint32_t* custom, uint64_t n_in, const int64_t* in_ids, const uint32_t* in_vals, uint32_t* out) {
  const uint64_t n = (uint64_t)1 << log_n;
  uint8_t f[PB_MAX_CUSTOM][3];
  for (int k = 0; k < n_custom; k++) {
    int s = 0;
    for (int w = 0; w < 6; w++)
      for (int t = 0; t < exps[6 * k + w]; t++) f[k][s++] = (uint8_t)w;
    while (s < 3) f[k][s++] = PB_FACTOR_ONE;
  }
  auto col = [&](const uint32_t* base, uint64_t c, uint64_t r) { return fp_to_mont(ld<Fr>(base + 8 * (c * n + r))); };
  std::unordered_map<int64_t, Fr> val;
  for (uint64_t k = 0; k < n_in; k++) val[in_ids[k]] = fp_to_mont(ld<Fr>(in_vals + 8 * k));
  auto get = [&](int64_t id, Fr* x) {
    if (id < 0) { *x = Fr::zero(); return true; }
    auto it = val.find(id);
    if (it == val.end()) return false;
    *x = it->second;
    return true;
  };
  for (uint64_t r = 0; r < m; r++) {
    const int64_t v = ids[3 * r + 2];
    SolveRow row;
    const Fr qo = col(sel, 3, r);
    bool defines = v >= 0 && !qo.is_zero() && !val.count(v);
    for (int k = 0; k < n_custom; k++) {
      row.q[k] = col(custom, k, r);
      if (solve_term_reads_c(f[k]) && !row.q[k].is_zero()) defines = false;
    }
    if (!defines) continue;
    Fr a, b;
    if (!get(ids[3 * r], &a) || !get(ids[3 * r + 1], &b)) return 1;
    row.ql = col(sel, 0, r);
    row.qr = col(sel, 1, r);
    row.qm = col(sel, 2, r);
    row.qc = col(sel, 4, r);
    row.neg_inv_qo = fp_neg(fp_inv_gcd(qo));
    val[v] = solve_gate(row, f, n_custom, a, b);
  }
  for (uint64_t c = 0; c < 3 * n; c++) {
    const uint64_t r = c / 3, w = c - 3 * r;
    Fr x = Fr::zero();
    if (r < m && !get(ids[c], &x)) return 1;
    st(out + 8 * (w * n + r), fp_from_mont(x));
  }
  return 0;
}

// hs_solve with rows that define from their table, through the same table index and solve_probe as solve.cu: qk and
// qt (NULL untagged) n canonical values each, tab the table columns t1 t2 t3 (t4) one after the other, rows values
// each.  The index is built here with std::sort and a fixed theta (stepped on a collision of words).  errs[0], errs[1]:
// the miss and ambiguous rows.  Returns 0, 1 as hs_solve, or 2 when errs is not zero.
int hs_solve_lookup(const int64_t* ids, int log_n, uint64_t m, const uint32_t* sel, int n_custom, const uint8_t* exps,
                    const uint32_t* custom, uint64_t n_in, const int64_t* in_ids, const uint32_t* in_vals,
                    const uint32_t* qk, const uint32_t* qt, const uint32_t* tab, uint64_t rows, uint32_t* out,
                    uint64_t* errs) {
  const uint64_t n = (uint64_t)1 << log_n;
  const int width = qt ? 4 : 3;
  uint8_t f[PB_MAX_CUSTOM][3];
  for (int k = 0; k < n_custom; k++) {
    int s = 0;
    for (int w = 0; w < 6; w++)
      for (int t = 0; t < exps[6 * k + w]; t++) f[k][s++] = (uint8_t)w;
    while (s < 3) f[k][s++] = PB_FACTOR_ONE;
  }
  // the index: distinct keys in ascending word order, none sharing a word
  std::vector<Fr> tm(width * rows);
  for (uint64_t k = 0; k < width * rows; k++) tm[k] = fp_to_mont(ld<Fr>(tab + 8 * k));
  SolveTable T = {};
  for (int w = 0; w < width; w++) T.t[w] = tm.data() + w * rows;
  auto tag_of = [&](uint64_t r) { return qt ? T.t[3][r] : Fr::zero(); };
  std::vector<std::pair<uint64_t, uint32_t>> kv(rows);
  std::vector<uint64_t> words;
  std::vector<uint32_t> keyrow;
  std::vector<uint8_t> amb;
  Fr seed = Fr::zero();
  seed.v[0] = 0x9e3779b9u;
  for (bool clean = false; !clean;) {
    seed.v[1]++;
    T.theta = fp_to_mont(seed);
    T.theta2 = fp_mul(T.theta, T.theta);
    for (uint64_t r = 0; r < rows; r++)
      kv[r] = {solve_table_word(tag_of(r), T.t[0][r], T.t[1][r], T.theta, T.theta2), (uint32_t)r};
    std::sort(kv.begin(), kv.end());
    words.clear(), keyrow.clear(), amb.clear();
    clean = true;
    for (uint64_t k = 0; k < rows && clean; k++) {
      const uint32_t r = kv[k].second;
      if (k == 0 || kv[k].first != kv[k - 1].first) {
        words.push_back(kv[k].first), keyrow.push_back(r), amb.push_back(0);
        continue;
      }
      const uint32_t p = kv[k - 1].second;
      if (T.t[0][r] != T.t[0][p] || T.t[1][r] != T.t[1][p] || tag_of(r) != tag_of(p)) clean = false;
      if (T.t[2][r] != T.t[2][p]) amb.back() = 1;
    }
  }
  T.word = words.data();
  T.row = keyrow.data();
  T.amb = amb.data();
  T.n_keys = words.size();

  auto col = [&](const uint32_t* base, uint64_t c, uint64_t r) { return fp_to_mont(ld<Fr>(base + 8 * (c * n + r))); };
  std::unordered_map<int64_t, Fr> val;
  for (uint64_t k = 0; k < n_in; k++) val[in_ids[k]] = fp_to_mont(ld<Fr>(in_vals + 8 * k));
  auto get = [&](int64_t id, Fr* x) {
    if (id < 0) { *x = Fr::zero(); return true; }
    auto it = val.find(id);
    if (it == val.end()) return false;
    *x = it->second;
    return true;
  };
  errs[0] = errs[1] = 0;
  for (uint64_t r = 0; r < m; r++) {
    const int64_t v = ids[3 * r + 2];
    if (v < 0 || val.count(v)) continue;
    SolveRow row;
    const Fr qo = col(sel, 3, r);
    bool gate = !qo.is_zero();
    for (int k = 0; k < n_custom; k++) {
      row.q[k] = col(custom, k, r);
      if (solve_term_reads_c(f[k]) && !row.q[k].is_zero()) gate = false;
    }
    const bool table = qo.is_zero() && !ld<Fr>(qk + 8 * r).is_zero();
    if (!gate && !table) continue;
    Fr a, b;
    if (!get(ids[3 * r], &a) || !get(ids[3 * r + 1], &b)) return 1;
    if (table) {
      Fr c;
      const Fr tag = qt ? fp_to_mont(ld<Fr>(qt + 8 * r)) : Fr::zero();
      const int e = solve_probe(T, tag, a, b, &c);
      if (e != PB_SOLVE_HIT) errs[e - 1]++;
      val[v] = c;
      continue;
    }
    row.ql = col(sel, 0, r);
    row.qr = col(sel, 1, r);
    row.qm = col(sel, 2, r);
    row.qc = col(sel, 4, r);
    row.neg_inv_qo = fp_neg(fp_inv_gcd(qo));
    val[v] = solve_gate(row, f, n_custom, a, b);
  }
  for (uint64_t c = 0; c < 3 * n; c++) {
    const uint64_t r = c / 3, w = c - 3 * r;
    Fr x = Fr::zero();
    if (r < m && !get(ids[c], &x)) return 1;
    st(out + 8 * (w * n + r), fp_from_mont(x));
  }
  return errs[0] || errs[1] ? 2 : 0;
}
}
