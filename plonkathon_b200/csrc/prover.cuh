// Prover state shared between prover.cu (the rounds) and capi.cu (the C ABI accessors).
#pragma once
#include "common.cuh"
#include "proof_layout.cuh"
#include "custom_terms.cuh"

namespace pb200 {

struct Srs;
void srs_msm(Context* ctx, Srs* srs, const Fr* d_scalars, uint64_t m, bool scalars_mont, uint8_t* out_xy, int* is_identity);
void srs_msm_batch(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t m, bool scalars_mont,
                   uint8_t* out_xy, int* is_identity);
void srs_msm_batch_partial(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t first,
                           uint64_t count, uint32_t bucket_lo, uint32_t bucket_hi, bool scalars_mont, G1XYZZ* out);
void srs_msm_batch_sharded(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t m,
                           bool scalars_mont, uint8_t* out_xy, int* is_identity);
uint32_t srs_bucket_count(Srs* s);

#define PB_SLICED_WHY "not available on a sliced prover (its 4n-coset cache does not fit in device memory, or PB200_SLICED=1): "
// sum_k Q_k[i] m_k(a, b, c), unrolled over the PB_MAX_CUSTOM slots so the kernel parameters are indexed statically
// (a dynamic index would copy them to local memory); count == 0 costs one uniform branch
#ifdef __CUDACC__
__device__ __forceinline__ Fr custom_gate_sum(const CustomTerms& t, uint64_t i, const Fr& a, const Fr& b, const Fr& c,
                                              Fr acc) {
#pragma unroll
  for (int k = 0; k < PB_MAX_CUSTOM; k++) {
    if (k >= t.count) break;
    const Fr q = ldg_fr(t.Q[k] + i);
    acc = fp_add(acc, fp_mul(custom_monomial(a, b, c, t.f[k]), q));
  }
  return acc;
}
// the same for a next-row prover: an, bn, cn are the wires of the next row (index + 1 mod n, or X -> wX on a coset)
__device__ __forceinline__ Fr custom_gate_sum_next(const CustomTerms& t, uint64_t i, const Fr& a, const Fr& b,
                                                   const Fr& c, const Fr& an, const Fr& bn, const Fr& cn, Fr acc) {
#pragma unroll
  for (int k = 0; k < PB_MAX_CUSTOM; k++) {
    if (k >= t.count) break;
    const Fr q = ldg_fr(t.Q[k] + i);
    acc = fp_add(acc, fp_mul(custom_monomial_next(a, b, c, an, bn, cn, t.f[k]), q));
  }
  return acc;
}
#endif

// the order of the sorted table copy: (t1, t2, t3[, t4]) lexicographically, each by Montgomery limbs from the top.
// width 3 for one untagged table, 4 with the table tag t4 (y[3] is read only then).  Unrolled, so y stays in registers.
// The prover's table index (k_lookup_index) and the witness check (k_check_lookup) both search with it.
PB_HD int lookup_cmp(const Fr* x, const Fr (&y)[4], int width) {
#pragma unroll
  for (int w = 0; w < 4; w++) {
    if (w == width) break;
#pragma unroll
    for (int l = 7; l >= 0; l--)
      if (x[w].v[l] != y[w].v[l]) return x[w].v[l] < y[w].v[l] ? -1 : 1;
  }
  return 0;
}

struct Prover {
  Context* ctx;
  Srs* srs;
  int log_n;
  uint64_t n;
  // One proof across the GPUs of a box (world > 1; the context carries the communicator): rank r owns every
  // world-th point of the 4n coset -- x_j = g mu^(world j + r), j < n_ext = 4n / world, itself a coset of the subgroup
  // of order n_ext -- so the coset extensions, the cached selector extensions and the quotient are local and divide by
  // world; inverse transforms are slab-sharded with one allgather at the join (ntt_shard.cuh); commitments split the
  // buckets (msm.cu).  world == 1 is the same code with n_ext = 4n.
  int world = 1, rank = 0, log_world = 0;
  int log_ext = 0;       // log2(n_ext)
  uint64_t n_ext = 0;
  uint32_t fold = 1;     // n / n_ext when the coset slice is shorter than a coefficient vector (world = 8), else 1
  uint64_t zw_shift = 4; // Z(w x_j) = Z-extension at local index j + 4 / world ...
  bool zw_separate = false;  // ... or, when 4 % world != 0, a separately extended vector (ext[5])
  // One GPU whose 4n-coset cache does not fit its memory (memory_plan.cuh), or PB200_SLICED=1: round 3 walks the four
  // n-point slices {g mu^(4j + r)} in turn, as the ranks of a 4-GPU sharded prover would, and joins them on the device.
  // sel_ext, xs, pi_basis[0] and ext[] then hold one slice (n points), recomputed for each; tq holds T's 3n
  // coefficients.  Plain circuits and same-row custom terms only: zero knowledge, lookups, shuffles and next-row terms
  // are refused (PB_SLICED_WHY).
  bool sliced = false;
  // per-circuit (all Montgomery)
  DevBuf sel_coeff[8 + PB_MAX_CUSTOM];   // QM QL QR QO QC S1 S2 S3, then the custom selectors; coefficient form
  DevBuf sel_lag[8 + PB_MAX_CUSTOM];     // same, Lagrange values (QM..QC and custom for the gate check, S1..S3 for round 2)
  DevBuf sel_ext[8 + PB_MAX_CUSTOM];     // same, on this rank's slice of the fixed 4n coset
  int n_custom = 0;
  uint8_t custom_f[PB_MAX_CUSTOM][3];    // monomial factors of each custom term (CustomTerms::f)
  // Next-row terms (pb200_prover_create_custom_next_row, one GPU): some term reads a(wX), b(wX) or c(wX).  Round 4 also
  // evaluates A, B, C at zeta w, the zeta w opening batches them with Z, and the proof has 864 bytes.
  bool next_row = false;
  Fr nr_ev[3];                           // a(zeta w), b(zeta w), c(zeta w), Montgomery
  DevBuf roots;          // w^i, i < n
  DevBuf gpow;           // (g mu^rank)^i, i < n     (coset shift on load)
  DevBuf gpow_w;         // (g mu^(rank+4))^i, i < n (only when zw_separate)
  DevBuf ginv_pow;       // g^-i, i < 4n            (undo the shift on store)
  DevBuf xs;             // x_j, j < n_ext
  Fr g, g_inv, zh_inv[4];
  Fr zh[4];              // Z_H(x_j) = x_j^n - 1 for j mod 4 (Montgomery)
  // per-proof state
  DevBuf lag[4];         // A B C Z Lagrange
  DevBuf coeff[5];       // a b c z pi coefficients
  DevBuf pi_lag;
  DevBuf ext[6];         // A B C Z PI Z(wX) on the slice
  DevBuf tq;             // quotient evaluations (n_ext) / coefficients (4n; sharded: 3n coefficients)
  DevBuf tq_loc;         // sharded: quotient evaluations on the slice
  DevBuf tmp[5];
  DevBuf aux_tmp;        // pass buffer of the side-stream coset transforms (n_ext)
  bool overlap = true;   // run the round-3 coset extensions of A, B, C (and Z) beside the round-1/2 MSMs
  DevBuf flags;
  Fr beta, gamma, alpha, fft_cofactor, zeta, v;   // Montgomery
  Fr ev[6];                                      // Montgomery evaluations (round 4)
  Fr pi_ev;
  // public inputs: when there are at most 8, PI is a combination of cached Lagrange-basis coset vectors
  uint64_t n_public = 0;
  bool pi_sparse = false;
  std::vector<DevBuf> pi_basis;   // L_i on the slice (n_ext each), i < 8; always holds L0 (the quotient's L0 term)
  std::vector<Fr> pub_neg;        // -public_i, Montgomery (host)
  // Zero knowledge (one GPU only): the blinding of the PLONK paper with 11 scalars b1..b11 per proof.  The unblinded
  // n-coefficient vectors above stay as they are (the coset extensions read them; k_quotient adds the Z_H multiples);
  // the blinded vectors, which are longer than n, live in their own zero-padded buffers of n + 8 elements.
  // With a lookup table (pb200_prover_set_zk_lookup) there are 21 scalars: b12..b21 blind F, H1, H2 and Z2.  A next-row
  // prover takes 14: b12..b14 give A, B, C a third blinder each (they are opened at zeta and at zeta w), so T3' has
  // n + 9 coefficients and the blinded vectors get ZK_NR_PAD elements of padding.
  // With a shuffle (pb200_prover_set_zk_shuffle) Z3 takes three more, always the last three: 14 scalars, 17 next-row.
  static const int ZK_BLINDERS = 11, ZK_LK_BLINDERS = 21, ZK_NR_BLINDERS = 14, ZK_PAD = 8, ZK_NR_PAD = 9;
  static const int ZK_SH_BLINDERS = 14, ZK_NR_SH_BLINDERS = 17;
  bool zk = false;
  bool zk_fixed = false;          // the same blinders for every proof (zk_fixed_b) instead of fresh OS randomness
  Fr zk_fixed_b[ZK_LK_BLINDERS];  // canonical
  Fr zk_b[ZK_LK_BLINDERS];        // this proof's b1..b11 (..b14 next-row, ..b21 lookups), Montgomery (drawn in round 1)
  DevBuf zk_coeff[4];             // A' B' C' (n + 2 coefficients, n + 3 next-row) Z' (n + 3)
  DevBuf zk_t[3];                 // T1' T2' (n + 1 coefficients) T3' (n + 6, n + 9 next-row)
  DevBuf zk_lk[5];                // lookups: T (n, zero padded) F' H2' (n + 2) H1' Z2' (n + 3), indexed by LK_*
  DevBuf zk_z3;                   // shuffles: Z3' (n + 3, zero padded)
  int zk_blinders() const {
    if (lk) return ZK_LK_BLINDERS;
    if (sh) return next_row ? ZK_NR_SH_BLINDERS : ZK_SH_BLINDERS;
    return next_row ? ZK_NR_BLINDERS : ZK_BLINDERS;
  }
  const Fr* zk_z3_b() const { return zk_b + zk_blinders() - 3; }  // Z3's X^2, X and constant blinders
  uint64_t zk_pad() const { return next_row ? ZK_NR_PAD : ZK_PAD; }
  uint64_t zk_t3_len() const { return n + (next_row ? 9 : 6); }  // coefficients of T3' (deg T <= 3n + 5, or 3n + 8)
  // Lookup argument (prover_set_lookup, one GPU): plookup over one fixed table of three columns, or over several
  // tables told apart by a tag column t4 and the selector Q_T, see "lookups" in prover.cu.  The proof gains f_1 h1_1
  // h2_1 z2_1 and six evaluations (1216 bytes).
  enum { LK_T = 0, LK_F, LK_H1, LK_H2, LK_Z2, LK_VECS };
  bool lk = false;
  // the coefficient vectors a lookup proof commits and opens: the unblinded lk_coeff, or zk_lk in zero-knowledge mode
  const Fr* lk_poly(int k) const { return (zk ? zk_lk[k] : lk_coeff[k]).as<Fr>(); }
  bool lk_tagged = false;              // several tables: t4 and Q_T are set (and lk_keys has 4 Fr per row)
  uint64_t lk_rows = 0;                // table rows before padding
  DevBuf lk_qk_coeff, lk_qk_ext;       // q_K: coefficients, on the 4n coset
  DevBuf lk_qk_lag;                    // q_K Lagrange values (Montgomery 0 / 1)
  DevBuf lk_qt_lag, lk_qt_coeff, lk_qt_ext;  // Q_T (table id per lookup row): Lagrange, coefficients, 4n coset
  DevBuf lk_tab[4];                    // t1 t2 t3 (t4 if tagged), Lagrange, padded to n by repeating the last row
  DevBuf lk_keys;                      // the table rows sorted by their Montgomery limbs (3 or 4 Fr per row) ...
  DevBuf lk_keys_idx;                  // ... and their original indices (uint32); equal rows keep table order
  DevBuf lk_j;                         // per row: table index j_i (uint32, n)
  DevBuf lk_cnt;                       // rows per table entry (uint32, n), zeroed by the scan
  DevBuf lk_off;                       // exclusive scan of lk_cnt (uint32, n + 1)
  DevBuf lk_sidx;                      // per position of s: its table entry (uint32, 2n)
  DevBuf lk_lag[LK_VECS];              // T F H1 H2 Z2: Lagrange values ...
  DevBuf lk_coeff[LK_VECS];            // ... coefficients ...
  DevBuf lk_ext[LK_VECS];              // ... on the 4n coset
  Fr eta, delta, epsilon;              // Montgomery
  Fr lk_ev[6];                         // f, t, t(zeta w), h2, h1(zeta w), z2(zeta w) at their points (Montgomery)
  // Shuffle argument (prover_set_shuffle, one GPU): the multiset of (a, b, c) over the rows with q_in = 1 equals the one
  // over the rows with q_out = 1, see "shuffle" in prover.cu.  The proof gains z3_1, q_in(zeta) and Z3(zeta w) (896
  // bytes, 992 on a next-row prover).
  enum { SH_IN = 0, SH_OUT };
  bool sh = false;
  DevBuf sh_lag[2];                    // Q_in Q_out: Lagrange values (Montgomery 0 / 1) ...
  DevBuf sh_coeff[2];                  // ... coefficients ...
  DevBuf sh_ext[2];                    // ... on the 4n coset
  DevBuf sh_z3_lag, sh_z3_coeff, sh_z3_ext;  // Z3: Lagrange values, coefficients, on the 4n coset
  // the coefficient vector of Z3 a proof commits and opens: the unblinded sh_z3_coeff, or zk_z3 in zero-knowledge mode
  const Fr* sh_z3_poly() const { return (zk ? zk_z3 : sh_z3_coeff).as<Fr>(); }
  Fr theta, kappa;                     // Montgomery
  Fr sh_ev[2];                         // q_in(zeta), Z3(zeta w) (Montgomery)
  // The proof's fields (proof_layout.cuh), canonical little-endian, indexed by ProofField: a point x||y, a scalar in
  // the first 32 bytes.  The rounds write them; only the fields of this prover's blocks are part of its proof.
  uint8_t fields[PROOF_FIELDS][64];
  // The witness check (check.cu): the copy permutation sigma as 3n uint32 cell indices, built on the first check and
  // kept (12n bytes).  No round reads it.
  DevBuf chk_sigma;
  bool sharded = false;  // made by a _sharded entry point (the witness check refuses it, whatever the world size)
  unsigned blocks() const {
    return (next_row ? BLOCK_NEXT_ROW : 0) | (sh ? BLOCK_SHUFFLE : 0) | (lk ? BLOCK_LOOKUP : 0);
  }

  enum { QM = 0, QL, QR, QO, QC, S1, S2, S3, CUSTOM0 };

  // the custom selectors from one of the per-circuit caches
  CustomTerms custom_terms(const DevBuf* sel) const {
    CustomTerms t;
    t.count = n_custom;
    for (int k = 0; k < PB_MAX_CUSTOM; k++) {
      t.Q[k] = k < n_custom ? sel[CUSTOM0 + k].as<Fr>() : nullptr;
      for (int s = 0; s < 3; s++) t.f[k][s] = custom_f[k][s];
    }
    return t;
  }

  // several commitments in one pass over the SRS (out: count * 64 bytes, contiguous)
  void commit_batch(const Fr* const* d_coeffs, uint32_t count, uint64_t m, uint8_t* out_xy) {
    int ident[4] = {0, 0, 0, 0};
    if (world > 1) srs_msm_batch_sharded(ctx, srs, d_coeffs, count, m, true, out_xy, ident);
    else srs_msm_batch(ctx, srs, d_coeffs, count, m, true, out_xy, ident);
    for (uint32_t k = 0; k < count; k++)
      PB_CHECK(!ident[k], "commitment is the point at infinity (unsupported by the reference transcript)");
  }
  void commit(const Fr* d_coeffs, uint64_t m, uint8_t* out_xy) { commit_batch(&d_coeffs, 1, m, out_xy); }
};


}  // namespace pb200
