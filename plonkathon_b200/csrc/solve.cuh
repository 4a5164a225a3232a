// Wire values of a circuit from its inputs (solve.cu): the gate body of a defining row and the table probe of a row
// that defines from its table, shared by the GPU solver and csrc/host_selftest.cpp, which runs them on the CPU in row
// order.
//
// A defining row r sets its O variable to c = -(QL a + QR b + QM a b + QC + sum_k Q_k m_k(a, b, 0)) / QO.  A row
// defines only when no custom term whose selector is non-zero there reads c or the next row, so m_k is evaluated
// with c and the next row's wires 0: every term that contributes is one in a and b alone.
#pragma once
#include "custom_terms.cuh"

namespace pb200 {

#define PB_SOLVE_NONE 0xffffffffu  // no defining row / no input

// ---- the arguments of solve_run (plonk_b200.h has their meaning) -----------------------------------------------------
// the circuit, its inputs and the outputs, as pb200_solve_wires takes them; lists holds 3, 5 (table) or 8 (shuffle)
// times limit entries, counts 2 or 4
struct SolveArgs {
  const int64_t* ids;
  int log_n;
  uint64_t n_constraints;
  const uint8_t* const* sel;  // QL QR QM QO QC
  int n_custom;
  const uint8_t* exps;
  const uint8_t* const* custom;
  uint64_t n_inputs;
  const int64_t* in_ids;
  const uint8_t* in_vals;
  uint32_t limit;
  uint64_t* counts;
  uint32_t* lists;
  void* const* out;
  bool out_on_device;
};
// rows that define from their table (pb200_solve_wires_lookup): q_K, Q_T and t4 (both null for one untagged table),
// t1 t2 t3, the table's rows, and where the listed miss and ambiguous rows' operands go (or null)
struct SolveTableArgs {
  const uint8_t* qk;
  const uint8_t* qtag;
  const uint8_t* tab[4];
  uint64_t rows;
  uint8_t* operands;
};
// a shuffle (pb200_solve_wires_shuffle): q_in and q_out
struct SolveShuffleArgs {
  const uint8_t* qin;
  const uint8_t* qout;
};

// the selectors of one row, Montgomery; neg_inv_qo = -1 / QO
struct SolveRow {
  Fr ql, qr, qm, qc, neg_inv_qo;
  Fr q[PB_MAX_CUSTOM];
};

// custom term factors (CustomTerms::f) that read c or the next row: a row where such a term's selector is non-zero
// does not define its O variable
PB_HD bool solve_term_reads_c(const uint8_t* f) {
  for (int s = 0; s < 3; s++)
    if (f[s] >= 2 && f[s] != PB_FACTOR_ONE) return true;
  return false;
}

// c of a defining row, Montgomery
PB_HD Fr solve_gate(const SolveRow& s, const uint8_t (*f)[3], int n_custom, const Fr& a, const Fr& b) {
  Fr acc = fp_add(fp_mul(a, s.ql), fp_mul(b, s.qr));
  acc = fp_add(acc, fp_mul(fp_mul(a, b), s.qm));
  acc = fp_add(acc, s.qc);
  const Fr z = Fr::zero();
  for (int k = 0; k < PB_MAX_CUSTOM; k++) {
    if (k >= n_custom) break;
    acc = fp_add(acc, fp_mul(custom_monomial_next(a, b, z, z, z, z, f[k]), s.q[k]));
  }
  return fp_mul(acc, s.neg_inv_qo);
}

// ---- rows that define from their table (pb200_solve_wires_lookup) ----------------------------------------------------
// A row r with q_K != 0 and QO = 0 sets c = t3 of the table rows whose (t4, t1, t2) equal (Q_T[r], a, b) (t4 = Q_T = 0
// for one untagged table).  The table index holds the distinct keys (tag, t1, t2) of the table in ascending order of
// their word (solve_table_word), with no two keys sharing a word (theta is drawn again until none do); for each key
// one table row that carries it, and whether the table rows with that key give two different t3.
struct SolveTable {
  const uint64_t* word;  // n_keys words, ascending and distinct
  const uint32_t* row;   // a table row with each key
  const uint8_t* amb;    // 1 where the rows with the key disagree on t3
  const Fr* t[4];        // t1 t2 t3 t4, Montgomery; t[3] null for one untagged table
  uint64_t n_keys;
  Fr theta, theta2;  // Montgomery
};

#define PB_SOLVE_HIT 0
#define PB_SOLVE_MISS 1
#define PB_SOLVE_AMBIGUOUS 2

// the 64-bit word of a key: the low word of t1 + theta t2 + theta^2 tag (Montgomery)
PB_HD uint64_t solve_table_word(const Fr& tag, const Fr& x, const Fr& y, const Fr& theta, const Fr& theta2) {
  const Fr h = fp_add(x, fp_add(fp_mul(theta, y), fp_mul(theta2, tag)));
  return (uint64_t)h.v[0] | ((uint64_t)h.v[1] << 32);
}

// c of a row that reads (a, b) from table `tag` (zero untagged), Montgomery.  The word only finds the one key that can
// match; whether it does is decided on full values.  PB_SOLVE_MISS: no table row has the key; PB_SOLVE_AMBIGUOUS: its
// rows give two different t3.  Both leave c = 0.
PB_HD int solve_probe(const SolveTable& T, const Fr& tag, const Fr& a, const Fr& b, Fr* c) {
  *c = Fr::zero();
  const uint64_t w = solve_table_word(tag, a, b, T.theta, T.theta2);
  uint64_t lo = 0, hi = T.n_keys;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) / 2;
    if (T.word[mid] < w) lo = mid + 1;
    else hi = mid;
  }
  if (lo == T.n_keys || T.word[lo] != w) return PB_SOLVE_MISS;
  const uint32_t r = T.row[lo];
  if (T.t[0][r] != a || T.t[1][r] != b || (T.t[3] && T.t[3][r] != tag)) return PB_SOLVE_MISS;
  if (T.amb[lo]) return PB_SOLVE_AMBIGUOUS;
  *c = T.t[2][r];
  return PB_SOLVE_HIT;
}

}  // namespace pb200
