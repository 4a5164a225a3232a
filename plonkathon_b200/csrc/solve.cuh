// Wire values of a circuit from its inputs (solve.cu): the gate body of a defining row, shared by the GPU solver and
// csrc/host_selftest.cpp, which runs it on the CPU in row order.
//
// A defining row r sets its O variable to c = -(QL a + QR b + QM a b + QC + sum_k Q_k m_k(a, b, 0)) / QO.  A row
// defines only when no custom term whose selector is non-zero there reads c or the next row, so m_k is evaluated
// with c and the next row's wires 0: every term that contributes is one in a and b alone.
#pragma once
#include "custom_terms.cuh"

namespace pb200 {

#define PB_SOLVE_NONE 0xffffffffu  // no defining row / no input

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

}  // namespace pb200
