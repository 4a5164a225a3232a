// Custom gate terms and their monomials, shared by the prover (prover.cuh), the wire solver (solve.cuh) and the CPU
// self-test (host_selftest.cpp).
#pragma once
#include "field.cuh"

namespace pb200 {

// Custom gate terms: the gate constraint gains sum_k Q_k a^i_k b^j_k c^l_k, total degree 2 or 3 (so T stays below
// degree 3n and the proof keeps its shape).  A term is stored as the factors of its monomial: up to 3 of {0 a, 1 b,
// 2 c, 3 a(wX), 4 b(wX), 5 c(wX)}, unused slots PB_FACTOR_ONE.  Factors 3..5 (next-row terms, degree 1 to 3) occur only
// on a prover made by pb200_prover_create_custom_next_row (Prover::next_row).
#define PB_MAX_CUSTOM 4
#define PB_FACTOR_ONE 6
struct CustomTerms {
  const Fr* Q[PB_MAX_CUSTOM];
  uint8_t f[PB_MAX_CUSTOM][3];
  int count;
};
// m_k(a, b, c) of a same-row term (degree 2 or 3) with degree - 1 products; the wires are selected by value so a, b, c
// stay in registers
PB_HD Fr custom_monomial(const Fr& a, const Fr& b, const Fr& c, const uint8_t* f) {
  auto pick = [&](uint8_t w) -> Fr { return w == 0 ? a : (w == 1 ? b : c); };
  Fr m = fp_mul(pick(f[0]), pick(f[1]));
  if (f[2] < 3) m = fp_mul(m, pick(f[2]));
  return m;
}
// m_k(a, b, c, a', b', c') of any term of a next-row prover (degree 1 to 3), a' = a(wX)
PB_HD Fr custom_monomial_next(const Fr& a, const Fr& b, const Fr& c, const Fr& an, const Fr& bn, const Fr& cn,
                              const uint8_t* f) {
  auto pick = [&](uint8_t w) -> Fr {
    return w == 0 ? a : w == 1 ? b : w == 2 ? c : w == 3 ? an : w == 4 ? bn : cn;
  };
  Fr m = pick(f[0]);
  if (f[1] != PB_FACTOR_ONE) m = fp_mul(m, pick(f[1]));
  if (f[2] != PB_FACTOR_ONE) m = fp_mul(m, pick(f[2]));
  return m;
}
}  // namespace pb200
