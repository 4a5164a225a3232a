// BN254 G1 (y^2 = x^3 + 3 over Fq) group law for the MSM kernels.
//
// Replaces py_ecc.bn128 `add` / `double` (one Fq inversion per operation; SURVEY App. A) as used by
// curve.py:38-111 `ec_lincomb`.  Accumulators use extended Jacobian "XYZZ" coordinates
// (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2; identity <=> ZZ == 0) so an affine point is added with
// 8 mul + 2 sqr and no inversion; a single inversion happens in g1_to_affine at the very end.
// Formulas: the standard madd-2008-s / add-2008-s / dbl-2008-s-1 sets for short Weierstrass curves
// with a = 0.  All coordinates are Montgomery-form Fq, fully reduced; inside an addition the intermediates are lazy
// (field.cuh: in [0, 2p)), which saves the final subtraction of most products, and Y3's difference of two products
// takes one reduction.  All exceptional cases the reference's tests reach are handled: identity operands, P + P
// (doubling), P + (-P).
#pragma once
#include "field.cuh"

namespace pb200 {

struct alignas(16) G1Affine {
  Fq x, y;
};

struct alignas(16) G1XYZZ {
  Fq X, Y, ZZ, ZZZ;
  PB_HD bool is_inf() const { return ZZ.is_zero(); }
  static PB_HD G1XYZZ identity() {
    G1XYZZ r;
    r.X = Fq::zero(); r.Y = Fq::zero(); r.ZZ = Fq::zero(); r.ZZZ = Fq::zero();
    return r;
  }
};

PB_HD G1XYZZ g1_from_affine(const G1Affine& p) {
  G1XYZZ r;
  r.X = p.x; r.Y = p.y; r.ZZ = Fq::one(); r.ZZZ = Fq::one();
  return r;
}

// acc = 2 * (affine p)
PB_HD void g1_double_affine(G1XYZZ& acc, const G1Affine& p) {
  Fq U = fp_dbl(p.y);
  Fq V = fp_sqr(U);
  Fq W = fp_mul(U, V);
  Fq S = fp_mul(p.x, V);
  Fq M = fp_sqr(p.x);
  M = fp_add(fp_dbl(M), M);
  Fq X3 = fp_sub(fp_sqr(M), fp_dbl(S));
  acc.Y = fp_mul2_lazy(M, fp_sub(S, X3), W, fp_neg_lazy(p.y));  // M (S - X3) - W y: all factors <= p
  fp_reduce_once(acc.Y);
  acc.X = X3;
  acc.ZZ = V;
  acc.ZZZ = W;
}

PB_HD void g1_double(G1XYZZ& a) {
  if (a.is_inf()) return;
  Fq U = fp_dbl(a.Y);
  Fq V = fp_sqr(U);
  Fq W = fp_mul(U, V);
  Fq S = fp_mul(a.X, V);
  Fq M = fp_sqr(a.X);
  M = fp_add(fp_dbl(M), M);
  Fq X3 = fp_sub(fp_sqr(M), fp_dbl(S));
  a.Y = fp_mul2_lazy(M, fp_sub(S, X3), W, fp_neg_lazy(a.Y));
  fp_reduce_once(a.Y);
  a.X = X3;
  a.ZZ = fp_mul(V, a.ZZ);
  a.ZZZ = fp_mul(W, a.ZZZ);
}

// The common part of the additions: from Pd = U2 - U1 (nonzero mod p) and Rd = S2 - S1,
//   PP = Pd^2, PPP = Pd PP, Q = U1 PP, X3 = Rd^2 - PPP - 2Q, Y3 = Rd (Q - X3) - S1 PPP,
//   ZZ3 = Z2 PP, ZZZ3 = Z3 PPP   (Z2, Z3: ZZ1 and ZZZ1, times ZZ2 and ZZZ2 in a full addition).
// Ranges, with p < 0.19 R: U1, S1 canonical; U2, S2 lazy products of canonical values (< 1.19p), so Pd, Rd =
// fp_sub(U2 or S2, canonical) < 1.19p; Z2, Z3 < 1.19p.  Then PP < 1.27p, PPP < 1.29p, Q < 1.24p, and Q - X3 < 1.24p,
// so Rd (Q - X3) + (p - S1) PPP < 2.77p^2 < pR and Y3 needs one reduction.  All four outputs leave canonical.
// The order (each factor used up as early as possible) keeps the accumulation kernel within 128 registers.
PB_HD void g1_add_tail(const Fq& U1, const Fq& S1, const Fq& Pd, const Fq& Rd, const Fq& Z2, const Fq& Z3, G1XYZZ& r) {
  const Fq PP = fp_sqr_lazy(Pd);
  r.ZZ = fp_mul(Z2, PP);
  const Fq PPP = fp_mul_lazy(Pd, PP);
  r.ZZZ = fp_mul(Z3, PPP);
  const Fq Q = fp_mul_lazy(U1, PP);
  r.X = fp_sub_lazy(fp_sub_lazy(fp_sub_lazy(fp_sqr_lazy(Rd), PPP), Q), Q);
  fp_reduce_once(r.X);
  r.Y = fp_mul2_lazy(Rd, fp_sub(Q, r.X), fp_neg_lazy(S1), PPP);
  fp_reduce_once(r.Y);
}

// acc += p (p affine, never the identity)
PB_HD void g1_add_mixed(G1XYZZ& acc, const G1Affine& p) {
  if (acc.is_inf()) {
    acc = g1_from_affine(p);
    return;
  }
  Fq U2 = fp_mul_lazy(p.x, acc.ZZ);
  Fq S2 = fp_mul_lazy(p.y, acc.ZZZ);
  Fq Pd = fp_sub(U2, acc.X);
  Fq Rd = fp_sub(S2, acc.Y);
  if (fp_is_zero_lazy(Pd)) {
    if (fp_is_zero_lazy(Rd)) g1_double_affine(acc, p);
    else acc = G1XYZZ::identity();
    return;
  }
  G1XYZZ r;
  g1_add_tail(acc.X, acc.Y, Pd, Rd, acc.ZZ, acc.ZZZ, r);
  acc = r;
}

// acc += p with (almost) uniform control flow for SIMT execution: every lane runs the same 8M + 2S
// sequence; an empty accumulator is handled by a select at the end instead of an early return, and only
// the rare P == +-Q cases branch.
PB_HD void g1_add_mixed_uniform(G1XYZZ& acc, const G1Affine& p) {
  const bool was_inf = acc.is_inf();
  Fq U2 = fp_mul_lazy(p.x, acc.ZZ);
  Fq S2 = fp_mul_lazy(p.y, acc.ZZZ);
  Fq Pd = fp_sub(U2, acc.X);
  Fq Rd = fp_sub(S2, acc.Y);
  if (!was_inf && fp_is_zero_lazy(Pd)) {
    if (fp_is_zero_lazy(Rd)) g1_double_affine(acc, p);
    else acc = G1XYZZ::identity();
    return;
  }
  G1XYZZ r;
  g1_add_tail(acc.X, acc.Y, Pd, Rd, acc.ZZ, acc.ZZZ, r);
  const Fq one = Fq::one();
#pragma unroll
  for (int i = 0; i < 8; i++) {
    acc.X.v[i] = was_inf ? p.x.v[i] : r.X.v[i];
    acc.Y.v[i] = was_inf ? p.y.v[i] : r.Y.v[i];
    acc.ZZ.v[i] = was_inf ? one.v[i] : r.ZZ.v[i];
    acc.ZZZ.v[i] = was_inf ? one.v[i] : r.ZZZ.v[i];
  }
}

// acc += q
PB_HD void g1_add(G1XYZZ& acc, const G1XYZZ& q) {
  if (q.is_inf()) return;
  if (acc.is_inf()) {
    acc = q;
    return;
  }
  Fq U1 = fp_mul(acc.X, q.ZZ);
  Fq U2 = fp_mul_lazy(q.X, acc.ZZ);
  Fq S1 = fp_mul(acc.Y, q.ZZZ);
  Fq S2 = fp_mul_lazy(q.Y, acc.ZZZ);
  Fq Pd = fp_sub(U2, U1);
  Fq Rd = fp_sub(S2, S1);
  if (fp_is_zero_lazy(Pd)) {
    if (fp_is_zero_lazy(Rd)) g1_double(acc);
    else acc = G1XYZZ::identity();
    return;
  }
  G1XYZZ r;
  g1_add_tail(U1, S1, Pd, Rd, fp_mul_lazy(acc.ZZ, q.ZZ), fp_mul_lazy(acc.ZZZ, q.ZZZ), r);
  acc = r;
}

// acc += q with select-based handling of identity operands (one instruction stream for all lanes, so two
// independent additions can be interleaved by the compiler); only the rare P == +-Q cases branch.
PB_HD void g1_add_uniform(G1XYZZ& acc, const G1XYZZ& q) {
  const bool a_inf = acc.is_inf(), q_inf = q.is_inf();
  Fq U1 = fp_mul(acc.X, q.ZZ);
  Fq U2 = fp_mul_lazy(q.X, acc.ZZ);
  Fq S1 = fp_mul(acc.Y, q.ZZZ);
  Fq S2 = fp_mul_lazy(q.Y, acc.ZZZ);
  Fq Pd = fp_sub(U2, U1);
  Fq Rd = fp_sub(S2, S1);
  if (!a_inf && !q_inf && fp_is_zero_lazy(Pd)) {
    if (fp_is_zero_lazy(Rd)) g1_double(acc);
    else acc = G1XYZZ::identity();
    return;
  }
  G1XYZZ r;
  g1_add_tail(U1, S1, Pd, Rd, fp_mul_lazy(acc.ZZ, q.ZZ), fp_mul_lazy(acc.ZZZ, q.ZZZ), r);
#pragma unroll
  for (int i = 0; i < 8; i++) {
    acc.X.v[i] = q_inf ? acc.X.v[i] : (a_inf ? q.X.v[i] : r.X.v[i]);
    acc.Y.v[i] = q_inf ? acc.Y.v[i] : (a_inf ? q.Y.v[i] : r.Y.v[i]);
    acc.ZZ.v[i] = q_inf ? acc.ZZ.v[i] : (a_inf ? q.ZZ.v[i] : r.ZZ.v[i]);
    acc.ZZZ.v[i] = q_inf ? acc.ZZZ.v[i] : (a_inf ? q.ZZZ.v[i] : r.ZZZ.v[i]);
  }
}

PB_HD G1Affine g1_neg_affine(const G1Affine& p) {
  G1Affine r;
  r.x = p.x;
  r.y = fp_neg(p.y);
  return r;
}

// returns true when a is the identity (out untouched -> zeros)
PB_HD bool g1_to_affine(const G1XYZZ& a, G1Affine& out) {
  if (a.is_inf()) {
    out.x = Fq::zero();
    out.y = Fq::zero();
    return true;
  }
  Fq A = fp_inv(a.ZZZ);                  // 1/ZZZ
  Fq izz = fp_sqr(fp_mul(a.ZZ, A));      // (ZZ/ZZZ)^2 = 1/ZZ   (ZZ^3 == ZZZ^2)
  out.x = fp_mul(a.X, izz);
  out.y = fp_mul(a.Y, A);
  return false;
}

}  // namespace pb200
