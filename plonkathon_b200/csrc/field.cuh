// BN254 prime fields Fr (scalar field, curve.py:11 `field_modulus = b.curve_order`) and
// Fq (base field, py_ecc.bn128 `field_modulus`) for sm_90a.
//
// Replaces every py_ecc `FQ` operation the reference's hot path performs
// (`FQ.__add__/__sub__/__mul__/__truediv__/__pow__`, SURVEY App. A).
//
// Representation: 8 x u32 little-endian limbs, Montgomery form with R = 2^256 (the same
// encoding the .ptau SRS file uses on disk, setup.py:36-40), always fully reduced to [0, p).
// Both moduli are < 2^254, so a + b never overflows 256 bits.
//
// Montgomery product: operand-scanning CIOS split into an "even" and an "odd" accumulator so
// every 32x32->64 partial product lands on an aligned register pair; written as
// mad.lo.cc / madc.hi.cc pairs, which ptxas fuses into one IMAD.WIDE.U32.X each
// (136 IMAD-class instructions per product; checked with cuobjdump -sass).
//
// For the group law (curve.cuh) there are cheaper variants: a dedicated squaring (36 partial products instead of
// 64, then the reduction), products that skip the final subtraction and return a value in [0, 2p), and the sum of
// two products with one reduction.  fp_mul itself, which the NTT and the quotient use, is unchanged.
//
// Every PTX instruction is wrapped in a tiny function that has a host emulation with an explicit
// carry flag, so the identical limb-level algorithm is unit-tested on the CPU
// (tests/test_host_arith.py via csrc/host_selftest.cpp) before it ever runs on a GPU.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define PB_HD __host__ __device__ __forceinline__
#define PB_D __device__ __forceinline__
#else
#define PB_HD inline
#define PB_D inline
#endif

namespace pb200 {

// --------------------------------------------------------------------------------------------
// carry-chain primitives (device: PTX; host: emulation with an explicit flag)
// --------------------------------------------------------------------------------------------
#if defined(__CUDA_ARCH__)
PB_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t mul_lo(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.lo.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t mul_hi(uint32_t a, uint32_t b) { uint32_t r; asm volatile("mul.hi.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
PB_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PB_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PB_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
PB_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
#else
static thread_local uint32_t g_cf = 0;  // emulated CC.CF
inline uint32_t add_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a + b + g_cf; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t addc(uint32_t a, uint32_t b) { return a + b + g_cf; }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b; g_cf = (uint32_t)((t >> 32) & 1); return (uint32_t)t; }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { uint64_t t = (uint64_t)a - b - g_cf; g_cf = (uint32_t)((t >> 32) & 1); return (uint32_t)t; }
inline uint32_t subc(uint32_t a, uint32_t b) { return a - b - g_cf; }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (uint64_t)(uint32_t)(a * b) + c + g_cf; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint64_t t = (((uint64_t)a * b) >> 32) + c + g_cf; g_cf = (uint32_t)(t >> 32); return (uint32_t)t; }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return (uint32_t)((((uint64_t)a * b) >> 32) + c + g_cf); }
#endif
// NB (device): borrow semantics of sub.cc/subc follow PTX: CC.CF holds the borrow-out and subc
// subtracts it; the host emulation mirrors that.

// --------------------------------------------------------------------------------------------
// field parameters
// --------------------------------------------------------------------------------------------
#define PB_LIMB_SWITCH(i, a0, a1, a2, a3, a4, a5, a6, a7) \
  ((i) == 0 ? a0 : (i) == 1 ? a1 : (i) == 2 ? a2 : (i) == 3 ? a3 : (i) == 4 ? a4 : (i) == 5 ? a5 : (i) == 6 ? a6 : a7)

struct FrParams {  // r = 21888242871839275222246405745257275088548364400416034343698204186575808495617
  static constexpr uint32_t NP0 = 0xefffffffu;  // -r^-1 mod 2^32
  static PB_HD constexpr uint32_t p(int i) { return PB_LIMB_SWITCH(i, 0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u); }
  static PB_HD constexpr uint32_t r1(int i) { return PB_LIMB_SWITCH(i, 0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u); }
  static PB_HD constexpr uint32_t r2(int i) { return PB_LIMB_SWITCH(i, 0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u); }
  static PB_HD constexpr uint32_t r3(int i) { return PB_LIMB_SWITCH(i, 0xb4bf0040u, 0x5e94d8e1u, 0x1cfbb6b8u, 0x2a489cbeu, 0xa19fcfedu, 0x893cc664u, 0x7fcc657cu, 0x0cf8594bu); }
};

struct FqParams {  // q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
  static constexpr uint32_t NP0 = 0xe4866389u;
  static PB_HD constexpr uint32_t p(int i) { return PB_LIMB_SWITCH(i, 0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u); }
  static PB_HD constexpr uint32_t r1(int i) { return PB_LIMB_SWITCH(i, 0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u); }
  static PB_HD constexpr uint32_t r2(int i) { return PB_LIMB_SWITCH(i, 0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u); }
  static PB_HD constexpr uint32_t r3(int i) { return PB_LIMB_SWITCH(i, 0xda1530dfu, 0xb1cd6dafu, 0xa7283db6u, 0x62f210e6u, 0x0ada0afbu, 0xef7f0b0cu, 0x2d592544u, 0x20fd6e90u); }
};

// --------------------------------------------------------------------------------------------
// field element
// --------------------------------------------------------------------------------------------
template <class P>
struct alignas(16) Fp {
  uint32_t v[8];

  static PB_HD Fp zero() { Fp r; for (int i = 0; i < 8; i++) r.v[i] = 0; return r; }
  static PB_HD Fp one() { Fp r; for (int i = 0; i < 8; i++) r.v[i] = P::r1(i); return r; }   // R mod p
  static PB_HD Fp r2() { Fp r; for (int i = 0; i < 8; i++) r.v[i] = P::r2(i); return r; }
  static PB_HD Fp r3() { Fp r; for (int i = 0; i < 8; i++) r.v[i] = P::r3(i); return r; }            // R^3 mod p
  static PB_HD Fp modulus() { Fp r; for (int i = 0; i < 8; i++) r.v[i] = P::p(i); return r; }

  PB_HD bool is_zero() const { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= v[i]; return o == 0; }
  PB_HD bool operator==(const Fp& b) const { uint32_t o = 0; for (int i = 0; i < 8; i++) o |= v[i] ^ b.v[i]; return o == 0; }
  PB_HD bool operator!=(const Fp& b) const { return !(*this == b); }
};

// a < p: a is the canonical (fully reduced) representative of its value
template <class P>
PB_HD bool fp_is_canonical(const Fp<P>& a) {
  const Fp<P> m = Fp<P>::modulus();
  for (int i = 7; i >= 0; i--)
    if (a.v[i] != m.v[i]) return a.v[i] < m.v[i];
  return false;
}

// r = a - p if a >= p else a     (a < 2p < 2^256)
template <class P>
PB_HD void fp_reduce_once(Fp<P>& a) {
  uint32_t t[8];
  t[0] = sub_cc(a.v[0], P::p(0));
#pragma unroll
  for (int i = 1; i < 8; i++) t[i] = subc_cc(a.v[i], P::p(i));
  uint32_t borrow = subc(0u, 0u);  // 0xffffffff if a < p
#pragma unroll
  for (int i = 0; i < 8; i++) a.v[i] = borrow ? a.v[i] : t[i];
}

template <class P>
PB_HD Fp<P> fp_add(const Fp<P>& a, const Fp<P>& b) {
  Fp<P> r;
  r.v[0] = add_cc(a.v[0], b.v[0]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = addc_cc(a.v[i], b.v[i]);
  r.v[7] = addc(a.v[7], b.v[7]);
  fp_reduce_once(r);
  return r;
}

template <class P>
PB_HD Fp<P> fp_sub(const Fp<P>& a, const Fp<P>& b) {
  Fp<P> r;
  r.v[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
  for (int i = 1; i < 8; i++) r.v[i] = subc_cc(a.v[i], b.v[i]);
  uint32_t mask = subc(0u, 0u);  // all ones if a < b
  r.v[0] = add_cc(r.v[0], P::p(0) & mask);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = addc_cc(r.v[i], P::p(i) & mask);
  r.v[7] = addc(r.v[7], P::p(7) & mask);
  return r;
}

template <class P>
PB_HD Fp<P> fp_neg(const Fp<P>& a) {
  Fp<P> r;
  r.v[0] = sub_cc(P::p(0), a.v[0]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = subc_cc(P::p(i), a.v[i]);
  r.v[7] = subc(P::p(7), a.v[7]);
  uint32_t nz = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) nz |= a.v[i];
#pragma unroll
  for (int i = 0; i < 8; i++) r.v[i] = nz ? r.v[i] : 0u;
  return r;
}

template <class P>
PB_HD Fp<P> fp_dbl(const Fp<P>& a) { return fp_add(a, a); }

// ---- Montgomery product -------------------------------------------------------------------
// T = X + 2^32 * Y.  X holds the products of even limbs of the multiplicand, Y those of odd limbs,
// so each 64-bit partial product lands on the limb pair (2k, 2k+1) of its accumulator.
// acc(pairs 0..3) += a(0,2,4,6) * b, returns with CC.CF = carry out of limb 7
template <class P>
PB_HD void fp_mad_row(uint32_t* acc, const uint32_t* a, uint32_t b) {
  acc[0] = mad_lo_cc(a[0], b, acc[0]);
  acc[1] = madc_hi_cc(a[0], b, acc[1]);
#pragma unroll
  for (int j = 2; j < 8; j += 2) {
    acc[j] = madc_lo_cc(a[j], b, acc[j]);
    acc[j + 1] = madc_hi_cc(a[j], b, acc[j + 1]);
  }
}
// same with the modulus as multiplicand: acc += p(off, off+2, ..) * m
template <class P, int OFF>
PB_HD void fp_mad_row_mod(uint32_t* acc, uint32_t m) {
  acc[0] = mad_lo_cc(P::p(OFF), m, acc[0]);
  acc[1] = madc_hi_cc(P::p(OFF), m, acc[1]);
#pragma unroll
  for (int j = 2; j < 8; j += 2) {
    acc[j] = madc_lo_cc(P::p(OFF + j), m, acc[j]);
    acc[j + 1] = madc_hi_cc(P::p(OFF + j), m, acc[j + 1]);
  }
}

// One CIOS step.  State: T = U + 2^32 * V + w, where U is the 0-aligned accumulator, V the
// 32-bit-shifted one and w a pending 32-bit word of weight 1.
//   FIRST: U = a_even*b, V = a_odd*b, w = 0.
//   else : the previous step left (with roles swapped) an accumulator V whose low limb, together
//          with the previous w, sums to 0 mod 2^32.  Dividing T by 2^32 turns that accumulator into
//          (V >> 64) in the shifted role, its limb 1 becomes the new pending word, and the carry of
//          (low limb + old w), which is simply (old w != 0), enters the U row as carry-in.
// No 32-bit add ever touches half of a register pair, which keeps every row fusable into
// IMAD.WIDE.U32.X.
template <class P, bool FIRST>
PB_HD void fp_cios_step(uint32_t* U, uint32_t* V, uint32_t& w, const uint32_t* a, uint32_t b) {
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      U[j] = mul_lo(a[j], b);
      U[j + 1] = mul_hi(a[j], b);
      V[j] = mul_lo(a[j + 1], b);
      V[j + 1] = mul_hi(a[j + 1], b);
    }
    w = 0;
  } else {
    (void)add_cc(w, 0xffffffffu);  // CF = (w != 0)
    U[0] = madc_lo_cc(a[0], b, U[0]);
    U[1] = madc_hi_cc(a[0], b, U[1]);
#pragma unroll
    for (int j = 2; j < 8; j += 2) {
      U[j] = madc_lo_cc(a[j], b, U[j]);
      U[j + 1] = madc_hi_cc(a[j], b, U[j + 1]);
    }
    uint32_t c1 = addc(0u, 0u);  // carry out of U limb 7 == weight of V' limb 7
    w = V[1];
    V[0] = mad_lo_cc(a[1], b, V[2]);
    V[1] = madc_hi_cc(a[1], b, V[3]);
    V[2] = madc_lo_cc(a[3], b, V[4]);
    V[3] = madc_hi_cc(a[3], b, V[5]);
    V[4] = madc_lo_cc(a[5], b, V[6]);
    V[5] = madc_hi_cc(a[5], b, V[7]);
    V[6] = madc_lo_cc(a[7], b, 0u);
    V[7] = madc_hi(a[7], b, c1);
  }
  uint32_t m = mul_lo(U[0] + w, P::NP0);
  fp_mad_row_mod<P, 1>(V, m);
  fp_mad_row_mod<P, 0>(U, m);
  V[7] = addc(V[7], 0u);
}

#if !defined(__CUDA_ARCH__) && defined(PB_HOST_FAST_MUL)
// Host-only shortcut used by the library's own host code (final Horner / inversion of a commitment,
// transcript challenge reduction): 4 x 64-bit CIOS with unsigned __int128.  Same function value as the limb
// code below; the CPU unit tests build WITHOUT this macro so they exercise the device algorithm.
template <class P>
inline Fp<P> fp_mul_host64(const Fp<P>& a, const Fp<P>& b) {
  typedef unsigned __int128 u128;
  uint64_t A[4], B[4], M[4], T[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    A[i] = (uint64_t)a.v[2 * i] | ((uint64_t)a.v[2 * i + 1] << 32);
    B[i] = (uint64_t)b.v[2 * i] | ((uint64_t)b.v[2 * i + 1] << 32);
    M[i] = (uint64_t)P::p(2 * i) | ((uint64_t)P::p(2 * i + 1) << 32);
  }
  uint64_t np = 1;  // -p^-1 mod 2^64 by Newton iteration from the 32-bit constant's defining property
  for (int k = 0; k < 6; k++) np *= 2 - M[0] * np;
  np = (uint64_t)0 - np;
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)A[j] * B[i] + T[j]; T[j] = (uint64_t)c; c >>= 64; }
    c += T[4]; T[4] = (uint64_t)c; T[5] = (uint64_t)(c >> 64);
    uint64_t m = T[0] * np;
    c = (u128)m * M[0] + T[0]; c >>= 64;
    for (int j = 1; j < 4; j++) { c += (u128)m * M[j] + T[j]; T[j - 1] = (uint64_t)c; c >>= 64; }
    c += T[4]; T[3] = (uint64_t)c; T[4] = T[5] + (uint64_t)(c >> 64); T[5] = 0;
  }
  // T < 2p: one conditional subtraction
  uint64_t r[4]; u128 br = 0; bool ge = T[4] != 0;
  if (!ge) { ge = true; for (int i = 3; i >= 0; i--) { if (T[i] != M[i]) { ge = T[i] > M[i]; break; } } }
  if (ge) { for (int i = 0; i < 4; i++) { u128 d = (u128)T[i] - M[i] - (uint64_t)br; r[i] = (uint64_t)d; br = (d >> 64) & 1; } }
  else { for (int i = 0; i < 4; i++) r[i] = T[i]; }
  Fp<P> o;
  for (int i = 0; i < 4; i++) { o.v[2 * i] = (uint32_t)r[i]; o.v[2 * i + 1] = (uint32_t)(r[i] >> 32); }
  return o;
}
#endif

// last CIOS step had U = Y, V = X:  T / 2^32 = X + (Y >> 32) + (w != 0)
template <class P>
PB_HD Fp<P> fp_cios_final(const uint32_t* X, const uint32_t* Y, uint32_t w) {
  Fp<P> r;
  (void)add_cc(w, 0xffffffffu);
  r.v[0] = addc_cc(X[0], Y[1]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = addc_cc(X[i], Y[i + 1]);
  r.v[7] = addc(X[7], 0u);
  return r;
}

template <class P>
PB_HD Fp<P> fp_mul(const Fp<P>& a, const Fp<P>& b) {
#if !defined(__CUDA_ARCH__) && defined(PB_HOST_FAST_MUL)
  return fp_mul_host64(a, b);
#else
  uint32_t X[8], Y[8], w;
  fp_cios_step<P, true>(X, Y, w, a.v, b.v[0]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[1]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[2]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[3]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[4]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[5]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[6]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[7]);
  Fp<P> r = fp_cios_final<P>(X, Y, w);
  fp_reduce_once(r);
  return r;
#endif
}

// ---- redundant ("lazy") representation ---------------------------------------------------------
// Both moduli satisfy 4p < R = 2^256 (p < 0.19 R), which gives the bounds below.  A lazy value is any
// integer in [0, 2p) congruent to the element; it is not unique (x and x + p), so it never leaves the
// function that made it: everything stored or compared is made canonical with fp_reduce_once.
//
// Montgomery reduction of T < p * R returns (T + m p) / R < 2p.  CIOS on a, b in [0, 2p) has
// T = a b < 4p^2 < p R, so dropping the final subtraction leaves a lazy result; fp_mul is this plus
// fp_reduce_once.
template <class P>
PB_HD Fp<P> fp_mul_lazy(const Fp<P>& a, const Fp<P>& b) {
#if !defined(__CUDA_ARCH__) && defined(PB_HOST_FAST_MUL)
  return fp_mul_host64(a, b);  // canonical, so also a valid lazy result
#else
  uint32_t X[8], Y[8], w;
  fp_cios_step<P, true>(X, Y, w, a.v, b.v[0]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[1]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[2]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[3]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[4]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[5]);
  fp_cios_step<P, false>(X, Y, w, a.v, b.v[6]);
  fp_cios_step<P, false>(Y, X, w, a.v, b.v[7]);
  return fp_cios_final<P>(X, Y, w);
#endif
}

// 2p, limb i
template <class P>
PB_HD constexpr uint32_t fp_2p(int i) { return (P::p(i) << 1) | (i ? P::p(i - 1) >> 31 : 0u); }

// a - b for a, b in [0, 2p): adds 2p on borrow, result in [0, 2p)
template <class P>
PB_HD Fp<P> fp_sub_lazy(const Fp<P>& a, const Fp<P>& b) {
  Fp<P> r;
  r.v[0] = sub_cc(a.v[0], b.v[0]);
#pragma unroll
  for (int i = 1; i < 8; i++) r.v[i] = subc_cc(a.v[i], b.v[i]);
  uint32_t mask = subc(0u, 0u);  // all ones if a < b
  r.v[0] = add_cc(r.v[0], fp_2p<P>(0) & mask);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = addc_cc(r.v[i], fp_2p<P>(i) & mask);
  r.v[7] = addc(r.v[7], fp_2p<P>(7) & mask);
  return r;
}
// (fp_sub is also exact for a in [0, 2p) and b in [0, p): it adds p on borrow, so the result is in [0, max(a, p)).)

// p - a for a in [0, p]: result in [0, p], congruent to -a (p for a == 0, unlike fp_neg)
template <class P>
PB_HD Fp<P> fp_neg_lazy(const Fp<P>& a) {
  Fp<P> r;
  r.v[0] = sub_cc(P::p(0), a.v[0]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = subc_cc(P::p(i), a.v[i]);
  r.v[7] = subc(P::p(7), a.v[7]);
  return r;
}

// a == 0 mod p for a in [0, 2p): a is 0 or p
template <class P>
PB_HD bool fp_is_zero_lazy(const Fp<P>& a) {
  uint32_t z = 0, q = 0;
#pragma unroll
  for (int i = 0; i < 8; i++) { z |= a.v[i]; q |= a.v[i] ^ P::p(i); }
  return z == 0 || q == 0;
}

// One CIOS step fed two rows: T += a * b + c * d (b, d: one limb each of the second factors), then one
// reduction row.  Same state and role swap as fp_cios_step; the second row adds into the accumulators
// without a shift, its carry out of limb 7 going to V limb 7 as the reduction rows do.
template <class P, bool FIRST>
PB_HD void fp_cios_step2(uint32_t* U, uint32_t* V, uint32_t& w, const uint32_t* a, uint32_t b, const uint32_t* c,
                         uint32_t d) {
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < 8; j += 2) {
      U[j] = mul_lo(a[j], b);
      U[j + 1] = mul_hi(a[j], b);
      V[j] = mul_lo(a[j + 1], b);
      V[j + 1] = mul_hi(a[j + 1], b);
    }
    w = 0;
  } else {
    (void)add_cc(w, 0xffffffffu);  // CF = (w != 0)
    U[0] = madc_lo_cc(a[0], b, U[0]);
    U[1] = madc_hi_cc(a[0], b, U[1]);
#pragma unroll
    for (int j = 2; j < 8; j += 2) {
      U[j] = madc_lo_cc(a[j], b, U[j]);
      U[j + 1] = madc_hi_cc(a[j], b, U[j + 1]);
    }
    uint32_t c1 = addc(0u, 0u);
    w = V[1];
    V[0] = mad_lo_cc(a[1], b, V[2]);
    V[1] = madc_hi_cc(a[1], b, V[3]);
    V[2] = madc_lo_cc(a[3], b, V[4]);
    V[3] = madc_hi_cc(a[3], b, V[5]);
    V[4] = madc_lo_cc(a[5], b, V[6]);
    V[5] = madc_hi_cc(a[5], b, V[7]);
    V[6] = madc_lo_cc(a[7], b, 0u);
    V[7] = madc_hi(a[7], b, c1);
  }
  fp_mad_row<P>(V, c + 1, d);
  fp_mad_row<P>(U, c, d);
  V[7] = addc(V[7], 0u);
  uint32_t m = mul_lo(U[0] + w, P::NP0);
  fp_mad_row_mod<P, 1>(V, m);
  fp_mad_row_mod<P, 0>(U, m);
  V[7] = addc(V[7], 0u);
}

// Sum of two products with one reduction: (a b + c d) / R mod p, lazy.  Needs a b + c d < p R, which holds
// e.g. when a, b, c, d < 2p and one factor of each product is below p (then a b + c d < 4p^2).
// Negate one operand (fp_neg_lazy / fp_sub_lazy) to get a difference of products.
template <class P>
PB_HD Fp<P> fp_mul2_lazy(const Fp<P>& a, const Fp<P>& b, const Fp<P>& c, const Fp<P>& d) {
#if !defined(__CUDA_ARCH__) && defined(PB_HOST_FAST_MUL)
  return fp_add(fp_mul_host64(a, b), fp_mul_host64(c, d));
#else
  uint32_t X[8], Y[8], w;
  fp_cios_step2<P, true>(X, Y, w, a.v, b.v[0], c.v, d.v[0]);
  fp_cios_step2<P, false>(Y, X, w, a.v, b.v[1], c.v, d.v[1]);
  fp_cios_step2<P, false>(X, Y, w, a.v, b.v[2], c.v, d.v[2]);
  fp_cios_step2<P, false>(Y, X, w, a.v, b.v[3], c.v, d.v[3]);
  fp_cios_step2<P, false>(X, Y, w, a.v, b.v[4], c.v, d.v[4]);
  fp_cios_step2<P, false>(Y, X, w, a.v, b.v[5], c.v, d.v[5]);
  fp_cios_step2<P, false>(X, Y, w, a.v, b.v[6], c.v, d.v[6]);
  fp_cios_step2<P, false>(Y, X, w, a.v, b.v[7], c.v, d.v[7]);
  return fp_cios_final<P>(X, Y, w);
#endif
}

// ---- squaring ----------------------------------------------------------------------------------
// The 512-bit square T = 2 * sum_{i<j} a_i a_j 2^(32(i+j)) + sum_i a_i^2 2^(64i) (28 + 8 partial products instead of
// 64), then Montgomery reduction of T.  The off-diagonal products go to two accumulators by the parity of i + j so
// every product lands on an aligned register pair: E[k] holds weight 2^(32k), O[k] weight 2^(32(k+1)).  Row i
// (multiplier a_i) is one carry chain into each; where a chain ends below a limb an earlier row wrote, its carry
// goes one limb up, into a limb no earlier row reached (the schedule is fixed, see the row comments).

// acc[2k..] += x[0] y, x[2] y, ... (n products, pairs at acc, acc + 2, ..); returns with CC.CF = carry out
PB_HD void fp_sqr_chain(uint32_t* acc, const uint32_t* x, uint32_t y, int n) {
  acc[0] = mad_lo_cc(x[0], y, acc[0]);
  acc[1] = madc_hi_cc(x[0], y, acc[1]);
#pragma unroll
  for (int k = 1; k < n; k++) {
    acc[2 * k] = madc_lo_cc(x[2 * k], y, acc[2 * k]);
    acc[2 * k + 1] = madc_hi_cc(x[2 * k], y, acc[2 * k + 1]);
  }
}

// T (16 limbs) = a^2 for a < 2^256
PB_HD void fp_sqr_wide(uint32_t* T, const uint32_t* a) {
  uint32_t E[16], O[16];
#pragma unroll
  for (int k = 0; k < 16; k++) { E[k] = 0; O[k] = 0; }
  // row 0: E limbs 2..7, O limbs 0..7 (weights 1..8); both top limbs were 0, no carry out
  fp_sqr_chain(E + 2, a + 2, a[0], 3);
  fp_sqr_chain(O + 0, a + 1, a[0], 4);
  // row 1: E 4..9 (new top); O weights 3..8, carry to weight 9
  fp_sqr_chain(E + 4, a + 3, a[1], 3);
  fp_sqr_chain(O + 2, a + 2, a[1], 3);
  O[8] = addc(0u, 0u);
  // row 2: E 6..9, carry to 10; O weights 5..10 (new top)
  fp_sqr_chain(E + 6, a + 4, a[2], 2);
  E[10] = addc(0u, 0u);
  fp_sqr_chain(O + 4, a + 3, a[2], 3);
  // row 3: E 8..11 (new top); O weights 7..10, carry to 11
  fp_sqr_chain(E + 8, a + 5, a[3], 2);
  fp_sqr_chain(O + 6, a + 4, a[3], 2);
  O[10] = addc(0u, 0u);
  // row 4: E 10..11, carry to 12; O weights 9..12 (new top)
  fp_sqr_chain(E + 10, a + 6, a[4], 1);
  E[12] = addc(0u, 0u);
  fp_sqr_chain(O + 8, a + 5, a[4], 2);
  // row 5: E 12..13 (new top); O weights 11..12, carry to 13
  fp_sqr_chain(E + 12, a + 7, a[5], 1);
  fp_sqr_chain(O + 10, a + 6, a[5], 1);
  O[12] = addc(0u, 0u);
  // row 6: O weights 13..14 (new top)
  fp_sqr_chain(O + 12, a + 7, a[6], 1);
  // S = E + O (weights 1..15), T = 2 S + diagonal
  uint32_t S[16];
  S[0] = 0;
  S[1] = O[0];
  S[2] = add_cc(E[2], O[1]);
#pragma unroll
  for (int k = 3; k < 14; k++) S[k] = addc_cc(E[k], O[k - 1]);
  S[14] = addc_cc(O[13], 0u);
  S[15] = addc(0u, 0u);
  S[1] = add_cc(S[1], S[1]);
#pragma unroll
  for (int k = 2; k < 15; k++) S[k] = addc_cc(S[k], S[k]);
  S[15] = addc(S[15], S[15]);
  T[0] = mad_lo_cc(a[0], a[0], 0u);
  T[1] = madc_hi_cc(a[0], a[0], S[1]);
#pragma unroll
  for (int i = 1; i < 7; i++) {
    T[2 * i] = madc_lo_cc(a[i], a[i], S[2 * i]);
    T[2 * i + 1] = madc_hi_cc(a[i], a[i], S[2 * i + 1]);
  }
  T[14] = madc_lo_cc(a[7], a[7], S[14]);
  T[15] = madc_hi(a[7], a[7], S[15]);
}

// One reduction-only CIOS step (no product row): same state and role swap as fp_cios_step.  FIRST starts from
// U = the value, V = 0.  Otherwise the pending carry (old w != 0) enters the reduction row of U as its carry-in
// instead of being propagated through U, and the shift of V by one limb pair is plain register renaming.
template <class P, bool FIRST>
PB_HD void fp_redc_step(uint32_t* U, uint32_t* V, uint32_t& w) {
  uint32_t cf = 0;
  if (FIRST) {
#pragma unroll
    for (int j = 0; j < 8; j++) V[j] = 0;
    w = 0;
  } else {
    cf = w != 0;
    w = V[1];
#pragma unroll
    for (int j = 0; j < 6; j++) V[j] = V[j + 2];
    V[6] = 0;
    V[7] = 0;
  }
  const uint32_t m = mul_lo(U[0] + w + cf, P::NP0);
  fp_mad_row_mod<P, 1>(V, m);
  (void)add_cc(cf, 0xffffffffu);  // CF = cf
  U[0] = madc_lo_cc(P::p(0), m, U[0]);
  U[1] = madc_hi_cc(P::p(0), m, U[1]);
#pragma unroll
  for (int j = 2; j < 8; j += 2) {
    U[j] = madc_lo_cc(P::p(j), m, U[j]);
    U[j + 1] = madc_hi_cc(P::p(j), m, U[j + 1]);
  }
  V[7] = addc(V[7], 0u);
}

// a^2 / R mod p, lazy, for a in [0, 2p).  T = a^2 = T_lo + R T_hi; the result is (T_lo + m p) / R + T_hi with
// (T_lo + m p) / R <= p and T_hi < 4p^2 / R < 0.76 p, so it is below 2p.
template <class P>
PB_HD Fp<P> fp_sqr_lazy(const Fp<P>& a) {
#if !defined(__CUDA_ARCH__) && defined(PB_HOST_FAST_MUL)
  return fp_mul_host64(a, a);
#else
  uint32_t T[16], Y[8], w;
  fp_sqr_wide(T, a.v);
  uint32_t* X = T;  // U of the first step: T_lo, reduced in place
  fp_redc_step<P, true>(X, Y, w);
  fp_redc_step<P, false>(Y, X, w);
  fp_redc_step<P, false>(X, Y, w);
  fp_redc_step<P, false>(Y, X, w);
  fp_redc_step<P, false>(X, Y, w);
  fp_redc_step<P, false>(Y, X, w);
  fp_redc_step<P, false>(X, Y, w);
  fp_redc_step<P, false>(Y, X, w);
  Fp<P> r = fp_cios_final<P>(X, Y, w);
  r.v[0] = add_cc(r.v[0], T[8]);
#pragma unroll
  for (int i = 1; i < 7; i++) r.v[i] = addc_cc(r.v[i], T[8 + i]);
  r.v[7] = addc(r.v[7], T[15]);
  return r;
#endif
}

// a^2: the dedicated squaring, fully reduced (bit-identical to fp_mul(a, a))
template <class P>
PB_HD Fp<P> fp_sqr(const Fp<P>& a) {
  Fp<P> r = fp_sqr_lazy(a);
  fp_reduce_once(r);
  return r;
}

template <class P>
PB_HD Fp<P> fp_to_mont(const Fp<P>& a) { return fp_mul(a, Fp<P>::r2()); }

// to_mont for an arbitrary 256-bit input (not necessarily < p): CIOS only needs one operand below p
template <class P>
PB_HD Fp<P> fp_to_mont_any(const Fp<P>& a) { return fp_mul(Fp<P>::r2(), a); }

template <class P>
PB_HD Fp<P> fp_from_mont(const Fp<P>& a) {
  Fp<P> o = Fp<P>::zero();
  o.v[0] = 1;
  return fp_mul(a, o);
}

// a^e for a 256-bit exponent given as 8 LE limbs (vartime in e; e is public everywhere it is used)
template <class P>
PB_HD Fp<P> fp_pow(const Fp<P>& a, const uint32_t* e) {
  Fp<P> r = Fp<P>::one();
  bool started = false;
  for (int i = 255; i >= 0; i--) {
    if (started) r = fp_sqr(r);
    if ((e[i >> 5] >> (i & 31)) & 1) {
      r = started ? fp_mul(r, a) : a;
      started = true;
    }
  }
  return r;
}

template <class P>
PB_HD Fp<P> fp_pow_u64(const Fp<P>& a, uint64_t e) {
  uint32_t ee[8] = {(uint32_t)e, (uint32_t)(e >> 32), 0, 0, 0, 0, 0, 0};
  return fp_pow(a, ee);
}

// inverse by Fermat (a^(p-2)); inv(0) == 0, matching py_ecc's prime_field_inv convention
template <class P>
PB_HD Fp<P> fp_inv(const Fp<P>& a) {
  uint32_t e[8];
#pragma unroll
  for (int i = 0; i < 8; i++) e[i] = P::p(i);
  e[0] -= 2;  // p is odd and p(0) >= 2 for both fields
  return fp_pow(a, e);
}

typedef Fp<FrParams> Fr;
typedef Fp<FqParams> Fq;

}  // namespace pb200
