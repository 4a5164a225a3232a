/* ORACLE / TEST INFRASTRUCTURE ONLY -- never linked into libplonk_b200.so.
 *
 * Plain-C CPU restatement of the two data-parallel cores of the reference's proving path, for exact
 * parity checks at sizes the pure-Python oracle (oracle/plonk_oracle.py) cannot reach in seconds:
 *
 *   oc_fr_fft      -- poly.py:113-149  Polynomial.fft / ifft: natural order in and out, w = 5^((r-1)/n)
 *                     (curve.py:15-16), inverse = reversed roots and a final multiplication by n^-1.
 *   oc_g1_lincomb  -- curve.py:38-44   ec_lincomb: sum_i s_i * P_i over BN254 G1, affine result or identity.
 *                     The function value is algorithm-independent; this file uses a plain bucket method
 *                     with Jacobian accumulators instead of the reference's bit-sliced multisubset tables
 *                     (which need one modular inversion per affine addition: minutes at 2^20).
 *   oc_fr_eval_lagrange -- value at x of the polynomial given by Lagrange values (used to re-derive KZG
 *                     commitments [f(tau)]G under a structured test SRS).
 *   oc_fr_eval_coeffs -- value at x of the polynomial given by its coefficients (Horner).  With eval_lagrange it
 *                     checks a whole transform in O(n): one identity at one random point.
 *
 * It is cross-checked against oracle/plonk_oracle.py (itself pinned by the reference's golden vectors) in
 * tests/test_oracle_c.py.  Arithmetic: 4 x 64-bit limbs, Montgomery form R = 2^256, unsigned __int128.
 * Build: make -C oracle  ->  oracle/c/libplonk_oracle_c.so                                               */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef unsigned __int128 u128;
typedef struct { uint64_t v[4]; } fe;

typedef struct { fe p, r1, r2; uint64_t np; } field_t;

static field_t FR, FQ;

static int fe_geq(const fe* a, const fe* b) {
  for (int i = 3; i >= 0; i--) if (a->v[i] != b->v[i]) return a->v[i] > b->v[i];
  return 1;
}
static void fe_sub_raw(fe* r, const fe* a, const fe* b) {
  u128 br = 0;
  for (int i = 0; i < 4; i++) { u128 d = (u128)a->v[i] - b->v[i] - (uint64_t)br; r->v[i] = (uint64_t)d; br = (d >> 64) & 1; }
}
static void fe_add(const field_t* F, fe* r, const fe* a, const fe* b) {
  u128 c = 0;
  for (int i = 0; i < 4; i++) { c += (u128)a->v[i] + b->v[i]; r->v[i] = (uint64_t)c; c >>= 64; }
  if (c || fe_geq(r, &F->p)) fe_sub_raw(r, r, &F->p);
}
static void fe_sub(const field_t* F, fe* r, const fe* a, const fe* b) {
  if (fe_geq(a, b)) fe_sub_raw(r, a, b);
  else { fe t; fe_sub_raw(&t, &F->p, b); u128 c = 0; for (int i = 0; i < 4; i++) { c += (u128)t.v[i] + a->v[i]; r->v[i] = (uint64_t)c; c >>= 64; } }
}
static int fe_is_zero(const fe* a) { return (a->v[0] | a->v[1] | a->v[2] | a->v[3]) == 0; }
static int fe_eq(const fe* a, const fe* b) { return memcmp(a, b, sizeof(fe)) == 0; }

/* Montgomery product (CIOS), result fully reduced */
static void fe_mul(const field_t* F, fe* r, const fe* a, const fe* b) {
  uint64_t T[6] = {0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 4; i++) {
    u128 c = 0;
    for (int j = 0; j < 4; j++) { c += (u128)a->v[j] * b->v[i] + T[j]; T[j] = (uint64_t)c; c >>= 64; }
    c += T[4]; T[4] = (uint64_t)c; T[5] = (uint64_t)(c >> 64);
    uint64_t m = T[0] * F->np;
    c = (u128)m * F->p.v[0] + T[0]; c >>= 64;
    for (int j = 1; j < 4; j++) { c += (u128)m * F->p.v[j] + T[j]; T[j - 1] = (uint64_t)c; c >>= 64; }
    c += T[4]; T[3] = (uint64_t)c; T[4] = T[5] + (uint64_t)(c >> 64); T[5] = 0;
  }
  fe t; memcpy(t.v, T, 32);
  if (T[4] || fe_geq(&t, &F->p)) fe_sub_raw(&t, &t, &F->p);
  *r = t;
}
static void fe_pow(const field_t* F, fe* r, const fe* a, const uint64_t e[4]) {
  fe acc = F->r1;
  for (int i = 255; i >= 0; i--) {
    fe_mul(F, &acc, &acc, &acc);
    if ((e[i >> 6] >> (i & 63)) & 1) fe_mul(F, &acc, &acc, a);
  }
  *r = acc;
}
static void fe_inv(const field_t* F, fe* r, const fe* a) { /* inv(0) == 0 like py_ecc */
  uint64_t e[4] = {F->p.v[0] - 2, F->p.v[1], F->p.v[2], F->p.v[3]};
  fe_pow(F, r, a, e);
}
static void fe_to_mont(const field_t* F, fe* r, const fe* a) { fe_mul(F, r, a, &F->r2); }
static void fe_from_mont(const field_t* F, fe* r, const fe* a) { fe one = {{1, 0, 0, 0}}; fe_mul(F, r, a, &one); }
static void fe_from_u64(const field_t* F, fe* r, uint64_t x) { fe t = {{x, 0, 0, 0}}; fe_to_mont(F, r, &t); }

static void field_init(field_t* F, const uint64_t p[4]) {
  memcpy(F->p.v, p, 32);
  uint64_t np = 1;
  for (int k = 0; k < 6; k++) np *= 2 - p[0] * np;
  F->np = (uint64_t)0 - np;
  /* R mod p and R^2 mod p by repeated doubling of 1 */
  fe x = {{1, 0, 0, 0}};
  for (int i = 0; i < 512; i++) {
    fe_add(F, &x, &x, &x);
    if (i == 255) F->r1 = x;
  }
  F->r2 = x;
}
static int g_init = 0;
static void ensure_init(void) {
  if (g_init) return;
  static const uint64_t r[4] = {0x43e1f593f0000001ULL, 0x2833e84879b97091ULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
  static const uint64_t q[4] = {0x3c208c16d87cfd47ULL, 0x97816a916871ca8dULL, 0xb85045b68181585dULL, 0x30644e72e131a029ULL};
  field_init(&FR, r);
  field_init(&FQ, q);
  g_init = 1;
}

/* ---------------------------------------------------------------------------------------------------- */
/* poly.py:113-149.  in/out: n x 32 bytes, canonical little-endian.  Returns 0 on success.              */
int oc_fr_fft(const uint8_t* in, uint8_t* out, unsigned log_n, int inverse) {
  ensure_init();
  size_t n = (size_t)1 << log_n;
  fe* a = (fe*)malloc(n * sizeof(fe));
  if (!a) return 1;
  /* load bit-reversed (the recursive even/odd split of poly.py:120-121 is a bit reversal) */
  for (size_t i = 0; i < n; i++) {
    size_t j = 0;
    for (unsigned b = 0; b < log_n; b++) if (i >> b & 1) j |= (size_t)1 << (log_n - 1 - b);
    fe t; memcpy(t.v, in + 32 * i, 32);
    fe_to_mont(&FR, &a[j], &t);
  }
  /* w = 5^((r-1)/n) (curve.py:15-16); inverse transform walks the roots backwards (poly.py:135) */
  uint64_t e[4] = {FR.p.v[0] - 1, FR.p.v[1], FR.p.v[2], FR.p.v[3]};
  for (unsigned s = 0; s < log_n; s++) { for (int i = 0; i < 4; i++) e[i] = (e[i] >> 1) | (i < 3 ? e[i + 1] << 63 : 0); }
  fe five, w;
  fe_from_u64(&FR, &five, 5);
  fe_pow(&FR, &w, &five, e);
  if (inverse) fe_inv(&FR, &w, &w);
  for (unsigned s = 0; s < log_n; s++) {
    size_t half = (size_t)1 << s;
    /* w_{2 half} = w^(n / (2 half)) */
    fe wl = w;
    for (unsigned k = s + 1; k < log_n; k++) fe_mul(&FR, &wl, &wl, &wl);
    for (size_t base = 0; base < n; base += 2 * half) {
      fe tw = FR.r1;
      for (size_t j = 0; j < half; j++) {
        fe t, u = a[base + j];
        fe_mul(&FR, &t, &a[base + j + half], &tw);
        fe_add(&FR, &a[base + j], &u, &t);          /* poly.py:124-125 */
        fe_sub(&FR, &a[base + j + half], &u, &t);
        fe_mul(&FR, &tw, &tw, &wl);
      }
    }
  }
  fe scale = FR.r1;
  if (inverse) { fe nn; fe_from_u64(&FR, &nn, (uint64_t)n); fe_inv(&FR, &scale, &nn); } /* poly.py:134,137 */
  for (size_t i = 0; i < n; i++) {
    fe t;
    if (inverse) fe_mul(&FR, &a[i], &a[i], &scale);
    fe_from_mont(&FR, &t, &a[i]);
    memcpy(out + 32 * i, t.v, 32);
  }
  free(a);
  return 0;
}

/* value at x of the polynomial with the given Lagrange values on the 2^log_n-th roots of unity (x off the domain) */
int oc_fr_eval_lagrange(const uint8_t* vals, unsigned log_n, const uint8_t* x32, uint8_t* out32) {
  ensure_init();
  size_t n = (size_t)1 << log_n;
  fe x; { fe t; memcpy(t.v, x32, 32); fe_to_mont(&FR, &x, &t); }
  uint64_t e[4] = {FR.p.v[0] - 1, FR.p.v[1], FR.p.v[2], FR.p.v[3]};
  for (unsigned s = 0; s < log_n; s++) { for (int i = 0; i < 4; i++) e[i] = (e[i] >> 1) | (i < 3 ? e[i + 1] << 63 : 0); }
  fe five, w, w_inv; fe_from_u64(&FR, &five, 5); fe_pow(&FR, &w, &five, e); fe_inv(&FR, &w_inv, &w);
  fe* d = (fe*)malloc(n * sizeof(fe)); fe* pref = (fe*)malloc(n * sizeof(fe));
  if (!d || !pref) { free(d); free(pref); return 1; }
  /* w^i / (x - w^i) = 1 / d_i with d_i = x w^-i - 1: one batch inversion of the d_i */
  fe cur = x, run = FR.r1;
  for (size_t i = 0; i < n; i++) {
    fe_sub(&FR, &d[i], &cur, &FR.r1);
    pref[i] = run; fe_mul(&FR, &run, &run, &d[i]);
    fe_mul(&FR, &cur, &cur, &w_inv);
  }
  fe inv; fe_inv(&FR, &inv, &run);
  fe acc = {{0, 0, 0, 0}};  /* canonical: a canonical value times a Montgomery-form 1/d_i is the plain quotient */
  for (size_t i = n; i-- > 0;) {
    fe di, t; fe_mul(&FR, &di, &inv, &pref[i]); fe_mul(&FR, &inv, &inv, &d[i]);
    memcpy(t.v, vals + 32 * i, 32);
    if (fe_is_zero(&t)) continue;
    fe_mul(&FR, &t, &t, &di); fe_add(&FR, &acc, &acc, &t);
  }
  /* (x^n - 1) / n */
  fe xn = x; for (unsigned s = 0; s < log_n; s++) fe_mul(&FR, &xn, &xn, &xn);
  fe num, nn, ninv; fe_sub(&FR, &num, &xn, &FR.r1); fe_from_u64(&FR, &nn, (uint64_t)n); fe_inv(&FR, &ninv, &nn);
  fe_mul(&FR, &acc, &acc, &num); fe_mul(&FR, &acc, &acc, &ninv);
  memcpy(out32, acc.v, 32);
  free(d); free(pref);
  return 0;
}

/* value at x of sum_{i < n} c_i x^i by Horner (any n >= 0; n == 0 gives 0).  coeffs: n x 32 bytes canonical.
 * The accumulator stays canonical: a Montgomery product with x in Montgomery form is a plain product.      */
int oc_fr_eval_coeffs(const uint8_t* coeffs, uint64_t n, const uint8_t* x32, uint8_t* out32) {
  ensure_init();
  fe x; { fe t; memcpy(t.v, x32, 32); fe_to_mont(&FR, &x, &t); }
  fe acc = {{0, 0, 0, 0}};
  for (uint64_t i = n; i-- > 0;) {
    fe c; memcpy(c.v, coeffs + 32 * i, 32);
    if (fe_geq(&c, &FR.p)) return 2;  /* not canonical */
    fe_mul(&FR, &acc, &acc, &x);
    fe_add(&FR, &acc, &acc, &c);
  }
  memcpy(out32, acc.v, 32);
  return 0;
}

/* ---------------------------------------------------------------------------------------------------- */
/* G1: y^2 = x^3 + 3 over Fq, Jacobian coordinates (X/Z^2, Y/Z^3), identity <=> Z == 0                   */
typedef struct { fe X, Y, Z; } jac;

static void jac_double(jac* r, const jac* p) {
  if (fe_is_zero(&p->Z)) { *r = *p; return; }
  fe A, B, C, D, E, F, t;
  fe_mul(&FQ, &A, &p->X, &p->X);
  fe_mul(&FQ, &B, &p->Y, &p->Y);
  fe_mul(&FQ, &C, &B, &B);
  fe_add(&FQ, &t, &p->X, &B); fe_mul(&FQ, &t, &t, &t); fe_sub(&FQ, &t, &t, &A); fe_sub(&FQ, &t, &t, &C);
  fe_add(&FQ, &D, &t, &t);
  fe_add(&FQ, &E, &A, &A); fe_add(&FQ, &E, &E, &A);
  fe_mul(&FQ, &F, &E, &E);
  jac o;
  fe_sub(&FQ, &o.X, &F, &D); fe_sub(&FQ, &o.X, &o.X, &D);
  fe_sub(&FQ, &t, &D, &o.X); fe_mul(&FQ, &t, &t, &E);
  fe c8; fe_add(&FQ, &c8, &C, &C); fe_add(&FQ, &c8, &c8, &c8); fe_add(&FQ, &c8, &c8, &c8);
  fe_sub(&FQ, &o.Y, &t, &c8);
  fe_mul(&FQ, &o.Z, &p->Y, &p->Z); fe_add(&FQ, &o.Z, &o.Z, &o.Z);
  *r = o;
}
static void jac_add(jac* r, const jac* p, const jac* q) {
  if (fe_is_zero(&p->Z)) { *r = *q; return; }
  if (fe_is_zero(&q->Z)) { *r = *p; return; }
  fe Z1Z1, Z2Z2, U1, U2, S1, S2, H, R, t;
  fe_mul(&FQ, &Z1Z1, &p->Z, &p->Z); fe_mul(&FQ, &Z2Z2, &q->Z, &q->Z);
  fe_mul(&FQ, &U1, &p->X, &Z2Z2); fe_mul(&FQ, &U2, &q->X, &Z1Z1);
  fe_mul(&FQ, &S1, &p->Y, &q->Z); fe_mul(&FQ, &S1, &S1, &Z2Z2);
  fe_mul(&FQ, &S2, &q->Y, &p->Z); fe_mul(&FQ, &S2, &S2, &Z1Z1);
  fe_sub(&FQ, &H, &U2, &U1); fe_sub(&FQ, &R, &S2, &S1);
  if (fe_is_zero(&H)) {
    if (fe_is_zero(&R)) { jac_double(r, p); return; }
    memset(r, 0, sizeof(jac)); return;  /* P + (-P) */
  }
  fe HH, HHH, V; jac o;
  fe_mul(&FQ, &HH, &H, &H); fe_mul(&FQ, &HHH, &HH, &H); fe_mul(&FQ, &V, &U1, &HH);
  fe_mul(&FQ, &o.X, &R, &R); fe_sub(&FQ, &o.X, &o.X, &HHH); fe_sub(&FQ, &o.X, &o.X, &V); fe_sub(&FQ, &o.X, &o.X, &V);
  fe_sub(&FQ, &t, &V, &o.X); fe_mul(&FQ, &t, &t, &R);
  fe s1h; fe_mul(&FQ, &s1h, &S1, &HHH); fe_sub(&FQ, &o.Y, &t, &s1h);
  fe_mul(&FQ, &o.Z, &p->Z, &q->Z); fe_mul(&FQ, &o.Z, &o.Z, &H);
  *r = o;
}

/* curve.py:38-44.  points: n x 64 bytes (x || y canonical little-endian, never the identity); scalars:
 * n x 32 bytes canonical (already reduced mod r, curve.py:41).  out_xy: 64 bytes; *is_identity set.     */
int oc_g1_lincomb(const uint8_t* points, const uint8_t* scalars, uint64_t n, uint8_t* out_xy, int* is_identity) {
  ensure_init();
  if (n == 0) return 2;  /* the reference raises ValueError (curve.py:93) */
  unsigned c = 4;
  while (c < 16 && ((uint64_t)1 << (c + 4)) < n) c++;
  unsigned W = (254 + c - 1) / c;
  size_t nb = (size_t)1 << c;
  jac* pts = (jac*)malloc(n * sizeof(jac));
  jac* buckets = (jac*)malloc(nb * sizeof(jac));
  if (!pts || !buckets) return 1;
  for (uint64_t i = 0; i < n; i++) {
    fe t; memcpy(t.v, points + 64 * i, 32); fe_to_mont(&FQ, &pts[i].X, &t);
    memcpy(t.v, points + 64 * i + 32, 32); fe_to_mont(&FQ, &pts[i].Y, &t);
    pts[i].Z = FQ.r1;
  }
  jac total; memset(&total, 0, sizeof total);
  for (int w = (int)W - 1; w >= 0; w--) {
    for (unsigned k = 0; k < c; k++) jac_double(&total, &total);
    memset(buckets, 0, nb * sizeof(jac));
    for (uint64_t i = 0; i < n; i++) {
      const uint64_t* s = (const uint64_t*)(scalars + 32 * i);
      unsigned bit = (unsigned)w * c, limb = bit >> 6, off = bit & 63;
      uint64_t d = s[limb] >> off;
      if (off + c > 64 && limb + 1 < 4) d |= s[limb + 1] << (64 - off);
      d &= nb - 1;
      if (d) jac_add(&buckets[d], &buckets[d], &pts[i]);
    }
    jac run, sum; memset(&run, 0, sizeof run); memset(&sum, 0, sizeof sum);
    for (size_t b = nb - 1; b >= 1; b--) { jac_add(&run, &run, &buckets[b]); jac_add(&sum, &sum, &run); }
    jac_add(&total, &total, &sum);
  }
  if (fe_is_zero(&total.Z)) { *is_identity = 1; memset(out_xy, 0, 64); }
  else {
    fe zi, zi2, zi3, x, y, t;
    fe_inv(&FQ, &zi, &total.Z); fe_mul(&FQ, &zi2, &zi, &zi); fe_mul(&FQ, &zi3, &zi2, &zi);
    fe_mul(&FQ, &x, &total.X, &zi2); fe_mul(&FQ, &y, &total.Y, &zi3);
    fe_from_mont(&FQ, &t, &x); memcpy(out_xy, t.v, 32);
    fe_from_mont(&FQ, &t, &y); memcpy(out_xy + 32, t.v, 32);
    *is_identity = 0;
  }
  free(pts); free(buckets);
  return 0;
}

/* Structured test SRS for sizes the reference's .ptau does not reach (setup.py:16-22 `powers_of_x` for a known
 * tau): out[i] = [tau^i] G, i < n, as x || y canonical little-endian.  G = (1, 2).  Fixed-base multiplication
 * with byte windows (table[w][d] = d * 2^(8w) * G) and one shared inversion per chunk of 1024 points. */
int oc_g1_powers(const uint8_t* tau32, uint64_t n, uint8_t* out) {
  ensure_init();
  jac (*table)[256] = (jac (*)[256])malloc(32 * 256 * sizeof(jac));
  enum { CH = 1024 };
  jac* acc = (jac*)malloc(CH * sizeof(jac));
  fe* pref = (fe*)malloc(CH * sizeof(fe));
  if (!table || !acc || !pref) return 1;
  jac base; fe two;
  base.X = FQ.r1; fe_add(&FQ, &two, &FQ.r1, &FQ.r1); base.Y = two; base.Z = FQ.r1;
  for (int w = 0; w < 32; w++) {
    memset(&table[w][0], 0, sizeof(jac));
    for (int d = 1; d < 256; d++) jac_add(&table[w][d], &table[w][d - 1], &base);
    for (int k = 0; k < 8; k++) jac_double(&base, &base);
  }
  fe tau, tau_m, cur; memcpy(tau.v, tau32, 32); fe_to_mont(&FR, &tau_m, &tau);
  cur = FR.r1;  /* tau^0 in Montgomery form */
  for (uint64_t i0 = 0; i0 < n; i0 += CH) {
    uint64_t cnt = n - i0 < CH ? n - i0 : CH;
    for (uint64_t k = 0; k < cnt; k++) {
      fe s; fe_from_mont(&FR, &s, &cur);
      const uint8_t* sb = (const uint8_t*)s.v;
      jac a; memset(&a, 0, sizeof a);
      for (int w = 0; w < 32; w++) if (sb[w]) jac_add(&a, &a, &table[w][sb[w]]);
      acc[k] = a;  /* never the identity: tau^i != 0 mod r */
      fe_mul(&FR, &cur, &cur, &tau_m);
    }
    fe run = FQ.r1;
    for (uint64_t k = 0; k < cnt; k++) { pref[k] = run; fe_mul(&FQ, &run, &run, &acc[k].Z); }
    fe inv; fe_inv(&FQ, &inv, &run);
    for (uint64_t k = cnt; k-- > 0;) {
      fe zi, zi2, zi3, x, y, t;
      fe_mul(&FQ, &zi, &inv, &pref[k]); fe_mul(&FQ, &inv, &inv, &acc[k].Z);
      fe_mul(&FQ, &zi2, &zi, &zi); fe_mul(&FQ, &zi3, &zi2, &zi);
      fe_mul(&FQ, &x, &acc[k].X, &zi2); fe_mul(&FQ, &y, &acc[k].Y, &zi3);
      fe_from_mont(&FQ, &t, &x); memcpy(out + 64 * (i0 + k), t.v, 32);
      fe_from_mont(&FQ, &t, &y); memcpy(out + 64 * (i0 + k) + 32, t.v, 32);
    }
  }
  free(table); free(acc); free(pref);
  return 0;
}
