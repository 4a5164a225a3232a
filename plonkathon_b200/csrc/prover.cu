// Device-resident PLONK prover: rounds 1-5 of prover.py:51-306 (`Prover.prove`, `round_1..5`).
//
// The reference's round bodies are stubs in the mounted branch; the computation follows the in-tree
// comments, the sanity asserts and the completed test verifier (see SURVEY App. D and
// oracle/plonk_oracle.py, which is pinned by test/proof.pickle).  Every output (9 G1 points, 6 scalars) is
// mathematically unique -- the reference prover has no blinding -- so the work is restructured freely:
//   * all vectors stay in HBM in Montgomery form; only the 15 proof values cross to the host, once per round,
//     because the Merlin transcript is host code;
//   * selector / permutation polynomials are converted to coefficients and coset-extended once per circuit
//     (Prover creation), on a FIXED coset g*<w_4n> (g = 5): the quotient T(X) does not depend on which coset
//     it is interpolated from, so the transcript's `fft_cofactor` challenge is drawn (it is part of the
//     transcript schedule, transcript.py:88-97) but not needed for the arithmetic;
//   * T1, T2, T3, R, W_z, W_zw are committed from their coefficients directly (the reference's
//     fft -> commit -> ifft round trip is the identity, setup.py:66-72);
//   * round 4 evaluates coefficient forms by parallel Horner instead of barycentric sums (same values);
//   * round 5 builds R(X) and the opening numerators in coefficient form; the divisions by (X - zeta) and
//     (X - zeta*w) are done on an n-point coset (quotient degree n-2 < n).
// The reference's run-time invariants are kept as checks that fail the call: gate satisfaction
// (prover.py:108-116), Z_n == 1 (prover.py:132), deg T < 3n (prover.py:205-208).
// Zero-knowledge mode (prover_set_zk, one GPU) blinds A, B, C, Z and the quotient pieces as in the PLONK paper; the
// proof keeps its 15 fields and the verifier does not change.  See "zero knowledge" below.
// A shuffle (Prover::sh, one GPU) proves that two sets of rows hold the same multiset of (a, b, c): one more grand
// product Z3 beside Z, see "shuffle" below; the proof gains z3_1 and two evaluations (896 bytes, 992 next-row).  In
// zero-knowledge mode (pb200_prover_set_zk_shuffle) Z3 takes three more blinders and the proof keeps its size.
// Custom terms over the next row (Prover::next_row, one GPU) read a(wX), b(wX), c(wX): k_gate_check<true> and
// k_quotient<ZK, true> read index + 1 (mod n) and coset index + 4, round 4 adds A, B, C at zeta w and round 5 opens them
// there with Z; the proof gains those three evaluations (864 bytes).
#include <algorithm>
#include <cerrno>
#include <sys/random.h>

#include "common.cuh"
#include "comm.cuh"
#include "transcript.cuh"
#include "prover.cuh"
#include "memory_plan.cuh"

namespace pb200 {

void ntt_run(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in, const Fr* in_scale,
             const Fr* out_scale);
void ntt_run_on(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add);
void ntt_run_fold(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                  uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add, uint32_t fold);
void ntt_sharded(Context* ctx, const Fr* const* in, Fr* const* out, int count, int log_n, bool inverse);
void ntt_shard_local(Context* ctx, const Fr* const* in, int count, int log_n, bool inverse, uint64_t in_mul,
                     uint64_t in_add, int log_g, int rank, Comm* cm);
void ntt_shard_combine(Context* ctx, const Fr* sub, uint64_t rank_stride, Fr* out, int log_n, bool inverse,
                       uint64_t limit, const Fr* post_scale, uint32_t* nonzero, int log_g, int rank);
uint32_t msm_default_window(uint64_t n, bool fixed_base);

// Coefficients (n) -> evaluations on this rank's slice of the fixed coset (n_ext points): one forward transform of
// size n_ext with the coset shift multiplied in on load, zero padding (n_ext > n) or wrap-around (n_ext < n).
static void coset_extend(Prover* P, cudaStream_t stream, Fr* tmp, const Fr* coeff, Fr* out, const Fr* shift_pow) {
  ntt_run_fold(P->ctx, stream, tmp, coeff, out, P->log_ext, false, P->n, shift_pow, nullptr, 1, 0, P->fold);
}

// n Lagrange values -> n coefficients for `count` vectors (poly.py:132-139): one device, or slab-sharded over the
// ranks with one allgather for the whole group
static void interpolate(Prover* P, const Fr* const* lag, Fr* const* coeff, int count) {
  if (P->world > 1) {
    ntt_sharded(P->ctx, lag, coeff, count, P->log_n, true);
  } else {
    for (int k = 0; k < count; k++) ntt_run(P->ctx, lag[k], coeff[k], P->log_n, true, P->n, nullptr, nullptr);
  }
}

// Launch the coset extension (to the fixed 4n coset) of coefficient vectors [first, first+count) on the side
// stream: it depends only on data already produced on the main stream, so it can fill the under-occupied
// tails of the commitments (bucket reduction, scan, host round trips) that follow on the main stream.
static void launch_coset_ext_async(Prover* P, int first, int count, int done_event) {
  Context* ctx = P->ctx;
  if (!ctx->aux_stream) {
    PB_CUDA(cudaStreamCreateWithFlags(&ctx->aux_stream, cudaStreamNonBlocking));
    for (auto& e : ctx->aux_ev) PB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  P->aux_tmp.ensure(P->n_ext * 32);
  PB_CUDA(cudaEventRecord(ctx->aux_ev[3], ctx->stream));          // inputs ready
  PB_CUDA(cudaStreamWaitEvent(ctx->aux_stream, ctx->aux_ev[3], 0));
  for (int k = first; k < first + count; k++) {
    coset_extend(P, ctx->aux_stream, P->aux_tmp.as<Fr>(), P->coeff[k].as<Fr>(), P->ext[k].as<Fr>(), P->gpow.as<Fr>());
    if (k == 3 && P->zw_separate)  // Z(wX) on the slice: the same coefficients on the coset shifted by w
      coset_extend(P, ctx->aux_stream, P->aux_tmp.as<Fr>(), P->coeff[3].as<Fr>(), P->ext[5].as<Fr>(), P->gpow_w.as<Fr>());
  }
  PB_CUDA(cudaEventRecord(ctx->aux_ev[done_event], ctx->aux_stream));
}
void launch_powers(Context* ctx, Fr* out, uint64_t n, const Fr& base, const Fr& scale);
Fr fr_from_u64(uint64_t x);
Fr fr_root_of_unity(int log_n);
void fr_to_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
struct Srs;
void srs_msm(Context* ctx, Srs* srs, const Fr* d_scalars, uint64_t m, bool scalars_mont, uint8_t* out_xy, int* is_identity);
uint64_t srs_size(Srs* s);

// ------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------
static Fr load_fr_checked(const uint8_t* h) {
  Fr a;
  memcpy(a.v, h, 32);
  PB_CHECK(fp_is_canonical(a), "public input not reduced below the field modulus");
  return a;
}

// wire values arrive canonical (< r): a value >= r would silently become a different field element in fp_to_mont
__global__ void k_count_noncanonical(const Fr* v, uint64_t n, uint32_t* bad) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !fp_is_canonical(ldg_fr(v + i))) atomicAdd(bad, 1u);
}

// prover.py:108-116: A*QL + B*QR + A*B*QM + C*QO + PI + QC (+ sum_k Q_k m_k(A, B, C)) == 0 on every row.
// NEXT: the custom terms also read the next row's wires, cyclically (row n - 1 reads row 0).
template <bool NEXT>
__global__ void k_gate_check(const Fr* A, const Fr* B, const Fr* C, const Fr* QL, const Fr* QR, const Fr* QM,
                             const Fr* QO, const Fr* QC, const Fr* PI, CustomTerms ct, uint64_t n, uint32_t* bad) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr a = ldg_fr(A + i), b = ldg_fr(B + i), c = ldg_fr(C + i);
  Fr s = fp_mul(a, ldg_fr(QL + i));
  s = fp_add(s, fp_mul(b, ldg_fr(QR + i)));
  s = fp_add(s, fp_mul(fp_mul(a, b), ldg_fr(QM + i)));
  s = fp_add(s, fp_mul(c, ldg_fr(QO + i)));
  s = fp_add(s, fp_add(ldg_fr(PI + i), ldg_fr(QC + i)));
  if constexpr (NEXT) {
    const uint64_t i1 = i + 1 == n ? 0 : i + 1;
    s = custom_gate_sum_next(ct, i, a, b, c, ldg_fr(A + i1), ldg_fr(B + i1), ldg_fr(C + i1), s);
  } else {
    s = custom_gate_sum(ct, i, a, b, c, s);
  }
  if (!s.is_zero()) atomicAdd(bad, 1u);
}

// prover.py:125-131: per-row numerator / denominator of the grand product
struct PermChallenges { Fr beta, gamma; };
__global__ void k_perm_terms(const Fr* A, const Fr* B, const Fr* C, const Fr* S1, const Fr* S2, const Fr* S3,
                             const Fr* roots, PermChallenges ch, uint64_t n, Fr* num, Fr* den) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr a = fp_add(ldg_fr(A + i), ch.gamma), b = fp_add(ldg_fr(B + i), ch.gamma), c = fp_add(ldg_fr(C + i), ch.gamma);
  Fr bw = fp_mul(ch.beta, ldg_fr(roots + i));
  Fr bw2 = fp_dbl(bw), bw3 = fp_add(bw2, bw);
  num[i] = fp_mul(fp_mul(fp_add(a, bw), fp_add(b, bw2)), fp_add(c, bw3));
  Fr d1 = fp_add(a, fp_mul(ch.beta, ldg_fr(S1 + i)));
  Fr d2 = fp_add(b, fp_mul(ch.beta, ldg_fr(S2 + i)));
  Fr d3 = fp_add(c, fp_mul(ch.beta, ldg_fr(S3 + i)));
  den[i] = fp_mul(fp_mul(d1, d2), d3);
}

// out[i] = num[i] / den[i] (inv(0) = 0), Montgomery's trick over the strided set {t, t+T, ...}
// (strided so the accesses of a warp are coalesced).  num may be null (plain inversion).
#define PB_BATCH_CH 16
__global__ void __launch_bounds__(128) k_batch_div(const Fr* num, const Fr* den, Fr* out, uint64_t n, uint64_t T) {
  const int CH = PB_BATCH_CH;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  Fr pref[CH];
  Fr run = Fr::one();
  int cnt = 0;
  for (int k = 0; k < CH; k++) {
    uint64_t i = t + (uint64_t)k * T;
    if (i >= n) break;
    Fr d = ldg_fr(den + i);
    if (d.is_zero()) d = Fr::one();
    pref[k] = run;
    run = fp_mul(run, d);
    cnt++;
  }
  Fr inv = fp_inv_gcd(run);
  for (int k = cnt - 1; k >= 0; k--) {
    uint64_t i = t + (uint64_t)k * T;
    Fr d = ldg_fr(den + i);
    bool z = d.is_zero();
    if (z) d = Fr::one();
    Fr ik = fp_mul(inv, pref[k]);
    inv = fp_mul(inv, d);
    Fr r = z ? Fr::zero() : ik;
    if (num) r = fp_mul(r, ldg_fr(num + i));
    out[i] = r;
  }
}

// ---- exclusive scans over a monoid, 3 kernels over tiles of 256 x 8: the vector's tiles (one total per tile), the
// tile totals (one block), then every element from its tile's start.  ScanMul is the grand product, ScanAdd the
// suffix sum of the division below.
#define PB_FR_TILE 2048
struct ScanMul {
  static __device__ __forceinline__ Fr id() { return Fr::one(); }
  static __device__ __forceinline__ Fr op(const Fr& a, const Fr& b) { return fp_mul(a, b); }
};
struct ScanAdd {
  static __device__ __forceinline__ Fr id() { return Fr::zero(); }
  static __device__ __forceinline__ Fr op(const Fr& a, const Fr& b) { return fp_add(a, b); }
};
template <class Op>
__device__ __forceinline__ Fr block_exclusive_scan_256(const Fr& v, Fr* sh, Fr* total) {
  // Hillis-Steele over 256 threads in shared memory (inclusive), then shift
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int d = 1; d < 256; d <<= 1) {
    Fr x = sh[threadIdx.x];
    Fr y = (int)threadIdx.x >= d ? sh[threadIdx.x - d] : Op::id();
    __syncthreads();
    if ((int)threadIdx.x >= d) sh[threadIdx.x] = Op::op(x, y);
    __syncthreads();
  }
  Fr excl = threadIdx.x ? sh[threadIdx.x - 1] : Op::id();
  *total = sh[255];
  __syncthreads();
  return excl;
}
// the tile totals in place -> the exclusive scan of them, and the grand total
template <class Op>
__global__ void __launch_bounds__(256) k_fr_scan_tiles(Fr* tiles, uint32_t n_tiles, Fr* total_out) {
  __shared__ Fr sh[256];
  uint32_t per = (n_tiles + 255) / 256;
  uint32_t lo = threadIdx.x * per, hi = min(lo + per, n_tiles);
  Fr p = Op::id();
  for (uint32_t i = lo; i < hi; i++) p = Op::op(p, tiles[i]);
  Fr total;
  Fr run = block_exclusive_scan_256<Op>(p, sh, &total);
  for (uint32_t i = lo; i < hi; i++) {
    Fr c = tiles[i];
    tiles[i] = run;
    run = Op::op(run, c);
  }
  if (threadIdx.x == 0) *total_out = total;
}

// ---- exclusive prefix product: Z[0] = 1, Z[i+1] = Z[i] * f[i] ----
__global__ void __launch_bounds__(256) k_prod_tiles(const Fr* f, uint64_t n, Fr* tile_prod) {
  __shared__ Fr sh[256];
  uint64_t base = (uint64_t)blockIdx.x * PB_FR_TILE + threadIdx.x * 8;
  Fr p = Fr::one();
  for (int k = 0; k < 8; k++) if (base + k < n) p = fp_mul(p, ldg_fr(f + base + k));
  Fr total;
  block_exclusive_scan_256<ScanMul>(p, sh, &total);
  if (threadIdx.x == 0) tile_prod[blockIdx.x] = total;
}
// carry (optional): the product of everything below this vector (the slabs of the lower ranks in a sharded round 2)
__global__ void __launch_bounds__(256) k_prod_apply(const Fr* f, uint64_t n, const Fr* tile_prod, const Fr* carry, Fr* Z) {
  __shared__ Fr sh[256];
  uint64_t base = (uint64_t)blockIdx.x * PB_FR_TILE + threadIdx.x * 8;
  Fr c[8];
  Fr p = Fr::one();
  for (int k = 0; k < 8; k++) { c[k] = base + k < n ? ldg_fr(f + base + k) : Fr::one(); p = fp_mul(p, c[k]); }
  Fr total;
  Fr start = tile_prod[blockIdx.x];
  if (carry) start = fp_mul(start, ldg_fr(carry));
  Fr run = fp_mul(start, block_exclusive_scan_256<ScanMul>(p, sh, &total));
  for (int k = 0; k < 8; k++) {
    if (base + k < n) Z[base + k] = run;
    run = fp_mul(run, c[k]);
  }
}

// sharded grand product: totals[r] = product of slab r (gathered).  carry = product of the slabs below `rank`,
// grand = product of all of them (Z_n, which must be 1: prover.py:132)
__global__ void k_prod_carry(const Fr* totals, uint32_t world, uint32_t rank, Fr* carry, Fr* grand) {
  if (threadIdx.x || blockIdx.x) return;
  Fr c = Fr::one(), all = Fr::one();
  for (uint32_t r = 0; r < world; r++) {
    Fr t = totals[r];
    if (r < rank) c = fp_mul(c, t);
    all = fp_mul(all, t);
  }
  *carry = c;
  *grand = all;
}

// ---- division by (X - z) in coefficient space ---------------------------------------------------------------
// q_(k-1) = s_k with s_k = N_k + z s_(k+1); multiplying through by z^k turns the recurrence into a plain suffix
// sum: s_k z^k = sum_(m >= k) N_m z^m.  So: u = N .* z^m, suffix-sum scan (additions only), multiply by z^-k.
// The tile and apply kernels walk the vector from the top: logical position i <-> index n-1-i
__global__ void __launch_bounds__(256) k_sufsum_tiles(const Fr* N, const Fr* zpow, uint64_t n, Fr* tile_sum) {
  __shared__ Fr sh[256];
  uint64_t base = (uint64_t)blockIdx.x * PB_FR_TILE + threadIdx.x * 8;
  Fr p = Fr::zero();
  for (int k = 0; k < 8; k++)
    if (base + k < n) { uint64_t m = n - 1 - (base + k); p = fp_add(p, fp_mul(ldg_fr(N + m), ldg_fr(zpow + m))); }
  Fr total;
  block_exclusive_scan_256<ScanAdd>(p, sh, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}
// out[m-1] = z^-m * (carry + sum_(m' >= m) N_m' z^m')  for m >= 1 ; out[n-1] = carry * z^-n ; the m = 0 sum is dropped.
// One device: carry = 0 (the m = 0 sum is N(z), the remainder).  Slab of a sharded division: N, zpow, zinvpow and out
// point at the slab, `carry` holds the sums of the slabs above it and last_scale = z^-(first index above the slab).
__global__ void __launch_bounds__(256) k_sufsum_apply(const Fr* N, const Fr* zpow, const Fr* zinvpow, uint64_t n,
                                                      const Fr* tile_sum, const Fr* carry, Fr last_scale, Fr* out) {
  __shared__ Fr sh[256];
  uint64_t base = (uint64_t)blockIdx.x * PB_FR_TILE + threadIdx.x * 8;
  Fr c[8];
  Fr p = Fr::zero();
  for (int k = 0; k < 8; k++) {
    if (base + k < n) { uint64_t m = n - 1 - (base + k); c[k] = fp_mul(ldg_fr(N + m), ldg_fr(zpow + m)); }
    else c[k] = Fr::zero();
    p = fp_add(p, c[k]);
  }
  const Fr cy = carry ? ldg_fr(carry) : Fr::zero();
  Fr total;
  Fr run = fp_add(fp_add(tile_sum[blockIdx.x], cy), block_exclusive_scan_256<ScanAdd>(p, sh, &total));
  for (int k = 0; k < 8; k++) {
    run = fp_add(run, c[k]);  // inclusive suffix sum at m
    if (base + k < n) {
      uint64_t m = n - 1 - (base + k);
      if (m >= 1) out[m - 1] = fp_mul(run, ldg_fr(zinvpow + m));
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n - 1] = fp_mul(cy, last_scale);
}

// sharded division: totals[r] = sum of slab r (gathered from all ranks).  carry = sum of the slabs above `rank`;
// the grand total is the remainder N(z), which must vanish
__global__ void k_sufsum_carry(const Fr* totals, uint32_t world, uint32_t rank, Fr* carry, uint32_t* nonzero) {
  if (threadIdx.x || blockIdx.x) return;
  Fr c = Fr::zero(), all = Fr::zero();
  for (uint32_t r = 0; r < world; r++) {
    Fr t = totals[r];
    all = fp_add(all, t);
    if (r > rank) c = fp_add(c, t);
  }
  *carry = c;
  if (!all.is_zero()) atomicAdd(nonzero, 1u);
}

// basis_i[j] = w^i * (x_j^n - 1) / (n (x_j - w^i)) : the i-th Lagrange basis polynomial on the coset
__global__ void k_lagrange_den(const Fr* X, uint64_t n4, Fr wi, Fr n_mont, Fr* den) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n4) den[j] = fp_mul(n_mont, fp_sub(ldg_fr(X + j), wi));
}

// ---- round 3: quotient on the fixed coset -----------------------------------------------------------------
struct QuotientArgs {
  const Fr *A, *B, *C, *Z, *Zw, *PI;                  // extended (this rank's slice); Zw[j + zw_shift] = Z(w x_j)
  const Fr *QL, *QR, *QM, *QO, *QC, *S1, *S2, *S3;    // extended, cached per circuit
  const Fr *L0, *X;                                   // extended L0 and the coset points
  Fr zh_inv[4];                                       // 1 / (x_j^n - 1) for j mod 4
  Fr alpha, alpha2, beta, gamma, one;
  uint64_t n4;                                         // points of the slice
  uint64_t zw_shift;
  uint32_t world, rank;                                // global coset index of local j: world * j + rank
  // public inputs: PI(x_j) = sum_i pi_coef[i] * pi_basis[i][j]  (pi_cnt > 0), else the extended vector PI
  int pi_cnt;
  const Fr* pi_basis[8];
  Fr pi_coef[8];
  CustomTerms custom;                                  // extended custom selectors (this rank's slice)
};
// Zero knowledge: A'(x) = A(x) + (b1 x + b2) Z_H(x) (B', C' likewise), Z'(x) = Z(x) + (b7 x^2 + b8 x + b9) Z_H(x) and
// Z'(w x) = Z(w x) + (b7 w^2 x^2 + b8 w x + b9) Z_H(x), since Z_H(w x) = Z_H(x).  Z_H takes four values on the coset, so
// the blinders come pre-multiplied by each of them: w[k] = Z_H class k times
//   (b1, b2, b3, b4, b5, b6,  b7, b8, b9,  b7 w^2, b8 w, b9)
// and a point costs 7 products.  A separate parameter after T, so the plain kernel's parameters keep their offsets.
struct ZkCoset { Fr w[4][12]; };
// Zero knowledge on a next-row prover: A' = A + (b12 X^2 + b1 X + b2) Z_H, B' = B + (b13 X^2 + b3 X + b4) Z_H,
// C' = C + (b14 X^2 + b5 X + b6) Z_H, and the shifted wires A'(w x) = A(w x) + (b12 w^2 x^2 + b1 w x + b2) Z_H(x) like
// Z'(w x).  w[k] = Z_H class k times
//   (b12, b1, b2,  b13, b3, b4,  b14, b5, b6,  b7, b8, b9,  b7 w^2, b8 w, b9,
//    b12 w^2, b1 w, b2,  b13 w^2, b3 w, b4,  b14 w^2, b5 w, b6)
// and a point costs 16 products.
struct ZkNextCoset { Fr w[4][24]; };
template <bool ZK_NEXT> struct ZkCosetOf { using type = ZkCoset; };
template <> struct ZkCosetOf<true> { using type = ZkNextCoset; };
static_assert(sizeof(QuotientArgs) + sizeof(Fr*) + sizeof(ZkNextCoset) <= 4096,
              "k_quotient's parameters must fit the 4 KiB parameter space");
// NEXT (a next-row prover, one GPU): the custom terms also read A, B, C at w x, the coset index + zw_shift as for Z.
template <bool ZK, bool NEXT>
__global__ void __launch_bounds__(128) k_quotient(QuotientArgs q, Fr* T, typename ZkCosetOf<ZK && NEXT>::type zk) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n4) return;
  uint64_t jw = j + q.zw_shift >= q.n4 ? j + q.zw_shift - q.n4 : j + q.zw_shift;
  Fr a = ldg_fr(q.A + j), b = ldg_fr(q.B + j), c = ldg_fr(q.C + j);
  // y + ((w_i x + w_i+1) x + w_i+2), the quadratic Z_H multiple of a next-row zero-knowledge vector
  auto quad = [&](Fr y, int i) {
    if constexpr (ZK && NEXT) {
      const uint32_t k = (uint32_t)j & 3;
      const Fr x = ldg_fr(q.X + j);
      y = fp_add(y, fp_add(fp_mul(fp_add(fp_mul(zk.w[k][i], x), zk.w[k][i + 1]), x), zk.w[k][i + 2]));
    }
    return y;
  };
  if constexpr (ZK && NEXT) {
    a = quad(a, 0);
    b = quad(b, 3);
    c = quad(c, 6);
  } else if constexpr (ZK) {
    const uint32_t k = (uint32_t)(j * q.world + q.rank) & 3;
    const Fr x = ldg_fr(q.X + j);
    a = fp_add(a, fp_add(fp_mul(zk.w[k][0], x), zk.w[k][1]));
    b = fp_add(b, fp_add(fp_mul(zk.w[k][2], x), zk.w[k][3]));
    c = fp_add(c, fp_add(fp_mul(zk.w[k][4], x), zk.w[k][5]));
  }
  Fr gate = fp_mul(a, ldg_fr(q.QL + j));
  gate = fp_add(gate, fp_mul(b, ldg_fr(q.QR + j)));
  gate = fp_add(gate, fp_mul(fp_mul(a, b), ldg_fr(q.QM + j)));
  gate = fp_add(gate, fp_mul(c, ldg_fr(q.QO + j)));
  Fr pi = Fr::zero();
  if (q.pi_cnt > 0) {
    for (int i = 0; i < q.pi_cnt; i++) pi = fp_add(pi, fp_mul(q.pi_coef[i], ldg_fr(q.pi_basis[i] + j)));
  } else if (q.PI) {
    pi = ldg_fr(q.PI + j);
  }
  gate = fp_add(gate, fp_add(pi, ldg_fr(q.QC + j)));
  if constexpr (NEXT) {
    const Fr an = quad(ldg_fr(q.A + jw), 15), bn = quad(ldg_fr(q.B + jw), 18), cn = quad(ldg_fr(q.C + jw), 21);
    gate = custom_gate_sum_next(q.custom, j, a, b, c, an, bn, cn, gate);
  } else {
    gate = custom_gate_sum(q.custom, j, a, b, c, gate);
  }
  Fr ag = fp_add(a, q.gamma), bg = fp_add(b, q.gamma), cg = fp_add(c, q.gamma);
  Fr bx = fp_mul(q.beta, ldg_fr(q.X + j));
  Fr bx2 = fp_dbl(bx), bx3 = fp_add(bx2, bx);
  Fr z = ldg_fr(q.Z + j), zw = ldg_fr(q.Zw + jw);
  if constexpr (ZK && NEXT) {
    z = quad(z, 9);
    zw = quad(zw, 12);
  } else if constexpr (ZK) {
    const uint32_t k = (uint32_t)(j * q.world + q.rank) & 3;
    const Fr x = ldg_fr(q.X + j);
    z = fp_add(z, fp_add(fp_mul(fp_add(fp_mul(zk.w[k][6], x), zk.w[k][7]), x), zk.w[k][8]));
    zw = fp_add(zw, fp_add(fp_mul(fp_add(fp_mul(zk.w[k][9], x), zk.w[k][10]), x), zk.w[k][11]));
  }
  Fr p1 = fp_mul(fp_mul(fp_mul(fp_add(ag, bx), fp_add(bg, bx2)), fp_add(cg, bx3)), z);
  Fr p2 = fp_mul(fp_mul(fp_mul(fp_add(ag, fp_mul(q.beta, ldg_fr(q.S1 + j))), fp_add(bg, fp_mul(q.beta, ldg_fr(q.S2 + j)))),
                        fp_add(cg, fp_mul(q.beta, ldg_fr(q.S3 + j)))),
                 zw);
  Fr perm = fp_mul(q.alpha, fp_sub(p1, p2));
  Fr l0 = fp_mul(q.alpha2, fp_mul(fp_sub(z, q.one), ldg_fr(q.L0 + j)));
  Fr num = fp_add(fp_add(gate, perm), l0);
  T[j] = fp_mul(num, q.zh_inv[(j * q.world + q.rank) & 3]);
}

// number of non-zero entries among v[0..n)
__global__ void k_count_nonzero(const Fr* v, uint64_t n, uint32_t* cnt) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && !ldg_fr(v + i).is_zero()) atomicAdd(cnt, 1u);
}

// ---- parallel Horner: polys[p] (n coefficients) at xs[p] ------------------------------------------------
// level 1: H[p][c] = sum_k coeff[p][k*NC + c] * (x^NC)^k  for c < NC   (coalesced across c)
struct EvalArgs { const Fr* poly[8]; Fr x_nc[8]; uint64_t n; uint32_t NC; };
__global__ void __launch_bounds__(128) k_horner_strided(EvalArgs a, Fr* H) {
  uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t p = blockIdx.y;
  if (c >= a.NC) return;
  const Fr* co = a.poly[p];
  uint64_t steps = a.n / a.NC;
  Fr acc = Fr::zero();
  for (uint64_t k = steps; k-- > 0;) acc = fp_add(fp_mul(acc, a.x_nc[p]), ldg_fr(co + k * a.NC + c));
  H[(uint64_t)p * a.NC + c] = acc;
}

// ---- coefficient-space linear combination: out[k] = sum_i w[i] * vec[i][k] (+ c0 at k == 0) -----------------
// indices [first, first + n) of the result (a slab of a sharded round 5; first = 0, n = everything on one device).
// 26 slots: round 5's largest batch is 19 plain terms (5 gate selectors, 4 custom, Z, S3, T1-T3, A, B, C, S1, S2) and
// 7 lookup terms (q_K, Q_T with a table tag, Z2, H1, F, T, H2).
struct LinCombArgs { const Fr* vec[26]; Fr w[26]; Fr c0; int count; uint64_t n, first; };
// A shuffle adds 3 (Q_out, Z3, Q_in) to the 19 plain terms: 22.
static_assert(5 + PB_MAX_CUSTOM + 10 + 7 <= 26, "round 5's largest batch must fit LinCombArgs");
static_assert(5 + PB_MAX_CUSTOM + 10 + 3 <= 26, "round 5's batch with a shuffle must fit LinCombArgs");
// Zero knowledge: the tail holds the blinded vectors, Z, T1-T3, A, B, C (7), and Z3' with a shuffle: 8.
static_assert(7 + 1 <= 26, "round 5's zero-knowledge tail with a shuffle must fit LinCombArgs");
__global__ void __launch_bounds__(128) k_lincomb(LinCombArgs a, Fr* out) {
  uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.n) return;
  k += a.first;
  Fr acc = k == 0 ? a.c0 : Fr::zero();
  for (int i = 0; i < a.count; i++) acc = fp_add(acc, fp_mul(a.w[i], ldg_fr(a.vec[i] + k)));
  out[k] = acc;
}

// den[j] = shift * roots[j] - point    (the n-point coset x_j = shift * w^j minus the opening point)
__global__ void k_coset_minus(const Fr* roots, Fr shift, Fr point, uint64_t n, Fr* den) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) den[j] = fp_sub(fp_mul(shift, ldg_fr(roots + j)), point);
}

struct Four { Fr v[4]; };
// v[j] *= m[(global coset index of j) mod 4], global index = world * j + rank
__global__ void k_scale_by4(Fr* v, uint64_t n4, Four m, uint32_t world, uint32_t rank) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n4) v[j] = fp_mul(v[j], m.v[(j * world + rank) & 3]);
}
__global__ void k_negate(Fr* v, uint64_t n) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) v[j] = fp_neg(v[j]);
}

// One blinded coefficient vector: out[k] = (k < n_in ? in[k] : 0) + lo[k] (k < 3) + hi[k - n] (n <= k < n + 3),
// k < n_out.  With n >= 8 the two patches never meet.
struct ZkPatch { Fr lo[3], hi[3]; };
__global__ void k_zk_blind(const Fr* in, uint64_t n_in, uint64_t n, ZkPatch p, uint64_t n_out, Fr* out) {
  uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_out) return;
  Fr v = k < n_in ? ldg_fr(in + k) : Fr::zero();
  if (k < 3) v = fp_add(v, p.lo[k]);
  else if (k >= n && k < n + 3) v = fp_add(v, p.hi[k - n]);
  out[k] = v;
}

// ---- lookups (plookup, cyclic alternating split) ------------------------------------------------------------------
// exclusive scan of a uint32 count array (msm.cu): offsets[0..nb) and the total at offsets[nb]; counts are zeroed
#define PB_SCAN_TILE 2048
__global__ void k_scan_tile_sums(const uint32_t* counts, uint32_t nb, uint32_t pad, uint32_t* tile_sums, uint32_t* max_out);
__global__ void k_scan_tiles(uint32_t* tile_sums, uint32_t n_tiles, uint32_t* total_out);
__global__ void k_scan_apply(uint32_t* counts, uint32_t nb, uint32_t pad, const uint32_t* tile_sums, uint32_t* offsets);

// j_i: for a lookup row (q_K = 1) the lowest table index of a row equal to (a_i, b_i, c_i[, Q_T[i]]) -- the first of
// the equal rows in the sorted copy, which keeps table order among them --, else 0.  QT == nullptr: one untagged table,
// keys of three columns.  A row not in the table: the lowest such i goes to *missing.
__global__ void __launch_bounds__(128) k_lookup_index(const Fr* A, const Fr* B, const Fr* C, const Fr* QK, const Fr* QT,
                                                      const Fr* keys, const uint32_t* keys_idx, uint64_t rows, uint64_t n,
                                                      uint32_t* j_out, uint32_t* missing) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (ldg_fr(QK + i).is_zero()) { j_out[i] = 0; return; }
  const int width = QT ? 4 : 3;
  const Fr key[4] = {ldg_fr(A + i), ldg_fr(B + i), ldg_fr(C + i), QT ? ldg_fr(QT + i) : Fr::zero()};
  uint64_t lo = 0, hi = rows;
  while (lo < hi) {
    uint64_t mid = (lo + hi) / 2;
    if (lookup_cmp(keys + width * mid, key, width) < 0) lo = mid + 1;
    else hi = mid;
  }
  if (lo < rows && lookup_cmp(keys + width * lo, key, width) == 0) {
    j_out[i] = keys_idx[lo];
  } else {
    j_out[i] = 0;
    atomicMin(missing, (uint32_t)i);
  }
}

// histogram of j over the n table entries.  Every non-lookup row has j = 0, so equal keys are first merged within the
// warp: one atomic per distinct key per warp instead of one per row on a single counter.
__global__ void __launch_bounds__(256) k_lookup_hist(const uint32_t* j, uint64_t n, uint32_t* cnt) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t key = i < n ? j[i] : 0xffffffffu;
  const uint32_t peers = __match_any_sync(0xffffffffu, key);
  if (key != 0xffffffffu && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(cnt + key, (uint32_t)__popc(peers));
}

// s (2n positions) is the table in order, entry j taking 1 + cnt_j positions from start_j = j + off_j on: position p
// belongs to the last entry with start_j <= p.  Each position finds its entry by binary search, so no thread writes a run.
__global__ void __launch_bounds__(256) k_lookup_place(const uint32_t* off, uint64_t n, uint32_t* sidx) {
  uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= 2 * n) return;
  uint64_t lo = 0, hi = n;  // first entry with start > p
  while (lo < hi) {
    uint64_t mid = (lo + hi) / 2;
    if (mid + off[mid] <= p) lo = mid + 1;
    else hi = mid;
  }
  sidx[p] = (uint32_t)(lo - 1);
}

// t = t1 + eta t2 + eta^2 t3 (+ eta^3 t4 with a table tag; t4 == nullptr without), then f_i = t[j_i], h1_i = s_2i,
// h2_i = s_2i+1
__global__ void k_lookup_compress(const Fr* t1, const Fr* t2, const Fr* t3, const Fr* t4, Fr eta, Fr eta2, Fr eta3,
                                  uint64_t n, Fr* t) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr x = fp_add(ldg_fr(t1 + i), fp_add(fp_mul(eta, ldg_fr(t2 + i)), fp_mul(eta2, ldg_fr(t3 + i))));
  if (t4) x = fp_add(x, fp_mul(eta3, ldg_fr(t4 + i)));
  t[i] = x;
}
__global__ void k_lookup_gather(const Fr* t, const uint32_t* j, const uint32_t* sidx, uint64_t n, Fr* f, Fr* h1, Fr* h2) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  f[i] = ldg_fr(t + j[i]);
  h1[i] = ldg_fr(t + sidx[2 * i]);
  h2[i] = ldg_fr(t + sidx[2 * i + 1]);
}

// per-row numerator / denominator of Z2 (indices wrap at n):
//   (1+d)(e+f_i)(e(1+d)+t_i+d t_i+1)  /  (e(1+d)+h1_i+d h2_i)(e(1+d)+h2_i+d h1_i+1)
struct LookupChallenges { Fr delta, eps, one_d, eps_one_d; };
__global__ void k_lookup_z2_terms(const Fr* t, const Fr* f, const Fr* h1, const Fr* h2, LookupChallenges ch, uint64_t n,
                                  Fr* num, Fr* den) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t i1 = i + 1 == n ? 0 : i + 1;
  const Fr x1 = ldg_fr(h1 + i), x2 = ldg_fr(h2 + i);
  num[i] = fp_mul(fp_mul(ch.one_d, fp_add(ch.eps, ldg_fr(f + i))),
                  fp_add(fp_add(ch.eps_one_d, ldg_fr(t + i)), fp_mul(ch.delta, ldg_fr(t + i1))));
  den[i] = fp_mul(fp_add(fp_add(ch.eps_one_d, x1), fp_mul(ch.delta, x2)),
                  fp_add(fp_add(ch.eps_one_d, x2), fp_mul(ch.delta, ldg_fr(h1 + i1))));
}

// the three lookup terms of the quotient, added to the plain quotient's evaluations on the 4n coset (one GPU):
//   a3 [q_K (A + eta B + eta^2 C - F) + eta^3 Q_T]
// + a4 [Z2 (1+d)(e+F)(e(1+d) + T + d T(wX)) - Z2(wX)(e(1+d) + H1 + d H2)(e(1+d) + H2 + d H1(wX))]
// + a5 L0 (Z2 - 1),   all over Z_H.  X -> wX is index + 4 on the coset, as for Z.  Q_T = q_K * tag, the table id of
// each lookup row; QT == nullptr for one untagged table (the term is zero).
struct LookupQuotientArgs {
  const Fr *A, *B, *C, *QK, *QT, *T, *F, *H1, *H2, *Z2, *L0;
  Fr zh_inv[4];
  Fr eta, eta2, eta3, delta, eps, one_d, eps_one_d, alpha3, alpha4, alpha5, one;
  uint64_t n4;
};
// Zero knowledge (pb200_prover_set_zk_lookup): the kernel reads the unblinded extensions and adds the Z_H multiples, as
// k_quotient<true> does.  F' = F + (b12 X + b13) Z_H, H1' = H1 + (b14 X^2 + b15 X + b16) Z_H, H2' = H2 + (b17 X + b18) Z_H,
// Z2' = Z2 + (b19 X^2 + b20 X + b21) Z_H, and A' + eta B' + eta^2 C' = A + eta B + eta^2 C + (e1 X + e0) Z_H with
// e1 = b1 + eta b3 + eta^2 b5, e0 = b2 + eta b4 + eta^2 b6.  w[k] = Z_H class k times
//   (e1, e0,  b12, b13,  b14, b15, b16,  b14 w^2, b15 w, b16,  b17, b18,  b19, b20, b21,  b19 w^2, b20 w, b21)
// (the terms at wX use Z_H(w x) = Z_H(x)): 11 products a point.  A separate parameter after out, so the plain kernel's
// parameters keep their offsets.
struct ZkLookupCoset { const Fr* X; Fr w[4][18]; };
static_assert(sizeof(LookupQuotientArgs) + sizeof(Fr*) + sizeof(ZkLookupCoset) <= 4096,
              "k_quotient_lookup's parameters must fit the 4 KiB parameter space");
template <bool ZK>
__global__ void __launch_bounds__(128) k_quotient_lookup(LookupQuotientArgs q, Fr* out, ZkLookupCoset zk) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n4) return;
  const uint64_t jw = j + 4 >= q.n4 ? j + 4 - q.n4 : j + 4;
  // zero knowledge: y + (w_i x + w_i+1) or y + ((w_i x + w_i+1) x + w_i+2), the Z_H multiple of the blinded polynomial;
  // in the plain instance both return y.  Indexed in the parameter space (a pointer to the weights would copy them)
  const uint32_t k = (uint32_t)j & 3;
  const Fr x = ZK ? ldg_fr(zk.X + j) : Fr::zero();
  auto lin = [&](Fr y, int i) {
    if constexpr (ZK) y = fp_add(y, fp_add(fp_mul(zk.w[k][i], x), zk.w[k][i + 1]));
    return y;
  };
  auto quad = [&](Fr y, int i) {
    if constexpr (ZK) y = fp_add(y, fp_add(fp_mul(fp_add(fp_mul(zk.w[k][i], x), zk.w[k][i + 1]), x), zk.w[k][i + 2]));
    return y;
  };
  const Fr f = lin(ldg_fr(q.F + j), 2);
  Fr w = lin(fp_add(ldg_fr(q.A + j), fp_add(fp_mul(q.eta, ldg_fr(q.B + j)), fp_mul(q.eta2, ldg_fr(q.C + j)))), 0);
  Fr acc = fp_mul(ldg_fr(q.QK + j), fp_sub(w, f));
  if (q.QT) acc = fp_add(acc, fp_mul(q.eta3, ldg_fr(q.QT + j)));
  acc = fp_mul(q.alpha3, acc);
  const Fr z2 = quad(ldg_fr(q.Z2 + j), 12), h1 = quad(ldg_fr(q.H1 + j), 4), h2 = lin(ldg_fr(q.H2 + j), 10);
  Fr p1 = fp_mul(fp_mul(fp_mul(z2, q.one_d), fp_add(q.eps, f)),
                 fp_add(fp_add(q.eps_one_d, ldg_fr(q.T + j)), fp_mul(q.delta, ldg_fr(q.T + jw))));
  Fr p2 = fp_mul(fp_mul(quad(ldg_fr(q.Z2 + jw), 15), fp_add(fp_add(q.eps_one_d, h1), fp_mul(q.delta, h2))),
                 fp_add(fp_add(q.eps_one_d, h2), fp_mul(q.delta, quad(ldg_fr(q.H1 + jw), 7))));
  acc = fp_add(acc, fp_mul(q.alpha4, fp_sub(p1, p2)));
  acc = fp_add(acc, fp_mul(q.alpha5, fp_mul(fp_sub(z2, q.one), ldg_fr(q.L0 + j))));
  out[j] = fp_add(out[j], fp_mul(acc, q.zh_inv[j & 3]));
}

// ---- shuffle ------------------------------------------------------------------------------------------------------
// per-row numerator / denominator of Z3: with w = a + theta b + theta^2 c, num = 1 + q_in (kappa + w - 1) and
// den = 1 + q_out (kappa + w - 1).  The selectors are 0 or 1 on the rows, so each is 1 or kappa + w.
struct ShuffleChallenges { Fr theta, theta2, kappa; };
__global__ void k_shuffle_terms(const Fr* A, const Fr* B, const Fr* C, const Fr* QIN, const Fr* QOUT,
                                ShuffleChallenges ch, uint64_t n, Fr* num, Fr* den) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr t = fp_add(ch.kappa, fp_add(ldg_fr(A + i), fp_add(fp_mul(ch.theta, ldg_fr(B + i)),
                                                              fp_mul(ch.theta2, ldg_fr(C + i)))));
  num[i] = ldg_fr(QIN + i).is_zero() ? Fr::one() : t;
  den[i] = ldg_fr(QOUT + i).is_zero() ? Fr::one() : t;
}

// the two shuffle terms of the quotient, added to the plain quotient's evaluations on the 4n coset (one GPU):
//   a3 [Z3(wX) (1 + Q_out (K + W - 1)) - Z3 (1 + Q_in (K + W - 1))] + a4 L0 (Z3 - 1),   over Z_H,
// W = A + theta B + theta^2 C.  X -> wX is index + 4 on the coset, as for Z.
struct ShuffleQuotientArgs {
  const Fr *A, *B, *C, *QIN, *QOUT, *Z3, *L0;
  Fr zh_inv[4];
  Fr theta, theta2, kappa_m1, alpha3, alpha4, one;
  uint64_t n4;
};
// Zero knowledge (pb200_prover_set_zk_shuffle): the kernel reads the unblinded extensions and adds the Z_H multiples, as
// k_quotient_lookup<true> does.  Z3' = Z3 + (c2 X^2 + c1 X + c0) Z_H with Z3's blinders c2, c1, c0 (the last three), and
// A' + theta B' + theta^2 C' = W + (e2 X^2 + e1 X + e0) Z_H with e1 = b1 + theta b3 + theta^2 b5, e0 = b2 + theta b4 +
// theta^2 b6, e2 = b12 + theta b13 + theta^2 b14 on a next-row prover and 0 otherwise.  w[k] = Z_H class k times
//   (e2, e1, e0,  c2, c1, c0,  c2 w^2, c1 w, c0)
// (Z3'(wX) uses Z_H(w x) = Z_H(x)): 6 products a point.  A separate parameter after out, so the plain kernel's parameters
// keep their offsets.
struct ZkShuffleCoset { const Fr* X; Fr w[4][9]; };
static_assert(sizeof(ShuffleQuotientArgs) + sizeof(Fr*) + sizeof(ZkShuffleCoset) <= 4096,
              "k_quotient_shuffle's parameters must fit the 4 KiB parameter space");
template <bool ZK>
__global__ void __launch_bounds__(128) k_quotient_shuffle(ShuffleQuotientArgs q, Fr* out, ZkShuffleCoset zk) {
  uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q.n4) return;
  const uint64_t jw = j + 4 >= q.n4 ? j + 4 - q.n4 : j + 4;
  // zero knowledge: y + ((w_i x + w_i+1) x + w_i+2), the Z_H multiple of the blinded polynomial; in the plain instance it
  // returns y.  Indexed in the parameter space (a pointer to the weights would copy them)
  const uint32_t kz = (uint32_t)j & 3;
  const Fr x = ZK ? ldg_fr(zk.X + j) : Fr::zero();
  auto quad = [&](Fr y, int i) {
    if constexpr (ZK) y = fp_add(y, fp_add(fp_mul(fp_add(fp_mul(zk.w[kz][i], x), zk.w[kz][i + 1]), x), zk.w[kz][i + 2]));
    return y;
  };
  const Fr k = fp_add(q.kappa_m1, quad(fp_add(ldg_fr(q.A + j), fp_add(fp_mul(q.theta, ldg_fr(q.B + j)),
                                                                        fp_mul(q.theta2, ldg_fr(q.C + j)))), 0));
  const Fr z3 = quad(ldg_fr(q.Z3 + j), 3);
  Fr acc = fp_sub(fp_mul(quad(ldg_fr(q.Z3 + jw), 6), fp_add(q.one, fp_mul(ldg_fr(q.QOUT + j), k))),
                  fp_mul(z3, fp_add(q.one, fp_mul(ldg_fr(q.QIN + j), k))));
  acc = fp_add(fp_mul(q.alpha3, acc), fp_mul(q.alpha4, fp_mul(fp_sub(z3, q.one), ldg_fr(q.L0 + j))));
  out[j] = fp_add(out[j], fp_mul(acc, q.zh_inv[j & 3]));
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------

static void upload_mont(Context* ctx, DevBuf& dst, const uint8_t* h, uint64_t n) {
  dst.ensure(n * 32);
  PB_CUDA(cudaMemcpyAsync(dst.p, h, n * 32, cudaMemcpyHostToDevice, ctx->stream));
  fr_to_mont(ctx, dst.as<Fr>(), dst.as<Fr>(), n);
}

Comm* ctx_comm(Context* ctx);

// cached per prover: pi_basis[i][j] = L_i(x_j) on this rank's slice of the fixed coset for the first `count` rows.
// L0 is made when the prover is created (the quotient's L0 term); the public inputs add the rows they need.
static void ensure_pi_basis(Prover* P, int count) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n, ne = P->n_ext;
  cudaStream_t st = ctx->stream;
  if ((int)P->pi_basis.size() >= count) return;
  Fr w = fr_root_of_unity(P->log_n);
  DevBuf den(ne * 32);
  for (int i = (int)P->pi_basis.size(); i < count; i++) {
    Fr wi = fp_pow_u64(w, (uint64_t)i);
    Four zh;  // w^i (x_j^n - 1): four values
    for (int k = 0; k < 4; k++) zh.v[k] = fp_mul(wi, P->zh[k]);
    P->pi_basis.emplace_back(ne * 32);
    Fr* out = P->pi_basis.back().as<Fr>();
    k_lagrange_den<<<PB_GRID(ne, 256), 0, st>>>(P->xs.as<Fr>(), ne, wi, fr_from_u64(n), den.as<Fr>());
    uint64_t T = (ne + PB_BATCH_CH - 1) / PB_BATCH_CH;
    k_batch_div<<<PB_GRID(T, 128), 0, st>>>(nullptr, den.as<Fr>(), out, ne, T);
    k_scale_by4<<<PB_GRID(ne, 256), 0, st>>>(out, ne, zh, (uint32_t)P->world, (uint32_t)P->rank);
    ctx->launches += 3;
  }
  PB_CUDA(cudaStreamSynchronize(st));
}

// Custom term exponents -> the factors of the monomial.  width 3: (i, j, l); width 6: (i, j, l, i', j', l'), the last
// three on a(wX), b(wX), c(wX).  A same-row term keeps its rules: degree 1 duplicates QL / QR / QO, degree 4 would need
// a fourth quotient piece, (1, 1, 0) is QM's term.  A term with a next-row exponent may have degree 1, 2 or 3 (no
// selector reads the next row).  A repeated term is one term split in two.  Sets P->next_row when some term reads the
// next row.
static void set_custom_terms(Prover* P, int n_custom, const uint8_t* h_exps, int width) {
  PB_CHECK(n_custom >= 0 && n_custom <= PB_MAX_CUSTOM, "at most 4 custom gate terms");
  PB_CHECK(n_custom == 0 || h_exps, "custom gate terms need their exponents");
  uint8_t six[PB_MAX_CUSTOM][6] = {};
  bool next_row = false;
  for (int k = 0; k < n_custom; k++) {
    uint8_t* e = six[k];
    memcpy(e, h_exps + width * k, width);
    const bool next = e[3] || e[4] || e[5];
    const int deg = e[0] + e[1] + e[2] + e[3] + e[4] + e[5];
    if (next) {
      PB_CHECK(deg >= 1 && deg <= 3, "custom gate term with next-row exponents must have total degree 1, 2 or 3");
    } else {
      PB_CHECK(deg >= 2 && deg <= 3, "custom gate term must have total degree 2 or 3");
      PB_CHECK(!(e[0] == 1 && e[1] == 1 && e[2] == 0), "custom gate term (1, 1, 0) duplicates QM");
    }
    for (int k2 = 0; k2 < k; k2++)
      PB_CHECK(memcmp(e, six[k2], 6) != 0, "custom gate terms must have distinct exponents");
    next_row = next_row || next;
  }
  for (int k = 0; k < n_custom; k++) {
    int s = 0;
    for (int w = 0; w < 6; w++)
      for (int t = 0; t < six[k][w]; t++) P->custom_f[k][s++] = (uint8_t)w;
    while (s < 3) P->custom_f[k][s++] = PB_FACTOR_ONE;
  }
  P->n_custom = n_custom;
  P->next_row = next_row;
}

// Which round-3 layout a one-GPU prover of 2^log_n rows takes (memory_plan.cuh): true for the sliced one.  Throws,
// before anything is allocated, when neither fits the free device memory.  PB200_SLICED=1 forces the sliced layout.
static bool plan_memory(Context* ctx, Srs* srs, int log_n, int n_custom) {
  size_t free_b = 0, total_b = 0;
  PB_CUDA(cudaMemGetInfo(&free_b, &total_b));
  // the largest MSM of a proof: three commitments on the fixed-base table, or one at a time on the generic path
  const uint32_t buckets = srs_bucket_count(srs);
  uint32_t c = 1, batch = buckets ? 3 : 1;
  if (buckets) while ((1u << (c - 1)) < buckets) c++;
  else c = msm_default_window((uint64_t)1 << log_n, false);
  uint64_t msm_now = 0;
  for (int k = 1; k < 10; k++) msm_now += ctx->scratch[k].bytes;
  const ProverMemory m = prover_memory(log_n, n_custom, c, batch, msm_now);
  const char* e = getenv("PB200_SLICED");
  const int choice = plan_choose(m, free_b, e && atoi(e) != 0);
  if (choice < 0) {
    char b[256];
    const double gib = 1024.0 * 1024.0 * 1024.0;
    snprintf(b, sizeof b, "a 2^%d prover needs %.1f GiB (%.1f GiB sliced), %.1f GiB free (%.1f GiB kept in reserve)",
             log_n, m.full.total() / gib, m.sliced.total() / gib, free_b / gib, PB_PLAN_MARGIN / gib);
    throw Error(b);
  }
  return choice == 1;
}

// h_pk: 8 vectors (QM QL QR QO QC S1 S2 S3), each n x 32 bytes canonical (compiler/program.py:10-30); h_custom:
// n_custom more selector vectors of the same shape, with their exponents h_exps (exp_width = 3 or 6 bytes per term).
// sharded: one proof across the ranks of the context's communicator (see Prover in prover.cuh).
Prover* prover_create(Context* ctx, Srs* srs, int log_n, const uint8_t* const* h_pk, int n_custom,
                      const uint8_t* h_exps, const uint8_t* const* h_custom, bool sharded, int exp_width) {
  auto P = std::make_unique<Prover>();
  P->ctx = ctx;
  P->srs = srs;
  P->log_n = log_n;
  const uint64_t n = (uint64_t)1 << log_n, n4 = 4 * n;
  P->n = n;
  P->sharded = sharded;
  PB_CHECK(log_n >= 1 && log_n <= 26, "group order must be 2^k, 1 <= k <= 26");
  PB_CHECK(n <= srs_size(srs), "Not enough powers in setup");
  set_custom_terms(P.get(), n_custom, h_exps, exp_width);
  PB_CHECK(n_custom == 0 || h_custom, "custom gate terms need their selector columns");
  PB_CHECK(!(sharded && P->next_row), "next-row custom gate terms are not available on the sharded prover (one GPU only)");
  if (sharded) {
    Comm* cm = ctx_comm(ctx);
    P->world = comm_world(cm);
    P->rank = comm_rank(cm);
    P->log_world = comm_log_world(cm);
    PB_CHECK(log_n > P->log_world, "sharded prover: fewer rows than ranks");
  } else {
    P->sliced = plan_memory(ctx, srs, log_n, n_custom);
    PB_CHECK(!(P->sliced && P->next_row), PB_SLICED_WHY "next-row custom gate terms need the whole coset in round 3");
  }
  const uint32_t G = (uint32_t)P->world, R = (uint32_t)P->rank;
  P->log_ext = P->sliced ? log_n : log_n + 2 - P->log_world;
  const uint64_t ne = P->n_ext = (uint64_t)1 << P->log_ext;
  P->fold = ne < n ? (uint32_t)(n / ne) : 1;
  P->zw_separate = (4 % G) != 0;
  P->zw_shift = P->sliced ? 1 : P->zw_separate ? 0 : 4 / G;
  cudaStream_t st = ctx->stream;
  P->g = fr_from_u64(5);
  P->g_inv = fp_inv(P->g);
  Fr one = Fr::one();
  const Fr mu = fr_root_of_unity(log_n + 2);
  const Fr shift = fp_mul(P->g, fp_pow_u64(mu, R));  // this rank's slice is shift * <mu^world>
  // tables
  P->roots.alloc(n * 32);
  launch_powers(ctx, P->roots.as<Fr>(), n, fr_root_of_unity(log_n), one);
  P->gpow.alloc(n * 32);
  launch_powers(ctx, P->gpow.as<Fr>(), n, shift, one);
  if (P->zw_separate) {
    P->gpow_w.alloc(n * 32);
    launch_powers(ctx, P->gpow_w.as<Fr>(), n, fp_mul(shift, fr_root_of_unity(log_n)), one);
  }
  const uint64_t n_ginv = P->sliced ? 3 * n : n4;  // sliced: only the join of T's 3n coefficients reads it
  P->ginv_pow.alloc(n_ginv * 32);
  launch_powers(ctx, P->ginv_pow.as<Fr>(), n_ginv, P->g_inv, one);
  P->xs.alloc(ne * 32);
  launch_powers(ctx, P->xs.as<Fr>(), ne, fp_pow_u64(mu, P->sliced ? 4 : G), shift);  // sliced: rewritten per slice
  // Z_H on the coset takes 4 values: g^n * i^(j mod 4) - 1, i = mu^n, j the global coset index
  Fr i4 = fp_pow_u64(mu, n);
  Fr cur = fp_pow_u64(P->g, n);
  for (int k = 0; k < 4; k++) {
    P->zh[k] = fp_sub(cur, one);
    P->zh_inv[k] = fp_inv(P->zh[k]);
    cur = fp_mul(cur, i4);
  }
  if (P->sliced) P->pi_basis.emplace_back(n * 32);  // L0 of the slice round 3 is on
  else ensure_pi_basis(P.get(), 1);                   // L0, for the quotient
  for (int k = 0; k < Prover::CUSTOM0 + n_custom; k++) {
    upload_mont(ctx, P->sel_lag[k], k < Prover::CUSTOM0 ? h_pk[k] : h_custom[k - Prover::CUSTOM0], n);
    P->sel_coeff[k].alloc(n * 32);
    ntt_run(ctx, P->sel_lag[k].as<Fr>(), P->sel_coeff[k].as<Fr>(), log_n, true, n, nullptr, nullptr);
    P->sel_ext[k].alloc(ne * 32);
    if (!P->sliced)  // sliced: recomputed for each slice in round 3
      coset_extend(P.get(), st, nullptr, P->sel_coeff[k].as<Fr>(), P->sel_ext[k].as<Fr>(), P->gpow.as<Fr>());
  }
  for (int k = 0; k < 4; k++) P->lag[k].alloc(n * 32);
  for (int k = 0; k < 5; k++) { P->coeff[k].alloc(n * 32); P->ext[k].alloc(ne * 32); }
  if (P->zw_separate) P->ext[5].alloc(ne * 32);
  P->pi_lag.alloc(n * 32);
  if (P->world > 1) {
    P->tq.alloc(3 * n * 32);
    P->tq_loc.alloc(ne * 32);
  } else if (P->sliced) {
    P->tq.alloc(3 * n * 32);  // the slices' evaluations go to the four slots of the join in ctx->gather
  } else {
    P->tq.alloc(n4 * 32);
  }
  for (int k = 0; k < 5; k++) P->tmp[k].alloc(n * 32);
  P->flags.alloc(64);
  if (const char* e = getenv("PB200_OVERLAP")) P->overlap = atoi(e) != 0;
  if (P->sliced) P->overlap = false;  // the side stream would extend onto one slice while round 3 walks all four
  PB_CUDA(cudaStreamSynchronize(st));
  PB_CUDA(cudaGetLastError());
  return P.release();
}

void prover_destroy(Prover* p) { delete p; }

static uint32_t read_flag(Prover* P, int idx) {
  uint32_t v;
  PB_CUDA(cudaMemcpyAsync(&v, P->flags.as<uint32_t>() + idx, 4, cudaMemcpyDeviceToHost, P->ctx->stream));
  PB_CUDA(cudaStreamSynchronize(P->ctx->stream));
  return v;
}

Comm* ctx_comm(Context* ctx);

// evaluate up to 8 coefficient-form polynomials (n coeffs each, Montgomery) at Montgomery points:
// two strided-Horner levels on the device (n -> 4096 -> 32 partial values), the last 32 on the host
static void eval_polys(Prover* P, int count, const Fr* const* polys, const Fr* xs, Fr* out) {
  Context* ctx = P->ctx;
  // one proof across G ranks: rank r evaluates the slab of coefficients [r n/G, (r+1) n/G) of every polynomial;
  // the G partial values x^(r n/G) * slab(x) are exchanged with one small allgather and added on the host
  const uint64_t n = P->n / (uint64_t)P->world, lo = n * (uint64_t)P->rank;
  uint32_t NC1 = (uint32_t)std::min<uint64_t>(n, 4096);
  uint32_t NC2 = std::min<uint32_t>(NC1, 32);
  ctx->scratch[0].ensure((size_t)count * (NC1 + NC2) * 32);
  Fr* H1 = ctx->scratch[0].as<Fr>();
  Fr* H2 = H1 + (size_t)count * NC1;
  EvalArgs a;
  a.n = n;
  a.NC = NC1;
  for (int p = 0; p < count; p++) { a.poly[p] = polys[p] + lo; a.x_nc[p] = fp_pow_u64(xs[p], NC1); }
  k_horner_strided<<<dim3((NC1 + 127) / 128, count), 128, 0, ctx->stream>>>(a, H1);
  EvalArgs b;
  b.n = NC1;
  b.NC = NC2;
  for (int p = 0; p < count; p++) { b.poly[p] = H1 + (size_t)p * NC1; b.x_nc[p] = fp_pow_u64(xs[p], NC2); }
  k_horner_strided<<<dim3((NC2 + 127) / 128, count), 128, 0, ctx->stream>>>(b, H2);
  ctx->launches += 2;
  std::vector<Fr> h((size_t)count * NC2);
  PB_CUDA(cudaMemcpyAsync(h.data(), H2, h.size() * 32, cudaMemcpyDeviceToHost, ctx->stream));
  PB_CUDA(cudaStreamSynchronize(ctx->stream));
  for (int p = 0; p < count; p++) {
    Fr acc = Fr::zero();
    for (uint32_t c = NC2; c-- > 0;) acc = fp_add(fp_mul(acc, xs[p]), h[(size_t)p * NC2 + c]);
    out[p] = P->world > 1 ? fp_mul(acc, fp_pow_u64(xs[p], lo)) : acc;
  }
  if (P->world > 1) {
    const size_t bytes = (size_t)count * 32;
    ctx->gather.ensure((size_t)P->world * bytes);
    Fr* all = ctx->gather.as<Fr>();
    PB_CUDA(cudaMemcpyAsync(all + (size_t)P->rank * count, out, bytes, cudaMemcpyHostToDevice, ctx->stream));
    comm_allgather_inplace(ctx_comm(ctx), all, bytes, ctx->stream);
    std::vector<Fr> parts((size_t)P->world * count);
    PB_CUDA(cudaMemcpyAsync(parts.data(), all, parts.size() * 32, cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(cudaStreamSynchronize(ctx->stream));
    for (int p = 0; p < count; p++) {
      Fr acc = Fr::zero();
      for (int r = 0; r < P->world; r++) acc = fp_add(acc, parts[(size_t)r * count + p]);
      out[p] = acc;
    }
  }
}

static void store_canonical(uint8_t* dst, const Fr& mont) {
  Fr c = fp_from_mont(mont);
  memcpy(dst, c.v, 32);
}

// ---- zero knowledge -----------------------------------------------------------------------------------------------
// The blinding of the PLONK paper (eprint 2019/953, prover rounds 1-3), b1..b11 = zk_b[0..10], Z_H = X^n - 1:
//   A' = A + (b1 X + b2) Z_H,  B' = B + (b3 X + b4) Z_H,  C' = C + (b5 X + b6) Z_H,  Z' = Z + (b7 X^2 + b8 X + b9) Z_H,
//   T = (gate + alpha perm + alpha^2 L0 (Z' - 1)) / Z_H of degree <= 3n + 5, cut at n and 2n, then
//   T1' = T1 + b10 X^n,  T2' = T2 - b10 + b11 X^n,  T3' = T3 - b11   (T1' + X^n T2' + X^2n T3' = T).
// On H every blinded polynomial equals the unblinded one, so rounds 1-2 check the same witness; commitments, openings
// and round 5 use the blinded polynomials, evaluations are corrected on the host.  The verifier does not change.
// A next-row prover opens A, B, C at zeta w too, so they take a third blinder each (b12..b14):
//   A' = A + (b12 X^2 + b1 X + b2) Z_H,  B' = B + (b13 X^2 + b3 X + b4) Z_H,  C' = C + (b14 X^2 + b5 X + b6) Z_H,
// the permutation product reaches degree 4n + 8, deg T <= 3n + 8 and T3' has n + 9 coefficients (zk_t3_len, ZK_NR_PAD).

// Fresh blinders from the OS CSPRNG: 64 bytes per scalar, reduced mod r (bias below 2^-250).  No other source: a failed
// read fails the proof.
static void zk_random_blinders(Fr* out_mont, int count) {
  std::vector<uint8_t> buf((size_t)count * 64);
  size_t got = 0;
  while (got < buf.size()) {
    ssize_t r = getrandom(buf.data() + got, buf.size() - got, 0);
    if (r < 0) {
      PB_CHECK(errno == EINTR, "zero-knowledge blinders: getrandom() failed (no fallback source is used)");
      continue;
    }
    got += (size_t)r;
  }
  const Fr m = Fr::modulus();
  auto reduce = [&](Fr x) {  // x < 2^256 < 6 r: subtract r while x >= r
    while (!fp_is_canonical(x)) {
      uint64_t borrow = 0;
      for (int i = 0; i < 8; i++) {
        uint64_t d = (uint64_t)x.v[i] - m.v[i] - borrow;
        x.v[i] = (uint32_t)d;
        borrow = (d >> 32) & 1;
      }
    }
    return x;
  };
  for (int k = 0; k < count; k++) {
    Fr lo, hi;
    memcpy(lo.v, buf.data() + 64 * k, 32);
    memcpy(hi.v, buf.data() + 64 * k + 32, 32);
    // lo + hi 2^256 mod r: fp_to_mont(hi) = hi R mod r with R = 2^256, and the sum is canonical
    Fr v = fp_add(reduce(lo), fp_to_mont(reduce(hi)));
    out_mont[k] = fp_to_mont(v);
  }
  std::fill(buf.begin(), buf.end(), 0);
}

// Switch zero-knowledge mode on with zk_blinders() scalars (h_blinders: that many canonical 32-byte words, or null for
// fresh ones per proof).  Every check comes before any change, so a refused call leaves the prover as it was.
static void zk_enable(Prover* P, const uint8_t* h_blinders) {
  if (P->next_row) {
    PB_CHECK(P->n >= 16, "zero-knowledge proving with next-row terms needs n >= 16 rows: the blinded quotient has "
                         "degree 3n + 8 < 4n");
    PB_CHECK(srs_size(P->srs) >= P->n + 9, "Not enough powers in setup: zero-knowledge proving with next-row terms "
                                           "needs n + 9 powers (T3' has n + 9 coefficients)");
  }
  PB_CHECK(P->n >= 8, "zero-knowledge proving needs n >= 8 rows: the blinded quotient has degree 3n + 5 < 4n");
  PB_CHECK(srs_size(P->srs) >= P->n + 6,
           "Not enough powers in setup: zero-knowledge proving needs n + 6 powers (T3' has n + 6 coefficients)");
  const int count = P->zk_blinders();
  Fr fixed[Prover::ZK_LK_BLINDERS];
  for (int k = 0; h_blinders && k < count; k++) {
    memcpy(fixed[k].v, h_blinders + 32 * k, 32);
    PB_CHECK(fp_is_canonical(fixed[k]), "zero-knowledge blinder not reduced below the field modulus");
  }
  const size_t bytes = (P->n + P->zk_pad()) * 32;
  for (auto& b : P->zk_coeff) b.ensure(bytes);
  for (auto& b : P->zk_t) b.ensure(bytes);
  for (auto& b : P->tmp) b.ensure(bytes);  // round 5 works on n + 8 coefficients (n + 9 next-row)
  if (P->lk)
    for (auto& b : P->zk_lk) b.ensure(bytes);
  if (P->sh) P->zk_z3.ensure(bytes);
  if (h_blinders) std::copy(fixed, fixed + count, P->zk_fixed_b);
  P->zk_fixed = h_blinders != nullptr;
  P->zk = true;
}

// Zero-knowledge mode through the entry point of `block`: pb200_prover_set_zk (BLOCK_PLAIN) on a prover without a
// lookup table or shuffle; pb200_prover_set_zk_lookup (BLOCK_LOOKUP), the 11 blinders and b12..b21 for F, H1, H2 and
// Z2 (see "zero knowledge with lookups" below); pb200_prover_set_zk_shuffle (BLOCK_SHUFFLE), the 11 blinders (14 on a
// next-row prover) and the last three for Z3 (see "zero knowledge with a shuffle").  Separate entry points because
// they take other numbers of blinders: the size of the caller's buffer never depends on the prover's state.
// Switching off through any of them ends zero-knowledge mode.
void prover_set_zk(Prover* P, unsigned block, bool enable, const uint8_t* h_blinders) {
  PB_CHECK(!(enable && P->sliced), PB_SLICED_WHY "zero knowledge blinds the quotient on the whole coset in round 3");
  if (block != BLOCK_PLAIN) {
    PB_CHECK(P->world == 1, "zero-knowledge proving is not available on the sharded prover (one GPU only)");
    PB_CHECK(P->blocks() & block, block == BLOCK_LOOKUP
                                      ? "this prover has no lookup table (pb200_prover_set_lookup): use pb200_prover_set_zk"
                                      : "this prover has no shuffle (pb200_prover_set_shuffle): use pb200_prover_set_zk");
  }
  if (!enable) {
    P->zk = P->zk_fixed = false;
    for (auto& b : P->zk_coeff) b.release();
    for (auto& b : P->zk_t) b.release();
    for (auto& b : P->zk_lk) b.release();
    P->zk_z3.release();
    return;
  }
  if (block == BLOCK_PLAIN) {
    PB_CHECK(P->world == 1, "zero-knowledge proving is not available on the sharded prover (one GPU only)");
    PB_CHECK(!P->sh, "zero-knowledge mode does not combine with a shuffle here: a shuffle prover takes 14 blinders (17 "
                     "with next-row terms) through pb200_prover_set_zk_shuffle");
    PB_CHECK(!P->lk, "zero-knowledge mode does not combine with lookups here: a lookup prover takes 21 blinders through "
                     "pb200_prover_set_zk_lookup");
  }
  zk_enable(P, h_blinders);
}

static void zk_draw_blinders(Prover* P) {
  const int count = P->zk_blinders();
  if (P->zk_fixed) {
    for (int k = 0; k < count; k++) P->zk_b[k] = fp_to_mont(P->zk_fixed_b[k]);
  } else {
    zk_random_blinders(P->zk_b, count);
  }
}

// out (n + zk_pad(), zero padded) = in (n_in coefficients) + c(X) Z_H(X) with c = c[0] + c[1] X + ... (deg < 3)
static void zk_blind(Prover* P, const Fr* in, uint64_t n_in, const ZkPatch& p, Fr* out) {
  const uint64_t len = P->n + P->zk_pad();
  k_zk_blind<<<PB_GRID(len, 256), 0, P->ctx->stream>>>(in, n_in, P->n, p, len, out);
  P->ctx->launches++;
}
static ZkPatch zh_multiple(std::initializer_list<Fr> c) {
  ZkPatch p;
  for (int i = 0; i < 3; i++) p.lo[i] = p.hi[i] = Fr::zero();
  int i = 0;
  for (const Fr& x : c) { p.lo[i] = fp_neg(x); p.hi[i] = x; i++; }
  return p;
}

// ---- lookups ------------------------------------------------------------------------------------------------------
// plookup (eprint 2020/315) in the cyclic, alternating-split form of PlonKup (eprint 2022/086).  A boolean selector q_K
// marks the rows whose (a, b, c) must be a row of one fixed table (t1, t2, t3).  Per proof, with t = t1 + eta t2 +
// eta^2 t3: f_i = t[j_i] (j_i the lowest matching table index, 0 on other rows); s (2n) is t in table order with every
// entry followed by one copy per row that looks it up; h1 = s[0::2], h2 = s[1::2]; Z2 is the grand product of
// k_lookup_z2_terms.  The quotient gains k_quotient_lookup's three terms (degree <= 3n); round 5 opens F, T, H2 at
// zeta and T, H1, Z2 at zeta w.  The index, histogram and placement do not depend on eta and run in round 1.
// Several tables (PlonKup's table tag): the tables are concatenated, t4 holds each table row's table id and Q_T the id
// of the table each lookup row reads (0 off lookup rows).  t gains eta^3 t4, the index matches (a, b, c, Q_T), the
// quotient's alpha^3 term gains eta^3 Q_T and round 5 one slot, alpha^3 eta^3 Q_T.  With t4 = Q_T = 0 every one of
// these terms vanishes, so one table proves the same bytes tagged or not.
// Zero knowledge with lookups (pb200_prover_set_zk_lookup): everything of plain zero-knowledge mode, and b12..b21 blind the
// lookup polynomials the proof commits to, one scalar more than the points each is revealed at (PlonKup, 2022/086):
//   F' = F + (b12 X + b13) Z_H,  H1' = H1 + (b14 X^2 + b15 X + b16) Z_H,  H2' = H2 + (b17 X + b18) Z_H,
//   Z2' = Z2 + (b19 X^2 + b20 X + b21) Z_H.
// T, q_K and Q_T are fixed or public and stay as they are.  Z2 is built from the unblinded values, as the checks are;
// k_quotient_lookup<true> adds the Z_H multiples on the coset (A', B', C' included), round 4 corrects f, h2, h1(zeta w)
// and z2(zeta w), and round 5 uses the blinded vectors.  deg T <= 3n + 5 still holds (the lookup products reach 2n + 6
// after the division), so T is split as in plain zero-knowledge mode and the proof keeps its 1216 bytes.

// q_K, Q_T and the table as prover_set_lookup takes them (and the wire solver, which reads the same table): refuses a
// missing column, an empty table, more table rows than n, q_K not 0 or 1, Q_T not canonical or not 0 where q_K = 0,
// and a table value not canonical, in that order.
void lookup_require(uint64_t n, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* const* h_tab,
                    uint64_t rows) {
  const bool tagged = h_qtag != nullptr;
  PB_CHECK(h_qk && h_tab && h_tab[0] && h_tab[1] && h_tab[2], "lookups need q_K and three table columns");
  PB_CHECK(!tagged || h_tab[3], "tagged lookups need the table tag column t4");
  PB_CHECK(rows >= 1, "the lookup table is empty");
  PB_CHECK(rows <= n, "the lookup table has more rows than the circuit");
  // q_K: 0 or 1 on every row; Q_T canonical and 0 where q_K = 0
  for (uint64_t i = 0; i < n; i++) {
    const uint8_t* e = h_qk + 32 * i;
    bool ok = e[0] <= 1;
    for (int k = 1; k < 32 && ok; k++) ok = e[k] == 0;
    PB_CHECK(ok, "q_K must be 0 or 1 on every row");
    if (!tagged) continue;
    Fr x;
    memcpy(x.v, h_qtag + 32 * i, 32);
    PB_CHECK(fp_is_canonical(x), ("Q_T on row " + std::to_string(i) + " not reduced below the field modulus").c_str());
    PB_CHECK(e[0] == 1 || x.is_zero(), ("Q_T must be 0 where q_K = 0: row " + std::to_string(i)).c_str());
  }
  for (int w = 0; w < (tagged ? 4 : 3); w++)
    for (uint64_t r = 0; r < rows; r++) {
      Fr x;
      memcpy(x.v, h_tab[w] + 32 * r, 32);
      PB_CHECK(fp_is_canonical(x), "lookup table value not reduced below the field modulus");
    }
}

// h_qtag == nullptr: one untagged table of three columns (h_tab[3] unused).  Otherwise several tables concatenated: the
// fourth column h_tab[3] holds each table row's table id and h_qtag = Q_T the id of the table each lookup row reads,
// zero wherever q_K = 0.  The rows are matched on (a, b, c, Q_T) and compressed with eta^3 t4 (eta^3 Q_T in the
// quotient), so a row can only match a row of its own table.
void prover_set_lookup(Prover* P, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* const* h_tab,
                       uint64_t rows) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  const bool tagged = h_qtag != nullptr;
  const int width = tagged ? 4 : 3;
  PB_CHECK(P->world == 1, "lookups are not available on the sharded prover (one GPU only)");
  PB_CHECK(!P->sliced, PB_SLICED_WHY "the lookup quotient needs the whole coset in round 3");
  PB_CHECK(!P->next_row, "lookups do not combine with next-row custom gate terms");
  PB_CHECK(!P->sh, "lookups do not combine with a shuffle");
  PB_CHECK(!P->zk, "lookups do not combine with zero-knowledge mode switched on first: set the table, then "
                   "pb200_prover_set_zk_lookup");
  PB_CHECK(!P->lk, "the lookup table is already set (set it once, before the first proof)");
  lookup_require(n, h_qk, h_qtag, h_tab, rows);
  // the table, padded to n rows by repeating its last row, in Montgomery form
  std::vector<Fr> tab[4];
  for (int w = 0; w < width; w++) {
    tab[w].resize(n);
    for (uint64_t r = 0; r < n; r++) {
      Fr x;
      memcpy(x.v, h_tab[w] + 32 * std::min(r, rows - 1), 32);
      tab[w][r] = fp_to_mont(x);
    }
  }
  // stable: equal rows keep table order, so the first of them in the sorted copy is the lowest table index
  std::vector<uint32_t> order(rows);
  for (uint64_t r = 0; r < rows; r++) order[r] = (uint32_t)r;
  const Fr zero = Fr::zero();
  std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
    const Fr kx[4] = {tab[0][x], tab[1][x], tab[2][x], tagged ? tab[3][x] : zero};
    const Fr ky[4] = {tab[0][y], tab[1][y], tab[2][y], tagged ? tab[3][y] : zero};
    return lookup_cmp(kx, ky, width) < 0;
  });
  std::vector<Fr> keys(width * rows);
  for (uint64_t r = 0; r < rows; r++)
    for (int w = 0; w < width; w++) keys[width * r + w] = tab[w][order[r]];
  cudaStream_t st = ctx->stream;
  P->lk_keys.alloc(keys.size() * 32);
  P->lk_keys_idx.alloc(rows * 4);
  PB_CUDA(cudaMemcpyAsync(P->lk_keys.p, keys.data(), keys.size() * 32, cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemcpyAsync(P->lk_keys_idx.p, order.data(), rows * 4, cudaMemcpyHostToDevice, st));
  for (int w = 0; w < width; w++) {
    P->lk_tab[w].alloc(n * 32);
    PB_CUDA(cudaMemcpyAsync(P->lk_tab[w].p, tab[w].data(), n * 32, cudaMemcpyHostToDevice, st));
  }
  upload_mont(ctx, P->lk_qk_lag, h_qk, n);
  P->lk_qk_coeff.alloc(n * 32);
  ntt_run(ctx, P->lk_qk_lag.as<Fr>(), P->lk_qk_coeff.as<Fr>(), P->log_n, true, n, nullptr, nullptr);
  P->lk_qk_ext.alloc(P->n_ext * 32);
  coset_extend(P, st, nullptr, P->lk_qk_coeff.as<Fr>(), P->lk_qk_ext.as<Fr>(), P->gpow.as<Fr>());
  if (tagged) {  // Q_T as q_K: Lagrange values (the index), coefficients (round 5), the 4n coset (the quotient)
    upload_mont(ctx, P->lk_qt_lag, h_qtag, n);
    P->lk_qt_coeff.alloc(n * 32);
    ntt_run(ctx, P->lk_qt_lag.as<Fr>(), P->lk_qt_coeff.as<Fr>(), P->log_n, true, n, nullptr, nullptr);
    P->lk_qt_ext.alloc(P->n_ext * 32);
    coset_extend(P, st, nullptr, P->lk_qt_coeff.as<Fr>(), P->lk_qt_ext.as<Fr>(), P->gpow.as<Fr>());
  }
  P->lk_j.alloc(n * 4);
  P->lk_cnt.alloc(n * 4);
  P->lk_off.alloc((n + 1) * 4);
  P->lk_sidx.alloc(2 * n * 4);
  for (int k = 0; k < Prover::LK_VECS; k++) {
    P->lk_lag[k].alloc(n * 32);
    P->lk_coeff[k].alloc(n * 32);
    P->lk_ext[k].alloc(P->n_ext * 32);
  }
  PB_CUDA(cudaStreamSynchronize(st));  // the host copies die here
  P->lk_rows = rows;
  P->lk_tagged = tagged;
  P->lk = true;
}

// round 1: table index of every row, the histogram over the table entries and each position's entry in s
static void lookup_index(Prover* P) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  uint32_t* missing = P->flags.as<uint32_t>() + 2;
  PB_CUDA(cudaMemsetAsync(missing, 0xff, 4, st));
  k_lookup_index<<<PB_GRID(n, 128), 0, st>>>(P->lag[0].as<Fr>(), P->lag[1].as<Fr>(), P->lag[2].as<Fr>(),
                                            P->lk_qk_lag.as<Fr>(), P->lk_tagged ? P->lk_qt_lag.as<Fr>() : nullptr,
                                            P->lk_keys.as<Fr>(), P->lk_keys_idx.as<uint32_t>(), P->lk_rows, n,
                                            P->lk_j.as<uint32_t>(), missing);
  PB_CUDA(cudaMemsetAsync(P->lk_cnt.p, 0, n * 4, st));
  k_lookup_hist<<<PB_GRID(n, 256), 0, st>>>(P->lk_j.as<uint32_t>(), n, P->lk_cnt.as<uint32_t>());
  const uint32_t n_tiles = (uint32_t)((n + PB_SCAN_TILE - 1) / PB_SCAN_TILE);
  ctx->scratch[0].ensure((size_t)n_tiles * 4);
  uint32_t* tiles = ctx->scratch[0].as<uint32_t>();
  uint32_t* off = P->lk_off.as<uint32_t>();
  k_scan_tile_sums<<<n_tiles, 256, 0, st>>>(P->lk_cnt.as<uint32_t>(), (uint32_t)n, 0, tiles, nullptr);
  k_scan_tiles<<<1, 256, 0, st>>>(tiles, n_tiles, off + n);
  k_scan_apply<<<n_tiles, 256, 0, st>>>(P->lk_cnt.as<uint32_t>(), (uint32_t)n, 0, tiles, off);
  k_lookup_place<<<PB_GRID(2 * n, 256), 0, st>>>(off, n, P->lk_sidx.as<uint32_t>());
  ctx->launches += 6;
  const uint32_t row = read_flag(P, 2);
  PB_CHECK(row == 0xffffffffu,
           ("AssertionError: lookup row " + std::to_string(row) + " is not in the table").c_str());
}

// step 1L: t, f, h1, h2 from eta, and one commitment pass over f, h1, h2
void prover_round_lookup(Prover* P, const Fr& eta_c) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  PB_CHECK(P->lk, "this prover has no lookup table (pb200_prover_set_lookup)");
  P->eta = fp_to_mont(eta_c);
  Fr* v[Prover::LK_VECS];
  for (int k = 0; k < Prover::LK_VECS; k++) v[k] = P->lk_lag[k].as<Fr>();
  const Fr eta2 = fp_sqr(P->eta);
  k_lookup_compress<<<PB_GRID(n, 256), 0, st>>>(P->lk_tab[0].as<Fr>(), P->lk_tab[1].as<Fr>(), P->lk_tab[2].as<Fr>(),
                                               P->lk_tagged ? P->lk_tab[3].as<Fr>() : nullptr, P->eta, eta2,
                                               fp_mul(eta2, P->eta), n, v[Prover::LK_T]);
  k_lookup_gather<<<PB_GRID(n, 256), 0, st>>>(v[Prover::LK_T], P->lk_j.as<uint32_t>(), P->lk_sidx.as<uint32_t>(), n,
                                             v[Prover::LK_F], v[Prover::LK_H1], v[Prover::LK_H2]);
  ctx->launches += 2;
  const Fr* lag[4] = {v[Prover::LK_T], v[Prover::LK_F], v[Prover::LK_H1], v[Prover::LK_H2]};
  Fr* coeff[4] = {P->lk_coeff[Prover::LK_T].as<Fr>(), P->lk_coeff[Prover::LK_F].as<Fr>(),
                  P->lk_coeff[Prover::LK_H1].as<Fr>(), P->lk_coeff[Prover::LK_H2].as<Fr>()};
  interpolate(P, lag, coeff, 4);
  if (P->zk) {  // F' H1' H2' (n + 2, n + 3, n + 2 coefficients), and T zero padded to n + 8 for round 5
    const Fr* b = P->zk_b;
    zk_blind(P, coeff[0], n, zh_multiple({}), P->zk_lk[Prover::LK_T].as<Fr>());
    zk_blind(P, coeff[1], n, zh_multiple({b[12], b[11]}), P->zk_lk[Prover::LK_F].as<Fr>());
    zk_blind(P, coeff[2], n, zh_multiple({b[15], b[14], b[13]}), P->zk_lk[Prover::LK_H1].as<Fr>());
    zk_blind(P, coeff[3], n, zh_multiple({b[17], b[16]}), P->zk_lk[Prover::LK_H2].as<Fr>());
  }
  const Fr* fh[3] = {P->lk_poly(Prover::LK_F), P->lk_poly(Prover::LK_H1), P->lk_poly(Prover::LK_H2)};
  P->commit_batch(fh, 3, P->zk ? n + 3 : n, P->fields[F_F]);
}

// A grand product (Z of the permutation argument, Z2 of the lookup argument) from its per-row numerators and
// denominators on this rank's slab [lo, lo + n/G) -- num and den point at the slab; num is overwritten with num / den.
// lag (all n rows) gets the exclusive prefix product, coeff its coefficients.  One proof across G ranks: the divisions
// and the in-slab prefix products are local; the slab products are exchanged with a 32-byte allgather (the product of
// the lower slabs is the slab's carry) and the values with one bulk allgather.  The product over all rows must be 1:
// `not_one` is the error otherwise.
static void grand_product(Prover* P, Fr* num, const Fr* den, Fr* lag, Fr* coeff, const char* not_one) {
  Context* ctx = P->ctx;
  cudaStream_t st = ctx->stream;
  const uint64_t ns = P->n / (uint64_t)P->world, lo = ns * (uint64_t)P->rank;
  uint64_t T = (ns + PB_BATCH_CH - 1) / PB_BATCH_CH;
  k_batch_div<<<PB_GRID(T, 128), 0, st>>>(num, den, num, ns, T);
  uint32_t n_tiles = (uint32_t)((ns + PB_FR_TILE - 1) / PB_FR_TILE);
  PB_CHECK(n_tiles <= 65536, "group order too large for the product scan");
  ctx->scratch[0].ensure((size_t)(n_tiles + 1 + 16) * 32);
  Fr* tiles = ctx->scratch[0].as<Fr>();
  Fr* totals = tiles + n_tiles + 1;  // [world] slab products, then carry and grand total
  k_prod_tiles<<<n_tiles, 256, 0, st>>>(num, ns, tiles);
  k_fr_scan_tiles<ScanMul><<<1, 256, 0, st>>>(tiles, n_tiles, tiles + n_tiles);
  const Fr* d_total = tiles + n_tiles;
  if (P->world > 1) {
    PB_CUDA(cudaMemcpyAsync(totals + P->rank, tiles + n_tiles, 32, cudaMemcpyDeviceToDevice, st));
    comm_allgather_inplace(ctx_comm(ctx), totals, 32, st);
    Fr* carry = totals + P->world;
    k_prod_carry<<<1, 32, 0, st>>>(totals, (uint32_t)P->world, (uint32_t)P->rank, carry, carry + 1);
    k_prod_apply<<<n_tiles, 256, 0, st>>>(num, ns, tiles, carry, lag + lo);
    comm_allgather_inplace(ctx_comm(ctx), lag, ns * 32, st);
    d_total = carry + 1;
    ctx->launches++;
  } else {
    k_prod_apply<<<n_tiles, 256, 0, st>>>(num, ns, tiles, nullptr, lag);
  }
  ctx->launches += 4;
  Fr total;
  PB_CUDA(cudaMemcpyAsync(&total, d_total, 32, cudaMemcpyDeviceToHost, st));
  const Fr* zl = lag;
  interpolate(P, &zl, &coeff, 1);
  PB_CUDA(cudaStreamSynchronize(st));
  PB_CHECK(total == Fr::one(), not_one);
}

// ---- shuffle ------------------------------------------------------------------------------------------------------
// Two fixed boolean selectors Q_in and Q_out claim that the multiset {(a_i, b_i, c_i) : q_in[i] = 1} equals the multiset
// {(a_i, b_i, c_i) : q_out[i] = 1}; no copy constraint joins the two sides.  After beta and gamma the transcript draws
// theta and kappa (no commitment in between).  With w_i = a_i + theta b_i + theta^2 c_i, Z3 is the grand product of
// num_i / den_i = (1 + q_in[i](kappa + w_i - 1)) / (1 + q_out[i](kappa + w_i - 1)) (k_shuffle_terms), Z3_n = 1 iff
// the two products agree.  The quotient gains k_quotient_shuffle's two terms at alpha^3, alpha^4 (degree <= 3n - 3, so T
// keeps three pieces); round 4 evaluates Q_in at zeta and Z3 at zeta w; round 5 keeps [Q_out] and [Z3] in the
// linearisation, opens Q_in at zeta (v^6) and Z3 at zeta w (v, or v^4 after A, B, C on a next-row prover).  A row with
// both selectors cancels out.  Not with lookups (their alpha^3..alpha^5 terms) or the sharded prover.
// Zero knowledge with a shuffle (pb200_prover_set_zk_shuffle): everything of zero-knowledge mode (b1..b11, or b1..b14 on a
// next-row prover), and Z3' = Z3 + (b_(m-2) X^2 + b_(m-1) X + b_m) Z_H with the last three of the m = 14 (17) blinders,
// one scalar more than the points Z3 is revealed at (zeta w and the linearisation).  Q_in and Q_out are fixed and stay
// as they are.  Z3 is built from the unblinded values, as the check is; k_quotient_shuffle<true> adds the Z_H multiples
// on the coset (A', B', C' included), round 4 corrects z3(zeta w) and round 5 uses Z3'.  deg T <= 3n + 5 (3n + 8) still
// holds (the shuffle products reach 2n + 2, 2n + 3 next-row, after the division), so T is split as in zero-knowledge
// mode and the proof keeps its 896 (992) bytes.

// q_in and q_out as prover_set_shuffle takes them (and the wire solver): n x 32 bytes canonical, 0 or 1 on every row,
// with as many ones in each
void shuffle_require(uint64_t n, const uint8_t* h_qin, const uint8_t* h_qout) {
  PB_CHECK(h_qin && h_qout, "a shuffle needs q_in and q_out");
  uint64_t ones[2] = {0, 0};
  const uint8_t* sel[2] = {h_qin, h_qout};
  for (int s = 0; s < 2; s++)
    for (uint64_t i = 0; i < n; i++) {
      const uint8_t* e = sel[s] + 32 * i;
      bool ok = e[0] <= 1;
      for (int k = 1; k < 32 && ok; k++) ok = e[k] == 0;
      PB_CHECK(ok, s ? "q_out must be 0 or 1 on every row" : "q_in must be 0 or 1 on every row");
      ones[s] += e[0];
    }
  PB_CHECK(ones[0] == ones[1], ("a shuffle needs as many q_in rows as q_out rows: " + std::to_string(ones[0]) +
                                " and " + std::to_string(ones[1])).c_str());
}

// Every check comes before any change, so a refused call leaves the prover as it was.
void prover_set_shuffle(Prover* P, const uint8_t* h_qin, const uint8_t* h_qout) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  PB_CHECK(P->world == 1, "shuffles are not available on the sharded prover (one GPU only)");
  PB_CHECK(!P->sliced, PB_SLICED_WHY "the shuffle quotient needs the whole coset in round 3");
  PB_CHECK(!P->lk, "shuffles do not combine with lookups");
  PB_CHECK(!P->zk, "shuffles do not combine with zero-knowledge mode switched on first: set the shuffle, then "
                   "pb200_prover_set_zk_shuffle");
  PB_CHECK(!P->sh, "the shuffle selectors are already set (set them once, before the first proof)");
  shuffle_require(n, h_qin, h_qout);
  const uint8_t* sel[2] = {h_qin, h_qout};
  cudaStream_t st = ctx->stream;
  for (int s = 0; s < 2; s++) {  // as q_K: Lagrange values (round 2), coefficients (rounds 4, 5), the 4n coset (round 3)
    upload_mont(ctx, P->sh_lag[s], sel[s], n);
    P->sh_coeff[s].alloc(n * 32);
    ntt_run(ctx, P->sh_lag[s].as<Fr>(), P->sh_coeff[s].as<Fr>(), P->log_n, true, n, nullptr, nullptr);
    P->sh_ext[s].alloc(P->n_ext * 32);
    coset_extend(P, st, nullptr, P->sh_coeff[s].as<Fr>(), P->sh_ext[s].as<Fr>(), P->gpow.as<Fr>());
  }
  P->sh_z3_lag.alloc(n * 32);
  P->sh_z3_coeff.alloc(n * 32);
  P->sh_z3_ext.alloc(P->n_ext * 32);
  PB_CUDA(cudaStreamSynchronize(st));  // the caller's host buffers may die after the call
  P->sh = true;
}

// round 2 of a shuffle proof, after Z: the grand product Z3, then one commitment pass over Z and Z3
static void shuffle_round2(Prover* P) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  ShuffleChallenges ch{P->theta, fp_sqr(P->theta), P->kappa};
  Fr* num = P->tmp[2].as<Fr>();
  Fr* den = P->tmp[3].as<Fr>();
  k_shuffle_terms<<<PB_GRID(n, 128), 0, st>>>(P->lag[0].as<Fr>(), P->lag[1].as<Fr>(), P->lag[2].as<Fr>(),
                                             P->sh_lag[Prover::SH_IN].as<Fr>(), P->sh_lag[Prover::SH_OUT].as<Fr>(), ch,
                                             n, num, den);
  ctx->launches++;
  grand_product(P, num, den, P->sh_z3_lag.as<Fr>(), P->sh_z3_coeff.as<Fr>(),
                "AssertionError: shuffle: the q_in rows and the q_out rows are not permutations of each other");
  if (P->zk) {  // Z' and Z3': n + 3 coefficients each
    const Fr *b = P->zk_b, *c = P->zk_z3_b();
    zk_blind(P, P->coeff[3].as<Fr>(), n, zh_multiple({b[8], b[7], b[6]}), P->zk_coeff[3].as<Fr>());
    zk_blind(P, P->sh_z3_coeff.as<Fr>(), n, zh_multiple({c[2], c[1], c[0]}), P->zk_z3.as<Fr>());
  }
  const Fr* zz[2] = {P->zk ? P->zk_coeff[3].as<Fr>() : P->coeff[3].as<Fr>(), P->sh_z3_poly()};
  uint8_t out[2][64];
  P->commit_batch(zz, 2, P->zk ? n + 3 : n, out[0]);
  memcpy(P->fields[F_Z], out[0], 64);
  memcpy(P->fields[F_Z3], out[1], 64);
}

// round 2 of a lookup proof, after Z: the grand product Z2, then one commitment pass over Z and Z2
static void lookup_round2(Prover* P) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  LookupChallenges ch;
  ch.delta = P->delta;
  ch.eps = P->epsilon;
  ch.one_d = fp_add(Fr::one(), P->delta);
  ch.eps_one_d = fp_mul(P->epsilon, ch.one_d);
  Fr* num = P->tmp[2].as<Fr>();
  Fr* den = P->tmp[3].as<Fr>();
  k_lookup_z2_terms<<<PB_GRID(n, 128), 0, st>>>(P->lk_lag[Prover::LK_T].as<Fr>(), P->lk_lag[Prover::LK_F].as<Fr>(),
                                               P->lk_lag[Prover::LK_H1].as<Fr>(), P->lk_lag[Prover::LK_H2].as<Fr>(), ch, n,
                                               num, den);
  ctx->launches++;
  Fr* zc = P->lk_coeff[Prover::LK_Z2].as<Fr>();
  grand_product(P, num, den, P->lk_lag[Prover::LK_Z2].as<Fr>(), zc,
                "AssertionError: lookup grand product does not close, Z2_n != 1");
  if (P->zk) {  // Z' and Z2': n + 3 coefficients each
    const Fr* b = P->zk_b;
    zk_blind(P, P->coeff[3].as<Fr>(), n, zh_multiple({b[8], b[7], b[6]}), P->zk_coeff[3].as<Fr>());
    zk_blind(P, zc, n, zh_multiple({b[20], b[19], b[18]}), P->zk_lk[Prover::LK_Z2].as<Fr>());
  }
  const Fr* zz[2] = {P->zk ? P->zk_coeff[3].as<Fr>() : P->coeff[3].as<Fr>(), P->lk_poly(Prover::LK_Z2)};
  uint8_t out[2][64];
  P->commit_batch(zz, 2, P->zk ? n + 3 : n, out[0]);
  memcpy(P->fields[F_Z], out[0], 64);
  memcpy(P->fields[F_Z2], out[1], 64);
}

// ---- round 1 (prover.py:86-119) -------------------------------------------------------------------------
void prover_round1(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                   uint64_t n_public, bool wires_on_device) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  PB_CHECK(n_public <= n, "more public inputs than rows");
  if (P->zk) zk_draw_blinders(P);  // here, so the whole-proof call and the round-by-round path behave alike
  if (ctx->aux_stream) {
    // a previous proof that failed a check may have left coset extensions running on the side stream: everything
    // this proof writes is ordered after them
    PB_CUDA(cudaEventRecord(ctx->aux_ev[2], ctx->aux_stream));
    PB_CUDA(cudaStreamWaitEvent(st, ctx->aux_ev[2], 0));
  }
  const uint8_t* src[3] = {hA, hB, hC};
  PB_CUDA(cudaMemsetAsync(P->flags.p, 0, 64, st));  // [0] gate check, [1] wire values not reduced below r
  for (uint64_t i = 0; i < n_public; i++) (void)load_fr_checked(h_public + 32 * i);
  if (wires_on_device) {
    for (int k = 0; k < 3; k++) {
      k_count_noncanonical<<<PB_GRID(n, 256), 0, st>>>(reinterpret_cast<const Fr*>(src[k]), n, P->flags.as<uint32_t>() + 1);
      fr_to_mont(ctx, reinterpret_cast<const Fr*>(src[k]), P->lag[k].as<Fr>(), n);
    }
    ctx->launches += 3;
  } else {
    // stage the three wire vectors on a copy stream so the transfers of B and C overlap the conversion and
    // transform of the previous vector (the copy engine runs beside the SMs)
    if (!ctx->copy_stream) {
      PB_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
      for (auto& e : ctx->copy_done) PB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    PB_CUDA(cudaEventRecord(ctx->copy_done[3], st));  // the destination buffers are free once prior work is done
    PB_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_done[3], 0));
    // one proof across G ranks: every rank stages only its 1/G slab of each wire column over PCIe and the ranks
    // exchange slabs over NVLink (one allgather per column) -- the host is read once, not G times
    const uint64_t slab = n / (uint64_t)P->world, first = slab * (uint64_t)P->rank;
    for (int k = 0; k < 3; k++) {
      PB_CUDA(cudaMemcpyAsync(P->lag[k].as<Fr>() + first, src[k] + first * 32, slab * 32, cudaMemcpyHostToDevice,
                              ctx->copy_stream));
      PB_CUDA(cudaEventRecord(ctx->copy_done[k], ctx->copy_stream));
    }
    for (int k = 0; k < 3; k++) {
      PB_CUDA(cudaStreamWaitEvent(st, ctx->copy_done[k], 0));
      if (P->world > 1) comm_allgather_inplace(ctx_comm(ctx), P->lag[k].p, slab * 32, st);
      k_count_noncanonical<<<PB_GRID(n, 256), 0, st>>>(P->lag[k].as<Fr>(), n, P->flags.as<uint32_t>() + 1);
      ctx->launches++;
      fr_to_mont(ctx, P->lag[k].as<Fr>(), P->lag[k].as<Fr>(), n);
      if (P->world == 1) ntt_run(ctx, P->lag[k].as<Fr>(), P->coeff[k].as<Fr>(), P->log_n, true, n, nullptr, nullptr);
    }
  }
  const Fr* abc_lag[3] = {P->lag[0].as<Fr>(), P->lag[1].as<Fr>(), P->lag[2].as<Fr>()};
  Fr* abc_coeff[3] = {P->coeff[0].as<Fr>(), P->coeff[1].as<Fr>(), P->coeff[2].as<Fr>()};
  // PI: Lagrange values -public_i (prover.py:57-62)
  PB_CUDA(cudaMemsetAsync(P->pi_lag.p, 0, n * 32, st));
  if (n_public) {
    PB_CUDA(cudaMemcpyAsync(P->pi_lag.p, h_public, n_public * 32, cudaMemcpyHostToDevice, st));
    fr_to_mont(ctx, P->pi_lag.as<Fr>(), P->pi_lag.as<Fr>(), n_public);
    k_negate<<<PB_GRID(n_public, 128), 0, st>>>(P->pi_lag.as<Fr>(), n_public);
    ctx->launches++;
  }
  (P->next_row ? k_gate_check<true> : k_gate_check<false>)<<<PB_GRID(n, 128), 0, st>>>(
      P->lag[0].as<Fr>(), P->lag[1].as<Fr>(), P->lag[2].as<Fr>(), P->sel_lag[Prover::QL].as<Fr>(),
      P->sel_lag[Prover::QR].as<Fr>(), P->sel_lag[Prover::QM].as<Fr>(), P->sel_lag[Prover::QO].as<Fr>(),
      P->sel_lag[Prover::QC].as<Fr>(), P->pi_lag.as<Fr>(), P->custom_terms(P->sel_lag), n, P->flags.as<uint32_t>());
  ctx->launches++;
  if (wires_on_device || P->world > 1) interpolate(P, abc_lag, abc_coeff, 3);
  // public inputs: few of them -> PI is a short combination of cached Lagrange-basis vectors (no transforms);
  // otherwise fall back to interpolating PI like any other column
  P->n_public = n_public;
  P->pi_sparse = n_public <= 8;
  if (P->pi_sparse) {
    if (!P->sliced) ensure_pi_basis(P, (int)n_public);  // sliced: made for each slice in round 3
    P->pub_neg.resize(n_public);
    for (uint64_t i = 0; i < n_public; i++) {
      Fr v;
      memcpy(v.v, h_public + 32 * i, 32);
      P->pub_neg[i] = fp_neg(fp_to_mont(v));
    }
  } else {
    const Fr* pl = P->pi_lag.as<Fr>();
    Fr* pc = P->coeff[4].as<Fr>();
    interpolate(P, &pl, &pc, 1);
  }
  uint32_t fl[2];
  PB_CUDA(cudaMemcpyAsync(fl, P->flags.p, 8, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  PB_CHECK(fl[1] == 0, "wire value not reduced below the field modulus (canonical 32-byte little-endian expected)");
  PB_CHECK(fl[0] == 0, "AssertionError: witness does not satisfy the gate constraints (prover.py:108-116)");
  if (P->lk) lookup_index(P);
  if (P->overlap) launch_coset_ext_async(P, 0, 3, 0);
  if (P->zk && P->next_row) {  // A' B' C': n + 3 coefficients (b12..b14 in front of the usual two)
    const Fr* b = P->zk_b;
    for (int k = 0; k < 3; k++)
      zk_blind(P, P->coeff[k].as<Fr>(), n, zh_multiple({b[2 * k + 1], b[2 * k], b[11 + k]}), P->zk_coeff[k].as<Fr>());
    const Fr* abc[3] = {P->zk_coeff[0].as<Fr>(), P->zk_coeff[1].as<Fr>(), P->zk_coeff[2].as<Fr>()};
    P->commit_batch(abc, 3, n + 3, P->fields[F_A]);
    return;
  }
  if (P->zk) {  // A' B' C': n + 2 coefficients
    const Fr* b = P->zk_b;
    for (int k = 0; k < 3; k++)
      zk_blind(P, P->coeff[k].as<Fr>(), n, zh_multiple({b[2 * k + 1], b[2 * k]}), P->zk_coeff[k].as<Fr>());
    const Fr* abc[3] = {P->zk_coeff[0].as<Fr>(), P->zk_coeff[1].as<Fr>(), P->zk_coeff[2].as<Fr>()};
    P->commit_batch(abc, 3, n + 2, P->fields[F_A]);
    return;
  }
  const Fr* abc[3] = {P->coeff[0].as<Fr>(), P->coeff[1].as<Fr>(), P->coeff[2].as<Fr>()};
  P->commit_batch(abc, 3, n, P->fields[F_A]);
}

// ---- round 2 (prover.py:121-152) -------------------------------------------------------------------------
// ch: the challenges drawn before round 2, canonical, indexed by ProofChallenge -- beta and gamma, theta and kappa for a
// shuffle, delta and epsilon for lookups (the ones of blocks the prover does not have are not read)
void prover_round2(Prover* P, const Fr* ch) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  P->beta = fp_to_mont(ch[CH_BETA]);
  P->gamma = fp_to_mont(ch[CH_GAMMA]);
  P->theta = fp_to_mont(ch[CH_THETA]);
  P->kappa = fp_to_mont(ch[CH_KAPPA]);
  P->delta = fp_to_mont(ch[CH_DELTA]);
  P->epsilon = fp_to_mont(ch[CH_EPSILON]);
  PermChallenges perm{P->beta, P->gamma};
  // one proof across G ranks: rank r builds the slab [r n/G, (r+1) n/G) of the grand product (see grand_product)
  const uint64_t ns = n / (uint64_t)P->world, lo = ns * (uint64_t)P->rank;
  Fr* num = P->tmp[0].as<Fr>() + lo;
  Fr* den = P->tmp[1].as<Fr>() + lo;
  k_perm_terms<<<PB_GRID(ns, 128), 0, st>>>(P->lag[0].as<Fr>() + lo, P->lag[1].as<Fr>() + lo, P->lag[2].as<Fr>() + lo,
                                           P->sel_lag[Prover::S1].as<Fr>() + lo, P->sel_lag[Prover::S2].as<Fr>() + lo,
                                           P->sel_lag[Prover::S3].as<Fr>() + lo, P->roots.as<Fr>() + lo, perm, ns, num, den);
  ctx->launches++;
  grand_product(P, num, den, P->lag[3].as<Fr>(), P->coeff[3].as<Fr>(),
                "AssertionError: permutation grand product does not close, Z_n != 1 (prover.py:132)");
  if (P->overlap) launch_coset_ext_async(P, 3, 1, 1);
  if (P->lk) {  // Z2, and Z with it in one commitment pass (both blinded in zero-knowledge mode)
    lookup_round2(P);
    return;
  }
  if (P->sh) {  // Z3, and Z with it in one commitment pass
    shuffle_round2(P);
    return;
  }
  if (P->zk) {  // Z': n + 3 coefficients
    const Fr* b = P->zk_b;
    zk_blind(P, P->coeff[3].as<Fr>(), n, zh_multiple({b[8], b[7], b[6]}), P->zk_coeff[3].as<Fr>());
    P->commit(P->zk_coeff[3].as<Fr>(), n + 3, P->fields[F_Z]);
    return;
  }
  P->commit(P->coeff[3].as<Fr>(), n, P->fields[F_Z]);
}

// ---- sliced round 3 -----------------------------------------------------------------------------------------
void fr_vec_op(Context* ctx, int op, const Fr* a, const Fr* b, const Fr& scalar_canonical, Fr* out, uint64_t n,
               uint64_t shift);

// out[j] = c L_i(x_j) on slice r: Z_H is the constant zh[r] there, so L_i(x) = w^i Z_H / (n (x - w^i)) is one
// denominator and one batched inversion (tmp[0] holds the denominators)
static void slice_lagrange(Prover* P, int r, uint64_t i, const Fr& c, Fr* out) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  const Fr wi = fp_pow_u64(fr_root_of_unity(P->log_n), i);
  const Fr scale = fp_mul(fr_from_u64(n), fp_inv(fp_mul(fp_mul(wi, P->zh[r]), c)));  // 1 / den = c L_i
  k_lagrange_den<<<PB_GRID(n, 256), 0, ctx->stream>>>(P->xs.as<Fr>(), n, wi, scale, P->tmp[0].as<Fr>());
  const uint64_t T = (n + PB_BATCH_CH - 1) / PB_BATCH_CH;
  k_batch_div<<<PB_GRID(T, 128), 0, ctx->stream>>>(nullptr, P->tmp[0].as<Fr>(), out, n, T);
  ctx->launches += 2;
}

// The quotient of a sliced prover: for r = 0..3 the n points {g mu^(4j + r)} of the 4n coset (world = 4, rank = r in
// k_quotient, so Z(w x_j) is the next point of the slice and Z_H is one constant): A, B, C, Z (PI when dense) and
// every selector are extended onto the slice, L0 and a sparse PI come from the closed form, and the slice's inverse
// transform goes to slot r of ctx->gather with the join's twiddle on the store (ntt_shard_local).  The join then keeps
// T's 3n coefficients in tq and counts the non-zero top n in flags[0] (prover.py:205-208).
static void quotient_sliced(Prover* P) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  const Fr mu = fr_root_of_unity(P->log_n + 2), w = fr_root_of_unity(P->log_n);
  ctx->gather.ensure(4 * n * 32);
  QuotientArgs q;
  q.pi_cnt = 0;
  q.A = P->ext[0].as<Fr>(); q.B = P->ext[1].as<Fr>(); q.C = P->ext[2].as<Fr>(); q.Z = P->ext[3].as<Fr>();
  q.Zw = q.Z;
  q.zw_shift = P->zw_shift;
  q.world = 4;
  q.PI = P->pi_sparse && P->n_public == 0 ? nullptr : P->ext[4].as<Fr>();
  q.QM = P->sel_ext[Prover::QM].as<Fr>(); q.QL = P->sel_ext[Prover::QL].as<Fr>(); q.QR = P->sel_ext[Prover::QR].as<Fr>();
  q.QO = P->sel_ext[Prover::QO].as<Fr>(); q.QC = P->sel_ext[Prover::QC].as<Fr>();
  q.S1 = P->sel_ext[Prover::S1].as<Fr>(); q.S2 = P->sel_ext[Prover::S2].as<Fr>(); q.S3 = P->sel_ext[Prover::S3].as<Fr>();
  q.custom = P->custom_terms(P->sel_ext);
  q.L0 = P->pi_basis[0].as<Fr>(); q.X = P->xs.as<Fr>();
  for (int k = 0; k < 4; k++) q.zh_inv[k] = P->zh_inv[k];
  q.alpha = P->alpha; q.alpha2 = fp_sqr(P->alpha); q.beta = P->beta; q.gamma = P->gamma; q.one = Fr::one();
  q.n4 = n;
  const ZkCoset zk{};
  for (int r = 0; r < 4; r++) {
    const Fr shift = fp_mul(P->g, fp_pow_u64(mu, (uint64_t)r));
    launch_powers(ctx, P->gpow.as<Fr>(), n, shift, Fr::one());
    launch_powers(ctx, P->xs.as<Fr>(), n, w, shift);
    for (int k = 0; k < (P->pi_sparse ? 4 : 5); k++)
      coset_extend(P, st, nullptr, P->coeff[k].as<Fr>(), P->ext[k].as<Fr>(), P->gpow.as<Fr>());
    for (int k = 0; k < Prover::CUSTOM0 + P->n_custom; k++)
      coset_extend(P, st, nullptr, P->sel_coeff[k].as<Fr>(), P->sel_ext[k].as<Fr>(), P->gpow.as<Fr>());
    slice_lagrange(P, r, 0, Fr::one(), P->pi_basis[0].as<Fr>());
    if (P->pi_sparse) {  // PI = sum_i -public_i L_i, summed into ext[4] (tmp[1] holds a term)
      bool first = true;
      for (uint64_t i = 0; i < P->n_public; i++) {
        if (P->pub_neg[i].is_zero()) continue;
        slice_lagrange(P, r, i, P->pub_neg[i], first ? P->ext[4].as<Fr>() : P->tmp[1].as<Fr>());
        if (!first) fr_vec_op(ctx, 0, P->ext[4].as<Fr>(), P->tmp[1].as<Fr>(), Fr::zero(), P->ext[4].as<Fr>(), n, 0);
        first = false;
      }
      if (first && P->n_public) PB_CUDA(cudaMemsetAsync(P->ext[4].p, 0, n * 32, st));
    }
    q.rank = (uint32_t)r;
    Fr* slot = ctx->gather.as<Fr>() + (uint64_t)r * n;
    k_quotient<false, false><<<PB_GRID(n, 128), 0, st>>>(q, slot, zk);
    ctx->launches++;
    const Fr* te = slot;
    ntt_shard_local(ctx, &te, 1, P->log_n + 2, true, 1, 0, 2, r, nullptr);
  }
  PB_CUDA(cudaMemsetAsync(P->flags.p, 0, 64, st));
  ntt_shard_combine(ctx, ctx->gather.as<Fr>(), n, P->tq.as<Fr>(), P->log_n + 2, true, 3 * n, P->ginv_pow.as<Fr>(),
                    P->flags.as<uint32_t>(), 2, 0);
}

// ---- round 3 (prover.py:154-226) -------------------------------------------------------------------------
void prover_round3(Prover* P, const Fr& alpha_c, const Fr& cofactor_c) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n, n4 = 4 * n, ne = P->n_ext;
  cudaStream_t st = ctx->stream;
  P->alpha = fp_to_mont(alpha_c);
  P->fft_cofactor = fp_to_mont(cofactor_c);
  if (P->sliced) {
    quotient_sliced(P);
    PB_CHECK(read_flag(P, 0) == 0, "AssertionError: quotient has degree >= 3n (prover.py:205-208)");
    const Fr* t123[3] = {P->tq.as<Fr>(), P->tq.as<Fr>() + n, P->tq.as<Fr>() + 2 * n};
    P->commit_batch(t123, 3, n, P->fields[F_T_LO]);
    return;
  }
  if (P->overlap) {  // A, B, C, Z were extended on the side stream during rounds 1 and 2
    PB_CUDA(cudaStreamWaitEvent(st, ctx->aux_ev[0], 0));
    PB_CUDA(cudaStreamWaitEvent(st, ctx->aux_ev[1], 0));
  }
  for (int k = (P->overlap ? 4 : 0); k < (P->pi_sparse ? 4 : 5); k++) {
    coset_extend(P, st, nullptr, P->coeff[k].as<Fr>(), P->ext[k].as<Fr>(), P->gpow.as<Fr>());
    if (k == 3 && P->zw_separate)
      coset_extend(P, st, nullptr, P->coeff[3].as<Fr>(), P->ext[5].as<Fr>(), P->gpow_w.as<Fr>());
  }
  QuotientArgs q;
  q.pi_cnt = P->pi_sparse ? (int)P->n_public : 0;
  for (int i = 0; i < q.pi_cnt; i++) { q.pi_basis[i] = P->pi_basis[i].as<Fr>(); q.pi_coef[i] = P->pub_neg[i]; }
  q.A = P->ext[0].as<Fr>(); q.B = P->ext[1].as<Fr>(); q.C = P->ext[2].as<Fr>(); q.Z = P->ext[3].as<Fr>();
  q.Zw = P->zw_separate ? P->ext[5].as<Fr>() : P->ext[3].as<Fr>();
  q.zw_shift = P->zw_shift;
  q.world = (uint32_t)P->world;
  q.rank = (uint32_t)P->rank;
  q.PI = P->pi_sparse ? nullptr : P->ext[4].as<Fr>();
  q.QM = P->sel_ext[Prover::QM].as<Fr>(); q.QL = P->sel_ext[Prover::QL].as<Fr>(); q.QR = P->sel_ext[Prover::QR].as<Fr>();
  q.QO = P->sel_ext[Prover::QO].as<Fr>(); q.QC = P->sel_ext[Prover::QC].as<Fr>();
  q.S1 = P->sel_ext[Prover::S1].as<Fr>(); q.S2 = P->sel_ext[Prover::S2].as<Fr>(); q.S3 = P->sel_ext[Prover::S3].as<Fr>();
  q.custom = P->custom_terms(P->sel_ext);
  q.L0 = P->pi_basis[0].as<Fr>(); q.X = P->xs.as<Fr>();
  for (int k = 0; k < 4; k++) q.zh_inv[k] = P->zh_inv[k];
  q.alpha = P->alpha; q.alpha2 = fp_sqr(P->alpha); q.beta = P->beta; q.gamma = P->gamma; q.one = Fr::one();
  q.n4 = ne;
  Fr* t_evals = P->world > 1 ? P->tq_loc.as<Fr>() : P->tq.as<Fr>();
  ZkCoset zk{};
  if (P->next_row && P->zk) {
    const Fr* b = P->zk_b;
    const Fr w = fr_root_of_unity(P->log_n), w2 = fp_sqr(w);
    const Fr per[24] = {b[11], b[0], b[1], b[12], b[2], b[3], b[13], b[4], b[5], b[6], b[7], b[8],
                        fp_mul(b[6], w2), fp_mul(b[7], w), b[8], fp_mul(b[11], w2), fp_mul(b[0], w), b[1],
                        fp_mul(b[12], w2), fp_mul(b[2], w), b[3], fp_mul(b[13], w2), fp_mul(b[4], w), b[5]};
    ZkNextCoset zn;
    for (int k = 0; k < 4; k++)
      for (int i = 0; i < 24; i++) zn.w[k][i] = fp_mul(per[i], P->zh[k]);
    k_quotient<true, true><<<PB_GRID(ne, 128), 0, st>>>(q, t_evals, zn);
  } else if (P->next_row) {
    k_quotient<false, true><<<PB_GRID(ne, 128), 0, st>>>(q, t_evals, zk);
  } else if (P->zk) {
    const Fr* b = P->zk_b;
    const Fr w = fr_root_of_unity(P->log_n);
    const Fr per[12] = {b[0], b[1], b[2], b[3], b[4], b[5], b[6], b[7], b[8], fp_mul(b[6], fp_sqr(w)), fp_mul(b[7], w), b[8]};
    for (int k = 0; k < 4; k++)
      for (int i = 0; i < 12; i++) zk.w[k][i] = fp_mul(per[i], P->zh[k]);
    k_quotient<true, false><<<PB_GRID(ne, 128), 0, st>>>(q, t_evals, zk);
  } else {
    k_quotient<false, false><<<PB_GRID(ne, 128), 0, st>>>(q, t_evals, zk);
  }
  ctx->launches++;
  if (P->lk) {  // one GPU: the slice is the whole 4n coset
    for (int k = 0; k < Prover::LK_VECS; k++)
      coset_extend(P, st, nullptr, P->lk_coeff[k].as<Fr>(), P->lk_ext[k].as<Fr>(), P->gpow.as<Fr>());
    LookupQuotientArgs lq;
    lq.A = q.A; lq.B = q.B; lq.C = q.C; lq.QK = P->lk_qk_ext.as<Fr>(); lq.L0 = q.L0;
    lq.QT = P->lk_tagged ? P->lk_qt_ext.as<Fr>() : nullptr;
    lq.T = P->lk_ext[Prover::LK_T].as<Fr>(); lq.F = P->lk_ext[Prover::LK_F].as<Fr>();
    lq.H1 = P->lk_ext[Prover::LK_H1].as<Fr>(); lq.H2 = P->lk_ext[Prover::LK_H2].as<Fr>();
    lq.Z2 = P->lk_ext[Prover::LK_Z2].as<Fr>();
    for (int k = 0; k < 4; k++) lq.zh_inv[k] = P->zh_inv[k];
    lq.eta = P->eta; lq.eta2 = fp_sqr(P->eta); lq.eta3 = fp_mul(lq.eta2, P->eta); lq.delta = P->delta; lq.eps = P->epsilon;
    lq.one_d = fp_add(Fr::one(), P->delta); lq.eps_one_d = fp_mul(P->epsilon, lq.one_d);
    lq.alpha3 = fp_mul(q.alpha2, P->alpha); lq.alpha4 = fp_sqr(q.alpha2); lq.alpha5 = fp_mul(lq.alpha4, P->alpha);
    lq.one = Fr::one();
    lq.n4 = ne;
    ZkLookupCoset zl{};
    if (P->zk) {
      const Fr* b = P->zk_b;
      const Fr w = fr_root_of_unity(P->log_n), w2 = fp_sqr(w);
      const Fr e1 = fp_add(b[0], fp_add(fp_mul(lq.eta, b[2]), fp_mul(lq.eta2, b[4])));
      const Fr e0 = fp_add(b[1], fp_add(fp_mul(lq.eta, b[3]), fp_mul(lq.eta2, b[5])));
      const Fr per[18] = {e1,    e0,    b[11], b[12], b[13], b[14], b[15], fp_mul(b[13], w2), fp_mul(b[14], w),
                          b[15], b[16], b[17], b[18], b[19], b[20], fp_mul(b[18], w2), fp_mul(b[19], w), b[20]};
      zl.X = P->xs.as<Fr>();
      for (int k = 0; k < 4; k++)
        for (int i = 0; i < 18; i++) zl.w[k][i] = fp_mul(per[i], P->zh[k]);
      k_quotient_lookup<true><<<PB_GRID(ne, 128), 0, st>>>(lq, t_evals, zl);
    } else {
      k_quotient_lookup<false><<<PB_GRID(ne, 128), 0, st>>>(lq, t_evals, zl);
    }
    ctx->launches++;
  }
  if (P->sh) {  // one GPU: the slice is the whole 4n coset
    coset_extend(P, st, nullptr, P->sh_z3_coeff.as<Fr>(), P->sh_z3_ext.as<Fr>(), P->gpow.as<Fr>());
    ShuffleQuotientArgs sq;
    sq.A = q.A; sq.B = q.B; sq.C = q.C; sq.L0 = q.L0;
    sq.QIN = P->sh_ext[Prover::SH_IN].as<Fr>(); sq.QOUT = P->sh_ext[Prover::SH_OUT].as<Fr>();
    sq.Z3 = P->sh_z3_ext.as<Fr>();
    for (int k = 0; k < 4; k++) sq.zh_inv[k] = P->zh_inv[k];
    sq.theta = P->theta; sq.theta2 = fp_sqr(P->theta); sq.kappa_m1 = fp_sub(P->kappa, Fr::one());
    sq.alpha3 = fp_mul(q.alpha2, P->alpha); sq.alpha4 = fp_sqr(q.alpha2); sq.one = Fr::one();
    sq.n4 = ne;
    ZkShuffleCoset zs{};
    if (P->zk) {
      const Fr *b = P->zk_b, *c = P->zk_z3_b();
      const Fr w = fr_root_of_unity(P->log_n), w2 = fp_sqr(w);
      auto wsum = [&](const Fr& x, const Fr& y, const Fr& z) {  // x + theta y + theta^2 z
        return fp_add(x, fp_add(fp_mul(sq.theta, y), fp_mul(sq.theta2, z)));
      };
      const Fr e2 = P->next_row ? wsum(b[11], b[12], b[13]) : Fr::zero();
      const Fr per[9] = {e2,   wsum(b[0], b[2], b[4]), wsum(b[1], b[3], b[5]), c[0], c[1], c[2],
                         fp_mul(c[0], w2), fp_mul(c[1], w), c[2]};
      zs.X = P->xs.as<Fr>();
      for (int k = 0; k < 4; k++)
        for (int i = 0; i < 9; i++) zs.w[k][i] = fp_mul(per[i], P->zh[k]);
      k_quotient_shuffle<true><<<PB_GRID(ne, 128), 0, st>>>(sq, t_evals, zs);
    } else {
      k_quotient_shuffle<false><<<PB_GRID(ne, 128), 0, st>>>(sq, t_evals, zs);
    }
    ctx->launches++;
  }
  PB_CUDA(cudaMemsetAsync(P->flags.p, 0, 64, st));
  if (P->world > 1) {
    // slab-sharded inverse over the 4n coset: the local inverse transform of the slice, ONE allgather, then the
    // join multiplies g^-i in and keeps the 3n coefficients (the top n must vanish: prover.py:205-208)
    const Fr* te = t_evals;
    ntt_shard_local(ctx, &te, 1, P->log_n + 2, true, 1, 0, P->log_world, P->rank, ctx_comm(ctx));
    ntt_shard_combine(ctx, ctx->gather.as<Fr>(), ne, P->tq.as<Fr>(), P->log_n + 2, true, 3 * n,
                      P->ginv_pow.as<Fr>(), P->flags.as<uint32_t>(), P->log_world, P->rank);
  } else {
    // back to coefficients: ifft(4n) then * g^-i (poly.py:169-177 with the fixed coset)
    ntt_run(ctx, P->tq.as<Fr>(), P->tq.as<Fr>(), P->log_n + 2, true, n4, nullptr, P->ginv_pow.as<Fr>());
    const uint64_t top = P->zk ? P->zk_t3_len() + 2 * n : 3 * n;  // zero knowledge: deg T <= 3n + 5 (3n + 8)
    k_count_nonzero<<<PB_GRID(n4 - top, 256), 0, st>>>(P->tq.as<Fr>() + top, n4 - top, P->flags.as<uint32_t>());
    ctx->launches++;
  }
  if (P->zk) {
    PB_CHECK(read_flag(P, 0) == 0, P->next_row
                 ? "AssertionError: quotient has degree >= 3n + 9 (zero-knowledge mode, next-row terms; prover.py:205-208)"
                 : "AssertionError: quotient has degree >= 3n + 6 (zero-knowledge mode; prover.py:205-208)");
    // the pieces overlap in tq once blinded (T1' reaches X^n), so each gets its own buffer; one commitment pass
    const Fr* t = P->tq.as<Fr>();
    const Fr b10 = P->zk_b[9], b11 = P->zk_b[10], zero = Fr::zero();
    zk_blind(P, t, n, ZkPatch{{zero, zero, zero}, {b10, zero, zero}}, P->zk_t[0].as<Fr>());
    zk_blind(P, t + n, n, ZkPatch{{fp_neg(b10), zero, zero}, {b11, zero, zero}}, P->zk_t[1].as<Fr>());
    const uint64_t t3 = P->zk_t3_len();
    zk_blind(P, t + 2 * n, t3, ZkPatch{{fp_neg(b11), zero, zero}, {zero, zero, zero}}, P->zk_t[2].as<Fr>());
    const Fr* t123[3] = {P->zk_t[0].as<Fr>(), P->zk_t[1].as<Fr>(), P->zk_t[2].as<Fr>()};
    P->commit_batch(t123, 3, t3, P->fields[F_T_LO]);
    return;
  }
  PB_CHECK(read_flag(P, 0) == 0, "AssertionError: quotient has degree >= 3n (prover.py:205-208)");
  const Fr* t123[3] = {P->tq.as<Fr>(), P->tq.as<Fr>() + n, P->tq.as<Fr>() + 2 * n};
  P->commit_batch(t123, 3, n, P->fields[F_T_LO]);
}

// ---- round 4 (prover.py:228-239) -------------------------------------------------------------------------
void prover_round4(Prover* P, const Fr& zeta_c) {
  P->zeta = fp_to_mont(zeta_c);
  Fr zw = fp_mul(P->zeta, fr_root_of_unity(P->log_n));
  const Fr* polys[7] = {P->coeff[0].as<Fr>(), P->coeff[1].as<Fr>(), P->coeff[2].as<Fr>(),
                        P->sel_coeff[Prover::S1].as<Fr>(), P->sel_coeff[Prover::S2].as<Fr>(),
                        P->coeff[3].as<Fr>(), P->coeff[4].as<Fr>()};
  Fr xs[7] = {P->zeta, P->zeta, P->zeta, P->zeta, P->zeta, zw, P->zeta};
  Fr out[7];
  eval_polys(P, P->pi_sparse ? 6 : 7, polys, xs, out);
  if (P->next_row) {  // A, B, C at zeta w, and the third blinder of zero-knowledge mode on all six wire evaluations
    const Fr* abc[3] = {P->coeff[0].as<Fr>(), P->coeff[1].as<Fr>(), P->coeff[2].as<Fr>()};
    const Fr zws[3] = {zw, zw, zw};
    eval_polys(P, 3, abc, zws, P->nr_ev);
    if (P->zk) {
      // A'(x) = A(x) + (b12 x^2 + b1 x + b2) Z_H(x) at x = zeta and x = zeta w, with Z_H(zeta w) = Z_H(zeta)
      const Fr* b = P->zk_b;
      const Fr zh = fp_sub(fp_pow_u64(P->zeta, P->n), Fr::one());
      auto blind = [&](int k, const Fr& x) {
        return fp_mul(fp_add(fp_mul(fp_add(fp_mul(b[11 + k], x), b[2 * k]), x), b[2 * k + 1]), zh);
      };
      for (int k = 0; k < 3; k++) {
        out[k] = fp_add(out[k], blind(k, P->zeta));
        P->nr_ev[k] = fp_add(P->nr_ev[k], blind(k, zw));
      }
      out[5] = fp_add(out[5], fp_mul(fp_add(fp_mul(fp_add(fp_mul(b[6], zw), b[7]), zw), b[8]), zh));
    }
    for (int k = 0; k < 3; k++) store_canonical(P->fields[F_A_SHIFTED_EVAL + k], P->nr_ev[k]);
  } else if (P->zk) {
    // the blinded polynomials at their points: A'(zeta) = A(zeta) + (b1 zeta + b2)(zeta^n - 1), ...,
    // Z'(zeta w) = Z(zeta w) + (b7 (zeta w)^2 + b8 zeta w + b9)(zeta^n - 1)
    const Fr* b = P->zk_b;
    const Fr zh = fp_sub(fp_pow_u64(P->zeta, P->n), Fr::one());
    for (int k = 0; k < 3; k++) out[k] = fp_add(out[k], fp_mul(fp_add(fp_mul(b[2 * k], P->zeta), b[2 * k + 1]), zh));
    out[5] = fp_add(out[5], fp_mul(fp_add(fp_mul(fp_add(fp_mul(b[6], zw), b[7]), zw), b[8]), zh));
  }
  for (int k = 0; k < 6; k++) { P->ev[k] = out[k]; store_canonical(P->fields[F_A_EVAL + k], out[k]); }
  if (P->pi_sparse) {
    // PI(zeta) = sum_i (-pub_i) w^i (zeta^n - 1) / (n (zeta - w^i)), one shared inversion (host arithmetic)
    const uint64_t n = P->n;
    Fr w = fr_root_of_unity(P->log_n), wi = Fr::one(), one = Fr::one();
    Fr zh = fp_sub(fp_pow_u64(P->zeta, n), one), nm = fr_from_u64(n);
    std::vector<Fr> den(P->n_public), pref(P->n_public), wis(P->n_public);
    Fr run = one;
    for (uint64_t i = 0; i < P->n_public; i++) {
      den[i] = fp_mul(nm, fp_sub(P->zeta, wi));
      wis[i] = wi;
      pref[i] = run;
      run = fp_mul(run, den[i]);
      wi = fp_mul(wi, w);
    }
    Fr inv = fp_inv(run), acc = Fr::zero();
    for (uint64_t i = P->n_public; i-- > 0;) {
      Fr di = fp_mul(inv, pref[i]);
      inv = fp_mul(inv, den[i]);
      acc = fp_add(acc, fp_mul(fp_mul(P->pub_neg[i], wis[i]), di));
    }
    P->pi_ev = fp_mul(acc, zh);
  } else {
    P->pi_ev = out[6];
  }
  if (P->lk) {  // the lookup evaluations: F, T at zeta, T at zeta w, H2 at zeta, H1 and Z2 at zeta w
    const Fr* lpolys[6] = {P->lk_coeff[Prover::LK_F].as<Fr>(), P->lk_coeff[Prover::LK_T].as<Fr>(),
                           P->lk_coeff[Prover::LK_T].as<Fr>(), P->lk_coeff[Prover::LK_H2].as<Fr>(),
                           P->lk_coeff[Prover::LK_H1].as<Fr>(), P->lk_coeff[Prover::LK_Z2].as<Fr>()};
    const Fr lxs[6] = {P->zeta, P->zeta, zw, P->zeta, zw, zw};
    eval_polys(P, 6, lpolys, lxs, P->lk_ev);
    if (P->zk) {  // F', H2' at zeta and H1', Z2' at zeta w, with Z_H(zeta w) = Z_H(zeta); T is not blinded
      const Fr* b = P->zk_b;
      const Fr zh = fp_sub(fp_pow_u64(P->zeta, P->n), Fr::one());
      Fr* e = P->lk_ev;
      e[0] = fp_add(e[0], fp_mul(fp_add(fp_mul(b[11], P->zeta), b[12]), zh));
      e[3] = fp_add(e[3], fp_mul(fp_add(fp_mul(b[16], P->zeta), b[17]), zh));
      e[4] = fp_add(e[4], fp_mul(fp_add(fp_mul(fp_add(fp_mul(b[13], zw), b[14]), zw), b[15]), zh));
      e[5] = fp_add(e[5], fp_mul(fp_add(fp_mul(fp_add(fp_mul(b[18], zw), b[19]), zw), b[20]), zh));
    }
    for (int k = 0; k < 6; k++) store_canonical(P->fields[F_F_EVAL + k], P->lk_ev[k]);
  }
  if (P->sh) {  // Q_in at zeta, Z3 at zeta w
    const Fr* spolys[2] = {P->sh_coeff[Prover::SH_IN].as<Fr>(), P->sh_z3_coeff.as<Fr>()};
    const Fr sxs[2] = {P->zeta, zw};
    eval_polys(P, 2, spolys, sxs, P->sh_ev);
    if (P->zk) {  // Z3'(zeta w) = Z3(zeta w) + (c2 (zeta w)^2 + c1 zeta w + c0)(zeta^n - 1); Q_in is not blinded
      const Fr* c = P->zk_z3_b();
      const Fr zh = fp_sub(fp_pow_u64(P->zeta, P->n), Fr::one());
      P->sh_ev[1] = fp_add(P->sh_ev[1], fp_mul(fp_add(fp_mul(fp_add(fp_mul(c[0], zw), c[1]), zw), c[2]), zh));
    }
    for (int k = 0; k < 2; k++) store_canonical(P->fields[F_QIN_EVAL + k], P->sh_ev[k]);
  }
}

// (num coefficients, n) / (X - point) -> quotient coefficients (out != num), remainder dropped.
// Coefficient-space synthetic division as a weighted suffix sum (see k_sufsum_*).  One proof across G ranks: rank r
// divides the slab of coefficients [r n/G, (r+1) n/G) -- `num` needs to be valid on that slab only --; the slab sums
// are exchanged with a 32-byte allgather (the sums of the slabs above are the slab's carry), the quotient slabs with
// one bulk allgather, so every rank ends up with the full quotient for its share of the commitment.
// len: coefficients of num (P->n, or n + 8 for the blinded numerators of zero-knowledge mode, which runs on one device)
static void divide_linear(Prover* P, const Fr* num, Fr* out, const Fr& point, Fr* pow_buf, Fr* invpow_buf,
                          uint64_t len) {
  Context* ctx = P->ctx;
  const uint64_t n = len / (uint64_t)P->world, lo = n * (uint64_t)P->rank;
  cudaStream_t st = ctx->stream;
  const Fr point_inv = fp_inv(point);
  launch_powers(ctx, pow_buf + lo, n, point, fp_pow_u64(point, lo));
  launch_powers(ctx, invpow_buf + lo, n, point_inv, fp_pow_u64(point_inv, lo));
  uint32_t n_tiles = (uint32_t)((n + PB_FR_TILE - 1) / PB_FR_TILE);
  ctx->scratch[0].ensure((size_t)(n_tiles + 1 + 16) * 32);
  Fr* tiles = ctx->scratch[0].as<Fr>();
  Fr* totals = tiles + n_tiles + 1;  // [world] slab sums, then the carry
  k_sufsum_tiles<<<n_tiles, 256, 0, st>>>(num + lo, pow_buf + lo, n, tiles);
  k_fr_scan_tiles<ScanAdd><<<1, 256, 0, st>>>(tiles, n_tiles, tiles + n_tiles);
  if (P->world > 1) {
    PB_CUDA(cudaMemcpyAsync(totals + P->rank, tiles + n_tiles, 32, cudaMemcpyDeviceToDevice, st));
    comm_allgather_inplace(ctx_comm(ctx), totals, 32, st);
    Fr* carry = totals + P->world;
    k_sufsum_carry<<<1, 32, 0, st>>>(totals, (uint32_t)P->world, (uint32_t)P->rank, carry, P->flags.as<uint32_t>());
    k_sufsum_apply<<<n_tiles, 256, 0, st>>>(num + lo, pow_buf + lo, invpow_buf + lo, n, tiles, carry,
                                           fp_pow_u64(point_inv, lo + n), out + lo);
    comm_allgather_inplace(ctx_comm(ctx), out, n * 32, st);
    ctx->launches += 5;
    return;
  }
  k_sufsum_apply<<<n_tiles, 256, 0, st>>>(num, pow_buf, invpow_buf, n, tiles, nullptr, Fr::zero(), out);
  // the grand total is the remainder num(point); it must vanish (prover.py:267 R(zeta) == 0 and the degree
  // asserts of prover.py:288,299 are equivalent to exact divisibility)
  k_count_nonzero<<<1, 32, 0, st>>>(tiles + n_tiles, 1, P->flags.as<uint32_t>());
  ctx->launches += 4;
}

// ---- round 5 (prover.py:241-306) -------------------------------------------------------------------------
void prover_round5(Prover* P, const Fr& v_c) {
  Context* ctx = P->ctx;
  const uint64_t n = P->n;
  cudaStream_t st = ctx->stream;
  P->v = fp_to_mont(v_c);
  const Fr one = Fr::one();
  const Fr &a = P->ev[0], &b = P->ev[1], &c = P->ev[2], &s1 = P->ev[3], &s2 = P->ev[4], &zw = P->ev[5];
  const Fr &al = P->alpha, &be = P->beta, &ga = P->gamma, &zeta = P->zeta, &v = P->v;
  Fr zn = fp_pow_u64(zeta, n);
  Fr zh_ev = fp_sub(zn, one);                                                   // Z_H(zeta)
  Fr l0_ev = fp_mul(zh_ev, fp_inv(fp_mul(fr_from_u64(n), fp_sub(zeta, one))));   // L0(zeta)
  Fr bz = fp_mul(be, zeta);
  Fr c1 = fp_mul(fp_mul(fp_mul(fp_add(fp_add(a, bz), ga), fp_add(fp_add(b, fp_dbl(bz)), ga)),
                        fp_add(fp_add(c, fp_add(fp_dbl(bz), bz)), ga)), al);
  Fr c2 = fp_mul(fp_mul(fp_mul(fp_add(fp_add(a, fp_mul(be, s1)), ga), fp_add(fp_add(b, fp_mul(be, s2)), ga)), al), zw);
  Fr al2l0 = fp_mul(fp_sqr(al), l0_ev);
  Fr v2 = fp_sqr(v), v3 = fp_mul(v2, v), v4 = fp_sqr(v2), v5 = fp_mul(v4, v);
  // W_z numerator = R + v(A - a) + v^2(B - b) + v^3(C - c) + v^4(S1 - s1) + v^5(S2 - s2), R per SURVEY App. D
  // zero knowledge: Z, T1..T3, A, B, C are the blinded vectors (n + 8 coefficients, zero padded); coefficients [n, n + 8)
  // of the numerator come from those alone (tail)
  const bool zk = P->zk;
  const Fr* wire[3];
  for (int i = 0; i < 3; i++) wire[i] = zk ? P->zk_coeff[i].as<Fr>() : P->coeff[i].as<Fr>();
  const Fr* zpoly = zk ? P->zk_coeff[3].as<Fr>() : P->coeff[3].as<Fr>();
  const Fr* tpiece[3];
  for (int i = 0; i < 3; i++) tpiece[i] = zk ? P->zk_t[i].as<Fr>() : P->tq.as<Fr>() + (uint64_t)i * n;
  LinCombArgs L, tail;
  int k = 0;
  tail.count = 0;
  auto add = [&](const Fr* vec, const Fr& w, bool blinded = false) {
    L.vec[k] = vec; L.w[k] = w; k++;
    if (blinded) { tail.vec[tail.count] = vec; tail.w[tail.count] = w; tail.count++; }
  };
  add(P->sel_coeff[Prover::QL].as<Fr>(), a);
  add(P->sel_coeff[Prover::QR].as<Fr>(), b);
  add(P->sel_coeff[Prover::QM].as<Fr>(), fp_mul(a, b));
  add(P->sel_coeff[Prover::QO].as<Fr>(), c);
  add(P->sel_coeff[Prover::QC].as<Fr>(), one);
  const Fr *aw = P->nr_ev, *bw = P->nr_ev + 1, *cw = P->nr_ev + 2;  // next-row provers: the wires at zeta w
  for (int t = 0; t < P->n_custom; t++)  // m_t(a, b, c) Q_t, or m_t(a, b, c, a(zeta w), b(zeta w), c(zeta w)) Q_t
    add(P->sel_coeff[Prover::CUSTOM0 + t].as<Fr>(),
        P->next_row ? custom_monomial_next(a, b, c, *aw, *bw, *cw, P->custom_f[t]) : custom_monomial(a, b, c, P->custom_f[t]));
  add(zpoly, fp_add(c1, al2l0), true);                                 // Z
  add(P->sel_coeff[Prover::S3].as<Fr>(), fp_neg(fp_mul(c2, be)));
  add(tpiece[0], fp_neg(zh_ev), true);                                 // T1
  add(tpiece[1], fp_neg(fp_mul(zh_ev, zn)), true);                     // T2
  add(tpiece[2], fp_neg(fp_mul(zh_ev, fp_sqr(zn))), true);             // T3
  add(wire[0], v, true);
  add(wire[1], v2, true);
  add(wire[2], v3, true);
  add(P->sel_coeff[Prover::S1].as<Fr>(), v4);
  add(P->sel_coeff[Prover::S2].as<Fr>(), v5);
  // constant term: PI(zeta) - c2 (c + gamma) - alpha^2 L0(zeta) - v a - v^2 b - v^3 c - v^4 s1 - v^5 s2
  Fr c0 = fp_sub(P->pi_ev, fp_mul(c2, fp_add(c, ga)));
  c0 = fp_sub(c0, al2l0);
  c0 = fp_sub(c0, fp_mul(v, a));
  c0 = fp_sub(c0, fp_mul(v2, b));
  c0 = fp_sub(c0, fp_mul(v3, c));
  c0 = fp_sub(c0, fp_mul(v4, s1));
  c0 = fp_sub(c0, fp_mul(v5, s2));
  // lookups: q_K, Z2 and H1 keep their commitments in the linearisation; F, T, H2 join the batch at zeta
  if (P->lk) {
    const Fr &fe = P->lk_ev[0], &te = P->lk_ev[1], &tw = P->lk_ev[2], &h2e = P->lk_ev[3], &h1w = P->lk_ev[4],
             &z2w = P->lk_ev[5];
    const Fr &eta = P->eta, &de = P->delta, &ep = P->epsilon;
    const Fr od = fp_add(one, de), eod = fp_mul(ep, od);
    const Fr al2 = fp_sqr(al), al3 = fp_mul(al2, al), al4 = fp_sqr(al2), al5 = fp_mul(al4, al);
    const Fr v6 = fp_mul(v5, v), v7 = fp_mul(v6, v), v8 = fp_mul(v7, v);
    const Fr abc = fp_add(a, fp_add(fp_mul(eta, b), fp_mul(fp_sqr(eta), c)));
    const Fr hw = fp_add(fp_add(eod, h2e), fp_mul(de, h1w));       // e(1+d) + h2 + d h1(zeta w)
    const Fr az2 = fp_mul(al4, z2w);
    // zero knowledge: Z2', H1', F', H2' (n + 3 or n + 2 coefficients) join the tail; T stays unblinded
    add(P->lk_qk_coeff.as<Fr>(), fp_mul(al3, fp_sub(abc, fe)));
    if (P->lk_tagged) add(P->lk_qt_coeff.as<Fr>(), fp_mul(al3, fp_mul(fp_sqr(eta), eta)));  // alpha^3 eta^3 Q_T
    add(P->lk_poly(Prover::LK_Z2),
        fp_add(fp_mul(fp_mul(fp_mul(al4, od), fp_add(ep, fe)), fp_add(fp_add(eod, te), fp_mul(de, tw))),
               fp_mul(al5, l0_ev)), true);
    add(P->lk_poly(Prover::LK_H1), fp_neg(fp_mul(az2, hw)), true);
    add(P->lk_poly(Prover::LK_F), v6, true);
    add(P->lk_poly(Prover::LK_T), v7);
    add(P->lk_poly(Prover::LK_H2), v8, true);
    // -a4 z2w (e(1+d) + d h2) hw - a5 L0(zeta) - v^6 f - v^7 t - v^8 h2
    Fr lc = fp_neg(fp_mul(fp_mul(az2, fp_add(eod, fp_mul(de, h2e))), hw));
    lc = fp_sub(lc, fp_mul(al5, l0_ev));
    c0 = fp_add(c0, fp_sub(lc, fp_add(fp_mul(v6, fe), fp_add(fp_mul(v7, te), fp_mul(v8, h2e)))));
  }
  // shuffle: [Q_out] and [Z3] keep their commitments in the linearisation; Q_in joins the batch at zeta.  Zero knowledge:
  // Z3' (n + 3 coefficients) joins the tail; Q_out and Q_in stay unblinded
  if (P->sh) {
    const Fr &qin = P->sh_ev[0], &z3w = P->sh_ev[1];
    const Fr al2 = fp_sqr(al), al3 = fp_mul(al2, al), al4 = fp_sqr(al2), v6 = fp_mul(v5, v);
    const Fr th = P->theta;
    const Fr km1 = fp_add(fp_sub(P->kappa, one), fp_add(a, fp_add(fp_mul(th, b), fp_mul(fp_sqr(th), c))));  // k + w - 1
    const Fr a3z = fp_mul(al3, z3w), a4l0 = fp_mul(al4, l0_ev);
    add(P->sh_coeff[Prover::SH_OUT].as<Fr>(), fp_mul(a3z, km1));                                    // a3 z3w (k + w - 1)
    add(P->sh_z3_poly(), fp_sub(a4l0, fp_mul(al3, fp_add(one, fp_mul(qin, km1)))), true);  // -a3 (1 + q_in(..)) + a4 L0
    add(P->sh_coeff[Prover::SH_IN].as<Fr>(), v6);
    // a3 z3w - a4 L0(zeta) - v^6 q_in(zeta)
    c0 = fp_add(c0, fp_sub(a3z, fp_add(a4l0, fp_mul(v6, qin))));
  }
  L.count = k;
  L.n = n / (uint64_t)P->world;          // one proof across G ranks: every rank builds (and divides) its slab only
  L.first = L.n * (uint64_t)P->rank;
  L.c0 = c0;
  Fr* wz = P->tmp[0].as<Fr>();
  PB_CUDA(cudaMemsetAsync(P->flags.p, 0, 64, st));
  k_lincomb<<<PB_GRID(L.n, 128), 0, st>>>(L, wz);
  ctx->launches++;
  const uint64_t len = zk ? n + P->zk_pad() : n;  // numerator coefficients
  if (zk) {
    tail.c0 = Fr::zero();
    tail.n = P->zk_pad();
    tail.first = n;
    k_lincomb<<<PB_GRID(tail.n, 128), 0, st>>>(tail, wz);
    ctx->launches++;
  }
  Fr* wz_q = P->tmp[1].as<Fr>();
  divide_linear(P, wz, wz_q, zeta, P->tmp[2].as<Fr>(), P->tmp[3].as<Fr>(), len);
  // W_zw numerator = Z - z_shifted_eval
  LinCombArgs M;
  M.vec[0] = zpoly; M.w[0] = one; M.count = 1; M.c0 = fp_neg(zw);
  M.n = zk ? len : L.n; M.first = L.first;
  if (P->lk) {  // + v (T - t(zeta w)) + v^2 (H1 - h1(zeta w)) + v^3 (Z2 - z2(zeta w)); zero knowledge: T zero padded
    M.vec[1] = P->lk_poly(Prover::LK_T); M.w[1] = v;
    M.vec[2] = P->lk_poly(Prover::LK_H1); M.w[2] = v2;
    M.vec[3] = P->lk_poly(Prover::LK_Z2); M.w[3] = v3;
    M.count = 4;
    M.c0 = fp_sub(M.c0, fp_add(fp_mul(v, P->lk_ev[2]), fp_add(fp_mul(v2, P->lk_ev[4]), fp_mul(v3, P->lk_ev[5]))));
  }
  if (P->next_row) {  // + v (A - a(zeta w)) + v^2 (B - b(zeta w)) + v^3 (C - c(zeta w)); zero knowledge: A', B', C'
    M.vec[1] = wire[0]; M.w[1] = v;
    M.vec[2] = wire[1]; M.w[2] = v2;
    M.vec[3] = wire[2]; M.w[3] = v3;
    M.count = 4;
    M.c0 = fp_sub(M.c0, fp_add(fp_mul(v, *aw), fp_add(fp_mul(v2, *bw), fp_mul(v3, *cw))));
  }
  if (P->sh) {  // + v^k (Z3 - z3(zeta w)): k = 1, or 4 after A, B, C on a next-row prover; zero knowledge: Z3', padded
    const Fr vk = P->next_row ? v4 : v;
    M.vec[M.count] = P->sh_z3_poly(); M.w[M.count] = vk; M.count++;
    M.c0 = fp_sub(M.c0, fp_mul(vk, P->sh_ev[1]));
  }
  Fr* wzw = P->tmp[0].as<Fr>();  // the W_z numerator is no longer needed
  k_lincomb<<<PB_GRID(M.n, 128), 0, st>>>(M, wzw);
  ctx->launches++;
  Fr* wzw_q = P->tmp[4].as<Fr>();
  divide_linear(P, wzw, wzw_q, fp_mul(zeta, fr_root_of_unity(P->log_n)), P->tmp[2].as<Fr>(), P->tmp[3].as<Fr>(), len);
  PB_CHECK(read_flag(P, 0) == 0,
           "AssertionError: opening numerator is not divisible by (X - point) (prover.py:267,288,299)");
  const Fr* ws[2] = {wz_q, wzw_q};
  // zero knowledge: W_z has n + 5 coefficients (numerator n + 6; next-row n + 8 and n + 9), W_zw n + 2; the rest of
  // the buffers is zero
  P->commit_batch(ws, 2, zk ? P->zk_t3_len() - 1 : n, P->fields[F_W_Z]);
}

// The canonical proof: the fields of the prover's blocks in table order (proof_layout.cuh), a G1 point as x||y, every
// integer 32-byte big-endian exactly as the transcript absorbs it (transcript.py); layout_bytes(P->blocks()) bytes
void prover_serialize(const Prover* P, uint8_t* out) {
  const unsigned blocks = P->blocks();
  for (int f = 0; f < PROOF_FIELDS; f++) {
    if (!block_present(PROOF_LAYOUT[f].block, blocks)) continue;
    for (int w = 0; w < (PROOF_LAYOUT[f].is_point ? 2 : 1); w++, out += 32)
      for (int i = 0; i < 32; i++) out[i] = P->fields[f][32 * w + 31 - i];
  }
}

// step's fields of the prover's blocks, little-endian, in table order (what each round entry point returns)
size_t copy_step(const Prover* P, int step, uint8_t* out) {
  const unsigned blocks = P->blocks();
  size_t o = 0;
  for (int f = 0; f < PROOF_FIELDS; f++) {
    const ProofFieldInfo& info = PROOF_LAYOUT[f];
    if (info.step != step || !block_present(info.block, blocks)) continue;
    const size_t bytes = info.is_point ? 64 : 32;
    memcpy(out + o, P->fields[f], bytes);
    o += bytes;
  }
  return o;
}

// prover.py:51-84: each step runs its round, absorbs its fields of the prover's blocks in table order and draws its
// challenges (step 1L only with lookups; u is the verifier's)
void prover_prove(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                  uint64_t n_public, uint8_t* out, bool wires_on_device) {
  PB_CUDA(cudaSetDevice(P->ctx->device));  // the calling host thread may not be the one that created the context
  const unsigned blocks = P->blocks();
  Transcript tr("plonk");  // prover.py:53
  Fr ch[PROOF_CHALLENGES] = {};  // canonical
  for (int step = 0; step < PROOF_STEPS; step++) {
    if (!layout_bytes(blocks, step)) continue;  // step 1L without lookups
    switch (step) {
      case STEP_1: prover_round1(P, hA, hB, hC, h_public, n_public, wires_on_device); break;
      case STEP_1L: prover_round_lookup(P, ch[CH_ETA]); break;
      case STEP_2: prover_round2(P, ch); break;
      case STEP_3: prover_round3(P, ch[CH_ALPHA], ch[CH_FFT_COFACTOR]); break;
      case STEP_4: prover_round4(P, ch[CH_ZETA]); break;
      case STEP_5: prover_round5(P, ch[CH_V]); prover_serialize(P, out); return;
    }
    for (int f = 0; f < PROOF_FIELDS; f++) {
      const ProofFieldInfo& info = PROOF_LAYOUT[f];
      if (info.step != step || !block_present(info.block, blocks)) continue;
      if (info.is_point) tr.append_point_le(info.label, P->fields[f]);
      else tr.append_scalar_le(info.label, P->fields[f]);
    }
    for (int c = 0; c < PROOF_CHALLENGES; c++)
      if (CHALLENGE_LAYOUT[c].step == step && block_present(CHALLENGE_LAYOUT[c].block, blocks))
        ch[c] = tr.get_and_append_challenge(CHALLENGE_LAYOUT[c].label);
  }
}

}  // namespace pb200
