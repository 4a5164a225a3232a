// Witness check without proving (pb200_prover_check): every gate, copy constraint, lookup row and shuffle row a
// witness fails on a one-GPU prover's own key, each category as an exact count and its lowest `limit` locations.
//
//   gate     rows i with A QL + B QR + A B QM + C QO + PI + QC + sum_k Q_k m_k != 0 (k_check_gate; next-row terms read
//            row i + 1 mod n, as k_gate_check<true> does).
//   copy     cells c = 3 row + col with v(c) != v(sigma(c)), sigma(c) the cell whose label omega^row' (col' + 1) is
//            S_col[row] (k_check_copy).
//   key      cells whose S entry is no label, or the label a lower cell's S entry already names: S is then not a
//            permutation and no witness closes Z.
//   lookup   rows with q_K = 1 whose (a, b, c[, Q_T]) is not a row of the table (k_check_lookup, over the sorted table
//            copy the prover holds).
//   shuffle  rows with q_in = 1 or q_out = 1 whose (a, b, c) occurs a different number of times among the q_in rows than
//            among the q_out rows (a row with both selectors counts on both sides).
//
// Every equality is decided on full field elements (Montgomery form, a bijection on canonical values).  Sorting uses
// 64-bit words of them, chosen so that the sort groups exactly: a label word that no two of the 3n labels share, and a
// shuffle fingerprint a + theta b + theta^2 c (theta from getrandom) drawn again until no two different tuples share
// its word.  So for S a permutation the report is empty iff Z_n = 1, up to the argument's own soundness error.
//
// sigma is built on the first check of a prover and cached in Prover::chk_sigma (3n uint32: the target cell,
// PB_SIGMA_DUP set when a lower cell names the same label, PB_SIGMA_NONE for a non-label).  Everything else is the
// call's own and freed before it returns; the prover's round state (lag, coeff, ext, fields, flags) is not touched.
#include <cerrno>
#include <sys/random.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"
#include "prover.cuh"

namespace pb200 {
// poly_ops.cu
void fr_to_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
// prover.cu
__global__ void k_count_noncanonical(const Fr* v, uint64_t n, uint32_t* bad);

#define PB_SIGMA_NONE 0xffffffffu
#define PB_SIGMA_DUP 0x80000000u

// 64-bit word w (0..3) of a value: limbs 2w and 2w + 1 (selected by value, so x stays in registers)
__device__ __forceinline__ uint64_t chk_word(const Fr& x, int w) {
  const uint32_t lo = w == 0 ? x.v[0] : w == 1 ? x.v[2] : w == 2 ? x.v[4] : x.v[6];
  const uint32_t hi = w == 0 ? x.v[1] : w == 1 ? x.v[3] : w == 2 ? x.v[5] : x.v[7];
  return (uint64_t)lo | ((uint64_t)hi << 32);
}
// label of cell c = 3 row + col: omega^row (col + 1), Montgomery (roots: omega^i Montgomery)
__device__ __forceinline__ Fr chk_label(const Fr* roots, uint32_t c) {
  const uint32_t row = c / 3, col = c - 3 * row;
  const Fr w = ldg_fr(roots + row);
  Fr x = w;
  if (col >= 1) x = fp_add(x, w);
  if (col == 2) x = fp_add(x, w);
  return x;
}
// S entry of cell c (S: the three n-value columns)
struct SCols { const Fr* s[3]; };
__device__ __forceinline__ Fr chk_s(const SCols& S, uint64_t n, uint32_t c) {
  const uint32_t row = c / 3, col = c - 3 * row;
  return ldg_fr((col == 0 ? S.s[0] : col == 1 ? S.s[1] : S.s[2]) + row);  // static indices: no local copy
}
// value of cell c in the column-major wire copy W = A | B | C
__device__ __forceinline__ Fr chk_v(const Fr* W, uint64_t n, uint32_t c) {
  const uint32_t row = c / 3, col = c - 3 * row;
  return ldg_fr(W + col * n + row);
}

// ---- sigma ---------------------------------------------------------------------------------------------------------
__global__ void k_check_label_keys(const Fr* roots, uint64_t m, int w, uint64_t* keys, uint32_t* cells) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  keys[c] = chk_word(chk_label(roots, (uint32_t)c), w);
  cells[c] = (uint32_t)c;
}
__global__ void k_check_s_keys(SCols S, uint64_t n, uint64_t m, int w, uint64_t* keys, uint32_t* cells) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  keys[c] = chk_word(chk_s(S, n, (uint32_t)c), w);
  cells[c] = (uint32_t)c;
}
// counts sorted positions whose key equals the previous one
__global__ void k_check_adjacent(const uint64_t* keys, uint64_t m, uint32_t* equal) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k > 0 && k < m && keys[k] == keys[k - 1]) atomicAdd(equal, 1u);
}
// sorted S position k: its cell's label cell by binary search over the sorted label words (collision-free, so at most
// one candidate), confirmed on the full value; first[label cell] gets the lowest cell naming it
__global__ void __launch_bounds__(128) k_check_sigma(const uint64_t* s_keys, const uint32_t* s_cells,
                                                     const uint64_t* l_keys, const uint32_t* l_cells, uint64_t m, SCols S,
                                                     const Fr* roots, uint64_t n, uint32_t* sigma, uint32_t* first) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const uint64_t key = s_keys[k];
  const uint32_t c = s_cells[k];
  uint64_t lo = 0, hi = m;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) / 2;
    if (l_keys[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  uint32_t t = PB_SIGMA_NONE;
  if (lo < m && l_keys[lo] == key) {
    const uint32_t lc = l_cells[lo];
    if (chk_s(S, n, c) == chk_label(roots, lc)) {
      t = lc;
      atomicMin(first + lc, c);
    }
  }
  sigma[c] = t;
}
__global__ void k_check_sigma_dups(uint32_t* sigma, const uint32_t* first, uint64_t m) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  const uint32_t t = sigma[c];
  if (t != PB_SIGMA_NONE && first[t] != (uint32_t)c) sigma[c] = t | PB_SIGMA_DUP;
}

// ---- per-call kernels ----------------------------------------------------------------------------------------------
// one flag per row: the gate residual is not zero.  pub: -public_i (Montgomery), i < n_public
template <bool NEXT>
__global__ void __launch_bounds__(128) k_check_gate(const Fr* W, const Fr* QL, const Fr* QR, const Fr* QM, const Fr* QO,
                                                    const Fr* QC, const Fr* pub, uint64_t n_public, CustomTerms ct,
                                                    uint64_t n, uint8_t* flag) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr *A = W, *B = W + n, *C = W + 2 * n;
  const Fr a = ldg_fr(A + i), b = ldg_fr(B + i), c = ldg_fr(C + i);
  Fr s = fp_mul(a, ldg_fr(QL + i));
  s = fp_add(s, fp_mul(b, ldg_fr(QR + i)));
  s = fp_add(s, fp_mul(fp_mul(a, b), ldg_fr(QM + i)));
  s = fp_add(s, fp_mul(c, ldg_fr(QO + i)));
  s = fp_add(s, ldg_fr(QC + i));
  if (i < n_public) s = fp_add(s, ldg_fr(pub + i));
  if constexpr (NEXT) {
    const uint64_t i1 = i + 1 == n ? 0 : i + 1;
    s = custom_gate_sum_next(ct, i, a, b, c, ldg_fr(A + i1), ldg_fr(B + i1), ldg_fr(C + i1), s);
  } else {
    s = custom_gate_sum(ct, i, a, b, c, s);
  }
  flag[i] = s.is_zero() ? 0 : 1;
}

// per cell: copy flag (sigma(c) defined and v(c) != v(sigma(c))) and key flag (no label, or a repeated one)
__global__ void k_check_copy(const Fr* W, const uint32_t* sigma, uint64_t n, uint64_t m, uint8_t* copy, uint8_t* key) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  const uint32_t t = sigma[c];
  key[c] = (t == PB_SIGMA_NONE || (t & PB_SIGMA_DUP)) ? 1 : 0;
  copy[c] = (t != PB_SIGMA_NONE && chk_v(W, n, (uint32_t)c) != chk_v(W, n, t & ~PB_SIGMA_DUP)) ? 1 : 0;
}

// one flag per row: q_K = 1 and (a, b, c[, Q_T]) is not among the `rows` sorted table rows (width 3, or 4 with QT)
__global__ void __launch_bounds__(128) k_check_lookup(const Fr* W, const Fr* QK, const Fr* QT, const Fr* keys,
                                                      uint64_t rows, uint64_t n, uint8_t* flag) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (ldg_fr(QK + i).is_zero()) { flag[i] = 0; return; }
  const int width = QT ? 4 : 3;
  const Fr key[4] = {ldg_fr(W + i), ldg_fr(W + n + i), ldg_fr(W + 2 * n + i), QT ? ldg_fr(QT + i) : Fr::zero()};
  uint64_t lo = 0, hi = rows;  // the prover's sorted table copy, in lookup_cmp's order
  while (lo < hi) {
    const uint64_t mid = (lo + hi) / 2;
    if (lookup_cmp(keys + width * mid, key, width) < 0) lo = mid + 1;
    else hi = mid;
  }
  flag[i] = (lo < rows && lookup_cmp(keys + width * lo, key, width) == 0) ? 0 : 1;
}

// shuffle: sort key of each row, the low word of a + theta b + theta^2 c
__global__ void k_check_sh_keys(const Fr* W, Fr theta, Fr theta2, uint64_t n, uint64_t* keys, uint32_t* rows) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr f = fp_add(ldg_fr(W + i), fp_add(fp_mul(theta, ldg_fr(W + n + i)), fp_mul(theta2, ldg_fr(W + 2 * n + i))));
  keys[i] = chk_word(f, 0);
  rows[i] = (uint32_t)i;
}
// sorted position k: head[k] = 1 where a run of equal keys starts; *impure counts neighbours with equal keys and
// different tuples (then theta is drawn again)
__global__ void k_check_sh_heads(const uint64_t* keys, const uint32_t* rows, const Fr* W, uint64_t n, uint32_t* head,
                                 uint32_t* impure) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const bool start = k == 0 || keys[k] != keys[k - 1];
  head[k] = start ? 1 : 0;
  if (!start) {
    const uint32_t r = rows[k], p = rows[k - 1];
    if (ldg_fr(W + r) != ldg_fr(W + p) || ldg_fr(W + n + r) != ldg_fr(W + n + p) ||
        ldg_fr(W + 2 * n + r) != ldg_fr(W + 2 * n + p))
      atomicAdd(impure, 1u);
  }
}
// per run (run[k]: 1-based run index of sorted position k): q_in count in the low 32 bits, q_out count in the high 32.
// A run's positions are contiguous, so each warp sums the lanes of one run first: one atomic per run and warp.
__global__ void __launch_bounds__(256) k_check_sh_count(const uint32_t* run, const uint32_t* rows, const Fr* QIN,
                                                        const Fr* QOUT, uint64_t n, unsigned long long* cnt) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t id = 0xffffffffu, in = 0, out = 0;
  if (k < n) {
    const uint32_t r = rows[k];
    id = run[k] - 1;
    in = ldg_fr(QIN + r).is_zero() ? 0 : 1;
    out = ldg_fr(QOUT + r).is_zero() ? 0 : 1;
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, id);
  in = __reduce_add_sync(peers, in);
  out = __reduce_add_sync(peers, out);
  if (id != 0xffffffffu && (int)(threadIdx.x & 31) == __ffs(peers) - 1 && (in | out))
    atomicAdd(cnt + id, (unsigned long long)in | ((unsigned long long)out << 32));
}
// one flag per row: q_in or q_out set and its run's two counts differ
__global__ void k_check_sh_flag(const uint32_t* run, const uint32_t* rows, const unsigned long long* cnt, const Fr* QIN,
                                const Fr* QOUT, uint64_t n, uint8_t* flag) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t r = rows[k];
  const unsigned long long v = cnt[run[k] - 1];
  const bool on = !ldg_fr(QIN + r).is_zero() || !ldg_fr(QOUT + r).is_zero();
  flag[r] = (on && (uint32_t)v != (uint32_t)(v >> 32)) ? 1 : 0;
}
// the copy list's pairs: (c, sigma(c)) for the `count` lowest failing cells
__global__ void k_check_pairs(const uint32_t* cells, uint32_t count, const uint32_t* sigma, uint32_t* pairs) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const uint32_t c = cells[k];
  pairs[2 * k] = c;
  pairs[2 * k + 1] = sigma[c] & ~PB_SIGMA_DUP;
}

// ---- host ----------------------------------------------------------------------------------------------------------
// a field element from getrandom(2), canonical and not zero, in Montgomery form (the wire solver's table index draws
// its theta here too)
Fr check_random_fr() {
  for (;;) {
    Fr x;
    size_t got = 0;
    while (got < 32) {
      const ssize_t r = getrandom(reinterpret_cast<uint8_t*>(x.v) + got, 32 - got, 0);
      if (r < 0) {
        PB_CHECK(errno == EINTR, "witness check: getrandom() failed (no fallback source is used)");
        continue;
      }
      got += (size_t)r;
    }
    x.v[7] &= 0x3fffffffu;  // below 2^254: r > 2^253, so at most half the draws are rejected
    if (fp_is_canonical(x) && !x.is_zero()) return fp_to_mont(x);
  }
}

// cub's temporary storage of the check's three kinds of pass over m items (sizes only, no device work)
struct CheckTemp {
  size_t sort = 0, scan = 0, select = 0;
  CheckTemp(uint64_t m_sort, uint64_t m_select) {
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    if (m_sort) {
      PB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, sort, k, v, (int)m_sort));
      PB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, scan, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m_sort));
    }
    PB_CUDA(cub::DeviceSelect::Flagged(nullptr, select, thrust::counting_iterator<uint32_t>(0), (const uint8_t*)nullptr,
                                       (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m_select));
  }
};

// sigma from the 3n labels and the 3n S entries, each sorted by its 64-bit word; the word is the first of the four
// that no two labels share
static void build_sigma(Prover* P, DevBuf& temp) {
  Context* ctx = P->ctx;
  cudaStream_t st = ctx->stream;
  const uint64_t n = P->n, m = 3 * n;
  const SCols S{{P->sel_lag[Prover::S1].as<Fr>(), P->sel_lag[Prover::S2].as<Fr>(), P->sel_lag[Prover::S3].as<Fr>()}};
  DevBuf lk(m * 8), lk2(m * 8), lc(m * 4), lc2(m * 4), sk(m * 8), sk2(m * 8), sc(m * 4), sc2(m * 4), first(m * 4),
      equal(4);
  cub::DoubleBuffer<uint64_t> lkeys(lk.as<uint64_t>(), lk2.as<uint64_t>());
  cub::DoubleBuffer<uint32_t> lcells(lc.as<uint32_t>(), lc2.as<uint32_t>());
  int w = 0;
  for (;; w++) {
    PB_CHECK(w < 4, "witness check: every 64-bit word of the cell labels repeats among them");
    k_check_label_keys<<<PB_GRID(m, 256), 0, st>>>(P->roots.as<Fr>(), m, w, lk.as<uint64_t>(), lc.as<uint32_t>());
    launched(ctx);
    lkeys = cub::DoubleBuffer<uint64_t>(lk.as<uint64_t>(), lk2.as<uint64_t>());
    lcells = cub::DoubleBuffer<uint32_t>(lc.as<uint32_t>(), lc2.as<uint32_t>());
    size_t tb = temp.bytes;
    PB_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, lkeys, lcells, (int)m, 0, 64, st));
    launched(ctx);
    PB_CUDA(cudaMemsetAsync(equal.p, 0, 4, st));
    k_check_adjacent<<<PB_GRID(m, 256), 0, st>>>(lkeys.Current(), m, equal.as<uint32_t>());
    launched(ctx);
    uint32_t eq = 0;
    PB_CUDA(cudaMemcpyAsync(&eq, equal.p, 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    if (eq == 0) break;
  }
  k_check_s_keys<<<PB_GRID(m, 256), 0, st>>>(S, n, m, w, sk.as<uint64_t>(), sc.as<uint32_t>());
  launched(ctx);
  cub::DoubleBuffer<uint64_t> skeys(sk.as<uint64_t>(), sk2.as<uint64_t>());
  cub::DoubleBuffer<uint32_t> scells(sc.as<uint32_t>(), sc2.as<uint32_t>());
  size_t tb = temp.bytes;
  PB_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, skeys, scells, (int)m, 0, 64, st));
  launched(ctx);
  DevBuf sigma(m * 4);
  PB_CUDA(cudaMemsetAsync(first.p, 0xff, m * 4, st));
  k_check_sigma<<<PB_GRID(m, 128), 0, st>>>(skeys.Current(), scells.Current(), lkeys.Current(), lcells.Current(), m,
                                                  S, P->roots.as<Fr>(), n, sigma.as<uint32_t>(), first.as<uint32_t>());
  launched(ctx);
  k_check_sigma_dups<<<PB_GRID(m, 256), 0, st>>>(sigma.as<uint32_t>(), first.as<uint32_t>(), m);
  launched(ctx);
  PB_CUDA(cudaStreamSynchronize(st));  // the temporaries die here
  P->chk_sigma = std::move(sigma);
}

// flags[0, m) -> the number of flagged indices, and the lowest min(count, limit) of them at h_out (null: the count
// only).  d_idx: m words, d_num: one; temp: at least cub::DeviceSelect::Flagged's storage over m items.  The wire
// solver lists its errors with it too.
uint64_t compact_flagged(Context* ctx, const uint8_t* flags, uint64_t m, DevBuf& temp, uint32_t* d_idx,
                         uint32_t* d_num, uint32_t limit, uint32_t* h_out) {
  cudaStream_t st = ctx->stream;
  size_t tb = temp.bytes;
  PB_CUDA(cub::DeviceSelect::Flagged(temp.p, tb, thrust::counting_iterator<uint32_t>(0), flags, d_idx, d_num, (int)m,
                                     st));
  launched(ctx);
  uint32_t num = 0;
  PB_CUDA(cudaMemcpyAsync(&num, d_num, 4, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  const uint32_t take = num < limit ? num : limit;
  if (take && h_out) {
    PB_CUDA(cudaMemcpyAsync(h_out, d_idx, (size_t)take * 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
  }
  return num;
}

// h_counts[5]: gate, copy, key, lookup, shuffle.  h_lists (6 limit uint32): gate rows, copy pairs (c, sigma(c)), key
// cells, lookup rows, shuffle rows, each ascending, unused entries 0xffffffff.  wires_on_device: A, B, C are device
// pointers.  Every refusal before the first device work leaves the prover as it was; later ones free what the call made.
void prover_check(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                  uint64_t n_public, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists, bool wires_on_device) {
  Context* ctx = P->ctx;
  cudaStream_t st = ctx->stream;
  const uint64_t n = P->n, m = 3 * n;
  PB_CHECK(!P->sharded && P->world == 1, "the witness check is not available on the sharded prover (one GPU only)");
  PB_CHECK(hA && hB && hC && h_counts && (h_lists || limit == 0) && (h_public || n_public == 0),
           "the witness check needs A, B, C, the public inputs and its outputs");
  PB_CHECK(n_public <= n, "more public inputs than rows");
  PB_CHECK(limit <= m, "limit above 3n, the most entries a list can have");
  std::vector<Fr> pub(n_public);
  for (uint64_t i = 0; i < n_public; i++) {
    memcpy(pub[i].v, h_public + 32 * i, 32);
    PB_CHECK(fp_is_canonical(pub[i]), "public input not reduced below the field modulus");
    pub[i] = fp_neg(fp_to_mont(pub[i]));
  }
  // device memory, before any device work: sigma (kept) and its build's sort buffers on the first call, then the
  // call's wire copy, flags, index list and the shuffle's sort
  const bool build = P->chk_sigma.p == nullptr;
  const CheckTemp t(std::max(build ? m : 0, P->sh ? n : 0), m);
  const uint64_t temp_need = std::max(std::max(t.sort, t.scan), t.select);
  const uint64_t build_need = build ? m * (4 * 8 + 4 * 4 + 4 + 4) : 0;     // keys, cells, first, sigma
  const uint64_t call_need = m * (32 + 2 + 4) + 64 + n_public * 32 + 12 * (uint64_t)limit +
                             (P->sh ? n * (2 * 8 + 2 * 4 + 4 + 8) : 0);     // W, flags, idx, pairs, the shuffle's sort
  const uint64_t need = temp_need + std::max(build_need, (build ? m * 4 : 0) + call_need);
  size_t free_b = 0, total_b = 0;
  PB_CUDA(cudaMemGetInfo(&free_b, &total_b));
  // PB200_CHECK_MAX_BYTES: the most device memory a check may take (read per call), so it leaves room for other work
  // on the card; without it, whatever is free
  if (const char* e = getenv("PB200_CHECK_MAX_BYTES")) free_b = std::min<size_t>(free_b, strtoull(e, nullptr, 10));
  if (need > free_b) {
    char b[256];
    snprintf(b, sizeof b, "the witness check of 2^%d rows needs %llu bytes of device memory, %llu are free", P->log_n,
             (unsigned long long)need, (unsigned long long)free_b);
    throw Error(b);
  }
  if (ctx->aux_stream) {  // coset extensions of a round 1 may still read lag on the side stream: nothing here writes it,
    PB_CUDA(cudaEventRecord(ctx->aux_ev[2], ctx->aux_stream));  // but the wire copy below is ordered after them
    PB_CUDA(cudaStreamWaitEvent(st, ctx->aux_ev[2], 0));
  }
  DevBuf temp(temp_need);
  if (build) build_sigma(P, temp);

  DevBuf W(m * 32), flags(2 * m), idx(m * 4), small(64), pubd(n_public * 32);
  uint32_t* bad = small.as<uint32_t>();
  uint32_t* num = bad + 1;
  uint32_t* impure = bad + 2;
  PB_CUDA(cudaMemsetAsync(small.p, 0, 64, st));
  const uint8_t* src[3] = {hA, hB, hC};
  for (int k = 0; k < 3; k++) {
    Fr* w = W.as<Fr>() + k * n;
    PB_CUDA(cudaMemcpyAsync(w, src[k], n * 32, wires_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    k_count_noncanonical<<<PB_GRID(n, 256), 0, st>>>(w, n, bad);
    launched(ctx);
    fr_to_mont(ctx, w, w, n);
  }
  uint32_t nbad = 0;
  PB_CUDA(cudaMemcpyAsync(&nbad, bad, 4, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  PB_CHECK(nbad == 0, "wire value not reduced below the field modulus (canonical 32-byte little-endian expected)");
  if (n_public) PB_CUDA(cudaMemcpyAsync(pubd.p, pub.data(), n_public * 32, cudaMemcpyHostToDevice, st));

  for (uint64_t k = 0; k < 5; k++) h_counts[k] = 0;
  for (uint64_t k = 0; k < 6 * (uint64_t)limit; k++) h_lists[k] = 0xffffffffu;
  uint32_t *l_gate = h_lists, *l_copy = h_lists + limit, *l_key = h_lists + 3 * (uint64_t)limit,
           *l_lookup = h_lists + 4 * (uint64_t)limit, *l_shuffle = h_lists + 5 * (uint64_t)limit;
  uint8_t* f = flags.as<uint8_t>();
  const Fr* Wp = W.as<Fr>();
  // gates
  (P->next_row ? k_check_gate<true> : k_check_gate<false>)<<<PB_GRID(n, 128), 0, st>>>(
      Wp, P->sel_lag[Prover::QL].as<Fr>(), P->sel_lag[Prover::QR].as<Fr>(), P->sel_lag[Prover::QM].as<Fr>(),
      P->sel_lag[Prover::QO].as<Fr>(), P->sel_lag[Prover::QC].as<Fr>(), pubd.as<Fr>(), n_public,
      P->custom_terms(P->sel_lag), n, f);
  launched(ctx);
  h_counts[0] = compact_flagged(ctx, f, n, temp, idx.as<uint32_t>(), num, limit, l_gate);
  // copy constraints and the key
  k_check_copy<<<PB_GRID(m, 256), 0, st>>>(Wp, P->chk_sigma.as<uint32_t>(), n, m, f, f + m);
  launched(ctx);
  std::vector<uint32_t> cells(limit);
  h_counts[1] = compact_flagged(ctx, f, m, temp, idx.as<uint32_t>(), num, limit, cells.data());
  const uint32_t pairs = (uint32_t)std::min<uint64_t>(h_counts[1], limit);
  if (pairs) {  // (c, sigma(c)) of the listed cells
    DevBuf pb((size_t)pairs * 12);
    PB_CUDA(cudaMemcpyAsync(pb.p, cells.data(), (size_t)pairs * 4, cudaMemcpyHostToDevice, st));
    k_check_pairs<<<PB_GRID(pairs, 128), 0, st>>>(pb.as<uint32_t>(), pairs, P->chk_sigma.as<uint32_t>(),
                                                        pb.as<uint32_t>() + pairs);
    launched(ctx);
    PB_CUDA(cudaMemcpyAsync(l_copy, pb.as<uint32_t>() + pairs, (size_t)pairs * 8, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
  }
  h_counts[2] = compact_flagged(ctx, f + m, m, temp, idx.as<uint32_t>(), num, limit, l_key);
  // lookup rows
  if (P->lk) {
    k_check_lookup<<<PB_GRID(n, 128), 0, st>>>(Wp, P->lk_qk_lag.as<Fr>(),
                                                     P->lk_tagged ? P->lk_qt_lag.as<Fr>() : nullptr, P->lk_keys.as<Fr>(),
                                                     P->lk_rows, n, f);
    launched(ctx);
    h_counts[3] = compact_flagged(ctx, f, n, temp, idx.as<uint32_t>(), num, limit, l_lookup);
  }
  // shuffle rows: sort by the fingerprint's word, count both sides per run of equal words
  if (P->sh) {
    const Fr* QIN = P->sh_lag[Prover::SH_IN].as<Fr>();
    const Fr* QOUT = P->sh_lag[Prover::SH_OUT].as<Fr>();
    DevBuf k1(n * 8), k2(n * 8), r1(n * 4), r2(n * 4), run(n * 4), cnt(n * 8);
    cub::DoubleBuffer<uint64_t> keys(k1.as<uint64_t>(), k2.as<uint64_t>());
    cub::DoubleBuffer<uint32_t> rows(r1.as<uint32_t>(), r2.as<uint32_t>());
    for (int draw = 0;; draw++) {
      PB_CHECK(draw < 8, "witness check: eight shuffle fingerprints in a row had colliding words");
      const Fr theta = check_random_fr();
      k_check_sh_keys<<<PB_GRID(n, 128), 0, st>>>(Wp, theta, fp_sqr(theta), n, k1.as<uint64_t>(), r1.as<uint32_t>());
      launched(ctx);
      keys = cub::DoubleBuffer<uint64_t>(k1.as<uint64_t>(), k2.as<uint64_t>());
      rows = cub::DoubleBuffer<uint32_t>(r1.as<uint32_t>(), r2.as<uint32_t>());
      size_t tb = temp.bytes;
      PB_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, keys, rows, (int)n, 0, 64, st));
      launched(ctx);
      PB_CUDA(cudaMemsetAsync(impure, 0, 4, st));
      k_check_sh_heads<<<PB_GRID(n, 256), 0, st>>>(keys.Current(), rows.Current(), Wp, n, run.as<uint32_t>(),
                                                         impure);
      launched(ctx);
      uint32_t imp = 0;
      PB_CUDA(cudaMemcpyAsync(&imp, impure, 4, cudaMemcpyDeviceToHost, st));
      PB_CUDA(cudaStreamSynchronize(st));
      if (imp == 0) break;
    }
    size_t tb = temp.bytes;
    // run index of every sorted position: the inclusive sum of the heads, into the free half of the row buffers
    uint32_t* run_id = rows.Alternate();
    PB_CUDA(cub::DeviceScan::InclusiveSum(temp.p, tb, run.as<uint32_t>(), run_id, (int)n, st));
    launched(ctx);
    PB_CUDA(cudaMemsetAsync(cnt.p, 0, n * 8, st));
    k_check_sh_count<<<PB_GRID(n, 256), 0, st>>>(run_id, rows.Current(), QIN, QOUT, n,
                                                       cnt.as<unsigned long long>());
    launched(ctx);
    k_check_sh_flag<<<PB_GRID(n, 256), 0, st>>>(run_id, rows.Current(), cnt.as<unsigned long long>(), QIN, QOUT,
                                                      n, f);
    launched(ctx);
    h_counts[4] = compact_flagged(ctx, f, n, temp, idx.as<uint32_t>(), num, limit, l_shuffle);
  }
  PB_CUDA(cudaStreamSynchronize(st));  // the call's buffers die here
}

}  // namespace pb200
