// Wire values A, B, C of a circuit from the values of its input variables (pb200_solve_wires), the way the reference
// runs a program (compiler/program.py:161-192), on the GPU.  solve.cuh has the gate body; DESIGN.md section 3 the rule.
//
//   1. group:    the 3n cells' keys (id + 1) << cb | cell are sorted as permutation.cu sorts them (perm_sort_keys); each
//                run of one id is one variable, numbered densely by an inclusive sum of the run heads.
//   2. source:   a variable is the constant 0 (id -1), an input (binary search of the sorted input ids), or defined by
//                the lowest row whose O cell carries it and that may define (k_solve_qualify): runs are in cell order,
//                so an atomicMin over the run's qualifying O cells finds it.  Errors, per cell in cell order:
//                  unset  the variable is neither an input nor defined by any row;
//                  order  an L or R cell of a defining row whose variable that row or a later one defines.
//                Each kind is an exact count and its lowest `limit` cells (cub::DeviceSelect::Flagged, as check.cu).
//   3. divisor:  1 / QO of every row by one batched inversion (k_batch_div); the body negates it.
//   4. evaluate: k_solve_eval<false>, persistent: each warp takes the next 32 defining rows in row order through one global
//                ticket; a lane computes its row once the ready flags of its L and R variables are set (acquire), then
//                stores c and sets its O variable's flag (release).  A lane whose operand a lower lane of its warp
//                defines sees it on a later pass of the warp's loop.  Every wait is bounded: a warp that makes no
//                progress for PB_SOLVE_STALL_NS sets the stall flag, and every warp leaves on it.
//   5. write:    every cell gets its variable's value, canonical, in A | B | C.
// Device memory: about 430 bytes a row plus the outputs (DESIGN.md section 2), all freed before the call returns.
//
// With a table (pb200_solve_wires_lookup) a row with q_K != 0 and QO = 0 may also define its O variable, as t3 of the
// table row matching its (tag, a, b).  k_solve_qualify flags it 2 beside the gate rows' 1, so both kinds go through
// steps 2 and 4 as one ascending list.  Before step 4 the table index is built (solve_table_index: words of the keys
// sorted, checked on full values, one entry per distinct key); k_solve_eval<true> probes it (solve.cuh, solve_probe)
// and flags miss and ambiguous rows, which still store 0 and release their flag.
//
// With a shuffle (pb200_solve_wires_shuffle) out-rows define nothing by the gate rule (k_solve_qualify); their
// variables are defined at the first out-row p (k_solve_claim_out), late and clash cells are flagged in step 2, and
// step 4 runs in two phases, the defining rows below p and the rest, with the sorted in-row tuples written into the
// out-rows between them (solve_shuffle).  DESIGN.md section 3 has the rule and the no-deadlock argument per phase.
#include <algorithm>
#include <cuda/atomic>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"
#include "permutation.cuh"
#include "solve.cuh"

namespace pb200 {
// poly_ops.cu
void fr_to_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
void fr_from_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
// prover.cu
__global__ void k_batch_div(const Fr* num, const Fr* den, Fr* out, uint64_t n, uint64_t T);
__global__ void k_count_noncanonical(const Fr* v, uint64_t n, uint32_t* bad);
// check.cu
Fr check_random_fr();
uint64_t compact_flagged(Context* ctx, const uint8_t* flags, uint64_t m, DevBuf& temp, uint32_t* d_idx,
                         uint32_t* d_num, uint32_t limit, uint32_t* h_out);
// prover.cu
void lookup_require(uint64_t n, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* const* h_tab,
                    uint64_t rows);
void shuffle_require(uint64_t n, const uint8_t* h_qin, const uint8_t* h_qout);
// permutation.cu
void perm_require_ids(const int64_t* h_ids, uint64_t m, int64_t* max_id);
uint64_t* perm_sort_keys(Context* ctx, const int64_t* h_ids, uint64_t m, int cb, int end_bit, DevBuf& keys, DevBuf& alt,
                         DevBuf& temp, size_t temp_bytes, uint64_t m_ids);

#define PB_SOLVE_BATCH_CH 16              // k_batch_div's chain length (PB_BATCH_CH)
#define PB_SOLVE_STALL_NS 10000000000ull  // 10 s without progress of a warp: the evaluation has stalled

struct SolveSel {
  const Fr *ql, *qr, *qm, *qo, *qc, *inv_qo;  // Montgomery, n each
  const Fr* q[PB_MAX_CUSTOM];
  uint8_t f[PB_MAX_CUSTOM][3];
  int n_custom;
};

// side[r] of a shuffle: PB_SOLVE_IN for an in-row (q_in = 1, q_out = 0), PB_SOLVE_OUT for an out-row (q_out = 1,
// q_in = 0), else 0
#define PB_SOLVE_IN 1
#define PB_SOLVE_OUT 2

// one flag per row r < n_rows: 1 where it defines its O variable by the gate rule (QO != 0 and no term whose selector
// is non-zero at r reads c or the next row), else PB_SOLVE_BY_TABLE where it defines from its table (qk not null:
// q_K != 0 and QO = 0, qk canonical), else 0.  Out-rows of a shuffle (side not null) define nothing: 0.
#define PB_SOLVE_BY_TABLE 2
__global__ void k_solve_qualify(SolveSel s, const Fr* qk, const uint8_t* side, uint64_t n_rows, uint8_t* qual) {
  const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n_rows) return;
  const bool qo = !ldg_fr(s.qo + r).is_zero();
  bool ok = qo;
#pragma unroll
  for (int k = 0; k < PB_MAX_CUSTOM; k++)
    if (k < s.n_custom && solve_term_reads_c(s.f[k]) && !ldg_fr(s.q[k] + r).is_zero()) ok = false;
  const bool table = qk && !qo && !ldg_fr(qk + r).is_zero();
  qual[r] = (side && side[r] == PB_SOLVE_OUT) ? 0 : ok ? 1 : table ? PB_SOLVE_BY_TABLE : 0;
}

// ---- the table index (solve.cuh, SolveTable) -----------------------------------------------------------------------
// table row k: the word of its key (t4, t1, t2) and k
__global__ void k_solve_tab_keys(SolveTable T, uint64_t rows, uint64_t* keys, uint32_t* idx) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows) return;
  const Fr tag = T.t[3] ? ldg_fr(T.t[3] + k) : Fr::zero();
  keys[k] = solve_table_word(tag, ldg_fr(T.t[0] + k), ldg_fr(T.t[1] + k), T.theta, T.theta2);
  idx[k] = (uint32_t)k;
}
// sorted position k: head[k] = 1 where a run of equal words starts; *impure counts neighbours with equal words and
// different keys (then theta is drawn again); split[k] = 1 where k's t3 differs from its neighbour's in the same run
__global__ void k_solve_tab_heads(SolveTable T, const uint64_t* keys, const uint32_t* idx, uint64_t rows,
                                  uint32_t* head, uint8_t* split, uint32_t* impure) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows) return;
  const bool start = k == 0 || keys[k] != keys[k - 1];
  head[k] = start ? 1 : 0;
  bool differs = false;
  if (!start) {
    const uint32_t r = idx[k], p = idx[k - 1];
    if (ldg_fr(T.t[0] + r) != ldg_fr(T.t[0] + p) || ldg_fr(T.t[1] + r) != ldg_fr(T.t[1] + p) ||
        (T.t[3] && ldg_fr(T.t[3] + r) != ldg_fr(T.t[3] + p)))
      atomicAdd(impure, 1u);
    differs = ldg_fr(T.t[2] + r) != ldg_fr(T.t[2] + p);
  }
  split[k] = differs ? 1 : 0;
}
// per run u (run[k]: 1-based run of sorted position k): its word, its first table row, and amb[u] = 1 when two of its
// rows give different t3 (amb zeroed before)
__global__ void k_solve_tab_unique(const uint64_t* keys, const uint32_t* idx, const uint32_t* head,
                                   const uint32_t* run, const uint8_t* split, uint64_t rows, uint64_t* word,
                                   uint32_t* row, uint8_t* amb) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= rows) return;
  const uint32_t u = run[k] - 1;
  if (head[k]) {
    word[u] = keys[k];
    row[u] = idx[k];
  }
  if (split[k]) amb[u] = 1;
}

__global__ void k_solve_heads(const uint64_t* keys, uint64_t m, int cb, uint32_t* head) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) head[k] = (k == 0 || (keys[k] >> cb) != (keys[k - 1] >> cb)) ? 1 : 0;
}

// sorted position k: its cell's variable; at a run head the variable's input (binary search of the sorted input ids,
// PB_SOLVE_NONE without one, PB_SOLVE_ZERO for id -1); at a qualifying O cell of a variable without input, a candidate
// defining row
#define PB_SOLVE_ZERO 0xfffffffeu
__global__ void k_solve_vars(const uint64_t* keys, const uint32_t* run, uint64_t m, int cb, const uint64_t* in_ids,
                             uint64_t n_in, const uint8_t* qual, uint32_t* var_of_cell, uint32_t* inp,
                             uint32_t* def_row) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const uint64_t key = keys[k], g = key >> cb;
  const uint32_t cell = (uint32_t)(key & (((uint64_t)1 << cb) - 1)), var = run[k] - 1;
  var_of_cell[cell] = var;
  uint32_t src = PB_SOLVE_ZERO;
  if (g != 0) {
    uint64_t lo = 0, hi = n_in;  // in_ids: id + 1, ascending
    while (lo < hi) {
      const uint64_t mid = (lo + hi) / 2;
      if (in_ids[mid] < g) lo = mid + 1;
      else hi = mid;
    }
    src = (lo < n_in && in_ids[lo] == g) ? (uint32_t)lo : PB_SOLVE_NONE;
  }
  if (k == 0 || (keys[k - 1] >> cb) != g) inp[var] = src;
  const uint32_t row = cell / 3;
  if (src == PB_SOLVE_NONE && cell - 3 * row == 2 && qual[row]) atomicMin(def_row + var, row);
}

// per cell: unset (a variable with no source) and order (an operand of a defining row that it or a later row defines);
// per row: whether it defines its O variable
__global__ void k_solve_flags(const uint32_t* var_of_cell, const uint32_t* inp, const uint32_t* def_row, uint64_t n,
                              uint8_t* unset, uint8_t* order, uint8_t* defines) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * n) return;
  const uint32_t row = (uint32_t)(c / 3), col = (uint32_t)(c - 3 * (uint64_t)row), v = var_of_cell[c];
  const uint32_t d = def_row[v];
  unset[c] = (inp[v] == PB_SOLVE_NONE && d == PB_SOLVE_NONE) ? 1 : 0;
  const bool row_defines = def_row[var_of_cell[3 * (uint64_t)row + 2]] == row;
  order[c] = (col < 2 && row_defines && d != PB_SOLVE_NONE && d >= row) ? 1 : 0;
  if (col == 2) defines[row] = row_defines ? 1 : 0;
}

// the variables' starting values: 0 for id -1, the inputs (canonical -> Montgomery); ready flag set for both
__global__ void k_solve_init(const uint32_t* inp, const Fr* in_vals, uint64_t n_vars, Fr* val, uint32_t* ready) {
  const uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n_vars) return;
  const uint32_t s = inp[v];
  if (s == PB_SOLVE_ZERO) val[v] = Fr::zero();
  else if (s != PB_SOLVE_NONE) val[v] = fp_to_mont(ldg_fr(in_vals + s));
  ready[v] = s != PB_SOLVE_NONE ? 1 : 0;
}

__device__ __forceinline__ uint64_t sv_now() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// what the evaluation of table-defining rows reads and writes: the qualify flags (PB_SOLVE_BY_TABLE), Q_T (Montgomery,
// null for one untagged table), the index, and per row a miss and an ambiguous flag
struct SolveLk {
  const uint8_t* qual;
  const Fr* qt;
  SolveTable T;
  uint8_t *miss, *amb;
};

// the defining rows rows[0, n_def), ascending, in dependency order (see the file comment).  status[0]: the ticket,
// status[1]: set when a warp stalled.  kTable: a row flagged PB_SOLVE_BY_TABLE probes the index (solve.cuh,
// solve_probe) instead of running the gate body; a miss or an ambiguous key sets the row's flag and still stores c = 0
// and the ready flag, so the rows that depend on it finish.  lk is read only then.
template <bool kTable>
__global__ void __launch_bounds__(128) k_solve_eval(SolveSel s, const uint32_t* rows, uint64_t n_def,
                                                    const uint32_t* var_of_cell, Fr* val, uint32_t* ready,
                                                    uint32_t* status, SolveLk lk) {
  const uint32_t lane = threadIdx.x & 31;
  cuda::atomic_ref<uint32_t, cuda::thread_scope_device> stalled(status[1]);
  for (;;) {
    uint32_t t = 0;
    if (lane == 0) t = atomicAdd(status, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    const uint64_t i = (uint64_t)t * 32 + lane;
    if ((uint64_t)t * 32 >= n_def) return;
    bool done = i >= n_def;
    uint32_t vl = 0, vr = 0, vo = 0;
    SolveRow sr;
    uint64_t row = 0;
    bool table = false;
    Fr tag;
    if (!done) {
      const uint64_t r = rows[i];
      vl = var_of_cell[3 * r];
      vr = var_of_cell[3 * r + 1];
      vo = var_of_cell[3 * r + 2];
      if constexpr (kTable) {
        row = r;
        table = lk.qual[r] == PB_SOLVE_BY_TABLE;
        if (table) tag = lk.qt ? ldg_fr(lk.qt + r) : Fr::zero();
      }
      if (!table) {
        sr.ql = ldg_fr(s.ql + r);
        sr.qr = ldg_fr(s.qr + r);
        sr.qm = ldg_fr(s.qm + r);
        sr.qc = ldg_fr(s.qc + r);
        sr.neg_inv_qo = fp_neg(ldg_fr(s.inv_qo + r));
#pragma unroll
        for (int k = 0; k < PB_MAX_CUSTOM; k++) sr.q[k] = k < s.n_custom ? ldg_fr(s.q[k] + r) : Fr::zero();
      }
    }
    uint64_t since = sv_now();
    while (!__all_sync(0xffffffffu, done)) {
      bool moved = false;
      if (!done) {
        cuda::atomic_ref<uint32_t, cuda::thread_scope_device> rl(ready[vl]), rr(ready[vr]);
        if (rl.load(cuda::memory_order_acquire) && rr.load(cuda::memory_order_acquire)) {
          const Fr a = val[vl], b = val[vr];
          if (table) {
            Fr c;
            const int e = solve_probe(lk.T, tag, a, b, &c);
            if (e == PB_SOLVE_MISS) lk.miss[row] = 1;
            if (e == PB_SOLVE_AMBIGUOUS) lk.amb[row] = 1;
            val[vo] = c;
          } else {
            val[vo] = solve_gate(sr, s.f, s.n_custom, a, b);
          }
          cuda::atomic_ref<uint32_t, cuda::thread_scope_device>(ready[vo]).store(1, cuda::memory_order_release);
          done = moved = true;
        }
      }
      if (__any_sync(0xffffffffu, moved)) {
        since = sv_now();
        continue;
      }
      // leave together: the decisions are the warp's, so no lane is left in a later __all_sync alone
      if (__any_sync(0xffffffffu, lane == 0 && stalled.load(cuda::memory_order_relaxed))) return;
      if (__any_sync(0xffffffffu, lane == 0 && sv_now() - since > PB_SOLVE_STALL_NS)) {
        if (lane == 0) stalled.store(1, cuda::memory_order_relaxed);
        return;
      }
      __nanosleep(64);
    }
  }
}

// ---- the shuffle (pb200_solve_wires_shuffle) ---------------------------------------------------------------------------
// side[r] as k_solve_qualify reads it; p: the first out-row.

// per out-row cell (after k_solve_vars): count the out-row cells of its variable, and let the shuffle define it at row p
// unless it is the constant 0 or an input.  A row below p that defines it keeps it (a clash); a row above p does not.
__global__ void k_solve_claim_out(const uint8_t* side, const uint32_t* var_of_cell, const uint32_t* inp, uint64_t n,
                                  uint32_t p, uint32_t* out_cells, uint32_t* def_row) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * n || side[c / 3] != PB_SOLVE_OUT) return;
  const uint32_t v = var_of_cell[c];
  atomicAdd(out_cells + v, 1u);
  if (inp[v] == PB_SOLVE_NONE) atomicMin(def_row + v, p);
}

// why an out-row cell cannot take the shuffled value, or PB_SOLVE_NONE when it can
#define PB_SOLVE_CLASH_NO_VAR 0   // the cell has no variable (-1)
#define PB_SOLVE_CLASH_INPUT 1    // its variable is an input
#define PB_SOLVE_CLASH_DEFINED 2  // a row below p defines its variable
#define PB_SOLVE_CLASH_SHARED 3   // its variable is on another out-row cell too
__device__ __forceinline__ uint32_t solve_clash(uint32_t v, const uint32_t* inp, const uint32_t* def_row,
                                                const uint32_t* out_cells, uint32_t p) {
  if (inp[v] == PB_SOLVE_ZERO) return PB_SOLVE_CLASH_NO_VAR;
  if (inp[v] != PB_SOLVE_NONE) return PB_SOLVE_CLASH_INPUT;
  if (def_row[v] < p) return PB_SOLVE_CLASH_DEFINED;
  if (out_cells[v] > 1) return PB_SOLVE_CLASH_SHARED;
  return PB_SOLVE_NONE;
}

// per cell: late (an in-row cell whose variable is defined at or after p: by the shuffle or by a row above p) and
// clash (an out-row cell that cannot take the shuffled value)
__global__ void k_solve_shuffle_flags(const uint8_t* side, const uint32_t* var_of_cell, const uint32_t* inp,
                                      const uint32_t* def_row, const uint32_t* out_cells, uint64_t n, uint32_t p,
                                      uint8_t* late, uint8_t* clash) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * n) return;
  const uint8_t sd = side[c / 3];
  const uint32_t v = var_of_cell[c], d = def_row[v];
  late[c] = (sd == PB_SOLVE_IN && inp[v] == PB_SOLVE_NONE && d != PB_SOLVE_NONE && d >= p) ? 1 : 0;
  clash[c] = (sd == PB_SOLVE_OUT && solve_clash(v, inp, def_row, out_cells, p) != PB_SOLVE_NONE) ? 1 : 0;
}

// the clash list's second and third entries: the reason of each listed cell, and the row below p that defines its
// variable (PB_SOLVE_NONE for the other reasons)
__global__ void k_solve_clash_reasons(const uint32_t* cells, uint32_t count, const uint32_t* var_of_cell,
                                      const uint32_t* inp, const uint32_t* def_row, const uint32_t* out_cells,
                                      uint32_t p, uint32_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const uint32_t v = var_of_cell[cells[k]], why = solve_clash(v, inp, def_row, out_cells, p);
  out[2 * k] = why;
  out[2 * k + 1] = why == PB_SOLVE_CLASH_DEFINED ? def_row[v] : PB_SOLVE_NONE;
}

// the K in-rows' tuples, canonical, as twelve columns of K 64-bit words: word w (0..11) is limb w % 4 of a, b, c for
// w / 4 = 0, 1, 2; and the starting positions 0..K-1
__global__ void k_solve_shuffle_gather(const uint32_t* in_rows, uint64_t K, const uint32_t* var_of_cell, const Fr* val,
                                       uint64_t* words, uint32_t* pos) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  const uint64_t r = in_rows[k];
#pragma unroll
  for (int col = 0; col < 3; col++) {
    const Fr x = fp_from_mont(val[var_of_cell[3 * r + col]]);
#pragma unroll
    for (int l = 0; l < 4; l++) words[(uint64_t)(4 * col + l) * K + k] = (uint64_t)x.v[2 * l] | ((uint64_t)x.v[2 * l + 1] << 32);
  }
  pos[k] = (uint32_t)k;
}

// the OR (acc[w]) and the AND (acc[12 + w]) of every word over the in-rows (acc set to 0 and ~0 before)
__global__ void __launch_bounds__(256) k_solve_shuffle_bits(const uint64_t* words, uint64_t K,
                                                            unsigned long long* acc) {
  __shared__ unsigned long long s_or[12], s_and[12];
  if (threadIdx.x < 12) {
    s_or[threadIdx.x] = 0;
    s_and[threadIdx.x] = ~0ull;
  }
  __syncthreads();
  unsigned long long o[12], a[12];
#pragma unroll
  for (int w = 0; w < 12; w++) o[w] = 0, a[w] = ~0ull;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < K; k += (uint64_t)gridDim.x * blockDim.x)
#pragma unroll
    for (int w = 0; w < 12; w++) {
      const unsigned long long x = words[(uint64_t)w * K + k];
      o[w] |= x;
      a[w] &= x;
    }
#pragma unroll
  for (int w = 0; w < 12; w++) {
    for (int s = 16; s; s >>= 1) {
      o[w] |= __shfl_xor_sync(0xffffffffu, o[w], s);
      a[w] &= __shfl_xor_sync(0xffffffffu, a[w], s);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicOr(s_or + w, o[w]);
      atomicAnd(s_and + w, a[w]);
    }
  }
  __syncthreads();
  if (threadIdx.x < 12) {
    atomicOr(acc + threadIdx.x, s_or[threadIdx.x]);
    atomicAnd(acc + 12 + threadIdx.x, s_and[threadIdx.x]);
  }
}

// one LSD pass: the word of the tuple at each sorted position, the key of the pass's stable sort
__global__ void k_solve_shuffle_key(const uint64_t* column, const uint32_t* pos, uint64_t K, uint64_t* key) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) key[k] = column[pos[k]];
}

// out-row j (ascending) takes the tuple of in-row in_rows[pos[j]] (the j-th in sorted order): its three variables get
// the in-row's values (Montgomery) and their ready flags
__global__ void k_solve_shuffle_put(const uint32_t* in_rows, const uint32_t* out_rows, const uint32_t* pos, uint64_t K,
                                    const uint32_t* var_of_cell, Fr* val, uint32_t* ready) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * K) return;
  const uint64_t j = c / 3, col = c - 3 * j;
  const uint32_t v = var_of_cell[3 * (uint64_t)out_rows[j] + col];
  val[v] = val[var_of_cell[3 * (uint64_t)in_rows[pos[j]] + col]];
  ready[v] = 1;
}

// a and b of each listed row, canonical, for the miss and ambiguous messages
__global__ void k_solve_operands(const uint32_t* rows, uint32_t count, const uint32_t* var_of_cell, const Fr* val,
                                 Fr* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= count) return;
  const uint64_t r = rows[k];
  out[2 * k] = fp_from_mont(val[var_of_cell[3 * r]]);
  out[2 * k + 1] = fp_from_mont(val[var_of_cell[3 * r + 1]]);
}

// every cell's value, canonical: W = A | B | C, column-major
__global__ void k_solve_write(const uint32_t* var_of_cell, const Fr* val, uint64_t n, Fr* A, Fr* B, Fr* C) {
  const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * n) return;
  const uint64_t row = c / 3, col = c - 3 * row;
  const Fr x = fp_from_mont(val[var_of_cell[c]]);
  (col == 0 ? A : col == 1 ? B : C)[row] = x;
}

// the order list's second entry: the row defining the variable of each listed cell
__global__ void k_solve_order_rows(const uint32_t* cells, uint32_t count, const uint32_t* var_of_cell,
                                   const uint32_t* def_row, uint32_t* out) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) out[k] = def_row[var_of_cell[cells[k]]];
}

// the table index of T's columns (rows table rows) into T.word / T.row / T.amb; sets T.theta, T.theta2 and T.n_keys.
// The (word, row) pairs are sorted; neighbours with equal words must have equal keys, else theta is drawn again.  The
// runs of equal words are then the distinct keys, in ascending word order.  temp: at least SortPairs' storage over rows
// items and InclusiveSum's; impure: one device word.
static void solve_table_index(Context* ctx, SolveTable& T, uint64_t rows, DevBuf& temp, uint32_t* impure) {
  cudaStream_t st = ctx->stream;
  DevBuf k1(rows * 8), k2(rows * 8), r1(rows * 4), r2(rows * 4), head(rows * 4), run(rows * 4), split(rows);
  cub::DoubleBuffer<uint64_t> keys(k1.as<uint64_t>(), k2.as<uint64_t>());
  cub::DoubleBuffer<uint32_t> idx(r1.as<uint32_t>(), r2.as<uint32_t>());
  for (int draw = 0;; draw++) {
    PB_CHECK(draw < 8, "solving the wires: eight table words in a row had colliding keys");
    T.theta = check_random_fr();
    T.theta2 = fp_sqr(T.theta);
    k_solve_tab_keys<<<PB_GRID(rows, 128), 0, st>>>(T, rows, k1.as<uint64_t>(), r1.as<uint32_t>());
    launched(ctx);
    keys = cub::DoubleBuffer<uint64_t>(k1.as<uint64_t>(), k2.as<uint64_t>());
    idx = cub::DoubleBuffer<uint32_t>(r1.as<uint32_t>(), r2.as<uint32_t>());
    size_t tb = temp.bytes;
    PB_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, keys, idx, (int)rows, 0, 64, st));
    ctx->launches++;
    PB_CUDA(cudaMemsetAsync(impure, 0, 4, st));
    k_solve_tab_heads<<<PB_GRID(rows, 256), 0, st>>>(T, keys.Current(), idx.Current(), rows, head.as<uint32_t>(),
                                                           split.as<uint8_t>(), impure);
    launched(ctx);
    uint32_t imp = 0;
    PB_CUDA(cudaMemcpyAsync(&imp, impure, 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    if (imp == 0) break;
  }
  size_t tb = temp.bytes;
  PB_CUDA(cub::DeviceScan::InclusiveSum(temp.p, tb, head.as<uint32_t>(), run.as<uint32_t>(), (int)rows, st));
  ctx->launches++;
  PB_CUDA(cudaMemsetAsync(const_cast<uint8_t*>(T.amb), 0, rows, st));
  k_solve_tab_unique<<<PB_GRID(rows, 256), 0, st>>>(keys.Current(), idx.Current(), head.as<uint32_t>(),
                                                          run.as<uint32_t>(), split.as<uint8_t>(), rows,
                                                          const_cast<uint64_t*>(T.word), const_cast<uint32_t*>(T.row),
                                                          const_cast<uint8_t*>(T.amb));
  launched(ctx);
  uint32_t keys_n = 0;
  PB_CUDA(cudaMemcpyAsync(&keys_n, run.as<uint32_t>() + rows - 1, 4, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));  // the index's temporaries die here
  T.n_keys = keys_n;
}

// the shuffle step, between the two phases of the evaluation: out-row j (out_rows ascending) takes the tuple of the j-th
// in-row in ascending (a, b, c) order, compared as canonical integers.  The positions 0..K-1 of the in-rows are sorted
// LSD by the twelve 64-bit words of their tuple, c's lowest first and a's highest last, one stable SortPairs a word.  A
// word equal on every in-row (OR = AND) is skipped, and the others sort only the bits from the lowest to the highest
// one where OR and AND differ: small integers (addresses, counters) cost a pass or two, random field elements twelve.
// temp: at least SortPairs' storage over K items; acc: 24 device words.
static void solve_shuffle(Context* ctx, const uint32_t* in_rows, const uint32_t* out_rows, uint64_t K,
                          const uint32_t* var_of_cell, Fr* val, uint32_t* ready, DevBuf& temp,
                          unsigned long long* acc) {
  cudaStream_t st = ctx->stream;
  DevBuf words(K * 96), k1(K * 8), k2(K * 8), p1(K * 4), p2(K * 4);
  k_solve_shuffle_gather<<<PB_GRID(K, 128), 0, st>>>(in_rows, K, var_of_cell, val, words.as<uint64_t>(),
                                                           p1.as<uint32_t>());
  launched(ctx);
  PB_CUDA(cudaMemsetAsync(acc, 0, 12 * 8, st));
  PB_CUDA(cudaMemsetAsync(acc + 12, 0xff, 12 * 8, st));
  const uint64_t blocks = std::min<uint64_t>((K + 255) / 256, 4 * (uint64_t)ctx->sm_count);
  k_solve_shuffle_bits<<<(unsigned)blocks, 256, 0, st>>>(words.as<uint64_t>(), K, acc);
  launched(ctx);
  unsigned long long bits[24];
  PB_CUDA(cudaMemcpyAsync(bits, acc, sizeof bits, cudaMemcpyDeviceToHost, st));
  PB_CUDA(cudaStreamSynchronize(st));
  cub::DoubleBuffer<uint64_t> keys(k1.as<uint64_t>(), k2.as<uint64_t>());
  cub::DoubleBuffer<uint32_t> pos(p1.as<uint32_t>(), p2.as<uint32_t>());
  for (int t = 2; t >= 0; t--)  // c, b, a
    for (int l = 0; l < 4; l++) {
      const int w = 4 * t + l;
      const unsigned long long diff = bits[w] ^ bits[12 + w];
      if (!diff) continue;
      k_solve_shuffle_key<<<PB_GRID(K, 256), 0, st>>>(words.as<uint64_t>() + (uint64_t)w * K, pos.Current(), K,
                                                            keys.Current());
      launched(ctx);
      size_t tb = temp.bytes;
      PB_CUDA(cub::DeviceRadixSort::SortPairs(temp.p, tb, keys, pos, (int)K, __builtin_ctzll(diff),
                                              64 - __builtin_clzll(diff), st));
      ctx->launches++;
    }
  k_solve_shuffle_put<<<PB_GRID(3 * K, 256), 0, st>>>(in_rows, out_rows, pos.Current(), K, var_of_cell, val,
                                                            ready);
  launched(ctx);
  PB_CUDA(cudaStreamSynchronize(st));  // the sort's buffers die here
}

namespace {
thread_local double g_solve_ms[3];  // the last shuffle solve: phase 1, the shuffle step, phase 2 (device events)
}
void solve_stages(double* out_ms, int count) {
  for (int k = 0; k < count && k < 3; k++) out_ms[k] = g_solve_ms[k];
}

namespace {
// one call of solve_run: its arguments, what the host checks made of them, and the device buffers of the steps
struct Solve {
  Context* ctx;
  cudaStream_t st;
  const SolveArgs& a;
  const SolveTableArgs* tb;    // null without a table
  const SolveShuffleArgs* sf;  // null without a shuffle
  uint64_t n = 0, m = 0;
  SolveSel s = {};
  int64_t max_id = -1;
  std::vector<uint64_t> in_keys;  // the inputs' ids + 1, ascending, and their values in that order
  std::vector<uint8_t> in_vals;
  // the shuffle: per row its side, K in-rows (as many out-rows), the first out-row p.  Without out-rows (q_in and q_out
  // all 0, or both 1 on the same rows) the solve is the one without a shuffle.
  std::vector<uint8_t> side;
  uint64_t K = 0;
  uint32_t p = PB_SOLVE_NONE;
  bool out_rows = false;
  uint64_t temp_bytes = 0;
  DevBuf temp, keys, alt, head, run, voc, inp, defr, ready, val, idx, flags, small, inids, invals, sel, qual, defines;
  DevBuf qkb, qtb, tabb, errf, ix_word, ix_row, ix_amb;  // the table
  DevBuf sideb, outc, shf;                                // the shuffle
  SolveLk lk = {};
  uint32_t *small_u = nullptr, *num = nullptr;

  Solve(Context* c, const SolveArgs& args, const SolveTableArgs* t, const SolveShuffleArgs* f)
      : ctx(c), st(c->stream), a(args), tb(t), sf(f) {}

  // the arguments, before any device work
  void require() {
    PB_CHECK(a.log_n >= 1 && a.log_n <= 26, "group order must be 2^k, 1 <= k <= 26 (the prover's range)");
    n = (uint64_t)1 << a.log_n;
    m = 3 * n;
    PB_CHECK(a.n_constraints <= n, "n_constraints above the group order");
    PB_CHECK(a.ids && a.sel && a.counts && (a.lists || a.limit == 0) && a.out && (a.in_ids || a.n_inputs == 0) &&
                 (a.in_vals || a.n_inputs == 0),
             "solving the wires needs the ids, the selectors, the inputs and the outputs");
    for (int k = 0; k < 5; k++) PB_CHECK(a.sel[k], "solving the wires needs QL, QR, QM, QO and QC");
    for (int k = 0; k < 3; k++) PB_CHECK(a.out[k], "solving the wires needs three output buffers");
    PB_CHECK(a.limit <= m, "limit above 3n, the most entries a list can have");
    PB_CHECK(a.n_custom >= 0 && a.n_custom <= PB_MAX_CUSTOM, "at most 4 custom gate terms");
    PB_CHECK(a.n_custom == 0 || (a.exps && a.custom), "custom gate terms need their exponents and selectors");
    s.n_custom = a.n_custom;
    for (int k = 0; k < a.n_custom; k++) {
      const uint8_t* e = a.exps + 6 * k;
      const int deg = e[0] + e[1] + e[2] + e[3] + e[4] + e[5];
      PB_CHECK(deg >= 1 && deg <= 3, "custom gate term must have total degree 1, 2 or 3");
      PB_CHECK(a.custom[k], "custom gate term without its selector");
      int f = 0;
      for (int w = 0; w < 6; w++)
        for (int t = 0; t < e[w]; t++) s.f[k][f++] = (uint8_t)w;
      while (f < 3) s.f[k][f++] = PB_FACTOR_ONE;
    }
    // ids (only rows below n_constraints are read), inputs and their values
    perm_require_ids(a.ids, 3 * a.n_constraints, &max_id);
    std::vector<uint64_t> order(a.n_inputs);
    for (uint64_t k = 0; k < a.n_inputs; k++) {
      const int64_t id = a.in_ids[k];
      if (id < 0 || id > PB_PERM_MAX_ID) {
        char b[256];
        snprintf(b, sizeof b, "input %llu: variable id %lld is outside [0, 2^32 - 2]", (unsigned long long)k,
                 (long long)id);
        throw Error(b);
      }
      Fr x;
      memcpy(x.v, a.in_vals + 32 * k, 32);
      if (!fp_is_canonical(x)) {
        char b[256];
        snprintf(b, sizeof b, "input %llu (variable %lld): value not reduced below the field modulus",
                 (unsigned long long)k, (long long)id);
        throw Error(b);
      }
      order[k] = k;
    }
    const int64_t* ids = a.in_ids;
    std::sort(order.begin(), order.end(),
              [ids](uint64_t x, uint64_t y) { return ids[x] != ids[y] ? ids[x] < ids[y] : x < y; });
    in_keys.resize(a.n_inputs);
    in_vals.resize(a.n_inputs * 32);
    for (uint64_t k = 0; k < a.n_inputs; k++) {
      if (k > 0 && a.in_ids[order[k]] == a.in_ids[order[k - 1]]) {
        char b[256];
        snprintf(b, sizeof b, "inputs %llu and %llu both name variable %lld", (unsigned long long)order[k - 1],
                 (unsigned long long)order[k], (long long)a.in_ids[order[k]]);
        throw Error(b);
      }
      in_keys[k] = (uint64_t)(a.in_ids[order[k]] + 1);
      memcpy(&in_vals[32 * k], a.in_vals + 32 * order[k], 32);
    }
    if (tb) lookup_require(n, tb->qk, tb->qtag, tb->tab, tb->rows);
    if (sf) {
      shuffle_require(n, sf->qin, sf->qout);
      side.resize(n);
      for (uint64_t i = 0; i < n; i++) {
        const uint8_t in = sf->qin[32 * i], out = sf->qout[32 * i];
        side[i] = in == out ? 0 : in ? PB_SOLVE_IN : PB_SOLVE_OUT;
        K += side[i] == PB_SOLVE_IN;
        if (side[i] == PB_SOLVE_OUT && p == PB_SOLVE_NONE) p = (uint32_t)i;
      }
    }
    out_rows = K > 0;
  }

  // the device memory the call needs, refused when more than is free; then the buffers
  void reserve() {
    const int end_bit = perm_sort_bits(a.log_n, max_id);
    const uint64_t rows = tb ? tb->rows : 0;
    size_t t_sort = 0, t_scan = 0, t_sel = 0, t_tab = 0, t_sh = 0;
    cub::DoubleBuffer<uint64_t> d(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    PB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t_sort, d, (int)m, 0, end_bit, st));
    PB_CUDA(cub::DeviceScan::InclusiveSum(nullptr, t_scan, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, st));
    PB_CUDA(cub::DeviceSelect::Flagged(nullptr, t_sel, thrust::counting_iterator<uint32_t>(0), (const uint8_t*)nullptr,
                                       (uint32_t*)nullptr, (uint32_t*)nullptr, (int)m, st));
    if (tb) PB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_tab, d, v, (int)rows, 0, 64, st));
    if (out_rows) PB_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_sh, d, v, (int)K, 0, 64, st));
    temp_bytes = std::max(std::max(std::max(t_sort, t_tab), std::max(t_scan, t_sel)), t_sh);
    // keys and alt (8 each), heads / run (4 each), var_of_cell, inp, def_row, ready (4 each), the values (32), the
    // index list (4), three flag bytes: per cell.  Selectors, 1 / QO and the custom selectors (32 each), the qualify
    // and defines flags: per row.  The inputs, the host outputs' staging and the sort's storage.
    const uint64_t limit = a.limit, n_custom = (uint64_t)a.n_custom;
    uint64_t need = m * (8 + 8 + 4 + 4 + 4 * 4 + 32 + 4 + 3) + n * (32 * (6 + n_custom) + 2) + a.n_inputs * 40 +
                    (a.out_on_device ? 0 : m * 32) + temp_bytes + 256;
    // with a table: q_K and Q_T (32 each) and the miss and ambiguous flags (1 each) per row; per table row its columns
    // (4 x 32), the sort's words and rows (2 x 8, 2 x 4), heads and runs (4 each), the split flag, the index
    // (8 + 4 + 1); the listed rows' operands
    if (tb) need += n * (32 + 32 + 2) + rows * (4 * 32 + 16 + 8 + 8 + 1 + 13) + limit * 2 * 64 + 256;
    // with a shuffle: the side and the in / out flags (1 each) per row; the out-row cell count (4) and the late and
    // clash flags (1 each) per cell; per in-row its tuple (96), the sort's words and positions (2 x 8, 2 x 4) and the
    // in-row and out-row lists (4 each); the listed cells' entries
    if (out_rows) need += n * 3 + m * (4 + 2) + K * (96 + 16 + 8 + 8) + limit * 5 * 4 + 256;
    size_t free_b = 0, total_b = 0;
    PB_CUDA(cudaMemGetInfo(&free_b, &total_b));
    // PB200_SOLVE_MAX_BYTES: the most device memory a solve may take (read per call), so it leaves room for other work
    if (const char* e = getenv("PB200_SOLVE_MAX_BYTES")) free_b = std::min<size_t>(free_b, strtoull(e, nullptr, 10));
    if (need > free_b) {
      char b[256];
      snprintf(b, sizeof b, "solving the wires of 2^%d rows needs %llu bytes of device memory, %llu are free", a.log_n,
               (unsigned long long)need, (unsigned long long)free_b);
      throw Error(b);
    }
    for (DevBuf* b : {&keys, &alt}) b->alloc(m * 8);
    for (DevBuf* b : {&head, &run, &voc, &inp, &defr, &ready, &idx}) b->alloc(m * 4);
    temp.alloc(temp_bytes);
    val.alloc(m * 32);
    flags.alloc(3 * m);
    small.alloc(out_rows ? 32 + 24 * 8 : 64);
    inids.alloc(a.n_inputs * 8 + 8);
    invals.alloc(a.n_inputs * 32 + 32);
    sel.alloc((6 + n_custom) * n * 32);
    qual.alloc(n);
    defines.alloc(n);
    small_u = small.as<uint32_t>();
    num = small_u + 1;
    if (tb) {
      qkb.alloc(n * 32);
      if (tb->qtag) qtb.alloc(n * 32);
      tabb.alloc((tb->qtag ? 4 : 3) * rows * 32);
      errf.alloc(2 * n);
    }
    if (out_rows) {
      sideb.alloc(3 * n);
      outc.alloc(m * 4);
      shf.alloc(2 * m);
    }
  }

  // the selectors, the inputs, the table and the shuffle's sides on the device; 1. group; 2. sources
  void sources() {
    Fr* selp = sel.as<Fr>();
    const uint64_t n_sel = (5 + (uint64_t)a.n_custom) * n;
    const Fr* sel_col[5];
    for (int k = 0; k < 5 + a.n_custom; k++) {
      Fr* col = selp + (uint64_t)k * n;
      PB_CUDA(cudaMemcpyAsync(col, k < 5 ? a.sel[k] : a.custom[k - 5], n * 32, cudaMemcpyHostToDevice, st));
      if (k < 5) sel_col[k] = col;
      else s.q[k - 5] = col;
    }
    PB_CUDA(cudaMemsetAsync(small.p, 0, 64, st));
    k_count_noncanonical<<<PB_GRID(n_sel, 256), 0, st>>>(selp, n_sel, small_u + 2);
    launched(ctx);
    fr_to_mont(ctx, selp, selp, n_sel);
    s.ql = sel_col[0];
    s.qr = sel_col[1];
    s.qm = sel_col[2];
    s.qo = sel_col[3];
    s.qc = sel_col[4];
    s.inv_qo = selp + n_sel;
    const uint64_t T = (n + PB_SOLVE_BATCH_CH - 1) / PB_SOLVE_BATCH_CH;
    k_batch_div<<<PB_GRID(T, 128), 0, st>>>(nullptr, s.qo, selp + n_sel, n, T);
    launched(ctx);
    uint32_t bad_sel = 0;
    PB_CUDA(cudaMemcpyAsync(&bad_sel, small_u + 2, 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    PB_CHECK(bad_sel == 0, "selector value not reduced below the field modulus");
    if (a.n_inputs) {
      PB_CUDA(cudaMemcpyAsync(inids.p, in_keys.data(), a.n_inputs * 8, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemcpyAsync(invals.p, in_vals.data(), a.n_inputs * 32, cudaMemcpyHostToDevice, st));
    }
    if (tb) {  // q_K (canonical), Q_T and the table columns (Montgomery), the per-row error flags
      const uint64_t rows = tb->rows;
      const int width = tb->qtag ? 4 : 3;
      PB_CUDA(cudaMemcpyAsync(qkb.p, tb->qk, n * 32, cudaMemcpyHostToDevice, st));
      if (tb->qtag) {
        PB_CUDA(cudaMemcpyAsync(qtb.p, tb->qtag, n * 32, cudaMemcpyHostToDevice, st));
        fr_to_mont(ctx, qtb.as<Fr>(), qtb.as<Fr>(), n);
      }
      for (int w = 0; w < width; w++) {
        lk.T.t[w] = tabb.as<Fr>() + (uint64_t)w * rows;
        PB_CUDA(cudaMemcpyAsync(tabb.as<Fr>() + (uint64_t)w * rows, tb->tab[w], rows * 32, cudaMemcpyHostToDevice, st));
      }
      fr_to_mont(ctx, tabb.as<Fr>(), tabb.as<Fr>(), width * rows);
      PB_CUDA(cudaMemsetAsync(errf.p, 0, 2 * n, st));
      lk.qual = qual.as<uint8_t>();
      lk.qt = tb->qtag ? qtb.as<Fr>() : nullptr;
      lk.miss = errf.as<uint8_t>();
      lk.amb = lk.miss + n;
    }
    if (out_rows) {  // per row its side, then the in-row and the out-row flags (for the row lists)
      std::vector<uint8_t> fl(2 * n);
      for (uint64_t i = 0; i < n; i++) {
        fl[i] = side[i] == PB_SOLVE_IN;
        fl[n + i] = side[i] == PB_SOLVE_OUT;
      }
      PB_CUDA(cudaMemcpyAsync(sideb.p, side.data(), n, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemcpyAsync(sideb.as<uint8_t>() + n, fl.data(), 2 * n, cudaMemcpyHostToDevice, st));
    }

    // 1. group
    const int cb = perm_cell_bits(a.log_n);
    const uint64_t* sorted = perm_sort_keys(ctx, a.ids, m, cb, perm_sort_bits(a.log_n, max_id), keys, alt, temp,
                                            temp_bytes, 3 * a.n_constraints);
    k_solve_heads<<<PB_GRID(m, 256), 0, st>>>(sorted, m, cb, head.as<uint32_t>());
    launched(ctx);
    size_t tb_bytes = temp.bytes;
    PB_CUDA(cub::DeviceScan::InclusiveSum(temp.p, tb_bytes, head.as<uint32_t>(), run.as<uint32_t>(), (int)m, st));
    ctx->launches++;
    // 2. sources
    k_solve_qualify<<<PB_GRID(n, 256), 0, st>>>(s, tb ? qkb.as<Fr>() : nullptr,
                                                out_rows ? sideb.as<uint8_t>() : nullptr, a.n_constraints,
                                                qual.as<uint8_t>());
    launched(ctx);
    PB_CUDA(cudaMemsetAsync(defr.p, 0xff, m * 4, st));
    PB_CUDA(cudaMemsetAsync(inp.p, 0xff, m * 4, st));  // variables past the last run: no source
    k_solve_vars<<<PB_GRID(m, 256), 0, st>>>(sorted, run.as<uint32_t>(), m, cb, inids.as<uint64_t>(), a.n_inputs,
                                             qual.as<uint8_t>(), voc.as<uint32_t>(), inp.as<uint32_t>(),
                                             defr.as<uint32_t>());
    launched(ctx);
    if (out_rows) {  // out-row variables: defined at row p
      PB_CUDA(cudaMemsetAsync(outc.p, 0, m * 4, st));
      k_solve_claim_out<<<PB_GRID(m, 256), 0, st>>>(sideb.as<uint8_t>(), voc.as<uint32_t>(), inp.as<uint32_t>(), n, p,
                                                    outc.as<uint32_t>(), defr.as<uint32_t>());
      launched(ctx);
    }
    k_solve_flags<<<PB_GRID(m, 256), 0, st>>>(voc.as<uint32_t>(), inp.as<uint32_t>(), defr.as<uint32_t>(), n,
                                              flags.as<uint8_t>(), flags.as<uint8_t>() + m, defines.as<uint8_t>());
    launched(ctx);
    if (out_rows) {  // row p defines nothing, though its O variable is defined at p: its flag and its operands' order
                     // flags off
      PB_CUDA(cudaMemsetAsync(defines.as<uint8_t>() + p, 0, 1, st));
      PB_CUDA(cudaMemsetAsync(flags.as<uint8_t>() + m + 3 * (uint64_t)p, 0, 2, st));
    }
  }

  // the cells flagged in f (m of them): their count, and at out the lowest `limit` of them, each followed by `extra`
  // entries that fill(d_cells, listed, d_entries) computes on the device
  template <class Fill>
  uint64_t list_cells(const uint8_t* f, uint32_t* out, int extra, Fill fill) {
    std::vector<uint32_t> cells(a.limit);
    const uint64_t count = compact_flagged(ctx, f, m, temp, idx.as<uint32_t>(), num, a.limit, cells.data());
    const uint32_t listed = (uint32_t)std::min<uint64_t>(count, a.limit);
    if (listed) {
      DevBuf d((size_t)listed * (1 + extra) * 4);
      PB_CUDA(cudaMemcpyAsync(d.p, cells.data(), (size_t)listed * 4, cudaMemcpyHostToDevice, st));
      fill(d.as<uint32_t>(), listed, d.as<uint32_t>() + listed);
      launched(ctx);
      std::vector<uint32_t> got((size_t)listed * extra);
      PB_CUDA(cudaMemcpyAsync(got.data(), d.as<uint32_t>() + listed, got.size() * 4, cudaMemcpyDeviceToHost, st));
      PB_CUDA(cudaStreamSynchronize(st));
      for (uint32_t k = 0; k < listed; k++) {
        out[(1 + extra) * (uint64_t)k] = cells[k];
        for (int j = 0; j < extra; j++) out[(1 + extra) * (uint64_t)k + 1 + j] = got[(uint64_t)extra * k + j];
      }
    }
    return count;
  }
  // the cells flagged in f, each with the row defining its variable
  uint64_t list_with_rows(const uint8_t* f, uint32_t* out) {
    return list_cells(f, out, 1, [&](const uint32_t* cells, uint32_t count, uint32_t* rows) {
      k_solve_order_rows<<<PB_GRID(count, 128), 0, st>>>(cells, count, voc.as<uint32_t>(), defr.as<uint32_t>(), rows);
    });
  }

  // the errors found before any row is evaluated: unset and order, and with out-rows late and clash; true with any
  bool errors() {
    const uint64_t limit = a.limit;
    uint64_t* counts = a.counts;
    for (uint64_t k = 0; k < (tb ? 5 : sf ? 8 : 3) * limit; k++) a.lists[k] = 0xffffffffu;
    counts[0] = compact_flagged(ctx, flags.as<uint8_t>(), m, temp, idx.as<uint32_t>(), num, a.limit, a.lists);
    counts[1] = list_with_rows(flags.as<uint8_t>() + m, a.lists + limit);
    if (tb || sf) counts[2] = counts[3] = 0;
    if (out_rows) {  // late in-row cells (with their defining row), clashing out-row cells (with reason and row)
      uint8_t* f_late = shf.as<uint8_t>();
      uint8_t* f_clash = f_late + m;
      k_solve_shuffle_flags<<<PB_GRID(m, 256), 0, st>>>(sideb.as<uint8_t>(), voc.as<uint32_t>(), inp.as<uint32_t>(),
                                                        defr.as<uint32_t>(), outc.as<uint32_t>(), n, p, f_late,
                                                        f_clash);
      launched(ctx);
      counts[2] = list_with_rows(f_late, a.lists + 3 * limit);
      counts[3] = list_cells(f_clash, a.lists + 5 * limit, 2, [&](const uint32_t* cells, uint32_t count, uint32_t* o) {
        k_solve_clash_reasons<<<PB_GRID(count, 128), 0, st>>>(cells, count, voc.as<uint32_t>(), inp.as<uint32_t>(),
                                                              defr.as<uint32_t>(), outc.as<uint32_t>(), p, o);
      });
    }
    return counts[0] || counts[1] || (sf && (counts[2] || counts[3]));
  }

  // the rows[0, count) through k_solve_eval, as many warps as fit on the device
  void evaluate(const uint32_t* rows, uint64_t count) {
    if (!count) return;
    const auto kernel = tb ? k_solve_eval<true> : k_solve_eval<false>;
    int per_sm = 0;
    PB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, 128, 0));
    const uint64_t warps = (count + 31) / 32;
    const uint64_t blocks = std::min<uint64_t>((uint64_t)std::max(per_sm, 1) * ctx->sm_count, (warps + 3) / 4);
    PB_CUDA(cudaMemsetAsync(small_u + 4, 0, 4, st));  // the ticket
    kernel<<<(unsigned)blocks, 128, 0, st>>>(s, rows, count, voc.as<uint32_t>(), val.as<Fr>(), ready.as<uint32_t>(),
                                             small_u + 4, lk);
    launched(ctx);
    uint32_t stalled = 0;
    PB_CUDA(cudaMemcpyAsync(&stalled, small_u + 5, 4, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    PB_CHECK(stalled == 0, "solving the wires stalled: a defining row waited too long for its operands");
  }

  // 3.-4. the defining rows in row order, evaluated: one phase, or with out-rows the defining rows below p (the
  // list's prefix idx[0, k_below)), the shuffle step and the rest
  void evaluate_all() {
    k_solve_init<<<PB_GRID(m, 256), 0, st>>>(inp.as<uint32_t>(), invals.as<Fr>(), m, val.as<Fr>(),
                                             ready.as<uint32_t>());
    launched(ctx);
    if (tb) {
      ix_word.alloc(tb->rows * 8);
      ix_row.alloc(tb->rows * 4);
      ix_amb.alloc(tb->rows);
      lk.T.word = ix_word.as<uint64_t>();
      lk.T.row = ix_row.as<uint32_t>();
      lk.T.amb = ix_amb.as<uint8_t>();
      solve_table_index(ctx, lk.T, tb->rows, temp, small_u + 6);
    }
    uint32_t* list = idx.as<uint32_t>();
    const uint8_t* def = defines.as<uint8_t>();
    const uint64_t k_below = out_rows ? compact_flagged(ctx, def, p, temp, list, num, 0, nullptr) : 0;
    const uint64_t n_def = compact_flagged(ctx, def, n, temp, list, num, 0, nullptr);
    if (!out_rows) {
      evaluate(list, n_def);
      return;
    }
    DevBuf rowl(2 * K * 4);  // the in-rows, then the out-rows, ascending
    const uint8_t* fl = sideb.as<uint8_t>() + n;
    const uint64_t got_in = compact_flagged(ctx, fl, n, temp, rowl.as<uint32_t>(), num, 0, nullptr);
    const uint64_t got_out = compact_flagged(ctx, fl + n, n, temp, rowl.as<uint32_t>() + K, num, 0, nullptr);
    PB_CHECK(got_in == K && got_out == K, "solving the wires: the shuffle's row lists disagree with q_in and q_out");
    cudaEvent_t ev[4];
    for (auto& e : ev) PB_CUDA(cudaEventCreate(&e));
    PB_CUDA(cudaEventRecord(ev[0], st));
    evaluate(list, k_below);
    PB_CUDA(cudaEventRecord(ev[1], st));
    solve_shuffle(ctx, rowl.as<uint32_t>(), rowl.as<uint32_t>() + K, K, voc.as<uint32_t>(), val.as<Fr>(),
                  ready.as<uint32_t>(), temp, reinterpret_cast<unsigned long long*>(small_u + 8));
    PB_CUDA(cudaEventRecord(ev[2], st));
    evaluate(list + k_below, n_def - k_below);
    PB_CUDA(cudaEventRecord(ev[3], st));
    PB_CUDA(cudaEventSynchronize(ev[3]));
    for (int k = 0; k < 3; k++) {
      float ms = 0;
      PB_CUDA(cudaEventElapsedTime(&ms, ev[k], ev[k + 1]));
      g_solve_ms[k] = ms;
    }
    for (auto& e : ev) PB_CUDA(cudaEventDestroy(e));
  }

  // with a table, the errors found while evaluating: miss and ambiguous rows, and the operands a, b of the listed
  // ones; true with any
  bool table_errors() {
    if (!tb) return false;
    const uint64_t limit = a.limit;
    uint64_t* counts = a.counts;
    uint32_t* l_miss = a.lists + 3 * limit;
    uint32_t* l_amb = l_miss + limit;
    counts[2] = compact_flagged(ctx, lk.miss, n, temp, idx.as<uint32_t>(), num, a.limit, l_miss);
    counts[3] = compact_flagged(ctx, lk.amb, n, temp, idx.as<uint32_t>(), num, a.limit, l_amb);
    const uint32_t take[2] = {(uint32_t)std::min<uint64_t>(counts[2], limit),
                              (uint32_t)std::min<uint64_t>(counts[3], limit)};
    if (tb->operands && take[0] + take[1]) {
      DevBuf lrows((size_t)(take[0] + take[1]) * 4), ops((size_t)(take[0] + take[1]) * 64);
      PB_CUDA(cudaMemcpyAsync(lrows.p, l_miss, (size_t)take[0] * 4, cudaMemcpyHostToDevice, st));
      PB_CUDA(cudaMemcpyAsync(lrows.as<uint32_t>() + take[0], l_amb, (size_t)take[1] * 4, cudaMemcpyHostToDevice, st));
      k_solve_operands<<<PB_GRID(take[0] + take[1], 128), 0, st>>>(lrows.as<uint32_t>(), take[0] + take[1],
                                                                   voc.as<uint32_t>(), val.as<Fr>(), ops.as<Fr>());
      launched(ctx);
      PB_CUDA(cudaMemcpyAsync(tb->operands, ops.p, (size_t)take[0] * 64, cudaMemcpyDeviceToHost, st));
      PB_CUDA(cudaMemcpyAsync(tb->operands + limit * 64, ops.as<uint8_t>() + (size_t)take[0] * 64,
                              (size_t)take[1] * 64, cudaMemcpyDeviceToHost, st));
      PB_CUDA(cudaStreamSynchronize(st));
    }
    return counts[2] || counts[3];
  }

  // 5. every cell's value into A, B, C
  void write() {
    DevBuf staging(a.out_on_device ? 0 : m * 32);
    Fr* W[3];
    for (int k = 0; k < 3; k++)
      W[k] = a.out_on_device ? reinterpret_cast<Fr*>(a.out[k]) : staging.as<Fr>() + (uint64_t)k * n;
    k_solve_write<<<PB_GRID(m, 256), 0, st>>>(voc.as<uint32_t>(), val.as<Fr>(), n, W[0], W[1], W[2]);
    launched(ctx);
    if (!a.out_on_device)
      for (int k = 0; k < 3; k++) PB_CUDA(cudaMemcpyAsync(a.out[k], W[k], n * 32, cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
  }
};
}  // namespace

// see plonk_b200.h: pb200_solve_wires, with `tb` pb200_solve_wires_lookup, with `sf` pb200_solve_wires_shuffle
void solve_run(Context* ctx, const SolveArgs& a, const SolveTableArgs* tb, const SolveShuffleArgs* sf) {
  Solve S(ctx, a, tb, sf);
  S.require();
  S.reserve();
  S.sources();
  if (!S.errors()) {
    S.evaluate_all();
    if (!S.table_errors()) S.write();
  }
  PB_CUDA(cudaStreamSynchronize(ctx->stream));  // the call's buffers die here
}

}  // namespace pb200
