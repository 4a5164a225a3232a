// Copy-constraint permutation S1, S2, S3 from a circuit's wiring (compiler/program.py:70-113, restated by
// synthetic.permutation_polys): the key packing, the host-side id check and the per-position body of the label
// kernel.  permutation.cu runs them on the GPU; csrc/host_selftest.cpp runs the same bodies on the CPU.
//
// Cell (row, col), col 0/1/2 for L/R/O, is cell = 3 row + col and carries a variable id, -1 for "no variable".  The
// cells of one id form a cycle in cell order; every cell stores the label omega^row' (col' + 1) of the previous cell
// of its cycle, the first cell that of the last.  All -1 cells form one more cycle.
//
// Each cell becomes one 64-bit key (id + 1) << cb | cell, cb = log_n + 2 = ceil(log2(3n)).  The keys are distinct, so
// after any correct sort a group's cells are consecutive and in cell order, which is exactly the cycle order.
#pragma once
#include "field.cuh"

namespace pb200 {

#define PB_PERM_MAX_ID 0xfffffffeLL  // largest wire variable id: id + 1 takes 32 bits of the key

PB_HD int perm_cell_bits(int log_n) { return log_n + 2; }
PB_HD uint64_t perm_key(int64_t id, uint64_t cell, int cb) { return ((uint64_t)(id + 1) << cb) | cell; }

// index of the first id outside [-1, PB_PERM_MAX_ID], or -1 when there is none; *max_id: the largest id
inline int64_t perm_check_ids(const int64_t* ids, uint64_t m, int64_t* max_id) {
  int64_t mx = -1;
  for (uint64_t k = 0; k < m; k++) {
    if (ids[k] < -1 || ids[k] > PB_PERM_MAX_ID) return (int64_t)k;
    mx = ids[k] > mx ? ids[k] : mx;
  }
  *max_id = mx;
  return -1;
}

// key bits the sort has to look at: the cell bits and the bits of the largest id + 1
inline int perm_sort_bits(int log_n, int64_t max_id) {
  int b = perm_cell_bits(log_n);
  for (uint64_t v = (uint64_t)(max_id + 1); v; v >>= 1) b++;
  return b;
}

struct PermArgs {
  const uint64_t* keys;  // the 3n keys, sorted
  const Fr* wpow;        // omega^row for row < n, canonical
  Fr* S;                 // S1 | S2 | S3, n values each, canonical
  uint64_t n;
  uint64_t m;            // 3n
  int cb;
};

// Sorted position of the last key of the group `g` that starts at position `first`: doubling steps from `first`
// until a key leaves the group, then bisection.  log2 of the group's size in reads, so the short cycles of a real
// circuit cost a few reads and the one large "no variable" group at most 2 log2(3n).
PB_HD uint64_t perm_group_last(const PermArgs& a, uint64_t first, uint64_t g) {
  uint64_t lo = first, hi, step = 1;
  for (;;) {
    hi = lo + step;
    if (hi >= a.m) { hi = a.m; break; }
    if ((a.keys[hi] >> a.cb) != g) break;
    lo = hi;
    step <<= 1;
  }
  while (hi - lo > 1) {  // keys[lo] is in the group, keys[hi] (or the end) is not
    const uint64_t mid = lo + (hi - lo) / 2;
    if ((a.keys[mid] >> a.cb) == g) lo = mid;
    else hi = mid;
  }
  return lo;
}

// Sorted position k: the label of the previous key of its group (of the group's last key at its first position),
// stored at S[col][row] of k's own cell.
PB_HD void perm_label(const PermArgs& a, uint64_t k) {
  const uint64_t key = a.keys[k], g = key >> a.cb, mask = ((uint64_t)1 << a.cb) - 1;
  uint64_t prev;
  if (k > 0 && (a.keys[k - 1] >> a.cb) == g) prev = a.keys[k - 1];
  else prev = a.keys[perm_group_last(a, k, g)];
  const uint32_t cell = (uint32_t)(key & mask), pcell = (uint32_t)(prev & mask);  // 3n <= 3 * 2^26
  const uint32_t row = cell / 3, col = cell - 3 * row, prow = pcell / 3, pcol = pcell - 3 * prow;
  const Fr w = a.wpow[prow];
  Fr x = w;  // omega^prow (pcol + 1): sums of canonical values stay canonical
  if (pcol >= 1) x = fp_add(x, w);
  if (pcol == 2) x = fp_add(x, w);
  a.S[col * a.n + row] = x;
}

}  // namespace pb200
