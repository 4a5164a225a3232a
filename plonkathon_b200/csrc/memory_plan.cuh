// Device bytes of a single-GPU prover, by count, for its two round-3 layouts (DESIGN.md section 2):
//   full:   everything on the 4n-point coset stays resident -- the cached selector extensions, L0, the coset points,
//           the five per-proof extensions and the 4n quotient, and the 4n NTT plans;
//   sliced: round 3 walks the four n-point slices {g mu^(4j + r)} of that coset one after the other (prover.cu,
//           "sliced round 3"), so every coset vector is n long and the selector extensions are recomputed per slice.
// prover_create picks the full layout when it fits the free device memory less PB_PLAN_MARGIN, else the sliced one,
// else refuses before allocating anything.  Host code (exported by csrc/host_selftest.cpp for the CPU tests).
#pragma once
#include <stdint.h>

#include "curve.cuh"
#include "msm_sort.cuh"

namespace pb200 {

// left free for what the count leaves out: the CUDA context's own growth, allocation granules, the small tables
#define PB_PLAN_MARGIN (4ull << 30)

struct MemoryCount {
  uint64_t circuit = 0;  // per-circuit cache (prover creation)
  uint64_t proof = 0;    // per-proof vectors (also allocated at creation)
  uint64_t ntt = 0;      // NTT plans, the sharded-join tables and the pass buffer in the context
  uint64_t msm = 0;      // growth of the context's MSM scratch for commitments of n coefficients
  uint64_t total() const { return circuit + proof + ntt + msm; }
};
struct ProverMemory {
  MemoryCount full, sliced;
};

// twiddle tables of one NTT plan of 2^log_n points (ntt.cu build_plan): the inter-pass tables of the first pass (N
// elements) and, with three passes, of the second (N / N1)
inline uint64_t plan_ntt_bytes(int log_n) {
  const uint64_t N = (uint64_t)1 << log_n;
  if (log_n <= 11) return 0;
  if (log_n <= 22) return N * 32;
  const int lb0 = (log_n + 2) / 3;
  return N * 32 + (N >> lb0) * 32;
}

// msm_c, msm_batch: the window bits and the number of commitments of the largest MSM a proof makes (three, on the
// fixed-base table); msm_now: bytes the context's MSM scratch already holds
inline ProverMemory prover_memory(int log_n, int n_custom, uint32_t msm_c, uint32_t msm_batch, uint64_t msm_now) {
  const uint64_t n = (uint64_t)1 << log_n, E = n * 32;
  const uint64_t sel = 8 + (uint64_t)n_custom;
  ProverMemory m;
  // full: sel_coeff, sel_lag (n each), sel_ext (4n); L0 and the coset points (4n each); roots, gpow (n), ginv_pow (4n)
  m.full.circuit = (sel * 6 + 4 + 4 + 1 + 1 + 4) * E;
  // lag (4), coeff (5), pi_lag (1), tmp (5) n each; five extensions, the quotient and the side stream's pass buffer 4n
  m.full.proof = (4 + 5 + 1 + 5) * E + (5 + 1 + 1) * 4 * E;
  // forward and inverse plans at n and 4n, the context's pass buffer (4n)
  m.full.ntt = 2 * plan_ntt_bytes(log_n) + 2 * plan_ntt_bytes(log_n + 2) + 4 * E;
  // sliced: sel_coeff, sel_lag and one slice of every selector extension (n each); the slice's points, its L0, roots,
  // gpow (n); ginv_pow for T's 3n coefficients
  m.sliced.circuit = (sel * 3 + 1 + 1 + 1 + 1 + 3) * E;
  // lag, coeff, pi_lag, tmp as above; five slice extensions (n), the quotient's 3n coefficients and the four slots of
  // the join in the context (4n)
  m.sliced.proof = (4 + 5 + 1 + 5) * E + 5 * E + 3 * E + 4 * E;
  // plans at n only; the join's multiply-on-store table of each slice (n); the pass buffer (n)
  m.sliced.ntt = 2 * plan_ntt_bytes(log_n) + 4 * E + E;
  // the MSM scratch of msm.cu: per entry (n * windows * batch) a binned entry and a sorted position; per segment of 32
  // entries two XYZZ partial sums, three words and a 24-byte heavy item; per bucket an XYZZ sum, a count and an offset
  const uint64_t W = (256 + msm_c - 1) / msm_c;
  const uint64_t entries = n * W * msm_batch, buckets = (uint64_t)msm_batch << (msm_c - 1);
  const uint64_t msm = entries * (sizeof(SortEntry) + 4) + (entries / 32 + 1) * (2 * sizeof(G1XYZZ) + 12 + 24) +
                       buckets * (sizeof(G1XYZZ) + 8);
  m.full.msm = m.sliced.msm = msm > msm_now ? msm - msm_now : 0;
  return m;
}

// 0: full, 1: sliced, -1: neither fits.  force_sliced (PB200_SLICED=1) can only force slicing, never prevent it.
inline int plan_choose(const ProverMemory& m, uint64_t free_bytes, bool force_sliced) {
  const uint64_t avail = free_bytes > PB_PLAN_MARGIN ? free_bytes - PB_PLAN_MARGIN : 0;
  if (!force_sliced && m.full.total() <= avail) return 0;
  if (m.sliced.total() <= avail) return 1;
  return -1;
}

}  // namespace pb200
