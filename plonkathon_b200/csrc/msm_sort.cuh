// Counting sort of the MSM's bucket entries (msm.cu, steps 1-3): the thread bodies.
//
// Every non-zero digit of every scalar is an entry (bucket key, point index | sign << 31).  The sort leaves the
// entries of bucket b at sorted[offsets[b] .. offsets[b] + counts[b]) in any order, with offsets the exclusive
// prefix sum of the counts (padded to even with `pad`, as msm_bucket.cuh needs).
//
// It runs in two levels so that no step does a global atomic per entry or a store into a write front larger than L2:
//   1. the keys are cut into at most PB_SORT_MAX_BINS coarse bins of 2^lb consecutive keys each;
//      k_msm_bin_count:   a shared-memory histogram over the bins per block, one global atomic per non-empty
//                         (block, bin);
//      (k_scan_* over the bin counts: bin_off, bin cursors zeroed)
//      k_msm_bin_scatter: the block counts again, reserves one contiguous range per non-empty bin with one global
//                         atomic, sorts its {key, value} pairs by bin in shared memory and copies them out, so
//                         consecutive threads store to consecutive addresses of a bin's range;
//   2. every bin is cut into chunks of at most T entries (a chunk never crosses a bin boundary, so heavy bins --
//      the short top window, skewed scalars -- spread over many blocks);
//      k_msm_chunk_map:   exclusive scan of the chunks per bin (chunk -> bin lookup);
//      k_msm_chunk_count: a shared-memory histogram over the bin's 2^lb buckets per chunk, added into counts[]
//                         with one global atomic per non-empty (chunk, bucket);
//      (k_scan_* over the bucket counts, as before: offsets, padding, max count, counts zeroed)
//      k_msm_chunk_place: the chunk's histogram again, one range per non-empty (chunk, bucket) reserved with an
//                         atomic on the zeroed counts (which leaves them equal to the raw counts), the 4-byte values
//                         sorted by bucket in shared memory and copied out into the bin's window of the sorted array.
// Staging matters: storing every entry straight to its rank (one 4-8 byte store per lane, 32 different sectors per
// warp instruction) measured about twice as slow for these two kernels (H100 SXM, 400 W: 0.58 + 0.32 ms against
// 0.22 + 0.18 ms for one 2^20 fixed-base commitment).
// Each kernel's body is split into per-thread phases at its __syncthreads points and takes its shared memory as
// explicit pointers, so csrc/host_selftest.cpp runs a block as a loop over phases (tests/test_host_arith.py); the
// __global__ wrappers live in msm.cu.
#pragma once
#include "msm_digits.cuh"

namespace pb200 {

#define PB_SORT_MAX_BINS 2048      // bins of the first level (shared histogram of the bin kernels)
#define PB_SORT_MAX_BIN_KEYS 2048  // buckets per bin (shared histogram of the chunk kernels): nb <= 2^22
#define PB_SORT_BIN_THREADS 512
#define PB_SORT_BIN_STAGE 8192     // entries a bin-kernel block stages in shared memory (64 KB)
#define PB_SORT_CHUNK_THREADS 512
#define PB_SORT_CHUNK 16384        // entries per chunk (staged: 64 KB)
static_assert(PB_SORT_MAX_BINS <= 256 * 8, "k_msm_chunk_map and the bin scan take one block of 256 x 8 bins");

struct alignas(8) SortEntry {
  uint32_t key, val;
};

struct SortArgs {
  ScalarBatch sb;
  uint64_t n;
  int from_mont;
  MsmGeom g;
  uint32_t spb;             // scalars per bin-kernel block: PB_SORT_BIN_STAGE / W, so its entries fit the stage
  uint32_t lb;              // bin of key k: k >> lb
  uint32_t nbins;           // ((nb - 1) >> lb) + 1 <= PB_SORT_MAX_BINS
  uint32_t T;               // entries per chunk
  uint32_t* bin_cnt;        // nbins: entries per bin (zeroed by the bin scan, restored by k_msm_bin_scatter)
  const uint32_t* bin_off;  // nbins + 1: exclusive prefix of bin_cnt
  SortEntry* binned;        // the entries grouped by bin
  uint32_t* chunk_first;    // nbins + 1: first chunk of every bin; [nbins] = number of chunks
  uint32_t* counts;         // nb bucket counts (+ the max count at [nb])
  const uint32_t* offsets;  // nb + 1
  uint32_t* sorted;         // the entries grouped by bucket
};

// key bits per bin: the fewest that leave at most PB_SORT_MAX_BINS bins (max(0, ceil(log2 nb) - 11))
PB_HD uint32_t sort_default_lb(uint32_t nb) {
  uint32_t lb = 0;
  while (((nb - 1) >> lb) >= PB_SORT_MAX_BINS) lb++;
  return lb;
}

// atomicAdd on the device; the host harness runs one thread at a time
PB_HD uint32_t sort_add(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
  return atomicAdd(p, v);
#else
  const uint32_t o = *p;
  *p = o + v;
  return o;
#endif
}

PB_HD void sort_zero(uint32_t* sh, uint32_t len, uint32_t t, uint32_t nt) {
  for (uint32_t b = t; b < len; b += nt) sh[b] = 0;
}

// A block-wide exclusive scan of sh[0..len) is split around a scan of one value per thread (the device's block scan,
// a loop on the host): thread t owns the segment [t * per, t * per + per) and contributes its sum.
PB_HD uint32_t scan_part_sum(const uint32_t* sh, uint32_t len, uint32_t t, uint32_t nt) {
  const uint32_t per = (len + nt - 1) / nt;
  uint32_t s = 0;
  for (uint32_t b = t * per; b < t * per + per && b < len; b++) s += sh[b];
  return s;
}

// f(key, value) for every owned non-zero digit of the scalars that thread t of bin-kernel block bx (scalar vector
// k) walks: scalars [bx * spb, (bx + 1) * spb), thread t takes every nt-th (coalesced loads)
template <class F>
PB_HD void sort_walk(const SortArgs& a, uint32_t bx, uint32_t k, uint32_t t, uint32_t nt, F f) {
  const uint64_t end = (uint64_t)(bx + 1) * a.spb < a.n ? (uint64_t)(bx + 1) * a.spb : a.n;
  for (uint64_t i = (uint64_t)bx * a.spb + t; i < end; i += nt) {
    DigitWalk dw(a.sb.p[k], i, a.from_mont);
    for (uint32_t w = 0; w < a.g.W; w++) {
      uint32_t neg, d = dw.next(w, a.g, neg);
      if (!d) continue;
      const uint32_t key = msm_bucket_key(a.g, k, w, d);
      if (key != 0xffffffffu) f(key, (uint32_t)((uint64_t)w * a.g.point_stride + i) | (neg << 31));
    }
  }
}

// ---- level 1: bins ------------------------------------------------------------------------------------------
// k_msm_bin_count and k_msm_bin_scatter, phase 1 (after sort_zero of sh_cnt): entries per bin of the block
PB_HD void bin_hist(const SortArgs& a, uint32_t bx, uint32_t k, uint32_t t, uint32_t nt, uint32_t* sh_cnt) {
  sort_walk(a, bx, k, t, nt, [&](uint32_t key, uint32_t) { sort_add(&sh_cnt[key >> a.lb], 1u); });
}

// k_msm_bin_count, phase 2: one global atomic per non-empty bin
PB_HD void bin_flush(const SortArgs& a, uint32_t t, uint32_t nt, const uint32_t* sh_cnt) {
  for (uint32_t b = t; b < a.nbins; b += nt)
    if (sh_cnt[b]) sort_add(&a.bin_cnt[b], sh_cnt[b]);
}

// k_msm_bin_scatter, phase 2 (run = block-wide exclusive prefix of the scan_part_sum of sh_cnt): the bins' offsets
// in the block's stage, and the block's range of every non-empty bin in `binned` reserved; the counters restart as
// cursors
PB_HD void bin_reserve(const SortArgs& a, uint32_t t, uint32_t nt, uint32_t run, uint32_t* sh_cnt, uint32_t* sh_loc,
                       uint32_t* sh_base) {
  const uint32_t per = (a.nbins + nt - 1) / nt;
  for (uint32_t b = t * per; b < t * per + per && b < a.nbins; b++) {
    const uint32_t c = sh_cnt[b];
    sh_loc[b] = run;
    run += c;
    if (c) sh_base[b] = a.bin_off[b] + sort_add(&a.bin_cnt[b], c);
    sh_cnt[b] = 0;
  }
}

// k_msm_bin_scatter, phase 3: the same walk again, the entries sorted by bin into the stage
PB_HD void bin_stage(const SortArgs& a, uint32_t bx, uint32_t k, uint32_t t, uint32_t nt, uint32_t* sh_cnt,
                     const uint32_t* sh_loc, SortEntry* stage) {
  sort_walk(a, bx, k, t, nt, [&](uint32_t key, uint32_t val) {
    const uint32_t b = key >> a.lb;
    SortEntry e;
    e.key = key;
    e.val = val;
    stage[sh_loc[b] + sort_add(&sh_cnt[b], 1u)] = e;
  });
}

// k_msm_bin_scatter, phase 4: the stage copied out, consecutive threads to consecutive positions of a bin's range
PB_HD void bin_copy_out(const SortArgs& a, uint32_t t, uint32_t nt, uint32_t total, const uint32_t* sh_loc,
                        const uint32_t* sh_base, const SortEntry* stage) {
  for (uint32_t p = t; p < total; p += nt) {
    const SortEntry e = stage[p];
    const uint32_t b = e.key >> a.lb;
    a.binned[sh_base[b] + p - sh_loc[b]] = e;
  }
}

// ---- chunk map (k_msm_chunk_map: one block of 256 threads, 8 bins each, a block scan in between) --------------
PB_HD uint32_t chunk_map_sum(const SortArgs& a, uint32_t t) {
  uint32_t s = 0;
  for (uint32_t b = 8 * t; b < 8 * t + 8 && b < a.nbins; b++) s += (a.bin_cnt[b] + a.T - 1) / a.T;
  return s;
}
PB_HD void chunk_map_write(const SortArgs& a, uint32_t t, uint32_t run, uint32_t total) {
  for (uint32_t b = 8 * t; b < 8 * t + 8 && b < a.nbins; b++) {
    a.chunk_first[b] = run;
    run += (a.bin_cnt[b] + a.T - 1) / a.T;
  }
  if (t == 0) a.chunk_first[a.nbins] = total;
}

// ---- level 2: chunks of one bin -----------------------------------------------------------------------------
struct SortChunk {
  uint32_t lo, hi;     // entry range in `binned`
  uint32_t key0, nkeys;  // the bin's keys [key0, key0 + nkeys)
};

// chunk c (the kernels walk the chunks grid-stride); false past the last chunk
PB_HD bool chunk_locate(const SortArgs& a, uint32_t c, SortChunk& ch) {
  if (c >= a.chunk_first[a.nbins]) return false;
  uint32_t l = 0, h = a.nbins;  // first bin whose first chunk is past c, minus one: c's bin (never an empty one)
  while (l < h) {
    const uint32_t m = (l + h) >> 1;
    if (a.chunk_first[m] > c) h = m; else l = m + 1;
  }
  const uint32_t b = l - 1;
  ch.lo = a.bin_off[b] + (c - a.chunk_first[b]) * a.T;
  ch.hi = a.bin_off[b + 1] - ch.lo > a.T ? ch.lo + a.T : a.bin_off[b + 1];
  ch.key0 = b << a.lb;
  ch.nkeys = a.g.nb - ch.key0 < (1u << a.lb) ? a.g.nb - ch.key0 : 1u << a.lb;  // the last bin may be partial
  return true;
}

// k_msm_chunk_count and k_msm_chunk_place, phase 1 (after sort_zero of sh_cnt): entries per bucket of the chunk
PB_HD void chunk_hist(const SortArgs& a, const SortChunk& ch, uint32_t t, uint32_t nt, uint32_t* sh_cnt) {
  for (uint32_t i = ch.lo + t; i < ch.hi; i += nt) sort_add(&sh_cnt[a.binned[i].key - ch.key0], 1u);
}

// k_msm_chunk_count, phase 2: one global atomic per non-empty bucket
PB_HD void chunk_flush(const SortArgs& a, const SortChunk& ch, uint32_t t, uint32_t nt, const uint32_t* sh_cnt) {
  for (uint32_t l = t; l < ch.nkeys; l += nt)
    if (sh_cnt[l]) sort_add(&a.counts[ch.key0 + l], sh_cnt[l]);
}

// k_msm_chunk_place, phase 2 (run = block-wide exclusive prefix of the scan_part_sum of sh_cnt): the buckets'
// offsets in the chunk's stage, and the chunk's range of every non-empty bucket reserved with an atomic on the zeroed
// counts; the counters restart as cursors
PB_HD void chunk_reserve(const SortArgs& a, const SortChunk& ch, uint32_t t, uint32_t nt, uint32_t run,
                         uint32_t* sh_cnt, uint32_t* sh_loc, uint32_t* sh_base) {
  const uint32_t per = (ch.nkeys + nt - 1) / nt;
  for (uint32_t l = t * per; l < t * per + per && l < ch.nkeys; l++) {
    const uint32_t c = sh_cnt[l];
    sh_loc[l] = run;
    run += c;
    if (c) sh_base[l] = a.offsets[ch.key0 + l] + sort_add(&a.counts[ch.key0 + l], c);
    sh_cnt[l] = 0;
  }
}

// k_msm_chunk_place, phase 3: the values sorted by bucket into the stage
PB_HD void chunk_stage(const SortArgs& a, const SortChunk& ch, uint32_t t, uint32_t nt, uint32_t* sh_cnt,
                       const uint32_t* sh_loc, uint32_t* stage) {
  for (uint32_t i = ch.lo + t; i < ch.hi; i += nt) {
    const SortEntry e = a.binned[i];
    const uint32_t l = e.key - ch.key0;
    stage[sh_loc[l] + sort_add(&sh_cnt[l], 1u)] = e.val;
  }
}

// k_msm_chunk_place, phase 4: the stage copied out, consecutive threads to consecutive positions of a bucket's range
// (the bucket of stage position p: the last one whose stage offset is <= p, never an empty one)
PB_HD void chunk_copy_out(const SortArgs& a, const SortChunk& ch, uint32_t t, uint32_t nt, const uint32_t* sh_loc,
                          const uint32_t* sh_base, const uint32_t* stage) {
  for (uint32_t p = t; p < ch.hi - ch.lo; p += nt) {
    uint32_t lo = 0, hi = ch.nkeys;
    while (lo < hi) {
      const uint32_t m = (lo + hi) >> 1;
      if (sh_loc[m] > p) hi = m; else lo = m + 1;
    }
    a.sorted[sh_base[lo - 1] + p - sh_loc[lo - 1]] = stage[p];
  }
}

}  // namespace pb200
