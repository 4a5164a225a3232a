// G1 multi-scalar multiplication (Pippenger / bucket method) for sm_90a.
//
// Replaces curve.py:38-111 (`ec_lincomb` -> `lincomb` -> `multisubset`) and the MSM half of
// setup.py:66-72 (`Setup.commit`).  The result sum_i s_i * P_i is algorithm-independent, so the
// reference's bit-sliced power-set method is replaced by:
//   1. signed-digit window slicing of every scalar (c-bit windows, digits in [-2^(c-1), 2^(c-1)]), with
//      per-block shared-memory histograms over coarse bins of buckets, and their scan  (k_msm_bin_count, k_scan_*)
//   2. scatter of (bucket, point index | sign) into the bins                     (k_msm_bin_scatter)
//   3. counting sort of every bin by bucket, in chunks: shared-memory histograms added into the bucket counts,
//      exclusive scan, placement           (k_msm_chunk_map, k_msm_chunk_count, k_scan_*, k_msm_chunk_place)
//      No step does a global atomic per entry or stores into a write front larger than L2 (msm_sort.cuh).
//   4. load-balanced bucket accumulation over fixed segments of the sorted entries: XYZZ accumulator += affine
//      point (8M+2S, no inversion), SIMT-uniform loop                            (k_msm_seg_accumulate)
//      + stitching of buckets that cross a segment boundary, block trees for heavy ones, piece-wise for buckets of
//      more than 1024 segments                                                   (k_msm_stitch[_pieces|_heavy])
//      [A/B alternative, PB200_MSM_ACC=affine: rounds of pairwise batched-affine additions, one safegcd inversion
//       per thread and round, 6 products per addition -- measured slower        (k_aff_round0 / k_aff_round / k_aff_tail)]
//   5. bucket reduction sum_b (b+1) * B_b by recursive grouping: running sums over 16 buckets per thread, then
//      block-wide suffix-scan levels over 512 elements                           (k_reduce_level0 / k_reduce_block)
//   6. the few remaining group operations (last <= 8 reduction pairs, bucket-range offset or the join of the ranks'
//      shares, window Horner, one inversion to affine) on the host, which has to read the point anyway to feed the
//      Fiat-Shamir transcript.
// Streams: steps 1-3, the stitch of step 4 and the upper levels of step 5 run on the context's high-priority stream,
// the accumulation and reduction level 0 on its main stream, joined by events, so the order of work is unchanged.
// With two contexts proving at once, the blocks of these short phases then take the SM slots that the other
// context's retiring accumulation blocks free, instead of waiting for its whole grid to drain (traces before and
// after, and what they gained: DESIGN.md section 5, profiles/h100_inflight_trace.md).  A retiring accumulation block
// frees 128 x 128 = 16,384 registers and no shared memory.  The bin kernels are held to 32 registers at 512 threads
// and the stitch kernels to 128 at 128 threads so that one block fits there.  k_reduce_block (168 registers at 128
// threads) needs the slots of two: capped at 128 registers it spills 224 bytes per thread in its chains of dependent
// additions, so it is left as it is.
// Multi-GPU: a call may own a sub-range of the buckets of every bucket set -- contiguous [bucket_lo, bucket_hi), or,
// with a communicator, every G-th bucket -- it walks all digits but sorts, accumulates and reduces only its own
// buckets, so the whole MSM (not just the accumulation) divides by the number of ranks; and/or a POINT RANGE (a
// sub-vector of the points).  It then returns partial sums; with a communicator the (S, R) pairs of the ranks are
// exchanged with one allgather and every rank returns the full result.
// Two modes: "generic" (arbitrary points: W windows x 2^(c-1) buckets) and "fixed-base" (SRS with the
// window multiples 2^(c*w) * P_i precomputed in HBM: one shared set of 2^(c-1) buckets, no Horner).
#include <algorithm>
#include <cstring>

#include "common.cuh"
#include "comm.cuh"
#include "msm_bucket.cuh"
#include "msm_digits.cuh"
#include "msm_sort.cuh"

namespace pb200 {

// ------------------------------------------------------------------------------------------
__device__ __forceinline__ G1Affine ld_affine(const G1Affine* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
  G1Affine r;
  r.x.v[0] = a.x; r.x.v[1] = a.y; r.x.v[2] = a.z; r.x.v[3] = a.w;
  r.x.v[4] = b.x; r.x.v[5] = b.y; r.x.v[6] = b.z; r.x.v[7] = b.w;
  r.y.v[0] = c.x; r.y.v[1] = c.y; r.y.v[2] = c.z; r.y.v[3] = c.w;
  r.y.v[4] = d.x; r.y.v[5] = d.y; r.y.v[6] = d.z; r.y.v[7] = d.w;
  return r;
}

// exclusive prefix of v across the block (a multiple of 32 threads, at most 1024), *total = block sum;
// sh: one word per warp
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* sh, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t x = v;
  for (int d = 1; d < 32; d <<= 1) {
    uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if ((int)lane >= d) x += y;
  }
  if (lane == 31) sh[wid] = x;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = lane < nw ? sh[lane] : 0;
    for (int d = 1; d < 32; d <<= 1) {
      uint32_t y = __shfl_up_sync(0xffffffffu, w, d);
      if ((int)lane >= d) w += y;
    }
    if (lane < nw) sh[lane] = w;  // inclusive warp totals
  }
  __syncthreads();
  uint32_t base = wid ? sh[wid - 1] : 0;
  *total = sh[nw - 1];
  __syncthreads();
  return base + x - v;
}

// ---- two-level counting sort of the bucket entries (msm_sort.cuh holds the thread bodies) -----------------------
__global__ void __launch_bounds__(PB_SORT_BIN_THREADS, 4) k_msm_bin_count(SortArgs a) {
  __shared__ uint32_t sh_cnt[PB_SORT_MAX_BINS];
  const uint32_t t = threadIdx.x, nt = blockDim.x;
  sort_zero(sh_cnt, a.nbins, t, nt);
  __syncthreads();
  bin_hist(a, blockIdx.x, blockIdx.y, t, nt, sh_cnt);
  __syncthreads();
  bin_flush(a, t, nt, sh_cnt);
}

// dynamic shared memory: the stage, PB_SORT_BIN_STAGE entries
__global__ void __launch_bounds__(PB_SORT_BIN_THREADS, 4) k_msm_bin_scatter(SortArgs a) {
  __shared__ uint32_t sh_cnt[PB_SORT_MAX_BINS], sh_loc[PB_SORT_MAX_BINS], sh_base[PB_SORT_MAX_BINS], sh_scan[32];
  extern __shared__ SortEntry stage[];
  const uint32_t t = threadIdx.x, nt = blockDim.x;
  sort_zero(sh_cnt, a.nbins, t, nt);
  __syncthreads();
  bin_hist(a, blockIdx.x, blockIdx.y, t, nt, sh_cnt);
  __syncthreads();
  uint32_t total;
  const uint32_t run = block_exclusive_scan(scan_part_sum(sh_cnt, a.nbins, t, nt), sh_scan, &total);
  bin_reserve(a, t, nt, run, sh_cnt, sh_loc, sh_base);
  __syncthreads();
  bin_stage(a, blockIdx.x, blockIdx.y, t, nt, sh_cnt, sh_loc, stage);
  __syncthreads();
  bin_copy_out(a, t, nt, total, sh_loc, sh_base, stage);
}

__global__ void __launch_bounds__(PB_SORT_CHUNK_THREADS) k_msm_chunk_count(SortArgs a) {
  __shared__ uint32_t sh_cnt[PB_SORT_MAX_BIN_KEYS];
  const uint32_t t = threadIdx.x, nt = blockDim.x;
  SortChunk ch;
  for (uint32_t c = blockIdx.x; chunk_locate(a, c, ch); c += gridDim.x) {
    sort_zero(sh_cnt, ch.nkeys, t, nt);
    __syncthreads();
    chunk_hist(a, ch, t, nt, sh_cnt);
    __syncthreads();
    chunk_flush(a, ch, t, nt, sh_cnt);
    __syncthreads();
  }
}

// dynamic shared memory: the stage, PB_SORT_CHUNK values
__global__ void __launch_bounds__(PB_SORT_CHUNK_THREADS) k_msm_chunk_place(SortArgs a) {
  __shared__ uint32_t sh_cnt[PB_SORT_MAX_BIN_KEYS], sh_loc[PB_SORT_MAX_BIN_KEYS], sh_base[PB_SORT_MAX_BIN_KEYS],
      sh_scan[32];
  extern __shared__ uint32_t stage_vals[];
  const uint32_t t = threadIdx.x, nt = blockDim.x;
  SortChunk ch;
  for (uint32_t c = blockIdx.x; chunk_locate(a, c, ch); c += gridDim.x) {
    sort_zero(sh_cnt, ch.nkeys, t, nt);
    __syncthreads();
    chunk_hist(a, ch, t, nt, sh_cnt);
    __syncthreads();
    uint32_t total;
    const uint32_t run = block_exclusive_scan(scan_part_sum(sh_cnt, ch.nkeys, t, nt), sh_scan, &total);
    chunk_reserve(a, ch, t, nt, run, sh_cnt, sh_loc, sh_base);
    __syncthreads();
    chunk_stage(a, ch, t, nt, sh_cnt, sh_loc, stage_vals);
    __syncthreads();
    chunk_copy_out(a, ch, t, nt, sh_loc, sh_base, stage_vals);
    __syncthreads();
  }
}

// ---- exclusive scan of a count array (3 small kernels): the bins and the buckets of the sort ---------------------
// offsets[0..nb] from counts[0..nb-1]; counts are zeroed on the way out (reused as cursors by the next placement
// kernel, which leaves them equal to the counts again).  pad != 0 rounds every count up to even, so all offsets are
// even (the slot layout of msm_bucket.cuh).
#define PB_SCAN_TILE 2048  // entries per block (256 threads x 8)

__global__ void __launch_bounds__(256) k_scan_tile_sums(const uint32_t* counts, uint32_t nb, uint32_t pad,
                                                        uint32_t* tile_sums, uint32_t* max_out) {
  __shared__ uint32_t sh[8];
  uint32_t base = blockIdx.x * PB_SCAN_TILE + threadIdx.x * 8;
  uint32_t s = 0, m = 0;
  for (int k = 0; k < 8; k++)
    if (base + k < nb) {
      uint32_t c = counts[base + k];
      m = max(m, c);
      s += (c + pad) & ~pad;
    }
  uint32_t total;
  block_exclusive_scan(s, sh, &total);
  if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
  if (max_out) {  // largest bucket of the launch (decides how many accumulation rounds do work)
    for (int d = 16; d > 0; d >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(max_out, m);
  }
}

// single block: exclusive scan of up to 256*32 tile sums in place; writes the grand total to *total_out
__global__ void __launch_bounds__(256) k_scan_tiles(uint32_t* tile_sums, uint32_t n_tiles, uint32_t* total_out) {
  __shared__ uint32_t sh[8];
  uint32_t per = (n_tiles + 255) / 256;
  uint32_t lo = threadIdx.x * per, hi = min(lo + per, n_tiles);
  uint32_t s = 0;
  for (uint32_t i = lo; i < hi; i++) s += tile_sums[i];
  uint32_t total;
  uint32_t run = block_exclusive_scan(s, sh, &total);
  for (uint32_t i = lo; i < hi; i++) {
    uint32_t c = tile_sums[i];
    tile_sums[i] = run;
    run += c;
  }
  if (threadIdx.x == 0) *total_out = total;
}

__global__ void __launch_bounds__(256) k_scan_apply(uint32_t* counts, uint32_t nb, uint32_t pad, const uint32_t* tile_sums,
                                                    uint32_t* offsets) {
  __shared__ uint32_t sh[8];
  uint32_t base = blockIdx.x * PB_SCAN_TILE + threadIdx.x * 8;
  uint32_t c[8];
  uint32_t s = 0;
  for (int k = 0; k < 8; k++) { c[k] = base + k < nb ? (counts[base + k] + pad) & ~pad : 0; s += c[k]; }
  uint32_t total;
  uint32_t run = tile_sums[blockIdx.x] + block_exclusive_scan(s, sh, &total);
  for (int k = 0; k < 8; k++) {
    if (base + k < nb) { offsets[base + k] = run; counts[base + k] = 0; }
    run += c[k];
  }
}

// one block: the first chunk of every bin (at most 256 x 8 = PB_SORT_MAX_BINS bins)
__global__ void __launch_bounds__(256) k_msm_chunk_map(SortArgs a) {
  __shared__ uint32_t sh[8];
  uint32_t total;
  const uint32_t run = block_exclusive_scan(chunk_map_sum(a, threadIdx.x), sh, &total);
  chunk_map_write(a, threadIdx.x, run, total);
}

// ---- batched-affine bucket accumulation (msm_bucket.cuh holds the thread bodies) -----------------------------
__global__ void __launch_bounds__(128, 4) k_aff_round0(AffAcc a) {
  Fq pref[PB_AFF_BMAX];
  uint32_t desc[PB_AFF_BMAX];
  aff_round0_thread(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, pref, desc);
}
__global__ void __launch_bounds__(128, 4) k_aff_round(AffAcc a) {
  Fq pref[PB_AFF_BMAX];
  uint32_t desc[PB_AFF_BMAX];
  aff_round_thread(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, pref, desc);
}
// rounds PB_AFF_GRID_ROUNDS.. of buckets with more than 2^PB_AFF_GRID_ROUNDS entries (skewed scalars only): one
// block walks the remaining rounds with a barrier in between; returns at once in the common case
__global__ void __launch_bounds__(256) k_aff_tail(AffAcc a, uint64_t s_bound) {
  Fq pref[PB_AFF_BMAX];
  uint32_t desc[PB_AFF_BMAX];
  const uint32_t maxc = *a.max_cnt;
  for (uint32_t r = PB_AFF_GRID_ROUNDS; r < 32 && maxc > (1u << r); r++) {
    a.r = r;
    const uint64_t T = aff_round_threads(s_bound, a.B, r);
    for (uint64_t t = threadIdx.x; t < T; t += blockDim.x) aff_round_thread(a, t, pref, desc);
    __syncthreads();
  }
}

// ---- A/B alternative: load-balanced XYZZ accumulation --------------------------------------------------------
// The sorted entry array (unpadded offsets) is cut into fixed segments of L entries, one thread each, so every
// thread does the same number of mixed additions no matter how skewed the bucket loads are.  A bucket that lies
// inside one segment is written directly.  A bucket that crosses a segment boundary leaves partial sums in two
// slots per segment (slot 2t: the segment's first run, slot 2t+1: its last run); the segment in which the bucket
// starts "owns" it and stitches the partials together afterwards: by itself when few segments are involved,
// through a block-wide tree for heavy buckets.
#define PB_MSM_EMPTY 0xffffffffu

__device__ __forceinline__ uint32_t upper_bound_u32(const uint32_t* a, uint32_t n, uint32_t key) {
  // first index i in [0, n) with a[i] > key (n if none)
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    if (__ldg(a + mid) > key) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// (128, 4): at most 128 registers, so 4 blocks fit an SM; unbounded, ptxas takes 134 and only 3 fit
__global__ void __launch_bounds__(128, 4) k_msm_seg_accumulate(const G1Affine* points, const uint32_t* offsets,
                                                            const uint32_t* sorted, uint32_t nb, uint32_t L,
                                                            G1XYZZ* buckets, G1XYZZ* slots, uint32_t* slot_bucket,
                                                            uint32_t* own_slot) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t M = offsets[nb];
  const uint64_t s64 = (uint64_t)t * L;
  if (s64 >= M) return;
  const uint32_t s = (uint32_t)s64;
  const uint32_t e = (uint32_t)min((uint64_t)M, s64 + L);
  uint32_t b = upper_bound_u32(offsets, nb + 1, s) - 1;  // offsets[b] <= s < offsets[b+1]
  uint32_t bstart = offsets[b], bend = offsets[b + 1];
  bool first = true;
  G1XYZZ acc = G1XYZZ::identity();
  // one flat loop over the segment: every lane does one mixed addition per iteration (uniform control
  // flow); run boundaries only cost a short predicated flush
  for (uint32_t pos = s; pos <= e; pos++) {
    if (pos == bend || pos == e) {
      if (bstart >= s && bend <= e) {
        buckets[b] = acc;
      } else {
        uint32_t slot = first ? 2 * t : 2 * t + 1;
        slots[slot] = acc;
        slot_bucket[slot] = b;
        if (bstart >= s) own_slot[t] = slot;  // the bucket starts here and continues past e
      }
      if (pos == e) break;
      first = false;
      acc = G1XYZZ::identity();
      b++;
      while (offsets[b + 1] <= pos) b++;  // skip empty buckets
      bstart = offsets[b];
      bend = offsets[b + 1];
    }
    uint32_t v = __ldg(sorted + pos);
    G1Affine p = ld_affine(points + (v & 0x7fffffffu));
    if (v >> 31) p.y = fp_neg(p.y);
    g1_add_mixed_uniform(acc, p);
  }
}

struct HeavyItem { uint32_t bucket, own_slot, t0, t1, piece_base, pieces; };
struct HeavyPiece { uint32_t item, index; };
#define PB_STITCH_PIECE 1024  // segments per piece of a very heavy bucket (a short top window puts n / 4 entries in one)

// one thread per segment: if it owns a boundary-crossing bucket, stitch it (or queue it as heavy; a bucket that
// spans more than PB_STITCH_PIECE segments is also cut into pieces that k_msm_stitch_pieces sums block by block)
__global__ void __launch_bounds__(128, 4) k_msm_stitch(const uint32_t* offsets, uint32_t nb, uint32_t L,
                                                    uint32_t n_segments, const G1XYZZ* slots,
                                                    const uint32_t* slot_bucket, const uint32_t* own_slot,
                                                    G1XYZZ* buckets, HeavyItem* heavy, uint32_t* heavy_count,
                                                    HeavyPiece* pieces, uint32_t small_limit) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_segments) return;
  const uint32_t os = own_slot[t];
  if (os == PB_MSM_EMPTY) return;
  const uint32_t b = slot_bucket[os];
  const uint32_t t1 = (offsets[b + 1] - 1) / L;  // last segment the bucket reaches
  if (t1 - t > small_limit) {
    uint32_t h = atomicAdd(heavy_count, 1u);
    HeavyItem it; it.bucket = b; it.own_slot = os; it.t0 = t; it.t1 = t1; it.piece_base = 0; it.pieces = 0;
    if (t1 - t > PB_STITCH_PIECE) {
      it.pieces = (t1 - t + PB_STITCH_PIECE - 1) / PB_STITCH_PIECE;
      it.piece_base = atomicAdd(heavy_count + 1, it.pieces);
      for (uint32_t p = 0; p < it.pieces; p++) { HeavyPiece hp; hp.item = h; hp.index = p; pieces[it.piece_base + p] = hp; }
    }
    heavy[h] = it;
    return;
  }
  G1XYZZ acc = slots[os];
  for (uint32_t k = t + 1; k <= t1; k++) {
    G1XYZZ piece = slots[2 * k];
    g1_add(acc, piece);
  }
  buckets[b] = acc;
}

// block-wide sum of one G1XYZZ per thread (128 threads); result in sh[0]
__device__ __forceinline__ void block_sum_xyzz(G1XYZZ* sh, const G1XYZZ& mine) {
  sh[threadIdx.x] = mine;
  __syncthreads();
  for (uint32_t d = blockDim.x >> 1; d > 0; d >>= 1) {
    if (threadIdx.x < d) {
      G1XYZZ a = sh[threadIdx.x], c = sh[threadIdx.x + d];
      g1_add(a, c);
      sh[threadIdx.x] = a;
    }
    __syncthreads();
  }
}

// pieces of very heavy buckets: one block each (grid-stride over the piece list): partial[p] = sum of the first-run
// slots of the piece's segments
__global__ void __launch_bounds__(128, 4) k_msm_stitch_pieces(const G1XYZZ* slots, const HeavyItem* heavy,
                                                           const uint32_t* heavy_count, const HeavyPiece* pieces,
                                                           G1XYZZ* partial) {
  __shared__ G1XYZZ sh[128];
  const uint32_t count = heavy_count[1];
  for (uint32_t p = blockIdx.x; p < count; p += gridDim.x) {
    const HeavyPiece hp = pieces[p];
    const HeavyItem it = heavy[hp.item];
    const uint32_t lo = it.t0 + 1 + hp.index * PB_STITCH_PIECE;
    const uint32_t hi = min(lo + PB_STITCH_PIECE - 1, it.t1);
    G1XYZZ acc = G1XYZZ::identity();
    for (uint32_t k = lo + threadIdx.x; k <= hi; k += blockDim.x) {
      G1XYZZ piece = slots[2 * k];
      g1_add(acc, piece);
    }
    block_sum_xyzz(sh, acc);
    if (threadIdx.x == 0) partial[p] = sh[0];
    __syncthreads();
  }
}

// heavy buckets: one block each (grid-stride over the queue), strided partial sums + shared-memory tree
__global__ void __launch_bounds__(128, 4) k_msm_stitch_heavy(const G1XYZZ* slots, const HeavyItem* heavy,
                                                          const uint32_t* heavy_count, const G1XYZZ* partial,
                                                          G1XYZZ* buckets) {
  __shared__ G1XYZZ sh[128];
  const uint32_t count = *heavy_count;
  for (uint32_t h = blockIdx.x; h < count; h += gridDim.x) {
    HeavyItem it = heavy[h];
    G1XYZZ acc = G1XYZZ::identity();
    if (threadIdx.x == 0) acc = slots[it.own_slot];
    if (it.pieces) {
      for (uint32_t p = threadIdx.x; p < it.pieces; p += blockDim.x) {
        G1XYZZ piece = partial[it.piece_base + p];
        g1_add(acc, piece);
      }
    } else {
      for (uint32_t k = it.t0 + 1 + threadIdx.x; k <= it.t1; k += blockDim.x) {
        G1XYZZ piece = slots[2 * k];
        g1_add(acc, piece);
      }
    }
    block_sum_xyzz(sh, acc);
    if (threadIdx.x == 0) buckets[it.bucket] = sh[0];
    __syncthreads();
  }
}

// ---- bucket reduction (msm_bucket.cuh) --------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_reduce_level0(ReduceArgs a) {
  reduce_level0_thread(a, (uint64_t)blockIdx.x * blockDim.x + threadIdx.x);
}
__global__ void __launch_bounds__(PB_REDUCE_THREADS) k_reduce_block(BlockLevelArgs a) {
  __shared__ G1XYZZ sh[PB_REDUCE_THREADS];
  const uint32_t t = threadIdx.x, chunk = blockIdx.x, set = blockIdx.y;
  G1XYZZ s, x;
  blk_local(a, set, chunk, t, s, x);
  sh[t] = s;
  __syncthreads();
#pragma unroll 1
  for (uint32_t d = 1; d < PB_REDUCE_THREADS; d <<= 1) {
    const G1XYZZ v = blk_scan_step(sh, t, d);
    __syncthreads();
    sh[t] = v;
    __syncthreads();
  }
  const G1XYZZ suf = sh[t];  // thread 0 keeps S' = suf_0
  const G1XYZZ y = blk_weight(a, t, x, suf);
  __syncthreads();
  sh[t] = y;
  __syncthreads();
#pragma unroll 1
  for (uint32_t d = PB_REDUCE_THREADS / 2; d > 0; d >>= 1) {
    blk_tree_step(sh, t, d);
    __syncthreads();
  }
  if (t == 0) {
    SR o;
    o.S = suf;
    o.R = sh[0];
    a.out[(uint64_t)set * gridDim.x + chunk] = o;
  }
}

// affine points: canonical <-> Montgomery (both coordinates)
__global__ void k_affine_to_mont(const G1Affine* in, G1Affine* out, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p = in[i];
  p.x = fp_to_mont(p.x);
  p.y = fp_to_mont(p.y);
  out[i] = p;
}

__global__ void k_affine_from_mont(const G1Affine* in, G1Affine* out, uint64_t n) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p = in[i];
  p.x = fp_from_mont(p.x);
  p.y = fp_from_mont(p.y);
  out[i] = p;
}

// out[i] = 2^c * in[i] as XYZZ
__global__ void __launch_bounds__(128) k_window_step(const G1Affine* in, G1XYZZ* out, uint64_t n, uint32_t c) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  G1Affine p = in[i];
  G1XYZZ a;
  g1_double_affine(a, p);
  for (uint32_t k = 1; k < c; k++) g1_double(a);
  out[i] = a;
}

void affine_to_mont(Context* ctx, const G1Affine* in, G1Affine* out, uint64_t n) {
  k_affine_to_mont<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(in, out, n);
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
}

// XYZZ -> affine with Montgomery's batch-inversion trick, CH points per thread.  No input may be the identity: one
// ZZZ == 0 zeroes the product of its chunk, and every point of that chunk comes out as (0, 0), which is neither the
// MSM's identity encoding nor on the curve.  Every caller converts k P for a point P != O and 0 < k < r (the group
// has prime order r); pb200_srs_generate / _lagrange refuse the taus that would make k = 0.
__global__ void __launch_bounds__(128) k_batch_to_affine(const G1XYZZ* in, G1Affine* out, uint64_t n) {
  const int CH = 16;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t i0 = t * CH;
  if (i0 >= n) return;
  int cnt = (int)min((uint64_t)CH, n - i0);
  Fq pref[CH];
  Fq run = Fq::one();
  for (int k = 0; k < cnt; k++) {
    pref[k] = run;                      // product of ZZZ[0..k)
    run = fp_mul(run, in[i0 + k].ZZZ);
  }
  Fq inv = fp_inv_gcd(run);
  for (int k = cnt - 1; k >= 0; k--) {
    G1XYZZ a = in[i0 + k];
    Fq A = fp_mul(inv, pref[k]);        // 1 / ZZZ_k
    inv = fp_mul(inv, a.ZZZ);
    Fq izz = fp_sqr(fp_mul(a.ZZ, A));
    G1Affine p;
    p.x = fp_mul(a.X, izz);
    p.y = fp_mul(a.Y, A);
    out[i0 + k] = p;
  }
}

// ------------------------------------------------------------------------------------------
// host orchestration
// ------------------------------------------------------------------------------------------
struct Srs {
  uint64_t n = 0;
  DevBuf base;       // n affine points, Montgomery form
  uint32_t c = 0, W = 0;
  DevBuf expanded;   // W * n affine points (window multiples), or empty
};

static uint32_t windows_for(uint32_t c) { return (256 + c - 1) / c; }

// Kernel attributes of the current device, set when a context (which is tied to one device) is created: the sort's
// shared-memory stages
void msm_init_device() {
  PB_CUDA(cudaFuncSetAttribute(k_msm_bin_scatter, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)(PB_SORT_BIN_STAGE * sizeof(SortEntry))));
  PB_CUDA(cudaFuncSetAttribute(k_msm_chunk_place, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(PB_SORT_CHUNK * 4)));
}

uint32_t msm_default_window(uint64_t n, bool fixed_base) {
  int lg = 0;
  while (((uint64_t)1 << lg) < n) lg++;
  int c = fixed_base ? lg : lg - 4;
  int lo = 4, hi = fixed_base ? 21 : 16;
  if (const char* e = getenv(fixed_base ? "PB200_MSM_C_FIXED" : "PB200_MSM_C")) { c = atoi(e); }
  if (c < lo) c = lo;
  if (c > hi) c = hi;
  return (uint32_t)c;
}

// k * p for a small k (host arithmetic, double-and-add)
static G1XYZZ host_mul_small(const G1XYZZ& p, uint32_t k) {
  G1XYZZ r = G1XYZZ::identity();
  for (int i = 31; i >= 0; i--) {
    g1_double(r);
    if ((k >> i) & 1) g1_add(r, p);
  }
  return r;
}

static void host_horner_to_affine(const std::vector<G1XYZZ>& ws, uint32_t c, uint8_t* out_xy, int* is_identity) {
  G1XYZZ r = G1XYZZ::identity();
  for (int w = (int)ws.size() - 1; w >= 0; w--) {
    if (w != (int)ws.size() - 1)
      for (uint32_t k = 0; k < c; k++) g1_double(r);
    g1_add(r, ws[w]);
  }
  G1Affine a;
  bool inf = g1_to_affine(r, a);
  *is_identity = inf ? 1 : 0;
  Fq x = fp_from_mont(a.x), y = fp_from_mont(a.y);
  memcpy(out_xy, x.v, 32);
  memcpy(out_xy + 32, y.v, 32);
}

static uint32_t env_u32(const char* name, uint32_t dflt) {
  const char* e = getenv(name);
  return e ? (uint32_t)atoi(e) : dflt;
}

// Chain length of an accumulation round (see AffAcc::B): as long as the launch still fills the machine.  A
// thread's safegcd inversion costs about as much as 8 additions, so short chains are expensive; the integer pipe is
// saturated by two resident warps per scheduler, so 256 threads per SM is "full".
static uint32_t pick_B(Context* ctx, uint64_t slots, uint32_t r) {
  static const uint32_t forced = env_u32("PB200_MSM_B", 0);
  const uint32_t cap = r == 0 ? 64 : PB_AFF_BMAX;  // round 0 is dense: B additions; later rounds: about B / 2
  if (forced) return std::min<uint32_t>(std::max<uint32_t>(r == 0 ? forced : 2 * forced, 2), cap);
  const uint64_t full = (uint64_t)ctx->sm_count * 256;
  for (uint32_t B = cap; B > 16; B >>= 1)
    if (slots / aff_round_span(B, r) >= 2 * full) return B;
  return 16;
}

// sum over ranks rho of (R_rho + rho * nloc * S_rho) for every bucket set: the partial sums of equal bucket ranges
// [rho * nloc, (rho + 1) * nloc), nloc a power of two.  all: [world][sets] (S, R) pairs.
// The same join for STRIDED shards (rank rho owns the buckets j = G k + rho; what the communicator path uses):
// sum_k (G k + rho + 1) B = G R_rho + (rho + 1 - G) S_rho, so the total is G sum R_rho - sum (G - 1 - rho) S_rho.
void host_join_bucket_shards_strided(const SR* all, uint32_t world, uint32_t sets, G1XYZZ* out) {
  uint32_t log_g = 0;
  while ((1u << log_g) < world) log_g++;
  PB_CHECK((1u << log_g) == world, "strided bucket shards need a power-of-two rank count");
  for (uint32_t s = 0; s < sets; s++) {
    G1XYZZ run = G1XYZZ::identity(), weighted = G1XYZZ::identity(), plain = G1XYZZ::identity();
    for (uint32_t rho = 0; rho < world; rho++) {
      const SR& e = all[(size_t)rho * sets + s];
      g1_add(plain, e.R);
      if (rho + 1 < world) {
        g1_add(run, e.S);       // sum_{rho' <= rho} S
        g1_add(weighted, run);  // -> sum (G - 1 - rho) S_rho
      }
    }
    for (uint32_t k = 0; k < log_g; k++) g1_double(plain);
    weighted.Y = fp_neg(weighted.Y);
    g1_add(plain, weighted);
    out[s] = plain;
  }
}

void host_join_bucket_shards(const SR* all, uint32_t world, uint32_t sets, uint32_t nloc, G1XYZZ* out) {
  uint32_t log_nloc = 0;
  while ((1u << log_nloc) < nloc) log_nloc++;
  PB_CHECK((1u << log_nloc) == nloc, "bucket shards must be a power of two wide");
  for (uint32_t s = 0; s < sets; s++) {
    G1XYZZ run = G1XYZZ::identity(), weighted = G1XYZZ::identity(), plain = G1XYZZ::identity();
    for (uint32_t rho = world; rho-- > 0;) {
      const SR& e = all[(size_t)rho * sets + s];
      g1_add(plain, e.R);
      if (rho >= 1) {
        g1_add(run, e.S);       // sum_{rho' >= rho} S
        g1_add(weighted, run);  // -> sum rho * S_rho
      }
    }
    for (uint32_t k = 0; k < log_nloc; k++) g1_double(weighted);
    g1_add(plain, weighted);
    out[s] = plain;
  }
}

// points: Montgomery affine (generic: n points; fixed-base: expanded table W*n).
// batch > 1 (fixed-base only): `batch` scalar vectors against the same points in one pass; the k-th MSM uses bucket
// set k.  [bucket_lo, bucket_hi): the bucket magnitudes this call owns (0, 2^(c-1) = everything); with a proper
// sub-range the result is this rank's partial sum.  comm != nullptr: the ranks of the communicator split the buckets
// evenly, exchange their 256-byte (S, R) pairs with one allgather and all return the full result.
void msm_run_batch(Context* ctx, const G1Affine* points, uint64_t n, const Fr* const* scalars, uint32_t batch,
                   bool scalars_mont, uint32_t c, bool fixed_base, uint64_t point_stride, uint32_t bucket_lo,
                   uint32_t bucket_hi, uint8_t* out_xy /*batch*64*/, int* is_identity /*batch*/,
                   G1XYZZ* raw_out /*optional: batch XYZZ sums instead of affine*/, Comm* comm = nullptr) {
  PB_CHECK(n > 0, "empty MSM");
  PB_CHECK(batch >= 1 && batch <= 4 && (fixed_base || batch == 1), "bad MSM batch");
  MsmGeom g;
  g.c = c;
  g.W = windows_for(c);
  g.half = 1u << (c - 1);
  g.fixed_base = fixed_base ? 1 : 0;
  g.point_stride = fixed_base ? point_stride : 0;
  g.batch = batch;
  g.own_log = 0;
  g.own_rank = 0;
  if (comm && comm_world(comm) > 1) {
    // strided ownership: rank r takes the buckets j = G k + r, so the few buckets a short top window (or a skewed
    // witness) concentrates on are spread over all ranks
    PB_CHECK((g.half >> comm_log_world(comm)) >= 1, "more ranks than buckets");
    static const bool contiguous = getenv("PB200_SHARD_CONTIGUOUS") != nullptr;  // A/B switch: r * nloc .. (r+1) * nloc
    if (contiguous) {
      const uint32_t per = g.half >> comm_log_world(comm);
      bucket_lo = per * (uint32_t)comm_rank(comm);
      bucket_hi = bucket_lo + per;
    } else {
      g.own_log = (uint32_t)comm_log_world(comm);
      g.own_rank = (uint32_t)comm_rank(comm);
      bucket_lo = 0;
      bucket_hi = g.half >> g.own_log;
    }
  } else {
    comm = nullptr;
  }
  if (bucket_hi > g.half) bucket_hi = g.half;
  PB_CHECK(bucket_lo < bucket_hi, "empty MSM bucket range");
  g.lo = bucket_lo;
  g.nloc = bucket_hi - bucket_lo;
  g.sets = fixed_base ? batch : g.W;
  g.nb = g.sets * g.nloc;
  PB_CHECK((fixed_base ? (uint64_t)g.W * point_stride : n) < (1ull << 31), "MSM too large for 31-bit point ids");
  ScalarBatch sb;
  for (uint32_t k = 0; k < 4; k++) sb.p[k] = k < batch ? scalars[k] : nullptr;

  // XYZZ segment accumulation is the default: measured on H100 (profiles/h100_bench_1gpu_msm_affine.json) the batched-affine
  // rounds spend in field additions and the safegcd inversion (ALU pipe) what they save in multiplications
  static const bool use_xyzz = [] { const char* e = getenv("PB200_MSM_ACC"); return !(e && !strcmp(e, "affine")); }();
  const uint32_t pad = use_xyzz ? 0 : 1;
  DevBuf& sorted = ctx->scratch[2];
  DevBuf& counts = ctx->scratch[3];
  DevBuf& offsets = ctx->scratch[4];
  DevBuf& lvl_a = ctx->scratch[6];
  DevBuf& lvl_b = ctx->scratch[7];
  const uint64_t entries = n * g.W * batch;           // upper bound (every digit non-zero and owned)
  const uint64_t positions = entries + (pad ? g.nb : 0);  // with the padding to even bucket sizes
  PB_CHECK(positions < (1ull << 30), "MSM too large (n * windows * batch must stay below 2^30)");
  sorted.ensure(positions * 4);
  counts.ensure((size_t)g.nb * 4 + 16);
  offsets.ensure((size_t)(g.nb + 1) * 4);
  uint32_t* max_cnt = counts.as<uint32_t>() + g.nb;
  const uint32_t n_tiles = (g.nb + PB_SCAN_TILE - 1) / PB_SCAN_TILE;
  PB_CHECK(n_tiles <= 8192, "too many buckets for the scan");
  ctx->msm_aff[1].ensure((size_t)8192 * 4);
  uint32_t* tile_sums = ctx->msm_aff[1].as<uint32_t>();

  // two-level sort (msm_sort.cuh): at most PB_SORT_MAX_BINS bins of 2^lb consecutive bucket keys
  const uint32_t lb = sort_default_lb(g.nb);
  PB_CHECK((1u << lb) <= PB_SORT_MAX_BIN_KEYS, "too many buckets for the sort");
  DevBuf& binned = ctx->scratch[8];
  DevBuf& bin_tab = ctx->scratch[9];
  binned.ensure(entries * sizeof(SortEntry));
  bin_tab.ensure((size_t)3 * (PB_SORT_MAX_BINS + 1) * 4);
  SortArgs sa;
  sa.sb = sb;
  sa.n = n;
  sa.from_mont = scalars_mont ? 1 : 0;
  sa.g = g;
  sa.lb = lb;
  sa.nbins = ((g.nb - 1) >> lb) + 1;
  sa.T = PB_SORT_CHUNK;
  uint32_t* bin_cnt = bin_tab.as<uint32_t>();
  uint32_t* bin_off = bin_cnt + PB_SORT_MAX_BINS + 1;
  sa.bin_cnt = bin_cnt;
  sa.bin_off = bin_off;
  sa.binned = binned.as<SortEntry>();
  sa.chunk_first = bin_off + PB_SORT_MAX_BINS + 1;
  sa.counts = counts.as<uint32_t>();
  sa.offsets = offsets.as<uint32_t>();
  sa.sorted = sorted.as<uint32_t>();
  sa.spb = PB_SORT_BIN_STAGE / g.W;
  const dim3 bin_grid((unsigned)((n + sa.spb - 1) / sa.spb), batch);
  // the chunk kernels walk the chunks grid-stride: (entries / T + bins) is a bound, the real count is on the device
  const uint64_t chunk_bound = entries / PB_SORT_CHUNK + sa.nbins;
  const uint32_t count_grid = (uint32_t)std::min<uint64_t>((uint64_t)ctx->sm_count * 4, chunk_bound);
  const uint32_t place_grid = (uint32_t)std::min<uint64_t>((uint64_t)ctx->sm_count * 2, chunk_bound);
  const size_t bin_stage_bytes = PB_SORT_BIN_STAGE * sizeof(SortEntry), chunk_stage_bytes = PB_SORT_CHUNK * 4;

  // The sort, the stitch and the upper reduction levels run on the context's high-priority stream, the accumulation
  // and reduction level 0 (bound by field products) on its main stream; every phase still waits for the one before.
  // Another context's accumulation fills the SMs with thousands of blocks: on the priority stream, these short
  // phases get each SM slot that one of its blocks frees instead of waiting for that whole grid to drain.
  cudaStream_t st = ctx->stream, ps = ctx->prio_stream;
  stream_join(ctx, ps, st);  // the scalars, and the previous call's last readers of this scratch
  ctx->time_begin(2, ps);
  PB_CUDA(cudaMemsetAsync(counts.p, 0, (size_t)g.nb * 4 + 16, ps));
  PB_CUDA(cudaMemsetAsync(bin_cnt, 0, (size_t)sa.nbins * 4, ps));
  if (pad) PB_CUDA(cudaMemsetAsync(sorted.p, 0xff, positions * 4, ps));
  k_msm_bin_count<<<bin_grid, PB_SORT_BIN_THREADS, 0, ps>>>(sa);
  k_scan_tile_sums<<<1, 256, 0, ps>>>(bin_cnt, sa.nbins, 0, tile_sums, nullptr);
  k_scan_tiles<<<1, 256, 0, ps>>>(tile_sums, 1, bin_off + sa.nbins);
  k_scan_apply<<<1, 256, 0, ps>>>(bin_cnt, sa.nbins, 0, tile_sums, bin_off);
  k_msm_bin_scatter<<<bin_grid, PB_SORT_BIN_THREADS, bin_stage_bytes, ps>>>(sa);
  k_msm_chunk_map<<<1, 256, 0, ps>>>(sa);
  k_msm_chunk_count<<<count_grid, PB_SORT_CHUNK_THREADS, 0, ps>>>(sa);
  k_scan_tile_sums<<<n_tiles, 256, 0, ps>>>(counts.as<uint32_t>(), g.nb, pad, tile_sums, max_cnt);
  k_scan_tiles<<<1, 256, 0, ps>>>(tile_sums, n_tiles, offsets.as<uint32_t>() + g.nb);
  k_scan_apply<<<n_tiles, 256, 0, ps>>>(counts.as<uint32_t>(), g.nb, pad, tile_sums, offsets.as<uint32_t>());
  k_msm_chunk_place<<<place_grid, PB_SORT_CHUNK_THREADS, chunk_stage_bytes, ps>>>(sa);
  ctx->time_end(2, ps);
  ctx->launches += 11;

  ReduceArgs ra;
  ra.pts = nullptr; ra.off = offsets.as<uint32_t>(); ra.cnt = counts.as<uint32_t>(); ra.xb = nullptr;
  if (!use_xyzz) {
    // rounds of batched affine additions, in place on the slot array (msm_bucket.cuh)
    const uint64_t s_bound = positions / 2;
    DevBuf& pts = ctx->msm_aff[0];
    pts.ensure(s_bound * sizeof(G1Affine));
    AffAcc a;
    a.table = points;
    a.sorted = sorted.as<uint32_t>();
    a.pts = pts.as<G1Affine>();
    a.off = offsets.as<uint32_t>();
    a.cnt = counts.as<uint32_t>();
    a.max_cnt = max_cnt;
    a.nbl = g.nb;
    // no bucket can hold more than n * W entries (fixed-base) / n entries (generic): rounds beyond that never run
    uint64_t cap = fixed_base ? n * g.W : n;
    uint32_t max_rounds = 1;
    while (max_rounds < 32 && (1ull << max_rounds) < cap) max_rounds++;
    stream_join(ctx, st, ps);
    ctx->time_begin(0);
    for (uint32_t r = 0; r < std::min<uint32_t>(max_rounds, PB_AFF_GRID_ROUNDS); r++) {
      a.r = r;
      a.B = pick_B(ctx, s_bound, r);
      const uint64_t threads = aff_round_threads(s_bound, a.B, r);
      if (r == 0) k_aff_round0<<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(a);
      else k_aff_round<<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(a);
      ctx->launches++;
    }
    if (max_rounds > PB_AFF_GRID_ROUNDS) {
      a.B = 32;
      k_aff_tail<<<1, 256, 0, st>>>(a, s_bound);
      ctx->launches++;
    }
    ctx->time_end(0);
    ra.pts = pts.as<G1Affine>();
  } else {
    // balanced XYZZ accumulation over fixed segments of L sorted entries
    DevBuf& buckets = ctx->scratch[5];
    DevBuf& seg = ctx->scratch[1];
    buckets.ensure((size_t)g.nb * sizeof(G1XYZZ));
    // entries per thread: 32 when there is plenty of work; a rank that owns a small share of the buckets (or a small
    // MSM) takes shorter segments so that the launch still has ~2 threads per resident slot -- its time is then the
    // length of one thread's chain of dependent additions, not throughput
    static const uint32_t seg_env = env_u32("PB200_MSM_SEG", 0);
    uint32_t L = 32;
    if (seg_env) {
      L = seg_env;
    } else {
      const uint64_t expected = entries / (g.half / g.nloc);  // digits are close to uniform over the buckets
      // (measured on a 1/8 share of a 2^20 commitment: L = 32 -> 453 us accumulate + 30 us stitch, L = 8 -> 296 + 223)
      while (L > 4 && expected / L < (uint64_t)ctx->sm_count * 512) L >>= 1;
      // the per-segment scratch is sized for the worst case (all entries owned): keep it below 1 GiB
      while (L < 32 && (entries / L) * (2 * sizeof(G1XYZZ) + 12 + sizeof(HeavyItem)) > (1ull << 30)) L <<= 1;
    }
    PB_CHECK(L >= 1 && L <= 4096, "bad PB200_MSM_SEG");
    const uint32_t n_seg = (uint32_t)((entries + L - 1) / L);
    const uint32_t max_pieces = 2 * (n_seg / PB_STITCH_PIECE) + 16;
    seg.ensure((size_t)n_seg * 2 * sizeof(G1XYZZ) + (size_t)n_seg * 3 * 4 + (size_t)n_seg * sizeof(HeavyItem) + 16 +
               (size_t)max_pieces * (sizeof(HeavyPiece) + sizeof(G1XYZZ)));
    G1XYZZ* slots = seg.as<G1XYZZ>();
    G1XYZZ* piece_partial = slots + (size_t)n_seg * 2;
    uint32_t* slot_bucket = reinterpret_cast<uint32_t*>(piece_partial + max_pieces);
    uint32_t* own_slot = slot_bucket + (size_t)n_seg * 2;
    uint32_t* heavy_count = own_slot + n_seg;  // [0] heavy items, [1] pieces
    HeavyItem* heavy = reinterpret_cast<HeavyItem*>(heavy_count + 4);
    HeavyPiece* pieces = reinterpret_cast<HeavyPiece*>(heavy + n_seg);
    PB_CUDA(cudaMemsetAsync(buckets.p, 0, (size_t)g.nb * sizeof(G1XYZZ), ps));
    PB_CUDA(cudaMemsetAsync(own_slot, 0xff, (size_t)n_seg * 4, ps));
    PB_CUDA(cudaMemsetAsync(heavy_count, 0, 16, ps));
    stream_join(ctx, st, ps);
    ctx->time_begin(0);
    k_msm_seg_accumulate<<<(n_seg + 127) / 128, 128, 0, st>>>(points, offsets.as<uint32_t>(), sorted.as<uint32_t>(),
                                                             g.nb, L, buckets.as<G1XYZZ>(), slots, slot_bucket, own_slot);
    ctx->time_end(0);
    stream_join(ctx, ps, st);
    k_msm_stitch<<<(n_seg + 127) / 128, 128, 0, ps>>>(offsets.as<uint32_t>(), g.nb, L, n_seg, slots, slot_bucket,
                                                     own_slot, buckets.as<G1XYZZ>(), heavy, heavy_count, pieces, 16);
    k_msm_stitch_pieces<<<std::min<uint32_t>(max_pieces, 592), 128, 0, ps>>>(slots, heavy, heavy_count, pieces, piece_partial);
    k_msm_stitch_heavy<<<296, 128, 0, ps>>>(slots, heavy, heavy_count, piece_partial, buckets.as<G1XYZZ>());
    ctx->launches += 4;
    ra.xb = buckets.as<G1XYZZ>();
  }
  stream_join(ctx, st, ps);

  // bucket reduction: levels of grouped running sums until one (S, R) pair per set is left
  // level-0 group size: 16 buckets per thread when that still fills the machine, down to 4 for small bucket counts
  // (a sharded rank, a small MSM), where the level is bound by the length of a thread's chain instead
  static const uint32_t g0_env = env_u32("PB200_MSM_G", 0);
  uint32_t log_g0 = 4;
  if (g0_env) {
    log_g0 = 1;
    while ((2u << log_g0) <= g0_env && log_g0 < 10) log_g0++;
  } else {
    while (log_g0 > 2 && (g.nb >> log_g0) < (uint32_t)ctx->sm_count * 256) log_g0--;
  }
  ctx->time_begin(3);
  ra.sets = g.sets;
  ra.m = g.nloc;
  ra.g = 1u << log_g0;
  {
    const uint64_t groups = (uint64_t)g.sets * reduce_groups(ra.m, ra.g);
    lvl_a.ensure(groups * sizeof(SR));
    lvl_b.ensure((groups / 16 + g.sets) * sizeof(SR));
    ra.out = lvl_a.as<SR>();
    k_reduce_level0<<<(unsigned)((groups + 127) / 128), 128, 0, st>>>(ra);
    ctx->launches++;
  }
  stream_join(ctx, ps, st);
  uint32_t m = reduce_groups(ra.m, ra.g), log_G = log_g0;
  SR* cur = lvl_a.as<SR>();
  SR* nxt = lvl_b.as<SR>();
  // the last few elements are folded on the host, which reads the result anyway; with a communicator every rank
  // reduces to ONE pair per set first, so the host join stays at world * sets additions
  const uint32_t m_stop = comm ? 1 : 8;
  while (m > m_stop) {
    BlockLevelArgs ba;
    ba.in = cur; ba.out = nxt; ba.sets = g.sets; ba.m = m; ba.log_G = log_G;
    k_reduce_block<<<dim3(reduce_chunks(m), g.sets), PB_REDUCE_THREADS, 0, ps>>>(ba);
    ctx->launches++;
    m = reduce_chunks(m);
    log_G += 9;  // log2(PB_REDUCE_CHUNK)
    std::swap(cur, nxt);
  }
  ctx->time_end(3, ps);
  stream_join(ctx, st, ps);  // the host reads the result on `st`
  PB_CUDA(cudaGetLastError());
  // the remaining m (<= 8) elements per set are folded on the host (reduce_fold_final)
  std::vector<G1XYZZ> ws(g.sets);
  if (comm) {
    // the MSM join: one allgather of sets * 256 bytes per rank, then a few host additions (the commitment has to
    // reach the host for the Fiat-Shamir transcript anyway)
    const uint32_t world = (uint32_t)comm_world(comm);
    DevBuf& gath = ctx->msm_aff[2];
    const size_t per_rank = (size_t)g.sets * m;  // every rank has the same m
    gath.ensure((size_t)world * per_rank * sizeof(SR));
    SR* all = gath.as<SR>();
    PB_CUDA(cudaMemcpyAsync(all + (size_t)comm_rank(comm) * per_rank, cur, per_rank * sizeof(SR), cudaMemcpyDeviceToDevice, st));
    comm_allgather_inplace(comm, all, per_rank * sizeof(SR), st);
    std::vector<SR> raw((size_t)world * per_rank), fin((size_t)world * g.sets);
    PB_CUDA(cudaMemcpyAsync(raw.data(), all, raw.size() * sizeof(SR), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t rho = 0; rho < world; rho++)
      for (uint32_t s = 0; s < g.sets; s++)
        fin[(size_t)rho * g.sets + s] = reduce_fold_final(raw.data() + (size_t)rho * per_rank + (size_t)s * m, m, log_G);
    if (g.own_log) host_join_bucket_shards_strided(fin.data(), world, g.sets, ws.data());
    else host_join_bucket_shards(fin.data(), world, g.sets, g.nloc, ws.data());
  } else {
    std::vector<SR> raw((size_t)g.sets * m), fin(g.sets);
    PB_CUDA(cudaMemcpyAsync(raw.data(), cur, raw.size() * sizeof(SR), cudaMemcpyDeviceToHost, st));
    PB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t s = 0; s < g.sets; s++) fin[s] = reduce_fold_final(raw.data() + (size_t)s * m, m, log_G);
    // set result = sum_j (lo + j + 1) B_j = R + lo * S
    for (uint32_t s = 0; s < g.sets; s++) {
      ws[s] = fin[s].R;
      if (g.lo) {
        G1XYZZ m_lo = host_mul_small(fin[s].S, g.lo);
        g1_add(ws[s], m_lo);
      }
    }
  }
  if (raw_out) {
    if (fixed_base) {
      for (uint32_t k = 0; k < batch; k++) raw_out[k] = ws[k];
    } else {  // window Horner without the final conversion
      G1XYZZ r = G1XYZZ::identity();
      for (int w = (int)g.W - 1; w >= 0; w--) {
        if (w != (int)g.W - 1) for (uint32_t k = 0; k < c; k++) g1_double(r);
        g1_add(r, ws[w]);
      }
      raw_out[0] = r;
    }
  } else if (fixed_base) {
    for (uint32_t k = 0; k < batch; k++) {
      std::vector<G1XYZZ> one(1, ws[k]);
      host_horner_to_affine(one, c, out_xy + 64 * k, is_identity + k);
    }
  } else {
    host_horner_to_affine(ws, c, out_xy, is_identity);
  }
}

void msm_run(Context* ctx, const G1Affine* points, uint64_t n, const Fr* scalars, bool scalars_mont, uint32_t c,
             bool fixed_base, uint64_t point_stride, uint8_t* out_xy, int* is_identity) {
  msm_run_batch(ctx, points, n, &scalars, 1, scalars_mont, c, fixed_base, point_stride, 0, 0xffffffffu, out_xy,
                is_identity, nullptr);
}

// ---- SRS --------------------------------------------------------------------------------
static void srs_finish(Context* ctx, Srs* srs, int precompute);

// h_points: n affine points, canonical little-endian (x || y), none the identity
Srs* srs_create(Context* ctx, const uint8_t* h_points, uint64_t n, int precompute) {
  auto srs = std::make_unique<Srs>();
  srs->n = n;
  srs->base.alloc(n * sizeof(G1Affine));
  DevBuf raw(n * sizeof(G1Affine));
  PB_CUDA(cudaMemcpyAsync(raw.p, h_points, n * sizeof(G1Affine), cudaMemcpyHostToDevice, ctx->stream));
  k_affine_to_mont<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(raw.as<G1Affine>(), srs->base.as<G1Affine>(), n);
  ctx->launches++;
  PB_CUDA(cudaStreamSynchronize(ctx->stream));
  srs_finish(ctx, srs.get(), precompute);
  return srs.release();
}

// base: n affine points already in HBM in Montgomery form (a checked .ptau section, ptau.cu), moved into the SRS
Srs* srs_adopt(Context* ctx, DevBuf&& base, uint64_t n, int precompute) {
  auto srs = std::make_unique<Srs>();
  srs->n = n;
  srs->base = std::move(base);
  srs_finish(ctx, srs.get(), precompute);
  return srs.release();
}

// builds the fixed-base window table 2^(c*w) * P_i, w < W, in HBM
static void srs_finish(Context* ctx, Srs* srs, int precompute) {
  const uint64_t n = srs->n;
  if (precompute) {
    uint32_t c = msm_default_window(n, true);
    uint32_t W = windows_for(c);
    srs->c = c;
    srs->W = W;
    srs->expanded.alloc((size_t)W * n * sizeof(G1Affine));
    G1Affine* ex = srs->expanded.as<G1Affine>();
    PB_CUDA(cudaMemcpyAsync(ex, srs->base.p, n * sizeof(G1Affine), cudaMemcpyDeviceToDevice, ctx->stream));
    DevBuf tmp(n * sizeof(G1XYZZ));
    for (uint32_t w = 1; w < W; w++) {
      k_window_step<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(ex + (uint64_t)(w - 1) * n, tmp.as<G1XYZZ>(), n, c);
      uint64_t threads = (n + 15) / 16;
      k_batch_to_affine<<<(unsigned)((threads + 127) / 128), 128, 0, ctx->stream>>>(tmp.as<G1XYZZ>(), ex + (uint64_t)w * n, n);
      ctx->launches += 2;
    }
    PB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  PB_CUDA(cudaGetLastError());
}

void srs_destroy(Srs* s) { delete s; }


// ---- structured SRS generation: [tau^i] G for i < n (setup.py:16-22 `powers_of_x` for a known test tau) --
// Fixed-base multiplication with byte windows: table[w][d-1] = d * 2^(8w) * G (32 x 255 affine points),
// then point_i = sum_w table[w][byte_w(tau^i)].
__global__ void __launch_bounds__(128) k_fb_table(G1XYZZ* out) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 32 * 255) return;
  uint32_t w = t / 255, d = t % 255 + 1;
  G1Affine g;
  g.x = Fq::one();
  g.y = fp_add(Fq::one(), Fq::one());  // generator (1, 2)
  G1XYZZ gx = g1_from_affine(g);
  G1XYZZ r = G1XYZZ::identity();
  for (int i = 7; i >= 0; i--) {
    g1_double(r);
    if ((d >> i) & 1) g1_add(r, gx);
  }
  for (uint32_t k = 0; k < 8 * w; k++) g1_double(r);
  out[t] = r;
}

__global__ void __launch_bounds__(128) k_fb_mul(const G1Affine* table, const Fr* scalars_mont, uint64_t n, G1XYZZ* out) {
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fr s = fp_from_mont(scalars_mont[i]);
  G1XYZZ acc = G1XYZZ::identity();
  for (uint32_t w = 0; w < 32; w++) {
    uint32_t d = (s.v[w >> 2] >> (8 * (w & 3))) & 0xff;
    if (d) {
      G1Affine p = ld_affine(table + w * 255 + (d - 1));
      g1_add_mixed(acc, p);
    }
  }
  out[i] = acc;
}

void launch_powers(Context* ctx, Fr* out, uint64_t n, const Fr& base, const Fr& scale);
static void srs_finish(Context* ctx, Srs* srs, int precompute);

void ntt_run(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in, const Fr* in_scale,
             const Fr* out_scale);

// tau: canonical Fr; generates on the device either the n monomial powers [tau^i] G or, with `lagrange`, the
// Lagrange-basis points [L_i(tau)] G of the domain of size n (n a power of two).  The Lagrange scalars are the
// inverse NTT of the power vector: sum_j c_j tau^j = sum_i v_i L_i(tau) with c = iNTT(v) gives
// L_i(tau) = (1/n) sum_j tau^j w^(-ij).
static Srs* srs_from_tau(Context* ctx, const Fr& tau_canonical, uint64_t n, int precompute, bool lagrange) {
  auto srs = std::make_unique<Srs>();
  srs->n = n;
  srs->base.alloc(n * sizeof(G1Affine));
  cudaStream_t st = ctx->stream;
  DevBuf tab_x(32 * 255 * sizeof(G1XYZZ)), tab(32 * 255 * sizeof(G1Affine));
  k_fb_table<<<(32 * 255 + 127) / 128, 128, 0, st>>>(tab_x.as<G1XYZZ>());
  k_batch_to_affine<<<((32 * 255 + 15) / 16 + 127) / 128, 128, 0, st>>>(tab_x.as<G1XYZZ>(), tab.as<G1Affine>(), 32 * 255);
  DevBuf pw(n * 32), pts(n * sizeof(G1XYZZ)), lag;
  launch_powers(ctx, pw.as<Fr>(), n, fp_to_mont(tau_canonical), Fr::one());
  const Fr* scalars = pw.as<Fr>();
  if (lagrange) {
    int log_n = 0;
    while (((uint64_t)1 << log_n) < n) log_n++;
    PB_CHECK(((uint64_t)1 << log_n) == n, "the Lagrange basis needs a power-of-two domain");
    lag.alloc(n * 32);
    ntt_run(ctx, pw.as<Fr>(), lag.as<Fr>(), log_n, true, n, nullptr, nullptr);
    scalars = lag.as<Fr>();
  }
  k_fb_mul<<<(unsigned)((n + 127) / 128), 128, 0, st>>>(tab.as<G1Affine>(), scalars, n, pts.as<G1XYZZ>());
  uint64_t threads = (n + 15) / 16;
  k_batch_to_affine<<<(unsigned)((threads + 127) / 128), 128, 0, st>>>(pts.as<G1XYZZ>(), srs->base.as<G1Affine>(), n);
  ctx->launches += 4;
  PB_CUDA(cudaStreamSynchronize(st));
  srs_finish(ctx, srs.get(), precompute);
  return srs.release();
}
Srs* srs_generate(Context* ctx, const Fr& tau_canonical, uint64_t n, int precompute) {
  return srs_from_tau(ctx, tau_canonical, n, precompute, false);
}
Srs* srs_generate_lagrange(Context* ctx, const Fr& tau_canonical, uint64_t n, int precompute) {
  return srs_from_tau(ctx, tau_canonical, n, precompute, true);
}

// copies the (canonical) affine points back to the host
void srs_export(Context* ctx, Srs* srs, uint8_t* h_points, uint64_t first, uint64_t count) {
  PB_CHECK(first + count <= srs->n, "SRS export out of range");
  DevBuf tmp(count * sizeof(G1Affine));
  k_affine_from_mont<<<(unsigned)((count + 127) / 128), 128, 0, ctx->stream>>>(srs->base.as<G1Affine>() + first,
                                                                          tmp.as<G1Affine>(), count);
  ctx->launches++;
  PB_CUDA(cudaMemcpyAsync(h_points, tmp.p, count * sizeof(G1Affine), cudaMemcpyDeviceToHost, ctx->stream));
  PB_CUDA(cudaStreamSynchronize(ctx->stream));
}

// commit to m <= n coefficients (device, Montgomery or canonical form)
void srs_msm(Context* ctx, Srs* srs, const Fr* d_scalars, uint64_t m, bool scalars_mont, uint8_t* out_xy, int* is_identity) {
  PB_CHECK(m <= srs->n, "Not enough powers in setup");
  if (srs->expanded.p) {
    msm_run(ctx, srs->expanded.as<G1Affine>(), m, d_scalars, scalars_mont, srs->c, true, srs->n, out_xy, is_identity);
  } else {
    msm_run(ctx, srs->base.as<G1Affine>(), m, d_scalars, scalars_mont, msm_default_window(m, false), false, 0, out_xy,
            is_identity);
  }
}

// `batch` commitments (<= 4) to coefficient vectors of the same length m in one pass over the SRS
void srs_msm_batch(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t m, bool scalars_mont,
                   uint8_t* out_xy, int* is_identity) {
  PB_CHECK(m <= srs->n, "Not enough powers in setup");
  if (srs->expanded.p && batch > 1) {
    msm_run_batch(ctx, srs->expanded.as<G1Affine>(), m, d_scalars, batch, scalars_mont, srs->c, true, srs->n, 0,
                  0xffffffffu, out_xy, is_identity, nullptr);
  } else {
    for (uint32_t k = 0; k < batch; k++) srs_msm(ctx, srs, d_scalars[k], m, scalars_mont, out_xy + 64 * k, is_identity + k);
  }
}

// Shard of `batch` commitments to m coefficients, returned as XYZZ partial sums (Montgomery) for the caller to
// exchange and add (multi-GPU MSM join).  Two ways to cut, which compose:
//   point range  [first, first + count): sum over those SRS powers only (each rank needs only its scalars' slab);
//   bucket range [bucket_lo, bucket_hi) of the 2^(c-1) signed-digit magnitudes: the rank walks all digits but sorts,
//                accumulates and reduces only its own buckets, so the bucket reduction divides by the rank count too.
void srs_msm_batch_partial(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t first,
                           uint64_t count, uint32_t bucket_lo, uint32_t bucket_hi, bool scalars_mont, G1XYZZ* out) {
  PB_CHECK(first + count <= srs->n, "Not enough powers in setup");
  PB_CHECK(srs->expanded.p, "sharded commitments need the fixed-base table (precompute)");
  const Fr* sh[4] = {nullptr, nullptr, nullptr, nullptr};
  for (uint32_t k = 0; k < batch; k++) sh[k] = d_scalars[k] + first;
  if (count == 0 || bucket_lo >= bucket_hi) {
    for (uint32_t k = 0; k < batch; k++) out[k] = G1XYZZ::identity();
    return;
  }
  msm_run_batch(ctx, srs->expanded.as<G1Affine>() + first, count, sh, batch, scalars_mont, srs->c, true, srs->n,
                bucket_lo, bucket_hi, nullptr, nullptr, out);
}
uint32_t srs_bucket_count(Srs* s) { return s->c ? 1u << (s->c - 1) : 0; }

// `batch` commitments with the buckets split over the ranks of the context's communicator (every rank holds the
// full scalar vectors and an SRS replica): one allgather of 256 bytes per commitment and rank at the join, the same
// affine results on every rank.
void srs_msm_batch_sharded(Context* ctx, Srs* srs, const Fr* const* d_scalars, uint32_t batch, uint64_t m,
                           bool scalars_mont, uint8_t* out_xy, int* is_identity) {
  PB_CHECK(m <= srs->n, "Not enough powers in setup");
  PB_CHECK(srs->expanded.p, "sharded commitments need the fixed-base table (precompute)");
  PB_CHECK(ctx->comm, "sharded commitments need a communicator on the context (pb200_comm_init)");
  msm_run_batch(ctx, srs->expanded.as<G1Affine>(), m, d_scalars, batch, scalars_mont, srs->c, true, srs->n, 0,
                0xffffffffu, out_xy, is_identity, nullptr, ctx->comm);
}

// sum of XYZZ partials -> canonical affine (host arithmetic; O(count) group operations)
void g1_combine_partials_host(const G1XYZZ* parts, uint32_t count, uint8_t* out_xy, int* is_identity) {
  std::vector<G1XYZZ> ws(1, G1XYZZ::identity());
  for (uint32_t k = 0; k < count; k++) g1_add(ws[0], parts[k]);
  host_horner_to_affine(ws, 1, out_xy, is_identity);
}

uint64_t srs_size(Srs* s) { return s->n; }
const G1Affine* srs_base(Srs* s) { return s->base.as<G1Affine>(); }

}  // namespace pb200
