// Fr radix-2 NTT / inverse NTT for sm_90a, natural order in -> natural order out.
//
// Replaces poly.py:113-149 (`Polynomial.fft` / `_fft` / `ifft`): forward computes
// o[k] = sum_j x[j] w^(jk) with w = 5^((r-1)/n) (curve.py:15-16); inverse uses the reversed roots
// (w^-1) and multiplies by n^-1 (poly.py:132-139).  Also carries the fused extras the coset
// transforms need (poly.py:156-177): multiply-on-load by a per-index table (offset^i), zero padding
// of the input (x4 extension), multiply-on-store by a per-index table (offset^-i).
//
// Decomposition (four-step, generalised to 1..3 passes): n = N1*N2(*N3).  Every pass transforms
// tiles of B = 2^logB points (up to 2048) x CC adjacent "batch" columns -- 2048 elements, 64 KiB -- held in
// shared memory as two 16-byte planes so 128-bit shared accesses are conflict-free.  The tile is bit-reversed
// on the way in; the in-tile DIT then runs in register-blocked radix-8 rounds (each thread owns 8 positions and
// does three radix-2 stages in registers between shared-memory exchanges) and leaves natural order.
// Non-final passes multiply by the inter-pass twiddles w_n^(j*k) from an HBM-resident table laid out exactly
// like the data (so the access is coalesced and costs no extra modmul), and write in place; the final pass
// writes transposed, CC x 32 B contiguous per row.  The per-pass local twiddles w_B^j are staged into shared
// memory with one TMA bulk copy (cp.async.bulk + mbarrier).
#include "common.cuh"
#include "comm.cuh"
#include "ntt_shard.cuh"

namespace pb200 {

// ------------------------------------------------------------------------------------------
// host-side Fr helpers (same limb code as the device, via the host emulation in field.cuh)
// ------------------------------------------------------------------------------------------
Fr fr_from_u64(uint64_t x) {
  Fr a = Fr::zero();
  a.v[0] = (uint32_t)x;
  a.v[1] = (uint32_t)(x >> 32);
  return fp_to_mont(a);
}

// w_{2^k} = 5^((r-1)/2^k) in Montgomery form (curve.py:15-16)
Fr fr_root_of_unity(int log_n) {
  // (r-1) >> log_n
  uint32_t e[8];
  for (int i = 0; i < 8; i++) e[i] = FrParams::p(i);
  e[0] -= 1;
  for (int s = 0; s < log_n; s++) {
    for (int i = 0; i < 8; i++) e[i] = (e[i] >> 1) | (i < 7 ? (e[i + 1] << 31) : 0);
  }
  return fp_pow(fr_from_u64(5), e);
}

// ------------------------------------------------------------------------------------------
// table generation kernels
// ------------------------------------------------------------------------------------------
// out[row * cols + j] = scale * w^(row * j)   (rows x cols, chunk of 64 columns per thread)
__global__ void k_gen_interpass(Fr* out, uint64_t rows, uint64_t cols, Fr w, Fr scale) {
  const int CH = 64;
  uint64_t chunks_per_row = (cols + CH - 1) / CH;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= rows * chunks_per_row) return;
  uint64_t row = t / chunks_per_row, j0 = (t % chunks_per_row) * CH;
  Fr wk = fp_pow_u64(w, row);
  Fr cur = fp_mul(fp_pow_u64(wk, j0), scale);
  for (int j = 0; j < CH && j0 + j < cols; j++) {
    out[row * cols + j0 + j] = cur;
    cur = fp_mul(cur, wk);
  }
}

// Position of local twiddle j inside its 16-byte plane: the higher 3-bit groups of j XOR-folded into the low three
// bits.  A stage reads the entries (low + m 2^t0) 2^s: eight lanes with different `low` would otherwise hit multiples
// of 8 entries -- one 16-byte column of the 128-byte wavefront -- and serialise 8-fold (ncu: 2.9 conflicts per element
// and pass after the data tile had been swizzled).  A bijection on [0, count) for any power-of-two count >= 8.
__host__ __device__ __forceinline__ uint32_t twiddle_slot(uint32_t j, uint32_t count) {
  return count >= 8 ? j ^ (((j >> 3) ^ (j >> 6) ^ (j >> 9)) & 7u) : j;
}

// planes[slot(j)] (lo 16 B) and planes[count + slot(j)] (hi 16 B) of w^j, j < count: stored pre-swizzled so that the
// TMA bulk copy of the kernel stays one linear transfer
__global__ void k_gen_local(uint4* planes, uint32_t count, Fr w) {
  uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= count) return;
  Fr x = fp_pow_u64(w, j);
  const uint32_t t = twiddle_slot(j, count);
  planes[t] = make_uint4(x.v[0], x.v[1], x.v[2], x.v[3]);
  planes[count + t] = make_uint4(x.v[4], x.v[5], x.v[6], x.v[7]);
}

// out[i] = scale * base^i
__global__ void k_powers(Fr* out, uint64_t n, Fr base, Fr scale) {
  const int CH = 64;
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t i0 = t * CH;
  if (i0 >= n) return;
  Fr cur = fp_mul(fp_pow_u64(base, i0), scale);
  for (int j = 0; j < CH && i0 + j < n; j++) {
    out[i0 + j] = cur;
    cur = fp_mul(cur, base);
  }
}

void launch_powers(Context* ctx, Fr* out, uint64_t n, const Fr& base, const Fr& scale) {
  uint64_t threads = (n + 63) / 64;
  k_powers<<<(unsigned)((threads + 127) / 128), 128, 0, ctx->stream>>>(out, n, base, scale);
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
}

// ------------------------------------------------------------------------------------------
// the pass kernel
// ------------------------------------------------------------------------------------------
struct PassParams {
  const Fr* in;
  Fr* out;
  const uint4* twl;     // local twiddles w_B^j, j < B/2, split planes
  const Fr* twg;        // inter-pass twiddle table (nullptr on the last pass)
  const Fr* in_scale;   // optional multiply-on-load table, indexed by global input index
  const Fr* out_scale;  // optional multiply-on-store table, indexed by global output index
  uint64_t n_in;        // input indices >= n_in read as zero
  uint64_t in_mul, in_add;  // physical input index = logical * in_mul + in_add (strided sub-sequence, first pass)
  uint32_t fold;            // first pass: logical input i is sum_f (in * in_scale)[i + f * 2^log_n], f < fold (a
                            // polynomial longer than the transform, reduced mod X^N - c^N on the fly)
  uint32_t log_b, log_cc, t_lo_count, b_fastest_load, has_final_scale, log_n;
  uint64_t r_hi, r_lo, r_cs, r_bs;
  uint64_t w_hi, w_lo, w_cs, w_bs;
  uint64_t g_hi, g_lo, g_cs, g_bs;
  Fr final_scale;
};

__device__ __forceinline__ Fr ld_planes(const uint4* lo, const uint4* hi, uint32_t i) {
  uint4 a = lo[i], b = hi[i];
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
__device__ __forceinline__ void st_planes(uint4* lo, uint4* hi, uint32_t i, const Fr& r) {
  lo[i] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  hi[i] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
// Data-tile accessors with an XOR swizzle of the low three index bits (a 16-byte access is served per quarter
// warp, 8 lanes x 16 B = one 128-byte wavefront when the 8 addresses differ in those bits).  Without it the
// bit-reversed tile load (lanes differ only in high index bits) and the first register-blocked round (lanes 8
// elements apart) put all 8 lanes of a wavefront on the same banks: ncu counted 3.5-4.7 M conflicts per pass.
// XOR-ing bits 3..5 and the top three bits of the index into bits 0..2 makes every access pattern of the kernel
// touch 8 distinct 16-byte columns; it is a bijection on the tile, so no padding is needed.
struct TileSwz {
  uint32_t top_shift, mask;  // mask = 7, or 0 for tiles too small to swizzle
  __device__ __forceinline__ uint32_t operator()(uint32_t i) const { return i ^ (((i >> 3) ^ (i >> top_shift)) & mask); }
};
__device__ __forceinline__ Fr ld_tile(const uint4* lo, const uint4* hi, uint32_t i, const TileSwz& z) {
  return ld_planes(lo, hi, z(i));
}
__device__ __forceinline__ void st_tile(uint4* lo, uint4* hi, uint32_t i, const Fr& r, const TileSwz& z) {
  st_planes(lo, hi, z(i), r);
}
__device__ __forceinline__ Fr ld_global(const Fr* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(q), b = __ldg(q + 1);
  Fr r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
  r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
  return r;
}
__device__ __forceinline__ void st_global(Fr* p, const Fr& r) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
  q[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

// --- TMA bulk copy (global -> shared) completed through an mbarrier -------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
      "r"(phase)
      : "memory");
}

// One register-blocked round: the thread owns the 8 tile positions base + k * 2^t0 (k = 0..7; base has three
// zero bits inserted at bit t0) of column c, runs the radix-2 DIT stages t0+s_first .. t0+2 on them in
// registers and writes them back.  Stage t0+s pairs k with k + 2^s and uses w_{2^(t0+s+1)}^j with
// j = (low t0 bits of base) + (k mod 2^s) * 2^t0.
__device__ __forceinline__ void ntt_round8(uint4* s_lo, uint4* s_hi, const uint4* t_lo, const uint4* t_hi, uint32_t q,
                                           uint32_t c, uint32_t t0, uint32_t s_first, uint32_t log_b,
                                           uint32_t log_cc, const TileSwz& z) {
  const uint32_t low = q & ((1u << t0) - 1);
  const uint32_t base = ((q >> t0) << (t0 + 3)) | low;
  Fr x[8];
#pragma unroll
  for (int k = 0; k < 8; k++) x[k] = ld_tile(s_lo, s_hi, ((base + ((uint32_t)k << t0)) << log_cc) | c, z);
#pragma unroll
  for (int s = 0; s < 3; s++) {
    if ((uint32_t)s < s_first) continue;
    const uint32_t st = t0 + s;
#pragma unroll
    for (int m = 0; m < (1 << s); m++) {
      Fr tw;
      const bool unit = (st == 0);
      if (!unit) tw = ld_planes(t_lo, t_hi, twiddle_slot((low + ((uint32_t)m << t0)) << (log_b - 1 - st), 1u << (log_b - 1)));
#pragma unroll
      for (int h = 0; h < (4 >> s); h++) {
        const int k = m + (h << (s + 1));
        Fr v = x[k + (1 << s)];
        if (!unit) v = fp_mul(v, tw);
        Fr u = x[k];
        x[k] = fp_add(u, v);
        x[k + (1 << s)] = fp_sub(u, v);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; k++) st_tile(s_lo, s_hi, ((base + ((uint32_t)k << t0)) << log_cc) | c, x[k], z);
}

#ifndef PB_NTT_THREADS
#define PB_NTT_THREADS 256
#define PB_NTT_BLOCKS 2
#endif
__global__ void __launch_bounds__(PB_NTT_THREADS, PB_NTT_BLOCKS) k_ntt_pass(PassParams p) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const uint32_t B = 1u << p.log_b, CC = 1u << p.log_cc, TE = B << p.log_cc;
  uint4* s_lo = reinterpret_cast<uint4*>(smem_raw);
  uint4* s_hi = s_lo + TE;
  uint4* t_lo = s_hi + TE;             // B/2 entries (at least 1)
  const uint32_t TW = B > 1 ? (B >> 1) : 1;
  uint4* t_hi = t_lo + TW;
  uint64_t* bar = reinterpret_cast<uint64_t*>(t_hi + TW);
  const uint32_t tid = threadIdx.x, nth = blockDim.x;
  const uint32_t log_te = p.log_b + p.log_cc;
  TileSwz z;
  z.mask = log_te >= 6 ? 7u : 0u;
  z.top_shift = log_te >= 6 ? log_te - 3 : 0;

  if (tid == 0) {
    mbar_init(bar, 1);
    mbar_expect_tx(bar, TW * 32);
    tma_bulk_g2s(t_lo, p.twl, TW * 32, bar);
  }

  const uint64_t tile = blockIdx.x;
  const uint64_t t_hi_i = tile / p.t_lo_count, t_lo_i = tile % p.t_lo_count;
  const uint64_t rbase = t_hi_i * p.r_hi + t_lo_i * p.r_lo;
  const uint64_t wbase = t_hi_i * p.w_hi + t_lo_i * p.w_lo;
  const uint64_t gbase = t_hi_i * p.g_hi + t_lo_i * p.g_lo;

  // ---- load tile (bit-reversed along the transform axis)
  for (uint32_t e = tid; e < TE; e += nth) {
    uint32_t c, b;
    if (p.b_fastest_load) { c = e >> p.log_b; b = e & (B - 1); }
    else { c = e & (CC - 1); b = e >> p.log_cc; }
    uint64_t gi = rbase + (uint64_t)c * p.r_cs + (uint64_t)b * p.r_bs;
    Fr x = Fr::zero();
    if (gi < p.n_in) {
      x = ld_global(p.in + gi * p.in_mul + p.in_add);
      if (p.in_scale) x = fp_mul(x, ld_global(p.in_scale + gi));
    }
    for (uint32_t f = 1; f < p.fold; f++) {
      const uint64_t gf = gi + ((uint64_t)f << p.log_n);
      if (gf < p.n_in) {
        Fr y = ld_global(p.in + gf * p.in_mul + p.in_add);
        if (p.in_scale) y = fp_mul(y, ld_global(p.in_scale + gf));
        x = fp_add(x, y);
      }
    }
    uint32_t br = p.log_b ? (__brev(b) >> (32 - p.log_b)) : 0;
    st_tile(s_lo, s_hi, (br << p.log_cc) | c, x, z);
  }
  __syncthreads();          // also orders tid 0's barrier init before the waits below
  mbar_wait(bar, 0);        // twiddles have landed

  if (p.log_b >= 3) {
    // ---- register-blocked rounds of three stages; a final partial round covers log_b mod 3 stages
    const uint32_t groups = TE >> 3;  // (B / 8) x CC threads' worth of work
    uint32_t t0 = 0;
    for (; t0 + 3 <= p.log_b; t0 += 3) {
      for (uint32_t w = tid; w < groups; w += nth) ntt_round8(s_lo, s_hi, t_lo, t_hi, w >> p.log_cc, w & (CC - 1), t0, 0, p.log_b, p.log_cc, z);
      __syncthreads();
    }
    if (t0 < p.log_b) {
      const uint32_t rem = p.log_b - t0;  // 1 or 2 stages left: run them as the tail of a group at log_b - 3
      for (uint32_t w = tid; w < groups; w += nth)
        ntt_round8(s_lo, s_hi, t_lo, t_hi, w >> p.log_cc, w & (CC - 1), p.log_b - 3, 3 - rem, p.log_b, p.log_cc, z);
      __syncthreads();
    }
  } else {
    // ---- tiny transforms: plain radix-2 stages in shared memory
    for (uint32_t t = 0; t < p.log_b; t++) {
      const uint32_t half = 1u << t;
      for (uint32_t q = tid; q < (TE >> 1); q += nth) {
        uint32_t c = q & (CC - 1), qq = q >> p.log_cc;
        uint32_t j = qq & (half - 1), grp = qq >> t;
        uint32_t i0 = (((grp << (t + 1)) + j) << p.log_cc) | c;
        uint32_t i1 = i0 + (half << p.log_cc);
        Fr u = ld_tile(s_lo, s_hi, i0, z);
        Fr v = ld_tile(s_lo, s_hi, i1, z);
        if (t > 0) v = fp_mul(v, ld_planes(t_lo, t_hi, twiddle_slot(j << (p.log_b - 1 - t), TW)));
        st_tile(s_lo, s_hi, i0, fp_add(u, v), z);
        st_tile(s_lo, s_hi, i1, fp_sub(u, v), z);
      }
      __syncthreads();
    }
  }

  // ---- store (batch index fastest)
  for (uint32_t e = tid; e < TE; e += nth) {
    uint32_t c = e & (CC - 1), k = e >> p.log_cc;
    Fr x = ld_tile(s_lo, s_hi, e, z);
    if (p.twg) x = fp_mul(x, ld_global(p.twg + gbase + (uint64_t)c * p.g_cs + (uint64_t)k * p.g_bs));
    if (p.has_final_scale) x = fp_mul(x, p.final_scale);
    uint64_t go = wbase + (uint64_t)c * p.w_cs + (uint64_t)k * p.w_bs;
    if (p.out_scale) x = fp_mul(x, ld_global(p.out_scale + go));
    st_global(p.out + go, x);
  }
}

// ------------------------------------------------------------------------------------------
// plans
// ------------------------------------------------------------------------------------------
struct NttPass {
  int log_b = 0, log_cc = 0;
  uint64_t tiles = 0;
  PassParams prm{};
  DevBuf twl, twg;
};

struct NttPlan {
  int log_n = 0;
  bool inverse = false;
  std::vector<NttPass> passes;
};

static const int kMaxLogB = 11;    // up to 2048-point tiles
#ifndef PB_NTT_TILE_LOG
#define PB_NTT_TILE_LOG 11
#endif
static const int kTileLog = PB_NTT_TILE_LOG;    // aim for 2048 elements (64 KiB) per tile: CC = 2048 / B adjacent columns

static size_t pass_smem_bytes(int log_b, int log_cc) {
  size_t B = (size_t)1 << log_b, TE = B << log_cc, TW = B > 1 ? B / 2 : 1;
  return TE * 32 + TW * 32 + 16;
}

static std::unique_ptr<NttPlan> build_plan(Context* ctx, int log_n, bool inverse) {
  PB_CHECK(log_n >= 0 && log_n <= 28, "NTT size must be 2^k with k <= 28 (Fr two-adicity)");
  auto plan = std::make_unique<NttPlan>();
  plan->log_n = log_n;
  plan->inverse = inverse;
  const uint64_t N = (uint64_t)1 << log_n;
  int npass = log_n <= kMaxLogB ? 1 : (log_n <= 2 * kMaxLogB ? 2 : 3);
  int lb[3] = {0, 0, 0};
  {
    int rem = log_n;
    for (int i = 0; i < npass; i++) {
      lb[i] = (rem + (npass - i) - 1) / (npass - i);
      rem -= lb[i];
    }
  }
  Fr w = fr_root_of_unity(log_n);
  if (inverse) w = fp_inv(w);
  Fr n_inv = fp_inv(fr_from_u64(N));
  plan->passes.resize(npass);
  uint64_t N1 = (uint64_t)1 << lb[0], N2 = (uint64_t)1 << lb[1], N3 = (uint64_t)1 << lb[2];
  for (int i = 0; i < npass; i++) {
    NttPass& ps = plan->passes[i];
    ps.log_b = lb[i];
    uint64_t B = (uint64_t)1 << lb[i];
    // local twiddles: w_B = w^(N/B)
    uint32_t TW = B > 1 ? (uint32_t)(B / 2) : 1;
    ps.twl.alloc((size_t)TW * 32);
    Fr wB = fp_pow_u64(w, N / B);
    k_gen_local<<<(TW + 127) / 128, 128, 0, ctx->stream>>>(ps.twl.as<uint4>(), TW, wB);
    ctx->launches++;
    PassParams& q = ps.prm;
    q.twl = ps.twl.as<uint4>();
    q.log_b = lb[i];
    q.has_final_scale = 0;
    q.final_scale = Fr::one();
    uint64_t batch;  // how many adjacent batch entries exist for this pass
    if (npass == 1) {
      batch = 1;
      ps.log_cc = 0;
      q.t_lo_count = 1;
      q.r_hi = q.r_lo = 0; q.r_cs = 0; q.r_bs = 1;
      q.w_hi = q.w_lo = 0; q.w_cs = 0; q.w_bs = 1;
      q.b_fastest_load = 1;
      q.twg = nullptr;
      if (inverse) { q.has_final_scale = 1; q.final_scale = n_inv; }
    } else if (i == 0) {
      // columns of length N1, stride C = N / N1; batch over adjacent columns
      uint64_t C = N / N1;
      batch = C;
      ps.log_cc = std::min(std::max(0, kTileLog - lb[0]), lb[1] + lb[2]);
      uint64_t CC = (uint64_t)1 << ps.log_cc;
      q.t_lo_count = (uint32_t)(C / CC);
      q.r_hi = 0; q.r_lo = CC; q.r_cs = 1; q.r_bs = C;
      q.w_hi = 0; q.w_lo = CC; q.w_cs = 1; q.w_bs = C;
      q.g_hi = 0; q.g_lo = CC; q.g_cs = 1; q.g_bs = C;
      q.b_fastest_load = 0;
      // table[k1 * C + j] = w^(j*k1) (* n^-1 for the inverse transform)
      ps.twg.alloc((size_t)N * 32);
      uint64_t threads = N1 * ((C + 63) / 64);
      k_gen_interpass<<<(unsigned)((threads + 127) / 128), 128, 0, ctx->stream>>>(
          ps.twg.as<Fr>(), N1, C, w, inverse ? n_inv : Fr::one());
      ctx->launches++;
      q.twg = ps.twg.as<Fr>();
    } else if (i == 1 && npass == 3) {
      // within row k1 (length M = N2*N3): columns of length N2, stride N3
      uint64_t M = N2 * N3;
      batch = N3;
      ps.log_cc = std::min(std::max(0, kTileLog - lb[1]), lb[2]);
      uint64_t CC = (uint64_t)1 << ps.log_cc;
      q.t_lo_count = (uint32_t)(N3 / CC);
      q.r_hi = M; q.r_lo = CC; q.r_cs = 1; q.r_bs = N3;
      q.w_hi = M; q.w_lo = CC; q.w_cs = 1; q.w_bs = N3;
      q.g_hi = 0; q.g_lo = CC; q.g_cs = 1; q.g_bs = N3;
      q.b_fastest_load = 0;
      ps.twg.alloc((size_t)M * 32);
      Fr wM = fp_pow_u64(w, N1);  // w_M = w^(N/M)
      uint64_t threads = N2 * ((N3 + 63) / 64);
      k_gen_interpass<<<(unsigned)((threads + 127) / 128), 128, 0, ctx->stream>>>(
          ps.twg.as<Fr>(), N2, N3, wM, Fr::one());
      ctx->launches++;
      q.twg = ps.twg.as<Fr>();
    } else {
      // last pass: contiguous rows of length B; batch over adjacent k1; transposed store
      q.twg = nullptr;
      q.b_fastest_load = 1;
      ps.log_cc = std::min(std::max(0, kTileLog - lb[i]), lb[0]);
      uint64_t CC = (uint64_t)1 << ps.log_cc;
      if (npass == 2) {
        batch = N1;
        q.t_lo_count = 1;  // tile = t_hi = k1 chunk
        q.r_hi = CC * N2; q.r_lo = 0; q.r_cs = N2; q.r_bs = 1;
        q.w_hi = CC; q.w_lo = 0; q.w_cs = 1; q.w_bs = N1;
      } else {
        batch = N1;
        q.t_lo_count = (uint32_t)N2;  // tile = (k1 chunk, k2)
        q.r_hi = CC * N2 * N3; q.r_lo = N3; q.r_cs = N2 * N3; q.r_bs = 1;
        q.w_hi = CC; q.w_lo = N1; q.w_cs = 1; q.w_bs = N1 * N2;
      }
    }
    (void)batch;
    q.log_cc = ps.log_cc;
    q.log_n = log_n;
    q.fold = 1;
    ps.tiles = N >> (lb[i] + ps.log_cc);
    size_t smem = pass_smem_bytes(ps.log_b, ps.log_cc);
    PB_CHECK(smem <= 227 * 1024, "NTT tile does not fit shared memory");
  }
  PB_CUDA(cudaGetLastError());
  return plan;
}

NttPlan* get_plan(Context* ctx, int log_n, bool inverse) {
  int key = log_n * 2 + (inverse ? 1 : 0);
  auto it = ctx->plans.find(key);
  if (it != ctx->plans.end()) return it->second.get();
  if (ctx->plans.empty())  // once per context, i.e. on this context's device (the attribute is per device)
    PB_CUDA(cudaFuncSetAttribute(k_ntt_pass, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  auto plan = build_plan(ctx, log_n, inverse);
  NttPlan* raw = plan.get();
  ctx->plans[key] = std::move(plan);
  return raw;
}

Context::Context() {}

Context::~Context() {
  plans.clear();
  shard_tables.clear();
  if (comm) comm_destroy(comm);
  for (auto& e : copy_done) if (e) cudaEventDestroy(e);
  for (auto& e : aux_ev) if (e) cudaEventDestroy(e);
  if (aux_stream) cudaStreamDestroy(aux_stream);
  if (copy_stream) cudaStreamDestroy(copy_stream);
  if (join_ev) cudaEventDestroy(join_ev);
  if (prio_stream) cudaStreamDestroy(prio_stream);
  if (own_stream && stream) cudaStreamDestroy(stream);
}

// out (2^log_n) = NTT(in), where `in` has n_in valid entries (rest read as zero).
// in_scale / out_scale: optional per-index multiplier tables.  `out` may alias `in` when
// n_in == 2^log_n.  Data form is irrelevant (the transform is linear and the twiddles are in
// Montgomery form): Montgomery in -> Montgomery out, canonical in -> canonical out.
void ntt_run_strided(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in,
                     const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add);

void ntt_run(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in,
             const Fr* in_scale, const Fr* out_scale) {
  ntt_run_strided(ctx, in, out, log_n, inverse, n_in, in_scale, out_scale, 1, 0);
}

void ntt_run_on(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add);
void ntt_run_fold(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                  uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add, uint32_t fold);

void ntt_run_strided(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in,
                     const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add) {
  ntt_run_on(ctx, ctx->stream, nullptr, in, out, log_n, inverse, n_in, in_scale, out_scale, in_mul, in_add);
}

// `stream` / `tmp`: run on another stream with a caller-owned pass buffer (2^log_n elements) so that the
// transform can overlap work on the context's main stream; tmp == nullptr uses the context's scratch.
void ntt_run_on(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add) {
  ntt_run_fold(ctx, stream, tmp, in, out, log_n, inverse, n_in, in_scale, out_scale, in_mul, in_add, 1);
}

// fold > 1: the logical input has fold * 2^log_n entries (of which n_in are non-zero) and is wrapped around the
// transform length on load -- evaluating a polynomial of degree >= 2^log_n on a 2^log_n-point (coset) domain.
void ntt_run_fold(Context* ctx, cudaStream_t stream, Fr* tmp, const Fr* in, Fr* out, int log_n, bool inverse,
                  uint64_t n_in, const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add, uint32_t fold) {
  NttPlan* plan = get_plan(ctx, log_n, inverse);
  const uint64_t N = (uint64_t)1 << log_n;
  int np = (int)plan->passes.size();
  const bool main_stream = stream == ctx->stream;
  if (np > 1 && !tmp) {
    PB_CHECK(main_stream, "a side-stream transform needs its own pass buffer");
    ctx->scratch[0].ensure((size_t)N * 32);
    tmp = ctx->scratch[0].as<Fr>();
  }
  for (int i = 0; i < np; i++) {
    NttPass& ps = plan->passes[i];
    PassParams q = ps.prm;
    q.in = (i == 0) ? in : tmp;
    q.out = (i == np - 1) ? out : tmp;
    q.n_in = (i == 0) ? n_in : N;
    q.in_mul = (i == 0) ? in_mul : 1;
    q.in_add = (i == 0) ? in_add : 0;
    q.in_scale = (i == 0) ? in_scale : nullptr;
    q.out_scale = (i == np - 1) ? out_scale : nullptr;
    q.fold = (i == 0) ? fold : 1;
    size_t smem = pass_smem_bytes(ps.log_b, ps.log_cc);
    if (main_stream) ctx->time_begin(1);
    k_ntt_pass<<<(unsigned)ps.tiles, PB_NTT_THREADS, smem, stream>>>(q);
    if (main_stream) ctx->time_end(1);
    ctx->launches++;
  }
  PB_CUDA(cudaGetLastError());
}

// ---- multi-GPU slab NTT (ntt_shard.cuh) -----------------------------------------------------------------------
struct ShardTables {
  DevBuf store_tw;  // w_N^(+-r k0) (* 1/G for the inverse), k0 < M: the local transform's multiply-on-store table
  DftTw dft;        // w_G^(+-k), k < G/2
};

struct CombineArgs {
  const Fr* sub;         // gathered sub-spectra: rank r's vector at sub + r * rank_stride
  Fr* out;
  uint64_t M, rank_stride;
  uint64_t limit;        // outputs with index >= limit are not stored; they must be zero (counted in *nonzero)
  const Fr* post_scale;  // optional per-output multiplier (indexed like out)
  uint32_t* nonzero;
  DftTw tw;
};
template <int LG>
__global__ void __launch_bounds__(128) k_shard_combine(CombineArgs a) {
  constexpr int G = 1 << LG;
  const uint64_t k0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k0 >= a.M) return;
  Fr x[G];
#pragma unroll
  for (int r = 0; r < G; r++) x[r] = ld_global(a.sub + (uint64_t)r * a.rank_stride + k0);
  small_dft<LG>(x, a.tw);
#pragma unroll
  for (int k1 = 0; k1 < G; k1++) {
    const uint64_t k = k0 + (uint64_t)k1 * a.M;
    if (k < a.limit) {
      Fr v = x[k1];
      if (a.post_scale) v = fp_mul(v, ld_global(a.post_scale + k));
      st_global(a.out + k, v);
    } else if (!x[k1].is_zero()) {
      atomicAdd(a.nonzero, 1u);
    }
  }
}

Comm* ctx_comm(Context* ctx);

// per (log_n, inverse, G, rank): a sliced prover joins the four slices of its coset on one device
static ShardTables* get_shard_tables(Context* ctx, int log_n, bool inverse, int log_g, int rank) {
  PB_CHECK(log_g >= 1 && log_g <= 3 && rank >= 0 && rank < (1 << log_g), "sharded transform: 2, 4 or 8 ranks");
  const int key = ((log_n * 2 + (inverse ? 1 : 0)) * 4 + log_g) * 8 + rank;
  auto it = ctx->shard_tables.find(key);
  if (it != ctx->shard_tables.end()) return it->second.get();
  PB_CHECK(log_n > log_g, "sharded transform: fewer points than ranks");
  const uint64_t M = (uint64_t)1 << (log_n - log_g);
  auto t = std::make_unique<ShardTables>();
  Fr w = fr_root_of_unity(log_n);
  if (inverse) w = fp_inv(w);
  Fr scale = inverse ? fp_inv(fr_from_u64((uint64_t)1 << log_g)) : Fr::one();
  t->store_tw.alloc(M * 32);
  launch_powers(ctx, t->store_tw.as<Fr>(), M, fp_pow_u64(w, (uint64_t)rank), scale);
  Fr wg = fp_pow_u64(w, M), cur = Fr::one();
  for (int k = 0; k < 4; k++) { t->dft.w[k] = cur; cur = fp_mul(cur, wg); }
  ShardTables* raw = t.get();
  ctx->shard_tables[key] = std::move(t);
  return raw;
}

// the join: `sub` holds the G = 2^log_g sub-spectra (rank r at r * rank_stride elements, M valid entries each);
// `rank` only picks a cached table (the join's twiddles do not depend on it)
void ntt_shard_combine(Context* ctx, const Fr* sub, uint64_t rank_stride, Fr* out, int log_n, bool inverse,
                       uint64_t limit, const Fr* post_scale, uint32_t* nonzero, int log_g, int rank) {
  ShardTables* t = get_shard_tables(ctx, log_n, inverse, log_g, rank);
  CombineArgs a;
  a.sub = sub; a.out = out; a.M = (uint64_t)1 << (log_n - log_g); a.rank_stride = rank_stride;
  a.limit = limit; a.post_scale = post_scale; a.nonzero = nonzero; a.tw = t->dft;
  const unsigned blocks = (unsigned)((a.M + 127) / 128);
  switch (log_g) {
    case 1: k_shard_combine<1><<<blocks, 128, 0, ctx->stream>>>(a); break;
    case 2: k_shard_combine<2><<<blocks, 128, 0, ctx->stream>>>(a); break;
    case 3: k_shard_combine<3><<<blocks, 128, 0, ctx->stream>>>(a); break;
    default: PB_CHECK(false, "sharded transform: 2, 4 or 8 ranks");
  }
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
}

// This rank's share of `count` transforms of the same size whose inputs are spread over the G ranks by decimation
// (logical input index i of rank r = global index G i + r; physical address in[v] + i * in_mul + in_add): local
// M-point transforms with the join twiddle fused into the store, written to the rank's place in ctx->gather
// ([G][count][M] layout), then ONE allgather over `cm`.  ntt_shard_combine finishes each vector.  cm == nullptr: one
// device plays every rank in turn (a sliced prover), no exchange; in[v] may then be the rank's own place in ctx->gather.
void ntt_shard_local(Context* ctx, const Fr* const* in, int count, int log_n, bool inverse, uint64_t in_mul,
                     uint64_t in_add, int log_g, int rank, Comm* cm) {
  const int G = 1 << log_g;
  ShardTables* t = get_shard_tables(ctx, log_n, inverse, log_g, rank);
  const uint64_t M = (uint64_t)1 << (log_n - log_g);
  ctx->gather.ensure((size_t)G * count * M * 32);
  Fr* mine = ctx->gather.as<Fr>() + (uint64_t)rank * count * M;
  for (int v = 0; v < count; v++)
    ntt_run_fold(ctx, ctx->stream, nullptr, in[v], mine + (uint64_t)v * M, log_n - log_g, inverse, M, nullptr,
                 t->store_tw.as<Fr>(), in_mul, in_add, 1);
  if (cm) comm_allgather_inplace(cm, ctx->gather.p, (size_t)count * M * 32, ctx->stream);
}

// full vector in (present on every rank) -> full vector out (on every rank): poly.py:113-149 across the ranks of the
// context's communicator with a single allgather at the join
void ntt_sharded(Context* ctx, const Fr* const* in, Fr* const* out, int count, int log_n, bool inverse) {
  Comm* cm = ctx_comm(ctx);
  const int log_g = comm_log_world(cm), rank = comm_rank(cm), G = 1 << log_g;
  if (G == 1) {  // a communicator of one rank: nothing to shard
    for (int v = 0; v < count; v++) ntt_run(ctx, in[v], out[v], log_n, inverse, (uint64_t)1 << log_n, nullptr, nullptr);
    return;
  }
  const uint64_t M = (uint64_t)1 << (log_n - log_g);
  ntt_shard_local(ctx, in, count, log_n, inverse, (uint64_t)G, (uint64_t)rank, log_g, rank, cm);
  for (int v = 0; v < count; v++)
    ntt_shard_combine(ctx, ctx->gather.as<Fr>() + (uint64_t)v * M, (uint64_t)count * M, out[v], log_n, inverse,
                      (uint64_t)1 << log_n, nullptr, nullptr, log_g, rank);
}

}  // namespace pb200
