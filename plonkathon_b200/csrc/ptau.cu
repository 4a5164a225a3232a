// Ceremony SRS from a snarkjs .ptau file, checked on the way in.
//
// A .ptau stores every coordinate as 32 little-endian bytes in Montgomery form with R = 2^256, which is the library's
// own device form, so the tauG1 section goes to HBM byte for byte (through pinned staging, in chunks) and becomes the
// SRS's base array with no conversion.  Before it is used it must pass:
//   1. every coordinate below q, and 2. every point on y^2 = x^3 + 3 (the identity, stored as (0, 0), is not)
//      -- one thread per point                                                      (k_ptau_check_g1)
//   3. point 0 is the generator (1, 2)
//   4. [tau]_2 on the twist and in G2: r [tau]_2 = O                                  (host G2 arithmetic, pairing.cuh)
//   5. the points are successive powers of the tau behind [tau]_2: for fresh 128-bit r_i from the OS CSPRNG,
//      e(sum_{i<m-1} r_i G_{i+1}, G2) = e(sum_{i<m-1} r_i G_i, [tau]_2), both sums one two-vector MSM over the SRS
//      itself (the second scalar vector is the first shifted by one place), then one product of two Miller loops.
// With 3 this makes G_i = [tau^i] G for the tau of [tau]_2, except with probability about 2^-128.
// A Lagrange block (section 12) passes 1 and 2 and must commit like the monomial SRS: for random values v,
// sum_i v_i [L_i(tau)] = sum_j c_j [tau^j] with c = iNTT(v).
#include <sys/random.h>

#include <cerrno>
#include <chrono>
#include <cstring>

#include "common.cuh"
#include "pairing.cuh"
#include "prover.cuh"

namespace pb200 {

Srs* srs_adopt(Context* ctx, DevBuf&& base, uint64_t n, int precompute);
void srs_destroy(Srs* s);
uint64_t srs_size(Srs* s);
void ntt_run(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in, const Fr* in_scale,
             const Fr* out_scale);
const Bn254Pairing& pairing_engine();

// bad[0]: lowest index of a point with a coordinate >= q; bad[1]: lowest index of a point with reduced coordinates
// that is not on y^2 = x^3 + 3 (Montgomery arithmetic throughout: the stored values are x R and y R)
__global__ void __launch_bounds__(256) k_ptau_check_g1(const G1Affine* pts, uint32_t n, uint32_t* bad) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint4* p = reinterpret_cast<const uint4*>(pts + i);
  const uint4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2), d = __ldg(p + 3);
  Fq x, y;
  x.v[0] = a.x; x.v[1] = a.y; x.v[2] = a.z; x.v[3] = a.w;
  x.v[4] = b.x; x.v[5] = b.y; x.v[6] = b.z; x.v[7] = b.w;
  y.v[0] = c.x; y.v[1] = c.y; y.v[2] = c.z; y.v[3] = c.w;
  y.v[4] = d.x; y.v[5] = d.y; y.v[6] = d.z; y.v[7] = d.w;
  if (!fp_is_canonical(x) || !fp_is_canonical(y)) {
    atomicMin(bad, i);
    return;
  }
  const Fq one = Fq::one();
  const Fq three = fp_add(fp_add(one, one), one);
  if (fp_sqr(y) != fp_add(fp_mul(fp_sqr(x), x), three)) atomicMin(bad + 1, i);
}

namespace {

enum { ST_H2D, ST_CHECK, ST_TABLE, ST_RANDOM, ST_MSM, ST_PAIRING, ST_G2, ST_COUNT };
thread_local double g_stage_ms[ST_COUNT];

double ms_since(std::chrono::steady_clock::time_point t0) {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
}

[[noreturn]] void refuse(const std::string& msg) { throw Error("ptau: " + msg); }

// host -> device through two pinned buffers: the copy into one overlaps the DMA out of the other
struct Staging {
  Context* ctx;
  size_t chunk;
  uint8_t* buf[2] = {nullptr, nullptr};
  cudaEvent_t done[2] = {nullptr, nullptr};
  Staging(Context* c, size_t bytes) : ctx(c), chunk(std::min<size_t>(bytes, (size_t)32 << 20)) {
    for (int k = 0; k < 2; k++) {
      PB_CUDA(cudaMallocHost((void**)&buf[k], chunk));
      PB_CUDA(cudaEventCreateWithFlags(&done[k], cudaEventDisableTiming));
    }
  }
  ~Staging() {
    cudaStreamSynchronize(ctx->stream);
    for (int k = 0; k < 2; k++) {
      if (done[k]) cudaEventDestroy(done[k]);
      if (buf[k]) cudaFreeHost(buf[k]);
    }
  }
  void upload(void* d, const uint8_t* h, size_t bytes) {
    int k = 0;
    for (size_t off = 0; off < bytes; off += chunk, k ^= 1) {
      const size_t len = std::min(chunk, bytes - off);
      PB_CUDA(cudaEventSynchronize(done[k]));  // the DMA out of this buffer (two chunks ago) has finished
      memcpy(buf[k], h + off, len);
      PB_CUDA(cudaMemcpyAsync((uint8_t*)d + off, buf[k], len, cudaMemcpyHostToDevice, ctx->stream));
      PB_CUDA(cudaEventRecord(done[k], ctx->stream));
    }
    PB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
};

// n points as stored (Montgomery x || y) -> HBM, refused unless checks 1 and 2 hold; `what` names a point in messages
DevBuf upload_checked(Context* ctx, const uint8_t* h, uint64_t n, const std::string& what) {
  PB_CHECK(n > 0, "empty SRS");
  PB_CHECK(n < (1ull << 31), "ptau: at most 2^31 - 1 points per load");
  auto t0 = std::chrono::steady_clock::now();
  DevBuf base(n * sizeof(G1Affine));
  {
    Staging st(ctx, n * sizeof(G1Affine));
    st.upload(base.p, h, n * sizeof(G1Affine));
  }
  g_stage_ms[ST_H2D] = ms_since(t0);
  DevBuf bad(8);
  PB_CUDA(cudaMemsetAsync(bad.p, 0xff, 8, ctx->stream));
  cudaEvent_t ev[2];
  PB_CUDA(cudaEventCreate(&ev[0]));
  PB_CUDA(cudaEventCreate(&ev[1]));
  cudaEventRecord(ev[0], ctx->stream);
  k_ptau_check_g1<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(base.as<G1Affine>(), (uint32_t)n,
                                                                       bad.as<uint32_t>());
  ctx->launches++;
  cudaEventRecord(ev[1], ctx->stream);
  uint32_t h_bad[2];
  cudaError_t e = cudaMemcpyAsync(h_bad, bad.p, 8, cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  float ms = 0;
  if (e == cudaSuccess) cudaEventElapsedTime(&ms, ev[0], ev[1]);
  cudaEventDestroy(ev[0]);
  cudaEventDestroy(ev[1]);
  PB_CUDA(e);
  PB_CUDA(cudaGetLastError());
  g_stage_ms[ST_CHECK] = ms;
  if (h_bad[0] != 0xffffffffu)
    refuse(what + " " + std::to_string(h_bad[0]) + " has a coordinate that is not below q");
  if (h_bad[1] != 0xffffffffu) {
    const uint8_t* p = h + 64 * (uint64_t)h_bad[1];
    bool zero = true;
    for (int k = 0; k < 64; k++) zero = zero && p[k] == 0;
    refuse(what + " " + std::to_string(h_bad[1]) + (zero ? " is the identity" : " is not on the curve"));
  }
  return base;
}

void os_random(uint8_t* out, size_t bytes) {
  size_t got = 0;
  while (got < bytes) {
    ssize_t r = getrandom(out + got, bytes - got, 0);
    if (r < 0) {
      PB_CHECK(errno == EINTR, "ptau: getrandom() failed (no fallback source is used)");
      continue;
    }
    got += (size_t)r;
  }
}

// `count` random canonical scalars below 2^128, then `zeros` zero scalars
std::vector<Fr> random_scalars128(uint64_t count, uint64_t zeros) {
  auto t0 = std::chrono::steady_clock::now();
  std::vector<Fr> s(count + zeros, Fr::zero());
  std::vector<uint8_t> raw((size_t)16 << 16);
  for (uint64_t i = 0; i < count; i += 1u << 16) {
    const uint64_t k = std::min<uint64_t>(1u << 16, count - i);
    os_random(raw.data(), 16 * k);
    for (uint64_t j = 0; j < k; j++) memcpy(s[i + j].v, raw.data() + 16 * j, 16);
  }
  g_stage_ms[ST_RANDOM] = ms_since(t0);
  return s;
}

G1Host g1_host(const uint8_t* xy_canonical, int is_identity) {
  G1Host p;
  p.inf = is_identity != 0;
  memcpy(p.x.v, xy_canonical, 32);
  memcpy(p.y.v, xy_canonical + 32, 32);
  p.x = fp_to_mont(p.x);
  p.y = fp_to_mont(p.y);
  return p;
}

// [tau]_2 as stored in section 3 (x.c0 x.c1 y.c0 y.c1, Montgomery): on the twist and in G2, or refused
G2Affine load_tau_g2(const uint8_t* h) {
  auto t0 = std::chrono::steady_clock::now();
  Fq c[4];
  for (int k = 0; k < 4; k++) {
    memcpy(c[k].v, h + 32 * k, 32);
    if (!fp_is_canonical(c[k])) refuse("[tau]_2 has a coordinate that is not below q");
  }
  G2Affine p{{c[0], c[1]}, {c[2], c[3]}, false};
  if (!g2_on_curve(p)) refuse("[tau]_2 is not on the twist curve");
  uint32_t r[8];
  for (int i = 0; i < 8; i++) r[i] = FrParams::p(i);
  if (!g2_mul(p, r).inf) refuse("[tau]_2 is not in G2 (r [tau]_2 is not the identity)");
  g_stage_ms[ST_G2] = ms_since(t0);
  return p;
}

G2Affine g2_generator() {
  static const uint32_t c[4][8] = {
      {0xd992f6edu, 0x46debd5cu, 0xf75edaddu, 0x674322d4u, 0x5e5c4479u, 0x426a0066u, 0x121f1e76u, 0x1800deefu},
      {0xaef312c2u, 0x97e485b7u, 0x35a9e712u, 0xf1aa4933u, 0x31fb5d25u, 0x7260bfb7u, 0x920d483au, 0x198e9393u},
      {0x66fa7daau, 0x4ce6cc01u, 0x0c43d37bu, 0xe3d1e769u, 0x8dcb408fu, 0x4aab7180u, 0xdb8c6debu, 0x12c85ea5u},
      {0xd122975bu, 0x55acdadcu, 0x70b38ef3u, 0xbc4b3133u, 0x690c3395u, 0xec9e99adu, 0x585ff075u, 0x090689d0u}};
  Fq f[4];
  for (int k = 0; k < 4; k++) {
    memcpy(f[k].v, c[k], 32);
    f[k] = fp_to_mont(f[k]);
  }
  return G2Affine{{f[0], f[1]}, {f[2], f[3]}, false};
}

// check 5: e(sum r_i G_{i+1}, G2) * e(-sum r_i G_i, [tau]_2) == 1
void check_powers(Context* ctx, Srs* srs, uint64_t n, const G2Affine& tau_g2) {
  if (n < 2) return;
  const std::vector<Fr> r = random_scalars128(n - 1, 1);  // r_0 .. r_(n-2), 0
  auto t0 = std::chrono::steady_clock::now();
  DevBuf s(2 * n * sizeof(Fr));
  Fr* s0 = s.as<Fr>();
  Fr* s1 = s0 + n;  // s1[i + 1] = r_i
  cudaStream_t st = ctx->stream;
  PB_CUDA(cudaMemcpyAsync(s0, r.data(), n * sizeof(Fr), cudaMemcpyHostToDevice, st));
  PB_CUDA(cudaMemsetAsync(s1, 0, sizeof(Fr), st));
  PB_CUDA(cudaMemcpyAsync(s1 + 1, s0, (n - 1) * sizeof(Fr), cudaMemcpyDeviceToDevice, st));
  const Fr* sc[2] = {s0, s1};
  uint8_t out[128];
  int ident[2];
  srs_msm_batch(ctx, srs, sc, 2, n, false, out, ident);
  g_stage_ms[ST_MSM] = ms_since(t0);
  t0 = std::chrono::steady_clock::now();
  G1Host lo = g1_host(out, ident[0]), hi = g1_host(out + 64, ident[1]);
  lo.y = fp_neg(lo.y);
  const bool ok = pairing_engine().product_is_one({hi, lo}, {g2_generator(), tau_g2});
  g_stage_ms[ST_PAIRING] = ms_since(t0);
  if (!ok) refuse("the tauG1 powers are not consistent with [tau]_2");
}

struct SrsDeleter {
  void operator()(Srs* s) const { srs_destroy(s); }
};

}  // namespace

Srs* srs_create_ptau(Context* ctx, const uint8_t* h_g1, uint64_t count, const uint8_t* h_tau_g2, int precompute) {
  for (double& t : g_stage_ms) t = 0;
  const G2Affine tau_g2 = load_tau_g2(h_tau_g2);
  DevBuf base = upload_checked(ctx, h_g1, count, "tauG1 point");
  const Fq one = Fq::one(), two = fp_add(one, one);
  if (memcmp(h_g1, one.v, 32) || memcmp(h_g1 + 32, two.v, 32)) refuse("tauG1 point 0 is not the generator (1, 2)");
  auto t0 = std::chrono::steady_clock::now();
  std::unique_ptr<Srs, SrsDeleter> srs(srs_adopt(ctx, std::move(base), count, precompute));
  g_stage_ms[ST_TABLE] = ms_since(t0);
  check_powers(ctx, srs.get(), count, tau_g2);
  return srs.release();
}

Srs* srs_create_ptau_lagrange(Context* ctx, const uint8_t* h_block, uint64_t n, Srs* monomial, int precompute) {
  for (double& t : g_stage_ms) t = 0;
  int log_n = 0;
  while (((uint64_t)1 << log_n) < n) log_n++;
  PB_CHECK(n > 0 && ((uint64_t)1 << log_n) == n, "ptau: a Lagrange block has a power-of-two size");
  if (srs_size(monomial) < n)
    refuse("the Lagrange block of size " + std::to_string(n) + " needs as many monomial powers, the SRS has " +
           std::to_string(srs_size(monomial)));
  DevBuf base = upload_checked(ctx, h_block, n, "Lagrange point");
  auto t0 = std::chrono::steady_clock::now();
  std::unique_ptr<Srs, SrsDeleter> srs(srs_adopt(ctx, std::move(base), n, precompute));
  g_stage_ms[ST_TABLE] = ms_since(t0);
  // values v (random, below 2^128) and coefficients c = iNTT(v) of the same polynomial f: [f(tau)] both ways
  const std::vector<Fr> v = random_scalars128(n, 0);
  t0 = std::chrono::steady_clock::now();
  DevBuf dv(n * sizeof(Fr)), dc(n * sizeof(Fr));
  PB_CUDA(cudaMemcpyAsync(dv.p, v.data(), n * sizeof(Fr), cudaMemcpyHostToDevice, ctx->stream));
  if (n == 1) PB_CUDA(cudaMemcpyAsync(dc.p, dv.p, sizeof(Fr), cudaMemcpyDeviceToDevice, ctx->stream));
  else ntt_run(ctx, dv.as<Fr>(), dc.as<Fr>(), log_n, true, n, nullptr, nullptr);
  uint8_t a[64], b[64];
  int ia = 0, ib = 0;
  srs_msm(ctx, srs.get(), dv.as<Fr>(), n, false, a, &ia);
  srs_msm(ctx, monomial, dc.as<Fr>(), n, false, b, &ib);
  g_stage_ms[ST_MSM] = ms_since(t0);
  if (ia != ib || (!ia && memcmp(a, b, 64)))
    refuse("the Lagrange block of size " + std::to_string(n) + " is not consistent with the tauG1 powers");
  return srs.release();
}

void ptau_stages(double* out_ms, int count) {
  for (int k = 0; k < count && k < ST_COUNT; k++) out_ms[k] = g_stage_ms[k];
}

}  // namespace pb200
