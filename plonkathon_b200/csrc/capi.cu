// extern "C" surface of libplonk_b200.so (declared in include/plonk_b200.h).
#include "../../include/plonk_b200.h"

#include <cstring>

#include "common.cuh"
#include "comm.cuh"
#include "msm_bucket.cuh"
#include "prover.cuh"
#include "pairing.cuh"
#include "solve.cuh"
#include "transcript.cuh"

namespace pb200 {
// ntt.cu
void ntt_run(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in, const Fr* in_scale,
             const Fr* out_scale);
void launch_powers(Context* ctx, Fr* out, uint64_t n, const Fr& base, const Fr& scale);
Fr fr_from_u64(uint64_t x);
void ntt_run_strided(Context* ctx, const Fr* in, Fr* out, int log_n, bool inverse, uint64_t n_in,
                     const Fr* in_scale, const Fr* out_scale, uint64_t in_mul, uint64_t in_add);
void ntt_sharded(Context* ctx, const Fr* const* in, Fr* const* out, int count, int log_n, bool inverse);
// poly_ops.cu
void fr_to_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
void fr_from_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);
void fr_vec_op(Context* ctx, int op, const Fr* a, const Fr* b, const Fr& scalar_canonical, Fr* out, uint64_t n,
               uint64_t shift);
void barycentric_eval(Context* ctx, const Fr* d_vals, int log_n, const Fr& x_mont, Fr* h_out);
float bench_modmul(Context* ctx, int field, uint64_t threads, uint32_t iters);
// msm.cu
struct Srs;
Srs* srs_create(Context* ctx, const uint8_t* h_points, uint64_t n, int precompute);
void srs_destroy(Srs* s);
Srs* srs_generate(Context* ctx, const Fr& tau_canonical, uint64_t n, int precompute);
Srs* srs_generate_lagrange(Context* ctx, const Fr& tau_canonical, uint64_t n, int precompute);
void srs_export(Context* ctx, Srs* srs, uint8_t* h_points, uint64_t first, uint64_t count);
void srs_msm(Context* ctx, Srs* srs, const Fr* d_scalars, uint64_t m, bool scalars_mont, uint8_t* out_xy, int* is_identity);
uint64_t srs_size(Srs* s);
uint32_t msm_default_window(uint64_t n, bool fixed_base);
void msm_init_device();
void msm_run(Context* ctx, const G1Affine* points, uint64_t n, const Fr* scalars, bool scalars_mont, uint32_t c,
             bool fixed_base, uint64_t point_stride, uint8_t* out_xy, int* is_identity);
void affine_to_mont(Context* ctx, const G1Affine* in, G1Affine* out, uint64_t n);
// prover.cu
Prover* prover_create(Context* ctx, Srs* srs, int log_n, const uint8_t* const* h_pk, int n_custom,
                      const uint8_t* h_exps, const uint8_t* const* h_custom, bool sharded, int exp_width);
void prover_destroy(Prover* p);
void prover_prove(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                  uint64_t n_public, uint8_t* out, bool wires_on_device);
void prover_round1(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                   uint64_t n_public, bool wires_on_device);
void prover_round2(Prover* P, const Fr* ch);
void prover_round3(Prover* P, const Fr& alpha_c, const Fr& cofactor_c);
void prover_round4(Prover* P, const Fr& zeta_c);
void prover_round5(Prover* P, const Fr& v_c);
void prover_serialize(const Prover* P, uint8_t* out);
size_t copy_step(const Prover* P, int step, uint8_t* out);
void prover_set_zk(Prover* P, unsigned block, bool enable, const uint8_t* h_blinders);
void prover_set_lookup(Prover* P, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* const* h_tab,
                       uint64_t rows);
void prover_round_lookup(Prover* P, const Fr& eta_c);
void prover_set_shuffle(Prover* P, const uint8_t* h_qin, const uint8_t* h_qout);
void g1_combine_partials_host(const G1XYZZ* parts, uint32_t count, uint8_t* out_xy, int* is_identity);
void host_join_bucket_shards(const SR* all, uint32_t world, uint32_t sets, uint32_t nloc, G1XYZZ* out);
void host_join_bucket_shards_strided(const SR* all, uint32_t world, uint32_t sets, G1XYZZ* out);
// check.cu
void prover_check(Prover* P, const uint8_t* hA, const uint8_t* hB, const uint8_t* hC, const uint8_t* h_public,
                  uint64_t n_public, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists, bool wires_on_device);
// permutation.cu
void permutation_run(Context* ctx, const int64_t* h_ids, int log_n, uint8_t* h_S);
// solve.cu
void solve_run(Context* ctx, const SolveArgs& a, const SolveTableArgs* tb, const SolveShuffleArgs* sf);
void solve_stages(double* out_ms, int count);
// ptau.cu
Srs* srs_create_ptau(Context* ctx, const uint8_t* h_g1, uint64_t count, const uint8_t* h_tau_g2, int precompute);
Srs* srs_create_ptau_lagrange(Context* ctx, const uint8_t* h_block, uint64_t n, Srs* monomial, int precompute);
void ptau_stages(double* out_ms, int count);

const Bn254Pairing& pairing_engine() {
  static const Bn254Pairing engine;  // constants derived once (thread-safe static initialisation)
  return engine;
}
}  // namespace pb200

using namespace pb200;

static thread_local std::string g_err;

#define PB_API_BEGIN try {
#define PB_API_END                        \
  return 0;                               \
  }                                       \
  catch (const std::exception& e) {       \
    g_err = e.what();                     \
    return 1;                             \
  }                                       \
  catch (...) {                           \
    g_err = "unknown error";              \
    return 1;                             \
  }

static Context* C(pb200_ctx* c) { return reinterpret_cast<Context*>(c); }

// Every entry point that touches the GPU runs on its context's device, whatever device the calling host thread had
// current (contexts on several GPUs in one process, provers driven from worker threads); the previous device is
// restored on the way out.
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(const Context* c) {
    int cur = -1;
    cudaGetDevice(&cur);
    if (cur != c->device) { cudaSetDevice(c->device); prev = cur; }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};
#define PB_ON_CTX(c) DeviceGuard guard__(c)

static Fr load_fr_canonical(const uint8_t* h) {
  Fr a;
  memcpy(a.v, h, 32);
  PB_CHECK(fp_is_canonical(a), "Fr value not reduced below the modulus");
  return a;
}

// ---- the proof-kind entry points ------------------------------------------------------------------------------------
// Each proof kind has its own prove, serialize and round entry points, so the size of the caller's buffer never
// depends on the prover's state.  An entry point of kind `kind` (a set of blocks, proof_layout.cuh) serves the provers
// that agree with it on the blocks adding fields to what it returns: one step's fields, or the whole proof.
static std::string kind_suffix(unsigned blocks) {
  std::string s;
  if (blocks & BLOCK_NEXT_ROW) s += "_next_row";
  if (blocks & BLOCK_SHUFFLE) s += "_shuffle";
  if (blocks & BLOCK_LOOKUP) s += "_lookup";
  return s;
}

// refuses a prover of another kind, naming its proof size and its entry point `fn`
static void require_kind(const Prover* P, unsigned kind, const char* fn, int step = -1, const char* note = "") {
  const unsigned blocks = P->blocks(), mask = step_blocks(step), have = blocks & mask;
  if (have == (kind & mask)) return;
  static const struct { unsigned block; const char *has, *lacks; } what[] = {
      {BLOCK_LOOKUP, "a lookup argument", "no lookup table"},
      {BLOCK_NEXT_ROW, "next-row custom gate terms", "no next-row custom gate terms"},
      {BLOCK_SHUFFLE, "a shuffle", "no shuffle"}};
  std::string msg = "this prover";
  const char* join = " has ";
  for (const auto& w : what)
    if ((have ^ kind) & mask & w.block) {
      msg += join;
      msg += have & w.block ? w.has : w.lacks;
      join = " and has ";
    }
  msg += ": its proofs have " + std::to_string(layout_bytes(blocks)) + " bytes";
  if (blocks & BLOCK_NEXT_ROW)
    msg += " (" + std::to_string(layout_bytes(blocks & ~BLOCK_NEXT_ROW)) + " without next-row terms, " +
           std::to_string(layout_bytes(blocks)) + " with next-row terms)";
  throw Error(msg + "; use pb200_prover_" + fn + kind_suffix(have) + note);
}

static int prove(pb200_prover* p, unsigned kind, const void* A, const void* B, const void* C, const uint8_t* h_public,
                 uint64_t n_public, uint8_t* out, bool wires_on_device = false) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  require_kind(P, kind, "prove", -1, wires_on_device ? " (wires in host memory)" : "");
  prover_prove(P, (const uint8_t*)A, (const uint8_t*)B, (const uint8_t*)C, h_public, n_public, out, wires_on_device);
  PB_API_END
}
static int serialize(pb200_prover* p, unsigned kind, uint8_t* out) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  require_kind(P, kind, "serialize");
  prover_serialize(P, out);
  PB_API_END
}
// x, y: theta and kappa for a shuffle, delta and epsilon for lookups
static int round2(pb200_prover* p, unsigned kind, const uint8_t* beta, const uint8_t* gamma, const uint8_t* x,
                  const uint8_t* y, uint8_t* out) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  require_kind(P, kind, "round2", STEP_2);
  Fr ch[PROOF_CHALLENGES] = {};
  ch[CH_BETA] = load_fr_canonical(beta);
  ch[CH_GAMMA] = load_fr_canonical(gamma);
  if (kind != BLOCK_PLAIN) {
    const bool sh = kind & BLOCK_SHUFFLE;
    ch[sh ? CH_THETA : CH_DELTA] = load_fr_canonical(x);
    ch[sh ? CH_KAPPA : CH_EPSILON] = load_fr_canonical(y);
  }
  prover_round2(P, ch);
  copy_step(P, STEP_2, out);
  PB_API_END
}
static int round4(pb200_prover* p, unsigned kind, const uint8_t* zeta, uint8_t* out) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  require_kind(P, kind, "round4", STEP_4);
  prover_round4(P, load_fr_canonical(zeta));
  copy_step(P, STEP_4, out);
  PB_API_END
}
static int set_zk(pb200_prover* p, unsigned block, int enable, const uint8_t* h_blinders) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  prover_set_zk(reinterpret_cast<Prover*>(p), block, enable != 0, h_blinders);
  PB_API_END
}

extern "C" {

const char* pb200_last_error(void) { return g_err.c_str(); }
const char* pb200_version(void) { return "plonk_b200 0.1 (sm_90a)"; }

int pb200_ctx_create(int device, void* cuda_stream, pb200_ctx** out) {
  PB_API_BEGIN
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  PB_CHECK(e == cudaSuccess && count > 0, "no CUDA device: libplonk_b200 has no CPU fallback");
  PB_CHECK(device >= 0 && device < count, "bad device ordinal");
  PB_CUDA(cudaSetDevice(device));
  auto ctx = std::make_unique<Context>();
  ctx->device = device;
  cudaDeviceProp prop;
  PB_CUDA(cudaGetDeviceProperties(&prop, device));
  ctx->sm_count = prop.multiProcessorCount;
  if (cuda_stream) {
    ctx->stream = reinterpret_cast<cudaStream_t>(cuda_stream);
  } else {
    PB_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
    ctx->own_stream = true;
  }
  int prio_least = 0, prio_greatest = 0;
  PB_CUDA(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
  PB_CUDA(cudaStreamCreateWithPriority(&ctx->prio_stream, cudaStreamNonBlocking, prio_greatest));
  PB_CUDA(cudaEventCreateWithFlags(&ctx->join_ev, cudaEventDisableTiming));
  msm_init_device();
  *out = reinterpret_cast<pb200_ctx*>(ctx.release());
  PB_API_END
}

void pb200_ctx_destroy(pb200_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(C(ctx)->device);
  cudaStreamSynchronize(C(ctx)->stream);
  delete C(ctx);
}

int pb200_ctx_sync(pb200_ctx* ctx) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CUDA(cudaStreamSynchronize(C(ctx)->stream));
  PB_API_END
}

uint64_t pb200_ctx_launches(pb200_ctx* ctx) { return C(ctx)->launches; }

int pb200_ctx_timing(pb200_ctx* ctx, int enable) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Context* c = C(ctx);
  PB_CUDA(cudaStreamSynchronize(c->stream));
  for (auto& v : c->timed) {
    for (auto& pr : v) { cudaEventDestroy(pr.first); cudaEventDestroy(pr.second); }
    v.clear();
  }
  c->timing = enable != 0;
  PB_API_END
}
int pb200_ctx_timing_read(pb200_ctx* ctx, int category, double* total_ms, uint64_t* count) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Context* c = C(ctx);
  PB_CHECK(category >= 0 && category < 4, "bad timing category");
  PB_CUDA(cudaStreamSynchronize(c->stream));
  double t = 0;
  for (auto& pr : c->timed[category]) {
    float ms = 0;
    PB_CUDA(cudaEventElapsedTime(&ms, pr.first, pr.second));
    t += ms;
  }
  *total_ms = t;
  *count = c->timed[category].size();
  PB_API_END
}
void* pb200_ctx_stream(pb200_ctx* ctx) { return (void*)C(ctx)->stream; }

int pb200_fr_to_mont(pb200_ctx* ctx, const void* d_in, void* d_out, uint64_t n) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  fr_to_mont(C(ctx), (const Fr*)d_in, (Fr*)d_out, n);
  PB_API_END
}
int pb200_fr_from_mont(pb200_ctx* ctx, const void* d_in, void* d_out, uint64_t n) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  fr_from_mont(C(ctx), (const Fr*)d_in, (Fr*)d_out, n);
  PB_API_END
}

int pb200_fr_vec_op(pb200_ctx* ctx, int op, const void* d_a, const void* d_b, const uint8_t* h_scalar, void* d_out,
                    uint64_t n, uint64_t shift) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Fr s = Fr::zero();
  if (h_scalar) s = load_fr_canonical(h_scalar);
  PB_CHECK(op < 4 ? d_b != nullptr : true, "missing second operand");
  fr_vec_op(C(ctx), op, (const Fr*)d_a, (const Fr*)d_b, s, (Fr*)d_out, n, shift);
  PB_API_END
}

int pb200_fr_ntt(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, int inverse) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  ntt_run(C(ctx), (const Fr*)d_in, (Fr*)d_out, (int)log_n, inverse != 0, (uint64_t)1 << log_n, nullptr, nullptr);
  PB_API_END
}

int pb200_fr_ntt_decimated(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_m, int inverse, uint64_t stride,
                           uint64_t offset) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(stride >= 1, "bad stride");
  ntt_run_strided(C(ctx), (const Fr*)d_in, (Fr*)d_out, (int)log_m, inverse != 0, (uint64_t)1 << log_m, nullptr, nullptr,
                  stride, offset);
  PB_API_END
}
int pb200_fr_ntt_sharded(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, int inverse) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  const Fr* in = (const Fr*)d_in;
  Fr* out = (Fr*)d_out;
  ntt_sharded(C(ctx), &in, &out, 1, (int)log_n, inverse != 0);
  PB_API_END
}

// ---- communicator ---------------------------------------------------------------------------------------------
int pb200_comm_unique_id(uint8_t* out128) {
  PB_API_BEGIN
  comm_unique_id(out128);
  PB_API_END
}
int pb200_comm_init(pb200_ctx* ctx, const uint8_t* id128, int rank, int world) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Context* c = C(ctx);
  PB_CHECK(!c->comm, "this context already has a communicator");
  c->comm = comm_create(id128, rank, world);
  PB_API_END
}
int pb200_comm_info(pb200_ctx* ctx, int* rank, int* world, uint64_t* collectives, uint64_t* bytes_received) {
  PB_API_BEGIN
  Context* c = C(ctx);
  *rank = c->comm ? c->comm->rank : 0;
  *world = c->comm ? c->comm->world : 1;
  *collectives = c->comm ? c->comm->collectives : 0;
  *bytes_received = c->comm ? c->comm->bytes_gathered : 0;
  PB_API_END
}

// staging helpers for the host-buffer entry points
struct HostStage {
  Context* ctx;
  DevBuf in, out;
  HostStage(Context* c, const uint8_t* h_in, size_t in_bytes, size_t out_bytes) : ctx(c), in(in_bytes), out(out_bytes) {
    if (in_bytes) PB_CUDA(cudaMemcpyAsync(in.p, h_in, in_bytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  void finish(uint8_t* h_out, size_t bytes) {
    PB_CUDA(cudaMemcpyAsync(h_out, out.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    PB_CUDA(cudaStreamSynchronize(ctx->stream));
  }
};

int pb200_fr_ntt_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n, int inverse) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  size_t bytes = ((size_t)1 << log_n) * 32;
  HostStage st(C(ctx), h_in, bytes, bytes);
  ntt_run(C(ctx), st.in.as<Fr>(), st.out.as<Fr>(), (int)log_n, inverse != 0, (uint64_t)1 << log_n, nullptr, nullptr);
  st.finish(h_out, bytes);
  PB_API_END
}

// poly.py:156-163: ifft(n) ; coefficient i *= offset^i ; zero-pad to 4n ; fft(4n)
static void coset_extend(Context* ctx, const Fr* d_in, Fr* d_out, int log_n, const uint8_t* h_offset) {
  uint64_t n = (uint64_t)1 << log_n;
  Fr off = fp_to_mont(load_fr_canonical(h_offset));
  DevBuf coeffs(n * 32), powers(n * 32);
  ntt_run(ctx, d_in, coeffs.as<Fr>(), log_n, true, n, nullptr, nullptr);
  launch_powers(ctx, powers.as<Fr>(), n, off, Fr::one());
  ntt_run(ctx, coeffs.as<Fr>(), d_out, log_n + 2, false, n, powers.as<Fr>(), nullptr);
  PB_CUDA(cudaStreamSynchronize(ctx->stream));  // temporaries die here
}

// poly.py:169-177: ifft(N) ; coefficient i *= offset^-i
static void coset_to_coeffs(Context* ctx, const Fr* d_in, Fr* d_out, int log_n, const uint8_t* h_offset) {
  uint64_t n = (uint64_t)1 << log_n;
  Fr off = fp_to_mont(load_fr_canonical(h_offset));
  Fr inv = fp_inv(off);  // inv(0) == 0 like py_ecc
  DevBuf powers(n * 32);
  launch_powers(ctx, powers.as<Fr>(), n, inv, Fr::one());
  ntt_run(ctx, d_in, d_out, log_n, true, n, nullptr, powers.as<Fr>());
  PB_CUDA(cudaStreamSynchronize(ctx->stream));
}

int pb200_fr_coset_extend(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, const uint8_t* h_offset) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  coset_extend(C(ctx), (const Fr*)d_in, (Fr*)d_out, (int)log_n, h_offset);
  PB_API_END
}
int pb200_fr_coset_extend_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n,
                               const uint8_t* h_offset) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  size_t bytes = ((size_t)1 << log_n) * 32;
  HostStage st(C(ctx), h_in, bytes, bytes * 4);
  coset_extend(C(ctx), st.in.as<Fr>(), st.out.as<Fr>(), (int)log_n, h_offset);
  st.finish(h_out, bytes * 4);
  PB_API_END
}
int pb200_fr_coset_to_coeffs(pb200_ctx* ctx, const void* d_in, void* d_out, unsigned log_n, const uint8_t* h_offset) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  coset_to_coeffs(C(ctx), (const Fr*)d_in, (Fr*)d_out, (int)log_n, h_offset);
  PB_API_END
}
int pb200_fr_coset_to_coeffs_host(pb200_ctx* ctx, const uint8_t* h_in, uint8_t* h_out, unsigned log_n,
                                  const uint8_t* h_offset) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  size_t bytes = ((size_t)1 << log_n) * 32;
  HostStage st(C(ctx), h_in, bytes, bytes);
  coset_to_coeffs(C(ctx), st.in.as<Fr>(), st.out.as<Fr>(), (int)log_n, h_offset);
  st.finish(h_out, bytes);
  PB_API_END
}

int pb200_fr_barycentric_eval(pb200_ctx* ctx, const void* d_vals, unsigned log_n, const uint8_t* h_x, uint8_t* h_out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Fr x = fp_to_mont(load_fr_canonical(h_x));
  Fr r;
  barycentric_eval(C(ctx), (const Fr*)d_vals, (int)log_n, x, &r);
  memcpy(h_out, r.v, 32);
  PB_API_END
}
int pb200_fr_barycentric_eval_host(pb200_ctx* ctx, const uint8_t* h_vals, unsigned log_n, const uint8_t* h_x,
                                   uint8_t* h_out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  size_t bytes = ((size_t)1 << log_n) * 32;
  HostStage st(C(ctx), h_vals, bytes, 0);
  Fr x = fp_to_mont(load_fr_canonical(h_x));
  Fr r;
  barycentric_eval(C(ctx), st.in.as<Fr>(), (int)log_n, x, &r);
  memcpy(h_out, r.v, 32);
  PB_API_END
}

int pb200_g1_msm(pb200_ctx* ctx, const void* d_points, const void* d_scalars, uint64_t n, uint8_t* h_out_xy,
                 int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(n > 0, "ec_lincomb of an empty list (the reference raises ValueError, curve.py:93)");
  Context* c = C(ctx);
  DevBuf mont(n * sizeof(G1Affine));
  affine_to_mont(c, (const G1Affine*)d_points, mont.as<G1Affine>(), n);
  msm_run(c, mont.as<G1Affine>(), n, (const Fr*)d_scalars, false, msm_default_window(n, false), false, 0, h_out_xy,
          is_identity);
  PB_API_END
}

int pb200_g1_msm_host(pb200_ctx* ctx, const uint8_t* h_points, const uint8_t* h_scalars, uint64_t n,
                      uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(n > 0, "ec_lincomb of an empty list (the reference raises ValueError, curve.py:93)");
  Context* c = C(ctx);
  DevBuf pts(n * 64), sc(n * 32);
  PB_CUDA(cudaMemcpyAsync(pts.p, h_points, n * 64, cudaMemcpyHostToDevice, c->stream));
  PB_CUDA(cudaMemcpyAsync(sc.p, h_scalars, n * 32, cudaMemcpyHostToDevice, c->stream));
  int rc = pb200_g1_msm(ctx, pts.p, sc.p, n, h_out_xy, is_identity);
  if (rc) throw Error(g_err);
  PB_API_END
}

int pb200_srs_create(pb200_ctx* ctx, const uint8_t* h_points, uint64_t n, int precompute, pb200_srs** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(n > 0, "empty SRS");
  *out = reinterpret_cast<pb200_srs*>(srs_create(C(ctx), h_points, n, precompute));
  PB_API_END
}
int pb200_srs_create_ptau(pb200_ctx* ctx, const uint8_t* h_g1, uint64_t count, const uint8_t* h_tau_g2, int precompute,
                          pb200_srs** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *out = reinterpret_cast<pb200_srs*>(srs_create_ptau(C(ctx), h_g1, count, h_tau_g2, precompute));
  PB_API_END
}
int pb200_srs_create_ptau_lagrange(pb200_ctx* ctx, const uint8_t* h_block, uint64_t n, pb200_srs* srs_monomial,
                                   int precompute, pb200_srs** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *out = reinterpret_cast<pb200_srs*>(
      srs_create_ptau_lagrange(C(ctx), h_block, n, reinterpret_cast<Srs*>(srs_monomial), precompute));
  PB_API_END
}
void pb200_srs_ptau_stages(double* ms, int count) { ptau_stages(ms, count); }
// Taus whose SRS would hold the identity are refused before any device work: tau = 0 makes [tau^i]G the identity for
// every i > 0, and tau^n = 1 makes L_i(tau) = 0 for all i but one.  The batched affine conversion cannot represent
// the identity (k_batch_to_affine), so such an SRS would commit to wrong points without an error.
int pb200_srs_generate(pb200_ctx* ctx, const uint8_t* h_tau, uint64_t n, int precompute, pb200_srs** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(n > 0, "empty SRS");
  const Fr tau = load_fr_canonical(h_tau);
  PB_CHECK(!tau.is_zero(), "tau == 0 mod r: every SRS point after the first would be the identity");
  *out = reinterpret_cast<pb200_srs*>(srs_generate(C(ctx), tau, n, precompute));
  PB_API_END
}
int pb200_srs_generate_lagrange(pb200_ctx* ctx, const uint8_t* h_tau, uint64_t n, int precompute, pb200_srs** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(n > 0, "empty SRS");
  const Fr tau = load_fr_canonical(h_tau);
  PB_CHECK(fp_pow_u64(fp_to_mont(tau), n) != Fr::one(),
           "tau^n == 1 mod r (tau is on the domain): every Lagrange point but one would be the identity");
  *out = reinterpret_cast<pb200_srs*>(srs_generate_lagrange(C(ctx), tau, n, precompute));
  PB_API_END
}
int pb200_srs_commit_coeffs_host(pb200_ctx* ctx, pb200_srs* srs, const uint8_t* h_coeffs, uint64_t m,
                                 uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  HostStage st(C(ctx), h_coeffs, (size_t)m * 32, 0);
  srs_msm(C(ctx), reinterpret_cast<Srs*>(srs), (const Fr*)st.in.p, m, false, h_out_xy, is_identity);
  PB_API_END
}
int pb200_srs_export(pb200_ctx* ctx, pb200_srs* srs, uint8_t* h_points, uint64_t first, uint64_t count) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  srs_export(C(ctx), reinterpret_cast<Srs*>(srs), h_points, first, count);
  PB_API_END
}
void pb200_srs_destroy(pb200_srs* srs) { srs_destroy(reinterpret_cast<Srs*>(srs)); }
uint64_t pb200_srs_size(pb200_srs* srs) { return srs_size(reinterpret_cast<Srs*>(srs)); }

int pb200_srs_commit_lagrange(pb200_ctx* ctx, pb200_srs* srs, const void* d_values, unsigned log_n, uint8_t* h_out_xy,
                              int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  Context* c = C(ctx);
  uint64_t n = (uint64_t)1 << log_n;
  PB_CHECK(n <= srs_size(reinterpret_cast<Srs*>(srs)), "Not enough powers in setup");
  DevBuf coeffs(n * 32);
  ntt_run(c, (const Fr*)d_values, coeffs.as<Fr>(), (int)log_n, true, n, nullptr, nullptr);
  srs_msm(c, reinterpret_cast<Srs*>(srs), coeffs.as<Fr>(), n, false, h_out_xy, is_identity);
  PB_API_END
}
int pb200_srs_commit_lagrange_host(pb200_ctx* ctx, pb200_srs* srs, const uint8_t* h_values, unsigned log_n,
                                   uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  size_t bytes = ((size_t)1 << log_n) * 32;
  HostStage st(C(ctx), h_values, bytes, 0);
  int rc = pb200_srs_commit_lagrange(ctx, srs, st.in.p, log_n, h_out_xy, is_identity);
  if (rc) throw Error(g_err);
  PB_API_END
}
int pb200_srs_commit_coeffs(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t m, int coeffs_montgomery,
                            uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  srs_msm(C(ctx), reinterpret_cast<Srs*>(srs), (const Fr*)d_coeffs, m, coeffs_montgomery != 0, h_out_xy, is_identity);
  PB_API_END
}

int pb200_prover_create(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                        pb200_prover** out) {
  return pb200_prover_create_custom(ctx, srs, log_n, h_pk, 0, nullptr, nullptr, out);
}
int pb200_prover_create_sharded(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                pb200_prover** out) {
  return pb200_prover_create_custom_sharded(ctx, srs, log_n, h_pk, 0, nullptr, nullptr, out);
}
int pb200_prover_create_custom(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                               unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                               pb200_prover** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *out = reinterpret_cast<pb200_prover*>(prover_create(C(ctx), reinterpret_cast<Srs*>(srs), (int)log_n, h_pk,
                                                       (int)n_custom, h_exps, h_custom, false, 3));
  PB_API_END
}
int pb200_prover_create_custom_next_row(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                        unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                                        pb200_prover** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *out = reinterpret_cast<pb200_prover*>(prover_create(C(ctx), reinterpret_cast<Srs*>(srs), (int)log_n, h_pk,
                                                       (int)n_custom, h_exps, h_custom, false, 6));
  PB_API_END
}
int pb200_prover_create_custom_sharded(pb200_ctx* ctx, pb200_srs* srs, unsigned log_n, const uint8_t* const* h_pk,
                                       unsigned n_custom, const uint8_t* h_exps, const uint8_t* const* h_custom,
                                       pb200_prover** out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *out = reinterpret_cast<pb200_prover*>(prover_create(C(ctx), reinterpret_cast<Srs*>(srs), (int)log_n, h_pk,
                                                       (int)n_custom, h_exps, h_custom, true, 3));
  PB_API_END
}
int pb200_permutation(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint8_t* h_S) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  permutation_run(C(ctx), h_ids, log_n, h_S);
  PB_API_END
}
int pb200_solve_wires(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                      const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                      const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                      const uint8_t* h_input_values, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists,
                      void* const* out, int out_on_device) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  const SolveArgs a{h_ids, log_n, n_constraints, h_sel, (int)n_custom, h_exps, h_custom, n_inputs, h_input_ids,
                    h_input_values, limit, h_counts, h_lists, out, out_on_device != 0};
  solve_run(C(ctx), a, nullptr, nullptr);
  PB_API_END
}
int pb200_solve_wires_lookup(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                             const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                             const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                             const uint8_t* h_input_values, const uint8_t* h_qk, const uint8_t* h_qtag,
                             const uint8_t* h_t1, const uint8_t* h_t2, const uint8_t* h_t3, const uint8_t* h_t4,
                             uint64_t table_rows, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists,
                             uint8_t* h_operands, void* const* out, int out_on_device) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  PB_CHECK(!h_qtag == !h_t4, "tagged lookups need both Q_T and the table tag column t4");
  const SolveArgs a{h_ids, log_n, n_constraints, h_sel, (int)n_custom, h_exps, h_custom, n_inputs, h_input_ids,
                    h_input_values, limit, h_counts, h_lists, out, out_on_device != 0};
  const SolveTableArgs tb{h_qk, h_qtag, {h_t1, h_t2, h_t3, h_t4}, table_rows, h_operands};
  solve_run(C(ctx), a, &tb, nullptr);
  PB_API_END
}
int pb200_solve_wires_shuffle(pb200_ctx* ctx, const int64_t* h_ids, int log_n, uint64_t n_constraints,
                              const uint8_t* const* h_sel, unsigned n_custom, const uint8_t* h_exps,
                              const uint8_t* const* h_custom, uint64_t n_inputs, const int64_t* h_input_ids,
                              const uint8_t* h_input_values, const uint8_t* h_qin, const uint8_t* h_qout,
                              uint32_t limit, uint64_t* h_counts, uint32_t* h_lists, void* const* out,
                              int out_on_device) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  const SolveArgs a{h_ids, log_n, n_constraints, h_sel, (int)n_custom, h_exps, h_custom, n_inputs, h_input_ids,
                    h_input_values, limit, h_counts, h_lists, out, out_on_device != 0};
  const SolveShuffleArgs sf{h_qin, h_qout};
  solve_run(C(ctx), a, nullptr, &sf);
  PB_API_END
}
void pb200_solve_shuffle_stages(double* ms, int count) { solve_stages(ms, count); }

void pb200_prover_destroy(pb200_prover* p) { prover_destroy(reinterpret_cast<Prover*>(p)); }
int pb200_prover_sliced(pb200_prover* p, int* out) {
  PB_API_BEGIN
  *out = reinterpret_cast<Prover*>(p)->sliced ? 1 : 0;
  PB_API_END
}

int pb200_prover_prove(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                       const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof768) {
  return prove(p, BLOCK_PLAIN, h_A, h_B, h_C, h_public, n_public, h_proof768);
}
int pb200_prover_prove_device(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                              const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof768) {
  return prove(p, BLOCK_PLAIN, d_A, d_B, d_C, h_public, n_public, h_proof768, true);
}
int pb200_prover_round1(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                        const uint8_t* h_public, uint64_t n_public, uint8_t* h_abc_xy) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  prover_round1(P, h_A, h_B, h_C, h_public, n_public, false);
  copy_step(P, STEP_1, h_abc_xy);
  PB_API_END
}
int pb200_prover_round2(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, uint8_t* h_z_xy) {
  return round2(p, BLOCK_PLAIN, beta, gamma, nullptr, nullptr, h_z_xy);
}
int pb200_prover_round3(pb200_prover* p, const uint8_t* alpha, const uint8_t* fft_cofactor, uint8_t* h_t_xy) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  prover_round3(P, load_fr_canonical(alpha), load_fr_canonical(fft_cofactor));
  copy_step(P, STEP_3, h_t_xy);
  PB_API_END
}
int pb200_prover_round4(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals) {
  return round4(p, BLOCK_PLAIN, zeta, h_evals);
}
int pb200_prover_round5(pb200_prover* p, const uint8_t* v, uint8_t* h_w_xy) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  prover_round5(P, load_fr_canonical(v));
  copy_step(P, STEP_5, h_w_xy);
  PB_API_END
}

int pb200_prover_read_vector(pb200_prover* p, int which, void* d_out) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  const Fr* src = nullptr;
  switch (which) {
    case 0: case 1: case 2: case 3: src = P->lag[which].as<Fr>(); break;   // A B C Z, Lagrange values
    case 4: src = P->pi_lag.as<Fr>(); break;                               // PI, Lagrange values
    case 5: case 6: case 7:  // T1 T2 T3, coefficients
      PB_CHECK(!P->zk, "T1, T2, T3 are not n-coefficient vectors in zero-knowledge mode (the blinded pieces have n + 1, "
                       "n + 1 and n + 6 coefficients)");
      src = P->tq.as<Fr>() + (uint64_t)(which - 5) * P->n;
      break;
    default: PB_CHECK(false, "unknown prover vector");
  }
  fr_from_mont(P->ctx, src, (Fr*)d_out, P->n);
  PB_CUDA(cudaStreamSynchronize(P->ctx->stream));
  PB_API_END
}
int pb200_prover_set_zk(pb200_prover* p, int enable, const uint8_t* h_blinders) {
  return set_zk(p, BLOCK_PLAIN, enable, h_blinders);
}
int pb200_prover_set_zk_lookup(pb200_prover* p, int enable, const uint8_t* h_blinders) {
  return set_zk(p, BLOCK_LOOKUP, enable, h_blinders);
}
int pb200_prover_set_zk_shuffle(pb200_prover* p, int enable, const uint8_t* h_blinders) {
  return set_zk(p, BLOCK_SHUFFLE, enable, h_blinders);
}
int pb200_prover_serialize(pb200_prover* p, uint8_t* h_proof768) { return serialize(p, BLOCK_PLAIN, h_proof768); }
int pb200_prover_set_lookup(pb200_prover* p, const uint8_t* h_qk, const uint8_t* h_t1, const uint8_t* h_t2,
                            const uint8_t* h_t3, uint64_t table_rows) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  const uint8_t* tab[4] = {h_t1, h_t2, h_t3, nullptr};
  prover_set_lookup(reinterpret_cast<Prover*>(p), h_qk, nullptr, tab, table_rows);
  PB_API_END
}
int pb200_prover_set_lookup_tagged(pb200_prover* p, const uint8_t* h_qk, const uint8_t* h_qtag, const uint8_t* h_t1,
                                   const uint8_t* h_t2, const uint8_t* h_t3, const uint8_t* h_t4, uint64_t table_rows) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  PB_CHECK(h_qtag && h_t4, "tagged lookups need Q_T and the table tag column t4");
  const uint8_t* tab[4] = {h_t1, h_t2, h_t3, h_t4};
  prover_set_lookup(reinterpret_cast<Prover*>(p), h_qk, h_qtag, tab, table_rows);
  PB_API_END
}
int pb200_prover_round_lookup(pb200_prover* p, const uint8_t* eta, uint8_t* h_fh_xy) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  Prover* P = reinterpret_cast<Prover*>(p);
  prover_round_lookup(P, load_fr_canonical(eta));
  copy_step(P, STEP_1L, h_fh_xy);
  PB_API_END
}
int pb200_prover_round2_lookup(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, const uint8_t* delta,
                               const uint8_t* epsilon, uint8_t* h_zz2_xy) {
  return round2(p, BLOCK_LOOKUP, beta, gamma, delta, epsilon, h_zz2_xy);
}
int pb200_prover_round4_lookup(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals) {
  return round4(p, BLOCK_LOOKUP, zeta, h_evals);
}
int pb200_prover_prove_lookup(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                              const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof1216) {
  return prove(p, BLOCK_LOOKUP, h_A, h_B, h_C, h_public, n_public, h_proof1216);
}
int pb200_prover_prove_device_lookup(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                     const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof1216) {
  return prove(p, BLOCK_LOOKUP, d_A, d_B, d_C, h_public, n_public, h_proof1216, true);
}
int pb200_prover_serialize_lookup(pb200_prover* p, uint8_t* h_proof1216) {
  return serialize(p, BLOCK_LOOKUP, h_proof1216);
}
int pb200_prover_round4_next_row(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals) {
  return round4(p, BLOCK_NEXT_ROW, zeta, h_evals);
}
int pb200_prover_prove_next_row(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                                const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof864) {
  return prove(p, BLOCK_NEXT_ROW, h_A, h_B, h_C, h_public, n_public, h_proof864);
}
int pb200_prover_prove_device_next_row(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                       const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof864) {
  return prove(p, BLOCK_NEXT_ROW, d_A, d_B, d_C, h_public, n_public, h_proof864, true);
}
int pb200_prover_serialize_next_row(pb200_prover* p, uint8_t* h_proof864) {
  return serialize(p, BLOCK_NEXT_ROW, h_proof864);
}
int pb200_prover_set_shuffle(pb200_prover* p, const uint8_t* h_qin, const uint8_t* h_qout) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  prover_set_shuffle(reinterpret_cast<Prover*>(p), h_qin, h_qout);
  PB_API_END
}
int pb200_prover_round2_shuffle(pb200_prover* p, const uint8_t* beta, const uint8_t* gamma, const uint8_t* theta,
                                const uint8_t* kappa, uint8_t* h_zz3_xy) {
  return round2(p, BLOCK_SHUFFLE, beta, gamma, theta, kappa, h_zz3_xy);
}
int pb200_prover_round4_shuffle(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals) {
  return round4(p, BLOCK_SHUFFLE, zeta, h_evals);
}
int pb200_prover_round4_next_row_shuffle(pb200_prover* p, const uint8_t* zeta, uint8_t* h_evals) {
  return round4(p, BLOCK_NEXT_ROW | BLOCK_SHUFFLE, zeta, h_evals);
}
int pb200_prover_prove_shuffle(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                               const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof896) {
  return prove(p, BLOCK_SHUFFLE, h_A, h_B, h_C, h_public, n_public, h_proof896);
}
int pb200_prover_prove_device_shuffle(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                      const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof896) {
  return prove(p, BLOCK_SHUFFLE, d_A, d_B, d_C, h_public, n_public, h_proof896, true);
}
int pb200_prover_serialize_shuffle(pb200_prover* p, uint8_t* h_proof896) {
  return serialize(p, BLOCK_SHUFFLE, h_proof896);
}
int pb200_prover_prove_next_row_shuffle(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                                        const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof992) {
  return prove(p, BLOCK_NEXT_ROW | BLOCK_SHUFFLE, h_A, h_B, h_C, h_public, n_public, h_proof992);
}
int pb200_prover_prove_device_next_row_shuffle(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                                               const uint8_t* h_public, uint64_t n_public, uint8_t* h_proof992) {
  return prove(p, BLOCK_NEXT_ROW | BLOCK_SHUFFLE, d_A, d_B, d_C, h_public, n_public, h_proof992, true);
}
int pb200_prover_serialize_next_row_shuffle(pb200_prover* p, uint8_t* h_proof992) {
  return serialize(p, BLOCK_NEXT_ROW | BLOCK_SHUFFLE, h_proof992);
}
int pb200_prover_check(pb200_prover* p, const uint8_t* h_A, const uint8_t* h_B, const uint8_t* h_C,
                       const uint8_t* h_public, uint64_t n_public, uint32_t limit, uint64_t* h_counts, uint32_t* h_lists) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  prover_check(reinterpret_cast<Prover*>(p), h_A, h_B, h_C, h_public, n_public, limit, h_counts, h_lists, false);
  PB_API_END
}
int pb200_prover_check_device(pb200_prover* p, const void* d_A, const void* d_B, const void* d_C,
                              const uint8_t* h_public, uint64_t n_public, uint32_t limit, uint64_t* h_counts,
                              uint32_t* h_lists) {
  PB_API_BEGIN PB_ON_CTX(reinterpret_cast<Prover*>(p)->ctx);
  prover_check(reinterpret_cast<Prover*>(p), (const uint8_t*)d_A, (const uint8_t*)d_B, (const uint8_t*)d_C, h_public,
               n_public, limit, h_counts, h_lists, true);
  PB_API_END
}
int pb200_g1_combine_partials_host(const uint8_t* h_xyzz, unsigned count, uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN
  std::vector<G1XYZZ> parts(count);
  memcpy(parts.data(), h_xyzz, (size_t)count * sizeof(G1XYZZ));
  g1_combine_partials_host(parts.data(), count, h_out_xy, is_identity);
  PB_API_END
}

int pb200_srs_commit_partial(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t first, uint64_t count,
                             uint32_t bucket_lo, uint32_t bucket_hi, int coeffs_montgomery, uint8_t* h_xyzz128) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  const Fr* sc = (const Fr*)d_coeffs;
  G1XYZZ part;
  srs_msm_batch_partial(C(ctx), reinterpret_cast<Srs*>(srs), &sc, 1, first, count, bucket_lo, bucket_hi,
                        coeffs_montgomery != 0, &part);
  memcpy(h_xyzz128, &part, sizeof(part));
  PB_API_END
}
int pb200_srs_bucket_count(pb200_srs* srs, uint32_t* out) {
  PB_API_BEGIN
  *out = srs_bucket_count(reinterpret_cast<Srs*>(srs));
  PB_API_END
}
int pb200_srs_commit_coeffs_sharded(pb200_ctx* ctx, pb200_srs* srs, const void* d_coeffs, uint64_t m,
                                    int coeffs_montgomery, uint8_t* h_out_xy, int* is_identity) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  const Fr* sc = (const Fr*)d_coeffs;
  srs_msm_batch_sharded(C(ctx), reinterpret_cast<Srs*>(srs), &sc, 1, m, coeffs_montgomery != 0, h_out_xy, is_identity);
  PB_API_END
}
int pb200_g1_join_bucket_shards_host(const uint8_t* h_sr, unsigned world, unsigned sets, uint32_t nloc, uint8_t* h_out_xy,
                                     int* is_identity) {
  PB_API_BEGIN
  std::vector<SR> all((size_t)world * sets);
  memcpy(all.data(), h_sr, all.size() * sizeof(SR));
  std::vector<G1XYZZ> ws(sets);
  if (nloc == 0) host_join_bucket_shards_strided(all.data(), world, sets, ws.data());
  else host_join_bucket_shards(all.data(), world, sets, nloc, ws.data());
  for (unsigned k = 0; k < sets; k++) g1_combine_partials_host(&ws[k], 1, h_out_xy + 64 * k, is_identity + k);
  PB_API_END
}

int pb200_transcript_create(const uint8_t* label, size_t label_len, pb200_transcript** out) {
  PB_API_BEGIN
  *out = reinterpret_cast<pb200_transcript*>(new Transcript(std::string((const char*)label, label_len)));
  PB_API_END
}
void pb200_transcript_destroy(pb200_transcript* t) { delete reinterpret_cast<Transcript*>(t); }
int pb200_transcript_append_message(pb200_transcript* t, const uint8_t* label, size_t label_len, const uint8_t* msg,
                                    size_t msg_len) {
  PB_API_BEGIN
  reinterpret_cast<Transcript*>(t)->append_message(std::string((const char*)label, label_len), msg, msg_len);
  PB_API_END
}
int pb200_transcript_challenge_bytes(pb200_transcript* t, const uint8_t* label, size_t label_len, uint8_t* out,
                                     size_t n) {
  PB_API_BEGIN
  reinterpret_cast<Transcript*>(t)->challenge_bytes(std::string((const char*)label, label_len), out, n);
  PB_API_END
}
int pb200_transcript_get_and_append_challenge(pb200_transcript* t, const uint8_t* label, size_t label_len,
                                              uint8_t* out_le32) {
  PB_API_BEGIN
  Fr f = reinterpret_cast<Transcript*>(t)->get_and_append_challenge(std::string((const char*)label, label_len));
  memcpy(out_le32, f.v, 32);
  PB_API_END
}

// ---- pairing / G2 (host code, pairing.cuh) ----
static Fq load_fq_canonical(const uint8_t* h) {
  Fq a;
  memcpy(a.v, h, 32);
  PB_CHECK(fp_is_canonical(a), "Fq value not reduced below the modulus");
  return fp_to_mont(a);
}
static G2Affine load_g2(const uint8_t* h, bool inf) {
  G2Affine q;
  q.inf = inf;
  q.x = {load_fq_canonical(h), load_fq_canonical(h + 32)};
  q.y = {load_fq_canonical(h + 64), load_fq_canonical(h + 96)};
  PB_CHECK(inf || g2_on_curve(q), "G2 point is not on the twist curve");
  return q;
}
static void store_g2(const G2Affine& q, uint8_t* out, int* is_identity) {
  *is_identity = q.inf ? 1 : 0;
  memset(out, 0, 128);
  if (q.inf) return;
  const Fq c[4] = {fp_from_mont(q.x.a), fp_from_mont(q.x.b), fp_from_mont(q.y.a), fp_from_mont(q.y.b)};
  for (int k = 0; k < 4; k++) memcpy(out + 32 * k, c[k].v, 32);
}
int pb200_pairing_check(const uint8_t* h_g1, const uint8_t* h_g1_identity, const uint8_t* h_g2,
                        const uint8_t* h_g2_identity, unsigned count, int* ok) {
  PB_API_BEGIN
  std::vector<G1Host> ps(count);
  std::vector<G2Affine> qs(count);
  const Fq three = fq_small(3);
  for (unsigned i = 0; i < count; i++) {
    ps[i].inf = h_g1_identity && h_g1_identity[i];
    if (!ps[i].inf) {
      ps[i].x = load_fq_canonical(h_g1 + 64 * i);
      ps[i].y = load_fq_canonical(h_g1 + 64 * i + 32);
      PB_CHECK(fp_sqr(ps[i].y) == fp_add(fp_mul(fp_sqr(ps[i].x), ps[i].x), three), "G1 point is not on the curve");
    }
    qs[i] = load_g2(h_g2 + 128 * i, h_g2_identity && h_g2_identity[i]);
  }
  *ok = pairing_engine().product_is_one(ps, qs) ? 1 : 0;
  PB_API_END
}
int pb200_g2_mul(const uint8_t* h_point, const uint8_t* h_scalar_le32, uint8_t* h_out, int* is_identity) {
  PB_API_BEGIN
  G2Affine p = load_g2(h_point, false);
  uint32_t k[8];
  memcpy(k, h_scalar_le32, 32);
  store_g2(g2_mul(p, k), h_out, is_identity);
  PB_API_END
}
int pb200_g2_add(const uint8_t* h_p, int p_identity, const uint8_t* h_q, int q_identity, uint8_t* h_out,
                 int* is_identity) {
  PB_API_BEGIN
  store_g2(g2_add(load_g2(h_p, p_identity != 0), load_g2(h_q, q_identity != 0)), h_out, is_identity);
  PB_API_END
}

int pb200_bench_modmul(pb200_ctx* ctx, int field, uint64_t threads, uint32_t iters, float* ms_out) {
  PB_API_BEGIN PB_ON_CTX(C(ctx));
  *ms_out = bench_modmul(C(ctx), field, threads, iters);
  PB_API_END
}

}  // extern "C"
