// Copy-constraint permutation S1, S2, S3 of a circuit's wiring on the GPU (permutation.cuh has the definition):
//   1. the 3n ids are checked on the host and copied as they are into the key buffer; k_perm_keys turns each into
//      its key (id + 1) << cb | cell in place;
//   2. cub::DeviceRadixSort sorts the keys over the bits in use, [0, cb + bits(max id + 1)) (perm_sort_keys, which
//      solve.cu shares);
//   3. k_perm_label writes every cell's label (perm_label) from a table of omega^row, canonical.
// Device memory: two key buffers of 24n bytes (the sort ping-pongs between them), the 96n-byte output, the 32n-byte
// table and the sort's temporary storage, all freed before the call returns.  At 2^24: 0.8 GB of keys, 1.6 GB of
// output and 0.5 GB of table.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "permutation.cuh"

namespace pb200 {
// ntt.cu
void launch_powers(Context* ctx, Fr* out, uint64_t n, const Fr& base, const Fr& scale);
Fr fr_root_of_unity(int log_n);
// poly_ops.cu
void fr_from_mont(Context* ctx, const Fr* in, Fr* out, uint64_t n);

__global__ void k_perm_keys(uint64_t* keys, uint64_t m, int cb) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < m) keys[k] = perm_key((int64_t)keys[k], k, cb);
}

__global__ void k_perm_label(PermArgs a) {
  const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < a.m) perm_label(a, k);
}

// refuses an id outside [-1, PB_PERM_MAX_ID], naming its cell; *max_id: the largest id
void perm_require_ids(const int64_t* h_ids, uint64_t m, int64_t* max_id) {
  const int64_t bad = perm_check_ids(h_ids, m, max_id);
  if (bad >= 0) {
    char b[256];
    snprintf(b, sizeof b, "wire variable id %lld at cell %lld (row %lld, wire %c) is outside [-1, 2^32 - 2]",
             (long long)h_ids[bad], (long long)bad, (long long)(bad / 3), "LRO"[bad % 3]);
    throw Error(b);
  }
}

// the m ids at h_ids -> their keys, sorted over bits [0, end_bit), in keys or alt (the returned one).  temp: the sort's
// storage of temp_bytes.  Keys of ids at or past h_ids + m_ids (m_ids < m) are those of -1: rows past n_constraints.
uint64_t* perm_sort_keys(Context* ctx, const int64_t* h_ids, uint64_t m, int cb, int end_bit, DevBuf& keys, DevBuf& alt,
                         DevBuf& temp, size_t temp_bytes, uint64_t m_ids) {
  if (m_ids > m) m_ids = m;
  PB_CUDA(cudaMemcpyAsync(keys.p, h_ids, m_ids * 8, cudaMemcpyHostToDevice, ctx->stream));
  if (m_ids < m) PB_CUDA(cudaMemsetAsync(keys.as<uint64_t>() + m_ids, 0xff, (m - m_ids) * 8, ctx->stream));
  k_perm_keys<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(keys.as<uint64_t>(), m, cb);
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
  cub::DoubleBuffer<uint64_t> dbuf(keys.as<uint64_t>(), alt.as<uint64_t>());
  PB_CUDA(cub::DeviceRadixSort::SortKeys(temp.p, temp_bytes, dbuf, (int)m, 0, end_bit, ctx->stream));
  ctx->launches++;  // the sort's passes counted as one launch
  return dbuf.Current();
}

void permutation_run(Context* ctx, const int64_t* h_ids, int log_n, uint8_t* h_S) {
  PB_CHECK(log_n >= 1 && log_n <= 26, "group order must be 2^k, 1 <= k <= 26 (the prover's range)");
  const uint64_t n = (uint64_t)1 << log_n, m = 3 * n;
  const int cb = perm_cell_bits(log_n);
  int64_t max_id = -1;
  perm_require_ids(h_ids, m, &max_id);
  const int end_bit = perm_sort_bits(log_n, max_id);

  cub::DoubleBuffer<uint64_t> dbuf(nullptr, nullptr);
  size_t temp_bytes = 0;
  PB_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, temp_bytes, dbuf, (int)m, 0, end_bit, ctx->stream));
  DevBuf& temp = ctx->scratch[0];
  const uint64_t need = 2 * m * 8 + m * 32 + n * 32 + (temp.bytes < temp_bytes ? temp_bytes : 0);
  size_t free_b = 0, total_b = 0;
  PB_CUDA(cudaMemGetInfo(&free_b, &total_b));
  if (need > free_b) {
    char b[256];
    snprintf(b, sizeof b, "the permutation of 2^%d rows needs %llu bytes of device memory, %llu are free", log_n,
             (unsigned long long)need, (unsigned long long)free_b);
    throw Error(b);
  }

  temp.ensure(temp_bytes);
  DevBuf keys(m * 8), alt(m * 8), S(m * 32), wpow(n * 32);
  launch_powers(ctx, wpow.as<Fr>(), n, fr_root_of_unity(log_n), Fr::one());
  fr_from_mont(ctx, wpow.as<Fr>(), wpow.as<Fr>(), n);
  PermArgs a;
  a.keys = perm_sort_keys(ctx, h_ids, m, cb, end_bit, keys, alt, temp, temp_bytes, m);
  a.wpow = wpow.as<Fr>();
  a.S = S.as<Fr>();
  a.n = n;
  a.m = m;
  a.cb = cb;
  k_perm_label<<<(unsigned)((m + 255) / 256), 256, 0, ctx->stream>>>(a);
  ctx->launches++;
  PB_CUDA(cudaGetLastError());
  PB_CUDA(cudaMemcpyAsync(h_S, S.p, m * 32, cudaMemcpyDeviceToHost, ctx->stream));
  PB_CUDA(cudaStreamSynchronize(ctx->stream));
}

}  // namespace pb200
