// modmul throughput: canonical CIOS products (fp_mul) and dedicated squarings (fp_sqr), both fully reduced
#include <cstdio>
#include "field.cuh"
using namespace pb200;
template <class F, bool SQR>
__global__ void __launch_bounds__(256) k(F* sink, uint32_t iters, F seed) {
  uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  F a = seed, b = seed;
  a.v[0] ^= t; b.v[1] ^= t * 2654435761u; a.v[7] &= 0x0fffffffu; b.v[7] &= 0x0fffffffu;
  if (SQR) {
    for (uint32_t i = 0; i < iters; i += 2) { a = fp_sqr(a); b = fp_sqr(b); }  // two independent chains, as below
  } else {
    for (uint32_t i = 0; i < iters; i += 2) { a = fp_mul(a, b); b = fp_mul(b, a); }
  }
  F r = fp_add(a, b);
  if (r.v[0] == 0x12345678u && r.v[3] == 42u) sink[t & 1023] = r;
}
template <bool SQR>
float run(Fq* sink, unsigned blocks, uint32_t iters, cudaEvent_t e0, cudaEvent_t e1) {
  k<Fq, SQR><<<blocks, 256>>>(sink, iters, Fq::r2());
  cudaEventRecord(e0);
  k<Fq, SQR><<<blocks, 256>>>(sink, iters, Fq::r2());
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}
int main() {
  Fq* sink; cudaMalloc(&sink, 1024 * 32);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int threads_per_sm : {1024, 2048}) {
    unsigned blocks = sms * threads_per_sm / 256; uint32_t iters = 4096;
    const float ms = run<false>(sink, blocks, iters, e0, e1), ms_sqr = run<true>(sink, blocks, iters, e0, e1);
    printf("threads/SM %d: products %.3f ms  %.2f Gmul/s   squarings %.3f ms  %.2f Gsqr/s\n", threads_per_sm, ms,
           (double)blocks * 256 * iters / ms / 1e6, ms_sqr, (double)blocks * 256 * iters / ms_sqr / 1e6);
  }
  return 0;
}
