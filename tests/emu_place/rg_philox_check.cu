/* rg_philox_check.cu -- TEST INFRASTRUCTURE ONLY: the engine's device Philox4x32-10 (rg_place.inl) against cuRAND's
 * curand_Philox4x32_10 on the same counters and key, on the GPU.  rg_philox_mismatches returns how many of the n counters
 * (i, i * 7919, i >> 3, i ^ 0x5bd1e995 for i = 0..n-1) give a different output word, or -1 on a CUDA error. */
#include <curand_philox4x32_x.h>
#include "../../robogym_b200/csrc/rg_place.inl"

__global__ void rg_philox_cmp(int n, uint32_t k0, uint32_t k1, unsigned long long* bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t u = (uint32_t)i;
  const RgU4 c = {u, u * 7919u, u >> 3, u ^ 0x5bd1e995u};
  const RgU4 r = rg_philox(c, k0, k1);
  const uint4 q = curand_Philox4x32_10(make_uint4(c.x, c.y, c.z, c.w), make_uint2(k0, k1));
  if (r.x != q.x || r.y != q.y || r.z != q.z || r.w != q.w) atomicAdd(bad, 1ull);
}

extern "C" long long rg_philox_mismatches(int n, uint32_t k0, uint32_t k1) {
  unsigned long long* d = nullptr;
  unsigned long long h = 0;
  if (cudaMalloc(&d, sizeof h) != cudaSuccess) return -1;
  cudaMemset(d, 0, sizeof h);
  rg_philox_cmp<<<(n + 255) / 256, 256>>>(n, k0, k1, d);
  const cudaError_t e = cudaMemcpy(&h, d, sizeof h, cudaMemcpyDeviceToHost);
  cudaFree(d);
  return e == cudaSuccess ? (long long)h : -1;
}
