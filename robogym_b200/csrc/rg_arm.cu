/* rg_arm.cu -- the arm controller's kernels (rg_arm_phase, rg_arm_sample_actions; the arithmetic is in rg_arm.inl).
 *
 * A translation unit of its own because its flags differ from the step kernel's: no -ftz, so subnormal operands and results
 * are kept as torch's float32 kernels keep them (under -ftz=true the rounded intrinsics become their .ftz forms and sinf / cosf
 * take their flush-to-zero paths), and -fmad=false besides the explicitly rounded intrinsics.  build.py compiles it to an
 * object and links it into the engine library. */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/robogym_b200.h"
#include "rg_arm.inl"

/* rg_arm_phase: one thread per environment */
__global__ void __launch_bounds__(128) rg_arm_kernel(const __grid_constant__ RgArmArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.nenv || (a.mask && !a.mask[e])) return;
  rg_arm_env(a, e);
}

/* rg_arm_sample_actions: one thread per (environment, component) */
__global__ void __launch_bounds__(128) rg_arm_sample_kernel(int nenv, int dim, uint32_t seed, uint32_t epoch, const uint8_t* mask, float* out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nenv * dim) return;
  const int e = i / dim, d = i - e * dim;
  if (mask && !mask[e]) return;
  out[i] = rg_arm_sample(seed, (uint32_t)e, epoch, (uint32_t)d);
}

cudaError_t rg_arm_launch(const RgArmArgs& a, cudaStream_t stream) {
  rg_arm_kernel<<<(a.nenv + 127) / 128, 128, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t rg_arm_sample_launch(int nenv, int dim, uint32_t seed, uint32_t epoch, const uint8_t* mask, float* out, cudaStream_t stream) {
  const int n = nenv * dim;
  rg_arm_sample_kernel<<<(n + 127) / 128, 128, 0, stream>>>(nenv, dim, seed, epoch, mask, out);
  return cudaGetLastError();
}
