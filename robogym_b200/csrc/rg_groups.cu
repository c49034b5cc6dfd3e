/* rg_groups.cu -- the object groups' kernel (rg_object_groups; the arithmetic is in rg_groups.inl, the ABI entry in
 * rg_engine.cu).  A translation unit of its own so that adding it leaves every kernel of rg_engine.cu as it was; it is
 * compiled with the engine's flags, which touch float32 arithmetic only, and its fp64 operations are explicitly rounded. */
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../include/robogym_b200.h"
#include "rg_groups.inl"

/* rg_object_groups: one thread per environment */
__global__ void __launch_bounds__(128) rg_groups_kernel(const __grid_constant__ RgGroupsArgs a) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.nenv || (a.mask && !a.mask[e])) return;
  rg_groups_env(a, (uint32_t)e);
}

/* copies the host inputs the kernel reads (palette, active counts, fixed counts) into one stream-ordered allocation, launches,
   and frees the allocation behind the launch; `a` holds the checked scalars and the outputs (rg_groups_check) */
static cudaError_t rg_groups_launch(const rg_groups_in* in, RgGroupsArgs a, const uint8_t* mask, cudaStream_t stream) {
  const size_t pal = (size_t)a.n_palette * 4 * sizeof(double), act = (size_t)a.nenv * sizeof(int);
  const size_t fix = in->group_mode == RG_GROUPS_FIXED ? (size_t)a.nenv * a.nobj * sizeof(int) : 0;
  char* buf = nullptr;
  cudaError_t e = cudaMallocAsync((void**)&buf, pal + act + fix, stream);
  if (e != cudaSuccess) return e;
  if (pal) e = cudaMemcpyAsync(buf, in->palette, pal, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(buf + pal, in->active, act, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess && fix) e = cudaMemcpyAsync(buf + pal + act, in->fixed_counts, fix, cudaMemcpyHostToDevice, stream);
  if (e == cudaSuccess) {
    a.palette = pal ? (const double*)buf : nullptr;
    a.active = (const int*)(buf + pal);
    a.fixed = fix ? (const int*)(buf + pal + act) : nullptr;
    a.mask = mask;
    rg_groups_kernel<<<(a.nenv + 127) / 128, 128, 0, stream>>>(a);
    e = cudaGetLastError();
  }
  const cudaError_t f = cudaFreeAsync(buf, stream);
  return e != cudaSuccess ? e : f;
}

/* rg_object_groups' work for rg_engine.cu, which keeps the error state: nullptr with *err the launch's CUDA status, or what is
   wrong with the arguments (nothing launched) */
const char* rg_groups_run(const rg_groups_in* in, const uint8_t* mask, int mask_len, const rg_groups_out* out, cudaStream_t stream, cudaError_t* err) {
  RgGroupsArgs a;
  memset(&a, 0, sizeof(a));
  const char* bad = rg_groups_check(in, mask_len, mask != nullptr, out, a);
  if (bad) return bad;
  *err = rg_groups_launch(in, a, mask, stream);
  return nullptr;
}
