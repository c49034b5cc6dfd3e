/* rg_cta.cu -- the step kernel with ONE ENVIRONMENT PER CTA of W warps (W = 2, 4, 8, 16), for models whose scratch leaves room for
 * a single environment per SM (dactyl/full_perpendicular): the one-warp kernel would keep one warp of the SM busy.  The same
 * sources as rg_step_kernel, compiled with -DRG_COOP (rg_defs.h, "Cooperative sections"): warp 0 runs every stage, and the
 * dense loops of the Newton solve spread over the CTA with bit-identical results.  Linked into librobogym_b200.so next to
 * rg_engine.cu, which selects it per batch (rg_batch_size).
 */
#define RG_COOP 1
#include "rg_kernel.inl"

/* The kernel's code does not depend on W (the cooperative loops stride by blockDim.x); W only sets the register budget:
   255 registers per thread up to 8 warps, 128 at 16. */
template <int MAXW>
__global__ void __launch_bounds__(MAXW * 32, 1) rg_step_cta_kernel(const __grid_constant__ RgKernelArgs args) {
  __shared__ __align__(8) unsigned long long mbar;
  float* s = rg_kernel_stage(args, &mbar);
  RgModelDev* wm = (RgModelDev*)rg_smem_raw;
  float* wover = nullptr;
  if (args.nover > 0 || args.env_pairs) {   /* the environment's own model view + its override rows, behind its scratch */
    wm = (RgModelDev*)(s + args.L.total);
    wover = (float*)((unsigned char*)wm + RG_MODEL_DEV_BYTES);
  }
  __shared__ int sh_slot;
  const int total = args.nslots ? *args.nslots : args.io.nenv;
  for (;;) {
    __syncthreads();                                   /* everybody is done with the previous environment (and with sh_slot) */
    if (threadIdx.x == 0) { sh_slot = atomicAdd(args.counter, 1); rg_coop_seq = 0; }
    __syncthreads();
    const int slot = sh_slot;
    if (slot >= total) break;
    if (threadIdx.x >= 32) { rg_coop_worker(); continue; }
    const int e = args.order ? args.order[slot] : slot;
    if (args.nover > 0 || args.env_pairs) rg_kernel_env_view(args, wm, wover, e);
    rg_kernel_env(args, wm, s, e);
    rg_coop_post(RG_COOP_EXIT, RgCtx{}, 0, 0, 0, 0, 0, 0, nullptr);
  }
}

static const void* rg_cta_fn(int warps_per_env) {
  return warps_per_env > 8 ? (const void*)rg_step_cta_kernel<16> : (const void*)rg_step_cta_kernel<8>;
}

cudaError_t rg_cta_prepare(int warps_per_env, int optin_smem, int* static_smem) {
  cudaFuncAttributes fa;
  cudaError_t e = cudaFuncGetAttributes(&fa, rg_cta_fn(warps_per_env));
  if (e != cudaSuccess) return e;
  *static_smem = (int)fa.sharedSizeBytes;
  return cudaFuncSetAttribute(rg_cta_fn(warps_per_env), cudaFuncAttributeMaxDynamicSharedMemorySize, optin_smem - *static_smem);
}

cudaError_t rg_cta_launch(int warps_per_env, int ctas, int smem, cudaStream_t stream, const RgKernelArgs& args) {
  if (warps_per_env > 8) rg_step_cta_kernel<16><<<ctas, 32 * warps_per_env, smem, stream>>>(args);
  else rg_step_cta_kernel<8><<<ctas, 32 * warps_per_env, smem, stream>>>(args);
  return cudaGetLastError();
}
