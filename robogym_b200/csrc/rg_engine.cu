/* rg_engine.cu -- sm_90a (H100) kernels + C ABI (include/robogym_b200.h) of the batched step engine.
 *
 * One persistent CTA per SM; each WARP owns one environment at a time and runs the whole fused
 * SimulationInterface.step() for it (robogym/mujoco/simulation_interface.py:176-189): state row
 * -> shared-memory scratch -> nsub x (kinematics, CRB mass matrix, RNE bias, tendons, PID,
 * collision, constraint rows, Newton solve, Euler) -> final forward -> state row + outputs.
 * The small per-model constant arrays are staged once per CTA into shared memory with a single
 * TMA bulk copy (cp.async.bulk + mbarrier); hull vertices / adjacency / pair list stay in global
 * memory behind the read-only path.  No tensor cores: nothing here is a dense contraction.
 */
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "../../include/robogym_b200.h"
#include "rg_step.inl"
#include "rg_place.inl"
#include "rg_goal.inl"
#include "rg_obs.inl"
#include "rg_arm.inl"
#include "rg_host.h"

/* The step kernel is built twice.  Registers are granted to a CTA in groups of four warps, so 12 warps (384 threads) may
   use 168 registers per thread, but 13 warps are granted the register file of 16 and get 128.  Up to RG_NARROW_WARPS warps
   per CTA run the 168-register build; a batch takes RG_MAX_WARPS only where the extra warp saves a round (rg_batch_size):
   held at 12 warps, the 128-register build is still about 5 % slower per warp (DESIGN.md section 4, "Residency").
   Shared memory decides how many fit. */
#ifndef RG_MAX_WARPS
#define RG_MAX_WARPS 13
#endif
#ifndef RG_NARROW_WARPS
#define RG_NARROW_WARPS 12
#endif
/* One environment per CTA of RG_CTA_WARPS warps (rg_cta.cu) for the models whose one-warp scratch leaves a single environment
   per SM and whose constraint solver has at least RG_CTA_MIN_NS dofs: there the dense solve is the part the other warps of the
   SM can take (DESIGN.md section 8, cfg 3).  RG_WARPS_PER_ENV=1|2|4|8|16 overrides the choice for any model. */
#ifndef RG_CTA_WARPS
#define RG_CTA_WARPS 8
#endif
#ifndef RG_CTA_MIN_NS
#define RG_CTA_MIN_NS 96
#endif

static thread_local std::string g_err;
static int rg_fail(int code, const std::string& msg) { g_err = msg; return code; }
#define RG_CUDA(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return rg_fail(-2, std::string(#call) + ": " + cudaGetErrorString(e_)); } while (0)

#include "rg_kernel.inl"

/* The step kernel's body.  SETTLE = the settle launch (rg_step_settle): the listed dofs' damping is overridden in the CTA's
   staged model and in each environment's own dof_damping row; every other line is the default kernel's. */
template <int MAXW, bool SETTLE>
__device__ __forceinline__ void rg_step_body(const RgKernelArgs& args, const RgSettleArgs* st) {
  __shared__ __align__(8) unsigned long long mbar;
  float* scratch0 = rg_kernel_stage(args, &mbar);
  if constexpr (SETTLE) {
    rg_settle_patch(*st, (float*)(rg_smem_raw + ((const RgModelDev*)rg_smem_raw)->dof_damping.off), threadIdx.x, blockDim.x);
    __syncthreads();
  }
  const int model_bytes = RG_MODEL_DEV_BYTES;
  const int warp = threadIdx.x >> 5;
  float* s = scratch0 + (size_t)warp * args.L.total;   /* L.total is a multiple of 4 floats: every per-warp area stays 16-byte aligned */
  /* with per-env overrides every warp keeps its own model view + a copy of this env's rows after the scratch */
  RgModelDev* wm = (RgModelDev*)rg_smem_raw;
  float* wover = nullptr;
  if (args.nover > 0 || args.env_pairs) {
    unsigned char* base = (unsigned char*)(scratch0 + (size_t)args.warps * args.L.total) + (size_t)warp * (model_bytes + 4 * args.over_floats);
    wm = (RgModelDev*)base;
    wover = (float*)(base + model_bytes);
  }
  /* Rounds: the CTA takes the next `warps` slots of the (cost-sorted) slot table from a device-wide counter, one slot per
     warp, and its warps walk the step in lock-step.  CTAs that finish early simply take more rounds (no static striding,
     no tail), and a partial last round runs with fewer warps instead of padding (the stage barriers count only the warps
     that hold an environment). */
  __shared__ int sh_slot0;
  const int total = args.nslots ? *args.nslots : args.io.nenv;
  for (;;) {
    __syncthreads();                                   /* everybody is done with the previous round (and with sh_slot0) */
    if (threadIdx.x == 0) sh_slot0 = atomicAdd(args.counter, args.warps);   /* (shrinking tail chunks measured worse: a round's length hardly depends on its warp count) */
    __syncthreads();
    const int slot0 = sh_slot0;
    if (slot0 >= total) break;
    const int nact = total - slot0 < args.warps ? total - slot0 : args.warps;
    if (threadIdx.x < nact) {                          /* warp w of this round: which barrier it meets at, with how many threads */
      const int w = threadIdx.x, G = args.groups < nact ? args.groups : nact;
      const int g = w * G / nact, lo = (g * nact + G - 1) / G, hi = ((g + 1) * nact + G - 1) / G;
      rg_bar_cfg[w] = ((1 + g) << 16) | (32 * (hi - lo));
    }
    __syncthreads();
    if (warp >= nact) continue;
    const int e = args.order ? args.order[slot0 + warp] : slot0 + warp;
    if (args.nover > 0 || args.env_pairs) rg_kernel_env_view(args, wm, wover, e);
    if constexpr (SETTLE) {
      if (st->row >= 0) { rg_settle_patch(*st, wover + st->row, threadIdx.x & 31, 32); __syncwarp(); }
    }
    rg_kernel_env(args, wm, s, e);
  }
}

template <int MAXW>
__global__ void __launch_bounds__(MAXW * 32, 1) rg_step_kernel(const __grid_constant__ RgKernelArgs args) {
  rg_step_body<MAXW, false>(args, nullptr);
}
/* the same kernel with the settle flag set (rg_step_settle) */
template <int MAXW>
__global__ void __launch_bounds__(MAXW * 32, 1) rg_settle_kernel(const __grid_constant__ RgKernelArgs args, const __grid_constant__ RgSettleArgs st) {
  rg_step_body<MAXW, true>(args, &st);
}

__global__ void rg_reset_kernel(RgModel m, RgBatchIO io, const uint8_t* mask) {
  const int env = blockIdx.x;
  if (env >= io.nenv || (mask && !mask[env])) return;
  for (int i = threadIdx.x; i < m.nq; i += blockDim.x) io.qpos[(size_t)env * m.nq + i] = m.qpos0[i];
  for (int i = threadIdx.x; i < m.nv; i += blockDim.x) { io.qvel[(size_t)env * m.nv + i] = 0.0f; io.warm[(size_t)env * m.nv + i] = 0.0f; }
  for (int i = threadIdx.x; i < m.nu; i += blockDim.x) io.ctrl[(size_t)env * m.nu + i] = 0.0f;
  for (int i = threadIdx.x; i < m.pidw * m.nu; i += blockDim.x) io.pid[(size_t)env * m.pidw * m.nu + i] = 0.0f;
  if (io.xfrc) for (int i = threadIdx.x; i < 6 * m.nbody; i += blockDim.x) ((float*)io.xfrc)[(size_t)env * 6 * m.nbody + i] = 0.0f;   /* mj_resetData clears xfrc_applied too */
  if (threadIdx.x == 0) { if (io.time) io.time[env] = 0.0f; if (io.warn) io.warn[env] = 0; }
}

/* Work-ordered scheduling.  The warps of a CTA meet at a barrier after every stage, so a CTA runs at the pace of
 * its slowest environment (most Newton iterations / narrow-phase pairs).  Contact configurations persist from one
 * env-step to the next, so the step kernel records a work estimate per environment and this kernel turns it into
 * the slot -> environment table of the NEXT launch (counting sort, one CTA): environments of similar cost share a
 * CTA.  Results do not depend on the table -- environments are independent -- only the barrier waits do. */
#define RG_ORDER_BINS 1024
__global__ void __launch_bounds__(1024) rg_order_kernel(const int* __restrict__ cost, int* __restrict__ order, int nenv) {
  __shared__ int bin[RG_ORDER_BINS];
  __shared__ int wsum[32];
  const int t = threadIdx.x;
  bin[t] = 0;
  __syncthreads();
  /* most expensive first: rounds are handed out in slot order, so the launch ends with the cheap environments (short tail) */
  for (int e = t; e < nenv; e += 1024) atomicAdd(&bin[RG_ORDER_BINS - 1 - min(max(cost[e], 0), RG_ORDER_BINS - 1)], 1);
  __syncthreads();
  /* exclusive scan of the 1024 bins */
  const int v = bin[t];
  int x = v;
  for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if ((t & 31) >= o) x += y; }
  if ((t & 31) == 31) wsum[t >> 5] = x;
  __syncthreads();
  if (t < 32) {
    int w = wsum[t];
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (t >= o) w += y; }
    wsum[t] = w;
  }
  __syncthreads();
  bin[t] = x - v + (t >= 32 ? wsum[(t >> 5) - 1] : 0);
  __syncthreads();
  for (int e = t; e < nenv; e += 1024) order[atomicAdd(&bin[RG_ORDER_BINS - 1 - min(max(cost[e], 0), RG_ORDER_BINS - 1)], 1)] = e;
}
/* slot table of a subset launch: the selected environments in ascending order (one CTA, ballot + scan compaction) */
__global__ void __launch_bounds__(1024) rg_subset_kernel(const uint8_t* __restrict__ mask, int* __restrict__ order, int* __restrict__ count, int nenv) {
  __shared__ int wsum[32];
  __shared__ int base;
  const int t = threadIdx.x;
  if (t == 0) base = 0;
  __syncthreads();
  for (int e0 = 0; e0 < nenv; e0 += 1024) {
    const int e = e0 + t;
    const int sel = e < nenv && mask[e] != 0;
    const unsigned bal = __ballot_sync(0xffffffffu, sel);
    if ((t & 31) == 0) wsum[t >> 5] = __popc(bal);
    __syncthreads();
    int before = base;
    for (int w = 0; w < (t >> 5); w++) before += wsum[w];
    if (sel) order[before + __popc(bal & ((1u << (t & 31)) - 1u))] = e;
    __syncthreads();
    if (t == 0) { int s = 0; for (int w = 0; w < 32; w++) s += wsum[w]; base += s; }
    __syncthreads();
  }
  if (t == 0) *count = base;
}
/* rg_batch_update_pairs: one warp per selected environment compacts the static pair list to the pairs whose geoms are both
   enabled in that environment's geom_dataid row (row stride 0: the shared row), clears its separating-axis cache, whose
   keys are indices into the list, and its "list is stale" flag.  `mask` may be the stale flags themselves (no __restrict__):
   every lane reads the environment's byte before lane 0 clears it. */
__global__ void __launch_bounds__(256) rg_pairs_kernel(RgModel m, const int* __restrict__ dataid, size_t stride, const uint8_t* mask, uint8_t* stale,
                                                       int nenv, unsigned* __restrict__ pairs, int* __restrict__ npair, int cap, int* __restrict__ sep, int* __restrict__ warn) {
  const int env = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (env >= nenv || (mask && !mask[env])) return;
  int w = 0;
  const int n = rg_env_pairs(m, dataid + (size_t)env * stride, pairs + (size_t)env * cap, cap, &w);
  for (int i = lane; i < RG_NSEP; i += 32) sep[(size_t)env * RG_NSEP + i] = 0xfff;
  if (lane == 0) { npair[env] = n; if (warn) warn[env] |= w; if (stale) stale[env] = 0; }
}
/* rg_batch_mark_pairs_stale with a mask */
__global__ void rg_mark_kernel(const uint8_t* __restrict__ mask, uint8_t* __restrict__ stale, int nenv) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < nenv && mask[e]) stale[e] = 1;
}
__global__ void rg_iota_kernel(int* order, int* cost, int* sep, int nenv) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e < nenv) { order[e] = e; cost[e] = 0; for (int i = 0; i < RG_NSEP; i++) sep[(size_t)e * RG_NSEP + i] = 0xfff; }
}

/* rg_batch_body_aabb: one warp per (environment, selected body); the lanes stride over the body's points, then a min / max
   reduction (exact, so the result does not depend on the order) */
struct RgAabbArgs {
  RgModel m;
  int nenv, nsel;
  int body[RG_AABB_MAXSEL];
  RgAabbRows rows;                 /* model arrays, or the first environment's bound rows ... */
  size_t stride[6];                /* ... and the row strides (0: the model's array) of dataid, pos, quat, size, mscale, gscale */
  const double* quat;              /* [nenv][nsel][4] */
  const uint8_t* mask;
  double* out;                     /* [nenv][nsel][2][3] */
};
__global__ void __launch_bounds__(256) rg_aabb_kernel(const __grid_constant__ RgAabbArgs a) {
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= a.nenv * a.nsel) return;
  const int env = w / a.nsel, k = w - env * a.nsel;
  if (a.mask && !a.mask[env]) return;
  RgAabbRows r = a.rows;
  r.dataid += env * a.stride[0]; r.pos += env * a.stride[1]; r.quat += env * a.stride[2]; r.size += env * a.stride[3];
  if (r.mscale) r.mscale += env * a.stride[4];
  if (r.gscale) r.gscale += env * a.stride[5];
  double R[9], lo[3], hi[3];
  rg_quat2mat_d(R, a.quat + (size_t)w * 4);
  rg_aabb_lane(a.m, r, a.body[k], R, lane, lo, hi);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    for (int c = 0; c < 3; c++) { lo[c] = fmin(lo[c], __shfl_xor_sync(0xffffffffu, lo[c], o)); hi[c] = fmax(hi[c], __shfl_xor_sync(0xffffffffu, hi[c], o)); }
  if (lane == 0) rg_aabb_finish(lo, hi, a.out + (size_t)w * 6);
}
/* rg_place_objects: one warp per selected environment */
__global__ void __launch_bounds__(128) rg_place_kernel(const __grid_constant__ RgPlaceArgs a) {
  const int env = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (env >= a.nenv || (a.mask && !a.mask[env])) return;
  rg_place_env(a, (uint32_t)env, threadIdx.x & 31);
}
/* rg_goal_modify: one thread per selected environment */
__global__ void __launch_bounds__(128) rg_modify_kernel(const __grid_constant__ RgModifyArgs a) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= a.nenv || (a.mask && !a.mask[env])) return;
  rg_modify_env(a, (uint32_t)env);
}
/* the arm controller's kernels live in rg_arm.cu, compiled without -ftz so that subnormals are kept as torch keeps them */
cudaError_t rg_arm_launch(const RgArmArgs& a, cudaStream_t stream);
cudaError_t rg_arm_sample_launch(int nenv, int dim, uint32_t seed, uint32_t epoch, const uint8_t* mask, float* out, cudaStream_t stream);
/* the object groups' kernel lives in rg_groups.cu: argument checks and launch (nullptr), or what is wrong with the arguments */
const char* rg_groups_run(const rg_groups_in* in, const uint8_t* mask, int mask_len, const rg_groups_out* out, cudaStream_t stream, cudaError_t* err);
/* rg_layout_goals: one warp per selected environment */
__global__ void __launch_bounds__(128) rg_layout_kernel(const __grid_constant__ RgLayoutArgs a) {
  const int env = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (env >= a.nenv || (a.mask && !a.mask[env])) return;
  rg_layout_env(a, (uint32_t)env, threadIdx.x & 31);
}
/* rg_rearrange_goal: one warp per selected environment, its working set in shared memory */
#define RG_GOAL_WARPS 4
__global__ void __launch_bounds__(32 * RG_GOAL_WARPS) rg_goal_kernel(const __grid_constant__ RgGoalArgs a) {
  __shared__ RgGoalScratch scratch[RG_GOAL_WARPS];
  const int w = threadIdx.x >> 5, env = blockIdx.x * RG_GOAL_WARPS + w;
  if (env >= a.nenv || (a.mask && !a.mask[env])) return;
  rg_goal_env(a, scratch[w], env, threadIdx.x & 31);
}
/* rg_goal_orientations: one warp per selected environment, a lane per slot */
__global__ void __launch_bounds__(128) rg_goal_rot_kernel(const __grid_constant__ RgGoalRotArgs a) {
  const int env = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (env >= a.nenv || (a.mask && !a.mask[env])) return;
  rg_goal_rot_env(a, env, threadIdx.x & 31);
}
/* rg_rearrange_obs: one warp per selected environment, no shared memory */
__global__ void __launch_bounds__(128) rg_obs_kernel(const __grid_constant__ RgObsArgs a) {
  const int env = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (env >= a.in.nenv || (a.mask && !a.mask[env])) return;
  rg_obs_env(a, env, threadIdx.x & 31);
}

/* ------------------------------------------------------------------ host objects */
struct rg_model {
  RgHostModel hm;
  RgModel dev;          /* same view with device pointers */
  char* d_arena = nullptr;
  int device = 0;
  RgLayout L;
  bool disabled_parts = false;   /* some mesh geom has geom_dataid -1: its batches always stream per-environment pair lists */
};
struct rg_batch {
  const rg_model* model;
  int nenv;
  void* ptr[RG_NFIELDS];
  int ctas, warps, smem;
  int env_warps = 1;       /* warps per environment: 1 = rg_step_kernel, 2..16 = rg_step_cta_kernel (one environment per CTA) */
  int nover = 0;
  int over_off[RG_MAX_PARAM_OVERRIDES], over_cnt[RG_MAX_PARAM_OVERRIDES], over_dst[RG_MAX_PARAM_OVERRIDES];
  int over_floats = 0;
  const float* over_ptr[RG_MAX_PARAM_OVERRIDES];
  std::string over_name[RG_MAX_PARAM_OVERRIDES];
  int* d_order = nullptr;  /* slot -> environment of the next launch */
  int* d_cost = nullptr;   /* work estimate written by the last launch */
  int* d_subset = nullptr; /* [nenv + 1] slot table of a subset launch, followed by its length */
  RgLayout L;              /* scratch layout for this batch's capacities */
  int* d_counter = nullptr; /* slot counter of the launch in flight */
  int* d_sep = nullptr;    /* [nenv][RG_NSEP] separating-axis cache of the narrow phase (speeds it up; results do not depend on it) */
  int balance = 1;
  int groups = 1;          /* barrier groups per round (rg_batch_set_barrier_groups) */
  unsigned* d_pairs = nullptr;  /* [nenv][pair_cap] per-environment pair lists (rg_batch_update_pairs), or nullptr */
  int* d_npair = nullptr;       /* [nenv] their lengths */
  int pair_cap = 0;
  uint8_t* d_stale = nullptr;   /* [nenv] the environment's geom_dataid row may have changed since its list was derived */
  bool any_stale = false;       /* some d_stale byte may be set: the next step rederives those lists first */
};

static void rg_wire_device_view(rg_model* mm) {
  mm->dev = mm->hm.view;
  const char* hbase = mm->hm.arena.data();
#define RG_DEVPTR(field) *(const void**)&mm->dev.field = (const void*)(mm->d_arena + ((const char*)mm->hm.view.field - hbase));
#define RG_DIM(n)
#define RG_I(n, c) RG_DEVPTR(n)
#define RG_F(n, c) RG_DEVPTR(n)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#define RG_DS(n, T, c) RG_DEVPTR(n)
#define RG_DSO(n, T, c, when) if (mm->hm.view.n) RG_DEVPTR(n)
#define RG_DG(n, T, c) RG_DEVPTR(n)
#include "rg_derived_fields.h"
#undef RG_DEVPTR
}

/* byte offset in RgModelDev of every array that lives in shared memory, which a warp's own view may point at a per-environment
   row instead (rg_batch_bind_param) */
static const struct { const char* name; int off; } rg_dev_arrays[] = {
#define RG_DIM(n)
#define RG_I(n, c) {#n, (int)offsetof(RgModelDev, n)},
#define RG_F(n, c) {#n, (int)offsetof(RgModelDev, n)},
#define RG_IB(n, c)
#define RG_FB(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#undef RG_IB
#undef RG_FB
#define RG_DS(n, T, c) {#n, (int)offsetof(RgModelDev, n)},
#define RG_DSO(n, T, c, when) {#n, (int)offsetof(RgModelDev, n)},
#define RG_DE(n, T, c) {#n, (int)offsetof(RgModelDev, n)},
#include "rg_derived_fields.h"
};

extern "C" {

const char* rg_last_error(void) { return g_err.c_str(); }

int rg_model_load(const void* blob, size_t len, int device, rg_model** out) {
  if (!blob || !out) return rg_fail(-1, "rg_model_load: null argument");
  rg_model* mm = new rg_model();
  std::string err;
  if (!rg_host_load(blob, len, mm->hm, err)) { delete mm; return rg_fail(-1, "rg_model_load: " + err); }
  mm->device = device;
  {
    const RgModel& v = mm->hm.view;
    for (int g = 0; g < v.ngeom; g++) {
      if (v.geom_type[g] != RG_GEOM_MESH) continue;
      if (v.geom_dataid[g] < -1 || v.geom_dataid[g] >= v.nmesh) { delete mm; return rg_fail(-1, "rg_model_load: geom_dataid of a mesh geom is neither -1 nor a mesh id"); }
      if (v.geom_dataid[g] == -1) mm->disabled_parts = true;
    }
    if (mm->disabled_parts && v.ngeom > 65536) { delete mm; return rg_fail(-1, "rg_model_load: disabled mesh parts need ngeom <= 65536 (16-bit ids in the pair lists)"); }
  }
  mm->L = rg_make_layout(mm->hm.view);
  cudaError_t e = cudaSetDevice(device);
  if (e == cudaSuccess) e = cudaMalloc((void**)&mm->d_arena, mm->hm.arena.size());
  if (e == cudaSuccess) e = cudaMemcpy(mm->d_arena, mm->hm.arena.data(), mm->hm.arena.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { std::string msg = std::string("rg_model_load: CUDA: ") + cudaGetErrorString(e); delete mm; return rg_fail(-2, msg); }
  rg_wire_device_view(mm);
  *out = mm;
  return 0;
}

void rg_model_destroy(rg_model* m) {
  if (!m) return;
  if (m->d_arena) cudaFree(m->d_arena);
  delete m;
}

int rg_model_dim(const rg_model* m, const char* name) {
  if (!m || !name) return -1;
#define RG_DIM(n) if (!strcmp(name, #n)) return m->hm.view.n;
#define RG_I(n, c)
#define RG_F(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  if (!strcmp(name, "npid")) return m->hm.view.pidw * m->hm.view.nu;   /* width of the RG_FIELD_PID row */
  return -1;
}

int rg_model_name2id(const rg_model* m, const char* objtype, const char* name) {
  if (!m || !objtype || !name) return -1;
  auto it = m->hm.names.find(objtype);
  if (it == m->hm.names.end()) return -1;
  for (size_t i = 0; i < it->second.size(); i++) if (it->second[i] == name) return (int)i;
  return -1;
}
const char* rg_model_id2name(const rg_model* m, const char* objtype, int id) {
  if (!m || !objtype) return nullptr;
  auto it = m->hm.names.find(objtype);
  if (it == m->hm.names.end() || id < 0 || (size_t)id >= it->second.size()) return nullptr;
  return it->second[(size_t)id].c_str();
}

int rg_model_set_field(rg_model* mm, const char* name, const void* data, size_t count) { return rg_model_set_field_async(mm, name, data, count, nullptr); }

int rg_model_set_field_async(rg_model* mm, const char* name, const void* data, size_t count, void* stream) {
  if (!mm || !name || !data) return rg_fail(-1, "rg_model_set_field: null argument");
  RgModel& m = mm->hm.view;
  if (!strcmp(name, "geom_mesh_scale"))
    return rg_fail(-1, "rg_model_set_field: geom_mesh_scale exists per environment only (rg_batch_bind_param); scale hulls model-wide with mesh_scale");
  const bool is_scale = !strcmp(name, "mesh_scale");   /* the one derived array of the engine that is a model parameter */
  RgHostField f;
  if (!rg_host_field(m, name, f) || (f.derived && !is_scale)) return rg_fail(-1, std::string("rg_model_set_field: unknown field ") + name);
  const size_t n = f.count;
  if (n != count) return rg_fail(-1, std::string("rg_model_set_field: size mismatch for ") + name);
  if (is_scale)
    for (size_t i = 0; i < n; i++)
      if (!(((const double*)data)[i] > 0.0) || !isfinite(((const double*)data)[i])) return rg_fail(-1, "rg_model_set_field: mesh_scale must be finite and positive");
  if (f.isint) memcpy(f.p, data, 4 * n);
  else {
    const double* s = (const double*)data;
    float* d = (float*)f.p;
    for (size_t i = 0; i < n; i++) d[i] = (float)s[i];
    if (!strcmp(name, "body_pos")) /* keep the fp32 world shift */
      for (int b = 1; b < m.nbody; b++)
        if (m.body_parentid[b] == 0) for (int a = 0; a < 3; a++) d[3 * b + a] = (float)(s[3 * b + a] - (double)m.origin[a]);
    if (!strcmp(name, "geom_pos")) for (int g = 0; g < m.ngeom; g++) if (m.geom_bodyid[g] == 0) for (int a = 0; a < 3; a++) d[3 * g + a] -= m.origin[a];
    if (!strcmp(name, "site_pos")) for (int k = 0; k < m.nsite; k++) if (m.site_bodyid[k] == 0) for (int a = 0; a < 3; a++) d[3 * k + a] -= m.origin[a];
  }
  RG_CUDA(cudaSetDevice(mm->device));
  /* stream-ordered: launches already queued on `stream` still see the old values, later ones the new; the host copy is
     pageable, so the runtime stages it before returning and `data` / the host arena may change right away */
  auto upload = [&](const char* array) {
    RgHostField u;
    rg_host_field(m, array, u);
    return cudaMemcpyAsync(mm->d_arena + ((const char*)u.p - mm->hm.arena.data()), u.p, 4 * u.count, cudaMemcpyHostToDevice, (cudaStream_t)stream);
  };
  RG_CUDA(upload(name));
  if (!strcmp(name, "mesh_vert")) {
    /* what the narrow phase derives from the hulls follows them: the float4-padded copy it scans, and the geom-frame box of
       every mesh geom that the OBB cull tests (the vertex bounding box, as the model compiler computes it) */
    rg_host_pad_verts(m);
    RG_CUDA(upload("mesh_vert4"));
    const double* v = (const double*)data;
    float* aabb = (float*)m.geom_aabb;
    for (int g = 0; g < m.ngeom; g++) {
      if (m.geom_type[g] != RG_GEOM_MESH) continue;
      const int mid = m.geom_dataid[g];
      if (mid < 0) continue;   /* a disabled part */
      const int a = m.mesh_vertadr[mid], nvt = m.mesh_vertnum[mid];
      for (int k = 0; k < 3 && nvt > 0; k++) {
        double lo = v[3 * a + k], hi = lo;
        for (int q = 1; q < nvt; q++) { lo = fmin(lo, v[3 * (a + q) + k]); hi = fmax(hi, v[3 * (a + q) + k]); }
        aabb[6 * g + k] = (float)(0.5 * (lo + hi));
        aabb[6 * g + 3 + k] = (float)(0.5 * (hi - lo));
      }
    }
    RG_CUDA(upload("geom_aabb"));
  }
  const bool vert = !strcmp(name, "mesh_vert"), layout = !strcmp(name, "mesh_vertadr") || !strcmp(name, "mesh_vertnum");
  if (vert || layout) {
    /* the hulls' support candidate lists follow their vertices; an edit of where the hulls are (vertadr / vertnum) switches
       every hull to the whole-hull scan instead (count -1), which needs no list */
    if (vert) rg_host_refresh_cells(m);
    else {
      m.ncand_cap = 0;
      rg_host_store_cells(m, std::vector<int>(2 * (size_t)m.nmesh * RG_NCELL, -1), std::vector<int>());
    }
    RG_CUDA(upload("mesh_cell"));
    if (m.ncand_cap > 0) RG_CUDA(upload("mesh_cand4"));
  }
  return 0;
}

int rg_dbg_size(const rg_model* m) { return m ? ::rg_dbg_size(m->hm.view, m->L.ncon) : -1; }
int rg_scratch_bytes(const rg_model* m) { return m ? 4 * m->L.total : -1; }

/* launch geometry: warps per CTA, dynamic shared memory, CTA count (re-run when the override set changes) */
static int rg_batch_size(rg_batch* b) {
  const rg_model* m = b->model;
  const int nenv = b->nenv;
  RG_CUDA(cudaSetDevice(m->device));
  int sms = 0, maxsmem = 0;
  RG_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->device));
  RG_CUDA(cudaDeviceGetAttribute(&maxsmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, m->device));
  cudaFuncAttributes fa;
  RG_CUDA(cudaFuncGetAttributes(&fa, rg_step_kernel<RG_MAX_WARPS>));   /* both builds declare the same static shared memory */
  maxsmem -= (int)fa.sharedSizeBytes;   /* the opt-in limit covers static + dynamic shared memory */
  const int model_bytes = RG_MODEL_DEV_BYTES;
  const int fixed = model_bytes + (int)((m->hm.small_bytes + 127) & ~(size_t)127) + 64;
  /* with per-env parameter overrides every warp also holds its own model view + this env's rows */
  const int per_warp = 4 * b->L.total + (b->nover > 0 || b->d_pairs ? model_bytes + 4 * b->over_floats : 0);
  int warps = (maxsmem - fixed) / per_warp;
  if (warps < 1) return rg_fail(-3, "rg_batch: model scratch does not fit in shared memory");
  int env_warps = warps == 1 && m->hm.view.ns >= RG_CTA_MIN_NS ? RG_CTA_WARPS : 1;
  const char* eenv = getenv("RG_WARPS_PER_ENV");
  if (eenv) {
    const int w = atoi(eenv);
    if (w == 1 || w == 2 || w == 4 || w == 8 || w == 16) env_warps = w;
  }
  b->env_warps = env_warps;
  if (env_warps > 1) {
    int cta_static = 0;
    RG_CUDA(rg_cta_prepare(env_warps, maxsmem + (int)fa.sharedSizeBytes, &cta_static));   /* (the opt-in limit, less its own static shared memory) */
    if (per_warp + fixed > maxsmem + (int)fa.sharedSizeBytes - cta_static) return rg_fail(-3, "rg_batch: model scratch does not fit in shared memory");
    b->warps = 1;   /* environments per CTA */
    b->smem = fixed - 64 + per_warp;
    b->ctas = nenv < sms ? nenv : sms;
    return 0;
  }
  if (warps > RG_MAX_WARPS) warps = RG_MAX_WARPS;
  /* rounds are handed out dynamically and a partial round runs with fewer warps, so more resident warps never cost padding */
  if (warps > nenv) warps = nenv;
  /* past RG_NARROW_WARPS every warp has fewer registers (see RG_MAX_WARPS): worth it only where the launch takes fewer rounds.
     dactyl/locked's 8192 environments take 5 rounds of 132 x 13 instead of 6 of 132 x 12 */
  if (warps > RG_NARROW_WARPS && (nenv + sms * warps - 1) / (sms * warps) >= (nenv + sms * RG_NARROW_WARPS - 1) / (sms * RG_NARROW_WARPS))
    warps = RG_NARROW_WARPS;
  /* a batch smaller than one full round is spread over all SMs (fewer warps per CTA) rather than packed into few of them:
     a round lasts as long as its slowest environment, and fewer resident warps make every one of them faster */
  if (nenv < sms * warps) { const int even = (nenv + sms - 1) / sms; if (even < warps) warps = even; }
  const char* wenv = getenv("RG_WARPS_PER_CTA");
  if (wenv && atoi(wenv) > 0 && atoi(wenv) <= RG_MAX_WARPS && per_warp * atoi(wenv) + fixed <= maxsmem) warps = atoi(wenv);
  b->warps = warps;
  b->smem = fixed - 64 + warps * per_warp;
  int ctas = (nenv + warps - 1) / warps;
  /* experiment hook: RG_CTAS_PER_SM=2 with RG_WARPS_PER_CTA=4 runs two independent barrier domains per SM */
  const char* cenv = getenv("RG_CTAS_PER_SM");
  const int per_sm = cenv && atoi(cenv) > 0 ? atoi(cenv) : 1;
  if (ctas > sms * per_sm) ctas = sms * per_sm;
  b->ctas = ctas;
  /* the attribute belongs to the kernel, not to this batch: batches with different footprints coexist, so opt in to the
     device maximum once rather than to this batch's size */
  RG_CUDA(cudaFuncSetAttribute(rg_step_kernel<RG_NARROW_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsmem));
  RG_CUDA(cudaFuncSetAttribute(rg_step_kernel<RG_MAX_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsmem));
  RG_CUDA(cudaFuncSetAttribute(rg_settle_kernel<RG_NARROW_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsmem));
  RG_CUDA(cudaFuncSetAttribute(rg_settle_kernel<RG_MAX_WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, maxsmem));
  return 0;
}

/* (re)allocate the per-environment pair lists with `cap` entries each (set-up call: synchronises) */
static int rg_pairs_alloc(rg_batch* b, int cap) {
  RG_CUDA(cudaSetDevice(b->model->device));
  if (b->d_pairs) { RG_CUDA(cudaFree(b->d_pairs)); b->d_pairs = nullptr; }
  if (!b->d_npair) RG_CUDA(cudaMalloc((void**)&b->d_npair, sizeof(int) * (size_t)b->nenv));
  if (!b->d_stale) { RG_CUDA(cudaMalloc((void**)&b->d_stale, (size_t)b->nenv)); RG_CUDA(cudaMemset(b->d_stale, 0, (size_t)b->nenv)); }
  b->pair_cap = cap > 0 ? cap : (b->model->hm.view.npair > 0 ? b->model->hm.view.npair : 1);
  RG_CUDA(cudaMalloc((void**)&b->d_pairs, sizeof(unsigned) * (size_t)b->nenv * b->pair_cap));
  return 0;
}
/* every environment's list from the shared geom_dataid row (a model with disabled parts, no per-environment row bound) */
static int rg_pairs_from_shared(rg_batch* b) {
  const rg_model* m = b->model;
  rg_pairs_kernel<<<(b->nenv + 7) / 8, 256>>>(m->dev, m->dev.geom_dataid, 0, nullptr, b->d_stale, b->nenv, b->d_pairs, b->d_npair, b->pair_cap, b->d_sep,
                                              (int*)b->ptr[RG_FIELD_WARN]);
  RG_CUDA(cudaGetLastError());
  RG_CUDA(cudaDeviceSynchronize());
  b->any_stale = false;
  return 0;
}
/* every list stale: derived from the per-environment rows before the next step (set-up call: synchronises) */
static int rg_pairs_all_stale(rg_batch* b) {
  RG_CUDA(cudaMemset(b->d_stale, 1, (size_t)b->nenv));
  b->any_stale = true;
  return 0;
}
static int rg_find_override(const rg_batch* b, const char* name) {
  for (int i = 0; i < b->nover; i++) if (b->over_name[i] == name) return i;
  return -1;
}

int rg_batch_create(const rg_model* m, int nenv, rg_batch** out) { return rg_batch_create_ex(m, nenv, 0, 0, 0, out); }

int rg_batch_create_ex(const rg_model* m, int nenv, int contact_capacity, int row_capacity, int dofs_per_contact, rg_batch** out) {
  if (!m || !out || nenv <= 0 || contact_capacity < 0 || row_capacity < 0 || dofs_per_contact < 0) return rg_fail(-1, "rg_batch_create: bad argument");
  rg_batch* b = new rg_batch();
  b->model = m;
  b->nenv = nenv;
  b->L = rg_make_layout(m->hm.view, contact_capacity ? contact_capacity : RG_NCON, row_capacity ? row_capacity : RG_NEL, dofs_per_contact ? dofs_per_contact : RG_TILE);
  for (int i = 0; i < RG_NFIELDS; i++) b->ptr[i] = nullptr;
  const int rc = rg_batch_size(b);
  if (rc) { delete b; return rc; }
  const char* benv = getenv("RG_BALANCE");
  if (benv) b->balance = atoi(benv) != 0;
  const char* genv = getenv("RG_BAR_GROUPS");
  if (genv && atoi(genv) >= 1 && atoi(genv) <= 12) b->groups = atoi(genv);
  cudaError_t e = cudaMalloc((void**)&b->d_order, sizeof(int) * (size_t)nenv);
  if (e == cudaSuccess) e = cudaMalloc((void**)&b->d_cost, sizeof(int) * (size_t)nenv);
  if (e == cudaSuccess) e = cudaMalloc((void**)&b->d_subset, sizeof(int) * ((size_t)nenv + 1));
  if (e == cudaSuccess) e = cudaMalloc((void**)&b->d_counter, sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc((void**)&b->d_sep, sizeof(int) * (size_t)nenv * RG_NSEP);
  if (e == cudaSuccess) { rg_iota_kernel<<<(nenv + 255) / 256, 256>>>(b->d_order, b->d_cost, b->d_sep, nenv); e = cudaDeviceSynchronize(); }   /* set-up call: may synchronise (the stepping calls never do) */
  if (e != cudaSuccess) { std::string msg = std::string("rg_batch_create: CUDA: ") + cudaGetErrorString(e); rg_batch_destroy(b); return rg_fail(-2, msg); }
  if (m->disabled_parts) {   /* the static list holds disabled parts: stream the shared draw's own pairs from the start */
    int rc2 = rg_pairs_alloc(b, 0);
    if (!rc2) rc2 = rg_batch_size(b);
    if (!rc2) rc2 = rg_pairs_from_shared(b);
    if (rc2) { const std::string msg = g_err; rg_batch_destroy(b); return rg_fail(rc2, msg); }
  }
  *out = b;
  return 0;
}
void rg_batch_destroy(rg_batch* b) {
  if (!b) return;
  if (b->d_order) cudaFree(b->d_order);
  if (b->d_cost) cudaFree(b->d_cost);
  if (b->d_subset) cudaFree(b->d_subset);
  if (b->d_sep) cudaFree(b->d_sep);
  if (b->d_counter) cudaFree(b->d_counter);
  if (b->d_pairs) cudaFree(b->d_pairs);
  if (b->d_npair) cudaFree(b->d_npair);
  if (b->d_stale) cudaFree(b->d_stale);
  delete b;
}

int rg_batch_set_balance(rg_batch* b, int on) {
  if (!b) return rg_fail(-1, "rg_batch_set_balance: null argument");
  b->balance = on != 0;
  return 0;
}

int rg_batch_bind(rg_batch* b, int field, void* p) {
  if (!b || field < 0 || field >= RG_NFIELDS) return rg_fail(-1, "rg_batch_bind: bad argument");
  b->ptr[field] = p;
  return 0;
}
int rg_model_origin(const rg_model* m, float origin[3]) {
  if (!m || !origin) return rg_fail(-1, "rg_model_origin: null argument");
  for (int a = 0; a < 3; a++) origin[a] = m->hm.view.origin[a];
  return 0;
}

int rg_batch_bind_param(rg_batch* b, const char* name, void* p) {
  if (!b || !name) return rg_fail(-1, "rg_batch_bind_param: null argument");
  const RgModel& m = b->model->hm.view;
  int off = -1;
  for (const auto& a : rg_dev_arrays) if (!strcmp(name, a.name)) off = a.off;
  const bool dataid = !strcmp(name, "geom_dataid");   /* the one int array: per-environment mesh draws (rg_batch_update_pairs) */
  RgHostField f;
  if (off < 0 || !rg_host_field(m, name, f) || (f.isint && !dataid))
    return rg_fail(-1, std::string("rg_batch_bind_param: not a (small) float model array: ") + name);
  const int cnt = (int)f.count;
  if (dataid && m.ngeom > 65536) return rg_fail(-1, "rg_batch_bind_param: geom_dataid per environment needs ngeom <= 65536 (16-bit ids in the pair lists)");
  int slot = -1;
  for (int i = 0; i < b->nover; i++) if (b->over_name[i] == name) slot = i;
  if (!p) {
    if (slot < 0) return 0;
    for (int i = slot; i + 1 < b->nover; i++) { b->over_off[i] = b->over_off[i + 1]; b->over_cnt[i] = b->over_cnt[i + 1]; b->over_ptr[i] = b->over_ptr[i + 1]; b->over_name[i] = b->over_name[i + 1]; }
    b->nover--;
  } else {
    if (slot < 0) { if (b->nover >= RG_MAX_PARAM_OVERRIDES) return rg_fail(-3, "rg_batch_bind_param: too many overrides"); slot = b->nover++; }
    b->over_off[slot] = off; b->over_cnt[slot] = cnt; b->over_ptr[slot] = (const float*)p; b->over_name[slot] = name;
  }
  int fl = 0;
  for (int i = 0; i < b->nover; i++) { b->over_dst[i] = fl; fl += (b->over_cnt[i] + 3) & ~3; }
  b->over_floats = fl;
  if (dataid && p) {
    /* the rows are the caller's to fill: every list is rederived from them before the next step (or by rg_batch_update_pairs) */
    if (!b->d_pairs) { const int rc = rg_pairs_alloc(b, 0); if (rc) return rc; }
    const int rc = rg_pairs_all_stale(b);
    if (rc) return rc;
  }
  const int rc = rg_batch_size(b);
  if (rc || !dataid || p) return rc;
  if (!b->model->disabled_parts) {   /* back to the static list */
    if (b->d_pairs) { cudaFree(b->d_pairs); b->d_pairs = nullptr; }
    b->any_stale = false;
    return rg_batch_size(b);
  }
  return rg_pairs_from_shared(b);
}

int rg_batch_set_pair_capacity(rg_batch* b, int capacity) {
  if (!b || capacity < 0) return rg_fail(-1, "rg_batch_set_pair_capacity: bad argument");
  if (!b->d_pairs) return rg_fail(-1, "rg_batch_set_pair_capacity: the batch has no per-environment pair lists (bind geom_dataid first)");
  int rc = rg_pairs_alloc(b, capacity);
  if (rc) return rc;
  if (rg_find_override(b, "geom_dataid") >= 0) return rg_pairs_all_stale(b);
  return rg_pairs_from_shared(b);
}

int rg_batch_mark_pairs_stale(rg_batch* b, const uint8_t* mask, void* stream) {
  if (!b) return rg_fail(-1, "rg_batch_mark_pairs_stale: null argument");
  if (rg_find_override(b, "geom_dataid") < 0 || !b->d_pairs) return rg_fail(-1, "rg_batch_mark_pairs_stale: geom_dataid is not bound per environment (rg_batch_bind_param)");
  RG_CUDA(cudaSetDevice(b->model->device));
  if (mask) rg_mark_kernel<<<(b->nenv + 255) / 256, 256, 0, (cudaStream_t)stream>>>(mask, b->d_stale, b->nenv);
  else RG_CUDA(cudaMemsetAsync(b->d_stale, 1, (size_t)b->nenv, (cudaStream_t)stream));
  RG_CUDA(cudaGetLastError());
  b->any_stale = true;
  return 0;
}

/* rederive the lists of the environments selected by `mask` (NULL: all) from the bound geom_dataid rows, on `stream` */
static int rg_pairs_launch(rg_batch* b, const uint8_t* mask, void* stream) {
  const int slot = rg_find_override(b, "geom_dataid");
  if (slot < 0 || !b->d_pairs) return rg_fail(-1, "rg_batch_update_pairs: geom_dataid is not bound per environment (rg_batch_bind_param)");
  const rg_model* m = b->model;
  RG_CUDA(cudaSetDevice(m->device));
  rg_pairs_kernel<<<(b->nenv + 7) / 8, 256, 0, (cudaStream_t)stream>>>(m->dev, (const int*)b->over_ptr[slot], (size_t)m->hm.view.ngeom, mask, b->d_stale, b->nenv,
                                                                       b->d_pairs, b->d_npair, b->pair_cap, b->d_sep, (int*)b->ptr[RG_FIELD_WARN]);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_batch_update_pairs(rg_batch* b, const uint8_t* mask, void* stream) {
  if (!b) return rg_fail(-1, "rg_batch_update_pairs: null argument");
  const int rc = rg_pairs_launch(b, mask, stream);
  if (!rc && !mask) b->any_stale = false;
  return rc;
}

int rg_batch_pair_info(const rg_batch* b, int* capacity, const int** counts_device) {
  if (!b) return rg_fail(-1, "rg_batch_pair_info: null argument");
  if (capacity) *capacity = b->d_pairs ? b->pair_cap : 0;
  if (counts_device) *counts_device = b->d_pairs ? b->d_npair : nullptr;
  return 0;
}

int rg_batch_capacity(const rg_batch* b, int* contacts, int* rows, int* dofs_per_contact) {
  if (!b) return -1;
  if (contacts) *contacts = b->L.ncon;
  if (rows) *rows = b->L.nel;
  if (dofs_per_contact) *dofs_per_contact = b->L.tile;
  return 0;
}
int rg_batch_dbg_size(const rg_batch* b) { return b ? ::rg_dbg_size(b->model->hm.view, b->L.ncon) : -1; }
int rg_batch_scratch_bytes(const rg_batch* b) { return b ? 4 * b->L.total : -1; }

int rg_batch_launch_info(const rg_batch* b, int* ctas, int* warps, int* smem) {
  if (!b) return -1;
  if (ctas) *ctas = b->ctas;
  if (warps) *warps = b->warps;
  if (smem) *smem = b->smem;
  return 0;
}

int rg_batch_env_warps(const rg_batch* b, int* warps_per_env) {
  if (!b || !warps_per_env) return rg_fail(-1, "rg_batch_env_warps: null argument");
  *warps_per_env = b->env_warps;
  return 0;
}

static int rg_fill_io(const rg_batch* b, RgBatchIO& io) {
  for (int f = RG_FIELD_QPOS; f <= RG_FIELD_WARMSTART; f++)
    if (!b->ptr[f] && !((f == RG_FIELD_CTRL || f == RG_FIELD_PID) && b->model->hm.view.nu == 0))   /* a model without actuators has no ctrl / PID rows */
      return rg_fail(-1, "rg_step: qpos, qvel, ctrl, pid and warmstart must be bound");
  io.nenv = b->nenv;
  io.qpos = (float*)b->ptr[RG_FIELD_QPOS]; io.qvel = (float*)b->ptr[RG_FIELD_QVEL]; io.ctrl = (float*)b->ptr[RG_FIELD_CTRL];
  io.pid = (float*)b->ptr[RG_FIELD_PID]; io.warm = (float*)b->ptr[RG_FIELD_WARMSTART]; io.time = (float*)b->ptr[RG_FIELD_TIME];
  io.xfrc = (const float*)b->ptr[RG_FIELD_XFRC]; io.timestep = (const float*)b->ptr[RG_FIELD_TIMESTEP];
  io.site_xpos = (float*)b->ptr[RG_FIELD_SITE_XPOS]; io.body_xpos = (float*)b->ptr[RG_FIELD_BODY_XPOS]; io.body_xquat = (float*)b->ptr[RG_FIELD_BODY_XQUAT];
  io.geom_xpos = (float*)b->ptr[RG_FIELD_GEOM_XPOS]; io.act_force = (float*)b->ptr[RG_FIELD_ACT_FORCE]; io.qacc = (float*)b->ptr[RG_FIELD_QACC];
  io.cost = b->balance ? b->d_cost : nullptr;
  io.sep = b->d_sep;
  io.body_xvel = (float*)b->ptr[RG_FIELD_BODY_XVEL];
  io.sensordata = (float*)b->ptr[RG_FIELD_SENSORDATA];
  io.mocap_pos = (const float*)b->ptr[RG_FIELD_MOCAP_POS]; io.mocap_quat = (const float*)b->ptr[RG_FIELD_MOCAP_QUAT];
  io.contact = (float*)b->ptr[RG_FIELD_CONTACT]; io.ncon = (int*)b->ptr[RG_FIELD_NCON]; io.warn = (int*)b->ptr[RG_FIELD_WARN]; io.dbg = (float*)b->ptr[RG_FIELD_DBG];
  return 0;
}

static int rg_launch_step(rg_batch* b, const uint8_t* mask, int nsub, int final_forward, void* stream, bool setconst = false, const RgSettleArgs* settle = nullptr) {
  if (!b || nsub < 0 || final_forward < 0 || final_forward > 4) return rg_fail(-1, "rg_step: bad argument");
  RgKernelArgs args;
  if (setconst) {
    /* mj_setConst writes into the per-environment rows the caller bound with rg_batch_bind_param: only bound constants exist
       per environment (the shared model is immutable while steps may be in flight) */
    static const char* names[6] = {"dof_invweight0", "body_invweight0", "tendon_invweight0", "tendon_length0", "body_subtreemass", "opt_meaninertia"};
    int any = 0;
    for (int k = 0; k < 6; k++) {
      args.setconst[k] = -1;
      for (int i = 0; i < b->nover; i++) if (b->over_name[i] == names[k]) { args.setconst[k] = i; any = 1; }
    }
    if (!any) return rg_fail(-3, "rg_set_const: bind at least one of dof_invweight0 / body_invweight0 / tendon_invweight0 / tendon_length0 / body_subtreemass / opt_meaninertia per environment first (rg_batch_bind_param)");
    nsub = -1;
  }
  const int rc = rg_fill_io(b, args.io);
  if (rc) return rc;
  if (b->any_stale && !setconst) {   /* geom_dataid rows written since their lists were derived: those lists first */
    const int rc2 = rg_pairs_launch(b, b->d_stale, stream);
    if (rc2) return rc2;
    b->any_stale = false;
  }
  args.env_pairs = b->d_pairs; args.env_npair = b->d_npair; args.pair_cap = b->pair_cap;
  args.m = b->model->dev;
  args.L = b->L;
  args.arena = b->model->d_arena;
  args.nsub = nsub; args.final_forward = final_forward; args.warps = b->warps; args.groups = b->groups;
  args.nover = b->nover;
  args.over_floats = b->over_floats;
  args.order = b->balance ? b->d_order : nullptr;
  args.nslots = nullptr;
  for (int i = 0; i < b->nover; i++) { args.over_off[i] = b->over_off[i]; args.over_cnt[i] = b->over_cnt[i]; args.over_dst[i] = b->over_dst[i]; args.over_ptr[i] = b->over_ptr[i]; }
  RG_CUDA(cudaSetDevice(b->model->device));
  if (mask) {
    rg_subset_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(mask, b->d_subset, b->d_subset + b->nenv, b->nenv);
    RG_CUDA(cudaGetLastError());
    args.order = b->d_subset;
    args.nslots = b->d_subset + b->nenv;
    args.io.cost = nullptr;
  }
  args.counter = b->d_counter;
  RG_CUDA(cudaMemsetAsync(b->d_counter, 0, sizeof(int), (cudaStream_t)stream));
  if (settle) {
    if (b->warps > RG_NARROW_WARPS) rg_settle_kernel<RG_MAX_WARPS><<<b->ctas, 32 * b->warps, b->smem, (cudaStream_t)stream>>>(args, *settle);
    else rg_settle_kernel<RG_NARROW_WARPS><<<b->ctas, 32 * b->warps, b->smem, (cudaStream_t)stream>>>(args, *settle);
  } else if (b->env_warps > 1) RG_CUDA(rg_cta_launch(b->env_warps, b->ctas, b->smem, (cudaStream_t)stream, args));
  else if (b->warps > RG_NARROW_WARPS) rg_step_kernel<RG_MAX_WARPS><<<b->ctas, 32 * b->warps, b->smem, (cudaStream_t)stream>>>(args);
  else rg_step_kernel<RG_NARROW_WARPS><<<b->ctas, 32 * b->warps, b->smem, (cudaStream_t)stream>>>(args);
  RG_CUDA(cudaGetLastError());
  if (!mask && b->balance && nsub > 0) {   /* (not after rg_set_const: it leaves no cost) */
    rg_order_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(b->d_cost, b->d_order, b->nenv);
    RG_CUDA(cudaGetLastError());
  }
  return 0;
}
int rg_step(rg_batch* b, int nsub, int final_forward, void* stream) { return rg_launch_step(b, nullptr, nsub, final_forward, stream); }
int rg_step_subset(rg_batch* b, const uint8_t* mask, int nsub, int final_forward, void* stream) {
  if (!mask) return rg_fail(-1, "rg_step_subset: null mask");
  return rg_launch_step(b, mask, nsub, final_forward, stream);
}
int rg_forward(rg_batch* b, void* stream) { return rg_step(b, 0, 1, stream); }
int rg_step_settle(rg_batch* b, const uint8_t* mask, const int* dofs, int ndof, double damping, int nsub, int final_forward, void* stream) {
  if (ndof < 1 || ndof > RG_SETTLE_MAXDOF || !dofs) return rg_fail(-1, "rg_step_settle: the dof list must hold 1 to " + std::to_string(RG_SETTLE_MAXDOF) + " dofs");
  if (!(damping >= 0.0) || !isfinite((float)damping)) return rg_fail(-1, "rg_step_settle: damping must be finite (in float32) and >= 0");
  if (nsub < 0 || final_forward < 0 || final_forward > 4) return rg_fail(-1, "rg_step_settle: nsub must be >= 0 and final_forward 0..4");
  if (!b) return rg_fail(-1, "rg_step_settle: null batch");
  if (b->env_warps > 1) return rg_fail(-1, "rg_step_settle: batches with one environment per CTA (rg_batch_env_warps > 1) have no settle kernel");
  RgSettleArgs st;
  st.ndof = ndof; st.damping = (float)damping; st.row = -1;
  const int nv = b->model->hm.view.nv;
  for (int i = 0; i < ndof; i++) {
    if (dofs[i] < 0 || dofs[i] >= nv) return rg_fail(-1, "rg_step_settle: dof id " + std::to_string(dofs[i]) + " out of range [0, " + std::to_string(nv) + ")");
    st.dofs[i] = dofs[i];
  }
  const int slot = rg_find_override(b, "dof_damping");
  if (slot >= 0) st.row = b->over_dst[slot];
  /* the substeps with the override, then the final forward passes with the model's (or the environment's) own damping, as
     the reference's forward() after restoring it: a launch of the default kernel */
  int rc = rg_launch_step(b, mask, nsub, 0, stream, false, &st);
  if (!rc && final_forward > 0) rc = rg_launch_step(b, mask, 0, final_forward, stream);
  return rc;
}
int rg_set_const(rg_batch* b, const uint8_t* mask, void* stream) { return rg_launch_step(b, mask, 0, 0, stream, true); }

int rg_reset(rg_batch* b, const uint8_t* mask, void* stream) {
  if (!b) return rg_fail(-1, "rg_reset: bad argument");
  RgBatchIO io;
  const int rc = rg_fill_io(b, io);
  if (rc) return rc;
  RG_CUDA(cudaSetDevice(b->model->device));
  rg_reset_kernel<<<b->nenv, 64, 0, (cudaStream_t)stream>>>(b->model->dev, io, mask);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_batch_body_aabb(rg_batch* b, const int* bodies, int nsel, const double* quat, const uint8_t* mask, double* out, void* stream) {
  if (!b || !bodies || !quat || !out || nsel <= 0) return rg_fail(-1, "rg_batch_body_aabb: bad argument");
  if (nsel > RG_AABB_MAXSEL) return rg_fail(-1, "rg_batch_body_aabb: at most " + std::to_string(RG_AABB_MAXSEL) + " bodies per call");
  const RgModel& hv = b->model->hm.view;
  RgAabbArgs a;
  a.m = b->model->dev;
  a.nenv = b->nenv; a.nsel = nsel;
  for (int k = 0; k < nsel; k++) {
    const int body = bodies[k];
    if (body <= 0 || body >= hv.nbody) return rg_fail(-1, "rg_batch_body_aabb: body id out of range");
    for (int g = hv.body_geomadr[body]; g < hv.body_geomadr[body] + hv.body_geomnum[body]; g++)
      if (hv.geom_type[g] != RG_GEOM_BOX && hv.geom_type[g] != RG_GEOM_MESH)
        return rg_fail(-1, "rg_batch_body_aabb: body " + std::to_string(body) + " has geom " + std::to_string(g) + " of type " + std::to_string(hv.geom_type[g]) +
                               "; only box and mesh geoms are boxed");
    a.body[k] = body;
  }
  /* each environment's bound row where there is one, the model's array where there is not */
  const char* names[6] = {"geom_dataid", "geom_pos", "geom_quat", "geom_size", "mesh_scale", "geom_mesh_scale"};
  const void* model_ptr[6] = {a.m.geom_dataid, a.m.geom_pos, a.m.geom_quat, a.m.geom_size, nullptr, nullptr};
  const void* ptr[6];
  for (int i = 0; i < 6; i++) {
    const int slot = rg_find_override(b, names[i]);
    ptr[i] = slot >= 0 ? (const void*)b->over_ptr[slot] : model_ptr[i];
    a.stride[i] = slot >= 0 ? (size_t)b->over_cnt[slot] : 0;
  }
  a.rows.dataid = (const int*)ptr[0]; a.rows.pos = (const float*)ptr[1]; a.rows.quat = (const float*)ptr[2]; a.rows.size = (const float*)ptr[3];
  a.rows.mscale = (const float*)ptr[4]; a.rows.gscale = (const float*)ptr[5];
  a.quat = quat; a.mask = mask; a.out = out;
  RG_CUDA(cudaSetDevice(b->model->device));
  const int warps = b->nenv * nsel;
  rg_aabb_kernel<<<(warps + 7) / 8, 256, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_place_objects(int nenv, int nobj, const double* bbox, const uint8_t* active, const double table[6], const double* area, int mode,
                     int max_trials, int max_per_object, double goal_distance_ratio, double goal_distance_min, const double* anchor,
                     uint32_t seed, uint32_t epoch, const uint8_t* mask, double* pos, int* status, void* stream) {
  if (nenv <= 0 || nobj <= 0 || !bbox || !active || !table || !area || !pos || !status) return rg_fail(-1, "rg_place_objects: bad argument");
  if (nobj > RG_PLACE_MAXOBJ) return rg_fail(-1, "rg_place_objects: at most " + std::to_string(RG_PLACE_MAXOBJ) + " objects per environment");
  if (mode < RG_PLACE_GRID || mode > RG_PLACE_GRID_THEN_UNIFORM) return rg_fail(-1, "rg_place_objects: unknown mode");
  if (max_trials < 1 || max_per_object < 1) return rg_fail(-1, "rg_place_objects: max_trials and max_per_object must be >= 1");
  if (mode == RG_PLACE_GOAL_DISTANCE && !anchor) return rg_fail(-1, "rg_place_objects: goal_distance_ratio needs the object placements (anchor)");
  RgPlaceArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.max_trials = max_trials; a.max_per_object = max_per_object;
  a.ratio = goal_distance_ratio; a.dmin = goal_distance_min;
  for (int k = 0; k < 3; k++) { a.table_pos[k] = table[k]; a.table_size[k] = table[3 + k]; }
  a.seed = seed; a.epoch = epoch;
  a.bbox = bbox; a.active = active; a.area = area; a.anchor = anchor; a.mask = mask; a.pos = pos; a.status = status;
  rg_place_kernel<<<(nenv + 3) / 4, 128, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_goal_modify(int nenv, int nobj, int kind, const uint8_t* active, const double* object_size, const double* goal_distance_ratio,
                   const double* target_height, double min_height, double max_height, double pickup_proba, double stacking_proba, int fixed_order,
                   uint32_t seed, uint32_t epoch, const uint8_t* mask, double* pos, void* stream) {
  RgModifyArgs a;
  const char* err = rg_modify_make_args(nenv, nobj, kind, active, object_size, goal_distance_ratio, target_height, min_height, max_height, pickup_proba,
                                        stacking_proba, fixed_order, seed, epoch, mask, pos, a);
  if (err) return rg_fail(-1, std::string("rg_goal_modify: ") + err);
  rg_modify_kernel<<<(nenv + 127) / 128, 128, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_layout_goals(int nenv, int nobj, int kind, const double* bbox, const uint8_t* active, const double table[6], const double* area,
                    const double* object_size, const double* distance_mul, const double* rel, int max_retry, uint32_t seed, uint32_t epoch,
                    const uint8_t* mask, double* pos, double* quat, int* status, double* angle, int* retry, void* stream) {
  RgLayoutArgs a;
  const char* err = rg_layout_make_args(nenv, nobj, kind, bbox, active, table, area, object_size, distance_mul, rel, max_retry, seed, epoch, mask, pos, quat,
                                        status, angle, retry, a);
  if (err) return rg_fail(-1, std::string("rg_layout_goals: ") + err);
  rg_layout_kernel<<<(nenv + 3) / 4, 128, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_rearrange_goal(const rg_goal_in* in, const uint8_t* mask, double* prev, const rg_goal_out* out, void* stream) {
  RgGoalArgs a;
  const char* err = rg_goal_make_args(in, mask, prev, out, a);
  if (err) return rg_fail(-1, std::string("rg_rearrange_goal: ") + err);
  rg_goal_kernel<<<(a.nenv + RG_GOAL_WARPS - 1) / RG_GOAL_WARPS, 32 * RG_GOAL_WARPS, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_goal_orientations(int nenv, int nobj, const double* base, const uint8_t* active, int mode, uint32_t seed, uint32_t epoch,
                         const uint8_t* mask, double* out, void* stream) {
  if (nenv <= 0 || nobj <= 0 || !base || !active || !out) return rg_fail(-1, "rg_goal_orientations: bad argument");
  if (nobj > RG_GOAL_MAXOBJ) return rg_fail(-1, "rg_goal_orientations: at most " + std::to_string(RG_GOAL_MAXOBJ) + " objects per environment");
  if (mode != RG_GOALROT_Z && mode != RG_GOALROT_BLOCK) return rg_fail(-1, "rg_goal_orientations: mode 1 z_axis or 2 block");
  RgGoalRotArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.seed = seed; a.epoch = epoch;
  a.base = base; a.active = active; a.mask = mask; a.out = out;
  rg_goal_rot_kernel<<<(nenv + 3) / 4, 128, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_rearrange_obs(const rg_obs_in* in, const uint8_t* mask, const rg_obs_out* out, void* stream) {
  RgObsArgs a;
  const char* err = rg_obs_make_args(in, mask, out, a);
  if (err) return rg_fail(-1, std::string("rg_rearrange_obs: ") + err);
  rg_obs_kernel<<<(a.in.nenv + 3) / 4, 128, 0, (cudaStream_t)stream>>>(a);
  RG_CUDA(cudaGetLastError());
  return 0;
}

int rg_arm_phase(const rg_arm_tables* tables, int phases, int nenv, const rg_arm_sim* main_sim, const rg_arm_sim* solver_sim, const float* action,
                 int action_dim, const uint8_t* mask, int mask_len, void* stream) {
  const char* err = rg_arm_check(tables, phases, nenv, main_sim, solver_sim, action, action_dim, mask, mask_len);
  if (err) return rg_fail(-1, std::string("rg_arm_phase: ") + err);
  RgArmArgs a;
  a.t = *tables; a.main = *main_sim; a.solver = *solver_sim;
  a.phases = phases; a.nenv = nenv; a.action_dim = action_dim; a.action = action; a.mask = mask;
  RG_CUDA(rg_arm_launch(a, (cudaStream_t)stream));
  return 0;
}

int rg_arm_sample_actions(int nenv, int action_dim, uint32_t seed, uint32_t epoch, const uint8_t* mask, int mask_len, float* out, void* stream) {
  if (nenv <= 0 || !out) return rg_fail(-1, "rg_arm_sample_actions: bad argument");
  if (action_dim < 1 || action_dim > RG_ARM_MAXACT) return rg_fail(-1, "rg_arm_sample_actions: action_dim must be 1..8");
  if (mask && mask_len != nenv) return rg_fail(-1, "rg_arm_sample_actions: the mask must hold one byte per environment (mask_len == nenv)");
  RG_CUDA(rg_arm_sample_launch(nenv, action_dim, seed, epoch, mask, out, (cudaStream_t)stream));
  return 0;
}

int rg_object_groups(const rg_groups_in* in, const uint8_t* mask, int mask_len, const rg_groups_out* out, void* stream) {
  cudaError_t e = cudaSuccess;
  const char* err = rg_groups_run(in, mask, mask_len, out, (cudaStream_t)stream, &e);
  if (err) return rg_fail(-1, std::string("rg_object_groups: ") + err);
  RG_CUDA(e);
  return 0;
}
}
