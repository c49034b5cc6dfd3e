/* rg_defs.h -- shared definitions of the batched rigid-body step engine.
 *
 * Execution model: ONE WARP PER ENVIRONMENT.  The device code is written as a sequence of
 * "phases": inside RG_PHASE_BEGIN/RG_PHASE_END every lane runs the body with its own `lane`
 * index; lanes exchange data only through the per-warp shared-memory scratch or through the
 * warp helpers below (sum/max/broadcast/compaction).  Everything outside a phase is warp-uniform.
 *
 * The same source compiles two ways:
 *   - nvcc, sm_90a (the product): a phase is straight-line SIMT code followed by __syncwarp();
 *     the warp helpers are shuffles / ballots.
 *   - g++ with -DRG_EMU (tests only, tests/emu): a phase is a `for (lane = 0..31)` loop and the
 *     helpers run the same butterfly order on arrays.  This lets the CPU-only CI check the
 *     kernel's logic against the fp64 oracle; it is never used as a product fallback.
 */
#pragma once
#include <stdint.h>
#include <math.h>

#ifdef RG_EMU
#include <string.h>
#define RG_DEV static inline
#define RG_DEV_NOINLINE static
#define RG_NOUNROLL
#define RG_UNROLL2
#define RG_UNROLL4
#define RG_UNROLL8
#define RG_PHASE_BEGIN for (int lane = 0; lane < 32; ++lane) {
#define RG_PHASE_END }
#define RG_LANE_DECL
#define LANEVAR(T, x) T x[32]
#define LANEARR(T, x, n) T x[32][n]
#define LV(x) x[lane]
#define LA(x, i) x[lane][i]
#define RG_LDG(p) (*(p))
#define RG_LDG4(base, idx, out) { const float* q_ = (base) + 4 * (size_t)(idx); (out)[0] = q_[0]; (out)[1] = q_[1]; (out)[2] = q_[2]; (out)[3] = q_[3]; }
#define RG_RSQRT(x) (1.0f / sqrtf(x))
#define RG_SCRATCH(c) ((c).s)
#define RG_CTA_SYNC()
#define RG_CTA_ANY(x) (x)
#define RG_SINCOS(x, sn, cs) { *(sn) = sinf(x); *(cs) = cosf(x); }
#else
#include <cuda_runtime.h>
#include <string.h>
#define RG_DEV __device__ __forceinline__
#ifdef RG_COOP   /* internal linkage: rg_cta.cu compiles the same functions again, into the same library as rg_engine.cu */
#define RG_DEV_NOINLINE static __device__ __noinline__
#else
#define RG_DEV_NOINLINE __device__ __noinline__
#endif
/* lane-strided loops run once or twice (n <= 64): unrolling them only bloats a kernel that is instruction-cache bound */
#define RG_NOUNROLL _Pragma("unroll 1")
#define RG_UNROLL2 _Pragma("unroll 2")
#define RG_UNROLL4 _Pragma("unroll 4")
#define RG_UNROLL8 _Pragma("unroll 8")
#define RG_PHASE_BEGIN {
#define RG_PHASE_END } __syncwarp();
#define RG_LANE_DECL const int lane = threadIdx.x & 31;
#define LANEVAR(T, x) T x
#define LANEARR(T, x, n) T x[n]
#define LV(x) x
#define LA(x, i) x[i]
#define RG_LDG(p) __ldg(p)
#define RG_LDG4(base, idx, out) { const float4 q_ = __ldg((const float4*)(base) + (idx)); (out)[0] = q_.x; (out)[1] = q_.y; (out)[2] = q_.z; (out)[3] = q_.w; }
#define RG_RSQRT(x) rsqrtf(x)
/* The per-warp scratch is addressed as (dynamic shared memory base + offset) so that the compiler can prove the
 * address space and emit LDS/STS with 32-bit addresses; a plain float* carried through the noinline stage
 * functions compiles to generic 64-bit LD/ST (measured: most of the instruction stream was address arithmetic). */
extern __shared__ __align__(128) unsigned char rg_smem_raw[];
#define RG_SCRATCH(c) (((float*)rg_smem_raw) + (c).soff)
/* The warps of a CTA walk the step in loose lock-step (one barrier per stage / Newton iteration): the
 * kernel's code is far larger than the instruction cache, so keeping the warps in the same stage lets
 * one instruction fetch feed all of them.  Every warp executes the same number of barriers. */
#ifndef RG_SKEW
#define RG_SKEW 0
#endif
#if RG_SKEW == 0
/* Only the warps that hold an environment in this round take part (the last round of a launch is usually partial): named
 * barrier 1 over rg_bar_threads threads; barrier 0 (__syncthreads) stays for the round boundaries in rg_step_kernel. */
/* The active warps of a round may be split into barrier GROUPS (rg_batch_set_barrier_groups / RG_BAR_GROUPS, default 1):
 * contiguous runs of warps, each with its own named barrier 1..G.  Barriers order nothing but the instruction stream, so
 * results do not depend on the grouping; fewer warps per barrier wait less for their slowest member, at the price of more
 * distinct code regions live in the instruction cache. */
__shared__ int rg_bar_cfg[16];   /* per warp: barrier id << 16 | threads taking part */
#define RG_CTA_SYNC() do { const int rg_cfg_ = rg_bar_cfg[threadIdx.x >> 5]; asm volatile("bar.sync %0, %1;" ::"r"(rg_cfg_ >> 16), "r"(rg_cfg_ & 0xffff) : "memory"); } while (0)
#else
/* Skewed variant: a warp may run up to RG_SKEW stages ahead of the slowest warp of its CTA.  Stage boundary k is an
 * mbarrier (ring of RG_SKEW+1): arrive on boundary k, then wait for boundary k-RG_SKEW.  A warp passes boundary k+R-1
 * only after boundary k completed, so a ring slot is never re-armed before its previous phase is over. */
#define RG_BAR_RING (RG_SKEW + 1)
__shared__ __align__(8) unsigned long long rg_stage_bar[RG_BAR_RING];
__shared__ int rg_stage_k[32];
__device__ __forceinline__ void rg_stage_sync() {
  __syncwarp();
  if ((threadIdx.x & 31) == 0) {
    const int w = threadIdx.x >> 5;
    const int k = rg_stage_k[w];
    rg_stage_k[w] = k + 1;
    const unsigned a = (unsigned)__cvta_generic_to_shared(&rg_stage_bar[k % RG_BAR_RING]);
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(a) : "memory");
    if (k >= RG_SKEW) {
      const int j = k - RG_SKEW;
      const unsigned b = (unsigned)__cvta_generic_to_shared(&rg_stage_bar[j % RG_BAR_RING]);
      const unsigned parity = (unsigned)((j / RG_BAR_RING) & 1);
      unsigned done = 0;
      while (!done)
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(done) : "r"(b), "r"(parity) : "memory");
    }
  }
  __syncwarp();
}
#define RG_CTA_SYNC() rg_stage_sync()
#endif
#define RG_CTA_ANY(x) __syncthreads_or(x)
#define RG_SINCOS(x, sn, cs) __sincosf(x, sn, cs)
#endif

/* Cooperative sections.  -DRG_COOP builds (rg_cta.cu, tests/emu/rg_emu_cta.cpp) run ONE environment per CTA of W warps: warp 0
 * runs every stage as above, and the dense per-element loops of the Newton solve (rg_sol.inl: the Hessian assembly, the
 * envelope Cholesky, the triangular solves, the matrix-vector products) spread their outputs over all RG_NT = 32 W threads.
 * Each output element is still computed by one thread with the same operation sequence, so the results are the one-warp
 * results bit for bit; only the owner of an element changes.  A cooperative phase ends at named barrier RG_COOP_BAR over the
 * CTA (the stage barriers use 0 and 1..RG_BAR_GROUPS).  A value one thread hands to all (RG_COOP_PUT / RG_COOP_BCAST) goes
 * through shared memory instead of a shuffle.  Without RG_COOP every macro below is the one-warp phase it stands for. */
#ifndef RG_COOP
#define RG_NT 32
#define RG_COOP_LANE_DECL RG_LANE_DECL
#define RG_COOP_BEGIN RG_PHASE_BEGIN
#define RG_COOP_END RG_PHASE_END
#define COOPVAR(T, x) LANEVAR(T, x)
#define COOPARR(T, x, n) LANEARR(T, x, n)
#define RG_COOP_PUT(k, who, v)
#define RG_COOP_BCAST(x, k, src) RG_WARP_BCAST(x, src)
#define RG_COOP_ENTER(id, c, a0, a1, a2, a3, a4, a5, p)
#elif defined(RG_EMU)
extern int rg_emu_coop_threads;   /* 32 W of the emulated CTA */
#define RG_NT rg_emu_coop_threads
#define RG_COOP_LANE_DECL
#define RG_COOP_BEGIN for (int lane = 0; lane < RG_NT; ++lane) {
#define RG_COOP_END }
#define COOPVAR(T, x) T x[512]
#define COOPARR(T, x, n) T x[512][n]
#define RG_COOP_PUT(k, who, v)
#define RG_COOP_BCAST(x, k, src) (x[src])
#define RG_COOP_ENTER(id, c, a0, a1, a2, a3, a4, a5, p)
#else
#define RG_COOP_BAR 15
#define RG_NT ((int)blockDim.x)
__shared__ float rg_coop_bc[2];   /* RG_COOP_PUT slots */
RG_DEV void rg_coop_sync() { asm volatile("bar.sync %0, %1;" ::"r"(RG_COOP_BAR), "r"((int)blockDim.x) : "memory"); }
#define RG_COOP_LANE_DECL const int lane = threadIdx.x;
#define RG_COOP_BEGIN {
#define RG_COOP_END } rg_coop_sync();
#define COOPVAR(T, x) T x
#define COOPARR(T, x, n) T x[n]
#define RG_COOP_PUT(k, who, v) if (who) rg_coop_bc[k] = (float)(v);
#define RG_COOP_BCAST(x, k, src) rg_coop_bc[k]
/* warp 0 enters a cooperative section: it posts the section and its arguments, and the other warps, waiting in rg_coop_worker
   (rg_sol.inl), join it */
#define RG_COOP_ENTER(id, c, a0, a1, a2, a3, a4, a5, p) if (threadIdx.x < 32) rg_coop_post(id, c, a0, a1, a2, a3, a4, a5, p);
/* one environment per CTA: warp 0 runs the stages alone, so the stage barriers have nobody to wait for */
#undef RG_CTA_SYNC
#undef RG_CTA_ANY
#define RG_CTA_SYNC() __syncwarp()
#define RG_CTA_ANY(x) (x)
#endif

#define RG_MINVAL 1e-15f
#define RG_EPS 1.1920929e-07f
/* Capacities are RUN-TIME parameters of a batch (rg_batch_create_ex): contacts kept per environment, single-row constraint
 * elements (friction loss + limits), dofs one contact may touch.  The defaults below are what the dactyl/locked model
 * needs in practice; the reference's own sizes (nconmax=100, njmax=500, assets.xml:5-6) are available at the price of
 * fewer resident environments per SM.  Overflow sets a warning bit, it never corrupts memory. */
#ifndef RG_NCON
#define RG_NCON 32
#endif
#ifndef RG_COST_ITER
#define RG_COST_ITER 3   /* weight of one Newton iteration against one narrow-phase pair in the work estimate (rg_order_kernel) */
#endif
#ifndef RG_NEL
#define RG_NEL 64
#endif
#define RG_CON_STRIDE 24
#define RG_CPRM 6           /* per-contact solver parameters: D, dim, first slot (rg_slot_col), unused, number of dofs, their sign bits (solimp[5] is staged there by the collision stage) */
#ifndef RG_GRP
#define RG_GRP 8           /* lanes that share one pair in the convex-convex narrow phase (rg_mpr_batch) */
#endif
#define RG_NSEP 64         /* words of the per-environment separating-axis cache (rg_mpr_batch) */
/* word offsets in the collision stage's narrow-phase staging area (L.stage, sized by rg_make_layout): [32][8] results of the
   convex-convex pairs from 0, their 32 candidate slots from RG_STAGE_SLOTS, the two geom views of each lane group's pair
   (rg_mpr_batch) from RG_STAGE_VIEWS */
#define RG_STAGE_SLOTS 256
#define RG_STAGE_VIEWS 288
#ifndef RG_CELLN
#define RG_CELLN 8         /* cells per cube-face edge of the hull support lists (rg_host_hull_cells, rg_hull_cell) */
#endif
#define RG_NCELL (6 * RG_CELLN * RG_CELLN)   /* direction cells per hull */
#define RG_TJ 8           /* max non-zeros of one tendon's Jacobian row */
#ifdef RG_PROFILE
#define RG_NPROF 16      /* per-stage cycle counters appended to the RG_DBG dump (-DRG_PROFILE builds only) */
#else
#define RG_NPROF 0
#endif
#define RG_TRI(i, j) ((((i) * ((i) + 1)) >> 1) + (j))   /* packed lower triangle, i >= j */
/* The solver's Hessian is stored with the dof order REVERSED (leaves of the kinematic tree first, roots and
 * free objects last): Cholesky then eliminates children before parents, so the tree-structured part
 * of the matrix produces no fill-in and the envelope of most rows is a handful of entries. */
#define RG_HS(a, b) ((a) >= (b) ? RG_TRI(a, b) : RG_TRI(b, a))   /* a, b = solver positions (dof_sidx) */
#ifndef RG_TILE
#define RG_TILE 16       /* default for the dofs one contact may touch (<= 32: their signs travel in one word) */
#endif

enum { RG_JNT_FREE = 0, RG_JNT_BALL = 1, RG_JNT_SLIDE = 2, RG_JNT_HINGE = 3 };
enum { RG_GEOM_PLANE = 0, RG_GEOM_SPHERE = 2, RG_GEOM_CAPSULE = 3, RG_GEOM_ELLIPSOID = 4, RG_GEOM_CYLINDER = 5, RG_GEOM_BOX = 6, RG_GEOM_MESH = 7 };
enum { RG_WRAP_JOINT = 1, RG_WRAP_PULLEY = 2, RG_WRAP_SITE = 3, RG_WRAP_SPHERE = 4, RG_WRAP_CYLINDER = 5 };
enum { RG_TRN_JOINT = 0, RG_TRN_TENDON = 3 };
enum { RG_GAIN_FIXED = 0, RG_GAIN_USER = 2, RG_BIAS_NONE = 0, RG_BIAS_AFFINE = 1, RG_BIAS_USER = 3 };
enum { RG_DSBL_CONSTRAINT = 1, RG_DSBL_EQUALITY = 2, RG_DSBL_FRICTIONLOSS = 4, RG_DSBL_LIMIT = 8, RG_DSBL_CONTACT = 16,
       RG_DSBL_PASSIVE = 32, RG_DSBL_GRAVITY = 64, RG_DSBL_CLAMPCTRL = 128, RG_DSBL_WARMSTART = 256,
       RG_DSBL_ACTUATION = 1024, RG_DSBL_REFSAFE = 2048 };
enum { RG_EL_FLOSS = 0, RG_EL_JLIMIT = 1, RG_EL_TLIMIT = 2 };
enum { RG_EQ_CONNECT = 0, RG_EQ_WELD = 1, RG_EQ_JOINT = 2 };
enum { RG_WARN_CONTACT_FULL = 1, RG_WARN_ROWS_FULL = 2, RG_WARN_BAD_STATE = 4, RG_WARN_MPR = 8, RG_WARN_TENDON_NNZ = 16, RG_WARN_DOFS_FULL = 32,
       RG_WARN_PAIRS_FULL = 64 /* rg_batch_update_pairs: the environment's pair list overflowed its capacity (surplus dropped) */,
       RG_WARN_BAD_DATAID = 128 /* rg_batch_update_pairs: a geom_dataid value that is neither -1 nor a mesh id of a mesh geom (geom disabled) */ };

/* Device view of the compiled model: fp32 / int32 copies of every rg_model_fields.h array, then the arrays the engine derives
   (rg_derived_fields.h) and its derived scalars. */
struct RgModel {
#define RG_DIM(n) int n;
#define RG_I(n, c) const int* n;
#define RG_F(n, c) const float* n;
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#define RG_DS(n, T, c) const T* n;
#define RG_DE(n, T, c) const T* n;
#define RG_DG(n, T, c) const T* n;
#include "rg_derived_fields.h"
  int ncand_cap;               /* entries mesh_cand4 has room for (rebuilt lists must fit in the arena allocated at load) */
#define RG_DSO(n, T, c, when) const T* n;
#include "rg_derived_fields.h"
  float origin[3];             /* world translation applied at load so coordinates stay small in fp32 */
  int small_bytes;             /* leading part of the arena that is staged into shared memory */
  int nM;                      /* entries of the tree-sparse mass matrix: sum over dofs of (depth + 1) */
  int ndoflevel;               /* depth levels of the dof tree */
  int ns;                      /* dofs in the constraint solver (<= nv) */
  int neqrow;                  /* rows of the active equality constraints */
  int pidw;                    /* floats of controller state per actuator: 3 (PID), 6 when the model has a cascaded-PI actuator */
};

/* Offsets (in floats) of the per-warp scratch arrays; computed once on the host (rg_make_layout). */
struct RgLayout {
  int qpos, qvel, ctrl, pid, warm;
  int lpos, lquat, xpos, xquat, gxpos, sxpos;
  int S, M, H;                       /* packed lower triangles; H aliases the block {Sdot,I10,crb} that is dead by then */
  int Sdot, I10, crb;
  int bias, smooth, qacc, Ma, search, Mv, qfc, tmp;
  int tlen, tvel, tJn, tJi, tJv, alen, aforce;
  int con, cu, cw, cF, cprm;         /* contacts + per-contact solver state */
  int el_i, el_D, el_jar, el_jv, el_f;
  int tileJ, tileWJ, tileDof, cand, cand2, scal, eldof, env, cdof, sep, stage;
  int mocap;                         /* [nmocap][7] pose of the mocap bodies (data.mocap_pos / mocap_quat) */
  int ncon, nel, tile;               /* capacities: contacts, single-row elements, dofs per contact */
  int total;
};

#ifndef RG_EMU
/* Device-side model view.  The small arrays of the model are staged in the CTA's dynamic shared memory, so
 * the view stores 32-bit OFFSETS from the shared-memory base instead of pointers: every `m.field[i]` then
 * compiles to an LDS with a 32-bit address instead of a generic 64-bit load.  The big read-only arrays
 * (hull vertices / adjacency, pair list) stay global pointers. */
template <class T>
struct RgArr {
  int off; /* bytes from rg_smem_raw */
  __device__ __forceinline__ const T* p() const { return (const T*)(rg_smem_raw + off); }
  __device__ __forceinline__ const T& operator[](int i) const { return p()[i]; }
  __device__ __forceinline__ const T* operator+(int i) const { return p() + i; }
};
struct RgModelDev {
#define RG_DIM(n) int n;
#define RG_I(n, c) RgArr<int> n;
#define RG_F(n, c) RgArr<float> n;
#define RG_IB(n, c) const int* n;
#define RG_FB(n, c) const float* n;
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#undef RG_IB
#undef RG_FB
  /* a per-environment array's offset is < 0 while no row is bound: it is never staged, so it costs no shared memory */
#define RG_DS(n, T, c) RgArr<T> n;
#define RG_DE(n, T, c) RgArr<T> n;
#include "rg_derived_fields.h"
#define RG_DSO(n, T, c, when) RgArr<T> n;
#include "rg_derived_fields.h"
  int has_pairs;
#define RG_DG(n, T, c) const T* n;
#define RG_DGH(n, T, c)
#include "rg_derived_fields.h"
  float origin[3];
  int small_bytes;
  int nM;
  int ndoflevel;
  int ns;
  int neqrow;
  int pidw;
  RgLayout L;                  /* per-warp scratch layout, kept next to the model so it is read with LDS too */
};
#define RG_MODEL_T RgModelDev
#define RG_HAS_PAIRS(m) ((m).has_pairs)
#define RG_GEOM_MESH_SCALE(m, g) ((m).geom_mesh_scale.off >= 0 ? (m).geom_mesh_scale[g] : 1.0f)
/* the model view is handed to non-inlined code as its byte offset in the CTA's dynamic shared memory, so that
   every access through it compiles to LDS rather than a generic load */
typedef int RgMRef;
#define RG_MDEREF(r) (*(const RgModelDev*)(rg_smem_raw + (r)))
#define RG_MREF(m) ((int)((const unsigned char*)&(m) - rg_smem_raw))
#else
#define RG_MODEL_T RgModel
#define RG_HAS_PAIRS(m) ((m).pair_packed != nullptr)
#define RG_GEOM_MESH_SCALE(m, g) ((m).geom_mesh_scale ? (m).geom_mesh_scale[g] : 1.0f)
typedef const RgModel* RgMRef;
#define RG_MDEREF(r) (*(r))
#define RG_MREF(m) (&(m))
#endif
/* the two reads of dof_damping: the passive force (rg_forces) and the implicit term of the Euler factor (rg_euler).  Both go
   through the model view, which is where the settle launch puts its override (rg_kernel.inl); the CPU emulation can redirect
   one of them at a time to show that the override reaches both (tests/emu/rg_emu_settle.cpp). */
#ifndef RG_DAMPING_PASSIVE
#define RG_DAMPING_PASSIVE(m) (m).dof_damping
#endif
#ifndef RG_DAMPING_IMPLICIT
#define RG_DAMPING_IMPLICIT(m) (m).dof_damping
#endif


#ifndef RG_EMU
/* ---- warp helpers (GPU) ---- */
RG_DEV float rg_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
RG_DEV float rg_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
RG_DEV int rg_warp_or(int v) { return __reduce_or_sync(0xffffffffu, (unsigned)v); }
RG_DEV int rg_warp_isum(int v) { return __reduce_add_sync(0xffffffffu, v); }
RG_DEV float rg_warp_bcast(float v, int src) { return __shfl_sync(0xffffffffu, v, src); }
/* exclusive prefix sum of small non-negative ints; returns total in *total */
RG_DEV int rg_warp_excl_scan(int v, int* total) {
  const int lane = threadIdx.x & 31;
  int x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
  *total = __shfl_sync(0xffffffffu, x, 31);
  return x - v;
}
#define RG_WARP_SUM(x) rg_warp_sum(x)
#define RG_WARP_MAX(x) rg_warp_max(x)
#define RG_WARP_OR(x) rg_warp_or(x)
#define RG_WARP_ISUM(x) rg_warp_isum(x)
#define RG_WARP_BCAST(x, src) rg_warp_bcast(x, src)
#define RG_WARP_SCAN(cnt, pos, total) pos = rg_warp_excl_scan(cnt, &(total))
/* arg-max over each group of RG_GRP consecutive lanes: every lane of a group ends up with the group's best value and the
   index that goes with it (ties: the smaller index, so the answer does not depend on which lane held it) */
RG_DEV void rg_group_argmax(float& v, int& i) {
#pragma unroll
  for (int o = RG_GRP / 2; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
}
#define RG_GROUP_ARGMAX(v, i) rg_group_argmax(v, i)
#else
/* ---- warp helpers (emulation: identical combination order) ---- */
static inline float rg_emu_sum(const float* x) {
  float t[32], u[32];
  memcpy(t, x, sizeof t);
  for (int o = 16; o > 0; o >>= 1) { for (int l = 0; l < 32; l++) u[l] = t[l] + t[l ^ o]; memcpy(t, u, sizeof t); }
  return t[0];
}
static inline float rg_emu_max(const float* x) { float m = x[0]; for (int l = 1; l < 32; l++) m = fmaxf(m, x[l]); return m; }
static inline int rg_emu_or(const int* x) { int m = 0; for (int l = 0; l < 32; l++) m |= x[l]; return m; }
static inline int rg_emu_isum(const int* x) { int m = 0; for (int l = 0; l < 32; l++) m += x[l]; return m; }
static inline int rg_emu_scan(const int* c, int* pos) { int s = 0; for (int l = 0; l < 32; l++) { pos[l] = s; s += c[l]; } return s; }
#define RG_WARP_SUM(x) rg_emu_sum(x)
#define RG_WARP_MAX(x) rg_emu_max(x)
#define RG_WARP_OR(x) rg_emu_or(x)
#define RG_WARP_ISUM(x) rg_emu_isum(x)
#define RG_WARP_BCAST(x, src) (x[src])
#define RG_WARP_SCAN(cnt, pos, total) total = rg_emu_scan(cnt, pos)
static inline void rg_emu_group_argmax(float* v, int* i) {
  for (int g = 0; g < 32; g += RG_GRP) {
    float bv = v[g]; int bi = i[g];
    for (int l = g + 1; l < g + RG_GRP; l++) if (v[l] > bv || (v[l] == bv && i[l] < bi)) { bv = v[l]; bi = i[l]; }
    for (int l = g; l < g + RG_GRP; l++) { v[l] = bv; i[l] = bi; }
  }
}
#define RG_GROUP_ARGMAX(v, i) rg_emu_group_argmax(v, i)
#endif

/* ---- small vector math ---- */
RG_DEV float rg_dot3(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
RG_DEV void rg_cross(float* r, const float* a, const float* b) {
  float x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  r[0] = x; r[1] = y; r[2] = z;
}
RG_DEV void rg_sub3(float* r, const float* a, const float* b) { r[0] = a[0] - b[0]; r[1] = a[1] - b[1]; r[2] = a[2] - b[2]; }
RG_DEV void rg_add3(float* r, const float* a, const float* b) { r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2]; }
RG_DEV void rg_copy3(float* r, const float* a) { r[0] = a[0]; r[1] = a[1]; r[2] = a[2]; }
RG_DEV void rg_scl3(float* r, const float* a, float s) { r[0] = a[0] * s; r[1] = a[1] * s; r[2] = a[2] * s; }
RG_DEV void rg_addscl3(float* r, const float* a, float s) { r[0] += a[0] * s; r[1] += a[1] * s; r[2] += a[2] * s; }
RG_DEV float rg_normalize3(float* a) {
  float n2 = rg_dot3(a, a);
  if (n2 < 1e-30f) { a[0] = 1; a[1] = 0; a[2] = 0; return 0.f; }
  float n = sqrtf(n2), inv = 1.0f / n;
  a[0] *= inv; a[1] *= inv; a[2] *= inv;
  return n;
}
RG_DEV void rg_quat_mul(float* r, const float* a, const float* b) {
  float w = a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3];
  float x = a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2];
  float y = a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1];
  float z = a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0];
  r[0] = w; r[1] = x; r[2] = y; r[3] = z;
}
RG_DEV void rg_quat_norm(float* q) {
  float n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
  if (n2 < 1e-30f) { q[0] = 1; q[1] = q[2] = q[3] = 0; return; }
  float inv = 1.0f / sqrtf(n2);
  q[0] *= inv; q[1] *= inv; q[2] *= inv; q[3] *= inv;
}
/* r = q v q^-1 */
RG_DEV void rg_rot(float* r, const float* q, const float* v) {
  float t[3], u[3] = {q[1], q[2], q[3]};
  rg_cross(t, u, v);
  t[0] *= 2; t[1] *= 2; t[2] *= 2;
  float c[3];
  rg_cross(c, u, t);
  r[0] = v[0] + q[0] * t[0] + c[0];
  r[1] = v[1] + q[0] * t[1] + c[1];
  r[2] = v[2] + q[0] * t[2] + c[2];
}
RG_DEV void rg_quat2mat(float* m, const float* q) {
  float w = q[0], x = q[1], y = q[2], z = q[3];
  m[0] = w * w + x * x - y * y - z * z; m[1] = 2 * (x * y - w * z); m[2] = 2 * (x * z + w * y);
  m[3] = 2 * (x * y + w * z); m[4] = w * w - x * x + y * y - z * z; m[5] = 2 * (y * z - w * x);
  m[6] = 2 * (x * z - w * y); m[7] = 2 * (y * z + w * x); m[8] = w * w - x * x - y * y + z * z;
}
RG_DEV void rg_mulmat3(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[1] * v[1] + m[2] * v[2], y = m[3] * v[0] + m[4] * v[1] + m[5] * v[2], z = m[6] * v[0] + m[7] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
RG_DEV void rg_mulmatT3(float* r, const float* m, const float* v) {
  float x = m[0] * v[0] + m[3] * v[1] + m[6] * v[2], y = m[1] * v[0] + m[4] * v[1] + m[7] * v[2], z = m[2] * v[0] + m[5] * v[1] + m[8] * v[2];
  r[0] = x; r[1] = y; r[2] = z;
}
RG_DEV int rg_f2i(float f) { int i; memcpy(&i, &f, 4); return i; }
RG_DEV float rg_i2f(int i) { float f; memcpy(&f, &i, 4); return f; }
RG_DEV float rg_clamp(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }
RG_DEV int rg_dof_in_body(const RG_MODEL_T& m, int body, int dof) {
  return ((unsigned)m.body_dofmask[body * m.nmaskw + (dof >> 5)] >> (dof & 31)) & 1u;
}
/* spatial vectors: V = [w; vO] (motion), F = [nO; f] (force), both about the (shifted) world origin */
RG_DEV float rg_dot6(const float* a, const float* b) { return rg_dot3(a, b) + rg_dot3(a + 3, b + 3); }
/* origin-form spatial inertia I = (m, h[3] = m*com, IO[6] = xx yy zz xy xz yz): F = I V */
RG_DEV void rg_inertia_mul(float* F, const float* I, const float* V) {
  float t[3], n[3];
  rg_cross(t, V, I + 1);                 /* w x h */
  float f0 = I[0] * V[3] + t[0], f1 = I[0] * V[4] + t[1], f2 = I[0] * V[5] + t[2];
  n[0] = I[4] * V[0] + I[7] * V[1] + I[8] * V[2];
  n[1] = I[7] * V[0] + I[5] * V[1] + I[9] * V[2];
  n[2] = I[8] * V[0] + I[9] * V[1] + I[6] * V[2];
  rg_cross(t, I + 1, V + 3);             /* h x vO */
  F[0] = n[0] + t[0]; F[1] = n[1] + t[1]; F[2] = n[2] + t[2];
  F[3] = f0; F[4] = f1; F[5] = f2;
}
RG_DEV void rg_cross_motion(float* r, const float* V, const float* S) {
  float a[3], b[3], c[3];
  rg_cross(a, V, S); rg_cross(b, V, S + 3); rg_cross(c, V + 3, S);
  r[0] = a[0]; r[1] = a[1]; r[2] = a[2];
  r[3] = b[0] + c[0]; r[4] = b[1] + c[1]; r[5] = b[2] + c[2];
}
RG_DEV void rg_cross_force(float* r, const float* V, const float* F) {
  float a[3], b[3], c[3];
  rg_cross(a, V, F); rg_cross(b, V + 3, F + 3); rg_cross(c, V, F + 3);
  r[0] = a[0] + b[0]; r[1] = a[1] + b[1]; r[2] = a[2] + b[2];
  r[3] = c[0]; r[4] = c[1]; r[5] = c[2];
}
/* velocity of the body point at `p` generated by unit rate of motion axis S */
RG_DEV void rg_jacp(float* jp, const float* S, const float* p) {
  float t[3];
  rg_cross(t, S, p);
  jp[0] = S[3] + t[0]; jp[1] = S[4] + t[1]; jp[2] = S[5] + t[2];
}
