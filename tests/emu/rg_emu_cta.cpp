/* rg_emu_cta.cpp -- CPU EMULATION BUILD of the step with one environment per CTA of W warps (robogym_b200/csrc/rg_cta.cu).  TEST
 * INFRASTRUCTURE ONLY.
 *
 * Built twice from this file (tests/emu/pyemu_cta.py): with -DRG_COOP the cooperative sections of the Newton solve loop over the
 * 32 W threads of the emulated CTA (rg_defs.h), without it they are the one-warp phases.  Both libraries export the same entry
 * points, so a test runs identical calls through both and compares the bytes.
 *   rgc_create / rgc_destroy: a model (blob) with the scratch layout of the given capacities (0 = engine default);
 *   rgc_ns:                   dofs in the model's constraint solver (what the engine's selection reads);
 *   rgc_set_warps:            W of the cooperative build (2, 4, 8, 16; the one-warp build ignores it);
 *   rgc_step:                 rg_env_step for every environment, per-environment timestep optional;
 *   rgc_chol:                 the envelope Cholesky of an n x n matrix (packed lower rows, right-hand side in row n) followed by
 *                             the back substitution, and a forward substitution of a second right-hand side with that factor.
 */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_step.inl"
#include "../../robogym_b200/csrc/rg_host.h"

#ifdef RG_COOP
int rg_emu_coop_threads = 64;
#endif

struct RgcHandle { RgHostModel hm; RgLayout L; std::vector<float> scratch; std::vector<int> sep; };

extern "C" {
void* rgc_create(const void* blob, size_t len, int ncon, int nel, int tile) {
  RgcHandle* h = new RgcHandle();
  std::string err;
  if (!rg_host_load(blob, len, h->hm, err)) { delete h; return nullptr; }
  h->L = rg_make_layout(h->hm.view, ncon ? ncon : RG_NCON, nel ? nel : RG_NEL, tile ? tile : RG_TILE);
  h->scratch.assign(h->L.total, 0.0f);
  return h;
}
void rgc_destroy(void* hv) { delete (RgcHandle*)hv; }
int rgc_ncon(void* hv) { return ((RgcHandle*)hv)->L.ncon; }
int rgc_ns(void* hv) { return ((RgcHandle*)hv)->hm.view.ns; }   /* dofs in the constraint solver */
int rgc_set_warps(int w) {
#ifdef RG_COOP
  rg_emu_coop_threads = 32 * w;
  return 1;
#else
  (void)w;
  return 0;
#endif
}
void rgc_step(void* hv, int nenv, float* qpos, float* qvel, float* ctrl, float* pid, float* warm, const float* timestep, float* sensordata,
              float* contact, int* ncon, int* warn, int nsub, int final_forward) {
  RgcHandle* h = (RgcHandle*)hv;
  RgBatchIO io;
  memset(&io, 0, sizeof io);
  io.nenv = nenv; io.qpos = qpos; io.qvel = qvel; io.ctrl = ctrl; io.pid = pid; io.warm = warm; io.timestep = timestep;
  io.sensordata = sensordata; io.contact = contact; io.ncon = ncon; io.warn = warn;
  if (h->sep.size() != (size_t)nenv * RG_NSEP) h->sep.assign((size_t)nenv * RG_NSEP, 0xfff);
  io.sep = h->sep.data();
  for (int env = 0; env < nenv; env++) rg_env_step(&h->hm.view, h->L, h->scratch.data(), 0, io, env, nsub, final_forward, 1);
}
/* a[(n+1)(n+2)/2] packed lower rows (row n = right-hand side), env[n] first nonzero column per row, b[n] a second right-hand side,
   sidx[2n] = dof -> solver position, solver position -> dof (identity is fine); out[n] = solution for row n, fwd[n] = L^-1 b */
void rgc_chol(int n, float* a, const int* env, const float* b, const int* sidx, float* out, float* fwd) {
  RgModel m;
  memset(&m, 0, sizeof m);
  m.ns = n; m.nv = n; m.dof_sidx = sidx;
  RgLayout L;
  memset(&L, 0, sizeof L);
  std::vector<float> s((size_t)(n + 1) * (n + 2) / 2 + 2 * n + 8);
  const int A = 0, o = (n + 1) * (n + 2) / 2;
  for (int i = 0; i < o; i++) s[A + i] = a[i];
  const RgCtx c = {&m, &L, s.data(), nullptr, 0.0f};
  rg_cholesky(c, A, env);
  for (int i = 0; i < o; i++) a[i] = s[A + i];   /* the factor, with y = L^-1 rhs in row n */
  rg_chol_back(c, A, env, o);
  for (int i = 0; i < n; i++) out[i] = s[o + i];
  for (int i = 0; i < n; i++) s[A + RG_TRI(n, 0) + i] = b[i];
  rg_chol_forward(c, A, env);
  for (int i = 0; i < n; i++) fwd[i] = s[A + RG_TRI(n, 0) + i];
}
}
