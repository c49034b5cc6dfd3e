/* rg_emu.cpp -- CPU EMULATION BUILD of the CUDA engine's device code.  TEST INFRASTRUCTURE ONLY.
 *
 * Compiles robogym_b200/csrc/rg_*.inl with -DRG_EMU: every warp phase becomes a loop over 32
 * lanes (see rg_defs.h).  It lets the CPU-only test tier (`pytest -m "not gpu"`) check the
 * kernel's fp32 logic against the fp64 oracle; it is not reachable from the package and the
 * product path never falls back to it.  One translation unit holds every entry point, so a
 * handle never crosses into a library with a different idea of RgeHandle.
 */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_step.inl"
#include "../../robogym_b200/csrc/rg_obs.inl"    /* with rg_goal.inl and rg_place.inl */
#include "../../robogym_b200/csrc/rg_host.h"

#include <stdio.h>
#include <stdlib.h>

#include <chrono>

struct RgeHandle { RgHostModel hm; RgLayout L; std::vector<float> scratch; std::vector<int> sep; const float* mocap_pos = nullptr; const float* mocap_quat = nullptr; float* sensordata = nullptr; };

/* the winner of rg_hull_scan over the RG_GRP lanes of a group (their arg-max, as rg_group_argmax combines it) */
static int rge_group_scan(const RgModel& m, const RgGeomView& v, const float* dl) {
  float best[RG_GRP]; int idx[RG_GRP];
  for (int gl = 0; gl < RG_GRP; gl++) rg_hull_scan(m, v, dl, 0, gl, RG_GRP, best[gl], idx[gl]);
  for (int o = RG_GRP / 2; o > 0; o >>= 1) {
    float nb[RG_GRP]; int ni[RG_GRP];
    for (int l = 0; l < RG_GRP; l++) {
      float bv = best[l]; int bi = idx[l];
      const float ov = best[l ^ o]; const int oi = idx[l ^ o];
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      nb[l] = bv; ni[l] = bi;
    }
    memcpy(best, nb, sizeof best); memcpy(idx, ni, sizeof idx);
  }
  return idx[0];
}

static const char* g_goal_err = "";
static const char* g_obs_err = "";

extern "C" {

/* ---- handles: load a model blob, edit its arrays, step a batch of environments */
void* rge_create_ex(const void* blob, size_t len, int ncon, int nel, int tile) {
  RgeHandle* h = new RgeHandle();
  std::string err;
  if (!rg_host_load(blob, len, h->hm, err)) { fprintf(stderr, "rge_create: %s\n", err.c_str()); delete h; return nullptr; }
  h->L = rg_make_layout(h->hm.view, ncon ? ncon : RG_NCON, nel ? nel : RG_NEL, tile ? tile : RG_TILE);
  h->scratch.assign(h->L.total, 0.0f);
  return h;
}
void* rge_create(const void* blob, size_t len) { return rge_create_ex(blob, len, 0, 0, 0); }
int rge_ncon(void* hv) { return ((RgeHandle*)hv)->L.ncon; }
int rge_pidw(void* hv) { return ((RgeHandle*)hv)->hm.view.pidw; }
/* the blob's name tables as parsed by the shared host loader (what rg_model_name2id serves) */
int rge_name2id(void* hv, const char* typ, const char* name) {
  RgeHandle* h = (RgeHandle*)hv;
  auto it = h->hm.names.find(typ);
  if (it == h->hm.names.end()) return -1;
  for (size_t i = 0; i < it->second.size(); i++) if (it->second[i] == name) return (int)i;
  return -1;
}
#ifdef RG_STATS
void rge_stats(long long* out) { out[0] = rg_stat_support; out[1] = rg_stat_climb; out[2] = rg_stat_mpr; out[3] = rg_stat_mpr_hit; out[4] = rg_stat_maxsup; for (int i = 0; i < 128; i++) out[8 + i] = rg_stat_hist[i / 64][i % 64]; for (int i = 0; i < 16; i++) out[136 + i] = rg_stat_x[i]; for (int i = 0; i < 16; i++) out[152 + i] = rg_stat_iterhist[i]; for (int i = 0; i < 16; i++) out[168 + i] = rg_stat_fliphist[i]; }
#endif
/* data.mocap_pos / mocap_quat rows ([nenv][nmocap*3], [nenv][nmocap*4]) used by the following rge_step calls (or null) */
void rge_set_mocap(void* hv, const float* pos, const float* quat) { ((RgeHandle*)hv)->mocap_pos = pos; ((RgeHandle*)hv)->mocap_quat = quat; }
void rge_set_sensordata(void* hv, float* out) { ((RgeHandle*)hv)->sensordata = out; }   /* [nenv][nsensordata] or null */
/* mj_setConst of the (edited) model: any output may be null */
void rge_set_const(void* hv, float* dof_invweight0, float* body_invweight0, float* tendon_invweight0, float* tendon_length0, float* body_subtreemass, float* opt_meaninertia) {
  RgeHandle* h = (RgeHandle*)hv;
  RgSetConstOut o = {dof_invweight0, body_invweight0, tendon_invweight0, tendon_length0, body_subtreemass, opt_meaninertia};
  rg_env_setconst(&h->hm.view, h->L, h->scratch.data(), 0, o);
}
void rge_destroy(void* hv) { delete (RgeHandle*)hv; }
int rge_dbg_size(void* hv) { return rg_dbg_size(((RgeHandle*)hv)->hm.view, ((RgeHandle*)hv)->L.ncon); }
int rge_scratch_floats(void* hv) { return ((RgeHandle*)hv)->L.total; }
/* the handle's scratch layout (rg_make_layout) as ints in RgLayout's declaration order; returns how many it has (copies at most n) */
int rge_layout(void* hv, int* out, int n) {
  const RgLayout& L = ((RgeHandle*)hv)->L;
  const int k = (int)(sizeof(RgLayout) / sizeof(int));
  memcpy(out, &L, sizeof(int) * (size_t)(n < k ? n : k));
  return k;
}
int rge_small_bytes(void* hv) { return (int)((RgeHandle*)hv)->hm.small_bytes; }
/* writable pointer to a model array, the blob's or a derived one (float32/int32 copy), so tests can edit parameters */
void* rge_model_field(void* hv, const char* name, int* count) {
  RgHostField f;
  if (!rg_host_field(((RgeHandle*)hv)->hm.view, name, f)) return nullptr;
  *count = (int)f.count;
  return f.p;
}

void rge_step(void* hv, int nenv, float* qpos, float* qvel, float* ctrl, float* pid, float* warm, float* time, const float* xfrc,
              const float* timestep, float* site_xpos, float* body_xpos, float* body_xquat, float* geom_xpos, float* act_force, float* qacc,
              float* contact, int* ncon, int* warn, float* dbg, int nsub, int final_forward) {
  RgeHandle* h = (RgeHandle*)hv;
  RgBatchIO io;
  io.nenv = nenv; io.qpos = qpos; io.qvel = qvel; io.ctrl = ctrl; io.pid = pid; io.warm = warm; io.time = time; io.xfrc = xfrc;
  io.timestep = timestep; io.site_xpos = site_xpos; io.body_xpos = body_xpos; io.body_xquat = body_xquat; io.geom_xpos = geom_xpos;
  io.act_force = act_force; io.qacc = qacc; io.contact = contact; io.ncon = ncon; io.warn = warn; io.dbg = dbg; io.cost = nullptr; io.body_xvel = nullptr; io.mocap_pos = h->mocap_pos; io.mocap_quat = h->mocap_quat; io.sensordata = h->sensordata;
  if (h->sep.size() != (size_t)nenv * RG_NSEP) h->sep.assign((size_t)nenv * RG_NSEP, 0xfff);   /* like the engine's per-batch buffer */
  io.sep = h->sep.data();
  for (int env = 0; env < nenv; env++) rg_env_step(&h->hm.view, h->L, h->scratch.data(), 0, io, env, nsub, final_forward, 1);
}

/* ---- per-environment pair lists (rg_batch_update_pairs)
 *   rge_pairs:     the device code's compaction (rg_env_pairs) of the handle's static pair list for one geom_dataid row;
 *   rge_use_pairs: make the handle's model view stream `list` (n pairs, packed g1 | g2 << 16) instead of the static list, as
 *                  the engine does for an environment with its own list.  `list` must outlive the following rge_step calls. */
int rge_pairs(void* hv, const int* dataid, unsigned* out, int cap, int* warn) {
  return rg_env_pairs(((RgeHandle*)hv)->hm.view, dataid, out, cap, warn);
}
void rge_use_pairs(void* hv, const unsigned* list, int n) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  m.pair_packed = nullptr;
  m.pair_geom1 = (const int*)list;
  m.pair_geom2 = nullptr;
  m.npair = n;
}

/* ---- per-environment geom scale (rg_batch_bind_param of geom_mesh_scale)
 *   rge_use_geom_scale: the handle's model view reads `row` ([ngeom] floats, or NULL = unbound: every factor 1) in the
 *                       following rge_step calls; `row` must outlive them.  Returns ngeom. */
int rge_use_geom_scale(void* hv, const float* row) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  m.geom_mesh_scale = row;
  return m.ngeom;
}

/* ---- hull support mapping: rg_hull_scan over the candidate list of the query direction's cell (rg_host.h:
 * rg_host_hull_cells), group-shared like rg_mpr_batch and one-lane like rg_support, next to the whole-hull scan */
int rge_support_ncell(void) { return RG_NCELL; }
int rge_support_celln(void) { return RG_CELLN; }
/* the lists: table [nmesh][RG_NCELL][2] (first entry, count) and the entries [ncand_cap][4] (x, y, z, vertex id bits) */
const int* rge_support_table(void* hv) { return ((RgeHandle*)hv)->hm.view.mesh_cell; }
const float* rge_support_entries(void* hv, int* cap) { *cap = ((RgeHandle*)hv)->hm.view.ncand_cap; return ((RgeHandle*)hv)->hm.view.mesh_cand4; }
int rge_support_cell(const float* dl) { return rg_hull_cell(dl); }
/* winners (vertex ids local to hull `mesh`) of n hull-frame directions dirs[n][3]: out[4 k] = group-shared list scan,
   out[4 k + 1] = group-shared whole-hull scan, out[4 k + 2] = one-lane list scan, out[4 k + 3] = one-lane whole-hull scan */
void rge_support_scan(void* hv, int mesh, const float* dirs, int n, int* out) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  RgModel full = m;
  std::vector<int> none(2 * (size_t)m.nmesh * RG_NCELL, -1);   /* every cell count -1: the whole-hull scan */
  full.mesh_cell = none.data();
  RgGeomView v;
  memset(&v, 0, sizeof v);
  v.type = RG_GEOM_MESH; v.mid = mesh;
  for (int k = 0; k < n; k++) {
    const float* dl = dirs + 3 * k;
    out[4 * k] = rge_group_scan(m, v, dl);
    out[4 * k + 1] = rge_group_scan(full, v, dl);
    float b;
    rg_hull_scan(m, v, dl, 0, 0, 1, b, out[4 * k + 2]);
    rg_hull_scan(full, v, dl, 0, 0, 1, b, out[4 * k + 3]);
  }
}
/* rg_model_set_field("mesh_vert", ...) on the emulated model: the float copy, the padded copy and the lists */
void rge_support_set_vert(void* hv, const double* v) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  float* d = (float*)m.mesh_vert;
  for (int k = 0; k < 3 * m.nmeshvert; k++) d[k] = (float)v[k];
  rg_host_pad_verts(m);
  rg_host_refresh_cells(m);
}
/* seconds one construction of every list of the model takes (rg_host_cells) */
double rge_support_build_seconds(void* hv) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  std::vector<int> table, ids;
  const auto t0 = std::chrono::steady_clock::now();
  rg_host_cells(m.mesh_vert4, m.mesh_vertadr, m.mesh_vertnum, m.nmesh, table, ids);
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

/* ---- placement (rg_place.inl)
 *   rge_philox:    n outputs of Philox4x32-10 for counters ctr[n][4] under key (k0, k1);
 *   rge_body_aabb: (center, half size) of one body of the handle's model rotated by quat (w x y z), from the given rows
 *                  (NULL: the model's array), reduced over the 32 emulated lanes;
 *   rge_place:     rg_place_objects for every environment whose mask byte is set (mask NULL: all). */
void rge_philox(int n, const uint32_t* ctr, uint32_t k0, uint32_t k1, uint32_t* out) {
  for (int i = 0; i < n; i++) {
    const RgU4 c = {ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]};
    const RgU4 r = rg_philox(c, k0, k1);
    out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
  }
}
void rge_body_aabb(void* hv, int body, const double* quat, const int* dataid, const float* pos, const float* gquat, const float* size,
                   const float* mscale, const float* gscale, double* out) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  const RgAabbRows r = {dataid ? dataid : m.geom_dataid, pos ? pos : m.geom_pos, gquat ? gquat : m.geom_quat, size ? size : m.geom_size, mscale, gscale};
  double R[9], lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  rg_quat2mat_d(R, quat);
  for (int lane = 0; lane < 32; lane++) {
    double l[3], h[3];
    rg_aabb_lane(m, r, body, R, lane, l, h);
    for (int a = 0; a < 3; a++) { lo[a] = fmin(lo[a], l[a]); hi[a] = fmax(hi[a], h[a]); }
  }
  rg_aabb_finish(lo, hi, out);
}
void rge_place(int nenv, int nobj, const double* bbox, const uint8_t* active, const double* table, const double* area, int mode, int max_trials,
               int max_per_object, double ratio, double dmin, const double* anchor, uint32_t seed, uint32_t epoch, const uint8_t* mask,
               double* pos, int* status) {
  RgPlaceArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.max_trials = max_trials; a.max_per_object = max_per_object;
  a.ratio = ratio; a.dmin = dmin;
  for (int k = 0; k < 3; k++) { a.table_pos[k] = table[k]; a.table_size[k] = table[3 + k]; }
  a.seed = seed; a.epoch = epoch;
  a.bbox = bbox; a.active = active; a.area = area; a.anchor = anchor; a.mask = mask; a.pos = pos; a.status = status;
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_place_env(a, (uint32_t)e, 0);
}

/* ---- goal evaluation and goal orientations (rg_goal.inl): a warp phase is one lane walking every slot
 *   rge_goal:           rg_rearrange_goal for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with
 *                       the message in rge_goal_error() for arguments the engine refuses;
 *   rge_goal_rot:       rg_goal_orientations likewise;
 *   rge_parallel_quats: the kernel's tables, PARALLEL_QUATS (24 x 4) then PARALLEL_QUATS_180 (4 x 4). */
const char* rge_goal_error(void) { return g_goal_err; }
int rge_goal(const rg_goal_in* in, const uint8_t* mask, double* prev, const rg_goal_out* out) {
  static RgGoalArgs a;
  static RgGoalScratch s;
  const char* err = rg_goal_make_args(in, mask, prev, out, a);
  if (err) { g_goal_err = err; return -1; }
  for (int e = 0; e < a.nenv; e++)
    if (!mask || mask[e]) rg_goal_env(a, s, e, 0);
  return 0;
}
void rge_goal_rot(int nenv, int nobj, const double* base, const uint8_t* active, int mode, uint32_t seed, uint32_t epoch,
                  const uint8_t* mask, double* out) {
  RgGoalRotArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.seed = seed; a.epoch = epoch;
  a.base = base; a.active = active; a.mask = mask; a.out = out;
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_goal_rot_env(a, e, 0);
}
void rge_parallel_quats(double* out) {
  for (int k = 0; k < 24; k++) for (int c = 0; c < 4; c++) out[4 * k + c] = rg_parallel_quats[k][c];
  for (int k = 0; k < 4; k++) for (int c = 0; c < 4; c++) out[96 + 4 * k + c] = rg_parallel_quats_180[k][c];
}

/* ---- rearrange observations (rg_obs.inl): a warp phase is one lane walking every contact and every slot
 *   rge_obs: rg_rearrange_obs for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with the message
 *            in rge_obs_error() for arguments the engine refuses. */
const char* rge_obs_error(void) { return g_obs_err; }
int rge_obs(const rg_obs_in* in, const uint8_t* mask, const rg_obs_out* out) {
  static RgObsArgs a;
  const char* err = rg_obs_make_args(in, mask, out, a);
  if (err) { g_obs_err = err; return -1; }
  for (int e = 0; e < a.in.nenv; e++)
    if (!mask || mask[e]) rg_obs_env(a, e, 0);
  return 0;
}
}
