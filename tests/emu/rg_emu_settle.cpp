/* rg_emu_settle.cpp -- CPU EMULATION BUILD of the settle launch (rg_step_settle).  TEST INFRASTRUCTURE ONLY.
 *
 * The emulation library (rg_emu.cpp, every entry point and its handles) compiled once more with the two reads of dof_damping
 * routed through rows the settle can redirect (RG_DAMPING_PASSIVE / RG_DAMPING_IMPLICIT, rg_defs.h), plus masked stepping and
 * the settle.  Its handles belong to this library only; tests/emu/pyemu_settle.py builds and loads it.
 *   rges_step:   rge_step for the environments whose mask byte is set (mask NULL: all), as rg_step_subset launches them;
 *   rges_settle: rg_step_settle: nsub substeps with dof_damping[dofs[i]] = damping, written into the model view's damping row
 *                as the kernel writes it into the CTA's staged copy, then final_forward forward passes with the model's row.
 *                `reads` 1 or 2 instead gives the override to the passive force only (1) or to the implicit term of the Euler
 *                factor only (2), the other read keeping the model's row: what a settle that missed one read would compute.
 *                The other arguments are rges_step's.
 */
#include <stdint.h>
static const float* rges_damp_passive = nullptr;
static const float* rges_damp_implicit = nullptr;
#define RG_DAMPING_PASSIVE(m) (rges_damp_passive ? rges_damp_passive : (m).dof_damping)
#define RG_DAMPING_IMPLICIT(m) (rges_damp_implicit ? rges_damp_implicit : (m).dof_damping)
#include "rg_emu.cpp"

extern "C" {

void rges_step(void* hv, const uint8_t* mask, int nenv, float* qpos, float* qvel, float* ctrl, float* pid, float* warm, float* time,
               const float* xfrc, const float* timestep, float* site_xpos, float* body_xpos, float* body_xquat, float* geom_xpos,
               float* act_force, float* qacc, float* contact, int* ncon, int* warn, float* dbg, int nsub, int final_forward) {
  RgeHandle* h = (RgeHandle*)hv;
  RgBatchIO io;
  io.nenv = nenv; io.qpos = qpos; io.qvel = qvel; io.ctrl = ctrl; io.pid = pid; io.warm = warm; io.time = time; io.xfrc = xfrc;
  io.timestep = timestep; io.site_xpos = site_xpos; io.body_xpos = body_xpos; io.body_xquat = body_xquat; io.geom_xpos = geom_xpos;
  io.act_force = act_force; io.qacc = qacc; io.contact = contact; io.ncon = ncon; io.warn = warn; io.dbg = dbg; io.cost = nullptr; io.body_xvel = nullptr;
  io.mocap_pos = h->mocap_pos; io.mocap_quat = h->mocap_quat; io.sensordata = h->sensordata;
  if (h->sep.size() != (size_t)nenv * RG_NSEP) h->sep.assign((size_t)nenv * RG_NSEP, 0xfff);
  io.sep = h->sep.data();
  for (int env = 0; env < nenv; env++)
    if (!mask || mask[env]) rg_env_step(&h->hm.view, h->L, h->scratch.data(), 0, io, env, nsub, final_forward, 1);
}

void rges_settle(void* hv, const uint8_t* mask, int nenv, float* qpos, float* qvel, float* ctrl, float* pid, float* warm, float* time,
                 const float* xfrc, const float* timestep, float* site_xpos, float* body_xpos, float* body_xquat, float* geom_xpos,
                 float* act_force, float* qacc, float* contact, int* ncon, int* warn, float* dbg, const int* dofs, int ndof, float damping,
                 int nsub, int final_forward, int reads) {
  RgeHandle* h = (RgeHandle*)hv;
  RgHostField f;
  rg_host_field(h->hm.view, "dof_damping", f);
  float* row = (float*)f.p;
  const std::vector<float> saved(row, row + f.count);
  std::vector<float> patched(saved);
  for (int i = 0; i < ndof; i++) patched[dofs[i]] = damping;
  if (reads == 3) memcpy(row, patched.data(), sizeof(float) * f.count);
  else if (reads == 1) rges_damp_passive = patched.data();
  else rges_damp_implicit = patched.data();
  rges_step(hv, mask, nenv, qpos, qvel, ctrl, pid, warm, time, xfrc, timestep, site_xpos, body_xpos, body_xquat, geom_xpos, act_force, qacc, contact,
            ncon, warn, dbg, nsub, 0);
  memcpy(row, saved.data(), sizeof(float) * f.count);
  rges_damp_passive = rges_damp_implicit = nullptr;
  if (final_forward > 0)
    rges_step(hv, mask, nenv, qpos, qvel, ctrl, pid, warm, time, xfrc, timestep, site_xpos, body_xpos, body_xquat, geom_xpos, act_force, qacc, contact,
              ncon, warn, dbg, 0, final_forward);
}
}
