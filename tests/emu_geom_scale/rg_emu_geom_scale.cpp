/* rg_emu_geom_scale.cpp -- TEST INFRASTRUCTURE ONLY: give a handle created by the CPU emulation build (tests/emu/librg_emu.so)
 * the per-mesh-geom scale row `geom_mesh_scale` that the engine binds per environment (rg_batch_bind_param).  Like
 * tests/emu_scale, this compiles the emulation build's own source with the same flags, so RgeHandle has the same layout as in
 * the library that created the handle.
 *   rge_use_geom_scale: the handle's model view reads `row` ([ngeom] floats, or NULL = unbound: every factor 1) in the
 *                       following rge_step calls; `row` must outlive them.  Returns ngeom. */
#include "../emu/rg_emu.cpp"

extern "C" int rge_use_geom_scale(void* hv, const float* row) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  m.geom_mesh_scale = row;
  return m.ngeom;
}
