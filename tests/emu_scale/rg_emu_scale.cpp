/* rg_emu_scale.cpp -- TEST INFRASTRUCTURE ONLY: reach the engine-derived `mesh_scale` array (rg_host.h) of a handle created by the
 * CPU emulation build (tests/emu/librg_emu.so).  `mesh_scale` is not an array of include/rg_model_fields.h, so rge_model_field does
 * not serve it.  This file compiles the emulation build's own source with the same flags, so RgeHandle has the same layout as in
 * the library that created the handle; it only reads the handle. */
#include "../emu/rg_emu.cpp"

extern "C" float* rge_mesh_scale(void* hv, int* count) {
  RgeHandle* h = (RgeHandle*)hv;
  *count = h->hm.view.nmesh;
  return (float*)h->hm.view.mesh_scale;
}
