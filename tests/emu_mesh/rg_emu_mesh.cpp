/* rg_emu_mesh.cpp -- TEST INFRASTRUCTURE ONLY: per-environment pair lists (rg_batch_update_pairs) for a handle created by the
 * CPU emulation build (tests/emu/librg_emu.so).  Like tests/emu_scale, this compiles the emulation build's own source with the
 * same flags, so RgeHandle has the same layout as in the library that created the handle.
 *   rge_pairs:     the device code's compaction (rg_env_pairs) of the handle's static pair list for one geom_dataid row;
 *   rge_use_pairs: make the handle's model view stream `list` (n pairs, packed g1 | g2 << 16) instead of the static list, as
 *                  the engine does for an environment with its own list.  `list` must outlive the following rge_step calls. */
#include "../emu/rg_emu.cpp"

extern "C" int rge_pairs(void* hv, const int* dataid, unsigned* out, int cap, int* warn) {
  return rg_env_pairs(((RgeHandle*)hv)->hm.view, dataid, out, cap, warn);
}
extern "C" void rge_use_pairs(void* hv, const unsigned* list, int n) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  m.pair_packed = nullptr;
  m.pair_geom1 = (const int*)list;
  m.pair_geom2 = nullptr;
  m.npair = n;
}
