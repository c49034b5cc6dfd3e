/* rg_emu_groups.cpp -- CPU EMULATION BUILD of the object groups (rg_object_groups, robogym_b200/csrc/rg_groups.inl).  TEST
 * INFRASTRUCTURE ONLY.
 *
 * Compiles rg_groups.inl with -DRG_EMU, as rg_emu.cpp compiles every kernel file: the same argument checks, then the kernel's
 * per-environment code on the host, reading the host inputs in place.  It holds no handles, so it lives in a library of its
 * own (tests/emu/pyemu_groups.py builds and loads it).
 *   rge_object_groups: rg_object_groups for every environment whose mask byte is set (mask NULL: all), outputs in host
 *                      memory; returns 0, or -1 with the message in rge_groups_error() for arguments the engine refuses.
 */
#define RG_EMU 1
#include <string.h>
#include "../../robogym_b200/csrc/rg_groups.inl"

static const char* g_groups_err = "";

extern "C" {
const char* rge_groups_error(void) { return g_groups_err; }
int rge_object_groups(const rg_groups_in* in, const uint8_t* mask, int mask_len, const rg_groups_out* out) {
  RgGroupsArgs a;
  memset(&a, 0, sizeof(a));
  const char* err = rg_groups_check(in, mask_len, mask != nullptr, out, a);
  if (err) { g_groups_err = err; return -1; }
  a.active = in->active;
  a.fixed = in->group_mode == RG_GROUPS_FIXED ? in->fixed_counts : nullptr;
  a.palette = a.n_palette ? in->palette : nullptr;
  a.mask = mask;
  for (int e = 0; e < a.nenv; e++)
    if (!mask || mask[e]) rg_groups_env(a, (uint32_t)e);
  return 0;
}
}
