/* rg_emu_modify.cpp -- CPU EMULATION BUILD of the goal modifier (rg_goal_modify, robogym_b200/csrc/rg_place.inl).  TEST
 * INFRASTRUCTURE ONLY.
 *
 * Compiles rg_place.inl with -DRG_EMU, as rg_emu.cpp compiles every kernel file; the modifier runs one thread per environment,
 * so the emulation is that thread's code called per environment.  It holds no handles, so it lives in a library of its own
 * (tests/emu/pyemu_modify.py builds and loads it).
 *   rge_goal_modify: rg_goal_modify for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with the
 *                    message in rge_modify_error() for arguments the engine refuses.
 */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_place.inl"

static const char* g_modify_err = "";

extern "C" {
const char* rge_modify_error(void) { return g_modify_err; }
int rge_goal_modify(int nenv, int nobj, int kind, const uint8_t* active, const double* object_size, const double* ratio, const double* target_height,
                    double min_h, double max_h, double pickup, double stacking, int fixed_order, uint32_t seed, uint32_t epoch, const uint8_t* mask,
                    double* pos) {
  RgModifyArgs a;
  const char* err = rg_modify_make_args(nenv, nobj, kind, active, object_size, ratio, target_height, min_h, max_h, pickup, stacking, fixed_order, seed, epoch,
                                        mask, pos, a);
  if (err) { g_modify_err = err; return -1; }
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_modify_env(a, (uint32_t)e);
  return 0;
}
}
