/* rg_emu_layout.cpp -- CPU EMULATION BUILD of the layout goals (rg_layout_goals, robogym_b200/csrc/rg_place.inl).  TEST
 * INFRASTRUCTURE ONLY.
 *
 * Compiles rg_place.inl with -DRG_EMU, as rg_emu.cpp compiles every kernel file: the warp's ballot over 32 retries becomes a
 * loop over them and the per-object work one lane's.  It holds no handles, so it lives in a library of its own
 * (tests/emu/pyemu_layout.py builds and loads it).
 *   rge_layout_goals: rg_layout_goals for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with the
 *                     message in rge_layout_error() for arguments the engine refuses.
 */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_place.inl"

static const char* g_layout_err = "";

extern "C" {
const char* rge_layout_error(void) { return g_layout_err; }
int rge_layout_goals(int nenv, int nobj, int kind, const double* bbox, const uint8_t* active, const double* table, const double* area,
                     const double* object_size, const double* distance_mul, const double* rel, int max_retry, uint32_t seed, uint32_t epoch,
                     const uint8_t* mask, double* pos, double* quat, int* status, double* angle, int* retry) {
  RgLayoutArgs a;
  const char* err = rg_layout_make_args(nenv, nobj, kind, bbox, active, table, area, object_size, distance_mul, rel, max_retry, seed, epoch, mask, pos,
                                        quat, status, angle, retry, a);
  if (err) { g_layout_err = err; return -1; }
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_layout_env(a, (uint32_t)e, 0);
  return 0;
}
}
