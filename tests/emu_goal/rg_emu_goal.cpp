/* rg_emu_goal.cpp -- TEST INFRASTRUCTURE ONLY: the device code of rg_goal.inl (goal evaluation and goal orientations) on the
 * CPU emulation build: a warp phase is one lane walking every slot.  Compiled with the emulation build's flags.
 *   rge_goal:          rg_rearrange_goal for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with
 *                      the message in rge_goal_error() for arguments the engine refuses;
 *   rge_goal_rot:      rg_goal_orientations likewise;
 *   rge_parallel_quats: the kernel's tables, PARALLEL_QUATS (24 x 4) then PARALLEL_QUATS_180 (4 x 4). */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_goal.inl"

static const char* g_goal_err = "";

extern "C" const char* rge_goal_error(void) { return g_goal_err; }

extern "C" int rge_goal(const rg_goal_in* in, const uint8_t* mask, double* prev, const rg_goal_out* out) {
  static RgGoalArgs a;
  static RgGoalScratch s;
  const char* err = rg_goal_make_args(in, mask, prev, out, a);
  if (err) { g_goal_err = err; return -1; }
  for (int e = 0; e < a.nenv; e++)
    if (!mask || mask[e]) rg_goal_env(a, s, e, 0);
  return 0;
}

extern "C" void rge_goal_rot(int nenv, int nobj, const double* base, const uint8_t* active, int mode, uint32_t seed, uint32_t epoch,
                             const uint8_t* mask, double* out) {
  RgGoalRotArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.seed = seed; a.epoch = epoch;
  a.base = base; a.active = active; a.mask = mask; a.out = out;
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_goal_rot_env(a, e, 0);
}

extern "C" void rge_parallel_quats(double* out) {
  for (int k = 0; k < 24; k++) for (int c = 0; c < 4; c++) out[4 * k + c] = rg_parallel_quats[k][c];
  for (int k = 0; k < 4; k++) for (int c = 0; c < 4; c++) out[96 + 4 * k + c] = rg_parallel_quats_180[k][c];
}
