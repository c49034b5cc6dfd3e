/* rg_emu_obs.cpp -- TEST INFRASTRUCTURE ONLY: the device code of rg_obs.inl (rearrange observations) on the CPU emulation
 * build: a warp phase is one lane walking every contact and every slot.  Compiled with the emulation build's flags.
 *   rge_obs: rg_rearrange_obs for every environment whose mask byte is set (mask NULL: all); returns 0, or -1 with the message
 *            in rge_obs_error() for arguments the engine refuses. */
#define RG_EMU 1
#include "../../robogym_b200/csrc/rg_obs.inl"

static const char* g_obs_err = "";

extern "C" const char* rge_obs_error(void) { return g_obs_err; }

extern "C" int rge_obs(const rg_obs_in* in, const uint8_t* mask, const rg_obs_out* out) {
  static RgObsArgs a;
  const char* err = rg_obs_make_args(in, mask, out, a);
  if (err) { g_obs_err = err; return -1; }
  for (int e = 0; e < a.in.nenv; e++)
    if (!mask || mask[e]) rg_obs_env(a, e, 0);
  return 0;
}
