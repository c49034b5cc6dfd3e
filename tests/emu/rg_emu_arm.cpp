/* rg_emu_arm.cpp -- CPU EMULATION BUILD of the robot reset's random action (rg_arm_sample_actions).  TEST INFRASTRUCTURE ONLY.
 * Compiles csrc/rg_arm.inl on the host; tests/emu/pyemu_arm.py builds and loads it.
 *   rgea_sample: component d of environment e for every environment of a [nenv] mask (NULL: all), as the kernel draws it. */
#define RG_EMU 1
#include <stdint.h>
#include "../../include/robogym_b200.h"
#include "../../robogym_b200/csrc/rg_step.inl"
#include "../../robogym_b200/csrc/rg_arm.inl"

extern "C" void rgea_sample(int nenv, int dim, uint32_t seed, uint32_t epoch, const uint8_t* mask, float* out) {
  for (int e = 0; e < nenv; e++) {
    if (mask && !mask[e]) continue;
    for (int d = 0; d < dim; d++) out[(size_t)e * dim + d] = rg_arm_sample(seed, (uint32_t)e, epoch, (uint32_t)d);
  }
}
