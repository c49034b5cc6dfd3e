/* rg_emu_place.cpp -- TEST INFRASTRUCTURE ONLY: the device code of rg_place.inl (Philox, rotated bounding boxes, placement) on
 * the CPU emulation build.  Like tests/emu_mesh, this compiles the emulation build's own source with the same flags, so a
 * handle created by tests/emu/librg_emu.so has the same layout here.
 *   rge_philox:    n outputs of Philox4x32-10 for counters ctr[n][4] under key (k0, k1);
 *   rge_body_aabb: (center, half size) of one body of the handle's model rotated by quat (w x y z), from the given rows
 *                  (NULL: the model's array), reduced over the 32 emulated lanes;
 *   rge_place:     rg_place_objects for every environment whose mask byte is set (mask NULL: all). */
#include "../emu/rg_emu.cpp"
#include "../../robogym_b200/csrc/rg_place.inl"

extern "C" void rge_philox(int n, const uint32_t* ctr, uint32_t k0, uint32_t k1, uint32_t* out) {
  for (int i = 0; i < n; i++) {
    const RgU4 c = {ctr[4 * i], ctr[4 * i + 1], ctr[4 * i + 2], ctr[4 * i + 3]};
    const RgU4 r = rg_philox(c, k0, k1);
    out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
  }
}

extern "C" void rge_body_aabb(void* hv, int body, const double* quat, const int* dataid, const float* pos, const float* gquat, const float* size,
                              const float* mscale, const float* gscale, double* out) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  const RgAabbRows r = {dataid ? dataid : m.geom_dataid, pos ? pos : m.geom_pos, gquat ? gquat : m.geom_quat, size ? size : m.geom_size, mscale, gscale};
  double R[9], lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  rg_quat2mat_d(R, quat);
  for (int lane = 0; lane < 32; lane++) {
    double l[3], h[3];
    rg_aabb_lane(m, r, body, R, lane, l, h);
    for (int a = 0; a < 3; a++) { lo[a] = fmin(lo[a], l[a]); hi[a] = fmax(hi[a], h[a]); }
  }
  rg_aabb_finish(lo, hi, out);
}

extern "C" void rge_place(int nenv, int nobj, const double* bbox, const uint8_t* active, const double* table, const double* area, int mode, int max_trials,
                          int max_per_object, double ratio, double dmin, const double* anchor, uint32_t seed, uint32_t epoch, const uint8_t* mask,
                          double* pos, int* status) {
  RgPlaceArgs a;
  a.nenv = nenv; a.nobj = nobj; a.mode = mode; a.max_trials = max_trials; a.max_per_object = max_per_object;
  a.ratio = ratio; a.dmin = dmin;
  for (int k = 0; k < 3; k++) { a.table_pos[k] = table[k]; a.table_size[k] = table[3 + k]; }
  a.seed = seed; a.epoch = epoch;
  a.bbox = bbox; a.active = active; a.area = area; a.anchor = anchor; a.mask = mask; a.pos = pos; a.status = status;
  for (int e = 0; e < nenv; e++)
    if (!mask || mask[e]) rg_place_env(a, (uint32_t)e, 0);
}
