/* rg_emu_support.cpp -- TEST INFRASTRUCTURE ONLY: the hull support mapping of the CPU emulation build (tests/emu/librg_emu.so)
 * on its own.  The narrow phase's rg_hull_scan scans the candidate list of the query direction's cell (rg_host.h:
 * rg_host_hull_cells); these entry points run it, group-shared like rg_mpr_batch and one-lane like rg_support, next to the
 * whole-hull scan, reach the lists, and apply a mesh_vert edit the way rg_model_set_field does.  This file compiles the
 * emulation build's own source with the same flags, so RgeHandle has the same layout as in the library that created the
 * handle. */
#include <chrono>

#include "../emu/rg_emu.cpp"

/* the winner of rg_hull_scan over the RG_GRP lanes of a group (their arg-max, as rg_group_argmax combines it) */
static int rge_group_scan(const RgModel& m, const RgGeomView& v, const float* dl) {
  float best[RG_GRP]; int idx[RG_GRP];
  for (int gl = 0; gl < RG_GRP; gl++) rg_hull_scan(m, v, dl, 0, gl, RG_GRP, best[gl], idx[gl]);
  for (int o = RG_GRP / 2; o > 0; o >>= 1) {
    float nb[RG_GRP]; int ni[RG_GRP];
    for (int l = 0; l < RG_GRP; l++) {
      float bv = best[l]; int bi = idx[l];
      const float ov = best[l ^ o]; const int oi = idx[l ^ o];
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
      nb[l] = bv; ni[l] = bi;
    }
    memcpy(best, nb, sizeof best); memcpy(idx, ni, sizeof idx);
  }
  return idx[0];
}

extern "C" {
int rge_support_ncell(void) { return RG_NCELL; }
int rge_support_celln(void) { return RG_CELLN; }
/* the lists: table [nmesh][RG_NCELL][2] (first entry, count) and the entries [ncand_cap][4] (x, y, z, vertex id bits) */
const int* rge_support_table(void* hv) { return ((RgeHandle*)hv)->hm.view.mesh_cell; }
const float* rge_support_entries(void* hv, int* cap) { *cap = ((RgeHandle*)hv)->hm.view.ncand_cap; return ((RgeHandle*)hv)->hm.view.mesh_cand4; }
int rge_support_cell(const float* dl) { return rg_hull_cell(dl); }
/* winners (vertex ids local to hull `mesh`) of n hull-frame directions dirs[n][3]: out[4 k] = group-shared list scan,
   out[4 k + 1] = group-shared whole-hull scan, out[4 k + 2] = one-lane list scan, out[4 k + 3] = one-lane whole-hull scan */
void rge_support_scan(void* hv, int mesh, const float* dirs, int n, int* out) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  RgModel full = m;
  std::vector<int> none(2 * (size_t)m.nmesh * RG_NCELL, -1);   /* every cell count -1: the whole-hull scan */
  full.mesh_cell = none.data();
  RgGeomView v;
  memset(&v, 0, sizeof v);
  v.type = RG_GEOM_MESH; v.mid = mesh;
  for (int k = 0; k < n; k++) {
    const float* dl = dirs + 3 * k;
    out[4 * k] = rge_group_scan(m, v, dl);
    out[4 * k + 1] = rge_group_scan(full, v, dl);
    float b;
    rg_hull_scan(m, v, dl, 0, 0, 1, b, out[4 * k + 2]);
    rg_hull_scan(full, v, dl, 0, 0, 1, b, out[4 * k + 3]);
  }
}
/* rg_model_set_field("mesh_vert", ...) on the emulated model: the float copy, the padded copy and the lists */
void rge_support_set_vert(void* hv, const double* v) {
  RgModel& m = ((RgeHandle*)hv)->hm.view;
  float* d = (float*)m.mesh_vert;
  for (int k = 0; k < 3 * m.nmeshvert; k++) d[k] = (float)v[k];
  rg_host_pad_verts(m);
  rg_host_refresh_cells(m);
}
/* seconds one construction of every list of the model takes (rg_host_cells) */
double rge_support_build_seconds(void* hv) {
  const RgModel& m = ((RgeHandle*)hv)->hm.view;
  std::vector<int> table, ids;
  const auto t0 = std::chrono::steady_clock::now();
  rg_host_cells(m.mesh_vert4, m.mesh_vertadr, m.mesh_vertnum, m.nmesh, table, ids);
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}
}
