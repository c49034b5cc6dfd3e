/* rg_host.h -- host-side model loading shared by the CUDA engine and the CPU emulation build:
 * unpack the model blob (include/rg_model_fields.h) into one contiguous fp32/int32 arena whose
 * leading `small_bytes` hold every small per-body/joint/dof/geom array (staged into shared memory
 * by the kernel with one bulk copy) followed by the big read-only arrays (hull vertices, hull
 * adjacency, candidate pair list) that stay in global memory.
 */
#pragma once
#include <stdint.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "rg_defs.h"

struct RgHostModel {
  std::vector<char> arena;
  RgModel view;                 /* pointers into `arena` (host) */
  std::vector<size_t> offsets;  /* byte offset of every RgModel pointer field, in struct order */
  size_t small_bytes = 0;
  std::map<std::string, std::vector<std::string>> names;   /* objtype -> names ("" = unnamed), from the blob's RGNAMES1 section */
};

static inline size_t rg_align16(size_t x) { return (x + 15) & ~(size_t)15; }

/* (re)build the float4-padded hull vertices the narrow phase reads from mesh_vert (at load, and after mesh_vert was edited) */
static inline void rg_host_pad_verts(RgModel& m) {
  float* v4 = (float*)m.mesh_vert4;
  for (int k = 0; k < m.nmeshvert; k++) { v4[4 * k] = m.mesh_vert[3 * k]; v4[4 * k + 1] = m.mesh_vert[3 * k + 1]; v4[4 * k + 2] = m.mesh_vert[3 * k + 2]; v4[4 * k + 3] = 0.0f; }
}

/* ---- support candidate lists of the hulls (the narrow phase's rg_hull_scan).
 * The arg-max of x . d over a hull's vertices is a vertex whose normal cone holds d.  The sphere of directions is split into
 * RG_NCELL cells, a cube map: face = axis f of the largest |d_f| and its sign s, then an RG_CELLN x RG_CELLN grid over the
 * gnomonic coordinates (u, v) = (d_a, d_b) / |d_f| in [-1, 1]^2, a = (f + 1) % 3, b = (f + 2) % 3; cell id =
 * ((2 f + (s < 0)) * RG_CELLN + i) * RG_CELLN + j with i from u, j from v.  Each cell lists the vertices that can win there.
 *
 * Invariant.  Let Q be the cell's (u, v) square dilated by RG_CELL_PAD (more than the device lookup's rounding, which is a
 * few ulp: < 1e-6 in u), R = max |x| over the hull (vertices are centred on the hull), eps = 1e-5 R.  The list holds every
 * vertex w with w . d >= max_x x . d - eps |d| for some d = s e_f + u e_a + v e_b, (u, v) in Q.  Any fp32 maximum of the
 * 3-term dot the device computes is within 2 * 3 * 2^-24 R |d| < eps |d| of the exact maximum, so every vertex that ties
 * for it is listed, and the list scan returns the lowest-id fp32 winner, as the whole-hull scan does.
 *
 * Construction (why it keeps the invariant).  h_w(u, v) = max_x (x - w) . d(u, v) is 2R-Lipschitz in (u, v): d moves by
 * du e_a + dv e_b and |x - w| <= 2R.  On the dilated cell |d| <= D = sqrt(1 + umax^2 + vmax^2), so a listed vertex only needs
 * h_w <= eps D somewhere in Q.  For a rectangle of Q with centre c and half-diagonal rho, every such w of the rectangle has
 * h_w(c) <= eps D + 2 R rho =: tol(rho); the set S(rect) = {w : h_w(c) <= tol(rho)} therefore covers the rectangle.  The
 * rectangle is split into quarters recursively (to RG_CELL_DEPTH levels, or until S holds one vertex) and the list is the
 * union of the leaves' sets.  A quarter's set is a subset of its parent's (its centre is rho / 2 from the parent's, and
 * tol(rho / 2) + 2 R rho / 2 = tol(rho)), and so is the arg-max at its centre (h = 0 there), so each set is computed over
 * the parent's set only, with the same result as over the whole hull.  The double-precision evaluation errs by ~1e-16 R,
 * far inside eps. */
#define RG_CELL_PAD 1e-4
#define RG_CELL_DEPTH 5
struct RgCellBuild {
  const float* v4; int nv; double R, epsD;
  int f, a, b; double s;
  std::vector<char> mark;
  std::vector<std::vector<int>> pool;   /* one candidate buffer per recursion level */
};
static inline void rg_cell_rect(RgCellBuild& B, double u0, double u1, double v0, double v1, int depth) {
  const std::vector<int>& par = B.pool[depth];
  std::vector<int>& cur = B.pool[depth + 1];
  const double uc = 0.5 * (u0 + u1), vc = 0.5 * (v0 + v1);
  double d[3];
  d[B.f] = B.s; d[B.a] = uc; d[B.b] = vc;
  const double tol = B.epsD + B.R * sqrt((u1 - u0) * (u1 - u0) + (v1 - v0) * (v1 - v0));   /* eps D + 2 R rho */
  double mx = -1e300;
  for (int k : par) { const float* p = B.v4 + 4 * k; mx = fmax(mx, p[0] * d[0] + p[1] * d[1] + p[2] * d[2]); }
  cur.clear();
  for (int k : par) { const float* p = B.v4 + 4 * k; if (p[0] * d[0] + p[1] * d[1] + p[2] * d[2] >= mx - tol) cur.push_back(k); }
  if (depth + 1 == RG_CELL_DEPTH || cur.size() <= 1) { for (int k : cur) B.mark[k] = 1; return; }
  for (int q = 0; q < 4; q++)
    rg_cell_rect(B, (q & 1) ? uc : u0, (q & 1) ? u1 : uc, (q & 2) ? vc : v0, (q & 2) ? v1 : vc, depth + 1);
}
/* candidate lists of one hull (v4: its float4-padded vertices): cells[2 c] = first entry (relative to the hull's first),
   cells[2 c + 1] = count; the entries (ascending vertex ids per cell) are appended to `ids` */
static inline void rg_host_hull_cells(const float* v4, int nv, int* cells, std::vector<int>& ids) {
  RgCellBuild B;
  B.v4 = v4; B.nv = nv; B.R = 0.0;
  for (int k = 0; k < nv; k++) B.R = fmax(B.R, sqrt((double)v4[4 * k] * v4[4 * k] + (double)v4[4 * k + 1] * v4[4 * k + 1] + (double)v4[4 * k + 2] * v4[4 * k + 2]));
  B.mark.assign(nv, 0);
  B.pool.assign(RG_CELL_DEPTH + 1, std::vector<int>());
  for (int k = 0; k < nv; k++) B.pool[0].push_back(k);
  const size_t base = ids.size();
  const double w = 2.0 / RG_CELLN, pad = RG_CELL_PAD;
  for (int c = 0; c < RG_NCELL; c++) {
    const int face = c / (RG_CELLN * RG_CELLN), i = (c / RG_CELLN) % RG_CELLN, j = c % RG_CELLN;
    B.f = face >> 1; B.s = (face & 1) ? -1.0 : 1.0; B.a = (B.f + 1) % 3; B.b = (B.f + 2) % 3;
    const double u0 = -1.0 + w * i - pad, u1 = -1.0 + w * (i + 1) + pad, v0 = -1.0 + w * j - pad, v1 = -1.0 + w * (j + 1) + pad;
    const double um = fmax(fabs(u0), fabs(u1)), vm = fmax(fabs(v0), fabs(v1));
    B.epsD = 1e-5 * B.R * sqrt(1.0 + um * um + vm * vm);
    if (nv > 0) rg_cell_rect(B, u0, u1, v0, v1, 0);
    cells[2 * c] = (int)(ids.size() - base);
    for (int k = 0; k < nv; k++) if (B.mark[k]) { ids.push_back(k); B.mark[k] = 0; }
    cells[2 * c + 1] = (int)(ids.size() - base) - cells[2 * c];
  }
}
/* candidate lists of every hull (v4: float4-padded vertices of all hulls): table [nmesh][RG_NCELL][2] with model-wide entry
   offsets, entries = vertex ids local to their hull */
static inline void rg_host_cells(const float* v4, const int* vertadr, const int* vertnum, int nmesh, std::vector<int>& table, std::vector<int>& ids) {
  table.assign(2 * (size_t)nmesh * RG_NCELL, 0);
  ids.clear();
  for (int h = 0; h < nmesh; h++) {
    const size_t base = ids.size();
    int* cells = table.data() + 2 * (size_t)h * RG_NCELL;
    rg_host_hull_cells(v4 + 4 * (size_t)vertadr[h], vertnum[h], cells, ids);
    for (int c = 0; c < RG_NCELL; c++) cells[2 * c] += (int)base;
  }
}
/* write the lists into the arena (m.mesh_cell, m.mesh_cand4): a hull whose entries no longer fit in the room allocated at
   load (an edited mesh_vert with longer lists), or that has no lists (count -1 in `table`), gets count -1 in every cell,
   i.e. the whole-hull scan */
static inline void rg_host_store_cells(RgModel& m, const std::vector<int>& table, const std::vector<int>& ids) {
  int* cell = (int*)m.mesh_cell;
  float* cand = (float*)m.mesh_cand4;
  int used = 0;
  for (int h = 0; h < m.nmesh; h++) {
    const int* src = table.data() + 2 * (size_t)h * RG_NCELL;
    int* dst = cell + 2 * (size_t)h * RG_NCELL;
    const int first = src[0], n = src[2 * (RG_NCELL - 1)] + src[2 * (RG_NCELL - 1) + 1] - first;
    if (n < 0 || used + n > m.ncand_cap) { for (int c = 0; c < RG_NCELL; c++) { dst[2 * c] = 0; dst[2 * c + 1] = -1; } continue; }
    for (int c = 0; c < RG_NCELL; c++) { dst[2 * c] = src[2 * c] - first + used; dst[2 * c + 1] = src[2 * c + 1]; }
    const int adr = m.mesh_vertadr[h];
    for (int q = 0; q < n; q++) {
      const int k = ids[(size_t)first + q];
      const float* p = m.mesh_vert4 + 4 * ((size_t)adr + k);
      float* e = cand + 4 * ((size_t)used + q);
      e[0] = p[0]; e[1] = p[1]; e[2] = p[2];
      memcpy(e + 3, &k, 4);
    }
    used += n;
  }
}

/* after an edit of mesh_vert (mesh_vert4 re-padded first): rebuild the lists in the arena */
static inline void rg_host_refresh_cells(RgModel& m) {
  std::vector<int> table, ids;
  rg_host_cells(m.mesh_vert4, m.mesh_vertadr, m.mesh_vertnum, m.nmesh, table, ids);
  rg_host_store_cells(m, table, ids);
}

static inline bool rg_host_load(const void* blob, size_t len, RgHostModel& hm, std::string& err) {
  const char* p = (const char*)blob;
  if (len < 12 || memcmp(p, "RGMODEL1", 8)) { err = "bad model blob magic"; return false; }
  int ndim;
  memcpy(&ndim, p + 8, 4);
  RgModel& m = hm.view;
  memset(&m, 0, sizeof m);
  const int* dims = (const int*)(p + 12);
  int k = 0;
#define RG_DIM(n) if (k < ndim) m.n = dims[k]; k++;
#define RG_I(n, c)
#define RG_F(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  if (k != ndim) { err = "model blob built against a different rg_model_fields.h"; return false; }
#define RG_DIM(n) const int n = m.n; (void)n;
#define RG_I(n, c)
#define RG_F(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  /* pass 1: sizes */
  size_t src = 12 + 4 * (size_t)ndim, dst = 0;
  std::vector<size_t> srcoff, dstoff, counts;
  std::vector<int> isint;
  std::vector<std::string> names;
#define RG_DIM(n)
#define RG_I(n, c) src = (src + 7) & ~(size_t)7; srcoff.push_back(src); src += 4 * (size_t)(c); dst = rg_align16(dst); dstoff.push_back(dst); dst += 4 * (size_t)(c); counts.push_back((size_t)(c)); isint.push_back(1); names.push_back(#n);
#define RG_F(n, c) src = (src + 7) & ~(size_t)7; srcoff.push_back(src); src += 8 * (size_t)(c); dst = rg_align16(dst); dstoff.push_back(dst); dst += 4 * (size_t)(c); counts.push_back((size_t)(c)); isint.push_back(0); names.push_back(#n);
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  if (src > len) { err = "model blob truncated"; return false; }
  /* optional name tables behind the arrays (mjModel.*_name2id): RGNAMES1, ntypes, then type\0 count name\0 ... */
  hm.names.clear();
  {
    size_t q = (src + 7) & ~(size_t)7;
    if (q + 12 <= len && !memcmp(p + q, "RGNAMES1", 8)) {
      int nt;
      memcpy(&nt, p + q + 8, 4);
      q += 12;
      for (int t = 0; t < nt && q < len; t++) {
        const size_t tl = strnlen(p + q, len - q);
        if (q + tl + 5 > len) { err = "model blob: bad name section"; return false; }
        std::string typ(p + q, tl);
        q += tl + 1;
        int cnt;
        memcpy(&cnt, p + q, 4);
        q += 4;
        std::vector<std::string>& v = hm.names[typ];
        for (int i = 0; i < cnt; i++) {
          if (q >= len) { err = "model blob: bad name section"; return false; }
          const size_t nl = strnlen(p + q, len - q);
          v.emplace_back(p + q, nl);
          q += nl + 1;
        }
      }
    }
  }
  /* the hulls' support candidate lists, built from the blob's vertices rounded to fp32 (the values mesh_vert4 holds) before the
     layout, which sizes their room: what they take now plus a quarter for later mesh_vert edits (rg_host_store_cells) */
  std::vector<int> cell_table, cell_ids;
  {
    size_t iv = 0, ia = 0, in = 0;
    for (size_t i = 0; i < names.size(); i++) {
      if (names[i] == "mesh_vert") iv = i;
      else if (names[i] == "mesh_vertadr") ia = i;
      else if (names[i] == "mesh_vertnum") in = i;
    }
    const int* va = (const int*)(p + srcoff[ia]); const int* vn = (const int*)(p + srcoff[in]);
    for (int h = 0; h < m.nmesh; h++)
      if (va[h] < 0 || vn[h] < 0 || va[h] > m.nmeshvert - vn[h]) { err = "mesh_vertadr / mesh_vertnum out of range"; return false; }
    const double* sv = (const double*)(p + srcoff[iv]);
    std::vector<float> v4(4 * (size_t)m.nmeshvert, 0.0f);
    for (size_t k = 0; k < (size_t)m.nmeshvert; k++) for (int a = 0; a < 3; a++) v4[4 * k + a] = (float)sv[3 * k + a];
    rg_host_cells(v4.data(), va, vn, m.nmesh, cell_table, cell_ids);
  }
  const size_t ncand_cap = cell_ids.size() + cell_ids.size() / 4;
  if (ncand_cap > (size_t)0x7fffffff) { err = "hull support lists too large"; return false; }
  /* derived arrays appended to the small section would disturb the order; put them right after the blob fields
     but account for them in small_bytes by placing them BEFORE the first big field. */
  size_t first_big = names.size();
  for (size_t i = 0; i < names.size(); i++) if (names[i] == "mesh_vert") { first_big = i; break; }
  /* re-run the destination layout: small fields, derived, big fields */
  dst = 0;
  for (size_t i = 0; i < first_big; i++) { dst = rg_align16(dst); dstoff[i] = dst; dst += 4 * counts[i]; }
  dst = rg_align16(dst); const size_t off_subtree = dst; dst += 4 * (size_t)m.nbody;
  dst = rg_align16(dst); const size_t off_mrow = dst; dst += 12 * (size_t)m.nv;
  dst = rg_align16(dst); const size_t off_dlvl = dst; dst += 4 * (2 * (size_t)m.nv + 2);
  dst = rg_align16(dst); const size_t off_xlvl = dst; dst += 4 * (2 * (size_t)m.nv + 2);
  dst = rg_align16(dst); const size_t off_sidx = dst; dst += 4 * (2 * (size_t)m.nv);
  dst = rg_align16(dst); const size_t off_eqrow = dst; dst += 4 * (6 * (size_t)m.neq + 1);
  dst = rg_align16(dst); const size_t off_pairs = dst; if (m.ngeom <= 256) dst += 2 * (size_t)m.npair;
  dst = rg_align16(dst); const size_t off_mscale = dst; dst += 4 * (size_t)m.nmesh;
  dst = rg_align16(dst);
  hm.small_bytes = dst;
  for (size_t i = first_big; i < names.size(); i++) { dst = rg_align16(dst); dstoff[i] = dst; dst += 4 * counts[i]; }
  dst = rg_align16(dst); const size_t off_v4 = dst; dst += 16 * (size_t)m.nmeshvert;
  dst = rg_align16(dst); const size_t off_cell = dst; dst += 8 * (size_t)m.nmesh * RG_NCELL;
  const size_t off_cand = dst; dst += 16 * ncand_cap;   /* right behind the table (8 * RG_NCELL is a multiple of 16): rg_hull_cands */
  dst = rg_align16(dst);
  hm.arena.assign(dst, 0);
  char* base = hm.arena.data();
  for (size_t i = 0; i < names.size(); i++) {
    if (isint[i]) memcpy(base + dstoff[i], p + srcoff[i], 4 * counts[i]);
    else {
      const double* s = (const double*)(p + srcoff[i]);
      float* d = (float*)(base + dstoff[i]);
      for (size_t q = 0; q < counts[i]; q++) d[q] = (float)s[q];
    }
  }
  /* wire the view */
  size_t idx = 0;
  hm.offsets.clear();
#define RG_DIM(n)
#define RG_I(n, c) m.n = (const int*)(base + dstoff[idx]); hm.offsets.push_back(dstoff[idx]); idx++;
#define RG_F(n, c) m.n = (const float*)(base + dstoff[idx]); hm.offsets.push_back(dstoff[idx]); idx++;
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  /* rows of the equality constraints (weld: 3 position + 3 orientation rows, joint coupling: 1) -- of all of them: eq_active is
     read at run time, robogym switches welds off and on (robogym/envs/rearrange/common/base.py:452).  Constraint types the
     compiler can describe but this engine does not simulate are refused instead of stepping wrong physics */
  {
    int* eqrow = (int*)(base + off_eqrow);
    int n = 0;
    for (int e = 0; e < m.neq; e++) {
      if (m.eq_type[e] == RG_EQ_WELD) {
        const int b1 = m.eq_obj1id[e], b2 = m.eq_obj2id[e];
        int nd = 0;
        for (int w = 0; w < m.nmaskw; w++) nd += __builtin_popcount((unsigned)(m.body_dofmask[b1 * m.nmaskw + w] | m.body_dofmask[b2 * m.nmaskw + w]));
        if (nd > RG_TJ) { err = "weld constraint touches more than RG_TJ dofs: not supported by this engine"; return false; }
        for (int k = 0; k < 6; k++) eqrow[n++] = 8 * e + k;
      } else if (m.eq_type[e] == RG_EQ_JOINT) eqrow[n++] = 8 * e;
      else { err = "equality constraint type other than weld / joint: not supported by this engine"; return false; }
    }
    m.neqrow = n;
    m.eqrow = eqrow;
  }
  /* mujoco-py's second user controller (actuator_user[0] = 1: the cascaded-PI law of the UR16e's default joint calibration,
     robogym/assets/xmls/robot/ur16e/jointspec/calibrations/cascaded_pi/joint_actuations.xml:4) keeps 6 floats of state per actuator */
  m.pidw = 3;
  for (int i = 0; i < m.nu; i++)
    if (m.actuator_user0[i] == 1.0f && m.actuator_biastype[i] == RG_BIAS_USER) m.pidw = 6;
  int* subtree = (int*)(base + off_subtree);
  int* mrow = (int*)(base + off_mrow);
  for (int b = 0; b < m.nbody; b++) subtree[b] = 1;
  for (int b = m.nbody - 1; b > 0; b--) subtree[m.body_parentid[b]] += subtree[b];
  /* tree-sparse mass matrix (MuJoCo's qM layout): row i holds M(i,i), M(i,parent(i)), M(i,parent(parent(i))), ... */
  {
    int nM = 0;
    for (int d = 0; d < m.nv; d++) {
      const int par = m.dof_parentid[d];
      if (par >= d) { err = "dofs are not numbered parent-first"; return false; }
      mrow[3 * d + 2] = par >= 0 ? mrow[3 * par + 2] + 1 : 0;
      mrow[3 * d] = nM;
      mrow[3 * d + 1] = 1;
      nM += mrow[3 * d + 2] + 1;
    }
    for (int d = m.nv - 1; d >= 0; d--) if (m.dof_parentid[d] >= 0) mrow[3 * m.dof_parentid[d] + 1] += mrow[3 * d + 1];
    for (int d = 0; d < m.nv; d++) {   /* a dof's descendants must be the dofs right behind it */
      const int par = m.dof_parentid[d];
      if (par >= 0 && d >= par + mrow[3 * par + 1]) { err = "dof subtrees are not contiguous"; return false; }
    }
    m.nM = nM;
    /* dofs sorted by depth (stable): dlvl[0..nv) = dof ids, dlvl[nv + l] = start of level l; the tree-sparse
       factorisation walks these levels leaves-first, the back substitution roots-first */
    int* dlvl = (int*)(base + off_dlvl);
    int maxd = 0;
    for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] > maxd) maxd = mrow[3 * d + 2];
    int pos = 0;
    for (int l = 0; l <= maxd; l++) {
      dlvl[m.nv + l] = pos;
      for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] == l) dlvl[pos++] = d;
    }
    dlvl[m.nv + maxd + 1] = pos;
    m.ndoflevel = m.nv > 0 ? maxd + 1 : 0;
    m.dof_lvl = dlvl;
    /* Kinematic trees that no constraint row can ever touch (no friction loss, no limited joint, no tendon, no geom in a
       collision pair -- e.g. the collision-free target cube of the dactyl scenes, robogym/envs/dactyl/locked.py:89-96) stay
       out of the constraint solver: their acceleration is M^-1 qfrc_smooth exactly (tree-sparse solve), and the dense
       Hessian is built over the remaining `ns` dofs only.  sidx[d] = position of dof d in the solver's order (reversed:
       leaves first) or -1; sidx[nv + k] = dof at solver position k. */
    std::vector<char> tree_con(m.nbody, 0);
    auto mark_body = [&](int b) { tree_con[m.body_rootid[b]] = 1; };
    for (int d = 0; d < m.nv; d++) if (m.dof_frictionloss[d] > 0.0f) mark_body(m.dof_bodyid[d]);
    for (int j = 0; j < m.njnt; j++) if (m.jnt_limited[j]) mark_body(m.jnt_bodyid[j]);
    for (int k = 0; k < m.npair; k++) { mark_body(m.geom_bodyid[m.pair_geom1[k]]); mark_body(m.geom_bodyid[m.pair_geom2[k]]); }
    for (int t = 0; t < m.ntendon; t++)
      for (int w = m.tendon_adr[t]; w < m.tendon_adr[t] + m.tendon_num[t]; w++) {
        if (m.wrap_type[w] == RG_WRAP_JOINT) mark_body(m.jnt_bodyid[m.wrap_objid[w]]);
        else if (m.wrap_type[w] == RG_WRAP_SITE) mark_body(m.site_bodyid[m.wrap_objid[w]]);
        else if (m.wrap_type[w] == RG_WRAP_SPHERE || m.wrap_type[w] == RG_WRAP_CYLINDER) mark_body(m.geom_bodyid[m.wrap_objid[w]]);
      }
    for (int e = 0; e < m.neq; e++) {
      if (m.eq_type[e] == RG_EQ_WELD) { mark_body(m.eq_obj1id[e]); mark_body(m.eq_obj2id[e]); }
      else { mark_body(m.jnt_bodyid[m.eq_obj1id[e]]); if (m.eq_obj2id[e] >= 0) mark_body(m.jnt_bodyid[m.eq_obj2id[e]]); }
    }
    int* sidx = (int*)(base + off_sidx);
    int ns = 0;
    for (int d = m.nv - 1; d >= 0; d--) {
      if (tree_con[m.body_rootid[m.dof_bodyid[d]]]) { sidx[d] = ns; sidx[m.nv + ns] = d; ns++; }
      else sidx[d] = -1;
    }
    m.ns = ns;
    m.dof_sidx = sidx;
    int* xlvl = (int*)(base + off_xlvl);
    pos = 0;
    for (int l = 0; l <= maxd; l++) {
      xlvl[m.nv + l] = pos;
      for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] == l && sidx[d] < 0) xlvl[pos++] = d;
    }
    xlvl[m.nv + maxd + 1] = pos;
    m.dof_xlvl = xlvl;
  }
  /* depth-first numbering check: every body's parent must precede it and subtrees must be contiguous */
  for (int b = 1; b < m.nbody; b++) {
    const int par = m.body_parentid[b];
    if (par >= b || b >= par + subtree[par]) { err = "bodies are not numbered depth-first"; return false; }
  }
  m.body_subtreesize = subtree;
  m.dof_mrow = mrow;
  hm.offsets.push_back(off_subtree);
  hm.offsets.push_back(off_mrow);
  hm.offsets.push_back(off_dlvl);
  hm.offsets.push_back(off_xlvl);
  hm.offsets.push_back(off_sidx);
  hm.offsets.push_back(off_eqrow);
  /* uniform hull scale: the narrow phase's support point of a mesh is mesh_scale * (arg-max vertex of the unscaled hull) */
  float* mscale = (float*)(base + off_mscale);
  for (int k = 0; k < m.nmesh; k++) mscale[k] = 1.0f;
  m.mesh_scale = mscale;
  m.geom_mesh_scale = nullptr;   /* per-environment only (rg_batch_bind_param): never part of the arena */
  hm.offsets.push_back(off_mscale);
  /* hull vertices padded to float4: the narrow phase scans a hull's vertices with one 16-byte load each */
  float* v4 = (float*)(base + off_v4);
  m.mesh_vert4 = v4;
  rg_host_pad_verts(m);
  m.pair_packed = nullptr;
  if (m.ngeom <= 256) {
    unsigned short* pk = (unsigned short*)(base + off_pairs);
    for (int k = 0; k < m.npair; k++) pk[k] = (unsigned short)(m.pair_geom1[k] | (m.pair_geom2[k] << 8));
    m.pair_packed = pk;
  }
  hm.offsets.push_back(off_v4);
  /* the hulls' support candidate lists (global memory, behind the staged section: shared memory per CTA is unchanged) */
  m.mesh_cell = (const int*)(base + off_cell);
  m.mesh_cand4 = (const float*)(base + off_cand);
  m.ncand_cap = (int)ncand_cap;
  rg_host_store_cells(m, cell_table, cell_ids);
  hm.offsets.push_back(off_cell);
  hm.offsets.push_back(off_cand);
  /* fp32 conditioning: translate the world so the scene sits near the origin */
  double o[3] = {0, 0, 0};
  int cnt = 0;
  const double* bp = nullptr;
  {
    size_t i = 0;
    for (; i < names.size(); i++) if (names[i] == "body_pos") break;
    bp = (const double*)(p + srcoff[i]);
  }
  for (int b = 1; b < m.nbody; b++) if (m.body_parentid[b] == 0) { for (int a = 0; a < 3; a++) o[a] += bp[3 * b + a]; cnt++; }
  for (int a = 0; a < 3; a++) m.origin[a] = cnt ? (float)(o[a] / cnt) : 0.0f;
  float* body_pos = (float*)m.body_pos;
  for (int b = 1; b < m.nbody; b++)
    if (m.body_parentid[b] == 0) for (int a = 0; a < 3; a++) body_pos[3 * b + a] = (float)(bp[3 * b + a] - (double)m.origin[a]);
  /* the world body stays at the (shifted) origin, so geoms and sites attached to it directly are shifted themselves */
  {
    float* gp = (float*)m.geom_pos; float* sp = (float*)m.site_pos;
    for (int g = 0; g < m.ngeom; g++) if (m.geom_bodyid[g] == 0) for (int a = 0; a < 3; a++) gp[3 * g + a] -= m.origin[a];
    for (int k = 0; k < m.nsite; k++) if (m.site_bodyid[k] == 0) for (int a = 0; a < 3; a++) sp[3 * k + a] -= m.origin[a];
  }
  m.small_bytes = (int)hm.small_bytes;
  if (m.nv > 32 * 8 || m.nmaskw > 8) { err = "model too large for the warp-per-env engine"; return false; }
  return true;
}
