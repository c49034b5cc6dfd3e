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
#include <type_traits>
#include <vector>

#include "rg_defs.h"

struct RgHostModel {
  std::vector<char> arena;
  RgModel view;                 /* pointers into `arena` (host) */
  size_t small_bytes = 0;
  std::map<std::string, std::vector<std::string>> names;   /* objtype -> names ("" = unnamed), from the blob's RGNAMES1 section */
};

/* the blob's arrays where they lie in the blob: int32 and fp64 */
struct RgBlob {
#define RG_DIM(n)
#define RG_I(n, c) const int* n;
#define RG_F(n, c) const double* n;
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
};

static inline size_t rg_align16(size_t x) { return (x + 15) & ~(size_t)15; }

/* A model array by name: one of the blob's (include/rg_model_fields.h) or one the engine derives (rg_derived_fields.h), with its
   element count.  The pointer is the view's: nullptr for an array the view does not hold (a per-environment one, or
   pair_packed when the pairs are not packed). */
struct RgHostField { void* p; size_t count; bool isint, derived; };
static inline bool rg_host_field(const RgModel& m, const char* name, RgHostField& f) {
#define RG_DIM(n) const int n = m.n; (void)n;
#define RG_I(n, c)
#define RG_F(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  const int ncand_cap = m.ncand_cap; (void)ncand_cap;
#define RG_FIELD(n, T, c, d) if (!strcmp(name, #n)) { f = {(void*)m.n, (size_t)(c), std::is_integral<T>::value, d}; return true; }
#define RG_DIM(n)
#define RG_I(n, c) RG_FIELD(n, int, c, false)
#define RG_F(n, c) RG_FIELD(n, float, c, false)
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#define RG_DS(n, T, c) RG_FIELD(n, T, c, true)
#define RG_DSO(n, T, c, when) RG_FIELD(n, T, (when) ? (c) : 0, true)
#define RG_DE(n, T, c) RG_FIELD(n, T, c, true)
#define RG_DG(n, T, c) RG_FIELD(n, T, c, true)
#include "rg_derived_fields.h"
#undef RG_FIELD
  return false;
}

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
  /* where the blob's arrays lie: each on an 8-byte boundary */
  RgBlob src;
  size_t at = 12 + 4 * (size_t)ndim;
#define RG_DIM(n)
#define RG_I(n, c) at = (at + 7) & ~(size_t)7; src.n = (const int*)(p + at); at += 4 * (size_t)(c);
#define RG_F(n, c) at = (at + 7) & ~(size_t)7; src.n = (const double*)(p + at); at += 8 * (size_t)(c);
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
  if (at > len) { err = "model blob truncated"; return false; }
  /* optional name tables behind the arrays (mjModel.*_name2id): RGNAMES1, ntypes, then type\0 count name\0 ... */
  hm.names.clear();
  {
    size_t q = (at + 7) & ~(size_t)7;
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
    const int* va = src.mesh_vertadr; const int* vn = src.mesh_vertnum;
    for (int h = 0; h < m.nmesh; h++)
      if (va[h] < 0 || vn[h] < 0 || va[h] > m.nmeshvert - vn[h]) { err = "mesh_vertadr / mesh_vertnum out of range"; return false; }
    std::vector<float> v4(4 * (size_t)m.nmeshvert, 0.0f);
    for (size_t k = 0; k < (size_t)m.nmeshvert; k++) for (int a = 0; a < 3; a++) v4[4 * k + a] = (float)src.mesh_vert[3 * k + a];
    rg_host_cells(v4.data(), va, vn, m.nmesh, cell_table, cell_ids);
  }
  const size_t ncand_cap = cell_ids.size() + cell_ids.size() / 4;
  if (ncand_cap > (size_t)0x7fffffff) { err = "hull support lists too large"; return false; }
  /* The arena, every array 16-byte aligned: the blob's small arrays and the derived staged ones (the leading small_bytes, which
     every CTA stages into shared memory), then the blob's big arrays and the derived global ones.  Walked once to size it, then
     once more to point the view's arrays into it and copy the blob's arrays there (fp64 -> fp32). */
  static_assert(8 * RG_NCELL % 16 == 0, "mesh_cand4 must start right behind mesh_cell (rg_hull_cands)");
  char* base = nullptr;
  size_t dst = 0;
  auto put = [&](auto& ptr, size_t count, bool present) {
    dst = rg_align16(dst);
    if (base) ptr = present ? (std::remove_reference_t<decltype(ptr)>)(base + dst) : nullptr;
    if (present) dst += sizeof(*ptr) * count;
  };
  auto put_i = [&](const int*& ptr, const int* s, size_t count) { put(ptr, count, true); if (base) memcpy((void*)ptr, s, 4 * count); };
  auto put_f = [&](const float*& ptr, const double* s, size_t count) { put(ptr, count, true); if (base) for (size_t q = 0; q < count; q++) ((float*)ptr)[q] = (float)s[q]; };
  auto layout = [&]() {
    dst = 0;
#define RG_DIM(n)
#define RG_I(n, c) put_i(m.n, src.n, (size_t)(c));
#define RG_F(n, c) put_f(m.n, src.n, (size_t)(c));
#define RG_IB(n, c)
#define RG_FB(n, c)
#include "../../include/rg_model_fields.h"
#undef RG_IB
#undef RG_FB
#define RG_DS(n, T, c) put(m.n, (size_t)(c), true);
#define RG_DSO(n, T, c, when) put(m.n, (size_t)(c), (when));
#include "rg_derived_fields.h"
    hm.small_bytes = dst = rg_align16(dst);
#undef RG_I
#undef RG_F
#define RG_I(n, c)
#define RG_F(n, c)
#define RG_IB(n, c) put_i(m.n, src.n, (size_t)(c));
#define RG_FB(n, c) put_f(m.n, src.n, (size_t)(c));
#include "../../include/rg_model_fields.h"
#undef RG_DIM
#undef RG_I
#undef RG_F
#undef RG_IB
#undef RG_FB
#define RG_DG(n, T, c) put(m.n, (size_t)(c), true);
#include "rg_derived_fields.h"
    dst = rg_align16(dst);
  };
  layout();
  hm.arena.assign(dst, 0);
  base = hm.arena.data();
  layout();
  /* rows of the equality constraints (weld: 3 position + 3 orientation rows, joint coupling: 1) -- of all of them: eq_active is
     read at run time, robogym switches welds off and on (robogym/envs/rearrange/common/base.py:452).  Constraint types the
     compiler can describe but this engine does not simulate are refused instead of stepping wrong physics */
  {
    int* eqrow = (int*)m.eqrow;
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
  }
  /* mujoco-py's second user controller (actuator_user[0] = 1: the cascaded-PI law of the UR16e's default joint calibration,
     robogym/assets/xmls/robot/ur16e/jointspec/calibrations/cascaded_pi/joint_actuations.xml:4) keeps 6 floats of state per actuator */
  m.pidw = 3;
  for (int i = 0; i < m.nu; i++)
    if (m.actuator_user0[i] == 1.0f && m.actuator_biastype[i] == RG_BIAS_USER) m.pidw = 6;
  int* subtree = (int*)m.body_subtreesize;
  int* mrow = (int*)m.dof_mrow;
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
    int* dlvl = (int*)m.dof_lvl;
    int maxd = 0;
    for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] > maxd) maxd = mrow[3 * d + 2];
    int pos = 0;
    for (int l = 0; l <= maxd; l++) {
      dlvl[m.nv + l] = pos;
      for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] == l) dlvl[pos++] = d;
    }
    dlvl[m.nv + maxd + 1] = pos;
    m.ndoflevel = m.nv > 0 ? maxd + 1 : 0;
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
    int* sidx = (int*)m.dof_sidx;
    int ns = 0;
    for (int d = m.nv - 1; d >= 0; d--) {
      if (tree_con[m.body_rootid[m.dof_bodyid[d]]]) { sidx[d] = ns; sidx[m.nv + ns] = d; ns++; }
      else sidx[d] = -1;
    }
    m.ns = ns;
    int* xlvl = (int*)m.dof_xlvl;
    pos = 0;
    for (int l = 0; l <= maxd; l++) {
      xlvl[m.nv + l] = pos;
      for (int d = 0; d < m.nv; d++) if (mrow[3 * d + 2] == l && sidx[d] < 0) xlvl[pos++] = d;
    }
    xlvl[m.nv + maxd + 1] = pos;
  }
  /* depth-first numbering check: every body's parent must precede it and subtrees must be contiguous */
  for (int b = 1; b < m.nbody; b++) {
    const int par = m.body_parentid[b];
    if (par >= b || b >= par + subtree[par]) { err = "bodies are not numbered depth-first"; return false; }
  }
  /* uniform hull scale: the narrow phase's support point of a mesh is mesh_scale * (arg-max vertex of the unscaled hull) */
  for (int k = 0; k < m.nmesh; k++) ((float*)m.mesh_scale)[k] = 1.0f;
  /* hull vertices padded to float4: the narrow phase scans a hull's vertices with one 16-byte load each */
  rg_host_pad_verts(m);
  if (m.pair_packed) {   /* ngeom <= 256 */
    unsigned short* pk = (unsigned short*)m.pair_packed;
    for (int k = 0; k < m.npair; k++) pk[k] = (unsigned short)(m.pair_geom1[k] | (m.pair_geom2[k] << 8));
  }
  /* the hulls' support candidate lists (global memory, behind the staged section: shared memory per CTA is unchanged) */
  m.ncand_cap = (int)ncand_cap;
  rg_host_store_cells(m, cell_table, cell_ids);
  /* fp32 conditioning: translate the world so the scene sits near the origin */
  double o[3] = {0, 0, 0};
  int cnt = 0;
  const double* bp = src.body_pos;
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
