/* rg_derived_fields.h -- the arrays the engine derives at load (rg_host_load) and adds to the arena of the blob's arrays
 * (include/rg_model_fields.h), as an X-macro list of (name, element type, count in elements over the dims and ncand_cap).
 *   RG_DS(n, T, c)        staged: inside the leading small_bytes that each CTA copies into shared memory (RgModelDev: an offset)
 *   RG_DSO(n, T, c, when) staged when `when` holds, else no room and a nullptr in the view
 *   RG_DE(n, T, c)        per environment only (rg_batch_bind_param): never in the arena, nullptr in the model's view
 *   RG_DG(n, T, c)        global: behind the blob's big arrays (RgModelDev: a pointer)
 *   RG_DGH(n, T, c)       global, and only RgModel holds it (defaults to RG_DG)
 * List order is arena order.  Define the macros you need, then include: the others expand to nothing, and all are #undef'd.
 */

#ifndef RG_DGH
#define RG_DGH(n, T, c) RG_DG(n, T, c)
#endif
#ifndef RG_DS
#define RG_DS(n, T, c)
#endif
#ifndef RG_DSO
#define RG_DSO(n, T, c, when)
#endif
#ifndef RG_DE
#define RG_DE(n, T, c)
#endif
#ifndef RG_DG
#define RG_DG(n, T, c)
#endif

RG_DS(body_subtreesize, int, nbody)   /* bodies are numbered depth-first: subtree(b) = [b, b+size) */
RG_DS(dof_mrow, int, 3 * nv)          /* [nv][3]: start of dof i's row in the tree-sparse mass matrix, dofs in its subtree, its depth */
RG_DS(dof_lvl, int, 2 * nv + 2)       /* dof ids sorted by depth, then the start of every depth level (ndoflevel + 1 entries) */
RG_DS(dof_xlvl, int, 2 * nv + 2)      /* the same lists restricted to the dofs that stay out of the constraint solver */
RG_DS(dof_sidx, int, 2 * nv)          /* solver position of every dof (or -1), then the dof at every solver position */
RG_DS(eqrow, int, 6 * neq + 1)        /* [neqrow]: equality id * 8 + row (weld: 6 rows, joint coupling: 1); row k is "virtual tendon" ntendon + k */
/* geom1 | geom2 << 8 of every pair when ngeom <= 256; a view without it streams an environment's own list instead (rg_pair) */
RG_DSO(pair_packed, unsigned short, npair, ngeom <= 256)
RG_DS(mesh_scale, float, nmesh)       /* uniform scale of every hull (1 at load; model-wide or per-environment parameter) */
RG_DE(geom_mesh_scale, float, ngeom)  /* uniform scale of every mesh geom on top of its hull's mesh_scale; unbound: 1 everywhere */
RG_DG(mesh_vert4, float, 4 * nmeshvert)          /* hull vertices padded to 16 bytes (one vector load each) */
RG_DG(mesh_cell, int, 2 * nmesh * RG_NCELL)      /* (first entry in mesh_cand4, count) of every direction cell's support
                                                    candidates; count -1: scan the whole hull (rg_host_store_cells) */
/* candidate vertices x, y, z and the vertex id's int bits, ascending ids per cell; right behind mesh_cell in the arena, where the
   device finds them (rg_hull_cands) */
RG_DGH(mesh_cand4, float, 4 * ncand_cap)

#undef RG_DS
#undef RG_DSO
#undef RG_DE
#undef RG_DG
#undef RG_DGH
