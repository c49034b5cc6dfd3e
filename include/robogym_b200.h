/* robogym_b200.h -- C ABI of the H100-native batched step engine (librobogym_b200.so).
 *
 * This is the drop-in boundary for robogym's physics path.  Each entry point names the
 * reference interface it replaces (paths relative to /root/reference/):
 *
 *   rg_model_load      <- mujoco_py.load_model_from_xml(xml) + MjSim(model, nsubsteps)
 *                         (robogym/mujoco/mujoco_xml.py:249-260).  The MJCF itself is compiled on
 *                         the host by robogym_b200.mjcf into the blob of include/rg_model_fields.h.
 *   rg_model_set_field <- in-place edits of sim.model.<array> by randomizers / modifiers
 *                         (robogym/wrappers/randomizations.py:84,139,188,302,589,643,713,745;
 *                          robogym/envs/dactyl/common/mujoco_modifiers.py:95-101).
 *   rg_batch_create/bind <- the mjData that MjSim owns (qpos, qvel, ctrl, userdata = PID state,
 *                         qacc_warmstart, xfrc_applied, time), here one row per environment in
 *                         caller-owned device tensors (torch) -- robogym reads/writes them through
 *                         SimulationInterface.qpos/qvel/set_qpos/... (simulation_interface.py:127-172)
 *                         and robot code writes sim.data.ctrl (robot/shadow_hand/mujoco/mujoco_shadow_hand.py:120-137).
 *   rg_step            <- SimulationInterface.step(): sim.step() [nsubsteps x mj_step, with the
 *                         mujoco-py PID callback enabled by cymj.set_pid_control,
 *                         simulation_interface.py:86-88] followed by sim.forward()
 *                         (robogym/mujoco/simulation_interface.py:176-189; robogym/robot_env.py:837).
 *   rg_forward         <- SimulationInterface.forward() (simulation_interface.py:203-207).
 *   rg_reset           <- SimulationInterface.reset() = mj_resetData (simulation_interface.py:191-195).
 *   rg_set_const       <- SimulationInterface.set_constants() = mj_setConst (simulation_interface.py:197-201).
 *
 * Conventions: every function returns 0 on success or a negative code and sets a thread-local
 * message readable with rg_last_error(); no exceptions or callbacks cross the ABI.  All device
 * work is stream-ordered and asynchronous on the stream the caller passes (a cudaStream_t as
 * void*).  The set-up calls (rg_model_load, rg_batch_create[_ex]) allocate engine-internal buffers and may synchronise with
 * the device; the stepping calls (rg_step, rg_step_subset, rg_forward, rg_reset, rg_model_set_field_async) never do, and
 * nothing ever allocates or frees the bound tensors.
 * State layout: row-major [nenv][n] float32 (int32 for ncon/warn); one environment per row.
 */
#ifndef ROBOGYM_B200_H
#define ROBOGYM_B200_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct rg_model rg_model;
typedef struct rg_batch rg_batch;

/* bindable per-environment arrays (rg_batch_bind) */
enum rg_field {
  RG_FIELD_QPOS = 0,       /* [nenv][nq]          in/out */
  RG_FIELD_QVEL = 1,       /* [nenv][nv]          in/out */
  RG_FIELD_CTRL = 2,       /* [nenv][nu]          in     */
  RG_FIELD_PID = 3,        /* [nenv][npid]        in/out : mujoco-py controller state in userdata; npid = rg_model_dim(m, "npid") = 3*nu
                              (PID: integral, last error, last derivative) or 6*nu when the model has a cascaded-PI actuator
                              (actuator user="1": + velocity-loop integral, smoothed set-point, step-taken flag) */
  RG_FIELD_WARMSTART = 4,  /* [nenv][nv]          in/out : qacc_warmstart */
  RG_FIELD_TIME = 5,       /* [nenv]              in/out (optional) */
  RG_FIELD_XFRC = 6,       /* [nenv][nbody*6]     in     (optional) : data.xfrc_applied */
  RG_FIELD_TIMESTEP = 7,   /* [nenv]              in     (optional) : per-env opt.timestep override */
  RG_FIELD_SITE_XPOS = 8,  /* [nenv][nsite*3]     out    (optional) */
  RG_FIELD_BODY_XPOS = 9,  /* [nenv][nbody*3]     out    (optional) */
  RG_FIELD_BODY_XQUAT = 10,/* [nenv][nbody*4]     out    (optional) */
  RG_FIELD_GEOM_XPOS = 11, /* [nenv][ngeom*3]     out    (optional) */
  RG_FIELD_ACT_FORCE = 12, /* [nenv][nu]          out    (optional) */
  RG_FIELD_QACC = 13,      /* [nenv][nv]          out    (optional) */
  RG_FIELD_CONTACT = 14,   /* [nenv][contact capacity][4] out (optional): geom1, geom2, dist, condim (rg_batch_capacity) */
  RG_FIELD_NCON = 15,      /* [nenv] int32        out    (optional) */
  RG_FIELD_WARN = 16,      /* [nenv] int32        in/out (optional): bit0 contact buffer full, bit1 row buffer full, bit2 bad state -> reset,
                              bit3 MPR, bit4 tendon Jacobian too dense, bit5 a contact touched more dofs than the batch allows (dropped),
                              bit6 rg_batch_update_pairs: pair list full (surplus dropped), bit7 rg_batch_update_pairs: a geom_dataid value
                              that is neither -1 nor a mesh id of a mesh geom (that geom is disabled) */
  RG_FIELD_DBG = 17,       /* [nenv][rg_batch_dbg_size] out (optional): stage dump used by the parity tests */
  RG_FIELD_BODY_XVEL = 18, /* [nenv][nbody*6]     out    (optional): angular, linear velocity of every body frame in world axes
                              = data.get_body_xvelr / get_body_xvelp (robogym/robot/ur16e/mujoco/joint_controlled_arm.py:32,
                              robogym/envs/rearrange/simulation/base.py:465-472) */
  RG_FIELD_MOCAP_POS = 19, /* [nenv][nmocap*3]    in     (optional): data.mocap_pos (world coordinates); unbound = the mocap bodies' model pose.
                              robogym moves the UR16e tool centre point by a mocap body welded to it
                              (robogym/robot/control/tcp/mocap_solver.py:41-46, robogym/assets/xmls/robot/ur16e/tcp_mocap.xml:2) */
  RG_FIELD_MOCAP_QUAT = 20,/* [nenv][nmocap*4]    in     (optional): data.mocap_quat */
  RG_FIELD_SENSORDATA = 21,/* [nenv][nsensordata] out    (optional): data.sensordata after the launch's last forward pass -- joint positions and
                              touch sensors (robogym/assets/xmls/robot/shadowhand/assets.xml:135-142); force / torque sensors
                              (robogym/assets/xmls/robot/ur16e/base.xml:48-49): wrench between the site's body and its parent
                              (cfrc_int of mj_rnePostConstraint), site frame */
  RG_NFIELDS = 22
};
#define RG_MAX_CONTACTS 32   /* DEFAULT contact capacity of a batch (rg_batch_create); rg_batch_create_ex picks another */
#define RG_MAX_PARAM_OVERRIDES 24

/* A mesh geom whose geom_dataid is -1 is a DISABLED part: an empty part slot of a model that holds a different object per
 * environment (robogym_b200.rearrange_mesh_scene).  It never reaches collision; batches of such a model stream
 * per-environment pair lists (rg_batch_update_pairs) from the start, derived from the shared geom_dataid row. */
int rg_model_load(const void* blob, size_t len, int device, rg_model** out);
void rg_model_destroy(rg_model* m);
/* value of a dimension of rg_model_fields.h (nq, nv, nu, nbody, ...) or -1 */
int rg_model_dim(const rg_model* m, const char* name);
/* id of a named object, as mjModel.body_name2id / joint_name2id / geom_name2id / site_name2id / actuator_name2id /
 * tendon_name2id / sensor_name2id do (robogym reaches them through sim.model, SURVEY App. B); objtype is "body", "joint",
 * "geom", "site", "actuator", "tendon", "mesh", "sensor" or "equality".  -1 when the name is unknown or the blob was
 * packed without its name tables. */
int rg_model_name2id(const rg_model* m, const char* objtype, const char* name);
const char* rg_model_id2name(const rg_model* m, const char* objtype, int id);   /* NULL when out of range; "" for an unnamed object */
/* overwrite a model array (host float64 / int32 values, `count` elements) and re-upload it.  The upload is ordered on
 * `stream` (set_field: the legacy default stream): launches queued before it keep the old values.  The host buffers may be
 * reused as soon as the call returns.  Do not call it from two threads for the same model at once.
 * Besides the arrays of include/rg_model_fields.h, `name` may be "mesh_scale": [nmesh] uniform scale of every convex hull
 * (1 at load; finite and > 0, else the call fails).  The narrow phase then uses the hull scaled by s about its frame origin --
 * support point s v*, with v* the support vertex of the unscaled hull -- and scales the hull's bounding box of the OBB cull
 * with it; geom_rbound (the broad phase) stays what the caller set, as in MuJoCo.  It is not part of the blob.  Editing
 * "mesh_vert" also rebuilds what the narrow phase derives from it (the padded vertex copy, the per-direction-cell candidate
 * lists of the support scan, the geom_aabb of mesh geoms); a hull whose rebuilt lists outgrow the room allocated at load falls
 * back to scanning all its vertices, with the same results.  Editing "mesh_vertadr" or "mesh_vertnum" switches every hull to
 * that whole-hull scan. */
int rg_model_set_field(rg_model* m, const char* name, const void* data, size_t count);
int rg_model_set_field_async(rg_model* m, const char* name, const void* data, size_t count, void* stream);
/* floats per environment of the RG_FIELD_DBG dump; bytes of shared memory per environment (one warp) */
int rg_dbg_size(const rg_model* m);
int rg_scratch_bytes(const rg_model* m);

int rg_batch_create(const rg_model* m, int nenv, rg_batch** out);
/* The same with explicit capacities per environment (0 = default): contacts kept (the reference compiles nconmax=100,
 * robogym/assets/xmls/robot/shadowhand/assets.xml:6), single-row constraint elements = friction-loss + limit rows
 * (reference njmax=500 counts these plus the contact rows, assets.xml:5), dofs one contact may touch (<= 32).  Larger
 * capacities mean more shared memory per environment, i.e. fewer environments resident per SM; overflow at run time sets
 * a warning bit (RG_FIELD_WARN) and drops the surplus, like mj_warning does. */
int rg_batch_create_ex(const rg_model* m, int nenv, int contact_capacity, int row_capacity, int dofs_per_contact, rg_batch** out);
int rg_batch_capacity(const rg_batch* b, int* contacts, int* rows, int* dofs_per_contact);
/* floats per environment of this batch's RG_FIELD_DBG dump; shared-memory bytes per environment */
int rg_batch_dbg_size(const rg_batch* b);
int rg_batch_scratch_bytes(const rg_batch* b);
void rg_batch_destroy(rg_batch* b);
int rg_batch_bind(rg_batch* b, int field, void* device_ptr);
/* Per-environment override of a float model array (domain randomisation, SURVEY 5.6: robogym's wrappers write
 * sim.model.geom_friction / dof_damping / actuator_gainprm / opt_gravity / ... per env and per episode):
 * device_ptr is a float32 [nenv][count(name)] tensor that replaces the shared array `name` for each environment.
 * Up to RG_MAX_PARAM_OVERRIDES arrays; device_ptr == NULL removes the override.  body_pos rows of bodies attached
 * to the world must be given relative to rg_model_origin().  "mesh_scale" ([nenv][nmesh], see rg_model_set_field) gives every
 * environment its own hull sizes; its values must be finite and > 0 (not checked on the device).
 * "geom_mesh_scale" ([nenv][ngeom], finite and > 0, not checked on the device) scales every mesh geom of an environment on
 * top of its hull's mesh_scale: the narrow phase uses the hull scaled by mesh_scale[dataid] * geom_mesh_scale[g], and the OBB
 * cull scales the geom's geom_aabb by the same product.  Two geoms that share a hull can so have different sizes.  It exists
 * per environment only (rg_model_set_field refuses it); while it is not bound every factor is 1.
 * "geom_dataid" is the one int array: an int32 [nenv][ngeom] row of mesh ids per environment (-1 = disabled part; every
 * other geom keeps -1), copied bit for bit into the environment's model view.  Binding it gives the batch per-environment
 * pair lists and marks them all stale: the next step (or rg_batch_update_pairs) derives them from the rows. */
int rg_batch_bind_param(rg_batch* b, const char* name, void* device_ptr);
/* Per-environment pair lists (reset time, not per step): one warp per environment whose mask byte is non-zero (mask == NULL:
 * all) compacts the static candidate pair list, in order, to the pairs whose two geoms are both enabled in that environment's
 * geom_dataid row, and clears its separating-axis cache.  The collision stage then streams that list instead of the static
 * one.  A full list sets warning bit 6 (surplus dropped), a bad geom_dataid value bit 7 (the geom counts as disabled).
 * Fails when geom_dataid is not bound per environment.  Asynchronous on `stream`. */
int rg_batch_update_pairs(rg_batch* b, const uint8_t* mask_device, void* stream);
/* The geom_dataid rows of the environments whose mask byte is non-zero (mask == NULL: all) were edited: their lists are stale.
 * The next rg_step / rg_step_subset / rg_forward first rederives every stale list (the same compaction, on its stream), so a
 * list never names a part that its row has disabled.  Call it after every write into the bound geom_dataid rows that is not
 * followed by rg_batch_update_pairs for the same environments (BatchedSim.set_param does).  Asynchronous on `stream`. */
int rg_batch_mark_pairs_stale(rg_batch* b, const uint8_t* mask_device, void* stream);
/* capacity of every environment's list (default, or 0: npair).  Set-up call (reallocates, synchronises); the lists are derived
 * again (from the per-environment rows before the next step, or at once from the shared row); overflow sets warning bit 6. */
int rg_batch_set_pair_capacity(rg_batch* b, int capacity);
/* capacity and the device array [nenv] of list lengths (0 / NULL when the batch streams the static list) */
int rg_batch_pair_info(const rg_batch* b, int* capacity, const int** counts_device);
int rg_model_origin(const rg_model* m, float origin[3]);
/* Work-ordered scheduling (default on; RG_BALANCE=0 in the environment turns it off at create): every launch records a
 * per-environment work estimate and the next launch groups environments of similar cost into the same CTA, which
 * shortens the waits at the per-stage CTA barriers.  Results are independent of the setting.  No reference
 * counterpart: mujoco-py steps one MjSim at a time (robogym/mujoco/simulation_interface.py:176). */
int rg_batch_set_balance(rg_batch* b, int on);
/* launch geometry actually used (for reporting): CTAs, warps per CTA, dynamic shared bytes */
int rg_batch_launch_info(const rg_batch* b, int* ctas, int* warps_per_cta, int* smem_bytes);
/* warps that step one environment: 1 = one warp per environment (warps_per_cta environments per CTA), 2..16 = one environment per
 * CTA of that many warps, which share the dense part of its constraint solve with bit-identical results.  Chosen at batch
 * creation for models whose scratch leaves a single environment per SM and whose solver is large; the environment variable
 * RG_WARPS_PER_ENV=1|2|4|8|16 forces it. */
int rg_batch_env_warps(const rg_batch* b, int* warps_per_env);

/* nsub x mj_step, then `final_forward` x mj_forward (0..4: SimulationInterface.step ends with one sim.forward(); the
 * observation path of RobotEnv runs more of them (robogym/robot_env.py:677, observation/mujoco.py:27) and mujoco-py's
 * PID state in userdata advances in each); derived outputs written once at the end */
int rg_step(rg_batch* b, int nsub, int final_forward, void* stream);
int rg_forward(rg_batch* b, void* stream);
/* the same for the environments whose mask byte (device memory, [nenv]) is non-zero; the others are untouched and cost
 * nothing (the launch covers only the selected environments).  What a Python loop over MjSim objects does when it
 * calls sim.forward()/sim.step() on some environments only (goal switches, resets). */
int rg_step_subset(rg_batch* b, const uint8_t* mask_device, int nsub, int final_forward, void* stream);
/* The reference's stabilize_objects (robogym/envs/rearrange/common/utils.py:76-93) for the environments whose mask byte is
 * non-zero (mask == NULL: all): nsub x mj_step with dof_damping[d] = `damping` for each of the `ndof` dof ids in the HOST array
 * `dofs` (1..64 ids in [0, nv); the same value for every selected environment, float32 on the device), then `final_forward` x
 * mj_forward (0..4) with each environment's own damping, as the reference's forward() after restoring it.  Neither the model
 * nor a per-environment dof_damping row changes.  The result is byte-identical to binding dof_damping per environment with
 * those entries set in the selected environments, rg_step_subset(mask, nsub, 0), restoring the rows and
 * rg_step_subset(mask, 0, final_forward); without the per-environment rows, which a batch would otherwise carry on every step.
 * Refused: an empty or out-of-range dof list, a negative or non-finite damping, and batches with rg_batch_env_warps > 1.
 * Two launches, asynchronous on `stream`. */
int rg_step_settle(rg_batch* b, const uint8_t* mask_device, const int* dofs, int ndof, double damping, int nsub, int final_forward, void* stream);
/* mj_setConst per environment (SimulationInterface.set_constants, robogym/mujoco/simulation_interface.py:197-201, which the
 * reference calls after its randomisers edited masses, inertias, armatures ...): recomputes, from each selected environment's
 * own parameter view at qpos0, the constants MuJoCo derives from the model -- dof_invweight0, body_invweight0,
 * tendon_invweight0, tendon_length0, body_subtreemass, opt_meaninertia -- and writes them into that environment's row of the
 * arrays bound with rg_batch_bind_param under those names (constants that are not bound per environment are not written:
 * the shared model is immutable while launches may be in flight; at least one must be bound).  One launch, asynchronous on
 * `stream`; mask as in rg_step_subset, NULL = every environment. */
int rg_set_const(rg_batch* b, const uint8_t* mask_device, void* stream);
/* mj_resetData for the environments whose mask byte is non-zero (mask == NULL: all) */
int rg_reset(rg_batch* b, const uint8_t* mask_device, void* stream);

/* Rotated bounding boxes of object bodies, the reference's `_get_bounding_box` (get_block_bounding_box /
 * get_mesh_bounding_box, robogym/envs/rearrange/common/utils.py:391-412): for every selected environment (mask as in
 * rg_step_subset, NULL = all) and each of the `nsel` (<= 64) body ids in the HOST array `bodies`, the body rotated by
 * quat[env][k] (device, fp64 [nenv][nsel][4], w x y z), out[env][k] = (center, half size) (device, fp64 [nenv][nsel][2][3]),
 * relative to the body origin in world-aligned axes.  The box covers what the narrow phase collides with: each environment's
 * bound geom_dataid / geom_pos / geom_quat / geom_size / mesh_scale / geom_mesh_scale rows where they are bound, the model's
 * arrays where they are not; mesh parts with geom_dataid -1 are skipped.  Only box and mesh geoms are boxed: a selected body
 * with any other geom is refused.  One warp per (environment, body); asynchronous on `stream`. */
int rg_batch_body_aabb(rg_batch* b, const int* bodies, int nsel, const double* quat, const uint8_t* mask_device, double* out, void* stream);
/* Reset-time placement of the rearrange objects, one warp per selected environment (mask as above; no model needed).
 * Device inputs: bbox [nenv][nobj][2][3] (rg_batch_body_aabb), active [nenv][nobj] (the active objects are placed in slot
 * order, as the reference places its num_objects; inactive slots are not written), area [nenv][6] (placement area offset,
 * full size), anchor [nenv][nobj][3] (goal_distance_ratio only: the object placements the goals are pulled toward).  Host:
 * table = table body pos, table geom half size.  mode 1 grid (place_objects_in_grid), 2 uniform
 * (place_objects_with_no_constraint), 3 goal_distance_ratio (place_targets_with_goal_distance_ratio), 4 grid then uniform
 * (RearrangeEnv._generate_object_placements); max_trials / max_per_object are the reference's max_placement_retry (also the
 * grid's trial count) / max_placement_retry_per_object.  Out: pos [nenv][nobj][3] body-origin positions (fp64) and status
 * [nenv]: the algorithm that succeeded (1, 2 or 3) or 0 = invalid (active slots zeroed; the reference raises
 * InvalidSimulationError and redraws the scene, here the caller redraws those environments).  Random numbers: Philox4x32-10
 * keyed by (seed, environment), counters (step, trial, 0, epoch) for the grid's shuffles and (proposal, 0, 1, epoch) for the
 * samplers' proposals (robogym_b200/csrc/rg_place.inl), so results do not depend on the mask.  Asynchronous on `stream`, on
 * the current device. */
int rg_place_objects(int nenv, int nobj, const double* bbox, const uint8_t* active, const double table[6], const double* area, int mode,
                     int max_trials, int max_per_object, double goal_distance_ratio, double goal_distance_min, const double* anchor,
                     uint32_t seed, uint32_t epoch, const uint8_t* mask_device, double* pos, int* status, void* stream);
/* The reference's other goal generators as edits of a placement, after rg_place_objects on the same stream, one thread per
 * selected environment (mask as above).  pos [nenv][nobj][3] (device, fp64) is edited in place on the active slots (uint8
 * [nenv][nobj], the reference's objects in slot order); inactive slots are not written.  kind:
 *   1 stack  (ObjectStackGoal._sample_next_goal_positions, goals/object_stack_goal.py): pos holds the bottom position in the
 *            first active slot; the active objects are taken in block order (0..n-1 with fixed_order, else numpy's shuffle)
 *            and object order[i] goes to the bottom position raised by i * object_size * 2;
 *   2 lift   (move_one_object_to_the_air, goals/pickandplace.py): one active object, randint(n), raised by
 *            uniform(min_height, max_height);
 *   3 train  (move_one_object_to_the_air_with_restrictions, goals/train_state.py): p = random(); nothing when
 *            p > pickup_proba + stacking_proba (or both are 0: no draw), a lift by the height times goal_distance_ratio when
 *            p < pickup_proba, otherwise (n >= 2) a tower of randint(2, n + 1) distinct objects on the first one's xy, member
 *            k + 1 raised by object_size * (k + 1) * 2.  The reference draws the members with the global np.random.choice;
 *            here they come from a partial Fisher-Yates draw on the environment's own stream;
 *   4 reach  (ObjectReachGoal._sample_next_goal_positions, goals/object_reach_goal.py): the one active object raised by
 *            target_height (an environment with another count is left alone).
 * object_size (stack, train), goal_distance_ratio (train) and target_height (reach) are fp64 [nenv] device arrays, NULL for
 * the kinds that do not read them.  Random numbers: Philox4x32-10 keyed by (seed, environment), draw d of the modifier at
 * counter (d, 0, 3, epoch) (robogym_b200/csrc/rg_place.inl lists d for every draw), so results do not depend on the mask.
 * Asynchronous on `stream`, on the current device. */
int rg_goal_modify(int nenv, int nobj, int kind, const uint8_t* active, const double* object_size, const double* goal_distance_ratio,
                   const double* target_height, double min_height, double max_height, double pickup_proba, double stacking_proba, int fixed_order,
                   uint32_t seed, uint32_t epoch, const uint8_t* mask_device, double* pos, void* stream);
/* The reference's layout goal generators, one warp per selected environment (mask as above), on the active slots (uint8
 * [nenv][nobj], the reference's objects in slot order; inactive slots are not written).  kind:
 *   1 domino   (DominoStateGoal, goals/dominos.py: _create_new_domino_position_and_rotation, _adjust_and_check_fit,
 *              _sample_next_goal_positions): up to max_retry arcs, each an offset random() * pi and a step
 *              random() * pi / 4 - pi / 8; domino i turned by i * step + (offset + step / 2) about z and laid along the arc's
 *              cumulative cos / sin steps of object_size * distance_mul; the first arc whose turned boxes fit in the placement
 *              area is moved to a uniform spot in it.  status 0 when none fits (positions zeroed, the last arc's rotations);
 *   2 attached (AttachedBlockStateGoal, goals/attached_block_state.py): exactly 8 active blocks (another count: status 0) in the
 *              reference's pattern of object_size cells, rows permuted, at a uniform origin; identity rotations;
 *   3 fixed    (ObjectFixedStateGoal, goals/object_state_fixed.py): rel [nenv][nobj][2], each object's placement relative to
 *              the placement area (values outside [0, 1] are taken as they are); identity rotations.
 * Attached and fixed are place_targets_with_fixed_position (common/utils.py): the proposal and _get_global_placement of
 * rg_place_objects, no collision or bounds check, status 1.  Device inputs: bbox [nenv][nobj][2][3] unrotated body boxes
 * (rg_batch_body_aabb with the identity), area [nenv][6], object_size / distance_mul fp64 [nenv] (NULL for the kinds that do
 * not read them); host: table as rg_place_objects.  Out (device): pos [nenv][nobj][3] fp64 body-origin positions, quat
 * [nenv][nobj][4] fp64 (w x y z), status int32 [nenv] (1 placed, 0 not); optional (NULL: not written, domino only): angle fp64
 * [nenv][nobj] the z angles, retry int32 [nenv] the arc that fitted (-1: none).  Random numbers: Philox4x32-10 keyed by (seed,
 * environment), draw d at counter (d, 0, 4, epoch) (robogym_b200/csrc/rg_place.inl lists d for every draw), so results do not
 * depend on the mask.  Asynchronous on `stream`, on the current device. */
int rg_layout_goals(int nenv, int nobj, int kind, const double* bbox, const uint8_t* active, const double table[6], const double* area,
                    const double* object_size, const double* distance_mul, const double* rel, int max_retry, uint32_t seed, uint32_t epoch,
                    const uint8_t* mask_device, double* pos, double* quat, int* status, double* angle, int* retry, void* stream);

/* Rearrange goal evaluation, once per env-step: the reference's ObjectStateGoal.relative_goal / goal_distance
 * (robogym/envs/rearrange/goals/object_state.py:492-599), RearrangeEnv._calculate_num_success /
 * _calculate_goal_distance_reward (envs/rearrange/common/base.py:824-848), RobotEnv._is_successful (robot_env.py:569-575)
 * and check_objects_off_table (envs/rearrange/simulation/base.py:805-832), one warp per selected environment.
 * Inputs (device unless noted):
 *   pos / quat: float32 object pose rows, read in place: slot k of environment e is pos[e * pos_stride + 3 * rows[k]] and
 *     quat[e * quat_stride + 4 * rows[k]] (w x y z).  A BatchedSim's body_xpos / body_xquat with rows = body ids, or
 *     [nenv][nobj] tensors with rows = 0..nobj-1.  rows is a HOST array of nobj (<= 64) ids.
 *   goal_pos / goal_quat: fp64 [nenv][nobj][3|4]; group: int32 [nenv][nobj], the object's group id (duplicates share one),
 *     -1 for an inactive (padded) slot; pos_offset / rot_weight: fp64 [nenv] (goal_pos_offset, goal_rot_weight).
 *   table: table body pos, table geom half size (as rg_place_objects); rot_dist_type 0 full, 1 mod90, 2 mod180;
 *   success_keys: bit 0 obj_pos, bit 1 obj_rot, bit 2 gripper_pos, bit 3 grasped in success_threshold (at least one), with
 *     their thresholds.
 *   Optional, at the end of the struct (NULL / 0: not read, and every other output is as without them), ObjectStackGoal's keys
 *   (goals/object_stack_goal.py): gripper_pos, float32, read in place at gripper_pos[e * gripper_stride] (a BatchedSim's
 *   site_xpos offset to the grip site's row, stride 3 * nsite); grasped, fp64 [nenv][nobj], the sum of the two pad contact
 *   flags per slot (is_object_grasped).  Bit 2 needs gripper_pos, bit 3 grasped.
 * Semantics: object angles are normalize_angles(mat2euler(quat2mat(q))) (get_object_rot), goal angles mat2euler(quat2mat(q))
 * (get_target_rot); inactive slots are zero on both sides.  Within every group of two or more active slots objects are
 * matched to goals greedily (the first flat argmin of the position distances, repeated); the others keep their own goal.
 * Padded slots count in num_success and goal_achieved, as in the reference.  `prev` ([nenv] fp64, in/out) holds the previous
 * evaluation's num_success; NaN marks "none since the goal reset" and gives reward 0.  Outputs per slot: obj_rot, rel_pos,
 * rel_rot ([nenv][nobj][3]), dist_pos, dist_rot ([nenv][nobj]), success, off_table (uint8 [nenv][nobj]); per environment:
 * num_success (count x reward_per_object), reward (num_success - prev), achieved, any_off (uint8).  pick (optional, int32
 * [nenv][nobj]): matched goal slot * 32 + index of the parallel quaternion taken (31: none).  rel_gripper [nenv][nobj][3] and
 * dist_gripper [nenv][nobj] (optional, with gripper_pos): obj_pos - gripper_pos and its norm, padded slots at -gripper_pos.  fp64 with explicitly rounded
 * operations in the reference's order (robogym_b200/csrc/rg_goal.inl).  Asynchronous on `stream`, on the current device. */
typedef struct rg_goal_in {
  int nenv, nobj;
  const float* pos; const float* quat;
  long long pos_stride, quat_stride;
  const int* rows;
  const double* goal_pos; const double* goal_quat;
  const int* group;
  const double* pos_offset; const double* rot_weight;
  double table[6];
  int rot_dist_type, success_keys;
  double pos_threshold, rot_threshold, reward_per_object;
  const float* gripper_pos; long long gripper_stride;
  const double* grasped;
  double gripper_threshold, grasped_threshold;
} rg_goal_in;
typedef struct rg_goal_out {
  double* obj_rot; double* rel_pos; double* rel_rot;
  double* dist_pos; double* dist_rot;
  uint8_t* success; uint8_t* off_table;
  double* num_success; double* reward;
  uint8_t* achieved; uint8_t* any_off;
  int* pick;
  double* rel_gripper; double* dist_gripper;
} rg_goal_out;
int rg_rearrange_goal(const rg_goal_in* in, const uint8_t* mask_device, double* prev, const rg_goal_out* out, void* stream);
/* Goal orientations at goal reset: randomize_quaternion_along_z (mode 1: quat_mul(z_quat, base)) or randomize_quaternion_block
 * (mode 2: quat_mul(z_quat, quat_mul(base, PARALLEL_QUATS[k]))), object_state.py:71-103, for the active slots (uint8
 * [nenv][nobj]) of the selected environments; base = the current target quaternions (fp64 [nenv][nobj][4]), out the same
 * shape (only those slots written; may alias base).  Random numbers: Philox4x32-10 keyed by (seed, environment); the i-th
 * active object reads counter (i, 0, 2, epoch): words x, y give its angle uniform(0, 2 pi), word z its face index in [0, 24)
 * (the constructions of rg_place_objects).  "full" (normal draws) is not provided. */
int rg_goal_orientations(int nenv, int nobj, const double* base_quat, const uint8_t* active, int mode, uint32_t seed, uint32_t epoch,
                         const uint8_t* mask_device, double* out, void* stream);

/* Rearrange observations, once per env-step after rg_rearrange_goal: the reference's RearrangeEnv._observe_simple with its
 * placement-area masks (envs/rearrange/common/base.py:311-421), the robot keys of MujocoObservation
 * (robot/ur16e/mujoco/joint_controlled_arm.py:22-85, robot/gripper/mujoco/mujoco_robotiq_gripper.py:12-35), the contact queries
 * get_gripper_table_contact / get_wrist_cam_collisions / get_object_gripper_contact and the penalty part of
 * _get_simulation_reward_with_done (common/base.py:768-795), one warp per selected environment.
 * Inputs (device unless noted):
 *   body_xpos / body_xquat / body_xvel / qpos / qvel / ctrl / sensordata / contact (float32) and ncon (int32): the main sim's
 *     rows, read in place; each environment's row is nbody * 3 | 4 | 6, nq, nv, nu, nsensordata, ncontact * 4 floats wide.
 *   obj_body / obj_qpos: HOST [nobj] (<= 64): body id and qpos address of the free joint of each object slot; tcp_body the
 *     robot0:gripper_tcp body; arm_qpos the arm joints' qpos addresses (<= 8), grip_qpos / grip_qvel the gripper joints'
 *     (<= 4), grip_act the gripper actuator; force_adr / torque_adr the sensor_adr of toolhead_force / toolhead_torque.
 *   geom_object: int32 [ngeom], the slot whose body owns the geom (-1: none); geom_flags: uint8 [ngeom], bit 0 a geom of a
 *     gripper body, bit 1 a robot geom (its name starts with the robot prefix); table_plane, wrist_sphere, pad[0..1]: the geoms
 *     table_collision_plane, robot0:wrist_cam_collision_sphere, robot0:left_contact_v, robot0:right_contact_v.
 *   goal_pos / goal_quat / rel_pos / rel_rot (fp64), achieved, off_table (uint8), group (int32, -1 inactive): the goal and the
 *     rg_rearrange_goal outputs of the same env-step; qpos_at_goal: float32 [nenv][nq], the qpos the goal was set on.
 *   bbox_size fp64 [nenv][nobj][3], colors fp64 [nenv][nobj][4], boundary fp64 [nenv][6] (min xyz, max xyz of the placement
 *     area); penalty: table_collision, wrist_collision, objects_off_table, safety_stop; mask_obs, mask_margin: the
 *     mask_obs_outside_placement_area keys (hard rule of check_objects_in_placement_area).
 * Outputs: fp64 [nenv][...] rows under the reference's key names; inactive slots are zero (placement masks 1).  The masked_*
 * and *_placement_mask outputs are written only with mask_obs (they may be NULL otherwise).  is_goal_achieved is int32,
 * safety_stop, gripper_table_contact, wrist_cam_contacts ([nenv][4]: table_collision_plane, robot, object, any) and sim_done
 * uint8.  fp64 with explicitly rounded operations in the reference's order (robogym_b200/csrc/rg_obs.inl).  Asynchronous on
 * `stream`, on the current device. */
typedef struct rg_obs_in {
  int nenv, nobj;
  const float* body_xpos; const float* body_xquat; const float* body_xvel;
  const float* qpos; const float* qvel; const float* ctrl; const float* sensordata; const float* contact;
  const int* ncon;
  int nbody, nq, nv, nu, nsensordata, ncontact, ngeom;
  const int* obj_body; const int* obj_qpos;
  int tcp_body;
  int narm, arm_qpos[8];
  int ngrip, grip_qpos[4], grip_qvel[4], grip_act;
  int force_adr, torque_adr;
  const int* geom_object; const uint8_t* geom_flags;
  int table_plane, wrist_sphere, pad[2];
  const double* goal_pos; const double* goal_quat; const double* rel_pos; const double* rel_rot;
  const uint8_t* achieved; const uint8_t* off_table; const int* group;
  const float* qpos_at_goal;
  const double* bbox_size; const double* colors; const double* boundary;
  double penalty[4];
  int mask_obs;
  double mask_margin;
} rg_obs_in;
typedef struct rg_obs_out {
  double* obj_pos; double* obj_rel_pos; double* obj_vel_pos; double* obj_rot; double* obj_vel_rot;   /* [nenv][nobj][3] */
  double* robot_joint_pos;                                      /* [nenv][narm] */
  double* gripper_pos; double* gripper_velp;                    /* [nenv][3] */
  double* gripper_controls;                                     /* [nenv][1] */
  double* gripper_qpos; double* gripper_vel;                    /* [nenv][ngrip] */
  double* qpos; double* qpos_goal;                              /* [nenv][nq] */
  double* goal_obj_pos; double* goal_obj_rot; double* rel_goal_obj_pos; double* rel_goal_obj_rot;   /* [nenv][nobj][3] */
  int* is_goal_achieved;                                        /* [nenv] */
  double* obj_gripper_contact;                                  /* [nenv][nobj][2] */
  double* obj_bbox_size; double* obj_colors;                    /* [nenv][nobj][3 | 4] */
  uint8_t* safety_stop;                                         /* [nenv] */
  double* tcp_force; double* tcp_torque;                        /* [nenv][3] */
  double* placement_mask; double* goal_placement_mask;          /* [nenv][nobj] */
  double* masked_obj_pos; double* masked_obj_rot; double* masked_obj_rel_pos; double* masked_obj_vel_pos; double* masked_obj_vel_rot;
  double* masked_obj_gripper_contact; double* masked_obj_bbox_size; double* masked_obj_colors;
  double* masked_goal_obj_pos; double* masked_goal_obj_rot; double* masked_rel_goal_obj_pos; double* masked_rel_goal_obj_rot;
  uint8_t* gripper_table_contact; uint8_t* wrist_cam_contacts;  /* [nenv], [nenv][4] */
  double* sim_reward; uint8_t* sim_done;                        /* [nenv] */
} rg_obs_out;
int rg_rearrange_obs(const rg_obs_in* in, const uint8_t* mask_device, const rg_obs_out* out, void* stream);

/* The dual-simulation arm controller's per-step arithmetic (robogym_b200.rearrange_arm.BatchedTcpArmController, TcpSolverMode.
 * MOCAP_IK): what runs between the solver and main simulations' launches, one thread per selected environment.
 * rg_arm_tables: the controller's index tables (host struct, passed by value to the kernel).  Ids are checked against the
 * dims of rg_arm_sim: qpos addresses < nq, actuators < nu, bodies in [1, nbody), mocap slots < nmocap.
 *   narm arm joints (<= 8): their qpos address in the main and solver models and the main actuator driving each;
 *   the gripper joint's qpos address and actuator in both; tcp_body: the solver's tool body;
 *   nweld (1..4) mocap welds of the solver model: mocap slot and welded body; the deltas move the first;
 *   ndof (1..3) tool rotations: euler_index (0..2, distinct), dof_joint (the arm joint whose range constrains it, -1: none),
 *   speed (rad per unit action, the mode's speed times max_position_change), lo_lim / hi_lim (the joint's range shrunk by the
 *   drift threshold); align_axis: -1, or the world axis (0..2) the commanded orientation is re-aligned with;
 *   max_position_change, grip_lo / grip_hi (the gripper's control range) and grip_half ((grip_hi - grip_lo) / 2).
 * All arithmetic is float32, each operation rounded as the float32 tensor path rounds it; constants are rounded to float32
 * where that path converts them. */
typedef struct rg_arm_tables {
  int narm;
  int arm_qpos_main[8]; int arm_qpos_solver[8]; int arm_act_main[8];
  int grip_qpos_main; int grip_qpos_solver; int grip_act_main; int grip_act_solver;
  int tcp_body;
  int nweld; int weld_mocap[4]; int weld_body[4];
  int ndof; int euler_index[3]; int dof_joint[3];
  int align_axis;
  double speed[3]; double lo_lim[8]; double hi_lim[8];
  double max_position_change; double grip_lo; double grip_hi; double grip_half;
} rg_arm_tables;
/* one simulation's rows as the controller reads and writes them (device, float32, row-major per environment): a BatchedSim's
 * bound qpos [nenv][nq], ctrl [nenv][nu], body_xpos [nenv][nbody][3], body_xquat [nenv][nbody][4], mocap_pos [nenv][nmocap][3],
 * mocap_quat [nenv][nmocap][4].  The main simulation's body and mocap rows are not read (NULL is fine). */
typedef struct rg_arm_sim {
  int nq; int nu; int nbody; int nmocap;
  float* qpos; float* ctrl; const float* body_xpos; const float* body_xquat; float* mocap_pos; float* mocap_quat;
} rg_arm_sim;
/* phase bits of rg_arm_phase; set bits run in this order, each on the environments whose mask byte is set:
 *   SYNC      solver arm qpos := main arm qpos (arm_reset_controller_error; free_dof_tcp_arm.py:215-226);
 *   GRIP      solver gripper qpos and ctrl := the main gripper's (on_observations_updated, joint_controlled_tcp_arm.py:129-140);
 *   SEAT      every weld's mocap body seated on its welded body (gym's reset_mocap2body_xpos);
 *   PRESOLVE  after the solver's forward: denormalize the action, constrain_quat_ctrl, euler2quat, the TCP quaternion product,
 *             align_axis, then SEAT and the deltas added to the first weld's mocap body (mocap_set_action);
 *   POSTSOLVE after the solver's substeps: main arm ctrl := solver arm qpos, main gripper ctrl := the gripper target. */
enum { RG_ARM_SYNC = 1, RG_ARM_GRIP = 2, RG_ARM_SEAT = 4, RG_ARM_PRESOLVE = 8, RG_ARM_POSTSOLVE = 16 };
/* `action` (device float32 [nenv][action_dim], action_dim = 3 + ndof + 1) is read by PRESOLVE and POSTSOLVE only (NULL
 * otherwise).  mask_device: uint8 [mask_len] with mask_len == nenv, or NULL (every environment).  Refuses out-of-range table
 * ids, a mask of another length and an action width that is not the mode's.  Asynchronous on `stream`. */
int rg_arm_phase(const rg_arm_tables* tables, int phases, int nenv, const rg_arm_sim* main_sim, const rg_arm_sim* solver_sim, const float* action,
                 int action_dim, const uint8_t* mask_device, int mask_len, void* stream);
/* _randomize_robot_initial_position's action_space.sample() for the masked environments: component d of environment e is
 * numpy's 53-bit double u from Philox4x32-10 keyed by (seed, e) at counter (d, 0, 5, epoch), words (x, y), mapped as gym
 * 0.15.3's Box.sample maps it for the bounded float32 box [-1, 1]: (float)(-1.0 + 2.0 * u) in fp64.  out: device float32
 * [nenv][action_dim] (1 <= action_dim <= 8); rows of unselected environments are not written. */
int rg_arm_sample_actions(int nenv, int action_dim, uint32_t seed, uint32_t epoch, const uint8_t* mask_device, int mask_len, float* out, void* stream);

/* The object groups of a rearrange reset, one thread per selected environment: RearrangeEnv._sample_random_object_groups
 * (with sample_group_counts), _sample_group_attributes and _sample_default_quaternions (robogym/envs/rearrange/common/
 * base.py:513-620, common/utils.py:47-73) and their overrides in blocks.py, blocks_duplicate.py, the dedupe environments,
 * holdout.py, common/mesh.py and ycb.py.  Environment e's objects are its first active[e] slots; its groups take them in
 * order.  Every input is HOST memory (the call copies what the kernel reads).
 *   active: int32 [nenv], each in [0, nobj] (nobj <= 64);
 *   group_mode: 1 random (sample_group_counts with lam ~ uniform(lam_low, lam_high)), 2 dedupe (every object its own group,
 *     no draws), 3 single (blocks_duplicate: the random counts drawn, then one group of all), 4 fixed (fixed_counts int32
 *     [nenv][nobj]: each row positive counts summing to the active count, then zeros, as holdout's task_object_configs);
 *   per group: a material index in [0, n_materials) (n_materials >= 1: choice(material_names)); a colour, color_mode 1 random
 *     (random((g, 4)), alpha 1), 2 palette (permutation(palette)[:g]; palette fp64 [n_palette][4], n_palette in
 *     [largest active count, 256]) or 3 grey ((0.5, 0.5, 0.5, 1), no draws); a size scale exp(uniform(-scale_low,
 *     scale_high)); with mesh_mode 1 (with replacement) or 2 (without: permutation(n_candidates)[:g], n_candidates <= 256 and
 *     no environment with more possible groups than candidates) a candidate index in [0, n_candidates), n_candidates >= 1;
 *   per object: the yaw uniform(0, 2 pi) and its quaternion about z (w, x, y, z).
 * Random numbers: Philox4x32-10 keyed by (seed, e); the groups and attributes take counter (d, 0, 6, epoch) for their d-th
 * draw in the reference's call order, object j's yaw counter (j, 1, 6, epoch) (robogym_b200/csrc/rg_groups.inl lists the
 * order).  Outputs (device, [nenv][nobj] row-major; rgba and quat [nenv][nobj][4]): group (the group id, 0-based in slot
 * order, the `group` of rg_goal_in), count (the group's size), material, rgba, scale, mesh (-1 without mesh draws), yaw,
 * quat; ngroups [nenv].  Slots past an environment's objects get -1 (group, material, mesh) or 0 (the rest).  Unselected
 * environments (mask_device: uint8 [mask_len], mask_len == nenv, or NULL) are not written.  Refuses more than 64 objects,
 * active counts outside [0, nobj], a non-finite lam or scale range, n_materials < 1, a palette with fewer rows than the
 * largest active count, mesh draws without candidates, more groups than candidates without replacement and a mask of
 * another length.  Asynchronous on `stream`; the host inputs are staged before the call returns, so the caller may reuse them. */
typedef struct rg_groups_in {
  int nenv; int nobj;
  const int* active;
  int group_mode; double lam_low; double lam_high; const int* fixed_counts;
  int n_materials;
  int color_mode; const double* palette; int n_palette;
  double scale_low; double scale_high;
  int mesh_mode; int n_candidates;
  uint32_t seed; uint32_t epoch;
} rg_groups_in;
typedef struct rg_groups_out {
  int* group; int* count; int* material; double* rgba; double* scale; int* mesh; double* yaw; double* quat; int* ngroups;
} rg_groups_out;
int rg_object_groups(const rg_groups_in* in, const uint8_t* mask_device, int mask_len, const rg_groups_out* out, void* stream);

const char* rg_last_error(void);

#ifdef __cplusplus
}
#endif
#endif
