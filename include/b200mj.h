/* b200mj.h — C ABI of the H100-native batched forward-dynamics engine (libb200mj.so).
 *
 * The reference has no C-ABI plugin seam of its own: dm_control reaches the engine through pybind11
 * calls on `mujoco.MjModel/MjData` handles. Each entry point below names the reference call it stands
 * in for (paths relative to the dm_control package of the reference):
 *
 *   b200mj_model_create   <- mujoco.MjModel.from_xml_string result          mujoco/wrapper/core.py:179-182
 *                            (the MJCF->tables compile itself is host Python, dm_control_b200/mjcf_compile.py)
 *   b200mj_step           <- mujoco.mj_step2 / mj_step / mj_step1 sequence  mujoco/engine.py:147-176
 *   b200mj_forward        <- mujoco.mj_forward (+ actuation-disabled form)  mujoco/engine.py:306-343
 *   b200mj_step_host      <- the same step as seen by rl/control.py:99-127 with HOST action/observation
 *                            buffers (host<->device copies inside the call)
 *   b200mj_reset          <- Physics.reset(keyframe_id): mj_resetData[Keyframe] + mj_forward   mujoco/engine.py:306-327
 *   b200mj_forward_masked <- Physics.after_reset() for the environments being reset           mujoco/engine.py:329-333
 *   b200mj_contact_force  <- mujoco.mj_contactForce                                           mujoco/wrapper/core.py:546-551
 *   b200mj_subtree_vel    <- mujoco.mj_subtreeVel (after a position/velocity stage)           locomotion/walkers/legacy_base.py:179-186
 *   b200mj_model_set_variable_geoms <- the per-episode recompile of the composer arenas       composer/environment.py:378-383
 *   b200mj_model_set_env_fields <- per-Physics model writes, e.g. PhysicsVariator.apply_variations   composer/variation/__init__.py:90-136
 *   b200mj_render         <- Physics.render / Camera.render (rgb, depth, segmentation)         mujoco/engine.py:178-233,840-946
 *                            (a ray caster over the model's primitives: hand-off images, not MuJoCo's OpenGL pixels)
 *   b200mj_workspace_bytes / b200mj_envs_per_block / b200mj_describe / b200mj_launch_count : instrumentation
 *
 * Threading: a b200mj_model handle owns streams, events and the handover buffers of its last call — like a reference
 * Physics instance it must be driven by one host thread at a time (the reference's contract: one Physics per thread).
 *
 * Conventions: all `*_dev` pointers are device pointers on the current CUDA device; batched arrays are
 * row-major [batch, n] (one environment's values contiguous: one warp owns one environment and reads its
 * row with coalesced loads). Any output pointer may be NULL (that field is then not materialised).
 * Return value: 0 ok; negative = configuration / launch error (see b200mj_error_string). Physics
 * warnings (mjtWarning) are per-environment counters in `warning` [batch, 8].
 * All calls are stream-ordered on `stream` (a cudaStream_t passed as void*), no host synchronisation
 * except in b200mj_step_host.
 */
#ifndef B200MJ_H_
#define B200MJ_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200mj_model b200mj_model;

/* Batched mjData slice crossing the ABI. State is read AND written; outputs are written. */
typedef struct b200mj_io {
  /* ---- physics state (in/out), [batch, n] ---- */
  double* qpos;            /* nq  */
  double* qvel;            /* nv  */
  double* act;             /* na  (may be NULL when na == 0) */
  double* qacc_warmstart;  /* nv  */
  double* time;            /* 1   */
  /* ---- inputs ---- */
  const double* ctrl;          /* nu  */
  const double* qfrc_applied;  /* nv, may be NULL */
  const double* xfrc_applied;  /* nbody*6 (force, torque), may be NULL */
  /* per-environment geoms (b200mj_model_set_variable_geoms names which; NULL = every environment uses the model's):
   * the composer corridor arenas re-draw wall / platform boxes every episode (locomotion/arenas/corridors.py:394-440)
   * and the reference recompiles its model for that (composer/environment.py:378-383); here the topology is shared and
   * only these two tables differ between environments */
  const double* var_geom_pos;   /* nvargeom*3 */
  const double* var_geom_size;  /* nvargeom*3 */
  /* ---- position / velocity stage outputs (consistent with the NEW state) ---- */
  double* xpos;            /* nbody*3 */
  double* xquat;           /* nbody*4 */
  double* xmat;            /* nbody*9 */
  double* xipos;           /* nbody*3 */
  double* geom_xpos;       /* ngeom*3 */
  double* geom_xmat;       /* ngeom*9 */
  double* site_xpos;       /* nsite*3 */
  double* site_xmat;       /* nsite*9 */
  double* subtree_com;     /* nbody*3 */
  double* subtree_linvel;  /* nbody*3 (mj_subtreeVel) */
  double* cvel;            /* nbody*6 */
  double* sensordata;      /* nsensordata (pos/vel sensors from the new state, acc sensors from the last step2) */
  double* qM;              /* nv*nv dense joint-space inertia */
  double* qfrc_bias;       /* nv */
  double* qfrc_passive;    /* nv */
  /* ---- acceleration stage outputs (from the last step2 / forward) ---- */
  double* qacc;            /* nv */
  double* qfrc_actuator;   /* nv */
  double* actuator_force;  /* nu */
  double* qfrc_constraint; /* nv */
  double* efc_force;       /* njmax */
  /* ---- contacts of the new state ---- */
  int32_t* ncon;           /* 1 */
  int32_t* contact_geom;   /* nconmax*2 (geom1, geom2) */
  int32_t* contact_efc_address; /* nconmax */
  double* contact_dist;    /* nconmax */
  double* contact_pos;     /* nconmax*3 */
  double* contact_frame;   /* nconmax*9 */
  int32_t* nefc;           /* 1 */
  int32_t* solver_niter;   /* 1 */
  /* ---- diagnostics ---- */
  int32_t* warning;        /* 8 counters per env, accumulated */
} b200mj_io;

enum {
  B200MJ_STEP_LEGACY = 1,      /* reference legacy ordering: step2,(step1+step2)*(n-1),step1 (engine.py:147-162) */
  B200MJ_STEP_FULL_FINAL = 2,  /* final position stage also runs collision + constraint assembly (ncon, contacts) */
  B200MJ_STEP_SENSORS = 4,     /* evaluate sensors */
  B200MJ_STEP_REUSE_POS = 8    /* the caller has not touched the state since the previous b200mj_step on this io: start from
                                  the position stage its trailing mj_step1 left behind, as the reference's legacy ordering
                                  does (engine.py:147-162: step2 first). Ignored unless that previous call ran with
                                  B200MJ_STEP_LEGACY | B200MJ_STEP_FULL_FINAL on the same (io->qpos, batch). */
};

/* Upload a compiled model blob (layout: b200mj_model_fields.h). */
int b200mj_model_create(const int32_t* idata, int ni, const double* rdata, int nr, b200mj_model** out);
void b200mj_model_destroy(b200mj_model* m);
/* Change opt.disableflags of an uploaded model (model.disable() context, wrapper/core.py:389-426). */
int b200mj_model_set_disableflags(b200mj_model* m, int disableflags);
/* Change per-env capacities (re-sizes the shared-memory workspace). */
int b200mj_model_set_capacity(b200mj_model* m, int nconmax, int njmax);

/* nstep physics steps for `batch` environments. flags: B200MJ_STEP_*. */
int b200mj_step(const b200mj_model* m, const b200mj_io* io, int batch, int nstep, int flags, void* stream);
/* mj_forward on the current state (no integration). extra_disableflags is OR-ed into opt.disableflags
 * (the reference's reset()/after_reset() pass mjDSBL_ACTUATION, engine.py:325-333). */
int b200mj_forward(const b200mj_model* m, const b200mj_io* io, int batch, int extra_disableflags, int flags,
                   void* stream);

/* Rendering hand-off (dm_control_b200/render.py). One camera per environment looks at that environment's geoms and
 * sites, whose world frames are outputs of b200mj_step / b200mj_forward (geom_xpos, geom_xmat, site_xpos, site_xmat).
 * Objects are `nobj` primitives per environment (geoms first, then sites): type (mjtGeom), kind (mjtObj: 5 geom, 6 site),
 * id within its kind, rgba (float), size (3 doubles; size_stride = doubles between environments, 0 when shared),
 * pos [batch, nobj, 3], mat [batch, nobj, 9]; objects with visible[i] == 0 are skipped. Camera: cam_xpos [batch, 3],
 * cam_xmat [batch, 9] (columns: right, up, backward — the camera looks along -z), vertical field of view `fovy` in
 * degrees; the pixel <-> ray map is the inverse of the reference's camera matrix (engine.py:759-810). Any of the three
 * outputs may be NULL: rgb uint8 [batch, H, W, 3] (headlight-shaded rgba, black background), depth float32
 * [batch, H, W] (distance along the optical axis, `zfar` where nothing is hit; hits nearer than `znear` are clipped),
 * seg int32 [batch, H, W, 2] = (object id, object kind), (-1, -1) for the background. */
typedef struct b200mj_render_scene {
  int nobj;
  const int32_t* obj_type; const int32_t* obj_kind; const int32_t* obj_id; const uint8_t* visible;
  const float* rgba;
  const double* size; long long size_stride;
  const double* pos; const double* mat;
  const double* cam_xpos; const double* cam_xmat;
  double fovy, znear, zfar;
} b200mj_render_scene;
int b200mj_render(const b200mj_render_scene* scene, int batch, int height, int width, uint8_t* rgb, float* depth, int32_t* seg,
                  void* stream);

/* End-to-end form with HOST buffers: copies ctrl_host [batch,nu] to the device, runs b200mj_step on the
 * device-resident io, copies `nobs` packed doubles per env (obs_dev -> obs_host) back, synchronises. */
int b200mj_step_host(const b200mj_model* m, const b200mj_io* io, int batch, int nstep, int flags,
                     const double* ctrl_host, double* ctrl_dev, const double* obs_dev, double* obs_host, int nobs,
                     void* stream);

/* mj_resetData / mj_resetDataKeyframe + mj_forward with actuation disabled (Physics.reset, engine.py:306-327) for the
 * environments whose env_mask byte is non-zero (env_mask == NULL: all), in two launches: qpos <- qpos0 or key_qpos[keyframe]
 * (keyframe < 0: qpos0), qvel / act / qacc_warmstart / ctrl / time <- 0, then the forward pass; the other
 * environments' state and outputs are left untouched. */
int b200mj_reset(const b200mj_model* m, const b200mj_io* io, int batch, const uint8_t* env_mask_dev, int keyframe, void* stream);
/* mj_forward restricted to the environments of env_mask (NULL: all): after_reset() of a masked reset (engine.py:329-333) */
int b200mj_forward_masked(const b200mj_model* m, const b200mj_io* io, int batch, const uint8_t* env_mask_dev,
                          int extra_disableflags, int flags, void* stream);
/* mj_contactForce (mujoco/wrapper/core.py:546-551) for contact `contact_id` of every environment, from the contact
 * and efc_force arrays of `io`: out6_dev [batch, 6] = force (normal, tangent1, tangent2) and torque (zero for condim
 * 1 / 3) in the contact frame; zeros where contact_id >= ncon or the contact has no constraint rows. */
int b200mj_contact_force(const b200mj_model* m, const b200mj_io* io, int batch, int contact_id, double* out6_dev, void* stream);
/* mj_step1-equivalent on the current state without integrating: position / velocity stage, mj_subtreeVel
 * (io->subtree_linvel; locomotion/walkers/legacy_base.py:179-186 calls it after every substep), position- and
 * velocity-stage sensors, outputs. */
int b200mj_subtree_vel(const b200mj_model* m, const b200mj_io* io, int batch, int flags, void* stream);
/* Name the geoms that take per-environment pos / size from io->var_geom_pos / var_geom_size (slot k <-> geom_ids[k]). */
int b200mj_model_set_variable_geoms(b200mj_model* m, const int32_t* geom_ids, int n);
/* Per-environment model fields: for each environment e < nrows, field field_ids[k] (its position in
 * B200MJ_MODEL_FIELDS) is read from rows_dev[e * row + off_k] instead of the shared model, where row is the sum of
 * the listed fields' full lengths in the order given and off_k the sum of the lengths before k. n == 0: off.
 * Supported (float64): body_mass, body_inertia, body_ipos, geom_friction, geom_solref, geom_solimp, dof_damping,
 * dof_armature, jnt_stiffness, actuator_gainprm, actuator_biasprm; nothing derived from them is recomputed (MuJoCo's
 * model-write rule without mj_setConst). An environment whose dof_damping row has a positive entry takes the implicit
 * damping update of mj_Euler. rows_dev is read by every later call until the next b200mj_model_set_env_fields (a
 * captured graph reads the live rows); calls that run physics on more than nrows environments return an error. */
int b200mj_model_set_env_fields(b200mj_model* m, const int32_t* field_ids, int n, const double* rows_dev, int nrows);

/* instrumentation */
int64_t b200mj_workspace_bytes(const b200mj_model* m);   /* shared memory per environment (bytes) */
int b200mj_envs_per_block(const b200mj_model* m);
/* JSON description of the kernel workspaces (fused, position, acceleration row-buckets) into buf[n]; 0 ok. */
int b200mj_describe(const b200mj_model* m, char* buf, int n);
int64_t b200mj_launch_count(void);                        /* kernels launched by this library so far */
const char* b200mj_error_string(int code);
const char* b200mj_version(void);

#ifdef __cplusplus
}
#endif
#endif /* B200MJ_H_ */
