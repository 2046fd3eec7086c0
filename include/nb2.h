/* nb2.h — C ABI of the H100 batched differentiable-timestep engine (libnb2.so).
 *
 * Drop-in boundary for the reference's hot path.  What each entry point replaces:
 *   nb2_step_forward   <- neural::forwardPass(world)            dart/neural/NeuralUtils.cpp:26-66
 *                         = World::setState/setAction/step      dart/simulation/World.cpp:2024-2086, 221-254
 *   nb2_step_backward  <- BackpropSnapshot::backpropState       dart/neural/BackpropSnapshot.cpp:382-420 (+ :121-194, :425-479)
 *   nb2_model_create   <- the World/Skeleton object graph a loader builds (dart/simulation/World.cpp:749-793), flattened
 *   nb2_rollout_*      <- trajectory::SingleShot::getSnapshots / backpropGradientWrt   dart/trajectory/SingleShot.cpp:635-686, 539-631
 * The pointer-style precedent inside the reference is SimpleFeatherstone::forwardDynamics(s_t*,s_t*,s_t*,s_t*)
 * (dart/dynamics/SimpleFeatherstone.hpp:61-65) and BoxedLcpSolver::solve(int, s_t*, ...) (dart/constraint/BoxedLcpSolver.hpp:125-135).
 *
 * Conventions: all batch buffers are row-major fp32, one row per world: state [B, 2*ndof] = [q ; qdot],
 * action [B, na].  Device entry points take DEVICE pointers and are stream-ordered (no hidden sync); the *_host
 * variants take HOST pointers and include the copies.  Every function returns 0 on success, a negative nb2_status
 * otherwise; nb2_last_error() describes the last failure of the calling thread.  There is no CPU fallback.
 */
#ifndef NB2_H_
#define NB2_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct nb2_model nb2_model; /* opaque: device model + launch configuration */

enum nb2_status {
  NB2_OK = 0,
  NB2_ERR_INVALID = -1,     /* bad argument / unsupported model */
  NB2_ERR_CUDA = -2,        /* CUDA runtime error (see nb2_last_error) */
  NB2_ERR_UNSUPPORTED = -3, /* model exceeds compiled limits */
};

enum nb2_precision { NB2_FP32 = 0, NB2_FP64 = 1 }; /* arithmetic type inside the kernels; I/O is always fp32 */

/* Canonical model description (see nimblephysics_b200/modelspec.py::compile_model for the producer and
 * nimblephysics_b200/csrc/nb2_model.h for the meaning of each field). All arrays are host memory, copied. */
typedef struct nb2_model_desc {
  int32_t nb, ndof, na, nslots;
  const int32_t* parent;      /* [nb]  canonical parent or -1 */
  const int32_t* jtype;       /* [nb]  1 revolute-z, 2 prismatic-z, 3 free */
  const int32_t* dof_off;     /* [nb] */
  const int32_t* flags;       /* [nb] */
  const int32_t* slot_self;   /* [nb] first accumulator slot owned by the body (or -1) */
  const int32_t* slot_parent; /* [nb] slot the body deposits into (or -1) */
  const int32_t* slot_count;  /* [nb] number of slots owned */
  const double* Xtree;        /* [nb*12] */
  const double* inertia;      /* [nb*10] */
  const double* damping;      /* [ndof] ... */
  const double* spring;
  const double* rest;
  const double* pos_lo;
  const double* pos_hi;
  const double* vel_lo;
  const double* vel_hi;
  const double* force_lo;
  const double* force_hi;
  const int32_t* action_map;  /* [na] */
  double gravity[3];
  double dt;
  /* ---- contact stage (nshapes == 0: contact-free world) ---- */
  int32_t nshapes, npairs;
  const int32_t* shape_body;      /* [nshapes] canonical body index, -1 = static (world-fixed) */
  const int32_t* shape_type;      /* 0 box (dims = full size), 1 sphere (dims[0] = r), 2 capsule (dims[0] = r, dims[1] = height) */
  const int32_t* shape_orig_body; /* reference BodyNode index, reported with the contacts */
  const double* shape_dims;       /* [nshapes*3] */
  const double* shape_T;          /* [nshapes*12] shape frame -> canonical body frame (or world) */
  const double* shape_mu;         /* friction coefficient of the owning body */
  const double* shape_rest;       /* restitution coefficient of the owning body */
  const int32_t* pair_a;          /* [npairs] collision pairs (shape indices) in the reference's enumeration order */
  const int32_t* pair_b;
  int32_t penetration_correction;
  double contact_clipping_depth, fallback_cfm;
  /* ---- cooperative schedule: `lanes` threads share one world (contact worlds must use 1). sched is
   * [trunk_n, lo, hi, ...,  then for each lane: limb_n, lo, hi, ...] with half-open canonical body ranges. */
  int32_t lanes, nsched;
  const int32_t* sched;
  /* ---- joints whose position limits are enforced (Joint::setPositionLimitEnforced, constraint/JointLimitConstraint.cpp): the bodies whose
   * parent joint (revolute / prismatic) it is, in the reference's joint order.  While q sits on or beyond pos_lo / pos_hi the contact stage
   * adds one LCP row for the joint after the contact rows (ConstraintSolver.cpp:642-695).  nlimits = 0: none (the loaders' default). */
  int32_t nlimits;
  const int32_t* limit_body;
} nb2_model_desc;

int nb2_model_create(const nb2_model_desc* desc, nb2_model** out);
/* Register one more sweep schedule of the SAME model (desc identical except lanes / flags / slot_* / nslots / sched).
 * The step entry points then pick, per launch, the schedule with the lowest estimated cost
 * (sequential depth of the schedule x waves the batch needs at that schedule's occupancy): small batches are latency
 * bound and get several threads per world, large ones fewer.  Register schedules before the first step call.
 * nb2_model_set_lanes pins the choice (0 = automatic); nb2_model_lanes_for reports it (backward: 0/1, precision: nb2_precision). */
int nb2_model_add_schedule(nb2_model* m, const nb2_model_desc* desc);
int nb2_model_set_lanes(nb2_model* m, int lanes);
int nb2_model_lanes_for(nb2_model* m, int B, int backward, int precision);
/* Replace the inertia parameters [nb*10] (m, h, Ibar as in nb2_model_desc.inertia) of every registered schedule:
 * what World::setMasses (World.cpp:1821-1825) changes; tree, limits and schedules stay.  Takes effect for launches
 * issued after the call (the model is a kernel parameter, copied at launch). */
int nb2_model_set_inertia(nb2_model* m, const double* inertia);
void nb2_model_destroy(nb2_model* m);
int nb2_model_ndof(const nb2_model* m);
int nb2_model_na(const nb2_model* m);

/* words per world the forward pass streams out for the backward pass ([words][B] layout); a word is 4 bytes
 * with NB2_FP32 and 8 bytes with NB2_FP64 (the stream is kept in the arithmetic type of the kernels) */
int nb2_saved_words_per_world(const nb2_model* m);

/* One differentiable timestep for B independent worlds.  `saved` may be NULL (no backward will follow),
 * otherwise it must hold nb2_saved_words_per_world(m)*B words.  `stream` is a cudaStream_t (NULL = default). */
int nb2_step_forward(const nb2_model* m, int B, const float* state, const float* action, float* next_state,
                     void* saved, int precision, void* stream);

/* Vector-Jacobian product of the same step: grad_next_state [B,2n] -> grad_state [B,2n], grad_action [B,na].
 * grad_inertia (may be NULL): [10*nb][B] floats, dL/d(m, h=m*c (3), Ibar xx,yy,zz,xy,xz,yz about the body origin) of every
 * canonical body and world — the raw material of lossWrtMass (BackpropSnapshot.cpp:167-178, WithRespectToMass.cpp);
 * the host contracts it with d(canonical inertia)/d(mass vector) (modelspec.inertia_param_jacobian). Contact-free step only. */
int nb2_step_backward(const nb2_model* m, int B, const float* state, const float* action, const void* saved,
                      const float* grad_next_state, float* grad_state, float* grad_action, float* grad_inertia,
                      int precision, void* stream);

/* Same two calls with HOST buffers (pageable or pinned): H2D copies, kernels, D2H copies, synchronised on return. */
int nb2_step_forward_host(nb2_model* m, int B, const float* state, const float* action, float* next_state,
                          int keep_for_backward, int precision);
int nb2_step_backward_host(nb2_model* m, int B, const float* grad_next_state, float* grad_state, float* grad_action,
                           int precision);

/* ---- per-world inertia: the *_pw variants of the step and rollout entry points ----------------------------------------------
 * world_inertia (may be NULL = the model's table): device memory, fp64, word-major [10*nb][B] (the layout of grad_inertia): word k of
 * canonical body i of world w at world_inertia[(10*i + k) * B + w], holding (m, h = m*c (3), Ibar xx,yy,zz,xy,xz,yz about the body origin)
 * exactly as nb2_model_desc.inertia does.  World w then steps with its own inertia; everything else of the model is shared.
 * A backward must be given the SAME world_inertia as the forward whose saved stream it consumes.  Masses are not checked on the device:
 * a world with a non-positive mass gets non-finite outputs; no other world is affected.  The existing entry points are these with NULL.
 * Not extended: the *_host entry points, nb2_forward_dynamics and the IKMapping kernels (COM entries use the model's masses). */
int nb2_step_forward_pw(const nb2_model* m, int B, const float* state, const float* action, const double* world_inertia, float* next_state,
                        void* saved, int precision, void* stream);
int nb2_step_backward_pw(const nb2_model* m, int B, const float* state, const float* action, const double* world_inertia, const void* saved,
                         const float* grad_next_state, float* grad_state, float* grad_action, float* grad_inertia,
                         int precision, void* stream);

#define NB2_MAX_CONTACTS 16
#define NB2_MAX_ROWS 48
/* ---- contact / boxed-LCP stage -------------------------------------------------------------------------------
 * Replaces ConstraintSolver::solve + World::integrateVelocitiesFromImpulses (dart/constraint/ConstraintSolver.cpp:376-823,
 * dart/constraint/BoxedLcpConstraintSolver.cpp:190-789, dart/simulation/World.cpp:283-304) for worlds whose model has shapes.
 * Arithmetic is fp64.  Buffers are device memory, one row per world:
 *   x_lcp   [B, NB2_MAX_ROWS] double   in: cached LCP solution (BoxedLcpConstraintSolver::mX), out: this step's solution
 *   m_lcp   [B] int32                  in: its size (-1: none), out: LCP dimension of this step
 *   labels  [B, NB2_MAX_ROWS] int32    out: ConstraintMapping per row (-2 clamping, -1 not clamping, >=0 upper-bound -> normal row)
 *   status  [B] int32                  out: bits 1 warm-start short-circuit, 2 Dantzig ran, 4 Dantzig failed, 8 PGS ran, 16 friction dropped,
 *            32 NaN reset, 64 standardisation kept the raw x, 128 unsupported geometry (capsule side contact), 256 contacts dropped (overflow),
 *            512 columns merged, 1024 restitution bounce active, 2048 backward failed (status_accum only), 4096 penetration correction
 *   ncontacts [B] int32                out
 *   cinfo   [B, NB2_MAX_CONTACTS, 10] float (optional, may be NULL): point(3) normal(3) depth bodyA bodyB type
 *   contact_record [B, nb2_contact_record_bytes/B/8] double (optional): what nb2_step_backward_contact needs (LCP size, labels,
 *            impulses, the velocity change they caused — ~1 KB per world; the clamping block of the LCP matrix is re-measured),
 *            the batched counterpart of the ConstrainedGroupGradientMatrices a BackpropSnapshot holds.
 */
size_t nb2_contact_workspace_bytes(const nb2_model* m, int B);
int nb2_model_has_contacts(const nb2_model* m);
/* forward step WITH the contact stage: one warp per world, the problem in shared memory; with a saved stream four kernels in stream order
 * (build -> solve head -> solve tail over the worlds that need the chain -> apply), without one a single fused kernel.  saved_fp64: nb2_saved_words_per_world(m) * B doubles (world-major; opaque), may be NULL when no backward will follow
 * (then contact_record must be NULL too).  workspace: nb2_contact_workspace_bytes(m, B) bytes of device memory — a pool of large
 * per-world workspaces for the rare worlds whose contact count exceeds the shared-memory capacity (nb2_model_set_contact_capacity).
 * status_accum (optional, [B] int32): every step ORs its status word into it — a sticky copy the caller reads once per rollout. */
int nb2_step_forward_contact(const nb2_model* m, int B, const float* state, const float* action, float* next_state,
                             void* saved_fp64, void* workspace, double* x_lcp, int32_t* m_lcp, int32_t* labels,
                             int32_t* status, int32_t* ncontacts, float* cinfo, double* contact_record, int32_t* status_accum, void* stream);
size_t nb2_contact_record_bytes(const nb2_model* m, int B);
/* VJP of a step taken with nb2_step_forward_contact (classification frozen at the forward solution), replaces
 * BackpropSnapshot::backpropState for steps with active contact constraints (dart/neural/BackpropSnapshot.cpp:980-1107,
 * 2723-3146), including steps with restitution (bounce diagonals, :2624-2680) and penetration correction.  Rows may act on one or two moving
 * bodies.  If a world cannot be back-propagated (the rows regenerated in the backward pass do not match the forward's, a compiled limit is exceeded) its gradients are NaN — never silent
 * garbage — and, when `status_accum` is given, bit NB2_ST_BWD_ERROR (2048) is OR-ed into status_accum[w]: callers check the array
 * once per rollout instead of scanning gradients.
 * grad_inertia: optional [10*nb][B] floats as in nb2_step_backward (mass gradient through the contact stage). */
int nb2_step_backward_contact(const nb2_model* m, int B, const float* state, const float* action, const void* saved_fp64,
                              const double* contact_record, void* workspace, const float* grad_next_state, float* grad_state,
                              float* grad_action, float* grad_inertia, int32_t* status_accum, void* stream);
/* per-world inertia (see nb2_step_forward_pw); the contact stage itself reads no inertia: it works from the forward's articulated quantities */
int nb2_step_forward_contact_pw(const nb2_model* m, int B, const float* state, const float* action, const double* world_inertia, float* next_state,
                                void* saved_fp64, void* workspace, double* x_lcp, int32_t* m_lcp, int32_t* labels,
                                int32_t* status, int32_t* ncontacts, float* cinfo, double* contact_record, int32_t* status_accum, void* stream);
int nb2_step_backward_contact_pw(const nb2_model* m, int B, const float* state, const float* action, const double* world_inertia, const void* saved_fp64,
                                 const double* contact_record, void* workspace, const float* grad_next_state, float* grad_state,
                                 float* grad_action, float* grad_inertia, int32_t* status_accum, void* stream);
/* contacts per world the shared-memory workspace of the fused contact kernels is sized for (LCP rows: 3x).  Default: 4 per box-box
 * pair + 1 per other pair, clamped to [2, NB2_MAX_CONTACTS].  Smaller = more resident worlds per SM, more worlds in the slow pool. */
/* The same two calls with HOST buffers (pageable or pinned): copies, kernels and a synchronise inside; the solver cache, the saved stream, the
 * contact record and the sticky status live in the model between calls (reset_cache != 0 forgets the cached LCP solutions first).
 * status_out (optional, [B]): this step's status words; sticky_out (optional, [B]): read-and-clear of the sticky word after the backward. */
int nb2_step_forward_contact_host(nb2_model* m, int B, const float* state, const float* action, float* next_state, int keep_for_backward,
                                  int reset_cache, int32_t* status_out);
int nb2_step_backward_contact_host(nb2_model* m, int B, const float* grad_next_state, float* grad_state, float* grad_action, int32_t* sticky_out);
int nb2_model_set_contact_capacity(nb2_model* m, int max_contacts_in_shared_memory);
int nb2_model_contact_capacity(const nb2_model* m);

/* Pointer-style forward dynamics q-ddot = FD(q, q-dot, tau) of B worlds (ABA, no integration, no contacts): the batched counterpart of
 * SimpleFeatherstone::forwardDynamics(s_t* pos, s_t* vel, s_t* force, s_t* accel) (dart/dynamics/SimpleFeatherstone.hpp:61-65,
 * SimpleFeatherstone.cpp:26-138) and of Skeleton::computeForwardDynamics + getAccelerations.  fp64 device arrays [B, ndof]; the model's
 * gravity applies (the reference's test zeroes it, unittests/comprehensive/test_SimpleFeatherstone.cpp:34).  Requires the default action
 * space (every dof).  It is one launch of the fp64 kernel of nb2_forward_dynamics_batch, reading pos and vel in place; a model whose fp64
 * working set fits no schedule's shared memory (which nb2_forward_dynamics_batch refuses with NB2_ERR_UNSUPPORTED) runs the same stages one
 * thread per world with scratch in global memory, allocated stream-ordered for the call. */
int nb2_forward_dynamics(const nb2_model* m, int B, const double* pos, const double* vel, const double* force, double* accel, void* stream);

/* Contact-free forward dynamics of B worlds: the acceleration accel [B, ndof] the contact-free step applies at state = [q ; qdot] under the
 * generalised force tau [B, ndof]:
 *     accel = M(q)^-1 ( tau - C(q, qdot) - g(q) - K (q - q0 + qdot dt) - D qdot )      (v+ = qdot + dt accel)
 * It is the exact inverse of nb2_inverse_dynamics: nb2_inverse_dynamics(state, qdot + dt accel) returns tau up to rounding.  tau is per dof,
 * not gathered through the action map, so any action space works; free joints use the step's conventions (body-twist velocities and
 * accelerations, the 6-vector joint force in the joint frame).  Contacts, joint-limit rows, velocity and force limits are ignored: a model with
 * collision pairs gets the accelerations of its trees, and no LCP cache is read or written.
 * Rows in the arithmetic type (float with NB2_FP32, double with NB2_FP64), device memory, one row per world.  world_inertia (may be NULL):
 * per-world inertia as for nb2_step_forward_pw.  saved (may be NULL when no backward will follow): nb2_saved_words_per_world(m) * B words of
 * the arithmetic type, [words][B], the step's saved-stream layout.  Launch shapes and lane schedules are picked per call as for the step;
 * NB2_ERR_UNSUPPORTED when no schedule's working set fits in shared memory (as for the step, e.g. a 64-body chain in fp64). */
int nb2_forward_dynamics_batch(const nb2_model* m, int B, const void* state, const void* tau, const double* world_inertia, void* accel, void* saved,
                               int precision, void* stream);
/* Vector-Jacobian product of the same call, with the SAME state, world_inertia and saved stream.  grad_accel [B, ndof] -> grad_state [B, 2*ndof]
 * = [dL/dq ; dL/dqdot], grad_tau [B, ndof] (all in the arithmetic type); grad_inertia (may be NULL): [10*nb][B] DOUBLES, dL/d(m, h, Ibar) of every
 * canonical body and world, laid out as nb2_inverse_dynamics_backward's.  No clipping is applied.  Allocates nothing. */
int nb2_forward_dynamics_backward(const nb2_model* m, int B, const void* state, const double* world_inertia, const void* saved, const void* grad_accel,
                                  void* grad_state, void* grad_tau, double* grad_inertia, int precision, void* stream);

/* Contact-free inverse dynamics of B worlds: the generalised force tau [B, ndof] for which the contact-free step started at
 * state = [q ; qdot] reaches the next velocity next_vel [B, ndof]:
 *     a = (next_vel - qdot) / dt ,   tau = M(q) a + C(q, qdot) + g(q) + K (q - q0 + qdot dt) + D qdot      (per dof)
 * (the step's semi-implicit spring and damping).  tau is in dof space, not gathered through the action map; free joints use the step's
 * conventions (rotation-vector positions, body-twist velocities, the 6-vector joint force in the joint frame).  Contacts, joint-limit rows
 * and force limits are ignored: a model with collision pairs gets the tau of its tree, and no LCP cache is read or written.  The round trip
 * holds: with an action space covering every dof, nb2_step_forward(state, tau) returns next_vel up to rounding.
 * UNLIKE the step entry points, the rows are in the arithmetic type: state, next_vel, tau, grad_* are float with NB2_FP32 and double
 * with NB2_FP64 (device memory, row-major, one row per world).  world_inertia (may be NULL): per-world inertia as for nb2_step_forward_pw.
 * saved (may be NULL when no backward will follow): nb2_saved_words_per_world(m) * B words of the arithmetic type, [words][B], the step's
 * saved-stream layout.  Launch shapes and lane schedules are picked per call as for the step (nb2_model_add_schedule). */
int nb2_inverse_dynamics(const nb2_model* m, int B, const void* state, const void* next_vel, const double* world_inertia, void* tau, void* saved,
                         int precision, void* stream);
/* Vector-Jacobian product of the same call, with the SAME state, world_inertia and saved stream (next_vel is not read: the saved stream
 * holds the accelerations it implies; it may be NULL).  grad_tau [B, ndof] -> grad_state [B, 2*ndof] = [dL/dq ; dL/dqdot], grad_next_vel
 * [B, ndof] (all in the arithmetic type); grad_inertia (may be NULL): [10*nb][B] DOUBLES, dL/d(m, h, Ibar) of every canonical body and
 * world, laid out as nb2_step_backward's (contract with modelspec.inertia_param_jacobian for dL/dmass).  No clipping is applied. */
int nb2_inverse_dynamics_backward(const nb2_model* m, int B, const void* state, const void* next_vel, const double* world_inertia, const void* saved,
                                  const void* grad_tau, void* grad_state, void* grad_next_vel, double* grad_inertia, int precision, void* stream);

/* Contact inverse dynamics of B worlds with one contact body: tau_ID of nb2_inverse_dynamics split into the contact wrench [B, 6] and the
 * joint torques tau [B, ndof] that remain:
 *     tau + J_c(q)^T wrench = tau_ID        on every dof,        tau = 0 on the six dofs of the contact body's free root,
 * where J_c maps qdot to the spatial velocity [omega; v_origin] of contact_body in world axes about the world origin, and wrench is
 * [torque; force] in the same axes about the same point.  The root's six tau_ID entries are its joint-frame force F_r (the step's free-joint
 * convention), so wrench = X*(root -> world) F_r, and tau differs from tau_ID only on the dofs of the joints between contact_body and the
 * root: tau_j = tau_ID,j - S_j^T F_j with F_j = F_r expressed in frame j.  Every other dof is tau_ID exactly.  The wrench is the same for
 * every body of the tree.  contact_body: canonical body index (modelspec body_owner); it must lie under a FREE root (NB2_ERR_INVALID
 * otherwise).  Rows, world_inertia and saved are those of nb2_inverse_dynamics (arithmetic type); tau, wrench: device, one row per world. */
int nb2_contact_inverse_dynamics(const nb2_model* m, int B, int contact_body, const void* state, const void* next_vel, const double* world_inertia,
                                 void* tau, void* wrench, void* saved, int precision, void* stream);
/* Vector-Jacobian product of the same call, with the SAME state, world_inertia, saved stream and the forward's wrench (next_vel is not
 * read).  grad_tau [B, ndof], grad_wrench [B, 6] -> grad_state, grad_next_vel, grad_inertia as in nb2_inverse_dynamics_backward.  seed:
 * caller-owned workspace [B, ndof] in the arithmetic type (the g_tau_ID handed to the inverse-dynamics backward); the call allocates nothing. */
int nb2_contact_inverse_dynamics_backward(const nb2_model* m, int B, int contact_body, const void* state, const void* next_vel,
                                          const double* world_inertia, const void* saved, const void* wrench, const void* grad_tau,
                                          const void* grad_wrench, void* seed, void* grad_state, void* grad_next_vel, double* grad_inertia,
                                          int precision, void* stream);

/* Multiple-contact inverse dynamics of B worlds: tau_ID of nb2_inverse_dynamics split over k = ncontact contact bodies of one tree, into
 * wrenches w_i [B, k, 6] and the joint torques tau [B, ndof] that remain:
 *     tau + sum_i J_i(q)^T w_i = tau_ID   on every dof,   tau = 0 on the six dofs of the bodies' free root,
 *     minimise sum_i | Gamma(p_i)^-1 (w_i - g_i) |^2,
 * J_i and the wrench convention ([torque; force], world axes, about the world origin) as nb2_contact_inverse_dynamics; p_i the world
 * position of contact point i, Gamma(p) = [[I, [p]x], [0, I]] (a wrench about p -> about the origin), so the deviation is measured as
 * [torque about p_i; force]; g_i the guesses.  The constraint is sum_i w_i = W (the one-body wrench) and
 *     lambda = H^-1 (W - sum_j g_j),  w_i = g_i + Gamma_i Gamma_i^T lambda,  H = sum_i Gamma_i Gamma_i^T.
 * contact_body [k]: canonical body indices (host); contact_point [k][3] (host): each point in its body's canonical frame.  1 <= k <=
 * NB2_MAX_CONTACT_BODIES; every body in range and under the same FREE root (NB2_ERR_INVALID otherwise).  guess [B, k, 6] or NULL (0).  With
 * k = 1 the result is nb2_contact_inverse_dynamics's (the guess is not read).  Rows, world_inertia and saved as nb2_inverse_dynamics. */
#define NB2_MAX_CONTACT_BODIES 4
int nb2_multiple_contact_inverse_dynamics(const nb2_model* m, int B, int ncontact, const int32_t* contact_body, const double* contact_point,
                                          const void* state, const void* next_vel, const double* world_inertia, const void* guess, void* tau,
                                          void* wrenches, void* saved, int precision, void* stream);
/* Vector-Jacobian product of the same call, with the SAME bodies, points, state, world_inertia, saved stream and guess, and the forward's
 * wrenches (next_vel is not read).  grad_tau [B, ndof], grad_wrenches [B, k, 6] -> grad_state, grad_next_vel, grad_inertia (may be NULL)
 * as nb2_inverse_dynamics_backward, and grad_guess [B, k, 6] (may be NULL).  seed: caller-owned workspace [B, ndof] in the arithmetic type;
 * the call allocates nothing. */
int nb2_multiple_contact_inverse_dynamics_backward(const nb2_model* m, int B, int ncontact, const int32_t* contact_body, const double* contact_point,
                                                   const void* state, const void* next_vel, const double* world_inertia, const void* saved,
                                                   const void* wrenches, const void* guess, const void* grad_tau, const void* grad_wrenches,
                                                   void* seed, void* grad_state, void* grad_next_vel, double* grad_inertia, void* grad_guess,
                                                   int precision, void* stream);
/* Dense Jacobians of nb2_multiple_contact_inverse_dynamics (DESIGN.md §6s), in one launch.  Arguments as that call (no saved stream), whose
 * tau [B, ndof] and wrenches [B, k, 6] it also writes, with m = 6k and row-major blocks in the arithmetic type, device memory:
 *     T_q, T_qdot, T_next_vel [B, ndof, ndof],  T_guess [B, ndof, m] :  T_x[w, i, j] = d tau[w, i] / d x[w, j] ,
 *     W_q, W_qdot, W_next_vel [B, m, ndof],     W_guess [B, m, m]    :  W_x[w, 6 i + c, j] = d wrenches[w, i, c] / d x[w, j] ,
 * next_vel held fixed in the q and qdot blocks.  Row i of each block is nb2_multiple_contact_inverse_dynamics_backward with the seed e_i on
 * that output (with k = 1 nb2_contact_inverse_dynamics_backward's), so free joints follow its conventions (position columns for the six
 * stored coordinates, body-twist velocity columns) and the blocks equal the VJP's rows up to rounding; the free root's six rows of every
 * T block are 0.  T_guess and W_guess may be NULL; with k = 1 they are 0 (the guess is not read).  tau and the wrenches are written by the
 * forward of nb2_multiple_contact_inverse_dynamics itself (further launches on the stream), so they equal its outputs bit for bit.  Masses
 * are held fixed.  Stateless, stream-ordered, nothing allocated, B = 0 only validates.  NB2_ERR_INVALID as
 * nb2_multiple_contact_inverse_dynamics; NB2_ERR_UNSUPPORTED when the working set does not fit shared memory even at 4 row slots. */
int nb2_multiple_contact_inverse_dynamics_jacobians(const nb2_model* m, int B, int ncontact, const int32_t* contact_body,
                                                    const double* contact_point, const void* state, const void* next_vel,
                                                    const double* world_inertia, const void* guess, void* tau, void* wrenches, void* T_q,
                                                    void* T_qdot, void* T_next_vel, void* T_guess, void* W_q, void* W_qdot, void* W_next_vel,
                                                    void* W_guess, int precision, void* stream);

/* Joint-space mass matrix M(q) [B, ndof, ndof] (row-major) of B worlds at the positions pos [B, ndof]: the matrix the step inverts, in its
 * velocity coordinates (free joints: body twist, S = I6), block-diagonal over trees; contacts, limits, springs and damping are not part of
 * it.  Rows in the arithmetic type of `precision` (NB2_FP64: double, else float); world_inertia as nb2_step_forward_pw (NULL: the model's).
 * Composite-rigid-body algorithm, one warp per world.  The result is exactly symmetric.  NB2_ERR_INVALID for a model without dofs. */
int nb2_mass_matrix(const nb2_model* m, int B, const void* pos, const double* world_inertia, void* M, int precision, void* stream);
/* M(q)^-1 [B, ndof, ndof]: the step's articulated inertias and one bias-free unit-force sweep pair per column (not a factorisation of M). */
int nb2_inverse_mass_matrix(const nb2_model* m, int B, const void* pos, const double* world_inertia, void* Minv, int precision, void* stream);
/* Vector-Jacobian products, L = <grad, out>.  grad_pos [B, ndof] (written; a free root's six entries are exactly 0), grad_inertia
 * [10 * nb][B] fp64 or NULL (written, as nb2_inverse_dynamics_backward).  The inverse's backward takes the forward's Minv and a caller-owned
 * workspace [B, ndof, ndof] in the arithmetic type; neither call allocates. */
int nb2_mass_matrix_backward(const nb2_model* m, int B, const void* pos, const double* world_inertia, const void* grad_M, void* grad_pos,
                             double* grad_inertia, int precision, void* stream);
int nb2_inverse_mass_matrix_backward(const nb2_model* m, int B, const void* pos, const double* world_inertia, const void* Minv, const void* grad_Minv,
                                     void* workspace, void* grad_pos, double* grad_inertia, int precision, void* stream);

/* Dense Jacobians of nb2_inverse_dynamics and nb2_forward_dynamics_batch, with their outputs, in one launch.  J[w][i][j] = d out_i / d in_j,
 * row-major [B, ndof, ndof] blocks in the arithmetic type of `precision`, device memory; state, next_vel, tau and world_inertia as for the
 * two calls.  Row i is the call's vector-Jacobian product with the seed e_i (free joints: body-twist velocity columns, position columns
 * through the six stored coordinates), so the blocks equal what the _backward entries give row by row:
 *   inverse dynamics  tau [B, ndof];  J_q = dtau/dq,  J_qdot = dtau/dqdot (next_vel held fixed),  J_next_vel = dtau/dnext_vel = M / dt
 *   forward dynamics  accel [B, ndof];  J_q = daccel/dq,  J_qdot = daccel/dqdot,  J_tau = daccel/dtau = M^-1
 * Contacts, limits and clipping are ignored; no LCP cache is read or written.  One warp per world, the working set in shared memory, which
 * every model of the mass-matrix envelope fits in both precisions (a 64-body chain in fp64 included).  Nothing is allocated.
 * NB2_ERR_INVALID for a model without dofs or a bad argument; NB2_ERR_UNSUPPORTED when the working set does not fit shared memory. */
int nb2_inverse_dynamics_jacobians(const nb2_model* m, int B, const void* state, const void* next_vel, const double* world_inertia, void* tau, void* J_q,
                                   void* J_qdot, void* J_next_vel, int precision, void* stream);
int nb2_forward_dynamics_jacobians(const nb2_model* m, int B, const void* state, const void* tau, const double* world_inertia, void* accel, void* J_q,
                                   void* J_qdot, void* J_tau, int precision, void* stream);

/* World Jacobians of body points [B, k, 6, ndof] (row-major per (world, node)) at the positions pos [B, ndof]: columns in the step's
 * velocity coordinates (free joints: body twist), J_e qdot = [omega_b ; d/dt p_e] in world axes for the point p_e = W_b T_e o_e of
 * canonical body b = body[e] (-1: static, an all-zero block).  T_owner_from_node [12k] (host, fp64: R row-major, p) places each node on
 * its body; offsets (device, arithmetic type): NULL (the nodes' origins), [k, 3] shared by the batch or [B, k, 3] (offsets_per_world = 1),
 * in each node's frame.  Rows in the arithmetic type of `precision`; world_inertia and mass play no part.  One warp per (world, node).
 * NB2_ERR_INVALID for k outside 1..NB2_MAX_JACOBIAN_NODES (32), a body outside -1..nb-1 or a model without dofs. */
#define NB2_MAX_JACOBIAN_NODES 32
int nb2_world_jacobian(const nb2_model* m, int B, const void* pos, int k, const int32_t* body, const double* T_owner_from_node, const void* offsets,
                       int offsets_per_world, void* J, int precision, void* stream);
/* VJP, L = <grad_J, J>: grad_pos [B, ndof] (written); grad_offsets NULL or [B, k, 3] (written, one row per world also for shared offsets:
 * their gradient is the sum over the batch, left to the caller so that it stays deterministic).  One warp per world owns its rows. */
int nb2_world_jacobian_backward(const nb2_model* m, int B, const void* pos, int k, const int32_t* body, const double* T_owner_from_node,
                                const void* offsets, int offsets_per_world, const void* grad_J, void* grad_pos, void* grad_offsets, int precision,
                                void* stream);
/* Centre-of-mass Jacobian [B, 3, ndof] of the tree rooted at canonical body root_body (Skeleton::getCOMLinearJacobian; columns of other
 * trees' dofs are 0); world_inertia as nb2_step_forward_pw (NULL: the model's).  Its VJP writes grad_pos [B, ndof] and, if not NULL,
 * grad_inertia [10 * nb][B] fp64 (as nb2_inverse_dynamics_backward; zero for bodies of other trees).  One warp per world.
 * NB2_ERR_INVALID for a root_body that is not a tree root or a model without dofs. */
int nb2_com_jacobian(const nb2_model* m, int B, const void* pos, int root_body, const double* world_inertia, void* J, int precision, void* stream);
int nb2_com_jacobian_backward(const nb2_model* m, int B, const void* pos, int root_body, const double* world_inertia, const void* grad_J,
                              void* grad_pos, double* grad_inertia, int precision, void* stream);

/* Time derivatives of the two Jacobians above at the states state [B, 2 ndof] = [q ; qdot] (Skeleton::getJacobianClassicDeriv,
 * getCOMLinearJacobianDeriv): dJ = d/dt J(q(t)) along a motion through q with velocity qdot (free joints: the tangent of the step's
 * position update), so that J qddot + dJ qdot is the acceleration.  Nodes, offsets, world_inertia, layouts and error cases as
 * nb2_world_jacobian / nb2_com_jacobian; B = 0 only validates.  The VJPs write grad_state [B, 2 ndof] = [dL/dq ; dL/dqdot] and, as the
 * Jacobians' VJPs, grad_offsets [B, k, 3] per world / grad_inertia [10 * nb][B].  Stateless, nothing allocated. */
int nb2_world_jacobian_deriv(const nb2_model* m, int B, const void* state, int k, const int32_t* body, const double* T_owner_from_node,
                             const void* offsets, int offsets_per_world, void* dJ, int precision, void* stream);
int nb2_world_jacobian_deriv_backward(const nb2_model* m, int B, const void* state, int k, const int32_t* body, const double* T_owner_from_node,
                                      const void* offsets, int offsets_per_world, const void* grad_dJ, void* grad_state, void* grad_offsets,
                                      int precision, void* stream);
int nb2_com_jacobian_deriv(const nb2_model* m, int B, const void* state, int root_body, const double* world_inertia, void* dJ, int precision,
                           void* stream);
int nb2_com_jacobian_deriv_backward(const nb2_model* m, int B, const void* state, int root_body, const double* world_inertia, const void* grad_dJ,
                                    void* grad_state, double* grad_inertia, int precision, void* stream);

/* Kinetic and potential energy and centroidal momentum of the tree rooted at canonical body root_body at the states state [B, 2 ndof]
 * (Skeleton::computeKineticEnergy / computePotentialEnergy, DESIGN.md §6m): kinetic [B] = 1/2 sum_i V_i . G_i V_i, potential [B] =
 * -g . sum_i (m_i p_i + R_i h_i) + 1/2 sum_d k_d (q_d - q0_d)^2 over the tree's bodies and dofs, momentum [B, 6] = [angular momentum about
 * the tree's COM ; linear momentum] in world axes.  Rows in the arithmetic type of `precision`; world_inertia as nb2_com_jacobian.  The
 * VJP reads grad_kinetic [B], grad_potential [B] and grad_momentum [B, 6] (each may be NULL: zero) and writes grad_state [B, 2 ndof] =
 * [dL/dq ; dL/dqdot] (0 on other trees' dofs) and, if not NULL, grad_inertia [10 * nb][B] fp64.  One warp per world; stateless, nothing
 * allocated, B = 0 only validates.  NB2_ERR_INVALID for a root_body that is not a tree root or a model without dofs. */
int nb2_energy_momentum(const nb2_model* m, int B, const void* state, int root_body, const double* world_inertia, void* kinetic, void* potential,
                        void* momentum, int precision, void* stream);
int nb2_energy_momentum_backward(const nb2_model* m, int B, const void* state, int root_body, const double* world_inertia, const void* grad_kinetic,
                                 const void* grad_potential, const void* grad_momentum, void* grad_state, double* grad_inertia, int precision,
                                 void* stream);

/* Inverse-dynamics regressor (DESIGN.md §6n): nb2_inverse_dynamics as a linear map of the canonical inertia table.  At state [B, 2 ndof]
 * and next_vel [B, ndof] it writes Y [B, ndof, nb, 10] and tau_passive [B, ndof] = K (q - q0 + qdot dt) + D qdot such that, for ANY
 * per-world inertia table pi ([nb][10] per world, the layout of world_inertia),
 *     nb2_inverse_dynamics(state, next_vel, world_inertia = pi)[w, d] = sum_{j,k} Y[w, d, j, k] pi[w, j, k] + tau_passive[w, d].
 * Y[w, d, j] is 0 unless dof d's joint is at or above canonical body j; every entry of the B rows is written.  Energy regressor: at state
 * [B, 2 ndof], Y_kinetic and Y_potential [B, nb, 10] and spring_energy [B] with sum_{j,k} Y_kinetic[w, j, k] pi[w, j, k] = 1/2 qdot^T M qdot,
 * sum_{j,k} Y_potential[w, j, k] pi[w, j, k] = -g . sum_j (m_j p_j + R_j h_j) (gravity at every body's COM), spring_energy =
 * 1/2 sum_d k_d (q_d - q0_d)^2 over all dofs.  Rows in the arithmetic type of `precision`.  Contacts, limits and clipping are ignored and
 * no LCP cache is read or written.  One warp per world; stateless, nothing allocated, B = 0 only validates.  NB2_ERR_INVALID for a model
 * without dofs. */
int nb2_inverse_dynamics_regressor(const nb2_model* m, int B, const void* state, const void* next_vel, void* Y, void* tau_passive, int precision,
                                   void* stream);
int nb2_energy_regressor(const nb2_model* m, int B, const void* state, void* Y_kinetic, void* Y_potential, void* spring_energy, int precision,
                         void* stream);

/* Constrained forward dynamics (DESIGN.md §6o): joint accelerations and contact wrenches of worlds whose k contact points are held by
 * bilateral constraints.  Contact i is canonical body body[i] (1 <= k <= NB2_MAX_CONTACT_BODIES, distinct, none static) at the point
 * T_owner_from_node[i] (R row-major 9, p 3: the node's placement on its body) applied to offsets[i] (NULL: the node's origin; [k, 3], or
 * [B, k, 3] with offsets_per_world).  It constrains the [omega ; pdot] rows of the point's world Jacobian J (nb2_world_jacobian), or only
 * its three linear rows with point_contacts.  With J [m, ndof] the stack, Jdot its time derivative (nb2_world_jacobian_deriv) and rho =
 * damping >= 0,
 *     M qdd + C + g + K (q - q0 + qdot dt) + D qdot = tau + J^T lam ,    J qdd + Jdot qdot = -rho lam ,
 * tau per dof as for nb2_forward_dynamics_batch.  accel [B, ndof] = qdd; wrenches [B, k, 6] = [lam_a + p_i x lam_l ; lam_l] (lam_i =
 * [torque about p_i ; force], world axes: the wrench about the world origin, as nb2_multiple_contact_inverse_dynamics) or, with
 * point_contacts, [B, k, 3] = the force.  A world whose J M^-1 J^T + rho I has a Cholesky pivot at or below 64 eps max(diagonal) gets NaN
 * rows.  The backward recomputes the forward and writes grad_state [B, 2 ndof], grad_tau [B, ndof], grad_offsets [B, k, 3] (or NULL, one
 * row per world also for shared offsets) and grad_inertia ([10 nb, B] fp64, or NULL).  Rows in the arithmetic type of `precision`;
 * contacts of the model, limits and the LCP cache play no part.  One warp per world; stateless, nothing allocated, B = 0 only validates.
 * NB2_ERR_INVALID for k out of range, a body out of range or repeated, a negative or non-finite damping or a model without dofs;
 * NB2_ERR_UNSUPPORTED when the working set does not fit shared memory. */
int nb2_constrained_forward_dynamics(const nb2_model* m, int B, const void* state, const void* tau, int k, const int32_t* body,
                                     const double* T_owner_from_node, const void* offsets, int offsets_per_world, int point_contacts, double damping,
                                     const double* world_inertia, void* accel, void* wrenches, int precision, void* stream);
int nb2_constrained_forward_dynamics_backward(const nb2_model* m, int B, const void* state, const void* tau, int k, const int32_t* body,
                                              const double* T_owner_from_node, const void* offsets, int offsets_per_world, int point_contacts,
                                              double damping, const double* world_inertia, const void* grad_accel, const void* grad_wrenches,
                                              void* grad_state, void* grad_tau, void* grad_offsets, double* grad_inertia, int precision,
                                              void* stream);
/* Dense Jacobians of constrained forward dynamics (DESIGN.md §6p), in one launch.  Arguments as nb2_constrained_forward_dynamics, whose
 * accel [B, ndof] and wrenches [B, k, r] (r = 6, or 3 with point_contacts) it also writes, with m = k r and
 *     J_q, J_qdot, J_tau [B, ndof, ndof] :  J_x[w, i, j] = d accel[w, i] / d x[w, j] ,
 *     W_q, W_qdot, W_tau [B, m, ndof]    :  W_x[w, i r + c, j] = d wrenches[w, i, c] / d x[w, j] ,
 * x = the positions, the velocities (both halves of state) and tau.  Row i of each block is nb2_constrained_forward_dynamics_backward
 * with the seed e_i on that output, so free joints follow its conventions (position columns for the six stored coordinates, body-twist
 * velocity columns) and the blocks equal the VJP's rows up to rounding.  accel and the wrenches are written by the forward of
 * nb2_constrained_forward_dynamics itself (a second launch on the stream), so they equal its outputs bit for bit.  Offsets and masses are
 * held fixed.  A singular world gets NaN in
 * its outputs and every block.  Stateless, stream-ordered, nothing allocated, B = 0 only validates.  NB2_ERR_INVALID as
 * nb2_constrained_forward_dynamics; NB2_ERR_UNSUPPORTED when the working set does not fit shared memory even at one row slot. */
int nb2_constrained_forward_dynamics_jacobians(const nb2_model* m, int B, const void* state, const void* tau, int k, const int32_t* body,
                                                const double* T_owner_from_node, const void* offsets, int offsets_per_world, int point_contacts,
                                                double damping, const double* world_inertia, void* accel, void* wrenches, void* J_q, void* J_qdot,
                                                void* J_tau, void* W_q, void* W_qdot, void* W_tau, int precision, void* stream);

/* Impulse dynamics (DESIGN.md §6q): the impact map of worlds whose k contact points strike and are held from then on.  Contacts, offsets,
 * point_contacts, damping and world_inertia as nb2_constrained_forward_dynamics, with J [m, ndof] the stack of the points' rows.  With
 * state [B, 2 ndof] = [q ; qdot-], e = restitution in [0, 1] and rho = damping,
 *     M (qdot+ - qdot-) = J^T Lam ,    J qdot+ = -e J qdot- - rho Lam ,
 * vel_after [B, ndof] = qdot+ (the step's velocity coordinates); impulses [B, k, 6] = [Lam_a + p_i x Lam_l ; Lam_l] (Lam_i = [angular
 * impulse about p_i ; linear impulse], world axes, N s: about the world origin) or, with point_contacts, [B, k, 3] = Lam_l.  Gravity, joint
 * springs and damping, limits, contacts of the model and the LCP cache play no part.  A world whose J M^-1 J^T + rho I has a Cholesky
 * pivot at or below 64 eps max(diagonal) gets NaN rows.  The backward recomputes the forward and writes grad_state [B, 2 ndof],
 * grad_offsets [B, k, 3] (or NULL) and grad_inertia ([10 nb, B] fp64, or NULL).  One warp per world; stateless, nothing allocated, B = 0
 * only validates.  NB2_ERR_INVALID as nb2_constrained_forward_dynamics and for a restitution outside [0, 1]; NB2_ERR_UNSUPPORTED when the
 * working set does not fit shared memory. */
int nb2_impulse_dynamics(const nb2_model* m, int B, const void* state, int k, const int32_t* body, const double* T_owner_from_node,
                         const void* offsets, int offsets_per_world, int point_contacts, double restitution, double damping,
                         const double* world_inertia, void* vel_after, void* impulses, int precision, void* stream);
int nb2_impulse_dynamics_backward(const nb2_model* m, int B, const void* state, int k, const int32_t* body, const double* T_owner_from_node,
                                  const void* offsets, int offsets_per_world, int point_contacts, double restitution, double damping,
                                  const double* world_inertia, const void* grad_vel, const void* grad_impulses, void* grad_state,
                                  void* grad_offsets, double* grad_inertia, int precision, void* stream);
/* Dense Jacobians of impulse dynamics (DESIGN.md §6r), in one launch.  Arguments as nb2_impulse_dynamics, whose vel_after [B, ndof] and
 * impulses [B, k, r] (r = 6, or 3 with point_contacts) it also writes, with m = k r and
 *     V_q, V_qdot [B, ndof, ndof] :  V_x[w, i, j] = d vel_after[w, i] / d x[w, j] ,
 *     I_q, I_qdot [B, m, ndof]    :  I_x[w, i r + c, j] = d impulses[w, i, c] / d x[w, j] ,
 * x = the positions or the pre-impact velocities (the two halves of state).  Row i of each block is nb2_impulse_dynamics_backward with
 * the seed e_i on that output, so free joints follow its conventions (position columns for the six stored coordinates, body-twist
 * velocity columns) and the blocks equal the VJP's rows up to rounding.  vel_after and the impulses are written by the forward of
 * nb2_impulse_dynamics itself (a second launch on the stream), so they equal its outputs bit for bit.  Offsets, masses, restitution and
 * damping are held fixed.  A singular world gets NaN in its outputs and every block.  Stateless, stream-ordered, nothing allocated, B = 0
 * only validates.  NB2_ERR_INVALID as nb2_impulse_dynamics; NB2_ERR_UNSUPPORTED when the working set does not fit shared memory even at
 * one row slot. */
int nb2_impulse_dynamics_jacobians(const nb2_model* m, int B, const void* state, int k, const int32_t* body, const double* T_owner_from_node,
                                   const void* offsets, int offsets_per_world, int point_contacts, double restitution, double damping,
                                   const double* world_inertia, void* vel_after, void* impulses, void* V_q, void* V_qdot, void* I_q,
                                   void* I_qdot, int precision, void* stream);

/* Batched boxed-LCP solves on the device: B independent problems, one warp each — the reference's pointer-style lower boundary
 * BoxedLcpSolver::solve(n, A, x, b, nub, lo, hi, findex, earlyTermination) (dart/constraint/BoxedLcpSolver.hpp:125-135) and the
 * solve chain of BoxedLcpConstraintSolver::solveLcp (BoxedLcpConstraintSolver.cpp:352-789).  Device pointers; problem w has dimension
 * m[w] <= mcap <= NB2_MAX_ROWS and sits at A[w][mcap][mcap] (row-major, symmetric), b / lo / hi / findex / x0 / x / labels [w][mcap].
 *   mode 0: Dantzig only (dSolveLCP, dart/external/odelcpsolver/lcp.cpp:780-1114); status[w] = 1 solved, 0 early termination, -1 cap
 *   mode 1: warm start (x0 or guessSolution) -> short-circuit -> Dantzig -> cfm + PGS -> friction drop -> classification;
 *           status[w] = NB2_ST_* bits, labels = ConstraintMapping per row.   x0 may be NULL. */
int nb2_lcp_solve_batch(int B, int mcap, int mode, int early_termination, double fallback_cfm, const int32_t* m, const double* A, const double* b,
                        const double* lo, const double* hi, const int32_t* findex, const double* x0, double* x, int32_t* labels, int32_t* status,
                        void* stream);

/* T-step rollout of a contact-free world and its reverse sweep — SingleShot::getSnapshots (dart/trajectory/SingleShot.cpp:635-686)
 * and SingleShot::backpropGradientWrt (:539-631).  All buffers are device memory, fp32, time-major:
 *   states  [T+1, B, 2n]: states[0] = x_0 on entry, the forward fills states[1..T];  actions [T, B, na];
 *   saved   T consecutive saved streams (nb2_saved_words_per_world * B words each); NULL = no backward will follow;
 *   grad_states [T+1, B, 2n]: on entry the gradient of the loss with respect to EVERY state of the trajectory (zeros where the
 *     loss does not look); on exit grad_states[t] holds the total dL/dx_t (grad_states[0] = dL/dx_0);
 *   grad_actions [T, B, na] out.
 * One call queues the 2T kernels on `stream`; nothing returns to the host in between. */
int nb2_rollout_forward(const nb2_model* m, int B, int T, float* states, const float* actions, void* saved, int precision, void* stream);
int nb2_rollout_backward(const nb2_model* m, int B, int T, const float* states, const float* actions, const void* saved,
                         float* grad_states, float* grad_actions, int precision, void* stream);
/* per-world inertia (see nb2_step_forward_pw), constant over the horizon.  grad_inertia (may be NULL): [10*nb][B] DOUBLES, accumulated in
 * place: every step adds its fp32 dL/d(inertia) term, so the caller zeroes it first and gets the sum over the T steps — the same fp64
 * sum, in the same order (t = T-1 .. 0), that chaining the single-step backward and adding its outputs gives. */
int nb2_rollout_forward_pw(const nb2_model* m, int B, int T, float* states, const float* actions, const double* world_inertia, void* saved, int precision,
                           void* stream);
int nb2_rollout_backward_pw(const nb2_model* m, int B, int T, const float* states, const float* actions, const double* world_inertia, const void* saved,
                            float* grad_states, float* grad_actions, double* grad_inertia, int precision, void* stream);

/* T-step rollout of a world WITH collision pairs and its reverse sweep (SingleShot::getSnapshots / backpropGradientWrt as above; every step
 * is World::step with the constraint solve, and the solver's cached LCP solution x_lcp / m_lcp flows from step to step on the device as
 * BoxedLcpConstraintSolver::mX does, dart/constraint/BoxedLcpConstraintSolver.cpp:263-306).  One call queues all kernels of the horizon on
 * `stream`; nothing returns to the host in between; failures surface through status_accum (read once per rollout).
 *   states / actions / grad_states / grad_actions: as for nb2_rollout_forward / _backward (grad_states accumulates in place);
 *   x_lcp [B, NB2_MAX_ROWS] double, m_lcp [B] int32: the solver cache (in: before step 0, out: after step T-1; the backward leaves it so);
 *   tape: nb2_rollout_contact_tape_bytes(m, B, T, checkpoint_every) bytes of device memory shared by the two calls;
 *   checkpoint_every k: 0 (or >= T) keeps the saved stream + contact record of every step (~(saved_words + record) * 8 B per world-step);
 *     0 < k < T keeps only ONE segment of k steps plus an LCP-cache snapshot per segment: the reverse sweep re-runs each segment's forward
 *     from states[t0] before back-propagating through it (one extra forward per step, memory / k) — results are bit-identical either way;
 *   workspace: nb2_contact_workspace_bytes(m, B). */
size_t nb2_rollout_contact_tape_bytes(const nb2_model* m, int B, int T, int checkpoint_every);
int nb2_rollout_forward_contact(const nb2_model* m, int B, int T, float* states, const float* actions, double* x_lcp, int32_t* m_lcp, void* tape,
                                int checkpoint_every, void* workspace, int32_t* status_accum, void* stream);
int nb2_rollout_backward_contact(const nb2_model* m, int B, int T, const float* states, const float* actions, double* x_lcp, int32_t* m_lcp, void* tape,
                                 int checkpoint_every, float* grad_states, float* grad_actions, void* workspace, int32_t* status_accum, void* stream);
/* per-world inertia: as nb2_rollout_forward_pw / nb2_rollout_backward_pw (grad_inertia: fp64 sum over the horizon, also under checkpointing) */
int nb2_rollout_forward_contact_pw(const nb2_model* m, int B, int T, float* states, const float* actions, const double* world_inertia, double* x_lcp,
                                   int32_t* m_lcp, void* tape, int checkpoint_every, void* workspace, int32_t* status_accum, void* stream);
int nb2_rollout_backward_contact_pw(const nb2_model* m, int B, int T, const float* states, const float* actions, const double* world_inertia, double* x_lcp,
                                    int32_t* m_lcp, void* tape, int checkpoint_every, float* grad_states, float* grad_actions, double* grad_inertia,
                                    void* workspace, int32_t* status_accum, void* stream);

/* IKMapping: task-space outputs of a state and their VJP, on the device (neural/IKMapping.cpp:146-237 getPositionsInPlace /
 * getVelocitiesInPlace; :371-476 getPosJacobian / getVelJacobian; python/nimblephysics/mapping.py:23-114 map_to_pos / map_to_vel).
 * An entry names a body node and what to report for it, in the order IKMapping::addSpatialBodyNode / addLinearBodyNode / addAngularBodyNode
 * were called:   type 0 SPATIAL -> pos [log(R_world) ; p_world] (6), vel [omega_world ; v_world] (6)   (IKMapping.cpp:160-170, 197-205)
 *                type 1 LINEAR  -> p_world (3), v_world (3);   type 2 ANGULAR -> log(R_world) (3), omega_world (3);
 *                type 3 COM     -> Skeleton::getCOM / getCOMLinearVelocity of the tree whose root body is `body` (3, 3).
 * body[e]: the moving body of the compiled model the node is (rigidly) part of, -1 for a static node; T_owner_from_body[e]: 12 doubles
 * (R row-major, p) placing the node's frame in that body's frame (the world frame for static nodes).
 *   mapped_pos [B, nb2_ik_pos_dim], mapped_vel [B, nb2_ik_vel_dim] float (either may be NULL);
 *   nb2_ik_backward: grad_state [B, 2n] = [J_pos^T grad_pos ; J_vel^T grad_vel] — positions feed only d/dq and velocities only d/dqdot,
 *   as MapToPosLayer / MapToVelLayer return them (mapping.py:36-47, 84-95); grad_pos / grad_vel may be NULL (= zeros). */
typedef struct nb2_ik_map nb2_ik_map;
int nb2_ik_create(const nb2_model* m, int nentries, const int32_t* type, const int32_t* body, const double* T_owner_from_body, nb2_ik_map** out);
void nb2_ik_destroy(nb2_ik_map* ik);
int nb2_ik_pos_dim(const nb2_ik_map* ik);
int nb2_ik_vel_dim(const nb2_ik_map* ik);
int nb2_ik_forward(const nb2_ik_map* ik, int B, const float* state, float* mapped_pos, float* mapped_vel, void* stream);
int nb2_ik_backward(const nb2_ik_map* ik, int B, const float* state, const float* grad_pos, const float* grad_vel, float* grad_state, void* stream);

/* number of kernels this library has launched since load (bench.py reports it as gpu_launches) */
long long nb2_launch_count(void);
const char* nb2_last_error(void);
const char* nb2_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NB2_H_ */
