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
 * space (every dof). */
int nb2_forward_dynamics(const nb2_model* m, int B, const double* pos, const double* vel, const double* force, double* accel, void* stream);

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
