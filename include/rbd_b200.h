/*
 * rbd_b200.h -- C ABI of librbd_b200.so: batched rigid-body dynamics on NVIDIA H100 (sm_90a).
 *
 * This is the drop-in boundary for ONE path of RigidBodyDynamics.jl v2.5.0 (the reference):
 * dynamics!, inverse_dynamics!, mass_matrix!, dynamics_bias! evaluated over a batch of (q, v, tau) states.
 * The reference has no FFI of its own (it is 100 % Julia; SURVEY.md finding 2), so each entry point below
 * names the Julia generic function it replaces; a Julia shim (julia/RBDB200.jl, INTEGRATION.md) `ccall`s
 * these symbols, and the Python host package binds the same symbols with ctypes.
 *
 * Conventions (identical to the reference):
 *   - 6-vectors are [angular; linear]                               src/spatial/common.jl:13
 *   - joint order == q/v/tau index order == tree_joints(mechanism)  src/mechanism_state.jl:101-104
 *   - QuaternionFloating: q = [w x y z px py pz], v = body-frame twist  src/joint_types/quaternion_floating.jl:9-17
 *   - external wrenches are given in the ROOT frame, one per non-root body, and are subtracted from the
 *     Newton-Euler wrench                                            src/mechanism_algorithms.jl:428-439
 *
 * Batched array layout: every array is "rows x batch" with the BATCH INDEX FASTEST (structure of arrays):
 * element (row k, sample b) lives at ptr[k * ld + b], ld >= B.  A Julia Matrix{T}(B, n) / CuArray{T,2}(B, n)
 * has exactly this layout with ld = B.  dtype selects float / double for ALL arrays of a call.
 *
 * Pointers of the plain entry points are DEVICE pointers; work is enqueued asynchronously on `stream`
 * (a cudaStream_t cast to void*; NULL = legacy default stream).  The *_host variants take HOST pointers
 * (pinned memory recommended), stage chunks through device buffers owned by the model handle, overlap
 * H2D / kernel / D2H on internal streams and return when the results are in host memory.
 *
 * All functions return an rbd_status (0 = RBD_OK) and never throw; rbd_last_error() returns a message for
 * the calling thread's last failure.  A model handle is immutable after creation and may be shared between
 * threads; concurrent calls on the same handle must use different streams only for the plain (device-pointer)
 * entry points -- the *_host variants serialise on the handle's staging buffers.
 */
#ifndef RBD_B200_H
#define RBD_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RBD_B200_VERSION 100 /* 0.1.0 */
#define RBD_MAX_BODIES 64    /* non-root bodies (== tree joints) per model */

typedef enum rbd_status {
  RBD_OK = 0,
  RBD_EINVAL = 1,       /* NULL pointer, bad enum, malformed description (ArgumentError in the reference)      */
  RBD_EDIM = 2,         /* size mismatch (DimensionMismatch, mechanism_algorithms.jl:250-251)                  */
  RBD_ELOOP = 3,        /* mechanism has non-tree joints ("can currently only handle tree Mechanisms", :549)   */
  RBD_ESTALE = 4,       /* modcount mismatch (ModificationCountMismatch, src/util.jl:56-72)                    */
  RBD_ECUDA = 5,        /* CUDA runtime error (message in rbd_last_error)                                      */
  RBD_EUNSUPPORTED = 6, /* model too large / dtype not built -- caller must fall back to the reference itself  */
  RBD_ENOMEM = 7
} rbd_status;

/* RBD_DUAL64X6: arrays of ForwardDiff.Dual{Tag,Float64,6} = 7 contiguous doubles (value, 6 partials) per element, i.e.
 * element (row k, sample b) starts at ((k * ld + b) * 7) doubles -- the memory layout of a Julia Matrix{Dual}(B, n).
 * Supported by rbd_dynamics (tau optional, no wext / q̇ output); other entry points return RBD_EUNSUPPORTED. */
typedef enum rbd_dtype { RBD_F32 = 0, RBD_F64 = 1, RBD_DUAL64X6 = 2 } rbd_dtype;

/* Joint type codes: the eight JointTypes of src/joint_types/ (file per line). */
typedef enum rbd_joint_type {
  RBD_JOINT_REVOLUTE = 0,             /* revolute.jl             nq 1 nv 1, jparam[0:3] = unit axis            */
  RBD_JOINT_PRISMATIC = 1,            /* prismatic.jl            nq 1 nv 1, jparam[0:3] = unit axis            */
  RBD_JOINT_FIXED = 2,                /* fixed.jl                nq 0 nv 0                                     */
  RBD_JOINT_PLANAR = 3,               /* planar.jl               nq 3 nv 3, jparam = x_axis, y_axis, rot_axis  */
  RBD_JOINT_QUATERNION_FLOATING = 4,  /* quaternion_floating.jl  nq 7 nv 6                                     */
  RBD_JOINT_SPQUAT_FLOATING = 5,      /* spquat_floating.jl      nq 6 nv 6                                     */
  RBD_JOINT_QUATERNION_SPHERICAL = 6, /* quaternion_spherical.jl nq 4 nv 3                                     */
  RBD_JOINT_SINCOS_REVOLUTE = 7       /* sin_cos_revolute.jl     nq 2 nv 1, jparam[0:3] = unit axis            */
} rbd_joint_type;

/*
 * Flattened tree Mechanism, in tree_joints(mechanism) order (joint i's successor is non-root body i).
 * What the shim reads from the reference objects:
 *   parent[i]    index of the joint whose successor is predecessor(joint i), -1 if the predecessor is the
 *                root body                                   predsucc, src/mechanism_state.jl:93-94
 *   jtype[i]     joint_type(joint)                           src/joint.jl:43-67
 *   X_tree[i]    joint_to_predecessor(joint): rotation (row-major 9) then translation (3)   src/joint.jl:49,77
 *   jparam[i]    joint-type constants (axes), see rbd_joint_type
 *   inertia[i]   spatial_inertia(successor) in the frame after the joint: moment about the frame origin
 *                (row-major 9), cross_part = m*com (3), mass (1)     src/rigid_body.jl:63,
 *                src/spatial/motion_force_interaction.jl:28-37
 *   gravity      mechanism.gravitational_acceleration.v      src/mechanism.jl:10-34
 *   modcount     modcount(mechanism)                         src/util.jl:56-72
 * q/v offsets are NOT passed: they follow from the joint order and the per-type nq/nv exactly as the
 * reference's qranges/vranges do (mechanism_state.jl:101-104); rbd_model_get_info returns them for checking.
 */
typedef struct rbd_model_desc {
  int32_t nb;
  int32_t num_non_tree_joints; /* > 0  =>  RBD_ELOOP, like inverse_dynamics! */
  const int32_t* parent;       /* [nb]     */
  const int32_t* jtype;        /* [nb]     */
  const double* X_tree;        /* [nb][12] */
  const double* jparam;        /* [nb][9]  */
  const double* inertia;       /* [nb][13] */
  double gravity[3];
  int64_t modcount;
} rbd_model_desc;

typedef struct rbd_model rbd_model; /* opaque handle */

typedef struct rbd_model_info {
  int32_t nb, nq, nv;
  int32_t stash_rows;        /* shared-memory rows per sample used by the ABA kernel                       */
  int32_t max_branch_depth;  /* simultaneously open branch nodes (pending-slot count)                      */
  int32_t general_path;      /* 1 if multi-DoF joints occur away from the first root joint                 */
  int64_t modcount;
  int32_t qstart[RBD_MAX_BODIES];
  int32_t vstart[RBD_MAX_BODIES];
  int32_t eval_order[RBD_MAX_BODIES]; /* depth-first preorder used on the device: position -> joint index */
} rbd_model_info;

/* Kernel launch statistics of the most recent call on this thread (for bench.py's gpu_launches / roofline). */
typedef struct rbd_launch_info {
  int32_t kernels_launched;
  int32_t grid, block;
  int32_t smem_bytes;
  int32_t blocks_per_sm;
  float last_kernel_ms; /* only filled by the *_host variants and rbd_*_timed helpers; else 0 */
  int32_t specialised;  /* 1 if the call ran the model-specialised (run-time compiled) kernels, 0 = generic kernels */
} rbd_launch_info;

int32_t rbd_version(void);
const char* rbd_last_error(void);
const char* rbd_status_string(int32_t status);

/* Flatten-once model handle: replaces constructing MechanismState/DynamicsResult caches
 * (src/mechanism_state.jl:79-172, src/dynamics_result.jl:11-85). */
int32_t rbd_model_create(const rbd_model_desc* desc, rbd_model** out);
int32_t rbd_model_destroy(rbd_model* model);
int32_t rbd_model_get_info(const rbd_model* model, rbd_model_info* info);
/* RBD_ESTALE if `modcount` differs from the one the handle was created with (@modcountcheck, util.jl:56-72). */
int32_t rbd_model_check_modcount(const rbd_model* model, int64_t modcount);
int32_t rbd_get_launch_info(rbd_launch_info* info);

/*
 * Model-specialised kernels.  For a given handle the library can generate straight-line CUDA code for dynamics! /
 * inverse_dynamics! / dynamics_bias! / mass_matrix! of THAT mechanism (tree walk unrolled, joint classes resolved, model constants folded,
 * structural zeros removed), compile it with NVRTC for sm_90a and keep the cubin in a disk cache
 * ($RBD_JIT_CACHE, else <library dir>/jit_cache, else ~/.cache/rbd_b200).  This is the analogue of the reference compiling
 * its generic functions for a concrete MechanismState{X,M,C} on first call (Julia's JIT).
 * Entry points use a specialised kernel when its cubin is cached or the batch is at least RBD_JIT_MIN_BATCH (default 32768)
 * samples -- the first such call then pays the compilation (seconds) -- and otherwise the generic kernels; RBD_JIT=0 disables.
 * rbd_model_precompile compiles ahead of time: `what` = OR of the RBD_SPEC_* bits, `load` != 0 also loads the kernels on the
 * current device (needs a GPU; load = 0 only fills the cache and works without one).  RBD_EUNSUPPORTED if NVRTC is not
 * available or the model does not qualify (callers keep working on the generic kernels).
 */
#define RBD_SPEC_DYNAMICS 1          /* dynamics!(result, state, torques)                */
#define RBD_SPEC_DYNAMICS_QDOT 2     /* ... with the q̇ output                             */
#define RBD_SPEC_DYNAMICS_NOTAU 4    /* ... with the zero-torque default (with / without q̇) */
#define RBD_SPEC_INVERSE_DYNAMICS 8  /* inverse_dynamics!                                */
#define RBD_SPEC_DYNAMICS_BIAS 16    /* dynamics_bias!                                   */
#define RBD_SPEC_DYNAMICS_GATHER 32  /* rbd_dynamics_gather (stores to peer GPUs)        */
#define RBD_SPEC_MASS_MATRIX 64      /* mass_matrix! (both triangles)                    */
#define RBD_SPEC_MASS_MATRIX_LOWER 128 /* mass_matrix! (lower triangle, RBD_UPLO_LOWER)  */
int32_t rbd_model_precompile(rbd_model* model, int32_t dtype, int32_t what, int32_t load);

/*
 * dynamics!(result, state, torques, externalwrenches)         src/mechanism_algorithms.jl:845-864
 *   q [nq x B], v [nv x B], tau [nv x B] or NULL (zero torques, the ConstVector default),
 *   wext [6*nb x B] or NULL (row 6*i+k = component k of the root-frame wrench on body i; NullDict default)
 *   -> vd_out [nv x B]  (result.v̇), qd_out [nq x B] or NULL (result.q̇, configuration_derivative!)
 * The reference solves M v̇ = tau - c by CRBA + RNEA + Cholesky; this library evaluates the same v̇ with the
 * Articulated-Body Algorithm (equal up to rounding; tolerance in tests/test_gpu_parity.py).
 */
int32_t rbd_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                     const void* tau, const void* wext, void* vd_out, void* qd_out, void* stream);

/*
 * dynamics! on a batch SHARDED over the GPUs of one box, with the result gather fused into the kernel (SURVEY 8(e), BASELINE
 * config 5).  Every process evaluates its own B samples exactly like rbd_dynamics, but v̇ is written into the GATHERED array
 * [nv x peer_ld] of EVERY GPU: vd_peers[p] is GPU p's array (peer-mapped into this process: CUDA IPC / symmetric memory / VMM;
 * this GPU's own array is one of them) and sample b lands in column col0 + b of each.  The output store is the gather: remote
 * rows are posted writes over NVLink / NVSwitch, no collective follows, and nothing in the kernel waits for them.  The caller
 * synchronises the GPUs (a barrier after the stream has drained) before reading the gathered arrays.
 * vd_multicast: NVLS multicast mapping of the same arrays (cuMulticast* / symmetric memory's multicast pointer) or NULL; with it
 * each row is ONE multimem.st that the NVSwitch replicates to all GPUs instead of npeers stores.
 * tau may be NULL (zero torques).  fp32 / fp64; no external wrenches / q̇ in this entry point.
 */
int32_t rbd_dynamics_gather(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* tau, int32_t npeers, void* const* vd_peers, void* vd_multicast, int64_t peer_ld,
                            int64_t col0, void* stream);

/* inverse_dynamics!(torquesout, jointwrenchesout, accelerations, state, v̇, externalwrenches)
 *                                                             src/mechanism_algorithms.jl:542-553
 *   vd [nv x B] -> tau_out [nv x B] = M(q) v̇ + c(q, v, wext)  (recursive Newton-Euler). */
int32_t rbd_inverse_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                             const void* v, const void* vd, const void* wext, void* tau_out, void* stream);

/* The per-body arguments of inverse_dynamics!(torquesout, jointwrenchesout, accelerations, state, v̇, externalwrenches)
 *                                                             src/mechanism_algorithms.jl:542-553, :387-459
 *   accelerations_out [6*nb x B]: rows 6 i .. 6 i + 5 = spatial acceleration [angular; linear] of the successor of tree joint i,
 *     expressed in the ROOT frame, gravity folded in as the root's fictitious acceleration -g exactly like spatial_accelerations!;
 *   jointwrenches_out [6*nb x B]: the wrench [torque; force] transmitted by tree joint i, ROOT frame (net wrench of the subtree,
 *     joint_wrenches_and_torques!).  Either may be NULL.  vd NULL = zero accelerations (the dynamics_bias! variant), wext as usual. */
int32_t rbd_inverse_dynamics_bodies(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                    const void* vd, const void* wext, void* accelerations_out, void* jointwrenches_out, void* stream);

/* Next row of the scope table (SURVEY 8(f) rank 4): soft point contact with half-spaces -- the batched contact_dynamics!
 *                                                             src/mechanism_algorithms.jl:680-723, src/contact.jl
 * with the reference's default SoftContactModel{HuntCrossleyModel, ViscoelasticCoulombModel} (contact.jl:104-118, :130-206; HalfSpace3D :219-239):
 *   normal force  f_n = max(lambda z^n zdot + k z^n, 0),   z = penetration, zdot = penetration velocity
 *   friction      f_stick = -k x - b v_t clipped to mu f_n;  xdot = (-k x - f_t) / b   (x: tangential displacement, the
 *                 3 "additional state" entries the reference keeps per (contact point, half-space) pair)
 * The descriptor is read on the host at call time (plain host arrays). */
typedef struct rbd_contact_desc {
  int32_t npoints;              /* <= 32 */
  const int32_t* body;          /* [npoints] tree-joint index whose successor carries the point (contact_points(body))      */
  const double* location;       /* [npoints][3] point in the frame after that joint (the frame of rbd_model_desc.inertia)    */
  const double* normal_model;   /* [npoints][3] HuntCrossleyModel k, lambda, n       (hunt_crossley_hertz: 50e3, 15e3, 1.5) */
  const double* friction_model; /* [npoints][3] ViscoelasticCoulombModel mu, k, b                                           */
  int32_t nhalfspaces;          /* <= 4 */
  const double* halfspace;      /* [nhalfspaces][6] HalfSpace3D: point (3), outward normal (3, normalised here), root frame */
} rbd_contact_desc;

/*   state           [3*npoints*nhalfspaces x B] or NULL (= all zero): tangential displacement of pair (p, h) at rows
 *                   3*(p*nhalfspaces + h) .. +2.  IN/OUT: pairs that are not in contact are reset to zero, as the reference does
 *                   inside contact_dynamics! (Contact.reset!).
 *   state_deriv_out same shape or NULL: xdot (zero for pairs not in contact) -- result.contact_state_derivatives
 *   wrenches_out    [6*nb x B]: rows 6 i .. 6 i + 5 = total contact wrench [torque; force] on the successor of tree joint i in the
 *                   ROOT frame -- result.contactwrenches; add the caller's externalwrenches and pass the sum as `wext` to
 *                   rbd_dynamics, which is exactly what dynamics! does (mechanism_algorithms.jl:850-856). */
int32_t rbd_contact_dynamics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                             const rbd_contact_desc* contact, void* state, void* state_deriv_out, void* wrenches_out, void* stream);

/* Next row of the scope table (SURVEY 8(f) rank 4, second half): dynamics! for mechanisms WITH kinematic loops
 *                                                             src/mechanism_algorithms.jl:845-864, :574-673, :747-822
 * The model handle stays a TREE handle (the spanning tree, num_non_tree_joints = 0); the non-tree joints arrive per call in this
 * descriptor (plain host arrays, read on the host), in non_tree_joints(mechanism) order.  Constraint rows are concatenated in that
 * order (mechanism_state.jl:105-107).  Per loop joint:
 *   predecessor / successor   tree-joint index whose successor is that body, -1 = the root body; predecessor != successor
 *   joint_to_predecessor      frame before the joint -> predecessor body frame: rotation row-major (9), translation (3)
 *   joint_to_successor        frame after the joint  -> successor body frame, same layout (Joint.joint_to_successor)
 *   nconstraints, wrench_basis  constraint_wrench_subspace(joint_type, tf): nconstraints (0..6) columns [torque; force] in the frame
 *                             after the joint, in the reference's column order (fixed.jl:42, revolute.jl:91, prismatic.jl:96,
 *                             planar.jl:95, quaternion_spherical.jl:60, sin_cos_revolute.jl:125; 0 columns for floating joints)
 *   gains                     Baumgarte stabilisation SE3PDGains: angular k, d, linear k, d (default 100, 20, 100, 20,
 *                             mechanism_algorithms.jl:610-612); gains == NULL disables stabilisation (stabilization_gains = nothing).
 * The library derives each loop's path (TreePath predecessor -> successor) from the model's parent[]. */
#define RBD_MAX_LOOP_JOINTS 16
#define RBD_MAX_CONSTRAINTS 96
typedef struct rbd_loop_desc {
  int32_t nloops;
  const int32_t* predecessor;          /* [nloops]                        */
  const int32_t* successor;            /* [nloops]                        */
  const double* joint_to_predecessor;  /* [nloops][12]                    */
  const double* joint_to_successor;    /* [nloops][12]                    */
  const int32_t* nconstraints;         /* [nloops] 0..6                   */
  const double* wrench_basis;          /* [sum nconstraints][6]           */
  const double* gains;                 /* [nloops][4] or NULL             */
} rbd_loop_desc;

/*   q [nq x B], v [nv x B], tau [nv x B] or NULL (zero), wext [6*nb x B] or NULL (root-frame wrenches as in rbd_dynamics)
 *   -> vd_out [nv x B] (result.v̇), qd_out [nq x B] (result.q̇), lambda_out [nl x B] (result.λ), K_out [nl*nv x B]
 *      (result.constraintjacobian, entry (c, j) at row c + j*nl, column-major), k_out [nl x B] (result.constraintbias);
 *      every output except vd_out may be NULL.  nl = sum of nconstraints.
 * The reference's BLAS solve (dynamics_solve!, :747-822):  M = L L^T,  Y = K L^-T,  z = L^-1 (tau - c),  A = Y Y^T,  b = Y z + k,
 * lambda = gelsy(A, b, rcond)  (minimum-norm solution of the rank-truncated system: A is only positive SEMI-definite),
 * v̇ = M^-1 (tau - c - K^T lambda).  Here the rank of A is decided by a diagonally pivoted Cholesky factorisation A ~ P^T G G^T P
 * that stops at the first pivot with  G_ii^2 <= rcond * G_11^2, and lambda = P^T G (G^T G)^-2 G^T P b, the minimum-norm
 * least-squares solution of the truncated system (equal to gelsy's wherever the rank gap is clear).
 * rcond: 1e-10 in fp64, the reference's constant (:804).  fp32: 1e-5 (about 100 fp32 epsilons): the Schur complement left by a
 * structurally zero constraint row (three of the five rows of a planar four-bar's revolute loop joint) carries rounding of order
 * eps_32 * G_11^2 ~ 1e-7 G_11^2, which 1e-10 would keep as rank and amplify into lambda.
 * fp32 / fp64 only (RBD_DUAL64X6 -> RBD_EUNSUPPORTED); more than RBD_MAX_LOOP_JOINTS loops or RBD_MAX_CONSTRAINTS rows ->
 * RBD_EUNSUPPORTED (callers fall back to the reference); a malformed descriptor (index out of range, predecessor == successor,
 * nconstraints outside 0..6) -> RBD_EINVAL.  With nloops = 0 the result is v̇ = M^-1 (tau - c). */
int32_t rbd_dynamics_loops(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                           const void* tau, const void* wext, const rbd_loop_desc* loops,
                           void* vd_out, void* qd_out, void* lambda_out, void* K_out, void* k_out, void* stream);

/* dynamics!(result, ...) INCLUDING the by-products the reference leaves in the DynamicsResult (src/dynamics_result.jl:11-85,
 * mechanism_algorithms.jl:849-863): besides v̇ / q̇, any of  result.massmatrix (M_out [nv*nv x B], see rbd_mass_matrix),
 * result.dynamicsbias (c_out [nv x B]), result.accelerations and result.jointwrenches (see rbd_inverse_dynamics_bodies, evaluated
 * at the v̇ just computed).  NULL = not wanted.  The forward dynamics itself does not need M or c (it is the Articulated-Body
 * Algorithm), so they cost extra launches only when asked for. */
int32_t rbd_dynamics_result(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* tau, const void* wext, void* vd_out, void* qd_out, void* M_out, void* c_out,
                            void* accelerations_out, void* jointwrenches_out, void* stream);

/* Next row of the scope table (SURVEY 8(f) rank 3): first derivatives of forward dynamics, analytically -- what the reference's
 * users obtain by pushing ForwardDiff.Dual numbers through dynamics! (examples/5. Derivatives and gradients using ForwardDiff,
 * test/test_mechanism_algorithms.jl:600-675, src/caches.jl:46-64), here in ONE call for the whole Jacobian of every sample:
 *   vd_out      [nv x B]     v̇ = dynamics!(...)                     (always written; it is the linearisation point)
 *   dvd_dq_out  [nv*nv x B]  entry (i, j) at row i + j*nv:  d v̇_i / d q_j  along velocity coordinate j, i.e. the derivative of
 *                            v̇ along q̇ = velocity_to_configuration_derivative(e_j) (mechanism_state.jl:905-910).  For joints with
 *                            nq == nv whose q̇ = v (revolute, prismatic, planar in its own axes) this is d v̇ / d q itself; in general
 *                            it equals  [d v̇ / d q] * velocity_to_configuration_derivative_jacobian(state)  -- the Jacobian in
 *                            the tangent space, which is what the Munthe-Kaas integrator's local coordinates need and which does
 *                            not depend on how the rotation is extended to non-unit quaternions.
 *   dvd_dv_out  [nv*nv x B]  d v̇_i / d v_j, same layout.
 * d v̇ / d tau is M^-1: mass_matrix! gives M.  tau may be NULL (zero torques).  fp32 / fp64; no external wrenches (RBD_EUNSUPPORTED
 * is never returned for them: the argument does not exist -- use the reference's Dual path, rbd_dynamics with RBD_DUAL64X6). */
int32_t rbd_dynamics_derivatives(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                 const void* tau, void* vd_out, void* dvd_dq_out, void* dvd_dv_out, void* stream);

/* Reverse mode (SURVEY 8(f) rank 3, second half): vector-Jacobian products of dynamics! / inverse_dynamics! -- what a reference user
 * gets from reverse-mode AD over those functions (ChainRules / ReverseDiff) -- in O(n) per sample, without forming any nv x nv
 * Jacobian (csrc/rbd_adjoint.cuh has the derivation).  Per sample, ID = inverse_dynamics! (mechanism_algorithms.jl:542-553):
 *
 * rbd_dynamics_vjp: the product  ν̄^T d v̇ / d(q, v, tau, wext)  of dynamics!(result, state, tau, wext) (:845-864).
 *   inputs   q [nq x B], v [nv x B], tau [nv x B] or NULL (zero), wext [6*nb x B] or NULL (root-frame wrenches as in rbd_dynamics),
 *            vd [nv x B] = v̇, which MUST be rbd_dynamics' result for the same q, v, tau, wext (the products are evaluated at this
 *            v̇; it is not recomputed -- tau enters only through it), vd_bar [nv x B] = ν̄
 *   outputs  tau_bar   [nv x B]    μ = M^-1 ν̄
 *            v_bar     [nv x B]    -(d ID / d v)^T μ
 *            q_bar_tan [nv x B]    -(d ID / d q)^T μ along q̇ = velocity_to_configuration_derivative(e_j): row j is
 *                                  sum_i ν̄_i dvd_dq[i + j*nv] of rbd_dynamics_derivatives
 *            q_bar_cfg [nq x B]    the same covector in configuration coordinates, mapped as configuration_derivative_to_velocity_adjoint!
 *                                  does (mechanism_state.jl:912-918, joint_types/*.jl): q_bar_cfg . (N(q) u) = q_bar_tan . u for every u
 *                                  (N: q̇ = N(q) v), also at non-unit quaternions; equal to q_bar_tan for revolute / prismatic joints.
 *                                  It has no component along the radial direction of a quaternion: that derivative depends on how the
 *                                  rotation formula is extended off the unit sphere, which no gradient should depend on.
 *            wext_bar  [6*nb x B]  ν̄^T d v̇ / d wext = -(d ID / d wext)^T μ: rows 6 i .. 6 i + 5 = the ROOT-frame twist [angular; linear]
 *                                  of the successor of tree joint i under the joint velocities μ (a motion vector: its pairing with a
 *                                  wrench perturbation [torque; force] gives the change of ν̄ . v̇)
 * rbd_inverse_dynamics_vjp: the product  τ̄^T d ID / d(q, v, v̇, wext)  of inverse_dynamics!.
 *   inputs   q, v, vd = v̇ [nv x B], wext or NULL, tau_bar [nv x B] = τ̄
 *   outputs  q_bar_tan [nv x B] (d ID / d q)^T τ̄ (tangent coordinates as above), q_bar_cfg [nq x B] (mapped as above),
 *            v_bar [nv x B] (d ID / d v)^T τ̄, vd_bar [nv x B] = M τ̄, wext_bar [6*nb x B] = (d ID / d wext)^T τ̄ = MINUS the root-frame
 *            twist of each body under the joint velocities τ̄ (external wrenches are subtracted in newton_euler!, :428-439)
 * Every output may be NULL (not computed, nothing written).  q, v, vd and the adjoint input must not be NULL (RBD_EINVAL).  fp32 /
 * fp64 (RBD_DUAL64X6 -> RBD_EUNSUPPORTED); the model limits of rbd_dynamics_derivatives apply; B == 0 or nv == 0: nothing to do. */
int32_t rbd_dynamics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld,
                         const void* q, const void* v, const void* tau, const void* wext, const void* vd,
                         const void* vd_bar,
                         void* q_bar_tan, void* q_bar_cfg, void* v_bar, void* tau_bar, void* wext_bar, void* stream);
int32_t rbd_inverse_dynamics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld,
                                 const void* q, const void* v, const void* vd, const void* wext,
                                 const void* tau_bar,
                                 void* q_bar_tan, void* q_bar_cfg, void* v_bar, void* vd_bar, void* wext_bar, void* stream);

/* The triangular solves of rbd_dynamics_derivatives also exist as a model-specialised kernel (every index a constant, right-hand
 * sides in registers; generated and NVRTC-compiled like the kernels of rbd_model_precompile, same cubin cache).  It is used when
 * its cubin is cached or the batch is at least RBD_JIT_MIN_BATCH (default 4096 for this entry point); RBD_DERIV_JIT=0 / RBD_JIT=0
 * keep the generic table-driven kernel.  This call compiles it ahead of time (no GPU needed). */
int32_t rbd_model_precompile_derivatives(rbd_model* model, int32_t dtype);

/* dynamics_bias!(result, state) / dynamics_bias!(torques, biasaccelerations, wrenches, state, externalwrenches)
 *                                                             src/mechanism_algorithms.jl:484-498
 *   -> c_out [nv x B] = c(q, v, wext) = inverse_dynamics with v̇ = 0. */
int32_t rbd_dynamics_bias(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                          const void* v, const void* wext, void* c_out, void* stream);

/* mass_matrix!(M::Symmetric, state)                           src/mechanism_algorithms.jl:248-272
 *   -> M_out [nv*nv x B]: entry (i, j) of sample b at row i + j*nv (column-major like M.data); BOTH
 *   triangles are written (the reference fills the lower one and wraps it in Symmetric(:L)). */
int32_t rbd_mass_matrix(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out,
                        void* stream);

/* Same with a choice of triangle (SURVEY 8(b) "full symmetric or lower-only flagged"): RBD_UPLO_LOWER writes only the entries
 * with row >= column -- exactly what the reference's mass_matrix! fills in M.data (Symmetric(:L)) -- and leaves the rest of
 * M_out untouched: half the output bytes (Atlas: 2.7 KB instead of 5.3 KB per sample). */
#define RBD_UPLO_FULL 0
#define RBD_UPLO_LOWER 1
int32_t rbd_mass_matrix_uplo(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out,
                             int32_t uplo, void* stream);

/* Next row of the scope table (SURVEY 8(f) rank 1), the main caller of dynamics!:
 * simulate(state0, final_time, control!; dt) with the default passive / constant-torque control
 *                                                             src/simulate.jl:36-55
 * = `nsteps` steps of MuntheKaasIntegrator with the runge_kutta_4 tableau   src/ode_integrators.jl:48-55, 233-300
 *   (stages in local coordinates around the configuration at the start of the step; local_coordinates! /
 *   global_coordinates! per joint type, src/mechanism_state.jl:1057-1085).
 *   q [nq x B], v [nv x B] are updated IN PLACE; tau [nv x B] or NULL is held constant over the call. */
int32_t rbd_integrate(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                      double dt, int32_t nsteps, void* stream);

/* The same with a TIME-VARYING open-loop control -- the batched form of the `control!(torques, t, state)` closure that simulate
 * evaluates at every stage of every step (src/simulate.jl:36-55, ode_integrators.jl:262-281): the torques of stage i (0..3, at
 * times t, t + dt/2, t + dt/2, t + dt) of step s are the [nv x B] block at  tau + s * tau_step_stride + i * tau_stage_stride
 * (strides in ELEMENTS; 0 / 0 = one block held over the whole call = rbd_integrate; stage stride 0 = zero-order hold over each
 * step).  No host round trip between steps.  State-feedback controllers still call rbd_integrate once per control interval. */
int32_t rbd_integrate_schedule(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                               int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps, void* stream);

/* rbd_integrate_schedule that also RECORDS the trajectory: q_traj [(nsteps+1) x nq x B] and v_traj [(nsteps+1) x nv x B] (leading
 * dimension B inside a block) receive the initial state in block 0 and the state after step s in block s.  q / v are advanced in
 * place exactly as by rbd_integrate_schedule (bit for bit, also every recorded block).  q_traj / v_traj must not be NULL. */
int32_t rbd_integrate_trajectory(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, const void* tau,
                                 int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps,
                                 void* q_traj, void* v_traj, void* stream);

/* Reverse mode through a rollout (DESIGN 4.13): the gradient of  L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s]
 * with respect to the initial state and the torques, for the trajectory rbd_integrate_trajectory recorded with the same tau,
 * strides, dt and nsteps.  Every array has leading dimension B; tau / tau_bar are the blocks of rbd_integrate_schedule.
 *   inputs   q_traj, v_traj (the recorded trajectory), tau or NULL (zero torques), q_traj_bar [(nsteps+1) x nq x B] and
 *            v_traj_bar [(nsteps+1) x nv x B] or NULL (zero)
 *   outputs  q0_bar_tan [nv x B] (tangent coordinates, the convention of rbd_dynamics_vjp), q0_bar_cfg [nq x B] (the minimal-norm
 *            configuration covector of rbd_dynamics_vjp), v0_bar [nv x B], and tau_bar (layout of tau; needs tau), which is ADDED TO:
 *            each (step, stage) adds its gradient to its block, so a block held over several stages or steps receives the sum of
 *            theirs, and a rollout split into consecutive calls (checkpointing) accumulates exactly like one call.  Each may be NULL.
 * Per step the four stages are recomputed from the recorded state, so memory is O((nq + nv) B) beyond the trajectory.  fp32 / fp64
 * only (RBD_EUNSUPPORTED); negative strides, nsteps < 0, dt <= 0, tau_bar without tau or NULL q_traj / v_traj: RBD_EINVAL.
 * B == 0: nothing to do; nsteps == 0: q0_bar_* from q_traj_bar[0], v0_bar = v_traj_bar[0].  Mechanisms with
 * loops are not supported (the Python layer refuses them with RBD_ELOOP). */
int32_t rbd_integrate_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                          const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride, double dt, int32_t nsteps,
                          const void* q_traj_bar, const void* v_traj_bar,
                          void* q0_bar_tan, void* q0_bar_cfg, void* v0_bar, void* tau_bar, void* stream);

/* simulate for a mechanism WITH contact points (DESIGN 4.14): rbd_integrate_schedule whose dynamics at every stage is dynamics! with
 * contact -- contact_dynamics! (see rbd_contact_dynamics) and the forward dynamics on its wrenches, in one kernel -- and which also
 * integrates the contact state s, the additional state of the reference's MechanismState, with the same RK4 tableau in plain
 * Euclidean form (MuntheKaasIntegrator.step, src/ode_integrators.jl:233-300; simulate, src/simulate.jl:36-55):
 *   stage i   s_i = s0 + dt a_i ṡ_{i-1},   step   s = s0 + dt sum_i b_i ṡ_i.
 *   q [nq x B], v [nv x B], s [3*npoints*nhalfspaces x B] (layout of rbd_contact_dynamics' state; leading dimension ld) are advanced
 *   IN PLACE; tau and its strides as in rbd_integrate_schedule; no external wrenches (simulate passes none).
 * Reset semantics: the reference's contact_dynamics! resets the state of a pair that is out of contact, but its integrator
 * overwrites the state with the stage value at every stage and with the step result at the end of the step, so within simulate a
 * reset never survives.  This call therefore never resets: a pair out of contact has ṡ = 0, keeps its last integrated s (frozen,
 * not zeroed) and resumes from it when it touches again.  s persists across calls exactly as the MechanismState's does, so
 * consecutive calls equal one call of the summed steps, bit for bit.
 * q_traj [(nsteps+1) x nq x B], v_traj [(nsteps+1) x nv x B], s_traj [(nsteps+1) x ns x B] (leading dimension B): all NULL, or all
 * set (s_traj may be NULL when ns = 0) to record the trajectory as rbd_integrate_trajectory does; recording does not change the
 * result.  Descriptor checks as rbd_contact_dynamics.  dtype other than fp32 / fp64: RBD_EUNSUPPORTED; nsteps < 0, dt <= 0, negative
 * strides, s == NULL with ns > 0, or a partial set of trajectory pointers: RBD_EINVAL; B == 0: nothing to do.  Kernels per step:
 * per stage the coordinate-map kernel(s) of rbd_integrate (1 or 2) and one forward-dynamics kernel, then the finishing kernel(s) of
 * rbd_integrate (1 or 2) and, when ns > 0, one for s -- 15 for a floating-base robot when B >= 1024 and B and ld are multiples of
 * 4 (fp32) / 2 (fp64) with 16-byte aligned q and v.  Mechanisms with loops are not supported (the Python layer refuses them with RBD_ELOOP). */
int32_t rbd_integrate_contact(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, void* s, const void* tau,
                              int64_t tau_step_stride, int64_t tau_stage_stride, const rbd_contact_desc* contact, double dt, int32_t nsteps,
                              void* q_traj, void* v_traj, void* s_traj, void* stream);

/* simulate for a mechanism WITH kinematic loops (DESIGN 4.16): simulate(state, final_time; Δt, stabilization_gains) (src/simulate.jl:
 * 36-55) -- the nsteps Munthe-Kaas RK4 steps of rbd_integrate_schedule, every stage evaluating dynamics! as the reference does
 * (mechanism_algorithms.jl:845-864): contact_dynamics! first when `contact` is given, then the KKT solve of rbd_dynamics_loops with
 * the contact wrenches as the external wrenches.  `loops` as rbd_dynamics_loops (gains NULL = stabilization_gains=nothing); nloops = 0
 * is a tree rollout on the M^-1 (tau - c) path.  `contact` NULL = no contact; otherwise s is integrated, never reset and persists
 * across calls exactly as in rbd_integrate_contact.  q, v, s (leading dimension ld) are advanced IN PLACE; tau and its strides as in
 * rbd_integrate_schedule; the trajectory pointers as in rbd_integrate_contact (all NULL or all set, s_traj may be NULL when ns = 0;
 * recording does not change the result); no external wrenches.  Descriptor checks as rbd_dynamics_loops and rbd_contact_dynamics;
 * dtype other than fp32 / fp64: RBD_EUNSUPPORTED; loops == NULL, nsteps < 0, dt <= 0, negative strides, s == NULL with ns > 0, or a
 * partial set of trajectory pointers: RBD_EINVAL; B == 0: nothing to do.  Kernels per step: per stage the coordinate-map kernel(s)
 * of rbd_integrate (1 or 2) and one KKT forward-dynamics kernel (with the contact pass in it when ns > 0), then the finishing
 * kernel(s) of rbd_integrate (1 or 2) and, when ns > 0, one for s -- 14 (15 with contact) for a floating-base robot when
 * B >= 1024 and B and ld are multiples of 4 (fp32) / 2 (fp64) with 16-byte aligned q and v; 9 for an all-revolute linkage
 * below that batch size. */
int32_t rbd_integrate_loops(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, void* s,
                            const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                            const rbd_loop_desc* loops, const rbd_contact_desc* contact /* NULL = no contact */,
                            double dt, int32_t nsteps, void* q_traj, void* v_traj, void* s_traj, void* stream);

/* Closed-loop rollouts (DESIGN 4.18): any of the three rollouts above -- the tree (rbd_integrate_schedule / _trajectory), contact
 * (`contact` set, rbd_integrate_contact) or loop rollout (`loops` set, rbd_integrate_loops; with `contact` too, its contact
 * variant) -- with joint-space feedback evaluated at EVERY RK4 stage on that stage's state (q_s, v_s), as the reference's
 * simulate calls control!(τ, t, state) at every stage (src/simulate.jl:36-55).  Per DoF, with e = local_coordinates!(q_ref, q_s)
 * (q_s - q_ref for Revolute, Prismatic, Planar, SPQuatFloating; the angle difference for SinCosRevolute; the rotation vector of
 * q_ref^-1 q_s for QuaternionSpherical; the SE(3) log of q_ref^-1 q_s for QuaternionFloating) and the reference's pd(gains, e, ė)
 * = -k e - d ė (src/pdcontrol.jl:35):
 *   RBD_PD_TORQUE            τ = τ_ff - Kp e - Kd (v_s - v_ref)
 *   RBD_PD_COMPUTED_TORQUE   v̇_des = v̇_ref - Kp e - Kd (v_s - v_ref),  τ = inverse_dynamics!(q_s, v_s, v̇_des) + τ_ff
 *                            (no contact wrenches in the inverse dynamics, as in the reference's PD tests' control!)
 * then, when effort bounds are given, τ_k is clamped to [lo_k, hi_k].  τ_ff is tau with its strides, exactly as in
 * rbd_integrate_schedule (NULL = 0).  The quaternions of q_ref must be unit quaternions (they are not normalised).
 * Every device array has the dtype of the call and leading dimension ld (kp / kd with gain_ld); q_ref of step s starts at
 * s * q_ref_step_stride elements, v_ref / vd_ref at s * v_ref_step_stride (0 = held over the call).  effort_lo / effort_hi are host
 * arrays, copied to the device on every call from pageable memory: that copy is not allowed during CUDA-graph stream capture, so a
 * captured rollout must pass them as NULL.
 * Everything else -- state, contact state, trajectories, return codes -- is as in the rollout the call runs.
 * Argument errors (before any CUDA call): pd, kp, kd or q_ref NULL, an unknown mode, vd_ref in RBD_PD_TORQUE mode, negative strides,
 * gain_ld other than 0 / ld, only one of effort_lo / effort_hi, or lo > hi: RBD_EINVAL; RBD_PD_COMPUTED_TORQUE with loops (nloops
 * > 0): RBD_ELOOP (inverse_dynamics! has no kinematic loops).  Kernels per stage: PD mode launches exactly the rollout's kernels
 * (the law runs in its coordinate-map kernels, which write the stage torques the dynamics reads); computed-torque mode adds the
 * inverse dynamics (1 kernel, 2 when the fp32 specialised kernel hands samples beyond its sin / cos range to the generic one) and
 * one elementwise kernel (τ_ff, clamp). */
#define RBD_PD_TORQUE 0
#define RBD_PD_COMPUTED_TORQUE 1
typedef struct rbd_pd_desc {
  int32_t mode;                          /* RBD_PD_TORQUE or RBD_PD_COMPUTED_TORQUE */
  const void* kp; const void* kd;        /* device [nv] (gain_ld = 0, shared by the batch) or [nv x B] (gain_ld = ld) */
  int64_t gain_ld;
  const void* q_ref;                     /* device [nq x B] block per step */
  const void* v_ref;                     /* device [nv x B] block per step, NULL = 0 */
  const void* vd_ref;                    /* device [nv x B] block per step, computed-torque mode only, NULL = 0 */
  int64_t q_ref_step_stride;             /* elements between the q_ref blocks of consecutive steps; 0 = held over the call */
  int64_t v_ref_step_stride;             /* the same for v_ref and vd_ref */
  const double* effort_lo;               /* host [nv], NULL = unbounded */
  const double* effort_hi;               /* host [nv], NULL = unbounded */
} rbd_pd_desc;
int32_t rbd_integrate_pd(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, void* s, const void* tau,
                         int64_t tau_step_stride, int64_t tau_stage_stride, const rbd_pd_desc* pd,
                         const rbd_loop_desc* loops /* NULL = tree or contact rollout */,
                         const rbd_contact_desc* contact /* NULL = no contact */, double dt, int32_t nsteps, void* q_traj, void* v_traj,
                         void* s_traj, void* stream);

/* Reverse mode through a contact rollout (DESIGN 4.15): the gradient of
 *   L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s] + s_traj_bar[s] . s_traj[s]
 * with respect to the initial state (q, v, s) and the torques, for the trajectory rbd_integrate_contact recorded with the same tau,
 * strides, contact descriptor, dt and nsteps.  The conventions are rbd_integrate_vjp's: leading dimension B; s_traj / s_traj_bar
 * [(nsteps+1) x ns x B] (ns = 3 npoints nhalfspaces); the *_bar inputs may be NULL (zero); outputs q0_bar_tan, q0_bar_cfg, v0_bar,
 * s0_bar [ns x B] may be NULL; tau_bar is ADDED TO, so a rollout split into consecutive calls gives the gradients of one call, bit
 * for bit; nsteps == 0 is the identity.  The contact force law is differentiated as implemented, on the branch each pair takes (in
 * or out of contact, f_n clamped at 0, stick or slip); a point exactly on the surface gets the one-sided derivative of z^n; a pair
 * out of contact passes its s adjoint through unchanged.  No gradient reaches the contact parameters or dt.  Descriptor checks as
 * rbd_contact_dynamics; dtype other than fp32 / fp64: RBD_EUNSUPPORTED; the argument errors of rbd_integrate_vjp and s_traj == NULL
 * with ns > 0: RBD_EINVAL; B == 0: nothing to do.  Kernels per step: the recompute of rbd_integrate_contact's step without its
 * finishing kernels, 5 elementwise phases (1 or 2 kernels each, as rbd_integrate_vjp), 4 stage adjoints (one kernel each), and
 * one configuration-covector kernel between steps.  Mechanisms with loops are not supported (the Python layer refuses them with
 * RBD_ELOOP). */
int32_t rbd_integrate_contact_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                  const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                                  const rbd_contact_desc* contact, double dt, int32_t nsteps, const void* q_traj_bar,
                                  const void* v_traj_bar, const void* s_traj_bar, void* q0_bar_tan, void* q0_bar_cfg, void* v0_bar,
                                  void* s0_bar, void* tau_bar, void* stream);

/* Reverse mode through a closed-loop rollout (DESIGN 4.19): the gradient of
 *   L = sum_s q_traj_bar[s] . q_traj[s] + v_traj_bar[s] . v_traj[s] (+ s_traj_bar[s] . s_traj[s] with contact)
 * for the trajectory rbd_integrate_pd recorded with the same controller `pd`, tau and strides, contact descriptor (NULL: the tree
 * rollout), dt and nsteps, leading dimension B (gain_ld 0 or B).  Gradients reach the initial state and τ_ff (the outputs of
 * rbd_integrate_vjp / rbd_integrate_contact_vjp, same shapes and conventions, tau_bar ADDED TO) and the controller's device arrays
 * through `pd_bar` (each ADDED TO, NULL = not wanted; pd_bar NULL: none):
 *   kp, kd          [nv x B]: per-sample contributions, also for shared gains (gain_ld = 0: the caller sums over the batch, so that a
 *                   rollout split into consecutive calls gives the gradients of one call, bit for bit)
 *   q_ref           the shape of pd->q_ref ([nq x B] held, or a block per step at q_ref_step_stride); the derivative with respect
 *                   to the nq coordinates as given (the law does not normalise q_ref)
 *   v_ref, vd_ref   the shapes of pd->v_ref / pd->vd_ref
 * The saturation's derivative is zero wherever the APPLIED torque equals a bound (1[lo < τ < hi]; torch.clamp's inclusive mask
 * differs from it only where τ is exactly on a bound).  Nothing reaches the effort bounds, dt or the contact parameters.
 * Argument errors (before any CUDA call): rbd_integrate_pd's controller checks, those of rbd_integrate_vjp /
 * rbd_integrate_contact_vjp, pd == NULL, and pd_bar->v_ref / vd_ref without pd->v_ref / vd_ref: RBD_EINVAL; in computed-torque
 * mode the model limits of rbd_inverse_dynamics_vjp: RBD_EUNSUPPORTED.  There is no loop rollout here.  Kernels per step: the
 * recompute of rbd_integrate_pd's step without its finishing kernels, then as rbd_integrate_vjp (or rbd_integrate_contact_vjp)
 * -- PD mode launches exactly their kernels; computed-torque mode adds per stage one inverse-dynamics VJP and, with effort bounds,
 * one elementwise mask kernel.  The effort bounds are copied to the device once per call (from pageable memory, so a call captured
 * in a CUDA graph must have none, as in rbd_integrate_pd); the per-step recompute reuses that copy. */
typedef struct rbd_pd_bar {
  void* kp; void* kd;                    /* [nv x B] */
  void* q_ref;                           /* the shape of pd->q_ref */
  void* v_ref; void* vd_ref;             /* the shapes of pd->v_ref / pd->vd_ref */
} rbd_pd_bar;
int32_t rbd_integrate_pd_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                             const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                             const rbd_pd_desc* pd, const rbd_contact_desc* contact /* NULL = tree rollout */, double dt,
                             int32_t nsteps, const void* q_traj_bar, const void* v_traj_bar, const void* s_traj_bar, void* q0_bar_tan,
                             void* q0_bar_cfg, void* v0_bar, void* s0_bar, void* tau_bar, const rbd_pd_bar* pd_bar, void* stream);

/* Next row of the scope table (SURVEY 8(f) rank 2): kinematics by-products of the same outward sweep, all expressed in the
 * mechanism's root frame, 6-vectors as [angular; linear].  Every output pointer may be NULL (not computed).
 *   transforms_to_root  [12*nb x B]  rows 12 i .. 12 i + 11 = transform_to_root(state, successor of tree joint i):
 *                                    rotation row-major (9) then translation (3)      src/mechanism_state.jl:687-714
 *   center_of_mass      [3 x B]      center_of_mass(state)                            src/mechanism_algorithms.jl:30-49
 *   kinetic_energy      [1 x B]      kinetic_energy(state)                            src/mechanism_state.jl:886-888, 989-994
 *   gravitational_potential_energy [1 x B]                                            src/mechanism_state.jl:897-903, 996-1000
 *   momentum            [6 x B]      momentum(state)                                  src/mechanism_state.jl:878-880, 975-980
 *   momentum_rate_bias  [6 x B]      momentum_rate_bias(state)                        src/mechanism_state.jl:882-884, 982-987
 *   momentum_matrix     [6*nv x B]   momentum_matrix!(A, state): column k at rows 6 k .. 6 k + 5
 *                                                                                     src/mechanism_algorithms.jl:313-327
 *   geometric_jacobian  [6*nv x B]   geometric_jacobian!(J, state, path), same column layout; requires `path_sign`
 *                                                                                     src/mechanism_algorithms.jl:80-100 */
typedef struct rbd_kinematics_out {
  void* transforms_to_root;
  void* center_of_mass;
  void* kinetic_energy;
  void* gravitational_potential_energy;
  void* momentum;
  void* momentum_rate_bias;
  void* momentum_matrix;
  void* geometric_jacobian;
} rbd_kinematics_out;

/* q [nq x B]; v [nv x B], may be NULL when none of kinetic_energy / momentum / momentum_rate_bias is requested (RBD_EINVAL
 * otherwise).  `path_sign` is a HOST array of nb entries (tree-joint order) describing a TreePath (src/graphs/tree_path.jl):
 * +1 for joints traversed from predecessor to successor (PathDirections.down), -1 for the opposite direction (up: the
 * reference negates those columns, mechanism_algorithms.jl:95), 0 for joints not on the path; NULL iff geometric_jacobian is
 * NULL.  fp32 / fp64 only. */
int32_t rbd_kinematics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                       const int8_t* path_sign, const rbd_kinematics_out* out, void* stream);

/* Task-space kinematics (DESIGN 4.17): point Jacobians, relative transforms, twists and accelerations of chosen bodies, in any
 * body frame, for up to RBD_MAX_TASKS tasks from ONE launch.  A task is a body of interest, a base body, a point fixed in the body
 * and a frame to express results in.  The descriptor holds plain HOST arrays, read at call time like rbd_contact_desc:
 *   body[t]   tree-joint index whose successor is the target body, -1 = the root body
 *   base[t]   the source body, same encoding; the path is path(mechanism, base, body)
 *   frame[t]  body whose default frame results are expressed in, -1 = the root frame; frame == NULL: the root frame for all tasks
 *   point[t]  [3] point fixed in `body`, in the frame after its joint (the frame of rbd_model_desc.inertia, as in
 *             rbd_contact_desc.location); point == NULL: every task uses its body's origin */
#define RBD_MAX_TASKS 32
typedef struct rbd_task_desc {
  int32_t ntasks;          /* 0 .. RBD_MAX_TASKS */
  const int32_t* body;     /* [ntasks] */
  const int32_t* base;     /* [ntasks] */
  const int32_t* frame;    /* [ntasks] or NULL */
  const double* point;     /* [ntasks][3] or NULL */
} rbd_task_desc;

/* Every output may be NULL (not computed).  Task t owns rows [t*R, (t+1)*R) of each array (R = the per-task row count below), K =
 * ntasks; 6-vectors are [angular; linear].  With F the task's frame, T_X = transform_to_root(state, X) (mechanism_state.jl:687-714):
 *   transform           [12 K x B]    relative_transform(state, frame(body), frame(base)) = inv(T_base) T_body: rotation row-major
 *                                     (9), translation (3); independent of `frame`                 mechanism_state.jl:1011-1014
 *   point               [3 K x B]     the point in F: transform(state, point, F)
 *   twist               [6 K x B]     relative_twist(state, body, base) expressed in F              mechanism_state.jl:1016-1038
 *   point_velocity      [3 K x B]     velocity of the point w.r.t. base, in F = point_velocity(twist, point) = point_jacobian * v
 *   geometric_jacobian  [6 nv K x B]  geometric_jacobian!(J, state, path) with J.frame = F: column k at rows 6k .. 6k+5 of the task's
 *                                     block; joints off the path give zero columns                 mechanism_algorithms.jl:101-132
 *   point_jacobian      [3 nv K x B]  point_jacobian!(Jp, state, path, point) in F: column k at rows 3k .. 3k+2
 *                                                                                                   mechanism_algorithms.jl:154-224
 *   acceleration        [6 K x B]     relative_acceleration(accels, body, base) with accels = spatial_accelerations!(state, v̇), then
 *                                     transform(state, accel, F)          mechanism_algorithms.jl:421-426, mechanism_state.jl:1049-1056
 *   point_acceleration  [3 K x B]     point_acceleration(twist, accel, point), all three in F       spatial/spatialmotion.jl:351-363
 * The point Jacobian takes the point in the BODY's frame, constant over the batch; the reference's point_jacobian! takes it in
 * Jp.frame.  Both give the same matrix for the same physical point. */
typedef struct rbd_task_out {
  void* transform;
  void* point;
  void* twist;
  void* point_velocity;
  void* geometric_jacobian;
  void* point_jacobian;
  void* acceleration;
  void* point_acceleration;
} rbd_task_out;

/* q [nq x B]; v [nv x B], may be NULL only when none of twist / point_velocity / acceleration / point_acceleration is requested
 * (RBD_EINVAL otherwise); vd [nv x B] or NULL = zero joint accelerations.  With vd == NULL, acceleration and point_acceleration are
 * exactly the velocity-product terms J̇ v that task-space controllers need (ẍ = J v̇ + J̇ v).  Gravity is in no output: the root's
 * acceleration -g of spatial_accelerations! is common to body and base and cancels.  body == base is allowed (identity transform;
 * zero twist, Jacobians and acceleration).  Errors, all decided on the host before any CUDA call: NULL model / q / tasks / out, an
 * index outside -1 .. nb-1 or ntasks < 0: RBD_EINVAL; ntasks > RBD_MAX_TASKS or a dtype other than fp32 / fp64: RBD_EUNSUPPORTED;
 * ld < B: RBD_EDIM.  B == 0 or ntasks == 0: RBD_OK, nothing written.  One kernel launch per call.  The per-sample working set
 * (the outward sweep's pending slots plus 12 to 24 rows for every distinct body the tasks name) lives in shared memory; if it does
 * not fit a block (fp64 with several dozen distinct bodies), the call returns RBD_EUNSUPPORTED: split the tasks over two calls. */
int32_t rbd_task_kinematics(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* vd, const rbd_task_desc* tasks, const rbd_task_out* out, void* stream);

/* Reverse mode of rbd_task_kinematics (DESIGN 4.20): for the same (q, v, vd, tasks), the product  Σ_outputs ȳ . ∂y/∂(q, v, v̇)  over
 * any subset of the eight outputs.  `out_bar` reuses rbd_task_out: each member is NULL (zero cotangent) or the cotangent ȳ with
 * exactly that output's layout and leading dimension ld.  Cotangent rows of Jacobian columns off a task's path are not read (those
 * columns are structurally zero).  Outputs, each [rows x B] with leading dimension ld or NULL (not wanted), are WRITTEN, not
 * accumulated, with the conventions of rbd_dynamics_vjp:
 *   q_bar_tan [nv]  derivative along velocity_to_configuration_derivative(e_j)
 *   q_bar_cfg [nq]  q_bar_tan mapped like configuration_derivative_to_velocity_adjoint! (no radial quaternion component)
 *   v_bar [nv], vd_bar [nv]  (zero when no velocity / acceleration cotangent is given)
 * Every forward quantity is recomputed from q, v and vd; the forward outputs are not needed.  Errors, all decided on the host before
 * any CUDA call: those of rbd_task_kinematics with out_bar in place of out (the descriptor checks with the same codes; a cotangent
 * on twist / point_velocity / acceleration / point_acceleration with v == NULL: RBD_EINVAL).  B == 0: RBD_OK, nothing written;
 * ntasks == 0: RBD_OK, the requested gradients set to zero.  Otherwise one kernel launch per call, with a stream-ordered workspace
 * of 42 rows per body plus 42 per distinct body the tasks name, per resident thread (at most 512 MB). */
int32_t rbd_task_kinematics_vjp(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                                const void* vd, const rbd_task_desc* tasks, const rbd_task_out* out_bar, void* q_bar_tan,
                                void* q_bar_cfg, void* v_bar, void* vd_bar, void* stream);

/* Task-space feedback (DESIGN 4.21): the closed-loop rollouts of rbd_integrate_pd with a controller built from up to RBD_MAX_TASKS
 * tasks of an rbd_task_desc, evaluated at EVERY RK4 stage on the stage state.  Each task yields f_t in its task frame and the
 * controller adds u_task = Σ_t J_t^T f_t, with the reference's pd(gains, e, ė) = -k e - d ė (src/pdcontrol.jl:35), gains diagonal:
 *   RBD_TASK_POINT (3 rows)  x = transform(state, point, base) in base coordinates, F = frame[t]:  e = R_F<-base (x - x_ref),
 *                            ė = point_velocity in F - R_F<-base ẋ_ref,  f = -Kp e - Kd ė,  J_t = point_jacobian in F
 *   RBD_TASK_POSE  (6 rows)  the frame C with origin at point[t] and the body's axes (frame[t] must equal body[t]); x = C -> base,
 *                            T = twist of C w.r.t. base in C; e = inv(x_ref) x, ψ = rotation vector of R_e, p_e its translation:
 *                            ang = -Kω ψ - Dω (ω - ω_ref),  lin = -Kv R_e^T p_e - Dv (v - v_ref)  (SE3PDGains, SE3PDMethod{:DoubleGeodesic},
 *                            src/pdcontrol.jl:83-107), f = [ang; lin],  J_t = geometric Jacobian of C in C
 * with R = Σ_t (3 | 6) gain / velocity rows and X = Σ_t (3 | 12) target rows in task order.  x_ref of a pose task is 12 rows in the
 * layout of rbd_task_kinematics' transform (rotation row-major, translation); its rotation must be orthonormal (it is not
 * re-orthonormalised).  Modes, with the optional joint-space term J = rbd_integrate_pd's law of `joint` (same mode):
 *   RBD_PD_TORQUE            τ = τ_ff + J + u_task
 *   RBD_PD_COMPUTED_TORQUE   v̇_des = J (with its v̇_ref) + u_task,  τ = inverse_dynamics!(q_s, v_s, v̇_des) + τ_ff
 * then the effort bounds clamp the sum once.  kp / kd: device [R] (gain_ld 0) or [R x B] (gain_ld = ld); x_ref [X x B] and xd_ref
 * [R x B] (NULL = 0) with leading dimension ld, the block of step s at s * step stride (0 = held over the call).  Everything else is
 * rbd_integrate_pd's, with `ctrl` in place of `pd`.  Argument errors (before any CUDA call): JointPD's checks on `joint` and the
 * descriptor checks of rbd_task_kinematics, with their codes; ctrl NULL, an unknown mode or kind, kind / kp / kd / x_ref NULL with
 * tasks, a pose task with frame != body, negative strides, gain_ld other than 0 / ld, a joint term whose mode differs or that has its
 * own effort bounds, only one of effort_lo / effort_hi, or lo > hi: RBD_EINVAL; RBD_PD_COMPUTED_TORQUE with loops: RBD_ELOOP.  When
 * the per-sample working set does not fit a block (as rbd_task_kinematics): RBD_EUNSUPPORTED, before any kernel.  Kernels per
 * stage: rbd_integrate_pd's with this controller's joint term (the open-loop rollout's without one), plus one task kernel. */
#define RBD_TASK_POINT 0
#define RBD_TASK_POSE 1
typedef struct rbd_task_pd_desc {
  int32_t mode;                          /* RBD_PD_TORQUE or RBD_PD_COMPUTED_TORQUE */
  rbd_task_desc tasks;                   /* host arrays; frame[t] == body[t] for pose tasks */
  const int32_t* kind;                   /* host [ntasks]: RBD_TASK_POINT / RBD_TASK_POSE */
  const void* kp; const void* kd;        /* device [R] (gain_ld 0) or [R x B] (gain_ld = ld) */
  int64_t gain_ld;
  const void* x_ref;                     /* device [X x B] block per step */
  int64_t x_ref_step_stride;             /* elements between the x_ref blocks of consecutive steps; 0 = held */
  const void* xd_ref;                    /* device [R x B] block per step, NULL = 0 */
  int64_t xd_ref_step_stride;
  const rbd_pd_desc* joint;              /* NULL = no joint-space term; same mode; its effort bounds NULL */
  const double* effort_lo;               /* host [nv], NULL = unbounded; clamp the sum */
  const double* effort_hi;
} rbd_task_pd_desc;
int32_t rbd_integrate_task_pd(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, void* q, void* v, void* s, const void* tau,
                              int64_t tau_step_stride, int64_t tau_stage_stride, const rbd_task_pd_desc* ctrl,
                              const rbd_loop_desc* loops /* NULL = tree or contact rollout */,
                              const rbd_contact_desc* contact /* NULL = no contact */, double dt, int32_t nsteps, void* q_traj,
                              void* v_traj, void* s_traj, void* stream);
/* The law of rbd_integrate_task_pd at one state (q, v) with the references of step `step`: tau_out [nv x B] = the torques the
 * rollout applies at a stage with that state (τ_ff = tau_ff, NULL = 0), every array with leading dimension ld.  The argument errors
 * of rbd_integrate_task_pd (step < 0: RBD_EINVAL); B == 0: nothing to do.  Kernels: one in RBD_PD_TORQUE mode; in computed-torque
 * mode the task kernel, the inverse dynamics and one elementwise kernel. */
int32_t rbd_task_pd_torques(const rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                            const void* tau_ff, const rbd_task_pd_desc* ctrl, int32_t step, void* tau_out, void* stream);

/* Reverse mode through a task-space closed-loop rollout (DESIGN 4.22): rbd_integrate_pd_vjp for the trajectory
 * rbd_integrate_task_pd recorded with the controller `ctrl` (tree or contact rollout, leading dimension B, gain_ld 0 or B).  Gradients
 * reach the initial state and τ_ff as there, and the controller's device arrays through `ctrl_bar` (each ADDED TO, NULL = not wanted;
 * ctrl_bar NULL: none):
 *   kp, kd          [R x B]: per-sample contributions, also for shared gains (the caller sums over the batch)
 *   x_ref, xd_ref   the shapes of ctrl->x_ref / ctrl->xd_ref; a pose target's 12 entries as given (the law does not re-orthonormalise)
 *   joint           the joint term's adjoints, as rbd_integrate_pd_vjp's pd_bar (needs ctrl->joint)
 * The saturation's derivative is rbd_integrate_pd_vjp's.  Nothing reaches the task points, the effort bounds, dt or the contact
 * parameters.  Argument errors (before any CUDA call): rbd_integrate_task_pd's controller checks, those of rbd_integrate_pd_vjp, a bar
 * without its array (xd_ref, joint, and the joint term's v_ref / vd_ref): RBD_EINVAL; in computed-torque mode the model limits of
 * rbd_inverse_dynamics_vjp: RBD_EUNSUPPORTED.  There is no loop rollout here.  Kernels per step: the recompute of
 * rbd_integrate_task_pd's step without its finishing kernels, then as rbd_integrate_pd_vjp with this controller's joint term
 * (rbd_integrate_vjp / rbd_integrate_contact_vjp without one), plus per stage one task-law adjoint kernel and, in torque mode with
 * effort bounds, one elementwise mask kernel. */
typedef struct rbd_task_pd_bar {
  void* kp; void* kd;                    /* [R x B] */
  void* x_ref; void* xd_ref;             /* the shapes of ctrl->x_ref / ctrl->xd_ref */
  const rbd_pd_bar* joint;               /* the joint term's, NULL = not wanted */
} rbd_task_pd_bar;
int32_t rbd_integrate_task_pd_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q_traj, const void* v_traj,
                                  const void* s_traj, const void* tau, int64_t tau_step_stride, int64_t tau_stage_stride,
                                  const rbd_task_pd_desc* ctrl, const rbd_contact_desc* contact /* NULL = tree rollout */, double dt,
                                  int32_t nsteps, const void* q_traj_bar, const void* v_traj_bar, const void* s_traj_bar,
                                  void* q0_bar_tan, void* q0_bar_cfg, void* v0_bar, void* s0_bar, void* tau_bar,
                                  const rbd_task_pd_bar* ctrl_bar, void* stream);
/* The adjoint of rbd_task_pd_torques at one state, every array [rows x B] (gain_ld 0 or B): for the cotangent tau_out_bar of the
 * torques, q_bar_tan [nv x B], q_bar_cfg [nq x B] (rbd_dynamics_vjp's conventions), v_bar [nv x B] and tau_ff_bar [nv x B] are
 * WRITTEN (each may be NULL), the controller's bars ADDED TO as in rbd_integrate_task_pd_vjp.  The saturation's derivative is
 * rbd_integrate_pd_vjp's.  Argument errors: those of rbd_task_pd_torques (leading dimension B), tau_ff_bar without tau_ff, a bar
 * without its array: RBD_EINVAL; in computed-torque mode the model limits of rbd_inverse_dynamics_vjp: RBD_EUNSUPPORTED; all before
 * any CUDA call.  Kernels: with effort bounds or in computed-torque mode the forward law first (rbd_task_pd_torques' kernels) and,
 * with bounds, one mask kernel; in computed-torque mode one inverse-dynamics VJP; then one task-adjoint kernel (the joint term's
 * adjoint in the same pass) and, when q_bar_tan or q_bar_cfg is wanted, one elementwise kernel. */
int32_t rbd_task_pd_torques_vjp(const rbd_model* model, int32_t dtype, int64_t B, const void* q, const void* v, const void* tau_ff,
                                const rbd_task_pd_desc* ctrl, int32_t step, const void* tau_out_bar, void* q_bar_tan, void* q_bar_cfg,
                                void* v_bar, void* tau_ff_bar, const rbd_task_pd_bar* ctrl_bar, void* stream);

/* Host-pointer variants: same semantics, host buffers in, host buffers out, copies inside the call. */
int32_t rbd_dynamics_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, const void* v,
                          const void* tau, const void* wext, void* vd_out, void* qd_out);
int32_t rbd_inverse_dynamics_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                                  const void* v, const void* vd, const void* wext, void* tau_out);
int32_t rbd_dynamics_bias_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q,
                               const void* v, const void* wext, void* c_out);
int32_t rbd_mass_matrix_host(rbd_model* model, int32_t dtype, int64_t B, int64_t ld, const void* q, void* M_out);

#ifdef __cplusplus
}
#endif
#endif /* RBD_B200_H */
