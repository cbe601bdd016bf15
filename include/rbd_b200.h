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
