# RBDB200.jl -- Julia shim over librbd_b200.so (C ABI in include/rbd_b200.h).
#
# UNTESTED: never executed (the build image has no Julia); it is the binding a RigidBodyDynamics.jl maintainer would add and
# must be run against the reference's test-suite before use.
# It keeps the reference's user-facing types: a reference `Mechanism` is flattened ONCE into an `rbd_model_desc`, and batched
# methods with the reference's names (`dynamics!`, `inverse_dynamics!`, `mass_matrix!`, `dynamics_bias!`) `ccall` the
# library.  Everything the GPU path does not cover (mechanisms with loops or contact points, scalar types other than
# Float32/Float64, additional state) is dispatched to the reference's own methods unchanged.
module RBDB200

using RigidBodyDynamics
using RigidBodyDynamics: Mechanism, Joint, JointType, Revolute, Prismatic, Fixed, Planar, QuaternionFloating,
    SPQuatFloating, QuaternionSpherical, SinCosRevolute, tree_joints, non_tree_joints, predecessor, successor,
    joint_to_predecessor, joint_type, spatial_inertia, root_body, num_positions, num_velocities, modcount,
    frame_after, fixed_transform, rotation, translation, transform, MechanismState, DynamicsResult,
    set_configuration!, set_velocity!
using StaticArrays
using CUDA   # CuArray provides device pointers; any device-pointer provider works

const librbd = get(ENV, "RBD_B200_LIB", "librbd_b200.so")

# ---- mirror of the C declarations (include/rbd_b200.h) ----------------------------------------------------------
const RBD_OK, RBD_EINVAL, RBD_EDIM, RBD_ELOOP, RBD_ESTALE, RBD_ECUDA, RBD_EUNSUPPORTED, RBD_ENOMEM = Int32.(0:7)
const RBD_F32, RBD_F64 = Int32(0), Int32(1)

struct rbd_model_desc
    nb::Int32
    num_non_tree_joints::Int32
    parent::Ptr{Int32}
    jtype::Ptr{Int32}
    X_tree::Ptr{Float64}
    jparam::Ptr{Float64}
    inertia::Ptr{Float64}
    gravity::NTuple{3, Float64}
    modcount::Int64
end

joint_code(::Revolute) = Int32(0);            joint_code(::Prismatic) = Int32(1)
joint_code(::Fixed) = Int32(2);               joint_code(::Planar) = Int32(3)
joint_code(::QuaternionFloating) = Int32(4);  joint_code(::SPQuatFloating) = Int32(5)
joint_code(::QuaternionSpherical) = Int32(6); joint_code(::SinCosRevolute) = Int32(7)

joint_params(jt::Union{Revolute, Prismatic, SinCosRevolute}) = vcat(Vector(jt.axis), zeros(6))
joint_params(jt::Planar) = vcat(Vector(jt.x_axis), Vector(jt.y_axis), Vector(jt.rot_axis))
joint_params(::JointType) = zeros(9)

function last_error()
    unsafe_string(ccall((:rbd_last_error, librbd), Cstring, ()))
end

"Thrown for RBD_EUNSUPPORTED / RBD_ELOOP: the batched methods catch it and run the reference's own methods sample by sample."
struct FallbackToReference <: Exception
    status::Int32
    msg::String
end

"Convert an rbd_status into the exception type the reference would have thrown (INTEGRATION.md, 'Errors')."
function check(status::Int32)
    status == RBD_OK && return nothing
    msg = last_error()
    status == RBD_EDIM && throw(DimensionMismatch(msg))
    status == RBD_EINVAL && throw(ArgumentError(msg))
    status == RBD_ESTALE && throw(RigidBodyDynamics.ModificationCountMismatch(msg))
    (status == RBD_EUNSUPPORTED || status == RBD_ELOOP) && throw(FallbackToReference(status, msg))
    error("rbd_b200 (status $status): $msg")
end

"""
The documented fallback: evaluate `f!(result, state, b)` with the reference's own `MechanismState` / `DynamicsResult` for every
sample b of the batch on the host (slow, but it keeps the shim a drop-in for mechanisms / scalar types the GPU path refuses).
`pull(state, b)` sets the single-sample state from row b; `push(result, b)` stores the result into the batched output.
"""
function reference_fallback(f!, mechanism::Mechanism, B::Integer, pull, push)
    state = MechanismState(mechanism)
    result = DynamicsResult(mechanism)
    for b in 1:B
        pull(state, b)
        f!(result, state, b)
        push(result, b)
    end
end

# ---- flatten-once model handle ---------------------------------------------------------------------------------
mutable struct Model
    handle::Ptr{Cvoid}
    mechanism::Mechanism
    modcount::Int
    nq::Int
    nv::Int
    nb::Int
end

"""
    Model(mechanism)

Flatten a tree `Mechanism{Float64}` (src/mechanism.jl:10-34) into the arrays of `rbd_model_desc`, in `tree_joints` order.
"""
function Model(mechanism::Mechanism{Float64})
    joints = collect(tree_joints(mechanism))
    nb = length(joints)
    succ_index = Dict(successor(j, mechanism) => i - 1 for (i, j) in enumerate(joints))
    parent = Int32[predecessor(j, mechanism) == root_body(mechanism) ? -1 : succ_index[predecessor(j, mechanism)] for j in joints]
    jtype = Int32[joint_code(joint_type(j)) for j in joints]
    X = zeros(12, nb); P = zeros(9, nb); I = zeros(13, nb)
    for (i, j) in enumerate(joints)
        T = joint_to_predecessor(j)                       # src/joint.jl:77
        R = rotation(T); p = translation(T)
        X[1:9, i] = vec(permutedims(Matrix(R)))           # row-major rotation
        X[10:12, i] = p
        P[:, i] = joint_params(joint_type(j))
        # The library wants the inertia in frame_after(joint).  That is where spatial_inertia(body) lives after
        # canonicalize_frame_definitions! / for URDF-parsed mechanisms, but a body attached with a `successor_pose` keeps its own
        # frame (mechanism_modification.jl:21-46): transform explicitly instead of assuming.
        body = successor(j, mechanism)
        inertia = spatial_inertia(body)
        if inertia.frame != frame_after(j)
            inertia = transform(inertia, fixed_transform(body, inertia.frame, frame_after(j)))
        end
        I[1:9, i] = vec(permutedims(Matrix(inertia.moment)))
        I[10:12, i] = inertia.cross_part
        I[13, i] = inertia.mass
    end
    g = mechanism.gravitational_acceleration.v
    handle = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve parent jtype X P I begin
        desc = rbd_model_desc(nb, length(non_tree_joints(mechanism)), pointer(parent), pointer(jtype), pointer(X),
                              pointer(P), pointer(I), (g[1], g[2], g[3]), modcount(mechanism))
        check(ccall((:rbd_model_create, librbd), Int32, (Ref{rbd_model_desc}, Ref{Ptr{Cvoid}}), desc, handle))
    end
    m = Model(handle[], mechanism, modcount(mechanism), num_positions(mechanism), num_velocities(mechanism), nb)
    finalizer(x -> ccall((:rbd_model_destroy, librbd), Int32, (Ptr{Cvoid},), x.handle), m)
    m
end

# ---- batched state / result: Matrix{T}(B, n) == rows x batch with the batch index fastest ------------------------
struct BatchedState{T, A <: AbstractMatrix{T}}
    model::Model
    q::A        # B x nq
    v::A        # B x nv
end
struct BatchedResult{T, A <: AbstractMatrix{T}}
    v̇::A        # B x nv
    q̇::A        # B x nq
    massmatrix::A   # B x nv^2
    dynamicsbias::A # B x nv
end

dtype_code(::Type{Float32}) = RBD_F32
dtype_code(::Type{Float64}) = RBD_F64
devptr(x::CuArray) = reinterpret(Ptr{Cvoid}, pointer(x))
devptr(::Nothing) = C_NULL
stream_ptr() = reinterpret(Ptr{Cvoid}, CUDA.stream().handle)

function checkstate(s::BatchedState)
    check(ccall((:rbd_model_check_modcount, librbd), Int32, (Ptr{Cvoid}, Int64), s.model.handle, modcount(s.model.mechanism)))
end

"""
`dynamics!(result, state, torques, externalwrenches)` -- src/mechanism_algorithms.jl:845-864, batched.  `byproducts = true` also
fills `result.massmatrix` and `result.dynamicsbias` like the reference does (`rbd_dynamics_result`); the Articulated-Body kernel
does not need them, so they are opt-in.
"""
function RigidBodyDynamics.dynamics!(result::BatchedResult{T}, state::BatchedState{T}, torques = nothing,
                                     externalwrenches = nothing; byproducts::Bool = false) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    try
        GC.@preserve result state torques externalwrenches begin
            check(ccall((:rbd_dynamics_result, librbd), Int32,
                        (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
                         Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                        state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), devptr(torques),
                        devptr(externalwrenches), devptr(result.v̇), devptr(result.q̇),
                        byproducts ? devptr(result.massmatrix) : C_NULL, byproducts ? devptr(result.dynamicsbias) : C_NULL,
                        C_NULL, C_NULL, stream_ptr()))
        end
    catch e
        e isa FallbackToReference || rethrow()
        # mechanisms / dtypes the GPU path refuses: the reference's own dynamics!, one sample at a time, on the host
        q, v = Array(state.q), Array(state.v)
        τ = torques === nothing ? nothing : Array(torques)
        v̇ = similar(v); q̇ = similar(q)
        reference_fallback(state.model.mechanism, B,
            (s, b) -> (set_configuration!(s, view(q, b, :)); set_velocity!(s, view(v, b, :))),
            (r, b) -> (v̇[b, :] .= r.v̇; q̇[b, :] .= r.q̇)) do r, s, b
            τ === nothing ? RigidBodyDynamics.dynamics!(r, s) : RigidBodyDynamics.dynamics!(r, s, τ[b, :])
        end
        copyto!(result.v̇, v̇); copyto!(result.q̇, q̇)
    end
    result
end

"`inverse_dynamics!(torquesout, ..., state, v̇, externalwrenches)` -- src/mechanism_algorithms.jl:542-553, batched."
function RigidBodyDynamics.inverse_dynamics!(torquesout::AbstractMatrix{T}, state::BatchedState{T}, v̇::AbstractMatrix{T},
                                             externalwrenches = nothing) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    size(torquesout) == (B, state.model.nv) || throw(DimensionMismatch("torquesout has wrong size"))
    GC.@preserve torquesout state v̇ externalwrenches begin
        check(ccall((:rbd_inverse_dynamics, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), devptr(v̇),
                    devptr(externalwrenches), devptr(torquesout), stream_ptr()))
    end
    torquesout
end

"`dynamics_bias!(result, state)` -- src/mechanism_algorithms.jl:484-498, batched."
function RigidBodyDynamics.dynamics_bias!(result::BatchedResult{T}, state::BatchedState{T},
                                          externalwrenches = nothing) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    GC.@preserve result state externalwrenches begin
        check(ccall((:rbd_dynamics_bias, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), devptr(externalwrenches),
                    devptr(result.dynamicsbias), stream_ptr()))
    end
    result.dynamicsbias
end

"""
`mass_matrix!(M, state)` -- src/mechanism_algorithms.jl:248-272, batched: `M` is B x nv^2, entry (i, j) in column i + (j-1) nv.
`uplo = :L` writes only the lower triangle, which is all the reference's `Symmetric(:L)` storage holds (half the bytes).
"""
function RigidBodyDynamics.mass_matrix!(M::AbstractMatrix{T}, state::BatchedState{T}; uplo::Symbol = :full) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    size(M) == (B, state.model.nv^2) || throw(DimensionMismatch("mass matrix has wrong size"))
    uplo in (:full, :L) || throw(ArgumentError("uplo must be :full or :L"))     # mechanism_algorithms.jl:251
    GC.@preserve M state begin
        check(ccall((:rbd_mass_matrix_uplo, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Int32, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(M), Int32(uplo == :L ? 1 : 0), stream_ptr()))
    end
    M
end

"Per-body outputs of `inverse_dynamics!` (`jointwrenchesout`, `accelerations`), B x 6nb each, root frame (`rbd_inverse_dynamics_bodies`)."
function inverse_dynamics_bodies!(jointwrenchesout, accelerations, state::BatchedState{T}, v̇, externalwrenches = nothing) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    GC.@preserve jointwrenchesout accelerations state v̇ externalwrenches begin
        check(ccall((:rbd_inverse_dynamics_bodies, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), devptr(v̇), devptr(externalwrenches),
                    devptr(accelerations), devptr(jointwrenchesout), stream_ptr()))
    end
    nothing
end

"""
Generate + NVRTC-compile the model-specialised kernels ahead of the first large call (`rbd_model_precompile`).  `what` = OR of the
RBD_SPEC_* bits of include/rbd_b200.h: 1 dynamics!, 2 ... with q̇, 4 zero-torque variants, 8 inverse_dynamics!, 16 dynamics_bias!,
32 multi-GPU gather, 64 mass_matrix! (both triangles), 128 mass_matrix! (lower triangle).
"""
precompile_kernels(model::Model, ::Type{T} = Float32; what::Integer = 31 | 64 | 128, load::Bool = true) where {T} =
    check(ccall((:rbd_model_precompile, librbd), Int32, (Ptr{Cvoid}, Int32, Int32, Int32), model.handle, dtype_code(T), Int32(what), Int32(load)))


# ---- SURVEY 8(f) rank 1 / rank 2: the callers and by-products either side of the path -----------------------------------

"`simulate(state, final_time; Δt)` with passive / constant-torque control (src/simulate.jl:36-55), whole batch on the GPU."
function RigidBodyDynamics.simulate(state::BatchedState{T}, final_time, torques = nothing; Δt = 1e-4) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    nsteps = 0; t = 0.0
    while t < final_time; t += Δt; nsteps += 1; end            # the reference's `while t < final_time` (ode_integrators.jl:311)
    GC.@preserve state torques begin
        check(ccall((:rbd_integrate, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Float64, Int32, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v),
                    torques === nothing ? C_NULL : devptr(torques), Float64(Δt), Int32(nsteps), stream_ptr()))
    end
    nsteps
end

"Mirror of `rbd_pd_desc` (include/rbd_b200.h)."
struct rbd_pd_desc
    mode::Int32
    kp::Ptr{Cvoid}
    kd::Ptr{Cvoid}
    gain_ld::Int64
    q_ref::Ptr{Cvoid}
    v_ref::Ptr{Cvoid}
    vd_ref::Ptr{Cvoid}
    q_ref_step_stride::Int64
    v_ref_step_stride::Int64
    effort_lo::Ptr{Float64}
    effort_hi::Ptr{Float64}
end

"""
`simulate` with joint-space feedback evaluated at every RK4 stage (rbd_integrate_pd, DESIGN 4.18): the `control!` of the
reference's PD tests, batched.  `kp`, `kd`: gains per velocity DoF, a vector (shared) or a B × nv matrix (per sample); `q_ref`
(B × nq, unit quaternions), `v_ref` / `v̇_ref` (B × nv, `nothing` = 0) held over the call; `computed_torque = true` gives
τ = inverse_dynamics!(q, v, v̇_ref - kp e - kd (v - v_ref)) + torques, otherwise τ = torques - kp e - kd (v - v_ref); `effort_bounds`
(a pair of nv-vectors, e.g. from `effort_bounds(joint)` of every tree joint) clamps τ.  Tree mechanisms without contact points.
(Not run here: no Julia installation is available to the project's tests; the Python binding exercises the same entry point.)
"""
function simulate_pd(state::BatchedState{T}, final_time, kp, kd, q_ref; v_ref = nothing, v̇_ref = nothing,
                     computed_torque::Bool = false, effort_bounds = nothing, torques = nothing, Δt = 1e-4) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    nsteps = 0; t = 0.0
    while t < final_time; t += Δt; nsteps += 1; end            # the reference's `while t < final_time` (ode_integrators.jl:311)
    lo, hi = effort_bounds === nothing ? (nothing, nothing) : (Vector{Float64}(effort_bounds[1]), Vector{Float64}(effort_bounds[2]))
    ptr(x) = x === nothing ? C_NULL : devptr(x)
    GC.@preserve state kp kd q_ref v_ref v̇_ref torques lo hi begin
        desc = rbd_pd_desc(Int32(computed_torque ? 1 : 0), devptr(kp), devptr(kd), ndims(kp) == 2 ? Int64(B) : Int64(0),
                           devptr(q_ref), ptr(v_ref), ptr(v̇_ref), 0, 0,
                           lo === nothing ? Ptr{Float64}(C_NULL) : pointer(lo), hi === nothing ? Ptr{Float64}(C_NULL) : pointer(hi))
        check(ccall((:rbd_integrate_pd, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ref{rbd_pd_desc},
                     Ptr{Cvoid}, Ptr{Cvoid}, Float64, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), C_NULL, ptr(torques), 0, 0, desc,
                    C_NULL, C_NULL, Float64(Δt), Int32(nsteps), C_NULL, C_NULL, C_NULL, stream_ptr()))
    end
    nsteps
end

"Mirror of `rbd_kinematics_out` (include/rbd_b200.h): eight device pointers, C_NULL = not requested."
struct rbd_kinematics_out
    transforms_to_root::Ptr{Cvoid}
    center_of_mass::Ptr{Cvoid}
    kinetic_energy::Ptr{Cvoid}
    gravitational_potential_energy::Ptr{Cvoid}
    momentum::Ptr{Cvoid}
    momentum_rate_bias::Ptr{Cvoid}
    momentum_matrix::Ptr{Cvoid}
    geometric_jacobian::Ptr{Cvoid}
end

"+1 / -1 / 0 per tree joint for a `TreePath` (src/graphs/tree_path.jl): down / up (column negated, mechanism_algorithms.jl:95) / absent."
function path_signs(model::Model, p::RigidBodyDynamics.TreePath)
    sign = zeros(Int8, model.nb)
    index = Dict(j => i for (i, j) in enumerate(tree_joints(model.mechanism)))
    for (joint, dir) in zip(p.edges, RigidBodyDynamics.Graphs.directions(p))
        sign[index[joint]] = dir == RigidBodyDynamics.Graphs.PathDirections.up ? Int8(-1) : Int8(1)
    end
    sign
end

"""
One launch of `rbd_kinematics`; every keyword is an optional B x rows output matrix (root frame, [angular; linear]):
`transforms_to_root` (12 nb), `center_of_mass` (3), `kinetic_energy` (1), `gravitational_potential_energy` (1), `momentum` (6),
`momentum_rate_bias` (6), `momentum_matrix` (6 nv), `geometric_jacobian` (6 nv, needs `path`).  The reference's single-output
names (`center_of_mass(state)`, `momentum_matrix!(A, state)`, `geometric_jacobian!(J, state, path)` ...) are one-line methods
over this.  src/mechanism_algorithms.jl:30-49, 80-100, 313-327; src/mechanism_state.jl:878-903, 975-1000.
"""
function kinematics!(state::BatchedState{T}; path = nothing, outs...) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    ptr(name) = haskey(outs, name) ? devptr(outs[name]) : C_NULL
    ko = rbd_kinematics_out(ptr(:transforms_to_root), ptr(:center_of_mass), ptr(:kinetic_energy),
                            ptr(:gravitational_potential_energy), ptr(:momentum), ptr(:momentum_rate_bias),
                            ptr(:momentum_matrix), ptr(:geometric_jacobian))
    sign = path === nothing ? nothing : path_signs(state.model, path)
    GC.@preserve state outs sign begin
        check(ccall((:rbd_kinematics, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Int8}, Ref{rbd_kinematics_out}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v),
                    sign === nothing ? C_NULL : pointer(sign), ko, stream_ptr()))
    end
    outs
end

RigidBodyDynamics.momentum_matrix!(A::AbstractMatrix, state::BatchedState) = (kinematics!(state; momentum_matrix = A); A)
RigidBodyDynamics.geometric_jacobian!(J::AbstractMatrix, state::BatchedState, p::RigidBodyDynamics.TreePath) =
    (kinematics!(state; path = p, geometric_jacobian = J); J)

"Mirror of `rbd_task_desc` (include/rbd_b200.h): host arrays, read during the call."
struct rbd_task_desc
    ntasks::Int32
    body::Ptr{Int32}
    base::Ptr{Int32}
    frame::Ptr{Int32}
    point::Ptr{Float64}
end

"Mirror of `rbd_task_out`: eight device pointers, C_NULL = not requested."
struct rbd_task_out
    transform::Ptr{Cvoid}
    point::Ptr{Cvoid}
    twist::Ptr{Cvoid}
    point_velocity::Ptr{Cvoid}
    geometric_jacobian::Ptr{Cvoid}
    point_jacobian::Ptr{Cvoid}
    acceleration::Ptr{Cvoid}
    point_acceleration::Ptr{Cvoid}
end

"Tree-joint index whose successor is `body`, -1 for the root body (the encoding of `rbd_task_desc`)."
function body_index(model::Model, body::RigidBody)
    body == root_body(model.mechanism) && return Int32(-1)
    for (i, j) in enumerate(tree_joints(model.mechanism))
        successor(j, model.mechanism) == body && return Int32(i - 1)
    end
    throw(ArgumentError("body $(body) is not part of the mechanism"))
end

"""
    task_kinematics!(state, tasks; vd = nothing, outs...)

One launch of `rbd_task_kinematics` for up to 32 tasks `(body, base, point, frame)`: `body`, `base` are `RigidBody`s, `point` is a
3-vector in the frame after `body`'s joint (`nothing` = its origin), `frame` is the `RigidBody` whose default frame results are
expressed in (`nothing` = the root frame).  Every keyword is an optional B x rows device matrix, task t owning rows
t*R+1 .. (t+1)*R: `transform` (12, `relative_transform`), `point` (3), `twist` (6, `relative_twist`), `point_velocity` (3),
`geometric_jacobian` (6 nv, `geometric_jacobian!` with J.frame = frame), `point_jacobian` (3 nv, `point_jacobian!`),
`acceleration` (6, `relative_acceleration` transformed to the frame) and `point_acceleration` (3).  `vd = nothing` gives the
velocity-product terms J̇ v.  src/mechanism_algorithms.jl:101-224, 421-426; src/mechanism_state.jl:1011-1056;
src/spatial/spatialmotion.jl:346-401.
"""
function task_kinematics!(state::BatchedState{T}, tasks; vd = nothing, outs...) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    model = state.model
    body = Int32[body_index(model, t[1]) for t in tasks]
    base = Int32[body_index(model, t[2]) for t in tasks]
    frame = Int32[t[4] === nothing ? Int32(-1) : body_index(model, t[4]) for t in tasks]
    point = zeros(Float64, 3, length(tasks))
    for (k, t) in enumerate(tasks)
        t[3] === nothing || (point[:, k] .= t[3])
    end
    ptr(name) = haskey(outs, name) ? devptr(outs[name]) : C_NULL
    to = rbd_task_out(ptr(:transform), ptr(:point), ptr(:twist), ptr(:point_velocity), ptr(:geometric_jacobian),
                      ptr(:point_jacobian), ptr(:acceleration), ptr(:point_acceleration))
    GC.@preserve state outs vd body base frame point begin
        td = rbd_task_desc(Int32(length(tasks)), pointer(body), pointer(base), pointer(frame), pointer(point))
        check(ccall((:rbd_task_kinematics, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ref{rbd_task_desc}, Ref{rbd_task_out}, Ptr{Cvoid}),
                    model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v),
                    vd === nothing ? C_NULL : devptr(vd), td, to, stream_ptr()))
    end
    outs
end

"Mirror of `rbd_task_pd_desc` (include/rbd_b200.h)."
struct rbd_task_pd_desc
    mode::Int32
    tasks::rbd_task_desc
    kind::Ptr{Int32}
    kp::Ptr{Cvoid}
    kd::Ptr{Cvoid}
    gain_ld::Int64
    x_ref::Ptr{Cvoid}
    x_ref_step_stride::Int64
    xd_ref::Ptr{Cvoid}
    xd_ref_step_stride::Int64
    joint::Ptr{rbd_pd_desc}
    effort_lo::Ptr{Float64}
    effort_hi::Ptr{Float64}
end

"""
    simulate_task_pd(state, final_time, tasks, kinds, kp, kd, x_ref; xd_ref = nothing, computed_torque = false,
                     effort_bounds = nothing, torques = nothing, Δt = 1e-4)

`simulate` with task-space feedback at every RK4 stage (rbd_integrate_task_pd, DESIGN 4.21): `tasks` as in `task_kinematics!`
(for a pose task `frame` must be `nothing` or the body), `kinds` a vector of `:point` / `:pose`.  Each task adds J_t' f_t with
f_t = -kp e - kd ė in its task frame: a point task's position relative to `base` (FramePDGains in `frame`), or the reference's
double-geodesic `pd(SE3PDGains, x, x_ref, T, T_ref)` on the frame at the task's point with the body's axes (pdcontrol.jl:83-107).
`kp`, `kd`: a vector of R = Σ (3 | 6) gains or a B × R matrix; `x_ref`: B × X (X = Σ (3 | 12), pose targets as `transform` of
`task_kinematics!`), `xd_ref`: B × R or `nothing`, held over the call.  No joint-space term here.  Tree mechanisms without contact
points.  (Not run here: no Julia installation is available to the project's tests; the Python binding exercises the same entry
point.)
"""
function simulate_task_pd(state::BatchedState{T}, final_time, tasks, kinds, kp, kd, x_ref; xd_ref = nothing,
                          computed_torque::Bool = false, effort_bounds = nothing, torques = nothing, Δt = 1e-4) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    model = state.model
    nsteps = 0; t = 0.0
    while t < final_time; t += Δt; nsteps += 1; end            # the reference's `while t < final_time` (ode_integrators.jl:311)
    body = Int32[body_index(model, t[1]) for t in tasks]
    base = Int32[body_index(model, t[2]) for t in tasks]
    frame = Int32[k == :pose ? body[i] : (t[4] === nothing ? Int32(-1) : body_index(model, t[4]))
                  for (i, (t, k)) in enumerate(zip(tasks, kinds))]
    point = zeros(Float64, 3, length(tasks))
    for (k, t) in enumerate(tasks)
        t[3] === nothing || (point[:, k] .= t[3])
    end
    kind = Int32[k == :pose ? 1 : 0 for k in kinds]
    lo, hi = effort_bounds === nothing ? (nothing, nothing) : (Vector{Float64}(effort_bounds[1]), Vector{Float64}(effort_bounds[2]))
    ptr(x) = x === nothing ? C_NULL : devptr(x)
    GC.@preserve state kp kd x_ref xd_ref torques lo hi body base frame point kind begin
        td = rbd_task_desc(Int32(length(tasks)), pointer(body), pointer(base), pointer(frame), pointer(point))
        desc = rbd_task_pd_desc(Int32(computed_torque ? 1 : 0), td, pointer(kind), devptr(kp), devptr(kd),
                                ndims(kp) == 2 ? Int64(B) : Int64(0), devptr(x_ref), 0, ptr(xd_ref), 0, Ptr{rbd_pd_desc}(C_NULL),
                                lo === nothing ? Ptr{Float64}(C_NULL) : pointer(lo), hi === nothing ? Ptr{Float64}(C_NULL) : pointer(hi))
        check(ccall((:rbd_integrate_task_pd, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Int64, Int64, Ref{rbd_task_pd_desc},
                     Ptr{Cvoid}, Ptr{Cvoid}, Float64, Int32, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                    model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), C_NULL, ptr(torques), 0, 0, desc,
                    C_NULL, C_NULL, Float64(Δt), Int32(nsteps), C_NULL, C_NULL, C_NULL, stream_ptr()))
    end
    nsteps
end

# ---- SURVEY 8(f) rank 3: Jacobians of forward dynamics ----------------------------------------------------------------------

"""
    dynamics_derivatives!(dvd_dq, dvd_dv, result, state, torques = nothing; externalwrenches = nothing, dvd_dtau = nothing)

Analytic `∂v̇/∂q` (tangent space) and `∂v̇/∂v` of `dynamics!` for every sample in one call -- what
`ForwardDiff.jacobian(x -> dynamics!(...), ...)` over the reference's generic path produces with 2 nv / 6 Dual sweeps per sample
(examples/5. Derivatives and gradients using ForwardDiff, test/test_mechanism_algorithms.jl:600-675).  `dvd_dq`, `dvd_dv` are
B x (nv*nv) device matrices, entry (i, j) of sample b at `[b, i + (j - 1) * nv]` (column-major like `M.data`);
`dvd_dq[:, :, j]` is the derivative along `velocity_to_configuration_derivative(e_j)`, i.e. `(∂v̇/∂q) * velocity_to_configuration_derivative_jacobian(state)`.
`result.v̇` receives v̇.  `externalwrenches`: B x 6nb root-frame wrenches as in `dynamics!`, held fixed while q moves; `dvd_dtau`:
a B x (nv*nv) matrix that receives `∂v̇/∂τ = M⁻¹` (rbd_dynamics_derivatives_ext).  (Not run here: no Julia installation is
available to the project's tests; the Python binding exercises the same entry points.)
"""
function dynamics_derivatives!(dvd_dq, dvd_dv, result::BatchedResult{T}, state::BatchedState{T}, torques = nothing;
                               externalwrenches = nothing, dvd_dtau = nothing) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    GC.@preserve state result torques dvd_dq dvd_dv externalwrenches dvd_dtau begin
        if externalwrenches === nothing && dvd_dtau === nothing
            check(ccall((:rbd_dynamics_derivatives, librbd), Int32,
                        (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}),
                        state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v),
                        torques === nothing ? C_NULL : devptr(torques), devptr(result.v̇), devptr(dvd_dq), devptr(dvd_dv), stream_ptr()))
        else
            check(ccall((:rbd_dynamics_derivatives_ext, librbd), Int32,
                        (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
                         Ptr{Cvoid}, Ptr{Cvoid}),
                        state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v),
                        torques === nothing ? C_NULL : devptr(torques), externalwrenches === nothing ? C_NULL : devptr(externalwrenches),
                        devptr(result.v̇), devptr(dvd_dq), devptr(dvd_dv), dvd_dtau === nothing ? C_NULL : devptr(dvd_dtau), stream_ptr()))
        end
    end
    dvd_dq, dvd_dv
end

"""
    inverse_dynamics_derivatives!(dtau_dq, dtau_dv, state, v̇, externalwrenches = nothing; torques = nothing, massmatrix = nothing)

Analytic `∂τ/∂q` (tangent space, as in `dynamics_derivatives!`) and `∂τ/∂v` of `inverse_dynamics!` at the given v̇ for every sample
in one call (rbd_inverse_dynamics_derivatives), B x (nv*nv) each in the layout of `dynamics_derivatives!`.  `torques` (B x nv)
receives τ itself and `massmatrix` (B x (nv*nv)) receives `∂τ/∂v̇ = M`, both triangles.  (Not run here: no Julia installation is
available to the project's tests; the Python binding exercises the same entry point.)
"""
function inverse_dynamics_derivatives!(dtau_dq, dtau_dv, state::BatchedState{T}, v̇::AbstractMatrix{T}, externalwrenches = nothing;
                                       torques = nothing, massmatrix = nothing) where {T <: Union{Float32, Float64}}
    checkstate(state)
    B = size(state.q, 1)
    GC.@preserve state v̇ externalwrenches dtau_dq dtau_dv torques massmatrix begin
        check(ccall((:rbd_inverse_dynamics_derivatives, librbd), Int32,
                    (Ptr{Cvoid}, Int32, Int64, Int64, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid},
                     Ptr{Cvoid}, Ptr{Cvoid}),
                    state.model.handle, dtype_code(T), B, B, devptr(state.q), devptr(state.v), devptr(v̇),
                    externalwrenches === nothing ? C_NULL : devptr(externalwrenches), torques === nothing ? C_NULL : devptr(torques),
                    devptr(dtau_dq), devptr(dtau_dv), massmatrix === nothing ? C_NULL : devptr(massmatrix), stream_ptr()))
    end
    dtau_dq, dtau_dv
end

"Compile the model-specialised solve kernel of `dynamics_derivatives!` ahead of time (cubin cache; no GPU needed)."
precompile_derivatives(model, ::Type{T}) where {T <: Union{Float32, Float64}} =
    check(ccall((:rbd_model_precompile_derivatives, librbd), Int32, (Ptr{Cvoid}, Int32), model.handle, dtype_code(T)))

end # module
