# DojoB200.jl -- Julia binding of libdojo_b200.so for Dojo.jl v0.7.6 (NOT runnable in the build image: no Julia there).
#
# It flattens a live `Dojo.Mechanism` into the C descriptor of include/dojo_b200.h and adds batched methods to the
# functions that enter / leave the per-timestep hot path, keeping their signatures:
#
#   Dojo.step!(mechanism, Z::Matrix, U::Matrix; opts)                 -> Z_next   (new batched method, 13Nb x B)
#   Dojo.get_maximal_gradients!(mechanism, Z::Matrix, U::Matrix; opts) -> (Fz, Fu) (12Nb x 12Nb x B, 12Nb x nu x B)
#   Dojo.minimal_to_maximal / maximal_to_minimal / step_minimal_coordinates!(mechanism, X::Matrix, ...)   (2nu x B)
#   Dojo.maximal_to_minimal_jacobian / minimal_to_maximal_jacobian / get_minimal_gradients!(mechanism, X::Matrix, ...)
#   DojoB200.env_step(mechanism, spec, S, A)                           -> (S_next, reward, done)  (DojoEnvironments.step! + get_state)
#   DojoB200.mehrotra_gpu!(mechanism; opts)                            -> :success / :failed  (B = 1 drop-in for mehrotra!)
#
# Node order = Julia ids (joints 1..Ne, bodies Ne+1..Ne+Nb, contacts after), exactly what the library assumes.
module DojoB200

using Dojo
using Dojo: Mechanism, JointConstraint, ContactConstraint, NonlinearContact, SolverOptions, vector

const LIB = get(ENV, "DOJO_B200_LIB", joinpath(@__DIR__, "..", "dojo.jl_b200", "libdojo_b200.so"))

struct BodyDesc
    mass::Float64
    inertia::NTuple{9,Float64}          # row-major
end
struct ElementDesc
    nlambda::Int32; nlimits::Int32
    axis_mask::NTuple{9,Float64}        # rows V1, V2, V3
    spring::Float64; damper::Float64
    spring_offset::NTuple{3,Float64}; limit_lo::NTuple{3,Float64}; limit_hi::NTuple{3,Float64}
end
struct JointDesc
    parent_body::Int32; child_body::Int32          # 0-based body index, -1 = origin
    vertex_parent::NTuple{3,Float64}; vertex_child::NTuple{3,Float64}
    orientation_offset::NTuple{4,Float64}
    tra::ElementDesc; rot::ElementDesc
end
struct ContactDesc
    type::Int32; parent_body::Int32
    friction_coefficient::Float64
    tangent::NTuple{6,Float64}; normal::NTuple{3,Float64}; origin::NTuple{3,Float64}
    radius::Float64; offset::NTuple{3,Float64}
end
struct MechanismDesc
    num_bodies::Int32; num_joints::Int32; num_contacts::Int32
    timestep::Float64; input_scaling::Float64; gravity::NTuple{3,Float64}
    bodies::Ptr{BodyDesc}; joints::Ptr{JointDesc}; contacts::Ptr{ContactDesc}
end
struct COptions
    rtol::Float64; btol::Float64; ls_scale::Float64
    max_iter::Int32; max_ls::Int32
    undercut::Float64; no_progress_max::Int32; no_progress_undercut::Float64; verbose::Int32
end
COptions(o::SolverOptions) = COptions(o.rtol, o.btol, o.ls_scale, o.max_iter, o.max_ls, o.undercut, o.no_progress_max,
                                      o.no_progress_undercut, o.verbose)

pad3(v) = ntuple(i -> i <= length(v) ? Float64(v[i]) : 0.0, 3)
rowmajor(M) = ntuple(k -> Float64(M[div(k - 1, 3) + 1, mod(k - 1, 3) + 1]), 9)

function element(el)
    Nλ = Dojo.joint_length(el); Nb½ = div(Dojo.limits_length(el), 2)
    mask = (vec(el.axis_mask1')..., vec(el.axis_mask2')..., vec(el.axis_mask3')...)
    lo = Nb½ > 0 ? el.joint_limits[1] : Float64[]; hi = Nb½ > 0 ? el.joint_limits[2] : Float64[]
    ElementDesc(Nλ, Nb½, Float64.(mask), el.spring, el.damper, pad3(el.spring_offset), pad3(lo), pad3(hi))
end

function flatten(mech::Mechanism{T,Nn,Ne,Nb,Ni}) where {T,Nn,Ne,Nb,Ni}
    bodies = [BodyDesc(b.mass, rowmajor(b.inertia)) for b in mech.bodies]
    bidx(id) = id == 0 ? Int32(-1) : Int32(id - Ne - 1)
    joints = [JointDesc(bidx(j.parent_id), bidx(j.child_id), Tuple(j.translational.vertices[1]), Tuple(j.translational.vertices[2]),
                        Tuple(vector(j.rotational.orientation_offset)), element(j.translational), element(j.rotational)) for j in mech.joints]
    contacts = map(mech.contacts) do c
        # contact_type (contacts/constructor.jl:117-128): 0 ImpactContact, 1 LinearContact, 2 NonlinearContact
        ctype = c.model isa NonlinearContact ? 2 : c.model isa LinearContact ? 1 : c.model isa ImpactContact ? 0 :
                error("DojoB200: unknown contact model $(typeof(c.model))")
        col = c.model.collision
        col isa SphereHalfSpaceCollision || error("DojoB200: only SphereHalfSpaceCollision is implemented")
        μf = ctype == 0 ? 0.0 : c.model.friction_coefficient                       # ImpactContact has no friction (impact.jl:8-11)
        tangent = ctype == 0 ? ntuple(_ -> 0.0, 6) : Tuple(vec(col.contact_tangent'))   # ... and a 0 x 3 contact_tangent (impact.jl:34)
        ContactDesc(ctype, bidx(c.parent_id), μf, tangent, Tuple(vec(col.contact_normal')),
                    Tuple(col.contact_origin), col.contact_radius, Tuple(col.contact_offset))
    end
    return bodies, joints, contacts
end

mutable struct Handle
    ptr::Ptr{Cvoid}
    nz::Int; nu::Int; ng::Int
end

function Handle(mech::Mechanism; device = 0, max_batch = 65536)
    bodies, joints, contacts = flatten(mech)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve bodies joints contacts begin
        desc = MechanismDesc(length(bodies), length(joints), length(contacts), mech.timestep, mech.input_scaling, Tuple(mech.gravity),
                             pointer(bodies), pointer(joints), pointer(contacts))
        rc = ccall((:dojo_create, LIB), Cint, (Ref{MechanismDesc}, Cint, Cint, Ref{Ptr{Cvoid}}), desc, device, max_batch, h)
        rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), C_NULL)))
    end
    hd = Handle(h[], 13 * length(bodies), Dojo.input_dimension(mech), 12 * length(bodies))
    finalizer(x -> ccall((:dojo_destroy, LIB), Cint, (Ptr{Cvoid},), x.ptr), hd)
    return hd
end

const HANDLES = IdDict{Mechanism,Handle}()
handle(mech) = get!(() -> Handle(mech), HANDLES, mech)

"batched step!: Z is 13Nb x B, U is nu x B (column = environment)"
function Dojo.step!(mech::Mechanism, Z::Matrix{Float64}, U::Matrix{Float64}; opts = SolverOptions{Float64}(), literal_q1 = false)
    h = handle(mech); B = size(Z, 2)
    Zn = similar(Z); status = zeros(Int32, B); iters = zeros(Int32, B)
    rc = ccall((:dojo_step, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, UInt32),
               h.ptr, COptions(opts), B, Z, U, C_NULL, Zn, C_NULL, status, iters, literal_q1 ? 1 : 0)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    B == 1 && status[1] == 2 && error("Excessive angular velocity.")   # reference behaviour: line_search.jl:18-20
    return Zn
end

"batched get_maximal_gradients!.  literal_q2 = true reproduces what the single-environment get_maximal_gradients! literally returns (data
 Jacobian built after update_state!, gradients/state.jl:69-76; DOJO_FLAG_Q2_LITERAL_GRADIENTS); the default is the consistent IFT gradient.
 literal_q17 = true leaves d(input impulse)/d(configuration) out of the data Jacobian as gradients/data.jl does
 (DOJO_FLAG_Q17_LITERAL_INPUT_JACOBIAN = 4); the reference's get_maximal_gradients! literally is literal_q2 = literal_q17 = true (flags 2 | 4)."
function Dojo.get_maximal_gradients!(mech::Mechanism, Z::Matrix{Float64}, U::Matrix{Float64}; opts = SolverOptions{Float64}(), literal_q2 = false,
                                     literal_q17 = false)
    h = handle(mech); B = size(Z, 2)
    Zn = similar(Z); Fz = zeros(h.ng, h.ng, B); Fu = zeros(h.ng, h.nu, B)
    status = zeros(Int32, B); iters = zeros(Int32, B)
    rc = ccall((:dojo_step_grad, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, UInt32),
               h.ptr, COptions(opts), B, Z, U, C_NULL, Zn, Fz, Fu, status, iters, (literal_q2 ? 2 : 0) | (literal_q17 ? 4 : 0))
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Fz, Fu
end

"batched get_contact_gradients (gradients/contact.jl:1-55): (Fz 12Nb x 12Nb x B, Fc 12Nb x 5Ni x B), contact data per contact =
 [friction_coefficient, contact_radius, contact_origin(3)]"
function get_contact_gradients!(mech::Mechanism, Z::Matrix{Float64}, U::Matrix{Float64}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(Z, 2); ng = 12 * length(mech.bodies); nc = 5 * length(mech.contacts)
    Zn = similar(Z); Fz = zeros(ng, ng, B); Fu = zeros(ng, h.nu, B); Fc = zeros(ng, nc, B); status = zeros(Int32, B); iters = zeros(Int32, B)
    rc = ccall((:dojo_step_grad_contact, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}),
               h.ptr, COptions(opts), B, Z, U, Zn, Fz, Fu, Fc, status, iters)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Fz, Fc
end
"swap the parameters of the live handle after the Mechanism's data changed (system identification): same topology"
function update_params!(mech::Mechanism)
    h = handle(mech); bodies, joints, contacts = flatten(mech)
    GC.@preserve bodies joints contacts begin
        desc = MechanismDesc(length(bodies), length(joints), length(contacts), mech.timestep, mech.input_scaling, Tuple(mech.gravity),
                             pointer(bodies), pointer(joints), pointer(contacts))
        rc = ccall((:dojo_update_params, LIB), Cint, (Ptr{Cvoid}, Ref{MechanismDesc}), h.ptr, desc)
        rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    end
    return nothing
end

"batched minimal_to_maximal / maximal_to_minimal: X is 2nu x B (per joint [c_tra; c_rot; v_tra; v_rot]), Z is 13Nb x B"
function Dojo.minimal_to_maximal(mech::Mechanism, X::Matrix{Float64})
    h = handle(mech); B = size(X, 2); Z = zeros(h.nz, B)
    rc = ccall((:dojo_minimal_to_maximal, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float64}, Ptr{Float64}), h.ptr, B, X, Z)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Z
end
function Dojo.maximal_to_minimal(mech::Mechanism, Z::Matrix{Float64})
    h = handle(mech); B = size(Z, 2); X = zeros(2 * h.nu, B)
    rc = ccall((:dojo_maximal_to_minimal, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float64}, Ptr{Float64}), h.ptr, B, Z, X)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return X
end

"batched step_minimal_coordinates! (simulation/step.jl:42-61): what DojoEnvironments.step! calls"
function Dojo.step_minimal_coordinates!(mech::Mechanism, X::Matrix{Float64}, U::Matrix{Float64}; opts = SolverOptions{Float64}(), literal::Bool = false)
    h = handle(mech); B = size(X, 2)
    Xn = similar(X); status = zeros(Int32, B); iters = zeros(Int32, B)
    # literal = true: the value step_minimal_coordinates! of Dojo.jl literally returns (step! advances the configuration a second time)
    rc = ccall((:dojo_step_minimal_flags, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, UInt32),
               h.ptr, COptions(opts), B, X, U, Xn, status, iters, literal ? UInt32(1) : UInt32(0))
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Xn
end

"batched maximal_to_minimal_jacobian (gradients/state.jl:9-56): 2nu x 12Nb x B"
function Dojo.maximal_to_minimal_jacobian(mech::Mechanism, Z::Matrix{Float64})
    h = handle(mech); B = size(Z, 2); J = zeros(2 * h.nu, 12 * length(mech.bodies), B)
    rc = ccall((:dojo_maximal_to_minimal_jacobian, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float64}, Ptr{Float64}), h.ptr, B, Z, J)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return J
end
"batched minimal_to_maximal_jacobian (gradients/state.jl:136-179) at x: 12Nb x 2nu x B (root -> leaves chain, see INTEGRATION.md)"
function Dojo.minimal_to_maximal_jacobian(mech::Mechanism, X::Matrix{Float64})
    h = handle(mech); B = size(X, 2); J = zeros(12 * length(mech.bodies), 2 * h.nu, B)
    Z = Dojo.minimal_to_maximal(mech, X)
    rc = ccall((:dojo_minimal_to_maximal_jacobian, LIB), Cint, (Ptr{Cvoid}, Cint, Ptr{Float64}, Ptr{Float64}), h.ptr, B, Z, J)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return J
end
"batched get_minimal_gradients! (gradients/state.jl:182-217): (2nu x 2nu x B, 2nu x nu x B)"
function Dojo.get_minimal_gradients!(mech::Mechanism, X::Matrix{Float64}, U::Matrix{Float64}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(X, 2); nm = 2 * h.nu
    Xn = similar(X); Gx = zeros(nm, nm, B); Gu = zeros(nm, h.nu, B); status = zeros(Int32, B); iters = zeros(Int32, B)
    rc = ccall((:dojo_minimal_gradients, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}),
               h.ptr, COptions(opts), B, X, U, Xn, Gx, Gu, status, iters)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Gx, Gu
end

# ---- DojoEnvironments on a batched axis (environments.jl:77-109, environments/ant_ars.jl): the spec carries state_map /
# input_map / get_state / the reward and failure test of examples/learning/ant_ars.jl:98-112
struct EnvSpec
    n_unactuated::Int32; contact_obs::Int32; forward_index::Int32; healthy_index::Int32; bound_index::Int32   # indices 0-based, -1 = off
    w_forward::Float64; w_control::Float64; w_contact::Float64; survive_reward::Float64
    healthy_min::Float64; healthy_max::Float64; bound_abs::Float64
end
const ANT_ARS = EnvSpec(6, 1, 0, 2, -1, 100.0, 0.05 / 10, 0.5e-3, 0.05, 0.2, 1.0, Inf)
const QUADRUPED_SAMPLING = EnvSpec(6, 0, -1, 2, 0, 0.0, 0.0, 0.0, 0.0, 0.0, Inf, 1000.0)

"step!(environment, S, A) for B environments: returns (S_next, reward, done); S is ns x B, A is na x B"
function env_step(mech::Mechanism, spec::EnvSpec, S::Matrix{Float64}, A::Matrix{Float64}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(S, 2)
    Sn = similar(S); reward = zeros(B); done = zeros(Int32, B); status = zeros(Int32, B); iters = zeros(Int32, B)
    rc = ccall((:dojo_env_step, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Ref{EnvSpec}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, Ptr{Int32}),
               h.ptr, COptions(opts), spec, B, S, A, Sn, reward, done, status, iters)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Sn, reward, done
end

"batched simulate!(...; record = true): returns (Z_traj 13Nb x B x T = Storage.x/q/v/ω, storage 12Nb x B x T = px pq vl ωl per body,
 diag 8 x B x T = momentum(6), kinetic, potential) -- save_to_storage! and mechanics/{momentum,energy}.jl evaluated on the device"
function simulate_record(mech::Mechanism, Z0::Matrix{Float64}, U::Array{Float64,3}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(Z0, 2); T = size(U, 3); Nb = length(mech.bodies)
    Zf = similar(Z0); traj = zeros(h.nz, B, T); sto = zeros(12 * Nb, B, T); diag = zeros(8, B, T); status = zeros(Int32, B)
    rc = ccall((:dojo_simulate_record, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}),
               h.ptr, COptions(opts), B, T, Z0, U, Zf, traj, sto, diag, status)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return traj, sto, diag
end

"open-loop batched simulate!: all T steps in one launch; U is nu x B x T, returns (Z_final, Z_traj 13Nb x B x T)"
function rollout(mech::Mechanism, Z0::Matrix{Float64}, U::Array{Float64,3}; opts = SolverOptions{Float64}(), record = true)
    h = handle(mech); B = size(Z0, 2); T = size(U, 3)
    Zf = similar(Z0); traj = record ? zeros(h.nz, B, T) : nothing; status = zeros(Int32, B)
    rc = ccall((:dojo_rollout, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}),
               h.ptr, COptions(opts), B, T, Z0, U, Zf, record ? traj : C_NULL, status)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Zf, traj
end

struct CFeedback  # = DojoFeedback (include/dojo_b200.h)
    steps::Int32; envs::Int32
    K::Ptr{Float64}; K_i::Ptr{Float64}; x_ref::Ptr{Float64}; u_ref::Ptr{Float64}
end
"closed-loop batched simulate! (examples/control: a controller! that reads get_minimal_state): before every step t the device applies
 u_t = u_ref - K (x_t - x_ref) - K_i xi_t, xi_t = xi_{t-1} + h (x_t - x_ref), on the minimal state x_t, all T steps in one launch.
 K, K_i: nu x 2nu, nu x 2nu x B or nu x 2nu x (1 or B) x T; x_ref (2nu) and u_ref (nu) likewise; every array is broadcast to the largest.
 xi (2nu x B, zeros when K_i is given without it) is updated in place.  Returns (Z_final, Z_traj 13Nb x B x T or nothing,
 U_applied nu x B x T, xi); rollout(mech, Z0, U_applied) reproduces the trajectory bit for bit"
function rollout_feedback(mech::Mechanism, Z0::Matrix{Float64}, T::Integer, K::AbstractArray; x_ref = nothing, u_ref = nothing, K_i = nothing,
                          xi = nothing, opts = SolverOptions{Float64}(), record = true)
    h = handle(mech); B = size(Z0, 2); nu = h.nu
    lay(A, tail) = A === nothing ? nothing : reshape(Float64.(A), tail..., size(A, length(tail) + 1), size(A, length(tail) + 2))
    arrs = (lay(K, (nu, 2nu)), lay(K_i, (nu, 2nu)), lay(x_ref, (2nu,)), lay(u_ref, (nu,)))
    given = [a for a in arrs if a !== nothing]
    envs = maximum(size(a, ndims(a) - 1) for a in given); steps = maximum(size(a, ndims(a)) for a in given)
    full(a) = a === nothing ? nothing : (o = zeros(size(a)[1:end-2]..., envs, steps); o .= a; o)
    Kf, Kif, xrf, urf = map(full, arrs)
    (Kif !== nothing && xi === nothing) && (xi = zeros(2nu, B))
    p(a) = a === nothing ? Ptr{Float64}(C_NULL) : pointer(a)
    Zf = similar(Z0); traj = record ? zeros(h.nz, B, T) : nothing; Ua = zeros(nu, B, T); status = zeros(Int32, B)
    rc = GC.@preserve Kf Kif xrf urf begin
        fb = CFeedback(Int32(steps), Int32(envs), p(Kf), p(Kif), p(xrf), p(urf))
        ccall((:dojo_rollout_feedback, LIB), Cint,
              (Ptr{Cvoid}, Ref{COptions}, Cint, Cint, Ptr{Float64}, Ref{CFeedback}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}),
              h.ptr, COptions(opts), B, T, Z0, fb, xi === nothing ? C_NULL : xi, Zf, record ? traj : C_NULL, Ua, status)
    end
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Zf, traj, Ua, xi
end

"simulate! + get_maximal_gradients! at every step, fused: U is nu x B x T; returns (Z_traj 13Nb x B x (T+1) with Z_traj[:, :, 1] = Z0,
 Fz 12Nb x 12Nb x B x T, Fu 12Nb x nu x B x T, status B x T) -- Fz[:, :, e, t] = dz_{t+1}/dz_t"
function rollout_gradients(mech::Mechanism, Z0::Matrix{Float64}, U::Array{Float64,3}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(Z0, 2); T = size(U, 3); ng = 12 * length(mech.bodies)
    traj = zeros(h.nz, B, T + 1); Fz = zeros(ng, ng, B, T); Fu = zeros(ng, h.nu, B, T); status = zeros(Int32, B, T); iters = zeros(Int32, B, T)
    rc = ccall((:dojo_rollout_grad, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}),
               h.ptr, COptions(opts), B, T, Z0, U, traj, Fz, Fu, status, iters)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return traj, Fz, Fu, status
end
"the same in minimal coordinates (get_minimal_gradients! at every step): X_traj 2nu x B x (T+1), Gx 2nu x 2nu x B x T, Gu 2nu x nu x B x T"
function rollout_minimal_gradients(mech::Mechanism, X0::Matrix{Float64}, U::Array{Float64,3}; opts = SolverOptions{Float64}())
    h = handle(mech); B = size(X0, 2); T = size(U, 3); nm = 2 * h.nu
    Xt = zeros(nm, B, T + 1); Gx = zeros(nm, nm, B, T); Gu = zeros(nm, h.nu, B, T); status = zeros(Int32, B, T); iters = zeros(Int32, B, T)
    rc = ccall((:dojo_rollout_minimal_gradients, LIB), Cint,
               (Ptr{Cvoid}, Ref{COptions}, Cint, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}),
               h.ptr, COptions(opts), B, T, X0, U, Xt, Gx, Gu, status, iters)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return Xt, Gx, Gu, status
end

struct CQuadraticCost  # = DojoQuadraticCost (include/dojo_b200.h)
    steps::Int32; envs::Int32
    Q::Ptr{Float64}; R::Ptr{Float64}; x_goal::Ptr{Float64}; u_goal::Ptr{Float64}; Q_final::Ptr{Float64}; x_goal_final::Ptr{Float64}
end
"Riccati backward pass of iLQR / TVLQR (the backward pass of IterativeLQR.jl's solve!) on rollout_minimal_gradients' output, all
 environments and steps in one launch: Xt 2nu x B x (T+1), U nu x B x T (or nothing), Gx 2nu x 2nu x B x T, Gu 2nu x nu x B x T.
 Cost sum_t 1/2 |x_t - x_goal|^2_Q + 1/2 |u_t - u_goal|^2_R + 1/2 |x_T - x_goal_final|^2_Q_final: Q, R, x_goal, u_goal as nxn, nxnxB or
 nxnx(1 or B)xT (broadcast to the largest, as rollout_feedback's arrays); Q_final (default: Q's last step) and x_goal_final (default:
 x_goal's last step) n x n or n x n x B.  active: nu mask (nothing: all inputs), mu: B regularisations.  Returns (K nu x 2nu x B x T,
 k nu x B x T, dV 2 x B, status B): u = U + alpha k - K (x - Xt) is rollout_feedback(mech, Z0, T, K; x_ref = Xt[:, :, 1:T],
 u_ref = U + alpha k); status[e] = t when the Cholesky of Quu + mu I failed at step t (1-based; K, k up to it and dV are NaN)"
function lqr_backward(mech::Mechanism, Xt::Array{Float64,3}, U, Gx::Array{Float64,4}, Gu::Array{Float64,4}; Q, R, x_goal = nothing,
                      u_goal = nothing, Q_final = nothing, x_goal_final = nothing, active = nothing, mu = nothing)
    h = handle(mech); B = size(Xt, 2); T = size(Xt, 3) - 1; nu = h.nu
    lay(A, tail) = A === nothing ? nothing : reshape(Float64.(A), tail..., size(A, length(tail) + 1), size(A, length(tail) + 2))
    arrs = (lay(Q, (2nu, 2nu)), lay(R, (nu, nu)), lay(x_goal, (2nu,)), lay(u_goal, (nu,)))
    given = [a for a in arrs if a !== nothing]
    fin = (Q_final === nothing ? nothing : reshape(Float64.(Q_final), 2nu, 2nu, :), x_goal_final === nothing ? nothing : reshape(Float64.(x_goal_final), 2nu, :))
    envs = max(maximum(size(a, ndims(a) - 1) for a in given), maximum((size(a, ndims(a)) for a in fin if a !== nothing); init = 1))
    steps = maximum(size(a, ndims(a)) for a in given)
    full(a) = a === nothing ? nothing : (o = zeros(size(a)[1:end-2]..., envs, steps); o .= a; o)
    Qs, Rs, xgs, ugs = map(full, arrs)
    Qf = fin[1] === nothing ? Qs[:, :, :, end] : (o = zeros(2nu, 2nu, envs); o .= fin[1]; o)
    xgf = fin[2] === nothing ? (xgs === nothing ? nothing : xgs[:, :, end]) : (o = zeros(2nu, envs); o .= fin[2]; o)
    act = active === nothing ? C_NULL : Int32.(collect(active))
    K = zeros(nu, 2nu, B, T); k = zeros(nu, B, T); dV = zeros(2, B); status = zeros(Int32, B)
    p(a) = a === nothing ? Ptr{Float64}(C_NULL) : pointer(a)
    rc = GC.@preserve Qs Rs xgs ugs Qf xgf begin
        cost = CQuadraticCost(Int32(steps), Int32(envs), p(Qs), p(Rs), p(xgs), p(ugs), p(Qf), p(xgf))
        ccall((:dojo_lqr_backward, LIB), Cint,
              (Ptr{Cvoid}, Cint, Cint, Ref{CQuadraticCost}, Ptr{Int32}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64},
               Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}),
              h.ptr, B, T, cost, act, Xt, U === nothing ? C_NULL : U, Gx, Gu, mu === nothing ? C_NULL : Float64.(mu), K, k, dV, status)
    end
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return K, k, dV, status
end

# ---- multi-GPU: one Julia process per GPU (e.g. MPI.jl ranks or Distributed workers); the exchange of the next states is fused into
# the step kernel (peer writes over NVLink, include/dojo_b200.h "Multi-GPU"): no NCCL.jl needed.  `allgather_bytes` is any host-side
# all-gather of a 128-byte blob per rank (MPI.Allgather, a shared file, ...), used ONCE at set-up.
mutable struct Gather
    ptr::Ptr{Cvoid}; world::Int; rank::Int; B::Int
end
function Gather(mech::Mechanism, world::Integer, rank::Integer, B_local::Integer, allgather_bytes::Function)
    h = handle(mech); g = Ref{Ptr{Cvoid}}(C_NULL)
    rc = ccall((:dojo_gather_create, LIB), Cint, (Ptr{Cvoid}, Cint, Cint, Cint, Ref{Ptr{Cvoid}}), h.ptr, world, rank, B_local, g)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    mine = zeros(UInt8, 128)
    ccall((:dojo_gather_export, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}), g[], mine) == 0 || error("dojo_gather_export")
    all = allgather_bytes(mine)::Vector{UInt8}                       # world * 128 bytes, rank order
    ccall((:dojo_gather_connect, LIB), Cint, (Ptr{Cvoid}, Ptr{UInt8}), g[], all) == 0 ||
        error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    gd = Gather(g[], world, rank, B_local)
    finalizer(x -> ccall((:dojo_gather_destroy, LIB), Cint, (Ptr{Cvoid},), x.ptr), gd)
    return gd
end
"step! of this rank's shard (device pointers, e.g. CuArray pointers) + exchange: afterwards `gathered(g)` on every rank holds the next
 states of all ranks, 13Nb x (world * B_local)"
function step_gather!(mech::Mechanism, g::Gather, dZ::Ptr{Float64}, dU::Ptr{Float64}, dZn::Ptr{Float64}; opts = SolverOptions{Float64}(), stream = C_NULL)
    h = handle(mech)
    rc = ccall((:dojo_step_gather_async, LIB), Cint,
               (Ptr{Cvoid}, Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, UInt32, Ptr{Cvoid}),
               h.ptr, g.ptr, COptions(opts), g.B, dZ, dU, C_NULL, dZn, C_NULL, C_NULL, 0, stream)
    rc == 0 || error(unsafe_string(ccall((:dojo_last_error, LIB), Cstring, (Ptr{Cvoid},), h.ptr)))
    return nothing
end
gathered(g::Gather) = ccall((:dojo_gather_buffer, LIB), Ptr{Float64}, (Ptr{Cvoid},), g.ptr)   # device pointer of the most recent step's gathered states (two alternating halves: ask after every step)

"B = 1 drop-in for mehrotra!(mechanism; opts): runs the step on the GPU and writes vsol / wsol back into the Mechanism"
function mehrotra_gpu!(mech::Mechanism; opts = SolverOptions{Float64}())
    h = handle(mech)
    z = Dojo.get_maximal_state(mech)
    # inputs were already turned into JF2 / Jτ2 by set_input!; they are passed as external impulses: Fext = J / timestep
    Fext = vcat([[b.state.Fext + b.state.JF2 / mech.timestep; b.state.τext + b.state.Jτ2 / mech.timestep] for b in mech.bodies]...)
    zn = zeros(h.nz); status = zeros(Int32, 1); iters = zeros(Int32, 1)
    ccall((:dojo_step, LIB), Cint,
          (Ptr{Cvoid}, Ref{COptions}, Cint, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Float64}, Ptr{Int32}, Ptr{Int32}, UInt32),
          h.ptr, COptions(opts), 1, z, C_NULL, Fext, zn, C_NULL, status, iters, 0)
    for (i, b) in enumerate(mech.bodies)
        b.state.vsol[2] = zn[13 * (i - 1) .+ (4:6)]; b.state.ωsol[2] = zn[13 * (i - 1) .+ (11:13)]
    end
    status[1] == 2 && error("Excessive angular velocity.")
    return status[1] == 0 ? :success : :failed
end

end # module
