# B200UDE.jl -- the reference-side binding of libb200ude.so (include/b200ude.h).
#
# SOURCE ONLY: `julia` is not installed in the build image nor on the GPU boxes, so this file has never been run.  It is the
# binding a maintainer of ChrisRackauckas/universal_differential_equations would add next to the scripts so that the call
# surface the scripts use --
#     concrete_solve(prob, Tsit5() / Vern7(), u0, p; saveat, abstol, reltol, sensealg = InterpolatingAdjoint(autojacvec = ReverseDiffVJP()))
#     DiffEqFlux.sciml_train(loss, theta, ADAM(eta); cb, maxiters)           (seir_exposure.jl:137-141,160-161; Fisher-KPP-CNN.jl:136,236-238)
# -- reaches the sm_90a kernels with ONE changed line per script: the line that builds the ODEProblem wraps the script's
# right-hand side in a `B200UDEFunction`, which names the UDE form (what a C ABI cannot learn from a closure):
#     prob_nn = ODEProblem(B200UDE.SEIRExposure(dudt_, ann, p_), u0, tspan, p)            # was ODEProblem(dudt_, u0, tspan, p)  seir_exposure.jl:131
#     prob_nn = ODEProblem(B200UDE.FisherKPP(nn_ode, rx_nn, Nx), rho0, (0.0, T), p)        # Fisher-KPP-CNN.jl:131
#     prob_nn = ODEProblem(B200UDE.LotkaVolterra(nn_dynamics!, U; rates = 0, consts = (p_[1], p_[4])), Xn[:, 1], tspan, p)   # scenario_1.jl:78
# Everything else -- predict(), loss(), callback, sciml_train(ADAM) -> sciml_train(BFGS) -- stays as written: the methods below
# are picked by dispatch on the problem's function type, and Zygote finds the reverse rule through DiffEqBase's own seam
# (`_concrete_solve_adjoint`, the function every `sensealg` of DiffEqSensitivity specialises).
#
# The Python module universal_differential_equations_b200.sciml mirrors these names and IS exercised by the test-suite
# (tests/test_gpu_parity.py::test_script_call_surface_*).
module B200UDE

using DiffEqBase, SciMLBase, OrdinaryDiffEq, DiffEqSensitivity, ChainRulesCore
import ComponentArrays

const lib = get(ENV, "B200UDE_LIB", "libb200ude")   # universal_differential_equations_b200/csrc/libb200ude.so

# ---- constants of include/b200ude.h ---------------------------------------------------------------------------------------
const F32 = Int32(0)
const MODEL_LV, MODEL_SEIR, MODEL_FKPP, MODEL_NODE, MODEL_SEIR_NODE, MODEL_FORCED, MODEL_OPERATOR = Int32.(0:6)

# operator UDE (MODEL_OPERATOR, npde.jl:75-78): du = D1 * re(p)(u) + D2 * u with fixed Julia matrices (column-major, as the ABI
# takes them); D2 = nothing is a zero D2
set_operators!(h, D1::Matrix{Float32}, D2::Union{Matrix{Float32},Nothing}=nothing) =
    check(h.ptr, ccall((:b200ude_set_operators, lib), Int32, (Ptr{Cvoid}, Ptr{Float32}, Ptr{Float32}, Int32, Ptr{Cvoid}),
                       h.ptr, D1, D2 === nothing ? Ptr{Float32}(C_NULL) : D2, HOST, C_NULL))

# forced neural ODE (MODEL_FORCED, FENEP.jl:41-62): per-trajectory forcing coefficients, a Julia Array of size (N, 3J) (the ABI's
# [3J][N]): columns A_j, ω_j, φ_j
set_forcing!(h, coef::Matrix{Float32}) =
    check(h.ptr, ccall((:b200ude_set_forcing, lib), Int32, (Ptr{Cvoid}, Ptr{Float32}, Csize_t, Int32, Ptr{Cvoid}), h.ptr, coef, size(coef, 1), HOST, C_NULL))
const ACT_IDENTITY, ACT_TANH, ACT_RBF = Int32.(0:2)
const TSIT5, VERN7, RKC2 = Int32.(0:2)
const INTERPOLATING_ADJOINT, DISCRETE_ADJOINT = Int32(0), Int32(1)
const HOST, DEVICE = Int32(0), Int32(1)
const FLAG_VERN7_DENSE = UInt32(2)
const FLAG_DISCRETE_DENSE = UInt32(4)
const FLAG_CHECKPOINT = UInt32(8)

Base.@kwdef mutable struct Desc            # mirrors struct b200ude_desc
    struct_size::UInt32 = 0;  device::Int32 = 0;  dtype::Int32 = F32;  model::Int32 = 0
    state_dim::Int32 = 2;     n_layers::Int32 = 0
    widths::NTuple{7,Int32} = ntuple(_ -> Int32(0), 7);  acts::NTuple{6,Int32} = ntuple(_ -> Int32(0), 6)
    n_prefix::Int32 = 0;      n_suffix::Int32 = 0;       n_consts::Int32 = 0
    consts::NTuple{16,Float64} = ntuple(_ -> 0.0, 16)
    solver::Int32 = 0;        sensealg::Int32 = 0
    t0::Float64 = 0.0;        dt::Float64 = 0.1;         n_steps::Int32 = 0;  save_every::Int32 = 1
    abstol::Float64 = 0.0;    reltol::Float64 = 0.0
    n_loss_weights::Int32 = 0; loss_weights::NTuple{16,Float64} = ntuple(_ -> 0.0, 16)
    max_trajectories::UInt64 = 1; flags::UInt32 = 0;     adaptive::Int32 = 0;  max_steps::Int32 = 0;  n_stages::Int32 = 0
end

Base.@kwdef mutable struct Adam            # mirrors struct b200ude_adam
    struct_size::UInt32 = 0; reserved::UInt32 = 0
    eta::Float64 = 0.001; beta1::Float64 = 0.9; beta2::Float64 = 0.999; eps::Float64 = 1e-8
    loss_scale::Float64 = 1.0; l2_reg::Float64 = 0.0
end

lasterr(h) = unsafe_string(ccall((:b200ude_last_error, lib), Cstring, (Ptr{Cvoid},), h))
check(h, rc) = rc == 0 || error("b200ude error $rc: " * lasterr(h))

mutable struct Handle
    ptr::Ptr{Cvoid}; P::Int; nsave::Int; d::Int; cap::Int
    function Handle(desc::Desc)
        desc.struct_size = sizeof(Desc)
        out = Ref{Ptr{Cvoid}}(C_NULL)
        check(C_NULL, ccall((:b200ude_create, lib), Int32, (Ref{Desc}, Ref{Ptr{Cvoid}}), desc, out))
        h = new(out[], 0, 0, desc.state_dim, desc.max_trajectories)
        h.P = ccall((:b200ude_num_params, lib), Csize_t, (Ptr{Cvoid},), h.ptr)
        h.nsave = ccall((:b200ude_num_save, lib), Csize_t, (Ptr{Cvoid},), h.ptr)
        finalizer(x -> ccall((:b200ude_destroy, lib), Cvoid, (Ptr{Cvoid},), x.ptr), h)
    end
end

# ---- the UDE forms the library recognises --------------------------------------------------------------------------------
"""An ODE function that ALSO says which UDE form it is.  `f` is the script's own closure: any code path that does not go
through the methods below (plotting solves with other algorithms, SINDy post-processing, ...) keeps calling it."""
struct B200UDEFunction{iip,F} <: SciMLBase.AbstractODEFunction{iip}
    f::F
    model::Int32; state_dim::Int32
    widths::Vector{Int32}; acts::Vector{Int32}     # chain layer widths (n_layers + 1) and activations (n_layers)
    n_prefix::Int32; n_suffix::Int32               # trainable physics scalars in front of / behind the chain parameters in theta
    consts::Vector{Float64}                        # the known-physics constants, in the order of include/b200ude.h
end
(f::B200UDEFunction)(args...) = f.f(args...)

act_code(a) = a === tanh ? ACT_TANH : a === identity ? ACT_IDENTITY : (string(a) == "rbf" ? ACT_RBF : error("activation $a has no kernel"))
# layer widths / activations of a DiffEqFlux.FastChain, a Lux.Chain or a Flux.Chain of dense layers
function chain_shape(chain)
    ls = collect(chain.layers)
    ins(l)  = hasproperty(l, :in)  ? l.in  : hasproperty(l, :in_dims)  ? l.in_dims  : size(l.weight, 2)
    outs(l) = hasproperty(l, :out) ? l.out : hasproperty(l, :out_dims) ? l.out_dims : size(l.weight, 1)
    act(l)  = hasproperty(l, :σ) ? l.σ : l.activation
    Int32[ins(ls[1]); outs.(ls)], Int32[act_code(act(l)) for l in ls]
end

"""LV UDE of LotkaVolterra/scenario_1.jl:69-76 (`rates = 0`, consts = (p_[1], p_[4])), scenario_2.jl:90-98 (`rates = 1`: theta[1] is
the trainable delta, consts = (p_[1],)), hudson_bay.jl:85-91 (`rates = 2`)."""
LotkaVolterra(f, chain; rates = 0, consts = (1.3, 1.8), iip = true) =
    B200UDEFunction{iip,typeof(f)}(f, MODEL_LV, 2, chain_shape(chain)..., rates, 0, collect(Float64, consts))
"""SEIR exposure UDE of SEIR_exposure/seir_exposure.jl:117-130; `p_` = (F, β0, α, κ, μ, σ, γ, d, λ) (`:33`)."""
SEIRExposure(f, ann, p_) = B200UDEFunction{false,typeof(f)}(f, MODEL_SEIR, 7, chain_shape(ann)..., 0, 0, collect(Float64, p_))
"""Black-box baseline `dudt_node` of seir_exposure.jl:55-64 (7 -> 64 -> 64 -> 64 -> 7)."""
SEIRNeuralODE(f, ann, p_) = B200UDEFunction{false,typeof(f)}(f, MODEL_SEIR_NODE, 7, chain_shape(ann)..., 0, 0, collect(Float64, p_))
"""Fisher-KPP UPDE of FisherKPP/Fisher-KPP-CNN.jl:111-126: theta = [destructure(rx_nn); conv taps (3); conv bias (1); D0]."""
FisherKPP(f, rx_nn, Nx) = B200UDEFunction{false,typeof(f)}(f, MODEL_FKPP, Nx, chain_shape(rx_nn)..., 0, 5, Float64[])

# ---- theta adapters: the scripts' parameter containers <-> the flat Float32 vector of the ABI (same element order) -----
flat32(p::AbstractVector) = Float32.(collect(p))                       # Vector (initial_params, destructure), ComponentVector
unflat(p::ComponentArrays.ComponentVector, g) = ComponentArrays.ComponentArray(eltype(p).(g), ComponentArrays.getaxes(p))
unflat(p::AbstractVector, g) = eltype(p).(g)

# ---- handles are cached per (function, solver, grid, tolerances, sensealg) -----------------------------------------------
const HANDLES = Dict{Any,Handle}()
solver_code(::Tsit5) = TSIT5
solver_code(::Vern7) = VERN7
# ROCK2 / ROCK4 (npde.jl:61,82,111,122) run as RKC2, the stabilised explicit method of the same class this library has (ROCK's own
# tables are not in the reference).  Their eigen_est is a callback that stores the bound in integ.eigen_est: it is called once
# on a probe to read the bound.  With dt: fixed-step RKC2 with the fewest stages whose stability interval covers 1.05 dt rho.
# Without dt on the operator model: adaptive RKC2, rho in consts[0], each step choosing its own stage count (at most 64).
solver_code(::Union{ROCK2,ROCK4}) = RKC2
mutable struct EigenProbe
    eigen_est::Float64
end
function eigen_est_of(alg)
    probe = EigenProbe(0.0)
    alg.eigen_est(probe)
    probe.eigen_est
end
function rkc2_beta(s)   # real stability interval of s-stage RKC2 (sciml._rkc2_beta)
    w0 = 1 + (2 / 13) / s^2
    T0, T1, d0, d1, e0, e1 = 1.0, w0, 0.0, 1.0, 0.0, 0.0
    for _ in 2:s
        T0, T1, d0, d1, e0, e1 = T1, 2w0 * T1 - T0, d1, 2T1 + 2w0 * d1 - d0, e1, 4d1 + 2w0 * e1 - e0
    end
    (w0 + 1) * e1 / d1
end
rock_stages(dt, rho) = something(findfirst(s -> s >= 2 && rkc2_beta(s) >= 1.05 * dt * rho, 1:64), 0)   # 0: create refuses it
sens_code(::InterpolatingAdjoint) = INTERPOLATING_ADJOINT
sens_code(::ForwardDiffSensitivity) = DISCRETE_ADJOINT      # same quantity (exact derivative of the discrete scheme), reverse mode
sens_code(::Nothing) = INTERPOLATING_ADJOINT
"""`B200UDE.vern7_dense[] = true`: Vern7 runs as OrdinaryDiffEq does -- saveat from Vern7's lazy dense output instead of tstops.
With the interpolating adjoint the adjoint runs over that dense output instead of a Tsit5 re-solve (B200UDE_FLAG_VERN7_DENSE); with
ForwardDiffSensitivity the discrete adjoint differentiates the interpolated saves (B200UDE_FLAG_DISCRETE_DENSE; the library ignores
it on a fixed grid, where the saves are step ends).  The Fisher-KPP UPDE with ForwardDiffSensitivity keeps its tstops kernels."""
const vern7_dense = Ref(false)
dense_flag(f, alg, sensealg) = !(vern7_dense[] && alg isa Vern7) ? UInt32(0) :
                               sens_code(sensealg) != DISCRETE_ADJOINT ? FLAG_VERN7_DENSE :
                               f.model == MODEL_FKPP ? UInt32(0) : FLAG_DISCRETE_DENSE

function handle_for(f::B200UDEFunction, alg, sensealg, tspan, saveat, dt, abstol, reltol, N)
    ts = saveat isa Number ? collect(tspan[1]:saveat:tspan[2]) : collect(saveat)
    save_dt = ts[2] - ts[1]
    all(isapprox.(diff(ts), save_dt; rtol = 1e-9)) || error("B200UDE: uniformly spaced saveat only")
    adaptive = dt === nothing
    step = adaptive ? save_dt : dt
    rock = alg isa Union{ROCK2,ROCK4}
    rho = rock ? eigen_est_of(alg) : 0.0
    key = (objectid(f), typeof(alg), rho, sens_code(sensealg), dense_flag(f, alg, sensealg), tspan, save_dt, step, adaptive, abstol, reltol)
    h = get(HANDLES, key, nothing)
    (h !== nothing && h.cap >= N) && return h
    nl = length(f.acts)
    cs = rock && adaptive && f.model == MODEL_OPERATOR ? [f.consts; rho] : f.consts
    d = Desc(model = f.model, state_dim = f.state_dim, n_layers = nl,
             widths = ntuple(i -> i <= nl + 1 ? f.widths[i] : Int32(0), 7), acts = ntuple(i -> i <= nl ? f.acts[i] : Int32(0), 6),
             n_prefix = f.n_prefix, n_suffix = f.n_suffix, n_consts = length(cs),
             consts = ntuple(i -> i <= length(cs) ? cs[i] : 0.0, 16),
             n_stages = !rock ? 0 : adaptive ? 64 : rock_stages(step, rho),
             solver = solver_code(alg), sensealg = sens_code(sensealg), t0 = tspan[1], dt = step,
             n_steps = round(Int32, (tspan[2] - tspan[1]) / step), save_every = round(Int32, save_dt / step),
             adaptive = adaptive ? 1 : 0, abstol = abstol, reltol = reltol, max_steps = adaptive ? 512 : 0, max_trajectories = N,
             flags = dense_flag(f, alg, sensealg))
    HANDLES[key] = Handle(d)
end

# ---- forward: Array-convertible solution of the ensemble (N = 1 for the scripts as written) -----------------------------
struct B200Solution{T} <: AbstractMatrix{T}     # d x n_save, what Array(concrete_solve(...)) and sol[2:4, :] index into
    u::Matrix{T}; t::Vector{Float64}; status::Vector{Int32}
end
Base.size(s::B200Solution) = size(s.u); Base.getindex(s::B200Solution, i...) = s.u[i...]

function forward(h::Handle, θ::Vector{Float32}, u0::Matrix{Float32})       # u0: (N, d); returns (N, d, n_save)
    N = size(u0, 1); out = Array{Float32}(undef, N, h.d, h.nsave); status = Vector{Int32}(undef, N)
    GC.@preserve θ u0 out status check(h.ptr, ccall((:b200ude_solve_host, lib), Int32,
        (Ptr{Cvoid}, Ptr{Float32}, Ptr{Float32}, Csize_t, Ptr{Float32}, Ptr{Int32}), h.ptr, θ, u0, N, out, status))
    any(!=(0), status) && @warn "B200UDE: $(count(!=(0), status)) of $N trajectories failed (1 = non-finite, 2 = maxiters); their unreached save points are NaN"
    out, status
end

# generic cotangent: the pullback of the solve.  The forward record lives in the handle (b200ude_solve_host kept it).
function pullback(h::Handle, Δ::Array{Float32,3}, N)
    gθ = Vector{Float32}(undef, h.P); gu0 = Matrix{Float32}(undef, N, h.d)
    dΔ = cu_upload(Δ)                                   # the adjoint entry point takes device pointers
    GC.@preserve gθ gu0 begin
        dg, dgu = cu_alloc(Float32, h.P), cu_alloc(Float32, N * h.d)
        check(h.ptr, ccall((:b200ude_adjoint, lib), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, dΔ, dg, dgu, C_NULL))
        cu_download!(gθ, dg); cu_download!(gu0, dgu)
    end
    gθ, gu0
end
# thin wrappers over CUDA.jl (kept out of line so that the module loads without CUDA.jl for host-buffer-only use)
cu_upload(a) = (CUDA = Base.require(Main, :CUDA); pointer(CUDA.CuArray(a)))
cu_alloc(T, n) = (CUDA = Base.require(Main, :CUDA); pointer(CUDA.CuArray{T}(undef, n)))
cu_download!(dst, src) = (CUDA = Base.require(Main, :CUDA); copyto!(dst, unsafe_wrap(CUDA.CuArray, src, length(dst))))

const B200Problem = ODEProblem{uType,tType,iip,P,<:B200UDEFunction} where {uType,tType,iip,P}

function DiffEqBase.concrete_solve(prob::B200Problem, alg::Union{Tsit5,Vern7}, u0 = prob.u0, p = prob.p; saveat = prob.tspan[2] - prob.tspan[1],
                                   sensealg = nothing, abstol = 1e-6, reltol = 1e-3, dt = nothing, kwargs...)
    u0m = u0 isa AbstractMatrix ? Float32.(permutedims(u0)) : reshape(Float32.(u0), 1, :)      # (N, d)
    h = handle_for(prob.f, alg, sensealg, prob.tspan, saveat, dt, abstol, reltol, size(u0m, 1))
    out, status = forward(h, flat32(p), u0m)
    ts = saveat isa Number ? collect(prob.tspan[1]:saveat:prob.tspan[2]) : collect(Float64, saveat)
    size(u0m, 1) == 1 ? B200Solution(eltype(u0).(out[1, :, :]), ts, status) : out
end

# DiffEqBase's reverse-mode seam: Zygote's adjoint of concrete_solve / solve calls this with the sensealg the script passed
for S in (:InterpolatingAdjoint, :ForwardDiffSensitivity)
    @eval function DiffEqBase._concrete_solve_adjoint(prob::B200Problem, alg::Union{Tsit5,Vern7}, sensealg::$S, u0, p, args...;
                                                     saveat = prob.tspan[2] - prob.tspan[1], abstol = 1e-6, reltol = 1e-3, dt = nothing, kwargs...)
        u0m = u0 isa AbstractMatrix ? Float32.(permutedims(u0)) : reshape(Float32.(u0), 1, :)
        N = size(u0m, 1)
        h = handle_for(prob.f, alg, sensealg, prob.tspan, saveat, dt, abstol, reltol, N)
        out, status = forward(h, flat32(p), u0m)
        ts = saveat isa Number ? collect(prob.tspan[1]:saveat:prob.tspan[2]) : collect(Float64, saveat)
        sol = N == 1 ? B200Solution(eltype(u0).(out[1, :, :]), ts, status) : out
        function b200_pullback(Δ)
            Δ3 = N == 1 ? reshape(Float32.(Array(Δ)), 1, h.d, h.nsave) : Float32.(Δ)
            gθ, gu0 = pullback(h, Δ3, N)
            (nothing, nothing, N == 1 ? eltype(u0).(vec(gu0)) : permutedims(gu0), unflat(p, gθ), ntuple(_ -> nothing, length(args))...)
        end
        sol, b200_pullback
    end
end

# ---- fused trajectory-matching loss (one call per optimiser iteration) and the on-device ADAM loop -------------------------
"""L = sum(abs2, w .* (data .- pred)) and dL/dtheta in one call (b200ude_loss_gradient_host): scenario_1.jl:91-94."""
function loss_gradient(h::Handle, θ::Vector{Float32}, u0::Matrix{Float32}, data::Array{Float32,3})
    N = size(u0, 1); g = Vector{Float32}(undef, h.P); L = Ref{Float64}(0)
    GC.@preserve θ u0 data g check(h.ptr, ccall((:b200ude_loss_gradient_host, lib), Int32,
        (Ptr{Cvoid}, Ptr{Float32}, Ptr{Float32}, Ptr{Float32}, Csize_t, Ref{Float64}, Ptr{Float32}, Ptr{Float32}),
        h.ptr, θ, u0, data, N, L, g, C_NULL))
    L[], g
end
b200_l2(h, θ, u0, data) = loss_gradient(h, flat32(θ), u0, data)[1]
function ChainRulesCore.rrule(::typeof(b200_l2), h, θ, u0, data)
    L, g = loss_gradient(h, flat32(θ), u0, data)
    L, Δ -> (NoTangent(), NoTangent(), unflat(θ, Δ .* g), NoTangent(), NoTangent())
end

"""`sciml_train(loss, θ, ADAM(η); cb, maxiters)` for the trajectory-matching loss with the whole iteration on the device
(b200ude_train_adam: forward + adjoint + reduce + ADAM replayed as one CUDA graph).  `u0`, `data` are CuArrays."""
function train_adam!(h::Handle, θ::Vector{Float32}, u0, data, opt::Adam, iters::Int; cb = (θ, l) -> false, chunk = 50)
    CUDA = Base.require(Main, :CUDA)
    opt.struct_size = sizeof(Adam)
    check(h.ptr, ccall((:b200ude_set_params, lib), Int32, (Ptr{Cvoid}, Ptr{Float32}, Csize_t, Int32, Ptr{Cvoid}), h.ptr, θ, h.P, HOST, C_NULL))
    check(h.ptr, ccall((:b200ude_adam_reset, lib), Int32, (Ptr{Cvoid}, Ptr{Cvoid}), h.ptr, C_NULL))
    hist = CUDA.zeros(Float32, chunk); done = 0
    while done < iters
        k = min(chunk, iters - done)
        check(h.ptr, ccall((:b200ude_train_adam, lib), Int32, (Ptr{Cvoid}, Ref{Adam}, Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Int32, Ptr{Cvoid}, Ptr{Cvoid}),
                           h.ptr, opt, pointer(u0), pointer(data), size(u0, 1), k, pointer(hist), C_NULL))
        done += k
        any(l -> cb(θ, l), Array(hist)[1:k]) && break          # the callback sees every recorded loss; halts at a chunk boundary
    end
    check(h.ptr, ccall((:b200ude_get_params, lib), Int32, (Ptr{Cvoid}, Ptr{Float32}, Csize_t, Int32, Ptr{Cvoid}), h.ptr, θ, h.P, HOST, C_NULL))
    θ
end

# ---------------------------------------------------------------------------------------------------------------------------
# Terminal-PDE path: highdim_pde/lambaem.jl:18-34   solve(TerminalPDEProblem(...), NNPDENS(u0, σᵀ∇u, opt = ADAM(η)); ...)
# (include/b200ude.h, b200ude_bsde_*).  g, f, μ, σ are closures in the script; the device path knows the script's family
#   μ = 0, σ = s I, f = -λ |σᵀ∇u|², g(X) = log(a + b |X|²)
# so the shim takes them as a tagged struct.  Source only (no `julia` in the build image).
struct HJB; λ::Float64; s::Float64; a::Float64; b::Float64; end
HJB(; λ = 1.0, s = sqrt(2.0), a = 0.5, b = 0.5) = HJB(λ, s, a, b)

mutable struct BsdeDesc
    struct_size::UInt32; device::Int32; dtype::Int32; dim::Int32; hidden::Int32; n_steps::Int32
    T::Float64; lambda::Float64; sigma::Float64; g_a::Float64; g_b::Float64
    x0::Ptr{Float64}; max_paths::UInt64
end

"""`solve_nnpdens(HJB(), x0, tspan, u0, σᵀ∇u; opt = Adam(0.03), maxiters = 500, trajectories = 100, dt = T/20, seed = 1, T = Float32)`:
`u0`, `σᵀ∇u` are the script's Flux chains (`Dense(d, hls, relu)` ... ); their parameters are read with `Flux.destructure`
(per layer vec(W), then b: the ABI's order), trained on the device and written back.  Returns u0(x0) (the script's `ans`)."""
function solve_nnpdens(fam::HJB, x0::AbstractVector, tspan, u0, σᵀ∇u; opt::Adam, maxiters = 500, trajectories = 100,
                       dt = (tspan[2] - tspan[1]) / 20, seed = 1, device = 0, T::Type = Float32, destructure)
    d = length(x0); θu, reu = destructure(u0); θz, rez = destructure(σᵀ∇u)
    # length(θu) = d h + h + h² + h + h + 1 = h² + (d + 3) h + 1  ->  h
    hls = Int(round((-(d + 3) + sqrt((d + 3)^2 - 4 * (1 - length(θu)))) / 2))
    x0d = Float64.(x0)
    desc = BsdeDesc(0, device, T === Float64 ? 1 : 0, d, hls, round(Int, (tspan[2] - tspan[1]) / dt), Float64(tspan[2]), fam.λ, fam.s, fam.a, fam.b,
                    pointer(x0d), trajectories)
    desc.struct_size = sizeof(BsdeDesc)
    h = Ref{Ptr{Cvoid}}(C_NULL)
    GC.@preserve x0d begin
        rc = ccall((:b200ude_bsde_create, lib), Int32, (Ref{BsdeDesc}, Ref{Ptr{Cvoid}}), desc, h)
    end
    rc == 0 || error(unsafe_string(ccall((:b200ude_bsde_last_error, lib), Cstring, (Ptr{Cvoid},), C_NULL)))
    bcheck(rc) = rc == 0 || error(unsafe_string(ccall((:b200ude_bsde_last_error, lib), Cstring, (Ptr{Cvoid},), h[])))
    try
        θ = T.(vcat(θu, θz)); P = length(θ)
        bcheck(ccall((:b200ude_bsde_set_params, lib), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Int32), h[], θ, P, HOST))
        opt.struct_size = sizeof(Adam)
        bcheck(ccall((:b200ude_bsde_train_adam, lib), Int32, (Ptr{Cvoid}, Ref{Adam}, Csize_t, Int32, UInt64, Ptr{Cvoid}, Ptr{Cvoid}),
                     h[], opt, trajectories, maxiters, seed, C_NULL, C_NULL))
        bcheck(ccall((:b200ude_bsde_get_params, lib), Int32, (Ptr{Cvoid}, Ptr{Cvoid}, Csize_t, Int32), h[], θ, P, HOST))
        u0t = reu(θ[1:length(θu)])                       # the trained networks, as Flux chains again
        return first(u0t(T.(x0))), u0t, rez(θ[length(θu)+1:end])
    finally
        ccall((:b200ude_bsde_destroy, lib), Cvoid, (Ptr{Cvoid},), h[])
    end
end

end # module
