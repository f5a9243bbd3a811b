/*
 * b200ude.h -- C ABI of the H100-native (sm_90a) UDE training path.
 *
 * This is the drop-in boundary for ONE hot path of
 * ChrisRackauckas/universal_differential_equations: the forward solve of a
 * universal differential equation (known physics + embedded dense chain) for an
 * ensemble of trajectories and its interpolating-adjoint gradient.  The
 * reference has no FFI of its own: the seam is Julia dispatch on
 *     concrete_solve(prob::ODEProblem, Tsit5()/Vern7(), u0, p; saveat, abstol,
 *                    reltol, sensealg = InterpolatingAdjoint(autojacvec = ReverseDiffVJP()))
 *         SEIR_exposure/seir_exposure.jl:137-141, FisherKPP/Fisher-KPP-CNN.jl:136,
 *         LotkaVolterra/scenario_1.jl:82-88
 * and its reverse rule (DiffEqSensitivity._concrete_solve_adjoint), driven by
 *     DiffEqFlux.sciml_train(loss, theta, opt; cb, maxiters)
 *         seir_exposure.jl:160-161, Fisher-KPP-CNN.jl:236-238.
 * A Julia shim (INTEGRATION.md) defines those methods on top of the entry
 * points below with `ccall`; the Python mirror in
 * universal_differential_equations_b200/sciml.py binds the same symbols with
 * ctypes and is what the tests and bench.py exercise.
 *
 * Conventions
 *  - every function returns int32_t: 0 = OK, <0 usage error, >0 CUDA runtime error
 *    (message via b200ude_last_error); nothing throws or longjmps across the ABI.
 *  - all arrays are plain pointers + sizes; the caller owns every array it passes;
 *    the handle owns theta's device copy, the stored forward solution and scratch.
 *  - ensemble layouts are trajectory-fastest (structure of arrays):
 *        u0 [d][N]      out / data / dL_dout [n_save][d][N]      grad_u0 [d][N]
 *    i.e. a Julia Array of size (N, d) / (N, d, n_save).
 *  - theta is the reference's own flat layout: [n_prefix trainable physics scalars |
 *    per dense layer: vec(W) column-major (W is out x in), then b | n_suffix scalars]
 *    (Lux ComponentVector scenario_1.jl:113, DiffEqFlux initial_params
 *    seir_exposure.jl:115, Flux.destructure Fisher-KPP-CNN.jl:106).
 *  - `stream` is a cudaStream_t passed as void* (NULL = default stream); calls taking a
 *    stream are asynchronous with respect to the host unless stated otherwise.
 *  - a handle is not thread-safe; use one handle per host thread and device.  The default kernels of the LV 2-32-32-2 chain
 *    (warp-collective family) and the fp64 kernels read theta from the handle's own device copy: any number of such handles
 *    can be in flight on a device.  The other kernel families read the active handle's theta and tables from the constant
 *    bank, so work of DIFFERENT handles of those kinds on one device must be stream-ordered (not concurrent).
 *  - the interpolating adjoint of a Vern7 handle runs over a Tsit5 re-solve from the same u0 with the same step / tolerances
 *    by default, and an adaptive Vern7 solve treats the save times as tstops: with the fused L2 entry point the reported loss is that of the re-solve.  With B200UDE_FLAG_VERN7_DENSE
 *    (below) it runs over the Vern7 solve's own lazy 7th-order dense output instead, and an adaptive Vern7 solve fills its
 *    save times from that interpolant rather than stopping at them -- the call of seir_exposure.jl:137-141 as written.
 *    The discrete adjoint of a Vern7 handle differentiates the Vern7 solve itself.
 */
#ifndef B200UDE_H
#define B200UDE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200UDE_ABI_VERSION 1

/* dtype */
#define B200UDE_F32 0
#define B200UDE_F64 1 /* double precision: EVERY device array of the calls (theta, u0, out, data, dL_dout, grad_theta, grad_u0, loss) is
                        * double.  Runtime-shape kernels for the LV / SEIR / NODE forms, Tsit5 and Vern7, fixed step and adaptive,
                        * and for the Fisher-KPP UPDE with adaptive Tsit5, or adaptive Vern7 with the discrete adjoint (fixed-step
                        * Fisher-KPP is fp32 only); interpolating adjoint, and the discrete adjoint of fixed-step Tsit5 / Vern7 and
                        * adaptive Vern7 -- the precision the reference's scenario 1 / 2, SEIR and Fisher-KPP scripts run in (Float64).  Entry points: create / set_params / get_params / forward / adjoint / adjoint_l2;
                        * the host-buffer, ADAM and peer entry points return B200UDE_EUNSUPPORTED for such handles. */

/* model kinds: the UDE right-hand sides of the reference */
#define B200UDE_MODEL_LV 0   /* du1 = a1*u1 + NN1(u), du2 = -a2*u2 + NN2(u)   scenario_1.jl:69-73,
                                a2 trainable (n_prefix=1) scenario_2.jl:90-95, a1,a2 trainable (n_prefix=2)
                                hudson_bay.jl:85-91; consts = {p_[1], p_[4]} */
#define B200UDE_MODEL_SEIR 1 /* 7-state exposure UDE, NN([S/N, I, D/N])      seir_exposure.jl:117-130;
                                consts = F,beta0,alpha,kappa,mu,sigma,gamma,d,lambda (:33) */
#define B200UDE_MODEL_FKPP 2 /* pointwise reaction net + D0 * 3-tap periodic stencil, n_suffix = 5
                                Fisher-KPP-CNN.jl:111-126, scenario_3.jl:103-114 */
#define B200UDE_MODEL_NODE 3 /* du = NN(u) */
#define B200UDE_MODEL_SEIR_NODE 4 /* the SEIR script's black-box baseline dudt_node: dS,dE,dI,dR,dD = first five outputs of
                                     NN([S/N,E,I,R,N,D/N,C]), dN = -mu N, dC = sigma E   seir_exposure.jl:52-64; consts as MODEL_SEIR */
#define B200UDE_MODEL_FORCED 5 /* forced neural ODE with a readout network (NonNewtonianFluids/FENEP.jl:41-62):
                                    du = f1([u; gamma(t)]),  readout y = f0([u; gamma(t)]),
                                    gamma_n(t) = sum_j A_jn cos(w_jn t + phi_jn), per-trajectory coefficients (b200ude_set_forcing).
                                  Descriptor: state_dim = d; consts[0] = L0 (layers of f0), consts[1] = J (harmonics, 1..4),
                                  n_consts = 2; n_layers = L0 + L1; widths[0 .. L0] = f0 (d+1 -> ... -> r), then
                                  widths[L0+1 .. L0+L1+1] = f1 (d+1 -> ... -> d), so L0 + L1 <= 5; acts[] in the same order
                                  (f0's then f1's).  theta = f0's layers then f1's, each vec(W) column-major then b
                                  (Flux.params(f0, f1), FENEP.jl:98); n_prefix = n_suffix = 0.  Envelope: widths <= 64, d + 1 <= 8,
                                  r <= 8, P <= 12288 in fp32.
                                  Rows: out, data and dL_dout have d + r rows per save, [n_save][d + r][N]: rows 0..d-1 the
                                  states, rows d..d+r-1 the readout at the saved states; grad_u0 stays [d][N]; n_loss_weights
                                  is 0 or d + r.  Tsit5, fixed step or adaptive, interpolating adjoint, fp32 and fp64 (the
                                  interpolating adjoint stands for the reference's Tracker gradient through the solver; the two
                                  agree to the solve tolerance).  The fused L2 recomputes the readout from the saved state.
                                  Vern7, RKC2, the discrete adjoint and the dense flags return B200UDE_EUNSUPPORTED. */
#define B200UDE_MODEL_OPERATOR 6 /* wide-state operator UDE (Climate/NeuralPDE/npde.jl:75-78):  du = D1 * NN(u) + D2 * u,
                                    NN: widths[0] = d -> ... -> widths[n_layers] = m; D1 (d x m) and D2 (d x d) fixed, column-major,
                                    set by b200ude_set_operators.  Envelope: d 1..64, every width 1..64, 1..5 layers, activations
                                    identity / tanh / rbf; n_prefix = n_suffix = n_consts = 0 (adaptive RKC2: n_consts = 1,
                                    consts[0] = eigen_est); n_loss_weights 0, or d when d <= 16.
                                    theta = per layer vec(W) then b (Flux.destructure).  A warp integrates one trajectory.
                                    Tsit5 fixed step or adaptive, RKC2 fixed step (2..64 stages) or adaptive (each step takes the
                                    fewest stages, up to n_stages, that are stable for h * eigen_est; eigen_est finite and > 0),
                                    interpolating adjoint, fp32 and fp64.  Vern7, the discrete adjoint and the dense flags return B200UDE_EUNSUPPORTED;
                                    B200UDE_FLAG_APPROX_TANH is accepted and ignored.  create returns B200UDE_EUNSUPPORTED when the
                                    staged operators, theta and one warp's gradient vector exceed the device's shared memory. */

/* activations of the dense chain */
#define B200UDE_ACT_IDENTITY 0
#define B200UDE_ACT_TANH 1
#define B200UDE_ACT_RBF 2 /* exp(-x^2), scenario_1.jl:59 */

/* solver (OrdinaryDiffEq algorithm the reference passes to solve/concrete_solve) */
#define B200UDE_TSIT5 0
#define B200UDE_VERN7 1
#define B200UDE_RKC2 2 /* second-order Runge-Kutta-Chebyshev with desc.n_stages stages per step: the closed-form stabilised explicit
                          method of the class of ROCK2 (Climate/NeuralPDE/npde.jl:61,82; ROCK2's own coefficient tables are not in the
                          reference); real stability interval ~ 0.65 n_stages^2; dense output = cubic Hermite; the interpolating
                          adjoint steps lambda backwards with RKC2 itself.  Fisher-KPP UPDE (1-16-16-1 chain, even grids), fixed step;
                          B200UDE_MODEL_OPERATOR, fixed step, or adaptive (ROCK2(eigen_est = rho) without dt): consts[0] = rho, an
                          upper bound of the spectral radius of df/du, n_consts = 1, n_stages = the cap on stages per step; each
                          step takes the fewest stages s with stability interval >= 1.05 h rho, the RKC error estimate and the
                          PI controller pick h, and the replay adjoint steps each recorded step with its own s */

/* sensealg */
#define B200UDE_INTERPOLATING_ADJOINT 0 /* InterpolatingAdjoint(autojacvec = ReverseDiffVJP())  seir_exposure.jl:71,140 */
#define B200UDE_DISCRETE_ADJOINT 1      /* exact gradient of the discrete scheme, the accepted step sequence held fixed, by reverse
                                           accumulation through the stages of every step: the quantity ForwardDiffSensitivity()
                                           computes in forward mode (scenario_1.jl:84-87, scenario_2.jl:106-108, hudson_bay.jl:99-102).
                                           Fixed-step Tsit5, fixed-step Vern7 and adaptive Vern7 on the LV / SEIR / SEIR_NODE /
                                           NODE forms, and adaptive Vern7 on the Fisher-KPP UPDE (scenario_3.jl:121-126), fp32 and
                                           fp64.  An adaptive Vern7 solve treats the save times as tstops by default; with
                                           B200UDE_FLAG_DISCRETE_DENSE (below) it steps freely, fills the save times from Vern7's
                                           lazy interpolant as OrdinaryDiffEq's saveat does, and the adjoint differentiates the
                                           interpolated saves too.  The fused L2 reads the saved states of the solve itself
                                           (recorded step ends, or `out` with the flag), so the loss reported is that solve's.
                                           Not for adaptive Tsit5 (its saveat values come from the interpolant), fixed-step
                                           Fisher-KPP or RKC2. */

/* memory space of a pointer argument */
#define B200UDE_HOST 0
#define B200UDE_DEVICE 1

/* flags */
#define B200UDE_FLAG_APPROX_TANH 1u /* tanh.approx.f32 (2^-11 rel. error) instead of the ex2/rcp form.  Honoured by the kernels
                                       of the LV 2-32-32-2 chain (warp-collective, tensor-core, packed, adaptive), of the SEIR
                                       3-64-64-1 chain (fixed-step Tsit5, Vern7, adaptive) and of the Fisher-KPP 1-16-16-1 chain
                                       (Tsit5, RKC2).  The LV 2-5-5-5-2, runtime-shape and fp64 kernels ignore it: their results
                                       are bitwise those without the flag. */
#define B200UDE_FLAG_VERN7_DENSE 2u /* Vern7 with its lazy 7th-order dense output (OrdinaryDiffEq's six extra stages and
                                       interpolation polynomials), for solver = B200UDE_VERN7 with the interpolating adjoint on the
                                       LV / SEIR / SEIR_NODE / NODE forms, fp32 and fp64, fixed step and adaptive:
                                       - adaptive: the steps stop only at the end of tspan; a save time inside a step is evaluated
                                         with the interpolant, one on a step end takes the step-end state (OrdinaryDiffEq's saveat);
                                       - fixed step: saves at step ends as without the flag, so the forward output is the same;
                                       - the interpolating adjoint runs over the Vern7 forward's own dense output (no Tsit5 re-solve):
                                         b200ude_adjoint_l2 reports the loss of the states b200ude_forward returned.  With adaptive = 1
                                         `out` must stay valid until the matching adjoint call (the fused L2 reads it).
                                       Every such handle, the SEIR 3-64-64-1 chain included, runs on the runtime-shape kernels
                                       (vern7_dense.cuh).  B200UDE_EUNSUPPORTED with the discrete adjoint, Tsit5, RKC2 or the
                                       Fisher-KPP UPDE. */
#define B200UDE_FLAG_DISCRETE_DENSE 4u /* the discrete adjoint through Vern7's interpolated saves, for solver = B200UDE_VERN7 with
                                       sensealg = B200UDE_DISCRETE_ADJOINT on the LV / SEIR / SEIR_NODE / NODE forms, fp32 and fp64:
                                       - adaptive: the forward is that of B200UDE_FLAG_VERN7_DENSE (steps stop only at the end of
                                         tspan, a save time inside a step comes from the interpolant, one on a step end takes the
                                         step-end state), and the discrete adjoint differentiates exactly that with the accepted
                                         step sizes held fixed: through the interpolation weights and the six extra stages of every
                                         step that holds a save time (vern7_dense_discrete.cuh).  This is
                                         solve(prob, Vern7(); saveat, abstol, reltol, sensealg = ForwardDiffSensitivity()) of
                                         scenario_1.jl:84-87, scenario_2.jl:106-108, hudson_bay.jl:99-102 as OrdinaryDiffEq steps it.
                                         `out` must stay valid until the matching adjoint call (the fused L2 reads it);
                                       - fixed step: saves are step ends; the flag is accepted and the results are bitwise those
                                         without it.
                                       B200UDE_EUNSUPPORTED with the interpolating adjoint, together with B200UDE_FLAG_VERN7_DENSE,
                                       with Tsit5, RKC2 or the Fisher-KPP UPDE. */
#define B200UDE_FLAG_CHECKPOINT 8u /* InterpolatingAdjoint(checkpointing = true): a checkpointed step record for adaptive Tsit5 with
                                       the interpolating adjoint on the Fisher-KPP UPDE (B200UDE_MODEL_FKPP, adaptive = 1), fp32 and
                                       fp64, every reaction chain and grid that configuration accepts (the 1-16-16-1 chain included).
                                       - the forward runs the same steps and returns bitwise the same out and status; it keeps u_n
                                         only every K accepted steps and the size of every accepted step, no stage derivatives;
                                       - the adjoint takes the segments of K steps last to first, recomputes each one's states and
                                         stages from its checkpoint with the recorded step sizes, and replays it as without the flag:
                                         the gradients are bitwise those without the flag, for about one more evaluation of the
                                         accepted steps' right-hand sides per adjoint.
                                       K = max(1, round(sqrt(max_steps / 7))).  Record per trajectory, in reals:
                                       (ceil(max_steps / K) + 1 + 7K + 2) * state_dim + (2 max_steps + 1) (checkpoints, scratch of one
                                       segment, step sizes and step times) instead of (7 max_steps + 2) * state_dim + max_steps + 1;
                                       b200ude_device_bytes reports it.  Deviation from SciMLSensitivity: its checkpointed adjoint
                                       re-solves each interval between checkpoints with error control, so its gradient moves by about
                                       the tolerance; here the forward's own accepted steps are replayed with their recorded sizes,
                                       so nothing moves.  B200UDE_EUNSUPPORTED on every other configuration: fixed step, Vern7, RKC2,
                                       the discrete adjoint, and every other model. */

/* per-trajectory status words written by b200ude_forward */
#define B200UDE_TRAJ_OK 0
#define B200UDE_TRAJ_NONFINITE 1
#define B200UDE_TRAJ_MAXSTEPS 2 /* adaptive: more than max_steps accepted steps needed */

/* error codes */
#define B200UDE_OK 0
#define B200UDE_EINVAL (-1)       /* bad descriptor / argument */
#define B200UDE_EUNSUPPORTED (-2) /* configuration has no sm_90a kernel in this build */
#define B200UDE_ESTATE (-3)       /* call order violated (e.g. adjoint before forward) */
#define B200UDE_ENOMEM (-4)
#define B200UDE_ENODEVICE (-5)    /* no CUDA device / not an sm_90 part */

#define B200UDE_MAX_LAYERS 6

typedef struct b200ude_handle b200ude_handle;

typedef struct b200ude_desc {
    uint32_t struct_size; /* = sizeof(b200ude_desc); checked */
    int32_t device;       /* CUDA device ordinal */
    int32_t dtype;        /* B200UDE_F32 | B200UDE_F64 */
    int32_t model;        /* B200UDE_MODEL_* */
    int32_t state_dim;    /* d */
    int32_t n_layers;     /* dense layers of the embedded chain */
    int32_t widths[B200UDE_MAX_LAYERS + 1]; /* widths[0] = chain input, widths[n_layers] = chain output */
    int32_t acts[B200UDE_MAX_LAYERS];
    int32_t n_prefix;     /* trainable physics scalars before the chain in theta */
    int32_t n_suffix;     /* trainable scalars after the chain in theta */
    int32_t n_consts;
    double consts[16];    /* fixed physics constants */
    int32_t solver;       /* B200UDE_TSIT5 | B200UDE_VERN7 | B200UDE_RKC2 */
    int32_t sensealg;     /* B200UDE_INTERPOLATING_ADJOINT | B200UDE_DISCRETE_ADJOINT */
    double t0;            /* tspan[1], the absolute start time.  Every kernel runs on s = t - t0, so step and save times keep the
                             float spacing of the span, whatever |t0| (at t0 = 1900, ulp(t) = 1.2e-4 in fp32).  The autonomous
                             models (LV, SEIR, NODE, Fisher-KPP, operator) never read t: their results do not depend on t0, bit
                             for bit.  B200UDE_MODEL_FORCED reads t in its forcing: b200ude_set_forcing folds w_j t0 into each
                             phase, phi_j + w_j t0 reduced mod 2 pi in double, so gamma(t) = sum A_j cos(w_j s + phi_j') is the
                             forcing at absolute t; with t0 = 0 the coefficients are used as given. */
    double dt;            /* fixed step (adaptive = false); saveat = t0 + i*save_every*dt */
    int32_t n_steps;      /* number of steps; tspan[2] = t0 + n_steps*dt */
    int32_t save_every;   /* save the state every this many steps (and at t0) */
    double abstol, reltol; /* adaptive stepping tolerances (used when adaptive = 1) */
    int32_t n_loss_weights; /* 0 => all ones; else = state_dim */
    double loss_weights[16]; /* per-component weight of the fused L2 loss (seir_exposure.jl:146 uses rows 2:4) */
    uint64_t max_trajectories; /* capacity: scratch is sized for this many trajectories */
    uint32_t flags;
    int32_t adaptive;   /* 0: fixed step dt (adaptive = false). 1: Tsit5 with OrdinaryDiffEq's PI controller, abstol / reltol;
                           saveat = t0 + i*save_every*dt, i = 0..n_steps/save_every (dt only defines the save grid).
                           LV / SEIR / NODE forms (Tsit5 or Vern7) and the Fisher-KPP UPDE (Tsit5, or Vern7 with the discrete
                           adjoint; its error norm is taken over the whole grid, as OrdinaryDiffEq's default norm over the state
                           vector), fp32 and fp64.  On B200UDE_MODEL_OPERATOR: Tsit5, or RKC2 with eigen_est in consts[0] */
    int32_t max_steps;  /* adaptive: capacity of ACCEPTED steps per trajectory (status 2 when exceeded) */
    int32_t n_stages;   /* B200UDE_RKC2: stages per step (2..64); choose dt * spectral_radius <= 0.65 n_stages^2.  0 otherwise */
} b200ude_desc;

int32_t b200ude_version(void);

/* Message of the last error on this handle (h may be NULL: last create() error of the calling thread). */
const char *b200ude_last_error(const b200ude_handle *h);

int32_t b200ude_create(const b200ude_desc *desc, b200ude_handle **out);
void b200ude_destroy(b200ude_handle *h);

/* length P of theta, number of saved time points, bytes of device memory held by the handle */
size_t b200ude_num_params(const b200ude_handle *h);
size_t b200ude_num_save(const b200ude_handle *h);
size_t b200ude_device_bytes(const b200ude_handle *h);

/* theta[P] (float) from host or device memory -> the handle's device copy. */
int32_t b200ude_set_params(b200ude_handle *h, const void *theta, size_t P, int32_t mem, void *stream);

/* FORCING of a B200UDE_MODEL_FORCED handle: coef [3J][N] in the handle's dtype (host or device memory per `mem`), rows
 * (A_j, w_j, phi_j) for j = 0..J-1, so that gamma_n(t) = sum_j A_jn cos(w_jn t + phi_jn).  The handle keeps a device copy
 * (capacity max_trajectories) that forward, solve_host, loss_gradient_host and train_adam read; calling them with more
 * trajectories than were last set is B200UDE_ESTATE.  Stream-ordered on `stream`.  Any other model: B200UDE_EUNSUPPORTED. */
int32_t b200ude_set_forcing(b200ude_handle *h, const void *coef, size_t N, int32_t mem, void *stream);

/* OPERATORS of a B200UDE_MODEL_OPERATOR handle: D1 [d x m] and D2 [d x d], column-major, in the handle's dtype (host or device
 * memory per `mem`).  D2 = NULL is a zero D2 (D1 = I, D2 = NULL: a plain wide neural ODE).  The handle keeps its own padded
 * device copies; forward or adjoint before the first call is B200UDE_ESTATE.  Stream-ordered on `stream`.  Any other model:
 * B200UDE_EUNSUPPORTED. */
int32_t b200ude_set_operators(b200ude_handle *h, const void *D1, const void *D2, int32_t mem, void *stream);

/* FORWARD  (replaces: the UDE RHS closure + OrdinaryDiffEq perform_step! loop behind
 * concrete_solve(prob, Tsit5(), u0, p; saveat, ...), one trajectory per ensemble member).
 * u0 [d][N], out [n_save][d][N], status [N] (may be NULL): DEVICE pointers.
 * Also stores the dense output (stage derivatives) the adjoint interpolates.  With adaptive = 1 `out` must stay valid
 * until the matching adjoint call (the fused L2 adjoint reads the interpolated saved states from it). */
int32_t b200ude_forward(b200ude_handle *h, const void *u0, size_t N, void *out, int32_t *status,
                        void *stream);

/* ADJOINT  (replaces: DiffEqSensitivity InterpolatingAdjoint backward solve + ReverseDiffVJP).
 * Uses the forward solution stored by the last b200ude_forward on this handle.
 * dL_dout [n_save][d][N]: cotangent of the saved states (the Zygote pullback's Delta).
 * grad_theta [P]: SUM over the N trajectories (overwritten). grad_u0 [d][N] or NULL. DEVICE pointers. */
int32_t b200ude_adjoint(b200ude_handle *h, const void *dL_dout, void *grad_theta, void *grad_u0,
                        void *stream);

/* ADJOINT with the L2 trajectory-matching loss fused (scenario_1.jl:91-94, seir_exposure.jl:144-147):
 * L = sum_n sum_i sum_k w_k (out - data)^2, Delta = 2 w (out - data) formed in-kernel.
 * data [n_save][d][N]; loss: float[1] (sum over the ensemble, overwritten). DEVICE pointers. */
int32_t b200ude_adjoint_l2(b200ude_handle *h, const void *data, void *loss, void *grad_theta,
                           void *grad_u0, void *stream);

/* HOST-BUFFER entry points (what a host-language binding calls with ordinary arrays): copy
 * inputs host->device, run the kernels, copy results back, synchronise.  Pinned host memory makes
 * the copies asynchronous; pageable memory works but is slower. */
int32_t b200ude_solve_host(b200ude_handle *h, const void *theta, const void *u0, size_t N, void *out,
                           int32_t *status);
int32_t b200ude_loss_gradient_host(b200ude_handle *h, const void *theta, const void *u0,
                                   const void *data, size_t N, double *loss, void *grad_theta,
                                   void *grad_u0 /* may be NULL */);

/* ON-DEVICE OPTIMISER  (replaces the ADAM phase of DiffEqFlux.sciml_train(loss, theta, ADAM(eta); cb, maxiters)
 * seir_exposure.jl:160, Fisher-KPP-CNN.jl:236, Optimization.solve(optprob, ADAM(0.1); maxiters) scenario_1.jl:114,
 * for the trajectory-matching loss  L = loss_scale * sum w (u - data)^2 + l2_reg * sum theta[n_prefix:]^2
 * (the L2 term skips the n_prefix trainable physics rates, as scenario_2.jl:113 does with theta[2:end])
 * (scenario_1.jl:91-94; scenario_2.jl:113-116 divides by the number of points and adds the L2 term).
 * The update is Flux.ADAM: m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2,
 * theta -= eta * (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + eps); the moments and t live in the handle. */
typedef struct b200ude_adam {
    uint32_t struct_size; /* = sizeof(b200ude_adam) */
    uint32_t reserved;
    double eta, beta1, beta2, eps; /* Flux defaults: 0.001, 0.9, 0.999, 1e-8 */
    double loss_scale;             /* 0 is read as 1 */
    double l2_reg;
} b200ude_adam;

/* the handle's current theta -> theta[P] (host: synchronises the stream; device: asynchronous) */
int32_t b200ude_get_params(b200ude_handle *h, void *theta, size_t P, int32_t mem, void *stream);
/* zero the ADAM moments and the step counter */
int32_t b200ude_adam_reset(b200ude_handle *h, void *stream);
/* one ADAM update of the handle's theta with a caller-supplied DEVICE gradient [P] (e.g. after an all-reduce over GPUs);
 * loss_scale / l2_reg are applied to it as above */
int32_t b200ude_adam_step(b200ude_handle *h, const b200ude_adam *opt, const void *grad_theta, void *stream);
/* `iters` full iterations without a host round trip: forward, fused-L2 adjoint, fixed-order reduce, ADAM update -- the first
 * launched directly, the rest as replays of one captured CUDA graph.  u0 [d][N], data [n_save][d][N]: DEVICE pointers.
 * loss_history: DEVICE float[iters] or NULL; slot i = loss at the pre-update theta of iteration i (what the reference's
 * callback records).  stream NULL = the handle's own stream, synchronised before returning.  With peers attached
 * (b200ude_peer_attach, below) every iteration uses the loss and gradient summed over ALL ranks: the call is then a collective,
 * every rank runs the same iterations in lock step and applies the identical update to its replica of theta. */
int32_t b200ude_train_adam(b200ude_handle *h, const b200ude_adam *opt, const void *u0, const void *data, size_t N,
                           int32_t iters, void *loss_history, void *stream);

/* MULTI-GPU (one process per GPU; the ensemble shards, theta is replicated -- SURVEY.md section 8e).  The only exchange of
 * the path, the sum over ranks of [grad_theta (P); loss], can run inside the final reduction kernel over NVLink peer memory:
 * every rank exports an exchange buffer (CUDA IPC), the host program gathers the `world` handles in rank order by whatever
 * means it has (MPI, torch.distributed, a file), attaches, and synchronises all ranks once (a host barrier) before the first
 * call.  b200ude_adjoint_l2_allreduce is then b200ude_adjoint_l2 whose loss and grad_theta are the sums over ALL ranks
 * (bitwise identical on every rank); it is a collective: every rank must call it the same number of times.  grad_u0 stays
 * local.  Fixed-step handles only.  A peer that never arrives turns the results into NaN after ~2 s instead of hanging. */
#define B200UDE_PEER_HANDLE_BYTES 64
int32_t b200ude_peer_export(b200ude_handle *h, void *handle_out /* B200UDE_PEER_HANDLE_BYTES */);
int32_t b200ude_peer_attach(b200ude_handle *h, int32_t rank, int32_t world, const void *handles /* world x 64 bytes, rank order */);
int32_t b200ude_peer_detach(b200ude_handle *h);
int32_t b200ude_adjoint_l2_allreduce(b200ude_handle *h, const void *data, void *loss, void *grad_theta, void *grad_u0,
                                     void *stream);

/* SELF-TEST of a device building block (no reference counterpart): y[i] = the kernels' tanh (1 - 2 / (1 + 2^(2 log2(e) x)) with one
 * reciprocal per four values, the variant the warp-collective LV kernels use) for n device floats; the parity tests compare it
 * with tanh in fp64.  device = CUDA ordinal. */
int32_t b200ude_selftest_tanh(int32_t device, const void *x, void *y, size_t n, void *stream);

/* TERMINAL-PDE / SDE PATH (SURVEY.md section 8 f4, BASELINE config 5) -- replaces, for highdim_pde/lambaem.jl:18-34,
 *     solve(TerminalPDEProblem(g, f, mu, sigma, x0, tspan), NNPDENS(u0, sigmaT_grad_u, opt = ADAM(eta));
 *           maxiters, trajectories = m, alg = LambaEM(), ...)                                   [EXT NeuralNetDiffEq 1.1.0]
 * i.e. the deep-BSDE method: dX = mu dt + sigma dW, du = -f dt + z . dW with z = sigmaT_grad_u([X; t]) and u(0) = u0(x0), all
 * `trajectories` paths advanced together, loss = mean (g(X_T) - u_T)^2, reverse-mode gradient through the discretised solve,
 * Flux.ADAM on both networks; the solution is u0(x0).  Problem family of the script (Hamilton-Jacobi-Bellman):
 *     mu = 0, sigma = sigma I, f(X, u, z, p, t) = -lambda |z|^2, g(X) = log(g_a + g_b |X|^2)
 * Networks as in the script: u0 = Dense(d, hidden, relu), Dense(hidden, hidden, relu), Dense(hidden, 1);
 * sigmaT_grad_u = Dense(d + 1, hidden, relu) x3 -> Dense(hidden, d); theta = [u0 net; sigmaT_grad_u net], each layer vec(W)
 * (out x in, column-major) then b -- Flux.params order.  relu'(0) = 1 (Flux 0.9 / Tracker differentiating max(zero(x), x)).
 * Time stepping: Euler-Maruyama with the fixed step T / n_steps (LambaEM is EM with step-size control).  Brownian increments:
 * sqrt(dt) * Box-Muller(Philox4x32-10) with counter (path, component / 4, step, 0) and key = seed; iteration i of
 * b200ude_bsde_train_adam uses seed0 + i.  dtype selects float or double for every buffer of the calls.
 * Streams: these calls take no stream; they run on the handle's own stream and return when the work is complete.  Device arrays
 * handed in (theta, a gradient for b200ude_bsde_adam_step) must be ready -- finish or synchronise the producing stream first. */
typedef struct b200ude_bsde_handle b200ude_bsde_handle;
typedef struct b200ude_bsde_desc {
    uint32_t struct_size; /* = sizeof(b200ude_bsde_desc) */
    int32_t device;
    int32_t dtype;        /* B200UDE_F32 | B200UDE_F64 */
    int32_t dim;          /* d */
    int32_t hidden;       /* hls (the script: 10 + d) */
    int32_t n_steps;
    double T;             /* tspan = (0, T) */
    double lambda, sigma; /* f = -lambda |z|^2; sigma = sqrt(2) in the script */
    double g_a, g_b;      /* g(X) = log(g_a + g_b |X|^2); 0.5, 0.5 in the script */
    const double *x0;     /* HOST double[dim]; copied by create */
    uint64_t max_paths;   /* capacity (trajectories) */
} b200ude_bsde_desc;
int32_t b200ude_bsde_create(const b200ude_bsde_desc *desc, b200ude_bsde_handle **out);
void b200ude_bsde_destroy(b200ude_bsde_handle *h);
const char *b200ude_bsde_last_error(const b200ude_bsde_handle *h);
size_t b200ude_bsde_num_params(const b200ude_bsde_handle *h);
/* mem = B200UDE_HOST | B200UDE_DEVICE; set_params also zeroes the ADAM state */
int32_t b200ude_bsde_set_params(b200ude_bsde_handle *h, const void *theta, size_t P, int32_t mem);
int32_t b200ude_bsde_get_params(b200ude_bsde_handle *h, void *theta, size_t P, int32_t mem);
/* one evaluation at the handle's theta: loss[1], grad[P], u0[1] = u0(x0) (host or device pointers of the handle's dtype; NULL =
 * not wanted).  path_offset shifts the Philox path counter and total_paths (0 = n_paths) is the denominator of the mean, so
 * that ranks of a multi-GPU job evaluate disjoint paths and their losses / gradients simply add. */
int32_t b200ude_bsde_loss_gradient(b200ude_bsde_handle *h, size_t n_paths, uint64_t seed, uint64_t path_offset, size_t total_paths,
                                   void *loss, void *grad, void *u0);
/* `iters` NNPDENS iterations on the device (forward paths, loss, backward sweep, ADAM), the first launched directly, the rest
 * as replays of one CUDA graph.  loss_history / u0_history: DEVICE arrays [iters] of the handle's dtype or NULL; slot i = the
 * loss / u0(x0) at the pre-update theta of iteration i (what the script's `verbose` callback prints). */
int32_t b200ude_bsde_train_adam(b200ude_bsde_handle *h, const b200ude_adam *opt, size_t n_paths, int32_t iters, uint64_t seed0,
                                void *loss_history, void *u0_history);
/* device time of the last b200ude_bsde_train_adam call in ms (CUDA events on the handle's stream around all its iterations) */
double b200ude_bsde_last_train_ms(const b200ude_bsde_handle *h);
/* fp64 handles with dim <= 110 and hidden <= 111 run fused sweeps (csrc/bsde.cu; the weight-gradient products on a fused kernel
 * too when dim and hidden are both even, else on library GEMMs); other handles return B200UDE_EUNSUPPORTED.  ms[0..2] = device time
 * of the forward sweep, the cotangent sweep and the batched weight-gradient GEMMs of the last b200ude_bsde_loss_gradient call
 * (CUDA events on the handle's stream) */
int32_t b200ude_bsde_last_sweep_ms(b200ude_bsde_handle *h, double *ms);
/* one ADAM update with a caller-supplied DEVICE gradient [P] of the handle's dtype (multi-GPU: b200ude_bsde_loss_gradient on
 * every rank's path shard, all-reduce of the gradient, then this call on every rank) */
int32_t b200ude_bsde_adam_step(b200ude_bsde_handle *h, const b200ude_adam *opt, const void *grad);

#ifdef __cplusplus
}
#endif
#endif /* B200UDE_H */
