// ude_generic.cuh -- shape-generic (runtime widths / activations) UDE kernels, written once over the real type.
//
// Functional coverage for every recognised UDE form whose chain has no specialised kernel: any dense chain
// with widths <= 64 and <= 5 layers, models LV (0/1/2 trainable rates), SEIR (7 states, chain on
// [S/N, I, D/N], SEIR_exposure/seir_exposure.jl:117-130), SEIR_NODE (the script's black-box baseline, :52-64) and NODE:
// Tsit5 / Vern7, fixed step and PI-controlled, the saveat interpolant, the interpolating adjoint on the fixed grid and the
// replay of an adaptive solve (the discrete adjoint of the Tsit5 / Vern7 solves is in discrete_adjoint.cuh, the Fisher-KPP
// kernels in fkpp_adaptive.cuh / k_generic.cu).  One trajectory per thread, weights read with runtime indices, activations
// in per-thread local arrays, Tsit5 forward with dense output and the interpolating adjoint exactly as in the specialised
// kernels.  The ensemble-summed parameter gradient is reduced deterministically: every contribution is summed over the
// warp's lanes with a fixed shuffle tree and added by lane 0 into a per-warp shared-memory vector.  Correctness first: these
// kernels are ~10-30x slower per FLOP than lv32::tc and are reported as such (DESIGN.md section 4.3).
//
// The precision comes in through `Ops`, which carries only what differs between fp32 and fp64:
//   real, MAXD, the kernels' parameter structs Fwd / Adj / Adapt (params.h);
//   model(), D(), din(), dout(), n_layers(), n_prefix(), P(), width(l), woff(l), layer_act(l) -- the runtime chain descriptor,
//     each field read by value straight from the __constant__ symbol (reading through a reference to the descriptor compiled
//     the chain loops differently and moved the register allocation of every kernel that calls chain_fwd);
//   theta(i), consts(i), lossw(c) -- the parameters, the model constants and the loss weights (returned by reference, so that
//     the LV rate selection stays a select of the address and one load, as when the kernels named the symbols directly);
//   act(k, a) -- activation k at pre-activation a.
// k_generic.cu instantiates it in fp32 (Ops32: theta and the tables in the constant bank, the approximate MUFU activations),
// k_f64.cu in fp64 (Ops64: the shape and tables in one __constant__ struct, theta in the handle's device copy).  The reference
// runs its LV scenario 1 / 2 and SEIR scripts in Float64 (scenario_1.jl:62-66, seir_exposure.jl:114-115) with abstol = reltol =
// 1e-6 -- tolerances fp32 cannot honour on the SEIR state (1.4e7 next to 10); H100's fp64 rate is half its fp32 rate.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "params.h"
#include "step_control.cuh"
#include "tsit5.cuh"
#include "vern7.cuh"

namespace b200ude {

namespace generic {

constexpr int MAXW = 64;   // max layer width
constexpr int MAXL = 5;    // max dense layers
constexpr int MAXD = 8;    // max state dimension / chain input / chain output

// derivative of activation k from pre-activation a and output h
template <typename R>
__device__ __forceinline__ R actder_rt(int k, R a, R h)
{
    return k == ACT_TANH ? fma(-h, h, (R)1) : (k == ACT_RBF ? (R)-2 * a * h : (R)1);
}

// chain forward; when KEEP, stores every layer's output (hs[l+1]) and pre-activation (pre[l])
template <class Ops, bool KEEP>
__device__ __noinline__ void chain_fwd(const typename Ops::real *x, typename Ops::real *y, typename Ops::real (*hs)[MAXW],
                                       typename Ops::real (*pre)[MAXW])
{
    using R = typename Ops::real;
    R cur[MAXW], nxt[MAXW];
    const int L = Ops::n_layers();
    for (int i = 0; i < Ops::width(0); ++i) {
        cur[i] = x[i];
        if (KEEP) hs[0][i] = x[i];
    }
    for (int l = 0; l < L; ++l) {
        const int nin = Ops::width(l), nout = Ops::width(l + 1), wo = Ops::woff(l), act = Ops::layer_act(l);
        for (int j = 0; j < nout; ++j) {
            R a = Ops::theta(wo + nin * nout + j);
            for (int i = 0; i < nin; ++i) a = fma(Ops::theta(wo + i * nout + j), cur[i], a);
            const R h = Ops::act(act, a);
            nxt[j] = h;
            if (KEEP) { pre[l][j] = a; hs[l + 1][j] = h; }
        }
        for (int j = 0; j < nout; ++j) cur[j] = nxt[j];
    }
    for (int j = 0; j < Ops::width(L); ++j) y[j] = cur[j];
}

template <class Ops>
__device__ __forceinline__ void model_inputs(const typename Ops::real *u, typename Ops::real *x)
{
    using R = typename Ops::real;
    if (Ops::model() == MODEL_SEIR) {
        const R invN = (R)1 / u[4];
        x[0] = u[0] * invN; x[1] = u[2]; x[2] = u[5] * invN;
    } else if (Ops::model() == MODEL_SEIR_NODE) {   // [S/N, E, I, R, N, D/N, C]  seir_exposure.jl:58
        const R invN = (R)1 / u[4];
        x[0] = u[0] * invN; x[1] = u[1]; x[2] = u[2]; x[3] = u[3]; x[4] = u[4]; x[5] = u[5] * invN; x[6] = u[6];
    } else {
        for (int i = 0; i < Ops::din(); ++i) x[i] = u[i];
    }
}

template <class Ops>
__device__ __forceinline__ void model_rhs(const typename Ops::real *u_in, typename Ops::real *du)
{
    using R = typename Ops::real;
    // private register copy of the state: the chain's scratch arrays (x, y, and chain_fwd's own) live in local memory, and the
    // state is read again after the chain -- with the caller's array that read came back clobbered by x in the Vern7 adaptive
    // kernel (stack-slot sharing after inlining; found with a device printf), which sent every SEIR solve to max_steps
    R u[MAXD];
#pragma unroll
    for (int c = 0; c < MAXD; ++c) u[c] = c < Ops::D() ? u_in[c] : (R)0;
    R x[MAXD], y[MAXD];
    model_inputs<Ops>(u, x);
    chain_fwd<Ops, false>(x, y, nullptr, nullptr);
    if (Ops::model() == MODEL_LV) {
        R a1 = Ops::consts(0), a2 = Ops::consts(1);
        if (Ops::n_prefix() == 1) a2 = Ops::theta(0);
        if (Ops::n_prefix() == 2) { a1 = Ops::theta(0); a2 = Ops::theta(1); }
        du[0] = fma(a1, u[0], y[0]);
        du[1] = fma(-a2, u[1], y[1]);
    } else if (Ops::model() == MODEL_SEIR) {
        // seir_exposure.jl:117-130; consts = F, beta0, alpha, kappa, mu, sigma, gamma, d, lambda (:33)
        const R F = Ops::consts(0), b0 = Ops::consts(1), mu = Ops::consts(4), sg = Ops::consts(5), gm = Ops::consts(6), dd = Ops::consts(7),
                lm = Ops::consts(8);
        const R S = u[0], E = u[1], I = u[2], R_ = u[3], N = u[4], Dd = u[5];
        const R inf = b0 * S * F / N, z = y[0];
        du[0] = -inf - z - mu * S;
        du[1] = inf + z - (sg + mu) * E;
        du[2] = sg * E - (gm + mu) * I;
        du[3] = gm * I - mu * R_;
        du[4] = -mu * N;
        du[5] = dd * gm * I - lm * Dd;
        du[6] = sg * E;
    } else if (Ops::model() == MODEL_SEIR_NODE) {   // dS,dE,dI,dR,dD = first five chain outputs; dN = -mu N; dC = sigma E  (seir_exposure.jl:55-64)
        du[0] = y[0]; du[1] = y[1]; du[2] = y[2]; du[3] = y[3];
        du[4] = -Ops::consts(4) * u[4];
        du[5] = y[4];
        du[6] = Ops::consts(5) * u[1];
    } else {
        for (int k = 0; k < Ops::D(); ++k) du[k] = y[k];
    }
}

// sum v over the warp's lanes with a fixed tree and add it into this warp's shared gradient vector
template <typename R>
__device__ __forceinline__ void warp_acc(R *gw, int idx, R v, int lane)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) gw[idx] += v;
}

// chain VJP: dx = (dchain/dx)^T dy; this warp's gradient vector += w * (dchain/dtheta)^T dy (w per lane; all lanes participate)
template <class Ops>
__device__ __noinline__ void chain_vjp(const typename Ops::real *x, const typename Ops::real *dy, typename Ops::real w, typename Ops::real *dx,
                                       typename Ops::real *gw, int lane)
{
    using R = typename Ops::real;
    R y[MAXD];
    R hs[MAXL + 1][MAXW], pre[MAXL][MAXW];
    chain_fwd<Ops, true>(x, y, hs, pre);
    const int L = Ops::n_layers();
    R q[MAXW], qn[MAXW];
    for (int j = 0; j < Ops::width(L); ++j) q[j] = dy[j];
    for (int l = L - 1; l >= 0; --l) {
        const int nin = Ops::width(l), nout = Ops::width(l + 1), wo = Ops::woff(l), act = Ops::layer_act(l);
        for (int j = 0; j < nout; ++j) q[j] *= actder_rt(act, pre[l][j], hs[l + 1][j]);
        for (int i = 0; i < nin; ++i) {
            R sacc = (R)0;
            const R hi = hs[l][i];
            for (int j = 0; j < nout; ++j) {
                sacc = fma(Ops::theta(wo + i * nout + j), q[j], sacc);
                warp_acc(gw, wo + i * nout + j, w * q[j] * hi, lane);
            }
            qn[i] = sacc;
        }
        for (int j = 0; j < nout; ++j) warp_acc(gw, wo + nin * nout + j, w * q[j], lane);
        for (int i = 0; i < nin; ++i) q[i] = qn[i];
    }
    for (int i = 0; i < Ops::width(0); ++i) dx[i] = q[i];
}

// kl = (df/du)^T g ; this warp's gradient vector += sc * lv * (df/dtheta)^T g   (all lanes of the warp participate)
template <class Ops>
__device__ __forceinline__ void model_vjp(const typename Ops::real *u_in, const typename Ops::real *g_in, typename Ops::real sc,
                                          typename Ops::real lv, typename Ops::real *kl, typename Ops::real *gw, int lane)
{
    using R = typename Ops::real;
    R u[MAXD], g[MAXD];   // private register copies, read again after the chain (see model_rhs)
#pragma unroll
    for (int c = 0; c < MAXD; ++c) { u[c] = c < Ops::D() ? u_in[c] : (R)0; g[c] = c < Ops::D() ? g_in[c] : (R)0; }
    R x[MAXD], dy[MAXD], dx[MAXD];
    model_inputs<Ops>(u, x);
    const R w = sc * lv;   // quadrature weight, zero for padding lanes
    if (Ops::model() == MODEL_SEIR) dy[0] = g[1] - g[0];   // z enters dS with -, dE with +
    else if (Ops::model() == MODEL_SEIR_NODE) { dy[0] = g[0]; dy[1] = g[1]; dy[2] = g[2]; dy[3] = g[3]; dy[4] = g[5]; dy[5] = (R)0; dy[6] = (R)0; }
    else for (int m = 0; m < Ops::dout(); ++m) dy[m] = g[m];
    chain_vjp<Ops>(x, dy, w, dx, gw, lane);
    if (Ops::model() == MODEL_LV) {
        R a1 = Ops::consts(0), a2 = Ops::consts(1);
        if (Ops::n_prefix() == 1) a2 = Ops::theta(0);
        if (Ops::n_prefix() == 2) { a1 = Ops::theta(0); a2 = Ops::theta(1); }
        kl[0] = fma(a1, g[0], dx[0]);
        kl[1] = fma(-a2, g[1], dx[1]);
        if (Ops::n_prefix() == 1) warp_acc(gw, 0, w * (-u[1] * g[1]), lane);
        if (Ops::n_prefix() == 2) {
            warp_acc(gw, 0, w * (u[0] * g[0]), lane);
            warp_acc(gw, 1, w * (-u[1] * g[1]), lane);
        }
    } else if (Ops::model() == MODEL_SEIR) {
        const R F = Ops::consts(0), b0 = Ops::consts(1), mu = Ops::consts(4), sg = Ops::consts(5), gm = Ops::consts(6), dd = Ops::consts(7),
                lm = Ops::consts(8);
        const R S = u[0], N = u[4], Dd = u[5];
        const R cS = b0 * F / N, cN = -b0 * S * F / (N * N);
        kl[0] = g[0] * (-cS - mu) + g[1] * cS + dx[0] / N;
        kl[1] = g[1] * (-(sg + mu)) + g[2] * sg + g[6] * sg;
        kl[2] = g[2] * (-(gm + mu)) + g[3] * gm + g[5] * dd * gm + dx[1];
        kl[3] = g[3] * (-mu);
        kl[4] = g[0] * (-cN) + g[1] * cN + g[4] * (-mu) - dx[0] * S / (N * N) - dx[2] * Dd / (N * N);
        kl[5] = g[5] * (-lm) + dx[2] / N;
        kl[6] = (R)0;
    } else if (Ops::model() == MODEL_SEIR_NODE) {
        const R S = u[0], N = u[4], Dd = u[5], mu = Ops::consts(4), sg = Ops::consts(5);
        kl[0] = dx[0] / N;
        kl[1] = dx[1] + sg * g[6];
        kl[2] = dx[2];
        kl[3] = dx[3];
        kl[4] = dx[4] - mu * g[4] - dx[0] * S / (N * N) - dx[5] * Dd / (N * N);
        kl[5] = dx[5] / N;
        kl[6] = dx[6];
    } else {
        for (int k = 0; k < Ops::D(); ++k) kl[k] = dx[k];
    }
}

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(typename Ops::Fwd p)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    const int D = Ops::D();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R dt = p.dt;
    R u[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](R *base, int row, const R *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    model_rhs<Ops>(u, k[0]);
    store(p.dense, 0, k[0]);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fma((R)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fma(dt, acc, u[c]);
            }
            if (i == 6) for (int c = 0; c < D; ++c) u[c] = g[c];
            model_rhs<Ops>(g, k[i]);
            store(p.dense, s * 6 + i, k[i]);
        }
        store(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store(p.out, isave, u); ++isave; }
        for (int c = 0; c < D; ++c) k[0][c] = k[6][c];
    }
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = ok ? 0 : 1;
    }
}

// Vern7 fixed-step forward solve (solve(prob, Vern7(); saveat, adaptive = false)): 9 stages per step, no FSAL.
// By default the interpolating adjoint of a Vern7 solve runs over a Tsit5 re-solve (b200ude.cu); with B200UDE_FLAG_VERN7_DENSE
// it runs over Vern7's own dense output (vern7_dense.cuh) from the step record this kernel writes.  With p.ustep set (discrete-adjoint handles) u_n of every step is recorded
// for the discrete adjoint (discrete_adjoint.cuh), which recomputes the stages from it.
template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_forward_kernel(typename Ops::Fwd p)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    const int D = Ops::D();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R dt = p.dt;
    R u[MAXD], g[MAXD], k[9][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) p.out[(size_t)c * N + n] = u[c];
    if (p.ustep)
        for (int c = 0; c < D; ++c) p.ustep[(size_t)c * N + n] = u[c];
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
        model_rhs<Ops>(u, k[0]);
#pragma unroll
        for (int i = 1; i < 9; ++i) {
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fma((R)Vern7::a(i, j), k[j][c], acc);
                g[c] = fma(dt, acc, u[c]);
            }
            model_rhs<Ops>(g, k[i]);
        }
        for (int c = 0; c < D; ++c) {
            R acc = (R)0;
#pragma unroll
            for (int j = 0; j < 9; ++j)
                if (Vern7::b(j) != 0.0) acc = fma((R)Vern7::b(j), k[j][c], acc);
            u[c] = fma(dt, acc, u[c]);
        }
        if (p.ustep)
            for (int c = 0; c < D; ++c) p.ustep[((size_t)(s + 1) * D + c) * N + n] = u[c];
        if ((s + 1) % p.save_every == 0) {
            for (int c = 0; c < D; ++c) p.out[((size_t)isave * D + c) * N + n] = u[c];
            ++isave;
        }
    }
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = ok ? 0 : 1;
    }
}

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(typename Ops::Adj p)
{
    using R = typename Ops::real;
    extern __shared__ __align__(16) unsigned char s_raw[];
    R *s_g = reinterpret_cast<R *>(s_raw);   // [BLOCK/32][P+1]
    const int D = Ops::D(), P = Ops::P();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    R *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = (R)0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const R lv = live ? (R)1 : (R)0;
    const R dt = p.dt;
    R lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    auto jump = [&](int isave) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)isave * D + c) * N + n;
            if (p.fused_l2) {
                const size_t idu = ((size_t)(isave * p.save_every) * D + c) * N + n;
                const R r = __ldg(p.ustep + idu) - __ldg(p.cot + idx);
                const R wgt = Ops::lossw(c);
                loss = fma(wgt * r, r, loss);
                lam[c] = fma((R)2 * wgt, r, lam[c]);
            } else {
                lam[c] += __ldg(p.cot + idx);
            }
        }
    };
    const int n_save = p.n_steps / p.save_every + 1;
    jump(n_save - 1);
    for (int s = p.n_steps - 1; s >= 0; --s) {
#pragma unroll
        for (int i = 0; i < 6; ++i) {   // k_7 of the backward step only feeds FSAL / error control
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < 7; ++j)
                    if (Tsit5::bw(i, j) != 0.0)
                        acc = fma((R)Tsit5::bw(i, j), __ldg(p.dense + ((size_t)(s * 6 + j) * D + c) * N + n), acc);
                x[c] = fma(dt, acc, __ldg(p.ustep + ((size_t)s * D + c) * N + n));
                R a2 = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) a2 = fma((R)Tsit5::a(i, j), kl[j][c], a2);
                g[c] = fma(dt, a2, lam[c]);
            }
            model_vjp<Ops>(x, g, dt * (R)Tsit5::b(i), lv, kl[i], gw, lane);
        }
        for (int c = 0; c < D; ++c) {
            R acc = (R)0;
#pragma unroll
            for (int j = 0; j < 6; ++j) acc = fma((R)Tsit5::b(j), kl[j][c], acc);
            lam[c] = fma(dt, acc, lam[c]);
        }
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    loss *= lv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

// =====================================================================================================
// Adaptive stepping (abstol / reltol as every reference call passes them: scenario_1.jl:85, seir_exposure.jl:139):
// Tsit5 with OrdinaryDiffEq's default PI controller and initial step (PIControl, step_control.cuh), one trajectory per
// thread with its own dt; saveat values come from the free 4th-order interpolant and do not alter the steps.  Every ACCEPTED
// step is recorded (tgrid, ustep, dense) so that the interpolating adjoint can replay the steps backwards, splitting them at
// the save times where the loss cotangent jumps in (oracle: ude_adjoint_replay; validated there against an
// error-controlled backward solve of [lambda; mu]).  The step record is Ops::Adapt (AdaptiveGrid / Adapt64Host, params.h).
// =====================================================================================================

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_forward_kernel(typename Ops::Fwd p, typename Ops::Adapt ap)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    const int D = Ops::D();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (R)(ap.n_save - 1);
    const R abstol = ap.abstol, reltol = ap.reltol;
    R u[MAXD], un[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](R *base, int row, const R *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    ap.tgrid[n] = t0;
    model_rhs<Ops>(u, k[0]);
    store(p.dense, 0, k[0]);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
    PIControl<R, 5> pi;
    {
        R d0 = 0, d1 = 0, d2 = 0;
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = PR::sq(d0 / D); d1 = PR::sq(d1 / D);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        model_rhs<Ops>(g, un);
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            const R e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = PR::sq(d2 / D) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    while (isave < ap.n_save) {
        R h = pi.dt;
        bool clipped = false;
        if (t + h >= t1 - PR::clip * fabs(t1)) { h = t1 - t; clipped = true; }
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fma((R)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fma(h, acc, u[c]);
            }
            if (i == 6) for (int c = 0; c < D; ++c) un[c] = g[c];
            model_rhs<Ops>(g, k[i]);
        }
        R ee = (R)0;
        for (int c = 0; c < D; ++c) {
            R e = (R)0;
#pragma unroll
            for (int j = 0; j < 7; ++j) e = fma((R)Tsit5::bt(j), k[j][c], e);
            e *= h;
            const R sc = abstol + reltol * fmax(fabs(u[c]), fabs(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const R EEst = PR::sq(ee / D);
        if (!(EEst <= PR::huge)) { bad = 1; break; }   // NaN / Inf
        if (pi.judge(EEst)) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            const R tn = clipped ? t1 : t + h;
            // dense record of this step: k_1..k_6 at rows nacc*6 + i, k_7 at (nacc+1)*6 (= k_1 of the next step)
            for (int i = 1; i < 7; ++i) store(p.dense, nacc * 6 + i, k[i]);
            while (isave < ap.n_save) {
                const R ts = t0 + ap.save_dt * (R)isave;
                if (ts > tn + PR::clip * fabs(tn)) break;
                R bw[7];
                Tsit5::weights(fmin((ts - t) / h, (R)1), bw);
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], k[j][c], acc);
                    p.out[((size_t)isave * D + c) * N + n] = fma(h, acc, u[c]);
                }
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = tn;
            ++nacc;
            ap.tgrid[(size_t)nacc * N + n] = t;
            for (int c = 0; c < D; ++c) { u[c] = un[c]; k[0][c] = k[6][c]; }
            store(p.ustep, nacc, u);
        } else {
            pi.reject(h);
        }
    }
    if (bad) {   // failed solve (non-finite error estimate / max_steps): the unreached save points are NaN, as a failed retcode would signal
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = PR::nan();
    }
    ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// Vern7 with OrdinaryDiffEq's PI controller (abstol / reltol; scenario_1.jl:84-85, seir_exposure.jl:138-139).  The save times
// are step end points (tstops), exactly as the oracle's Vern7 path does (saveat through the lazy 7th-order interpolant:
// B200UDE_FLAG_VERN7_DENSE, vern7_dense.cuh); the step sequence between save points is the controller's own.  No dense record is written
// (the interpolating adjoint of a Vern7 solve is taken over a Tsit5 re-solve, see b200ude.cu).  With p.ustep set
// (discrete-adjoint handles) every accepted step is recorded -- tgrid, ustep, hstep, nacc -- for the discrete adjoint: the caller
// then passes all four arrays; with p.ustep null, ap.tgrid, ap.hstep and ap.nacc are not touched.
template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_adaptive_forward_kernel(typename Ops::Fwd p, typename Ops::Adapt ap)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    const int D = Ops::D();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (R)(ap.n_save - 1);
    const R abstol = ap.abstol, reltol = ap.reltol;
    const bool record = p.ustep != nullptr;
    R u[MAXD], un[MAXD], g[MAXD], k[10][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) p.out[(size_t)c * N + n] = u[c];
    if (record) {
        ap.tgrid[n] = t0;
        for (int c = 0; c < D; ++c) p.ustep[(size_t)c * N + n] = u[c];
    }
    model_rhs<Ops>(u, k[0]);
    PIControl<R, 7> pi;
    {
        R d0 = 0, d1 = 0, d2 = 0;
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = PR::sq(d0 / D); d1 = PR::sq(d1 / D);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        model_rhs<Ops>(g, un);
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            const R e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = PR::sq(d2 / D) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    bool have_k1 = true;
    while (isave < ap.n_save) {
        const R tend = t0 + ap.save_dt * (R)isave;
        R h = pi.dt;
        bool clipped = false;
        if (t + h >= tend - PR::clip * fabs(tend)) { h = tend - t; clipped = true; }
        if (!have_k1) model_rhs<Ops>(u, k[0]);
#pragma unroll
        for (int i = 1; i < 10; ++i) {
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fma((R)Vern7::a(i, j), k[j][c], acc);
                g[c] = fma(h, acc, u[c]);
            }
            model_rhs<Ops>(g, k[i]);
        }
        R ee = (R)0;
        for (int c = 0; c < D; ++c) {
            R acc = (R)0, e = (R)0;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                if (Vern7::b(j) != 0.0) acc = fma((R)Vern7::b(j), k[j][c], acc);
                if (Vern7::bt(j) != 0.0) e = fma((R)Vern7::bt(j), k[j][c], e);
            }
            un[c] = fma(h, acc, u[c]);
            e *= h;
            const R sc = abstol + reltol * fmax(fabs(u[c]), fabs(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const R EEst = PR::sq(ee / D);
        if (!(EEst <= PR::huge)) { bad = 1; break; }
        if (pi.judge(EEst)) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            if (record) ap.hstep[(size_t)nacc * N + n] = h;
            ++nacc;
            if (clipped) {
                for (int c = 0; c < D; ++c) p.out[((size_t)isave * D + c) * N + n] = un[c];
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = clipped ? tend : t + h;
            if (record) {
                ap.tgrid[(size_t)nacc * N + n] = t;
                for (int c = 0; c < D; ++c) p.ustep[((size_t)nacc * D + c) * N + n] = un[c];
            }
            for (int c = 0; c < D; ++c) u[c] = un[c];
            have_k1 = false;   // not FSAL
        } else {
            pi.reject(h);
            have_k1 = true;    // k_1 = f(u) is still valid after a rejection
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = PR::nan();
    }
    if (record) ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_adjoint_kernel(typename Ops::Adj p, typename Ops::Adapt ap)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    R *s_g = reinterpret_cast<R *>(s_raw);   // [BLOCK/32][P+1]
    const int D = Ops::D(), P = Ops::P();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    R *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = (R)0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const int nacc = ap.nacc[n];
    int nmax = live ? nacc : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    R lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD], un_[MAXD];
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    int isave = ap.n_save - 1;
    auto jump = [&](int is) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)is * D + c) * N + n;
            lam[c] += __ldg(p.cot + idx);
        }
    };
    if (live) jump(isave);
    --isave;
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act_s = live && s < nacc;
        const int sc_ = act_s ? s : 0;                 // inactive lanes shadow step 0 (finite data), weight 0
        const R tn = ap.tgrid[(size_t)sc_ * N + n], tn1 = ap.tgrid[(size_t)(sc_ + 1) * N + n], hn = tn1 - tn;
        const R eps = PR::eta * hn;
        for (int c = 0; c < D; ++c) un_[c] = __ldg(p.ustep + ((size_t)sc_ * D + c) * N + n);
        R cur = tn1;
        while (true) {
            const bool has = act_s && cur > tn + eps;
            if (!__any_sync(0xffffffffu, has)) break;
            R ta = tn;
            const R ts = ap.t0 + ap.save_dt * (R)isave;
            if (has && isave >= 0 && ts > tn + eps) ta = ts;
            const R h = has ? cur - ta : (R)0;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                R bw[7];
                const R Th = fmin(fmax((cur - (R)Tsit5::c(i) * h - tn) / hn, (R)0), (R)1);
                Tsit5::weights(Th, bw);
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * D + c) * N + n), acc);
                    x[c] = fma(hn, acc, un_[c]);
                    R a2 = (R)0;
#pragma unroll
                    for (int j = 0; j < i; ++j)
                        if (Tsit5::a(i, j) != 0.0) a2 = fma((R)Tsit5::a(i, j), kl[j][c], a2);
                    g[c] = fma(h, a2, lam[c]);
                }
                model_vjp<Ops>(x, g, h * (R)Tsit5::b(i), has ? (R)1 : (R)0, kl[i], gw, lane);
            }
            if (has) {
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 6; ++j) acc = fma((R)Tsit5::b(j), kl[j][c], acc);
                    lam[c] = fma(h, acc, lam[c]);
                }
                cur = ta;
                if (isave >= 0 && fabs(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
    }
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    if (lane == 0) gw[P] = (R)0;   // the adaptive path takes a generic cotangent; no fused loss
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace generic
}  // namespace b200ude
