// ude_f64.cuh -- double-precision twin of the runtime-shape kernels (ude_generic.cuh): dtype = B200UDE_F64 handles.
//
// The reference runs its LV scenario 1 / 2 and SEIR scripts in Float64 (scenario_1.jl:62-66, seir_exposure.jl:114-115) with
// abstol = reltol = 1e-6 -- tolerances the fp32 kernels cannot honour on the SEIR state (1.4e7 next to 10).  These kernels
// carry the same algorithms -- Tsit5 / Vern7, fixed step and PI-controlled, the saveat interpolant, the interpolating adjoint
// on the fixed grid and the replay of an adaptive solve -- in fp64: one trajectory per thread, runtime chain shape (widths
// <= 64, <= 5 layers), models LV (0/1/2 trainable rates), SEIR, SEIR_NODE, NODE.  theta is read from the handle's device
// copy (global memory, L1-resident), the shape / constants from one small __constant__ struct.  Reference precision, not
// throughput: H100's fp64 rate is half its fp32 rate and these are the untuned one-thread-per-trajectory kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tsit5.cuh"
#include "vern7.cuh"

namespace b200ude {
namespace f64 {

constexpr int MODEL_LV = 0, MODEL_SEIR = 1, MODEL_FKPP = 2, MODEL_NODE = 3, MODEL_SEIR_NODE = 4;
constexpr int ACT_IDENTITY = 0, ACT_TANH = 1, ACT_RBF = 2;

struct Shape64 {
    uint64_t serial;
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[6];
    int acts[5];
    int woff[5];          // offset of layer l's W in theta (column-major, out x in), its bias follows at woff + in*out
    const double *theta;  // the handle's device copy
    double consts[16], lossw[16];
};
static __constant__ Shape64 c_gen;

struct Fwd64 {
    const double *u0;
    double *out, *ustep, *dense;
    int32_t *status;
    int N, n_steps, save_every;
    double dt;
};
struct Adj64 {
    const double *ustep, *dense, *cot;
    double *grad_u0, *partial;
    int N, n_steps, save_every, fused_l2;
    double dt;
};
struct Adapt64 {
    double t0, save_dt, abstol, reltol;
    int n_save, max_steps;
    double *tgrid;   // [max_steps+1][N]
    int *nacc;       // [N]
    double *hstep;   // [max_steps][N] step sizes of the accepted steps (Vern7 record for the discrete adjoint) or nullptr
};

constexpr int MAXW = 64;   // max layer width
constexpr int MAXL = 5;    // max dense layers
constexpr int MAXD = 8;    // max state dimension / chain input / chain output

__device__ __forceinline__ double act_rt(int k, double a)
{
    return k == ACT_TANH ? tanh(a) : (k == ACT_RBF ? exp(-a * a) : a);
}
__device__ __forceinline__ double actder_rt(int k, double a, double h)
{
    return k == ACT_TANH ? fma(-h, h, 1.0) : (k == ACT_RBF ? -2.0 * a * h : 1.0);
}

// chain forward; when KEEP, stores every layer's output (hs[l+1]) and pre-activation (pre[l])
template <bool KEEP>
__device__ __noinline__ void chain_fwd(const double *x, double *y, double (*hs)[MAXW], double (*pre)[MAXW])
{
    double cur[MAXW], nxt[MAXW];
    const int L = c_gen.n_layers;
    for (int i = 0; i < c_gen.widths[0]; ++i) {
        cur[i] = x[i];
        if (KEEP) hs[0][i] = x[i];
    }
    for (int l = 0; l < L; ++l) {
        const int nin = c_gen.widths[l], nout = c_gen.widths[l + 1], wo = c_gen.woff[l], act = c_gen.acts[l];
        for (int j = 0; j < nout; ++j) {
            double a = c_gen.theta[wo + nin * nout + j];
            for (int i = 0; i < nin; ++i) a = fma(c_gen.theta[wo + i * nout + j], cur[i], a);
            const double h = act_rt(act, a);
            nxt[j] = h;
            if (KEEP) { pre[l][j] = a; hs[l + 1][j] = h; }
        }
        for (int j = 0; j < nout; ++j) cur[j] = nxt[j];
    }
    for (int j = 0; j < c_gen.widths[L]; ++j) y[j] = cur[j];
}

__device__ __forceinline__ void model_inputs(const double *u, double *x)
{
    if (c_gen.model == MODEL_SEIR) {
        const double invN = 1.0 / u[4];
        x[0] = u[0] * invN; x[1] = u[2]; x[2] = u[5] * invN;
    } else if (c_gen.model == MODEL_SEIR_NODE) {   // [S/N, E, I, R, N, D/N, C]  seir_exposure.jl:58
        const double invN = 1.0 / u[4];
        x[0] = u[0] * invN; x[1] = u[1]; x[2] = u[2]; x[3] = u[3]; x[4] = u[4]; x[5] = u[5] * invN; x[6] = u[6];
    } else {
        for (int i = 0; i < c_gen.din; ++i) x[i] = u[i];
    }
}

__device__ __forceinline__ void model_rhs(const double *u_in, double *du)
{
    // private register copy of the state: the chain's scratch arrays (x, y, and chain_fwd's own) live in local memory, and the
    // state is read again after the chain -- with the caller's array that read came back clobbered by x in the Vern7 adaptive
    // kernel (stack-slot sharing after inlining; found with a device printf), which sent every SEIR solve to max_steps
    double u[MAXD];
#pragma unroll
    for (int c = 0; c < MAXD; ++c) u[c] = c < c_gen.D ? u_in[c] : 0.0;
    double x[MAXD], y[MAXD];
    model_inputs(u, x);
    chain_fwd<false>(x, y, nullptr, nullptr);
    if (c_gen.model == MODEL_LV) {
        double a1 = c_gen.consts[0], a2 = c_gen.consts[1];
        if (c_gen.n_prefix == 1) a2 = c_gen.theta[0];
        if (c_gen.n_prefix == 2) { a1 = c_gen.theta[0]; a2 = c_gen.theta[1]; }
        du[0] = fma(a1, u[0], y[0]);
        du[1] = fma(-a2, u[1], y[1]);
    } else if (c_gen.model == MODEL_SEIR) {
        // seir_exposure.jl:117-130; consts = F, beta0, alpha, kappa, mu, sigma, gamma, d, lambda (:33)
        const double F = c_gen.consts[0], b0 = c_gen.consts[1], mu = c_gen.consts[4], sg = c_gen.consts[5], gm = c_gen.consts[6], dd = c_gen.consts[7], lm = c_gen.consts[8];
        const double S = u[0], E = u[1], I = u[2], R = u[3], N = u[4], Dd = u[5];
        const double inf = b0 * S * F / N, z = y[0];
        du[0] = -inf - z - mu * S;
        du[1] = inf + z - (sg + mu) * E;
        du[2] = sg * E - (gm + mu) * I;
        du[3] = gm * I - mu * R;
        du[4] = -mu * N;
        du[5] = dd * gm * I - lm * Dd;
        du[6] = sg * E;
    } else if (c_gen.model == MODEL_SEIR_NODE) {   // dS,dE,dI,dR,dD = first five chain outputs; dN = -mu N; dC = sigma E  (seir_exposure.jl:55-64)
        du[0] = y[0]; du[1] = y[1]; du[2] = y[2]; du[3] = y[3];
        du[4] = -c_gen.consts[4] * u[4];
        du[5] = y[4];
        du[6] = c_gen.consts[5] * u[1];
    } else {
        for (int k = 0; k < c_gen.D; ++k) du[k] = y[k];
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(Fwd64 p)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const double dt = p.dt;
    double u[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](double *base, int row, const double *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    model_rhs(u, k[0]);
    store(p.dense, 0, k[0]);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            for (int c = 0; c < D; ++c) {
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fma((double)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fma(dt, acc, u[c]);
            }
            if (i == 6) for (int c = 0; c < D; ++c) u[c] = g[c];
            model_rhs(g, k[i]);
            store(p.dense, s * 6 + i, k[i]);
        }
        store(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store(p.out, isave, u); ++isave; }
        for (int c = 0; c < D; ++c) k[0][c] = k[6][c];
    }
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= 1.0e300);
        p.status[n] = ok ? 0 : 1;
    }
}

// Vern7 fixed-step forward solve (solve(prob, Vern7(); saveat, adaptive = false)): 9 stages per step, no FSAL.
// By default the interpolating adjoint of a Vern7 solve runs over a Tsit5 re-solve (b200ude.cu); with B200UDE_FLAG_VERN7_DENSE
// it runs over Vern7's own dense output (vern7_dense.cuh) from the step record this kernel writes.  With p.ustep set (discrete-adjoint handles) u_n of every step is recorded
// for the discrete adjoint (discrete_adjoint.cuh), which recomputes the stages from it.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_forward_kernel(Fwd64 p)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const double dt = p.dt;
    double u[MAXD], g[MAXD], k[9][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) p.out[(size_t)c * N + n] = u[c];
    if (p.ustep)
        for (int c = 0; c < D; ++c) p.ustep[(size_t)c * N + n] = u[c];
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
        model_rhs(u, k[0]);
#pragma unroll
        for (int i = 1; i < 9; ++i) {
            for (int c = 0; c < D; ++c) {
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fma((double)Vern7::a(i, j), k[j][c], acc);
                g[c] = fma(dt, acc, u[c]);
            }
            model_rhs(g, k[i]);
        }
        for (int c = 0; c < D; ++c) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j < 9; ++j)
                if (Vern7::b(j) != 0.0) acc = fma((double)Vern7::b(j), k[j][c], acc);
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
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= 1.0e300);
        p.status[n] = ok ? 0 : 1;
    }
}

// sum v over the warp's lanes with a fixed tree and add it into this warp's shared gradient vector
__device__ __forceinline__ void warp_acc(double *gw, int idx, double v, int lane)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) gw[idx] += v;
}

// chain VJP: dx = (dchain/dx)^T dy; this warp's gradient vector += w * (dchain/dtheta)^T dy (w per lane; all lanes participate)
__device__ __noinline__ void chain_vjp(const double *x, const double *dy, double w, double *dx, double *gw, int lane)
{
    double y[MAXD];
    double hs[MAXL + 1][MAXW], pre[MAXL][MAXW];
    chain_fwd<true>(x, y, hs, pre);
    const int L = c_gen.n_layers;
    double q[MAXW], qn[MAXW];
    for (int j = 0; j < c_gen.widths[L]; ++j) q[j] = dy[j];
    for (int l = L - 1; l >= 0; --l) {
        const int nin = c_gen.widths[l], nout = c_gen.widths[l + 1], wo = c_gen.woff[l], act = c_gen.acts[l];
        for (int j = 0; j < nout; ++j) q[j] *= actder_rt(act, pre[l][j], hs[l + 1][j]);
        for (int i = 0; i < nin; ++i) {
            double sacc = 0.0;
            const double hi = hs[l][i];
            for (int j = 0; j < nout; ++j) {
                sacc = fma(c_gen.theta[wo + i * nout + j], q[j], sacc);
                warp_acc(gw, wo + i * nout + j, w * q[j] * hi, lane);
            }
            qn[i] = sacc;
        }
        for (int j = 0; j < nout; ++j) warp_acc(gw, wo + nin * nout + j, w * q[j], lane);
        for (int i = 0; i < nin; ++i) q[i] = qn[i];
    }
    for (int i = 0; i < c_gen.widths[0]; ++i) dx[i] = q[i];
}

// kl = (df/du)^T g ; this warp's gradient vector += sc * (df/dtheta)^T g   (all lanes of the warp participate)
__device__ __forceinline__ void model_vjp(const double *u_in, const double *g_in, double sc, double lv, double *kl, double *gw, int lane)
{
    double u[MAXD], g[MAXD];   // private register copies, read again after the chain (see model_rhs)
#pragma unroll
    for (int c = 0; c < MAXD; ++c) { u[c] = c < c_gen.D ? u_in[c] : 0.0; g[c] = c < c_gen.D ? g_in[c] : 0.0; }
    double x[MAXD], dy[MAXD], dx[MAXD];
    model_inputs(u, x);
    const double w = sc * lv;   // quadrature weight, zero for padding lanes
    if (c_gen.model == MODEL_SEIR) dy[0] = g[1] - g[0];   // z enters dS with -, dE with +
    else if (c_gen.model == MODEL_SEIR_NODE) { dy[0] = g[0]; dy[1] = g[1]; dy[2] = g[2]; dy[3] = g[3]; dy[4] = g[5]; dy[5] = 0.0; dy[6] = 0.0; }
    else for (int m = 0; m < c_gen.dout; ++m) dy[m] = g[m];
    chain_vjp(x, dy, w, dx, gw, lane);
    if (c_gen.model == MODEL_LV) {
        double a1 = c_gen.consts[0], a2 = c_gen.consts[1];
        if (c_gen.n_prefix == 1) a2 = c_gen.theta[0];
        if (c_gen.n_prefix == 2) { a1 = c_gen.theta[0]; a2 = c_gen.theta[1]; }
        kl[0] = fma(a1, g[0], dx[0]);
        kl[1] = fma(-a2, g[1], dx[1]);
        if (c_gen.n_prefix == 1) warp_acc(gw, 0, w * (-u[1] * g[1]), lane);
        if (c_gen.n_prefix == 2) {
            warp_acc(gw, 0, w * (u[0] * g[0]), lane);
            warp_acc(gw, 1, w * (-u[1] * g[1]), lane);
        }
    } else if (c_gen.model == MODEL_SEIR) {
        const double F = c_gen.consts[0], b0 = c_gen.consts[1], mu = c_gen.consts[4], sg = c_gen.consts[5], gm = c_gen.consts[6], dd = c_gen.consts[7], lm = c_gen.consts[8];
        const double S = u[0], N = u[4], Dd = u[5];
        const double cS = b0 * F / N, cN = -b0 * S * F / (N * N);
        kl[0] = g[0] * (-cS - mu) + g[1] * cS + dx[0] / N;
        kl[1] = g[1] * (-(sg + mu)) + g[2] * sg + g[6] * sg;
        kl[2] = g[2] * (-(gm + mu)) + g[3] * gm + g[5] * dd * gm + dx[1];
        kl[3] = g[3] * (-mu);
        kl[4] = g[0] * (-cN) + g[1] * cN + g[4] * (-mu) - dx[0] * S / (N * N) - dx[2] * Dd / (N * N);
        kl[5] = g[5] * (-lm) + dx[2] / N;
        kl[6] = 0.0;
    } else if (c_gen.model == MODEL_SEIR_NODE) {
        const double S = u[0], N = u[4], Dd = u[5], mu = c_gen.consts[4], sg = c_gen.consts[5];
        kl[0] = dx[0] / N;
        kl[1] = dx[1] + sg * g[6];
        kl[2] = dx[2];
        kl[3] = dx[3];
        kl[4] = dx[4] - mu * g[4] - dx[0] * S / (N * N) - dx[5] * Dd / (N * N);
        kl[5] = dx[5] / N;
        kl[6] = dx[6];
    } else {
        for (int k = 0; k < c_gen.D; ++k) kl[k] = dx[k];
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(Adj64 p)
{
    extern __shared__ __align__(16) double s_g[];   // [BLOCK/32][P+1]
    const int D = c_gen.D, P = c_gen.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const double lv = live ? 1.0 : 0.0;
    const double dt = p.dt;
    double lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD];
    double loss = 0.0;
    for (int c = 0; c < D; ++c) lam[c] = 0.0;
    auto jump = [&](int isave) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)isave * D + c) * N + n;
            if (p.fused_l2) {
                const size_t idu = ((size_t)(isave * p.save_every) * D + c) * N + n;
                const double r = __ldg(p.ustep + idu) - __ldg(p.cot + idx);
                const double wgt = c_gen.lossw[c];
                loss = fma(wgt * r, r, loss);
                lam[c] = fma(2.0 * wgt, r, lam[c]);
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
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < 7; ++j)
                    if (Tsit5::bw(i, j) != 0.0)
                        acc = fma((double)Tsit5::bw(i, j), __ldg(p.dense + ((size_t)(s * 6 + j) * D + c) * N + n), acc);
                x[c] = fma(dt, acc, __ldg(p.ustep + ((size_t)s * D + c) * N + n));
                double a2 = 0.0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) a2 = fma((double)Tsit5::a(i, j), kl[j][c], a2);
                g[c] = fma(dt, a2, lam[c]);
            }
            model_vjp(x, g, dt * (double)Tsit5::b(i), lv, kl[i], gw, lane);
        }
        for (int c = 0; c < D; ++c) {
            double acc = 0.0;
#pragma unroll
            for (int j = 0; j < 6; ++j) acc = fma((double)Tsit5::b(j), kl[j][c], acc);
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
    double *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

// =====================================================================================================
// Adaptive stepping (abstol / reltol as every reference call passes them: scenario_1.jl:85, seir_exposure.jl:139):
// Tsit5 with OrdinaryDiffEq's default PI controller (gamma 0.9, qmin 1/5, qmax 10, beta1 7/50, beta2 2/25,
// steady band [1, 1.2], Hairer initial step), one trajectory per thread with its own dt; saveat values come from
// the free 4th-order interpolant and do not alter the steps.  Every ACCEPTED step is recorded
// (tgrid, ustep, dense) so that the interpolating adjoint can replay the steps backwards, splitting them at
// the save times where the loss cotangent jumps in (oracle: ude_adjoint_replay; validated there against an
// error-controlled backward solve of [lambda; mu]).
// =====================================================================================================

__device__ __forceinline__ void tsit5_bw_rt(double Th, double *bw)
{
    bw[0] = Th * ((double)Tsit5::r(0, 1) + Th * ((double)Tsit5::r(0, 2) + Th * ((double)Tsit5::r(0, 3) + Th * (double)Tsit5::r(0, 4))));
#pragma unroll
    for (int j = 1; j < 7; ++j) bw[j] = Th * Th * ((double)Tsit5::r(j, 2) + Th * ((double)Tsit5::r(j, 3) + Th * (double)Tsit5::r(j, 4)));
}
__device__ __forceinline__ double tsit5_btilde(int j)
{
    return j == 0 ? -0.001780011052225777 : j == 1 ? -0.0008164344596567469 : j == 2 ? 0.007880878010261995
         : j == 3 ? -0.1447110071732629 : j == 4 ? 0.5823571654525552 : j == 5 ? -0.45808210592918697 : 0.015151515151515152;
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_forward_kernel(Fwd64 p, Adapt64 ap)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const double t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (double)(ap.n_save - 1);
    const double abstol = ap.abstol, reltol = ap.reltol;
    const double gamma = 0.9, qmin = 0.2, qmax = 10.0, beta1 = 7.0 / 50.0, beta2 = 2.0 / 25.0;
    double u[MAXD], un[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](double *base, int row, const double *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    ap.tgrid[n] = t0;
    model_rhs(u, k[0]);
    store(p.dense, 0, k[0]);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
    double dt;
    {
        double d0 = 0.f, d1 = 0.f, d2 = 0.f;
        for (int c = 0; c < D; ++c) {
            const double sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = sqrt(d0 / D); d1 = sqrt(d1 / D);
        double dt0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
        dt0 = fmin(dt0, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        model_rhs(g, un);
        for (int c = 0; c < D; ++c) {
            const double sk = abstol + reltol * fabs(u[c]);
            const double e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = sqrt(d2 / D) / dt0;
        const double dm = fmax(d1, d2);
        const double dt1 = dm <= 1e-15 ? fmax(1e-6, dt0 * 1e-3) : exp10(-(2.0 + log10(dm)) / 5.0);
        dt = fmin(fmin(100.0 * dt0, dt1), t1 - t0);
    }
    double t = t0, qold = 1e-4;
    int nacc = 0, isave = 1, bad = 0;
    while (isave < ap.n_save) {
        double h = dt;
        bool clipped = false;
        if (t + h >= t1 - 1e-12 * fabs(t1)) { h = t1 - t; clipped = true; }
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            for (int c = 0; c < D; ++c) {
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fma((double)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fma(h, acc, u[c]);
            }
            if (i == 6) for (int c = 0; c < D; ++c) un[c] = g[c];
            model_rhs(g, k[i]);
        }
        double ee = 0.0;
        for (int c = 0; c < D; ++c) {
            double e = 0.0;
#pragma unroll
            for (int j = 0; j < 7; ++j) e = fma(tsit5_btilde(j), k[j][c], e);
            e *= h;
            const double sc = abstol + reltol * fmax(fabs(u[c]), fabs(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const double EEst = sqrt(ee / D);
        if (!(EEst <= 1.0e300)) { bad = 1; break; }   // NaN / Inf
        const double q11 = pow(EEst, beta1);
        double q = fmin(fmax(q11 / pow(qold, beta2) / gamma, 1.0 / qmax), 1.0 / qmin);
        if (EEst <= 1.0) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            const double tn = clipped ? t1 : t + h;
            // dense record of this step: k_1..k_6 at rows nacc*6 + i, k_7 at (nacc+1)*6 (= k_1 of the next step)
            for (int i = 1; i < 7; ++i) store(p.dense, nacc * 6 + i, k[i]);
            while (isave < ap.n_save) {
                const double ts = t0 + ap.save_dt * (double)isave;
                if (ts > tn + 1e-12 * fabs(tn)) break;
                double bw[7];
                tsit5_bw_rt(fmin((ts - t) / h, 1.0), bw);
                for (int c = 0; c < D; ++c) {
                    double acc = 0.0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], k[j][c], acc);
                    p.out[((size_t)isave * D + c) * N + n] = fma(h, acc, u[c]);
                }
                ++isave;
            }
            qold = fmax(EEst, 1e-4);
            // qsteady_min = qsteady_max = 1 for explicit RK methods in OrdinaryDiffEq (the 6/5 band is the implicit-solver default): no dead band
            if (!clipped || h >= dt) dt = h / q;
            else dt = fmax(dt, h / q);
            t = tn;
            ++nacc;
            ap.tgrid[(size_t)nacc * N + n] = t;
            for (int c = 0; c < D; ++c) { u[c] = un[c]; k[0][c] = k[6][c]; }
            store(p.ustep, nacc, u);
        } else {
            dt = h / fmin(1.0 / qmin, q11 / gamma);
        }
    }
    if (bad) {   // failed solve (non-finite error estimate / max_steps): the unreached save points are NaN, as a failed retcode would signal
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = __longlong_as_double(0x7ff8000000000000LL);
    }
    ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= 1.0e300);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// Vern7 with OrdinaryDiffEq's PI controller (abstol / reltol; scenario_1.jl:84-85, seir_exposure.jl:138-139).  The save times
// are step end points (tstops), exactly as the oracle's Vern7 path does (saveat through the lazy 7th-order interpolant:
// B200UDE_FLAG_VERN7_DENSE, vern7_dense.cuh); the step sequence between save points is the controller's own.  No dense record is written
// (the interpolating adjoint of a Vern7 solve is taken over a Tsit5 re-solve, see b200ude.cu).  With ap.tgrid set
// (discrete-adjoint handles) every accepted step is recorded -- tgrid, ustep, hstep, nacc -- for the discrete adjoint.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_adaptive_forward_kernel(Fwd64 p, Adapt64 ap)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const double t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (double)(ap.n_save - 1);
    const double abstol = ap.abstol, reltol = ap.reltol;
    const double gamma = 0.9, qmin = 0.2, qmax = 10.0, beta1 = 7.0 / 70.0, beta2 = 2.0 / 35.0;   // order 7
    const bool record = ap.tgrid != nullptr;
    double u[MAXD], un[MAXD], g[MAXD], k[10][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) p.out[(size_t)c * N + n] = u[c];
    if (record) {
        ap.tgrid[n] = t0;
        for (int c = 0; c < D; ++c) p.ustep[(size_t)c * N + n] = u[c];
    }
    model_rhs(u, k[0]);
    double dt;
    {
        double d0 = 0.f, d1 = 0.f, d2 = 0.f;
        for (int c = 0; c < D; ++c) {
            const double sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = sqrt(d0 / D); d1 = sqrt(d1 / D);
        double dt0 = (d0 < 1e-5 || d1 < 1e-5) ? 1e-6 : 0.01 * d0 / d1;
        dt0 = fmin(dt0, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        model_rhs(g, un);
        for (int c = 0; c < D; ++c) {
            const double sk = abstol + reltol * fabs(u[c]);
            const double e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = sqrt(d2 / D) / dt0;
        const double dm = fmax(d1, d2);
        const double dt1 = dm <= 1e-15 ? fmax(1e-6, dt0 * 1e-3) : exp10(-(2.0 + log10(dm)) / 7.0);
        dt = fmin(fmin(100.0 * dt0, dt1), t1 - t0);
    }
    double t = t0, qold = 1e-4;
    int nacc = 0, isave = 1, bad = 0;
    bool have_k1 = true;
    while (isave < ap.n_save) {
        const double tend = t0 + ap.save_dt * (double)isave;
        double h = dt;
        bool clipped = false;
        if (t + h >= tend - 1e-12 * fabs(tend)) { h = tend - t; clipped = true; }
        if (!have_k1) model_rhs(u, k[0]);
#pragma unroll
        for (int i = 1; i < 10; ++i) {
            for (int c = 0; c < D; ++c) {
                double acc = 0.0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fma((double)Vern7::a(i, j), k[j][c], acc);
                g[c] = fma(h, acc, u[c]);
            }
            model_rhs(g, k[i]);
        }
        double ee = 0.0;
        for (int c = 0; c < D; ++c) {
            double acc = 0.0, e = 0.0;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                if (Vern7::b(j) != 0.0) acc = fma((double)Vern7::b(j), k[j][c], acc);
                if (Vern7::bt(j) != 0.0) e = fma((double)Vern7::bt(j), k[j][c], e);
            }
            un[c] = fma(h, acc, u[c]);
            e *= h;
            const double sc = abstol + reltol * fmax(fabs(u[c]), fabs(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const double EEst = sqrt(ee / D);
        if (!(EEst <= 1.0e300)) { bad = 1; break; }
        const double q11 = pow(EEst, beta1);
        double q = fmin(fmax(q11 / pow(qold, beta2) / gamma, 1.0 / qmax), 1.0 / qmin);
        if (EEst <= 1.0) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            if (record) ap.hstep[(size_t)nacc * N + n] = h;
            ++nacc;
            if (clipped) {
                for (int c = 0; c < D; ++c) p.out[((size_t)isave * D + c) * N + n] = un[c];
                ++isave;
            }
            qold = fmax(EEst, 1e-4);
            // qsteady_min = qsteady_max = 1 for explicit RK methods in OrdinaryDiffEq (the 6/5 band is the implicit-solver default): no dead band
            if (!clipped || h >= dt) dt = h / q;
            else dt = fmax(dt, h / q);
            t = clipped ? tend : t + h;
            if (record) {
                ap.tgrid[(size_t)nacc * N + n] = t;
                for (int c = 0; c < D; ++c) p.ustep[((size_t)nacc * D + c) * N + n] = un[c];
            }
            for (int c = 0; c < D; ++c) u[c] = un[c];
            have_k1 = false;   // not FSAL
        } else {
            dt = h / fmin(1.0 / qmin, q11 / gamma);
            have_k1 = true;    // k_1 = f(u) is still valid after a rejection
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = __longlong_as_double(0x7ff8000000000000LL);
    }
    if (ap.nacc) ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= 1.0e300);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_adjoint_kernel(Adj64 p, Adapt64 ap)
{
    extern __shared__ __align__(16) double s_g[];   // [BLOCK/32][P+1]
    const int D = c_gen.D, P = c_gen.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const int nacc = ap.nacc[n];
    int nmax = live ? nacc : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    double lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD], un_[MAXD];
    double loss = 0.0;
    for (int c = 0; c < D; ++c) lam[c] = 0.0;
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
        const double tn = ap.tgrid[(size_t)sc_ * N + n], tn1 = ap.tgrid[(size_t)(sc_ + 1) * N + n], hn = tn1 - tn;
        const double eps = 1e-10 * hn;
        for (int c = 0; c < D; ++c) un_[c] = __ldg(p.ustep + ((size_t)sc_ * D + c) * N + n);
        double cur = tn1;
        while (true) {
            const bool has = act_s && cur > tn + eps;
            if (!__any_sync(0xffffffffu, has)) break;
            double ta = tn;
            const double ts = ap.t0 + ap.save_dt * (double)isave;
            if (has && isave >= 0 && ts > tn + eps) ta = ts;
            const double h = has ? cur - ta : 0.0;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                double bw[7];
                const double Th = fmin(fmax((cur - (double)Tsit5::c(i) * h - tn) / hn, 0.0), 1.0);
                tsit5_bw_rt(Th, bw);
                for (int c = 0; c < D; ++c) {
                    double acc = 0.0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * D + c) * N + n), acc);
                    x[c] = fma(hn, acc, un_[c]);
                    double a2 = 0.0;
#pragma unroll
                    for (int j = 0; j < i; ++j)
                        if (Tsit5::a(i, j) != 0.0) a2 = fma((double)Tsit5::a(i, j), kl[j][c], a2);
                    g[c] = fma(h, a2, lam[c]);
                }
                model_vjp(x, g, h * (double)Tsit5::b(i), has ? 1.0 : 0.0, kl[i], gw, lane);
            }
            if (has) {
                for (int c = 0; c < D; ++c) {
                    double acc = 0.0;
#pragma unroll
                    for (int j = 0; j < 6; ++j) acc = fma((double)Tsit5::b(j), kl[j][c], acc);
                    lam[c] = fma(h, acc, lam[c]);
                }
                cur = ta;
                if (isave >= 0 && fabs(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
    }
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    if (lane == 0) gw[P] = 0.0;   // the adaptive path takes a generic cotangent; no fused loss
    (void)loss;
    __syncwarp();
    double *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}


}  // namespace f64
}  // namespace b200ude
