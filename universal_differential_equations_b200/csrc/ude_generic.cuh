// ude_generic.cuh -- shape-generic (runtime widths / activations) UDE kernels.
//
// Functional coverage for every recognised UDE form whose chain has no specialised kernel: any dense chain
// with widths <= 64 and <= 5 layers, models LV (0/1/2 trainable rates), SEIR (7 states, chain on
// [S/N, I, D/N], SEIR_exposure/seir_exposure.jl:117-130), SEIR_NODE (the script's black-box baseline, :52-64) and NODE;
// also the adaptive Tsit5 forward / replay-adjoint kernels, the Vern7 forward kernels and the runtime-shape Fisher-KPP kernels
// (the discrete adjoint of the Tsit5 / Vern7 solves is in discrete_adjoint.cuh).  One trajectory per thread, weights read
// from the constant bank with runtime indices, activations in per-thread local arrays, Tsit5 forward with
// dense output and the interpolating adjoint exactly as in the specialised kernels.  The ensemble-summed
// parameter gradient is reduced deterministically: every contribution is summed over the warp's lanes with a
// fixed shuffle tree and added by lane 0 into a per-warp shared-memory vector.  Correctness first: these
// kernels are ~10-30x slower per FLOP than lv32::tc and are reported as such (DESIGN.md section 4.3).
#pragma once
#include "ude_adjoint.cuh"
#include "vern7.cuh"

namespace b200ude {
namespace generic {

constexpr int MAXW = 64;   // max layer width
constexpr int MAXL = 5;    // max dense layers
constexpr int MAXD = 8;    // max state dimension / chain input / chain output

struct GenDesc {
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[MAXL + 1];
    int acts[MAXL];
    int woff[MAXL];   // offset of layer l's W in theta (column-major, out x in), its bias follows at woff + in*out
};
static __constant__ GenDesc c_gen;

__device__ __forceinline__ float act_rt(int k, float a)
{
    return k == ACT_TANH ? tanh_dev<0>(a) : (k == ACT_RBF ? rbf_dev(a) : a);
}
__device__ __forceinline__ float actder_rt(int k, float a, float h)
{
    return k == ACT_TANH ? fmaf(-h, h, 1.0f) : (k == ACT_RBF ? -2.0f * a * h : 1.0f);
}

// chain forward; when KEEP, stores every layer's output (hs[l+1]) and pre-activation (pre[l])
template <bool KEEP>
__device__ __noinline__ void chain_fwd(const float *x, float *y, float (*hs)[MAXW], float (*pre)[MAXW])
{
    float cur[MAXW], nxt[MAXW];
    const int L = c_gen.n_layers;
    for (int i = 0; i < c_gen.widths[0]; ++i) {
        cur[i] = x[i];
        if (KEEP) hs[0][i] = x[i];
    }
    for (int l = 0; l < L; ++l) {
        const int nin = c_gen.widths[l], nout = c_gen.widths[l + 1], wo = c_gen.woff[l], act = c_gen.acts[l];
        for (int j = 0; j < nout; ++j) {
            float a = c_theta[wo + nin * nout + j];
            for (int i = 0; i < nin; ++i) a = fmaf(c_theta[wo + i * nout + j], cur[i], a);
            const float h = act_rt(act, a);
            nxt[j] = h;
            if (KEEP) { pre[l][j] = a; hs[l + 1][j] = h; }
        }
        for (int j = 0; j < nout; ++j) cur[j] = nxt[j];
    }
    for (int j = 0; j < c_gen.widths[L]; ++j) y[j] = cur[j];
}

__device__ __forceinline__ void model_inputs(const float *u, float *x)
{
    if (c_gen.model == MODEL_SEIR) {
        const float invN = 1.0f / u[4];
        x[0] = u[0] * invN; x[1] = u[2]; x[2] = u[5] * invN;
    } else if (c_gen.model == MODEL_SEIR_NODE) {   // [S/N, E, I, R, N, D/N, C]  seir_exposure.jl:58
        const float invN = 1.0f / u[4];
        x[0] = u[0] * invN; x[1] = u[1]; x[2] = u[2]; x[3] = u[3]; x[4] = u[4]; x[5] = u[5] * invN; x[6] = u[6];
    } else {
        for (int i = 0; i < c_gen.din; ++i) x[i] = u[i];
    }
}

__device__ __forceinline__ void model_rhs(const float *u_in, float *du)
{
    // private register copy of the state: the chain's scratch arrays (x, y, and chain_fwd's own) live in local memory, and the
    // state is read again after the chain -- with the caller's array that read came back clobbered by x in the Vern7 adaptive
    // kernel (stack-slot sharing after inlining; found with a device printf), which sent every SEIR solve to max_steps
    float u[MAXD];
#pragma unroll
    for (int c = 0; c < MAXD; ++c) u[c] = c < c_gen.D ? u_in[c] : 0.0f;
    float x[MAXD], y[MAXD];
    model_inputs(u, x);
    chain_fwd<false>(x, y, nullptr, nullptr);
    if (c_gen.model == MODEL_LV) {
        float a1 = c_consts[0], a2 = c_consts[1];
        if (c_gen.n_prefix == 1) a2 = c_theta[0];
        if (c_gen.n_prefix == 2) { a1 = c_theta[0]; a2 = c_theta[1]; }
        du[0] = fmaf(a1, u[0], y[0]);
        du[1] = fmaf(-a2, u[1], y[1]);
    } else if (c_gen.model == MODEL_SEIR) {
        // seir_exposure.jl:117-130; consts = F, beta0, alpha, kappa, mu, sigma, gamma, d, lambda (:33)
        const float F = c_consts[0], b0 = c_consts[1], mu = c_consts[4], sg = c_consts[5], gm = c_consts[6], dd = c_consts[7], lm = c_consts[8];
        const float S = u[0], E = u[1], I = u[2], R = u[3], N = u[4], Dd = u[5];
        const float inf = b0 * S * F / N, z = y[0];
        du[0] = -inf - z - mu * S;
        du[1] = inf + z - (sg + mu) * E;
        du[2] = sg * E - (gm + mu) * I;
        du[3] = gm * I - mu * R;
        du[4] = -mu * N;
        du[5] = dd * gm * I - lm * Dd;
        du[6] = sg * E;
    } else if (c_gen.model == MODEL_SEIR_NODE) {   // dS,dE,dI,dR,dD = first five chain outputs; dN = -mu N; dC = sigma E  (seir_exposure.jl:55-64)
        du[0] = y[0]; du[1] = y[1]; du[2] = y[2]; du[3] = y[3];
        du[4] = -c_consts[4] * u[4];
        du[5] = y[4];
        du[6] = c_consts[5] * u[1];
    } else {
        for (int k = 0; k < c_gen.D; ++k) du[k] = y[k];
    }
}

struct GenFwdParams {
    FwdParams f;
};

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(FwdParams p)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const float dt = p.dt;
    float u[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](float *base, int row, const float *v) {
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
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fmaf((float)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fmaf(dt, acc, u[c]);
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
        for (int c = 0; c < D; ++c) ok = ok && (fabsf(u[c]) <= 3.0e38f);
        p.status[n] = ok ? 0 : 1;
    }
}

// Vern7 fixed-step forward solve (solve(prob, Vern7(); saveat, adaptive = false)): 9 stages per step, no FSAL.
// By default the interpolating adjoint of a Vern7 solve runs over a Tsit5 re-solve (b200ude.cu); with B200UDE_FLAG_VERN7_DENSE
// it runs over Vern7's own dense output (vern7_dense.cuh) from the step record this kernel writes.  With p.ustep set (discrete-adjoint handles) u_n of every step is recorded
// for the discrete adjoint (discrete_adjoint.cuh), which recomputes the stages from it.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_forward_kernel(FwdParams p)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const float dt = p.dt;
    float u[MAXD], g[MAXD], k[9][MAXD];
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
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fmaf((float)Vern7::a(i, j), k[j][c], acc);
                g[c] = fmaf(dt, acc, u[c]);
            }
            model_rhs(g, k[i]);
        }
        for (int c = 0; c < D; ++c) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < 9; ++j)
                if (Vern7::b(j) != 0.0) acc = fmaf((float)Vern7::b(j), k[j][c], acc);
            u[c] = fmaf(dt, acc, u[c]);
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
        for (int c = 0; c < D; ++c) ok = ok && (fabsf(u[c]) <= 3.0e38f);
        p.status[n] = ok ? 0 : 1;
    }
}

// sum v over the warp's lanes with a fixed tree and add it into this warp's shared gradient vector
__device__ __forceinline__ void warp_acc(float *gw, int idx, float v, int lane)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) gw[idx] += v;
}

// chain VJP: dx = (dchain/dx)^T dy; this warp's gradient vector += w * (dchain/dtheta)^T dy (w per lane; all lanes participate)
__device__ __noinline__ void chain_vjp(const float *x, const float *dy, float w, float *dx, float *gw, int lane)
{
    float y[MAXD];
    float hs[MAXL + 1][MAXW], pre[MAXL][MAXW];
    chain_fwd<true>(x, y, hs, pre);
    const int L = c_gen.n_layers;
    float q[MAXW], qn[MAXW];
    for (int j = 0; j < c_gen.widths[L]; ++j) q[j] = dy[j];
    for (int l = L - 1; l >= 0; --l) {
        const int nin = c_gen.widths[l], nout = c_gen.widths[l + 1], wo = c_gen.woff[l], act = c_gen.acts[l];
        for (int j = 0; j < nout; ++j) q[j] *= actder_rt(act, pre[l][j], hs[l + 1][j]);
        for (int i = 0; i < nin; ++i) {
            float sacc = 0.0f;
            const float hi = hs[l][i];
            for (int j = 0; j < nout; ++j) {
                sacc = fmaf(c_theta[wo + i * nout + j], q[j], sacc);
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
__device__ __forceinline__ void model_vjp(const float *u_in, const float *g_in, float sc, float lv, float *kl, float *gw, int lane)
{
    float u[MAXD], g[MAXD];   // private register copies, read again after the chain (see model_rhs)
#pragma unroll
    for (int c = 0; c < MAXD; ++c) { u[c] = c < c_gen.D ? u_in[c] : 0.0f; g[c] = c < c_gen.D ? g_in[c] : 0.0f; }
    float x[MAXD], dy[MAXD], dx[MAXD];
    model_inputs(u, x);
    const float w = sc * lv;   // quadrature weight, zero for padding lanes
    if (c_gen.model == MODEL_SEIR) dy[0] = g[1] - g[0];   // z enters dS with -, dE with +
    else if (c_gen.model == MODEL_SEIR_NODE) { dy[0] = g[0]; dy[1] = g[1]; dy[2] = g[2]; dy[3] = g[3]; dy[4] = g[5]; dy[5] = 0.0f; dy[6] = 0.0f; }
    else for (int m = 0; m < c_gen.dout; ++m) dy[m] = g[m];
    chain_vjp(x, dy, w, dx, gw, lane);
    if (c_gen.model == MODEL_LV) {
        float a1 = c_consts[0], a2 = c_consts[1];
        if (c_gen.n_prefix == 1) a2 = c_theta[0];
        if (c_gen.n_prefix == 2) { a1 = c_theta[0]; a2 = c_theta[1]; }
        kl[0] = fmaf(a1, g[0], dx[0]);
        kl[1] = fmaf(-a2, g[1], dx[1]);
        if (c_gen.n_prefix == 1) warp_acc(gw, 0, w * (-u[1] * g[1]), lane);
        if (c_gen.n_prefix == 2) {
            warp_acc(gw, 0, w * (u[0] * g[0]), lane);
            warp_acc(gw, 1, w * (-u[1] * g[1]), lane);
        }
    } else if (c_gen.model == MODEL_SEIR) {
        const float F = c_consts[0], b0 = c_consts[1], mu = c_consts[4], sg = c_consts[5], gm = c_consts[6], dd = c_consts[7], lm = c_consts[8];
        const float S = u[0], N = u[4], Dd = u[5];
        const float cS = b0 * F / N, cN = -b0 * S * F / (N * N);
        kl[0] = g[0] * (-cS - mu) + g[1] * cS + dx[0] / N;
        kl[1] = g[1] * (-(sg + mu)) + g[2] * sg + g[6] * sg;
        kl[2] = g[2] * (-(gm + mu)) + g[3] * gm + g[5] * dd * gm + dx[1];
        kl[3] = g[3] * (-mu);
        kl[4] = g[0] * (-cN) + g[1] * cN + g[4] * (-mu) - dx[0] * S / (N * N) - dx[2] * Dd / (N * N);
        kl[5] = g[5] * (-lm) + dx[2] / N;
        kl[6] = 0.0f;
    } else if (c_gen.model == MODEL_SEIR_NODE) {
        const float S = u[0], N = u[4], Dd = u[5], mu = c_consts[4], sg = c_consts[5];
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
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(AdjParams p)
{
    extern __shared__ __align__(16) float s_g[];   // [BLOCK/32][P+1]
    const int D = c_gen.D, P = c_gen.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0f;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt;
    float lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD];
    float loss = 0.0f;
    for (int c = 0; c < D; ++c) lam[c] = 0.0f;
    auto jump = [&](int isave) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)isave * D + c) * N + n;
            if (p.fused_l2) {
                const size_t idu = ((size_t)(isave * p.save_every) * D + c) * N + n;
                const float r = __ldg(p.ustep + idu) - __ldg(p.cot + idx);
                const float wgt = c_lossw[c];
                loss = fmaf(wgt * r, r, loss);
                lam[c] = fmaf(2.0f * wgt, r, lam[c]);
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
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < 7; ++j)
                    if (Tsit5::bw(i, j) != 0.0)
                        acc = fmaf((float)Tsit5::bw(i, j), __ldg(p.dense + ((size_t)(s * 6 + j) * D + c) * N + n), acc);
                x[c] = fmaf(dt, acc, __ldg(p.ustep + ((size_t)s * D + c) * N + n));
                float a2 = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) a2 = fmaf((float)Tsit5::a(i, j), kl[j][c], a2);
                g[c] = fmaf(dt, a2, lam[c]);
            }
            model_vjp(x, g, dt * (float)Tsit5::b(i), lv, kl[i], gw, lane);
        }
        for (int c = 0; c < D; ++c) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < 6; ++j) acc = fmaf((float)Tsit5::b(j), kl[j][c], acc);
            lam[c] = fmaf(dt, acc, lam[c]);
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
    float *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
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
struct AdaptParams {
    float t0, save_dt, abstol, reltol;
    int n_save, max_steps;
    float *tgrid;     // [max_steps+1][N]
    int *nacc;        // [N]
    float *hstep;     // [max_steps][N] step sizes of the accepted steps (Vern7 record for the discrete adjoint) or nullptr
};

__device__ __forceinline__ void tsit5_bw_rt(float Th, float *bw)
{
    bw[0] = Th * ((float)Tsit5::r(0, 1) + Th * ((float)Tsit5::r(0, 2) + Th * ((float)Tsit5::r(0, 3) + Th * (float)Tsit5::r(0, 4))));
#pragma unroll
    for (int j = 1; j < 7; ++j) bw[j] = Th * Th * ((float)Tsit5::r(j, 2) + Th * ((float)Tsit5::r(j, 3) + Th * (float)Tsit5::r(j, 4)));
}
__device__ __forceinline__ float tsit5_btilde(int j)
{
    return j == 0 ? -0.001780011052225777f : j == 1 ? -0.0008164344596567469f : j == 2 ? 0.007880878010261995f
         : j == 3 ? -0.1447110071732629f : j == 4 ? 0.5823571654525552f : j == 5 ? -0.45808210592918697f : 0.015151515151515152f;
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_forward_kernel(FwdParams p, AdaptParams ap)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const float t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (float)(ap.n_save - 1);
    const float abstol = ap.abstol, reltol = ap.reltol;
    const float gamma = 0.9f, qmin = 0.2f, qmax = 10.0f, beta1 = 7.0f / 50.0f, beta2 = 2.0f / 25.0f;
    float u[MAXD], un[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](float *base, int row, const float *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    ap.tgrid[n] = t0;
    model_rhs(u, k[0]);
    store(p.dense, 0, k[0]);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
    float dt;
    {
        float d0 = 0.f, d1 = 0.f, d2 = 0.f;
        for (int c = 0; c < D; ++c) {
            const float sk = abstol + reltol * fabsf(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = sqrtf(d0 / D); d1 = sqrtf(d1 / D);
        float dt0 = (d0 < 1e-5f || d1 < 1e-5f) ? 1e-6f : 0.01f * d0 / d1;
        dt0 = fminf(dt0, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fmaf(dt0, k[0][c], u[c]);
        model_rhs(g, un);
        for (int c = 0; c < D; ++c) {
            const float sk = abstol + reltol * fabsf(u[c]);
            const float e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = sqrtf(d2 / D) / dt0;
        const float dm = fmaxf(d1, d2);
        const float dt1 = dm <= 1e-15f ? fmaxf(1e-6f, dt0 * 1e-3f) : exp10f(-(2.0f + log10f(dm)) / 5.0f);
        dt = fminf(fminf(100.0f * dt0, dt1), t1 - t0);
    }
    float t = t0, qold = 1e-4f;
    int nacc = 0, isave = 1, bad = 0;
    while (isave < ap.n_save) {
        float h = dt;
        bool clipped = false;
        if (t + h >= t1 - 1e-6f * fabsf(t1)) { h = t1 - t; clipped = true; }
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            for (int c = 0; c < D; ++c) {
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) acc = fmaf((float)Tsit5::a(i, j), k[j][c], acc);
                g[c] = fmaf(h, acc, u[c]);
            }
            if (i == 6) for (int c = 0; c < D; ++c) un[c] = g[c];
            model_rhs(g, k[i]);
        }
        float ee = 0.0f;
        for (int c = 0; c < D; ++c) {
            float e = 0.0f;
#pragma unroll
            for (int j = 0; j < 7; ++j) e = fmaf(tsit5_btilde(j), k[j][c], e);
            e *= h;
            const float sc = abstol + reltol * fmaxf(fabsf(u[c]), fabsf(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const float EEst = sqrtf(ee / D);
        if (!(EEst <= 3.0e38f)) { bad = 1; break; }   // NaN / Inf
        const float q11 = powf(EEst, beta1);
        float q = fminf(fmaxf(q11 / powf(qold, beta2) / gamma, 1.0f / qmax), 1.0f / qmin);
        if (EEst <= 1.0f) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            const float tn = clipped ? t1 : t + h;
            // dense record of this step: k_1..k_6 at rows nacc*6 + i, k_7 at (nacc+1)*6 (= k_1 of the next step)
            for (int i = 1; i < 7; ++i) store(p.dense, nacc * 6 + i, k[i]);
            while (isave < ap.n_save) {
                const float ts = t0 + ap.save_dt * (float)isave;
                if (ts > tn + 1e-6f * fabsf(tn)) break;
                float bw[7];
                tsit5_bw_rt(fminf((ts - t) / h, 1.0f), bw);
                for (int c = 0; c < D; ++c) {
                    float acc = 0.0f;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fmaf(bw[j], k[j][c], acc);
                    p.out[((size_t)isave * D + c) * N + n] = fmaf(h, acc, u[c]);
                }
                ++isave;
            }
            qold = fmaxf(EEst, 1e-4f);
            // qsteady_min = qsteady_max = 1 for explicit RK methods in OrdinaryDiffEq (the 6/5 band is the implicit-solver default): no dead band
            if (!clipped || h >= dt) dt = h / q;
            else dt = fmaxf(dt, h / q);
            t = tn;
            ++nacc;
            ap.tgrid[(size_t)nacc * N + n] = t;
            for (int c = 0; c < D; ++c) { u[c] = un[c]; k[0][c] = k[6][c]; }
            store(p.ustep, nacc, u);
        } else {
            dt = h / fminf(1.0f / qmin, q11 / gamma);
        }
    }
    if (bad) {   // failed solve (non-finite error estimate / max_steps): the unreached save points are NaN, as a failed retcode would signal
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = __int_as_float(0x7fc00000);
    }
    ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabsf(u[c]) <= 3.0e38f);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// Vern7 with OrdinaryDiffEq's PI controller (abstol / reltol; scenario_1.jl:84-85, seir_exposure.jl:138-139).  The save times
// are step end points (tstops), exactly as the oracle's Vern7 path does (saveat through the lazy 7th-order interpolant:
// B200UDE_FLAG_VERN7_DENSE, vern7_dense.cuh); the step sequence between save points is the controller's own.  No dense record is written
// (the interpolating adjoint of a Vern7 solve is taken over a Tsit5 re-solve, see b200ude.cu).  With ap.tgrid set
// (discrete-adjoint handles) every accepted step is recorded -- tgrid, ustep, hstep, nacc -- for the discrete adjoint.
template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) vern7_adaptive_forward_kernel(FwdParams p, AdaptParams ap)
{
    const int D = c_gen.D;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const float t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (float)(ap.n_save - 1);
    const float abstol = ap.abstol, reltol = ap.reltol;
    const float gamma = 0.9f, qmin = 0.2f, qmax = 10.0f, beta1 = 7.0f / 70.0f, beta2 = 2.0f / 35.0f;   // order 7
    const bool record = ap.tgrid != nullptr;
    float u[MAXD], un[MAXD], g[MAXD], k[10][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    for (int c = 0; c < D; ++c) p.out[(size_t)c * N + n] = u[c];
    if (record) {
        ap.tgrid[n] = t0;
        for (int c = 0; c < D; ++c) p.ustep[(size_t)c * N + n] = u[c];
    }
    model_rhs(u, k[0]);
    float dt;
    {
        float d0 = 0.f, d1 = 0.f, d2 = 0.f;
        for (int c = 0; c < D; ++c) {
            const float sk = abstol + reltol * fabsf(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = sqrtf(d0 / D); d1 = sqrtf(d1 / D);
        float dt0 = (d0 < 1e-5f || d1 < 1e-5f) ? 1e-6f : 0.01f * d0 / d1;
        dt0 = fminf(dt0, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fmaf(dt0, k[0][c], u[c]);
        model_rhs(g, un);
        for (int c = 0; c < D; ++c) {
            const float sk = abstol + reltol * fabsf(u[c]);
            const float e = (un[c] - k[0][c]) / sk;
            d2 += e * e;
        }
        d2 = sqrtf(d2 / D) / dt0;
        const float dm = fmaxf(d1, d2);
        const float dt1 = dm <= 1e-15f ? fmaxf(1e-6f, dt0 * 1e-3f) : exp10f(-(2.0f + log10f(dm)) / 7.0f);
        dt = fminf(fminf(100.0f * dt0, dt1), t1 - t0);
    }
    float t = t0, qold = 1e-4f;
    int nacc = 0, isave = 1, bad = 0;
    bool have_k1 = true;
    while (isave < ap.n_save) {
        const float tend = t0 + ap.save_dt * (float)isave;
        float h = dt;
        bool clipped = false;
        if (t + h >= tend - 1e-6f * fabsf(tend)) { h = tend - t; clipped = true; }
        if (!have_k1) model_rhs(u, k[0]);
#pragma unroll
        for (int i = 1; i < 10; ++i) {
            for (int c = 0; c < D; ++c) {
                float acc = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) acc = fmaf((float)Vern7::a(i, j), k[j][c], acc);
                g[c] = fmaf(h, acc, u[c]);
            }
            model_rhs(g, k[i]);
        }
        float ee = 0.0f;
        for (int c = 0; c < D; ++c) {
            float acc = 0.0f, e = 0.0f;
#pragma unroll
            for (int j = 0; j < 10; ++j) {
                if (Vern7::b(j) != 0.0) acc = fmaf((float)Vern7::b(j), k[j][c], acc);
                if (Vern7::bt(j) != 0.0) e = fmaf((float)Vern7::bt(j), k[j][c], e);
            }
            un[c] = fmaf(h, acc, u[c]);
            e *= h;
            const float sc = abstol + reltol * fmaxf(fabsf(u[c]), fabsf(un[c]));
            ee += (e / sc) * (e / sc);
        }
        const float EEst = sqrtf(ee / D);
        if (!(EEst <= 3.0e38f)) { bad = 1; break; }
        const float q11 = powf(EEst, beta1);
        float q = fminf(fmaxf(q11 / powf(qold, beta2) / gamma, 1.0f / qmax), 1.0f / qmin);
        if (EEst <= 1.0f) {
            if (nacc >= ap.max_steps) { bad = 2; break; }
            if (record) ap.hstep[(size_t)nacc * N + n] = h;
            ++nacc;
            if (clipped) {
                for (int c = 0; c < D; ++c) p.out[((size_t)isave * D + c) * N + n] = un[c];
                ++isave;
            }
            qold = fmaxf(EEst, 1e-4f);
            // qsteady_min = qsteady_max = 1 for explicit RK methods in OrdinaryDiffEq (the 6/5 band is the implicit-solver default): no dead band
            if (!clipped || h >= dt) dt = h / q;
            else dt = fmaxf(dt, h / q);
            t = clipped ? tend : t + h;
            if (record) {
                ap.tgrid[(size_t)nacc * N + n] = t;
                for (int c = 0; c < D; ++c) p.ustep[((size_t)nacc * D + c) * N + n] = un[c];
            }
            for (int c = 0; c < D; ++c) u[c] = un[c];
            have_k1 = false;   // not FSAL
        } else {
            dt = h / fminf(1.0f / qmin, q11 / gamma);
            have_k1 = true;    // k_1 = f(u) is still valid after a rejection
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < ap.n_save; ++is)
            for (int c = 0; c < D; ++c) p.out[((size_t)is * D + c) * N + n] = __int_as_float(0x7fc00000);
    }
    if (ap.nacc) ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabsf(u[c]) <= 3.0e38f);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

template <int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_adjoint_kernel(AdjParams p, AdaptParams ap)
{
    extern __shared__ __align__(16) float s_g[];   // [BLOCK/32][P+1]
    const int D = c_gen.D, P = c_gen.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0f;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const int nacc = ap.nacc[n];
    int nmax = live ? nacc : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    float lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD], un_[MAXD];
    float loss = 0.0f;
    for (int c = 0; c < D; ++c) lam[c] = 0.0f;
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
        const float tn = ap.tgrid[(size_t)sc_ * N + n], tn1 = ap.tgrid[(size_t)(sc_ + 1) * N + n], hn = tn1 - tn;
        const float eps = 1e-5f * hn;
        for (int c = 0; c < D; ++c) un_[c] = __ldg(p.ustep + ((size_t)sc_ * D + c) * N + n);
        float cur = tn1;
        while (true) {
            const bool has = act_s && cur > tn + eps;
            if (!__any_sync(0xffffffffu, has)) break;
            float ta = tn;
            const float ts = ap.t0 + ap.save_dt * (float)isave;
            if (has && isave >= 0 && ts > tn + eps) ta = ts;
            const float h = has ? cur - ta : 0.0f;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                float bw[7];
                const float Th = fminf(fmaxf((cur - (float)Tsit5::c(i) * h - tn) / hn, 0.0f), 1.0f);
                tsit5_bw_rt(Th, bw);
                for (int c = 0; c < D; ++c) {
                    float acc = 0.0f;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fmaf(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * D + c) * N + n), acc);
                    x[c] = fmaf(hn, acc, un_[c]);
                    float a2 = 0.0f;
#pragma unroll
                    for (int j = 0; j < i; ++j)
                        if (Tsit5::a(i, j) != 0.0) a2 = fmaf((float)Tsit5::a(i, j), kl[j][c], a2);
                    g[c] = fmaf(h, a2, lam[c]);
                }
                model_vjp(x, g, h * (float)Tsit5::b(i), has ? 1.0f : 0.0f, kl[i], gw, lane);
            }
            if (has) {
                for (int c = 0; c < D; ++c) {
                    float acc = 0.0f;
#pragma unroll
                    for (int j = 0; j < 6; ++j) acc = fmaf((float)Tsit5::b(j), kl[j][c], acc);
                    lam[c] = fmaf(h, acc, lam[c]);
                }
                cur = ta;
                if (isave >= 0 && fabsf(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
    }
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    if (lane == 0) gw[P] = 0.0f;   // the adaptive path takes a generic cotangent; no fused loss
    (void)loss;
    __syncwarp();
    float *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

// =====================================================================================================
// Fisher-KPP UPDE (FisherKPP/Fisher-KPP-CNN.jl:111-126, LotkaVolterra/scenario_3.jl:103-114):
//   du_i = NN(u_i) + D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1}),  periodic, theta = [chain | w1 w2 w3 b | D0].
// One thread per grid point; a CTA holds `tpc` whole trajectories (tpc * Nx threads, rounded up to a warp
// multiple); neighbours are exchanged through shared memory.  The handle's internal stores (ustep, dense)
// are point-fastest ([row][trajectory][point]) so that every warp access is contiguous; the ABI arrays
// (u0, out, data, grad_u0) keep the documented trajectory-fastest layout.
// =====================================================================================================
struct FkppGeom {
    int Nx, tpc;
};

__device__ __forceinline__ float fkpp_exchange(float *sU, int slot, int base, int i, int Nx, bool valid, float v, float &vm, float &vp)
{
    if (valid) sU[slot] = v;
    __syncthreads();
    vm = sU[base + (i + Nx - 1) % Nx];
    vp = sU[base + (i + 1) % Nx];
    __syncthreads();
    return v;
}

template <int DUMMY>
__global__ void fkpp_forward_kernel(FwdParams p, FkppGeom geo)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sU = s_dyn;
    const int Nx = geo.Nx, slots = geo.tpc * Nx;
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float dt = p.dt;
    const int sx = c_gen.P - 5;
    const float w1 = c_theta[sx], w2 = c_theta[sx + 1], w3 = c_theta[sx + 2], D0 = c_theta[sx + 4];
    float u = __ldg(p.u0 + (size_t)i * N + n);
    auto rhs = [&](float g) {
        float gm, gp, y;
        fkpp_exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
        chain_fwd<false>(&g, &y, nullptr, nullptr);
        return fmaf(D0, fmaf(w1, gm, fmaf(w2, g, w3 * gp)), y);
    };
    auto store_int = [&](float *b, int row, float v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
    auto store_abi = [&](float *b, int row, float v) { if (live) b[((size_t)row * Nx + i) * N + n] = v; };
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    float k[7];
    k[0] = rhs(u);
    store_int(p.dense, 0, k[0]);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll
        for (int st = 1; st < 7; ++st) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Tsit5::a(st, j) != 0.0) acc = fmaf((float)Tsit5::a(st, j), k[j], acc);
            const float g = fmaf(dt, acc, u);
            if (st == 6) u = g;
            k[st] = rhs(g);
            store_int(p.dense, s * 6 + st, k[st]);
        }
        store_int(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store_abi(p.out, isave, u); ++isave; }
        k[0] = k[6];
    }
    if (p.status) {
        // a trajectory is flagged when any of its points is non-finite
        const int bad = __syncthreads_or((live && !(fabsf(u) <= 3.0e38f)) ? 1 : 0);   // CTA-wide; refined per trajectory below
        if (bad) {
            if (valid) sU[slot] = (fabsf(u) <= 3.0e38f) ? 0.0f : 1.0f;
            __syncthreads();
            if (live && i == 0) {
                float any = 0.0f;
                for (int q = 0; q < Nx; ++q) any += sU[base + q];
                p.status[n] = any > 0.0f ? 1 : 0;
            }
        } else if (live && i == 0) {
            p.status[n] = 0;
        }
    }
}

template <int DUMMY>
__global__ void fkpp_adjoint_kernel(AdjParams p, FkppGeom geo)
{
    extern __shared__ __align__(16) float s_dyn[];
    const int Nx = geo.Nx, slots = geo.tpc * Nx, P = c_gen.P;
    float *sU = s_dyn;                                   // [slots] neighbour exchange
    float *s_g = s_dyn + ((slots + 3) / 4) * 4;          // [nwarps][P+1]
    const int slot = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0f;
    __syncwarp();
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt;
    const int sx = P - 5;
    const float w1 = c_theta[sx], w2 = c_theta[sx + 1], w3 = c_theta[sx + 2], D0 = c_theta[sx + 4];
    float lam = 0.0f, loss = 0.0f, kl[6];
    auto jump = [&](int isave) {
        const size_t idx = ((size_t)isave * Nx + i) * N + n;   // ABI layout
        if (p.fused_l2) {
            const float r = __ldg(p.ustep + ((size_t)(isave * p.save_every) * N + n) * Nx + i) - __ldg(p.cot + idx);
            loss = fmaf(r, r, loss);
            lam = fmaf(2.0f, r, lam);
        } else {
            lam += __ldg(p.cot + idx);
        }
    };
    const int n_save = p.n_steps / p.save_every + 1;
    jump(n_save - 1);
    for (int s = p.n_steps - 1; s >= 0; --s) {
#pragma unroll
        for (int st = 0; st < 6; ++st) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < 7; ++j)
                if (Tsit5::bw(st, j) != 0.0)
                    acc = fmaf((float)Tsit5::bw(st, j), __ldg(p.dense + ((size_t)(s * 6 + j) * N + n) * Nx + i), acc);
            const float x = fmaf(dt, acc, __ldg(p.ustep + ((size_t)s * N + n) * Nx + i));
            float a2 = 0.0f;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Tsit5::a(st, j) != 0.0) a2 = fmaf((float)Tsit5::a(st, j), kl[j], a2);
            const float g = fmaf(dt, a2, lam);
            const float w = dt * (float)Tsit5::b(st) * lv;
            // neighbours of u (for the stencil-weight gradients) and of lambda (for the transposed stencil)
            float xm, xp, gm, gp, dx;
            fkpp_exchange(sU, slot, base, i, Nx, valid, x, xm, xp);
            fkpp_exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
            chain_vjp(&x, &g, w, &dx, gw, lane);
            kl[st] = dx + D0 * fmaf(w2, g, fmaf(w1, gp, w3 * gm));   // (J^T g)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
            warp_acc(gw, sx + 0, w * D0 * xm * g, lane);
            warp_acc(gw, sx + 1, w * D0 * x * g, lane);
            warp_acc(gw, sx + 2, w * D0 * xp * g, lane);
            warp_acc(gw, sx + 4, w * fmaf(w1, xm, fmaf(w2, x, w3 * xp)) * g, lane);
        }
        float acc = 0.0f;
#pragma unroll
        for (int j = 0; j < 6; ++j) acc = fmaf((float)Tsit5::b(j), kl[j], acc);
        lam = fmaf(dt, acc, lam);
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    if (p.grad_u0 && live) p.grad_u0[(size_t)i * N + n] = lam;
    loss *= lv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    float *dst = p.partial + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace generic
}  // namespace b200ude
