// seir_tc.cuh -- tensor-core kernels of the SEIR exposure UDE (SEIR_exposure/seir_exposure.jl:114-130):
// 7 states (S, E, I, R, N, D, C), chain 3 -> 64 -> 64 -> 1 (tanh, tanh, linear) on [S/N, I, D/N], P = 4481.
//
// Same building block as lv32_tc.cuh, one size up: the 64 x 64 layer of the 32 trajectories of a warp is a
// [32 x 64] x [64 x 64] GEMM of 3xTF32 mma.sync.m16n8k8 tiles (384 HMMA per warp and sweep), activations passed through
// the warp's rows in shared memory by the thread that owns the trajectory.  A CTA holds TWO independent groups of 128
// trajectories (256 threads) that share one staged copy of W2 (hi/lo; the transposed product reads it transposed); each
// group has its own named barrier and staging buffers.  One CTA per SM (up to 209 KB of shared memory).
// Adjoint: the two sweeps (chain forward, W2^T q2) on the tensor core; the ensemble-summed dW2 += q2 (x) h1
// (64 x 64 outputs, K = the group's 128 trajectories) is a 3xTF32 mma.sync GEMM (or FFMA 8 x 4 register tiles) over the
// staged rows; the thin layers are thread-owned column sums.  Deterministic: per-group partials, fixed-order final reduce.
#pragma once
#include "vern7.cuh"
#include "lv32_tc.cuh"
#include "step_control.cuh"

namespace b200ude {
namespace seir {

using lv32::ldw4;
using lv32::bc;
using lv32::fma2;
using namespace lv32::tc;   // tensor-core helpers (warp_gemm, split_tf32, tf32_rna, row load / store)

constexpr int D = 7, DIN = 3, HS = 64;
constexpr int OFF_W1 = 0;               // W1[j, m] at m*64 + j
constexpr int OFF_B1 = 3 * HS;          // 192
constexpr int OFF_W2 = OFF_B1 + HS;     // 256, W2[j, i] at i*64 + j
constexpr int OFF_B2 = OFF_W2 + HS * HS; // 4352
constexpr int OFF_W3 = OFF_B2 + HS;     // 4416, W3[0, j] at j
constexpr int OFF_B3 = OFF_W3 + HS;     // 4480
constexpr int PS = OFF_B3 + 1;          // 4481

constexpr int SWS = HS + 4;   // row stride (floats) of the staged W2: conflict-free B fragments of the forward product
constexpr int SLD64 = 68;     // staged activation row stride (floats): 64 + 4
constexpr int GROUP = 128, GROUPS = 2, BLOCK = GROUP * GROUPS;

// W2[j][i] (theta[OFF_W2 + i*64 + j]) at j * SWS + i, hi / lo split: B(k = i, n = j) of the forward product h1 W2^T and,
// read transposed, B(k = j, n = i) of q2 W2
__device__ __forceinline__ void stage_weights64(const float *__restrict__ theta, float *sBhi, float *sBlo, int tid, int nthreads)
{
    for (int e = tid; e < HS * HS; e += nthreads) {
        const int j = e >> 6, i = e & 63;
        const float x = theta[OFF_W2 + i * HS + j];
        const float hi = tf32_rna(x);
        sBhi[j * SWS + i] = hi;
        sBlo[j * SWS + i] = x - hi;
    }
}

struct GrpCtx {
    float *rows;   // this warp's 32 activation rows (row r belongs to lane r)
    int bar_id;    // named barrier of this group (1 + group)
};
__device__ __forceinline__ void group_sync(int id) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(GROUP) : "memory"); }
__device__ __forceinline__ GrpCtx group_ctx(float *cta_rows) { return GrpCtx{cta_rows + (threadIdx.x >> 5) * 32 * SLD64, 1 + (int)(threadIdx.x / GROUP)}; }

// d = a W2^T for this thread's 64-wide row a, through the warp's rows
__device__ __forceinline__ void gemm_row64(const GrpCtx &c, const float (&a)[HS], const float *sBhi, const float *sBlo, float (&d)[HS])
{
    float *row = c.rows + (threadIdx.x & 31) * SLD64;
    store_row(row, a);
    warp_gemm<HS, HS, SLD64, SWS, false>(c.rows, c.rows, sBhi, sBlo);
    load_row(row, d);
}

struct State7 {
    float v[D];
};

// chain input [S/N, I, D/N] (seir_exposure.jl:120)
__device__ __forceinline__ void seir_inputs(const float (&u)[D], float (&x)[3])
{
    const float invN = 1.0f / u[4];
    x[0] = u[0] * invN;
    x[1] = u[2];
    x[2] = u[5] * invN;
}

// ---- UDE right-hand side (seir_exposure.jl:117-130), the 64 x 64 layer on the tensor core ----
template <int TM>
__device__ __noinline__ State7 rhs_seir(const GrpCtx *cp, const float *sWhi, const float *sWlo, State7 us, int zsel)
{
    const GrpCtx c = *cp;
    const int zb = lv32::c_zero[zsel & 7] << 2;
    float x[3];
    seir_inputs(us.v, x);
    float h[HS];
#pragma unroll
    for (int j4 = 0; j4 < HS; j4 += 4) {
        const float4 wb = ldw4(zb + OFF_B1 + j4), w0 = ldw4(zb + OFF_W1 + j4), w1 = ldw4(zb + OFF_W1 + HS + j4), w2 = ldw4(zb + OFF_W1 + 2 * HS + j4);
        const float b_[4] = {wb.x, wb.y, wb.z, wb.w}, w0_[4] = {w0.x, w0.y, w0.z, w0.w}, w1_[4] = {w1.x, w1.y, w1.z, w1.w}, w2_[4] = {w2.x, w2.y, w2.z, w2.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) h[j4 + k] = fmaf(w2_[k], x[2], fmaf(w1_[k], x[1], fmaf(w0_[k], x[0], b_[k])));
        lv32::tanh_quad_s<TM>(h[j4], h[j4 + 1], h[j4 + 2], h[j4 + 3]);   // one reciprocal per four values (lv32_packed.cuh)
    }
    gemm_row64(c, h, sWhi, sWlo, h);
    float z = c_theta[zb + OFF_B3];
#pragma unroll
    for (int j4 = 0; j4 < HS; j4 += 4) {
        const float4 b2 = ldw4(zb + OFF_B2 + j4), w3 = ldw4(zb + OFF_W3 + j4);
        const float b_[4] = {b2.x, b2.y, b2.z, b2.w}, w3_[4] = {w3.x, w3.y, w3.z, w3.w};
        float t_[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) t_[k] = h[j4 + k] + b_[k];
        lv32::tanh_quad_s<TM>(t_[0], t_[1], t_[2], t_[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) z = fmaf(w3_[k], t_[k], z);
    }
    // consts = F, beta0, alpha, kappa, mu, sigma, gamma, d, lambda (seir_exposure.jl:33)
    const float F = c_consts[0], b0 = c_consts[1], mu = c_consts[4], sg = c_consts[5], gm = c_consts[6], dd = c_consts[7], lm = c_consts[8];
    const float S = us.v[0], E = us.v[1], I = us.v[2], R = us.v[3], N = us.v[4], Dd = us.v[5];
    const float inf = b0 * S * F / N;
    State7 du;
    du.v[0] = -inf - z - mu * S;
    du.v[1] = inf + z - (sg + mu) * E;
    du.v[2] = sg * E - (gm + mu) * I;
    du.v[3] = gm * I - mu * R;
    du.v[4] = -mu * N;
    du.v[5] = dd * gm * I - lm * Dd;
    du.v[6] = sg * E;
    return du;
}

// ---- forward kernel --------------------------------------------------------------------------------------
template <int TM>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(FwdParams p)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sWf_hi = s_dyn, *sWf_lo = s_dyn + HS * SWS;
    const GrpCtx c = group_ctx(s_dyn + 2 * HS * SWS);
    stage_weights64(p.theta, sWf_hi, sWf_lo, threadIdx.x, BLOCK);
    __syncthreads();

    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float dt = p.dt;
    State7 u;
#pragma unroll
    for (int cc = 0; cc < D; ++cc) u.v[cc] = __ldg(p.u0 + (size_t)cc * N + n);
    auto store = [&](float *base, int row, const State7 &v) {
        if (live) {
#pragma unroll
            for (int cc = 0; cc < D; ++cc) base[((size_t)row * D + cc) * N + n] = v.v[cc];
        }
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    State7 k[7];
#pragma unroll
    for (int j = 0; j < 7; ++j)
#pragma unroll
        for (int cc = 0; cc < D; ++cc) k[j].v[cc] = 0.0f;
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll 1
        for (int i = (s == 0 ? 0 : 1); i < 7; ++i) {
            State7 g;
#pragma unroll
            for (int cc = 0; cc < D; ++cc) g.v[cc] = 0.0f;
#define B200UDE_SEIR_COMB(I)                                                              \
    case I: {                                                                             \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) {        \
            _Pragma("unroll") for (int cc = 0; cc < D; ++cc)                              \
                g.v[cc] = fmaf((float)Tsit5::a(I, j), k[j].v[cc], g.v[cc]);               \
        }                                                                                 \
    } break;
            switch (i) {
                B200UDE_SEIR_COMB(1)
                B200UDE_SEIR_COMB(2)
                B200UDE_SEIR_COMB(3)
                B200UDE_SEIR_COMB(4)
                B200UDE_SEIR_COMB(5)
                B200UDE_SEIR_COMB(6)
            default: break;
            }
#undef B200UDE_SEIR_COMB
#pragma unroll
            for (int cc = 0; cc < D; ++cc) g.v[cc] = fmaf(dt, g.v[cc], u.v[cc]);
            if (i == 6) u = g;   // stage 7's argument is u_{n+1} (row 7 = b, FSAL)
            const State7 kk = rhs_seir<TM>(&c, sWf_hi, sWf_lo, g, i);
            switch (i) {
            case 0: k[0] = kk; break;
            case 1: k[1] = kk; break;
            case 2: k[2] = kk; break;
            case 3: k[3] = kk; break;
            case 4: k[4] = kk; break;
            case 5: k[5] = kk; break;
            default: k[6] = kk; break;
            }
            store(p.dense, s * 6 + i, kk);
        }
        store(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) {
            store(p.out, isave, u);
            ++isave;
        }
        k[0] = k[6];
    }
    if (p.status && live) {
        bool ok = true;
#pragma unroll
        for (int cc = 0; cc < D; ++cc) ok = ok && (fabsf(u.v[cc]) <= 3.0e38f);
        p.status[n] = ok ? 0 : 1;
    }
}

// ---- Vern7 forward kernel (fixed step): the reference's solver for this model (seir_exposure.jl:138, Vern7()), 9 stages per step
// (the 10th only feeds the error estimate of the adaptive controller), saved states only -- Vern7's lazy dense output is not
// available (DESIGN.md section 1), so the interpolating adjoint of a Vern7 handle runs over a Tsit5 re-solve on these same
// tensor-core kernels.  Stage loop fully unrolled: the tableau entries are FFMA immediates, the right-hand side stays one function.
template <int TM>
__global__ void __launch_bounds__(BLOCK, 1) vern7_forward_kernel(FwdParams p)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sWf_hi = s_dyn, *sWf_lo = s_dyn + HS * SWS;
    const GrpCtx c = group_ctx(s_dyn + 2 * HS * SWS);
    stage_weights64(p.theta, sWf_hi, sWf_lo, threadIdx.x, BLOCK);
    __syncthreads();

    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float dt = p.dt;
    State7 u;
#pragma unroll
    for (int cc = 0; cc < D; ++cc) u.v[cc] = __ldg(p.u0 + (size_t)cc * N + n);
    auto store = [&](float *base, int row, const State7 &v) {
        if (live) {
#pragma unroll
            for (int cc = 0; cc < D; ++cc) base[((size_t)row * D + cc) * N + n] = v.v[cc];
        }
    };
    store(p.out, 0, u);
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
        State7 k[9];
#pragma unroll
        for (int i = 0; i < 9; ++i) {
            State7 g;
#pragma unroll
            for (int cc = 0; cc < D; ++cc) {
                float a = 0.0f;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Vern7::a(i, j) != 0.0) a = fmaf((float)Vern7::a(i, j), k[j].v[cc], a);
                g.v[cc] = fmaf(dt, a, u.v[cc]);
            }
            k[i] = rhs_seir<TM>(&c, sWf_hi, sWf_lo, g, i);
        }
#pragma unroll
        for (int cc = 0; cc < D; ++cc) {
            float a = 0.0f;
#pragma unroll
            for (int j = 0; j < 9; ++j)
                if (Vern7::b(j) != 0.0) a = fmaf((float)Vern7::b(j), k[j].v[cc], a);
            u.v[cc] = fmaf(dt, a, u.v[cc]);
        }
        if ((s + 1) % p.save_every == 0) {
            store(p.out, isave, u);
            ++isave;
        }
    }
    if (p.status && live) {
        bool ok = true;
#pragma unroll
        for (int cc = 0; cc < D; ++cc) ok = ok && (fabsf(u.v[cc]) <= 3.0e38f);
        p.status[n] = ok ? 0 : 1;
    }
}

// ---- adaptive forward kernel (abstol / reltol): Tsit5 + OrdinaryDiffEq's PI controller per trajectory, saveat by the free
// interpolant, step record for the replay adjoint; CTA-uniform attempt loop (see lv32::tc::adaptive_forward_kernel) ----------
template <int TM>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_forward_kernel(FwdParams p, AdaptiveGrid ag)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sWf_hi = s_dyn, *sWf_lo = s_dyn + HS * SWS;
    const GrpCtx c = group_ctx(s_dyn + 2 * HS * SWS);
    stage_weights64(p.theta, sWf_hi, sWf_lo, threadIdx.x, BLOCK);
    __syncthreads();

    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float t0 = ag.t0, t1 = ag.t0 + ag.save_dt * (float)(ag.n_save - 1);
    const float abstol = ag.abstol, reltol = ag.reltol;
    State7 u;
#pragma unroll
    for (int cc = 0; cc < D; ++cc) u.v[cc] = __ldg(p.u0 + (size_t)cc * N + n);
    auto store = [&](float *base, int row, const State7 &v) {
        if (live) {
#pragma unroll
            for (int cc = 0; cc < D; ++cc) base[((size_t)row * D + cc) * N + n] = v.v[cc];
        }
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    if (live) ag.tgrid[n] = t0;
    State7 k[7];
#pragma unroll
    for (int j = 0; j < 7; ++j)
#pragma unroll
        for (int cc = 0; cc < D; ++cc) k[j].v[cc] = 0.0f;
    k[0] = rhs_seir<TM>(&c, sWf_hi, sWf_lo, u, 0);
    store(p.dense, 0, k[0]);
    PIControl<float, 5> pi;
    {   // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
        float d0 = 0.f, d1 = 0.f, d2 = 0.f;
#pragma unroll
        for (int cc = 0; cc < D; ++cc) {
            const float sk = abstol + reltol * fabsf(u.v[cc]);
            d0 += (u.v[cc] / sk) * (u.v[cc] / sk);
            d1 += (k[0].v[cc] / sk) * (k[0].v[cc] / sk);
        }
        d0 = Prec<float>::sq(d0 / D); d1 = Prec<float>::sq(d1 / D);
        const float dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        State7 g;
#pragma unroll
        for (int cc = 0; cc < D; ++cc) g.v[cc] = fmaf(dt0, k[0].v[cc], u.v[cc]);
        const State7 f1 = rhs_seir<TM>(&c, sWf_hi, sWf_lo, g, 1);
#pragma unroll
        for (int cc = 0; cc < D; ++cc) {
            const float sk = abstol + reltol * fabsf(u.v[cc]);
            const float e = (f1.v[cc] - k[0].v[cc]) / sk;
            d2 += e * e;
        }
        d2 = Prec<float>::sq(d2 / D) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    float t = t0;
    int nacc = 0, isave = 1, bad = 0;
#pragma unroll 1
    while (true) {
        const bool active = (isave < ag.n_save) && !bad;
        if (!__syncthreads_or(active ? 1 : 0)) break;
        float h = pi.dt;
        bool clipped = false;
        if (t + h >= t1 - Prec<float>::clip * fabsf(t1)) { h = t1 - t; clipped = true; }
        if (!active) h = 0.0f;
        State7 un = u;
#pragma unroll 1
        for (int i = 1; i < 7; ++i) {
            State7 g;
#pragma unroll
            for (int cc = 0; cc < D; ++cc) g.v[cc] = 0.0f;
#define B200UDE_SEIR_COMB(I)                                                              \
    case I: {                                                                             \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) {        \
            _Pragma("unroll") for (int cc = 0; cc < D; ++cc)                              \
                g.v[cc] = fmaf((float)Tsit5::a(I, j), k[j].v[cc], g.v[cc]);               \
        }                                                                                 \
    } break;
            switch (i) {
                B200UDE_SEIR_COMB(1)
                B200UDE_SEIR_COMB(2)
                B200UDE_SEIR_COMB(3)
                B200UDE_SEIR_COMB(4)
                B200UDE_SEIR_COMB(5)
            default:
                B200UDE_SEIR_COMB(6)
            }
#undef B200UDE_SEIR_COMB
#pragma unroll
            for (int cc = 0; cc < D; ++cc) g.v[cc] = fmaf(h, g.v[cc], u.v[cc]);
            if (i == 6) un = g;
            const State7 kk = rhs_seir<TM>(&c, sWf_hi, sWf_lo, g, i);
            switch (i) {
            case 1: k[1] = kk; break;
            case 2: k[2] = kk; break;
            case 3: k[3] = kk; break;
            case 4: k[4] = kk; break;
            case 5: k[5] = kk; break;
            default: k[6] = kk; break;
            }
        }
        if (active) {
            float ee = 0.0f;
#pragma unroll
            for (int cc = 0; cc < D; ++cc) {
                float e = 0.0f;
#pragma unroll
                for (int j = 0; j < 7; ++j) e = fmaf((float)Tsit5::bt(j), k[j].v[cc], e);
                e *= h;
                const float sc = abstol + reltol * fmaxf(fabsf(u.v[cc]), fabsf(un.v[cc]));
                ee += (e / sc) * (e / sc);
            }
            const float EEst = Prec<float>::sq(ee / D);
            if (!(EEst <= Prec<float>::huge)) {
                bad = 1;
            } else {
                if (pi.judge(EEst)) {
                    if (nacc >= ag.max_steps) {
                        bad = 2;
                    } else {
                        const float tn = clipped ? t1 : t + h;
#pragma unroll
                        for (int i = 1; i < 7; ++i) store(p.dense, nacc * 6 + i, k[i]);
                        while (isave < ag.n_save) {
                            const float ts = t0 + ag.save_dt * (float)isave;
                            if (ts > tn + Prec<float>::clip * fabsf(tn)) break;
                            float bw[7];
                            Tsit5::weights(fminf((ts - t) / h, 1.0f), bw);
                            State7 o;
#pragma unroll
                            for (int cc = 0; cc < D; ++cc) {
                                float acc = 0.0f;
#pragma unroll
                                for (int j = 0; j < 7; ++j) acc = fmaf(bw[j], k[j].v[cc], acc);
                                o.v[cc] = fmaf(h, acc, u.v[cc]);
                            }
                            store(p.out, isave, o);
                            ++isave;
                        }
                        pi.accept(EEst, h, clipped);
                        t = tn;
                        ++nacc;
                        if (live) ag.tgrid[(size_t)nacc * N + n] = t;
                        u = un;
                        k[0] = k[6];
                        store(p.ustep, nacc, u);
                    }
                } else {
                    pi.reject(h);
                }
            }
        }
    }
    if (bad && live) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < ag.n_save; ++is)
#pragma unroll
            for (int cc = 0; cc < D; ++cc) p.out[((size_t)is * D + cc) * N + n] = Prec<float>::nan();
    }
    if (live) ag.nacc[n] = nacc;
    if (p.status && live) {
        bool ok = true;
#pragma unroll
        for (int cc = 0; cc < D; ++cc) ok = ok && (fabsf(u.v[cc]) <= Prec<float>::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// ---- adjoint kernel --------------------------------------------------------------------------------------
struct __align__(16) GroupStage {
    float B1[GROUP * SLD64];   // h2 rows, then q2 rows, then q1 rows   [trajectory][j]
    float B2[GROUP * SLD64];   // h1 rows                                [trajectory][i]
    float SG[GROUP];           // scaled, masked chain-output cotangent
    float U[GROUP * 4];        // chain input [x0, x1, x2, -]
    float RED[GROUP];          // loss reduction scratch
};

// GEMM = 1: the group's gradient GEMM dW2 += q2 (x) h1 (64 x 64 outputs, K = 128 trajectories) as 3xTF32 warp-level
// mma.sync.m16n8k8 -- warp w of the group owns the 16 rows j = 16 w .. 16 w + 15 and all 8 column tiles; fragments are read
// from the staged rows with the bank-conflict-free k permutation of lv32_tc.cuh.  GEMM = 0: FFMA 8 x 4 register tiles.
template <int TM, int GEMM, bool ADAPT = false>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(AdjParams p, AdaptiveGrid ag)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sW_hi = s_dyn, *sW_lo = s_dyn + HS * SWS;
    stage_weights64(p.theta, sW_hi, sW_lo, threadIdx.x, BLOCK);
    __syncthreads();

    const int group = threadIdx.x / GROUP, tg = threadIdx.x % GROUP;
    GroupStage *st = reinterpret_cast<GroupStage *>(s_dyn + 2 * HS * SWS) + group;
    float *const rowB1 = st->B1 + tg * SLD64, *const rowB2 = st->B2 + tg * SLD64;
    const GrpCtx c{st->B1 + (tg & ~31) * SLD64, 1 + group};   // this warp's q2 / q1 rows, the group's barrier
    const int jt = tg >> 4, it = tg & 15;        // dW2 tile: j = jt*8 + jj, i = it*4 + {0,1},{2,3}
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt, inv_dt = 1.0f / dt;
    const float F = c_consts[0], b0 = c_consts[1], mu = c_consts[4], sgm = c_consts[5], gm = c_consts[6], dd = c_consts[7], lm = c_consts[8];

    float2 acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = bc(0.0f);
    float macc[32];   // GEMM = 1: C fragments of this warp's 8 column tiles, tile nt at 4 nt
#pragma unroll
    for (int q = 0; q < 32; ++q) macc[q] = 0.0f;
    float *const sum_row = reinterpret_cast<float *>(reinterpret_cast<GroupStage *>(s_dyn + 2 * HS * SWS) + GROUPS) + threadIdx.x * 33;   // running dW2 sums
    const int lane = threadIdx.x & 31, fg = lane >> 2, tig = lane & 3, wg = tg >> 5;
    // thin layers: thread tg owns column j = tg % 64 over the staged rows [64 * (tg / 64), +64) of its group:
    // a_w3 (dW3[j]), a_b2 (db2[j]), a_b3 (db3), a_w1[m] (dW1[j][m]), a_b1 (db1[j]); the two halves are added at the end
    float a_w3 = 0.f, a_b2 = 0.f, a_b3 = 0.f, a_w10 = 0.f, a_w11 = 0.f, a_w12 = 0.f, a_b1 = 0.f;
    const int jc = tg & 63, tlo = (tg >> 6) * 64;

    float lam[D];
#pragma unroll
    for (int cc = 0; cc < D; ++cc) lam[cc] = 0.0f;
    float loss = 0.0f;
    const int n_save = p.n_steps / p.save_every + 1;
    bool first_flush = true;

    // One evaluation of (df/du)^T g (-> kn) and of the theta-gradient quadrature term at state u, stage argument g:
    // sc = quadrature weight (h b_i), isc = 1 / sc (0 for a masked thread), lvm = 0/1 mask.
    auto eval_core = [&](int stage, const float (&u)[D], const float (&g)[D], float sc, float isc, float lvm, float (&kn)[D]) {
        const int zb = lv32::c_zero[stage] << 2;
        float x[3];
        seir_inputs(u, x);
        const float sg = lvm * sc * (g[1] - g[0]);   // z enters dS with -, dE with +
        group_sync(c.bar_id);                       // the previous stage's column passes are done with SG / U / B1
        st->SG[tg] = sg;
        *reinterpret_cast<float4 *>(&st->U[tg * 4]) = make_float4(x[0], x[1], x[2], 0.0f);

        // ---- chain forward ----
        float v[HS];
#pragma unroll
        for (int j4 = 0; j4 < HS; j4 += 4) {
            const float4 wb = ldw4(zb + OFF_B1 + j4), w0 = ldw4(zb + OFF_W1 + j4), w1 = ldw4(zb + OFF_W1 + HS + j4), w2 = ldw4(zb + OFF_W1 + 2 * HS + j4);
            const float b_[4] = {wb.x, wb.y, wb.z, wb.w}, w0_[4] = {w0.x, w0.y, w0.z, w0.w}, w1_[4] = {w1.x, w1.y, w1.z, w1.w}, w2_[4] = {w2.x, w2.y, w2.z, w2.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) v[j4 + k] = fmaf(w2_[k], x[2], fmaf(w1_[k], x[1], fmaf(w0_[k], x[0], b_[k])));
            lv32::tanh_quad_s<TM>(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);
            *reinterpret_cast<float4 *>(rowB2 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // h1 row
        }
        warp_gemm<HS, HS, SLD64, SWS, false>(st->B2 + (tg & ~31) * SLD64, c.rows, sW_hi, sW_lo);
        load_row(rowB1, v);   // v = W2 h1
        // h2 = tanh(. + b2) -> B1 row;  q2 = W3 * sg * (1 - h2^2) stays in v
#pragma unroll
        for (int j4 = 0; j4 < HS; j4 += 4) {
            const float4 b2 = ldw4(zb + OFF_B2 + j4), w3 = ldw4(zb + OFF_W3 + j4);
            const float b_[4] = {b2.x, b2.y, b2.z, b2.w}, w3_[4] = {w3.x, w3.y, w3.z, w3.w};
            float h2[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) h2[k] = v[j4 + k] + b_[k];
            lv32::tanh_quad_s<TM>(h2[0], h2[1], h2[2], h2[3]);
#pragma unroll
            for (int k = 0; k < 4; ++k) v[j4 + k] = w3_[k] * sg * fmaf(-h2[k], h2[k], 1.0f);
            *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(h2[0], h2[1], h2[2], h2[3]);
        }
        group_sync(c.bar_id);
        // column pass A: dW3[j] += sum_t SG[t] h2[t][j];  db3 += sum_t SG[t]
#pragma unroll 8
        for (int t = tlo; t < tlo + 64; ++t) {
            const float sgt = st->SG[t];
            a_w3 = fmaf(sgt, st->B1[t * SLD64 + jc], a_w3);
            a_b3 += sgt;
        }
        group_sync(c.bar_id);
#pragma unroll
        for (int j4 = 0; j4 < HS; j4 += 4) *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // q2 row
        // ---- gradient GEMM of the group, then W2^T q2 on the tensor core (in place over the q2 rows) ----
        group_sync(c.bar_id);
        if constexpr (GEMM == 1) {
#pragma unroll 1
            for (int ks = 0; ks < GROUP / 8; ++ks) {
                const float *q0 = st->B1 + (8 * ks + 2 * tig) * SLD64 + 16 * wg + fg, *q1 = q0 + SLD64;
                const float *h0 = st->B2 + (8 * ks + 2 * tig) * SLD64 + fg, *h1r = h0 + SLD64;
                uint32_t ah[4], al[4];
                lv32::tc::split_tf32(q0[0], ah[0], al[0]);
                lv32::tc::split_tf32(q0[8], ah[1], al[1]);
                lv32::tc::split_tf32(q1[0], ah[2], al[2]);
                lv32::tc::split_tf32(q1[8], ah[3], al[3]);
#pragma unroll
                for (int half = 0; half < 2; ++half) {
                    uint32_t bh[4][2], bl[4][2];
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        lv32::tc::split_tf32(h0[8 * (4 * half + k)], bh[k][0], bl[k][0]);
                        lv32::tc::split_tf32(h1r[8 * (4 * half + k)], bh[k][1], bl[k][1]);
                    }
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        float (&cf)[4] = *reinterpret_cast<float (*)[4]>(&macc[4 * (4 * half + k)]);
                        lv32::tc::mma_m16n8k8(cf, al, bh[k]);
                        lv32::tc::mma_m16n8k8(cf, ah, bl[k]);
                        lv32::tc::mma_m16n8k8(cf, ah, bh[k]);
                    }
                }
            }
            lv32::tc::flush32(sum_row, macc, first_flush); first_flush = false;   // per evaluation: 48-MMA chains
#pragma unroll 8
            for (int t = tlo; t < tlo + 64; ++t) a_b2 += st->B1[t * SLD64 + jc];   // db2[j] += sum_t q2[t][j]
        } else {
            float4 G0[2], G1[2], Hh[2];
            auto load_row = [&](int t, int b) {
                const float *r1 = st->B1 + t * SLD64, *r2 = st->B2 + t * SLD64;
                G0[b] = *reinterpret_cast<const float4 *>(r1 + jt * 8);
                G1[b] = *reinterpret_cast<const float4 *>(r1 + jt * 8 + 4);
                Hh[b] = *reinterpret_cast<const float4 *>(r2 + it * 4);
            };
            auto use_row = [&](int b) {
                const float gj[8] = {G0[b].x, G0[b].y, G0[b].z, G0[b].w, G1[b].x, G1[b].y, G1[b].z, G1[b].w};
                const float2 h01 = make_float2(Hh[b].x, Hh[b].y), h23 = make_float2(Hh[b].z, Hh[b].w);
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    acc[2 * jj] = fma2(bc(gj[jj]), h01, acc[2 * jj]);
                    acc[2 * jj + 1] = fma2(bc(gj[jj]), h23, acc[2 * jj + 1]);
                }
            };
            load_row(0, 0);
#pragma unroll 1
            for (int t = 0; t < GROUP; t += 2) {
                load_row(t + 1, 1);
                use_row(0);
                if (t + 2 < GROUP) load_row(t + 2, 0);
                use_row(1);
            }
#pragma unroll 8
            for (int t = tlo; t < tlo + 64; ++t) a_b2 += st->B1[t * SLD64 + jc];   // db2[j] += sum_t q2[t][j]
        }
        group_sync(c.bar_id);  // everyone is done reading q2 / h1 rows
        warp_gemm<HS, HS, SLD64, SWS, true>(c.rows, c.rows, sW_hi, sW_lo);
        load_row(rowB1, v);   // v = W2^T q2
        float dx0 = 0.0f, dx1 = 0.0f, dx2 = 0.0f;
#pragma unroll
        for (int j4 = 0; j4 < HS; j4 += 4) {
            const float4 hh = *reinterpret_cast<const float4 *>(rowB2 + j4);
            const float4 w0 = ldw4(zb + OFF_W1 + j4), w1 = ldw4(zb + OFF_W1 + HS + j4), w2 = ldw4(zb + OFF_W1 + 2 * HS + j4);
            const float h_[4] = {hh.x, hh.y, hh.z, hh.w}, w0_[4] = {w0.x, w0.y, w0.z, w0.w}, w1_[4] = {w1.x, w1.y, w1.z, w1.w}, w2_[4] = {w2.x, w2.y, w2.z, w2.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                v[j4 + k] *= fmaf(-h_[k], h_[k], 1.0f);   // q1
                dx0 = fmaf(w0_[k], v[j4 + k], dx0);
                dx1 = fmaf(w1_[k], v[j4 + k], dx1);
                dx2 = fmaf(w2_[k], v[j4 + k], dx2);
            }
            *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // q1 row
        }
        dx0 *= isc; dx1 *= isc; dx2 *= isc;   // cotangent of the chain input, quadrature weight removed
        // (df/du)^T g: physics Jacobian of seir_exposure.jl:117-130 plus the chain-input map [S/N, I, D/N]
        {
            const float S = u[0], Nn = u[4], Dd = u[5];
            const float cS = b0 * F / Nn, cN = -b0 * S * F / (Nn * Nn), invN = 1.0f / Nn;
                        kn[0] = g[0] * (-cS - mu) + g[1] * cS + dx0 * invN;
            kn[1] = g[1] * (-(sgm + mu)) + g[2] * sgm + g[6] * sgm;
            kn[2] = g[2] * (-(gm + mu)) + g[3] * gm + g[5] * dd * gm + dx1;
            kn[3] = g[3] * (-mu);
            kn[4] = g[0] * (-cN) + g[1] * cN + g[4] * (-mu) - dx0 * S * invN * invN - dx2 * Dd * invN * invN;
            kn[5] = g[5] * (-lm) + dx2 * invN;
            kn[6] = 0.0f;
        }
        group_sync(c.bar_id);
        // column pass B: dW1[j][m] += sum_t q1[t][j] x[t][m];  db1[j] += sum_t q1[t][j]
#pragma unroll 8
        for (int t = tlo; t < tlo + 64; ++t) {
            const float qq = st->B1[t * SLD64 + jc];
            const float4 u4 = *reinterpret_cast<const float4 *>(&st->U[t * 4]);
            a_w10 = fmaf(qq, u4.x, a_w10);
            a_w11 = fmaf(qq, u4.y, a_w11);
            a_w12 = fmaf(qq, u4.z, a_w12);
            a_b1 += qq;
        }
    };
#define B200UDE_SEIR_SETKL_ALL()                                                                      \
    switch (stage) {                                                                                  \
    case 0: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[0][cc] = kn[cc]; break;               \
    case 1: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[1][cc] = kn[cc]; break;               \
    case 2: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[2][cc] = kn[cc]; break;               \
    case 3: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[3][cc] = kn[cc]; break;               \
    case 4: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[4][cc] = kn[cc]; break;               \
    default: _Pragma("unroll") for (int cc = 0; cc < D; ++cc) kl[5][cc] = kn[cc]; break;              \
    }

    if constexpr (!ADAPT) {
    loss_jump<D>(p, n_save - 1, n, N, lam, loss);
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        float kl[6][D];
#pragma unroll
        for (int j = 0; j < 6; ++j)
#pragma unroll
            for (int cc = 0; cc < D; ++cc) kl[j][cc] = 0.0f;
#pragma unroll 1
        for (int stage = 0; stage < 6; ++stage) {
            float u[D], g[D], sc, isc;
#define B200UDE_SEIR_PRE(I)                                        \
    case I: {                                                      \
        interp_state<D, I>(p, s, n, N, dt, u);                     \
        stage_arg<D, I>(lam, kl, dt, g);                           \
        sc = dt * (float)Tsit5::b(I);                              \
        isc = inv_dt * (float)(1.0 / Tsit5::b(I));                 \
    } break;
            switch (stage) {
                B200UDE_SEIR_PRE(0)
                B200UDE_SEIR_PRE(1)
                B200UDE_SEIR_PRE(2)
                B200UDE_SEIR_PRE(3)
                B200UDE_SEIR_PRE(4)
            default:
                B200UDE_SEIR_PRE(5)
            }
#undef B200UDE_SEIR_PRE
            float kn[D];
            eval_core(stage, u, g, sc, isc, lv, kn);
            B200UDE_SEIR_SETKL_ALL()
        }
#pragma unroll
        for (int cc = 0; cc < D; ++cc) {
            float a = 0.0f;
#pragma unroll
            for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j][cc], a);
            lam[cc] = fmaf(dt, a, lam[cc]);
        }
        if (s % p.save_every == 0) loss_jump<D>(p, s / p.save_every, n, N, lam, loss);
    }
    } else {
    // ---- adaptive: replay the accepted forward steps backwards, split at the save times (see lv32_tc.cuh); CTA-uniform loops ----
    __shared__ int s_nmax;
    if (threadIdx.x == 0) s_nmax = 0;
    __syncthreads();
    const int nacc = ag.nacc[n];
    atomicMax(&s_nmax, live ? nacc : 0);
    __syncthreads();
    const int nmax = s_nmax;
    int isave = ag.n_save - 1;
    auto jump = [&](int is) {
#pragma unroll
        for (int cc = 0; cc < D; ++cc) lam[cc] += __ldg(p.cot + ((size_t)is * D + cc) * N + n);
    };
    if (live) jump(isave);
    --isave;
#pragma unroll 1
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act_s = live && s < nacc;
        const int sc_ = act_s ? s : 0;
        const float tn = ag.tgrid[(size_t)sc_ * N + n], tn1 = ag.tgrid[(size_t)(sc_ + 1) * N + n], hn = tn1 - tn;
        const float eps = 1e-5f * hn, inv_hn = 1.0f / hn;
        float cur = tn1;
#pragma unroll 1
        while (true) {
            const bool has = act_s && cur > tn + eps;
            if (!__syncthreads_or(has ? 1 : 0)) break;
            float ta = tn;
            const float ts = ag.t0 + ag.save_dt * (float)isave;
            if (has && isave >= 0 && ts > tn + eps) ta = ts;
            const float h = has ? cur - ta : 0.0f;
            const float lvm = has ? 1.0f : 0.0f, inv_h = has ? 1.0f / h : 0.0f;
            float kl[6][D];
#pragma unroll
            for (int j = 0; j < 6; ++j)
#pragma unroll
                for (int cc = 0; cc < D; ++cc) kl[j][cc] = 0.0f;
#pragma unroll 1
            for (int stage = 0; stage < 6; ++stage) {
                float u[D], g[D], sc, isc, ci;
#define B200UDE_SEIR_PRE(I)                                        \
    case I: {                                                      \
        stage_arg<D, I>(lam, kl, h, g);                            \
        sc = h * (float)Tsit5::b(I);                               \
        isc = inv_h * (float)(1.0 / Tsit5::b(I));                  \
        ci = (float)Tsit5::c(I);                                   \
    } break;
                switch (stage) {
                    B200UDE_SEIR_PRE(0)
                    B200UDE_SEIR_PRE(1)
                    B200UDE_SEIR_PRE(2)
                    B200UDE_SEIR_PRE(3)
                    B200UDE_SEIR_PRE(4)
                default:
                    B200UDE_SEIR_PRE(5)
                }
#undef B200UDE_SEIR_PRE
                {
                    const float Th = fminf(fmaxf((cur - ci * h - tn) * inv_hn, 0.0f), 1.0f);
                    float bw[7];
                    Tsit5::weights(Th, bw);
#pragma unroll
                    for (int cc = 0; cc < D; ++cc) {
                        float acc2 = 0.0f;
#pragma unroll
                        for (int j = 0; j < 7; ++j) acc2 = fmaf(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * D + cc) * N + n), acc2);
                        u[cc] = fmaf(hn, acc2, __ldg(p.ustep + ((size_t)sc_ * D + cc) * N + n));
                    }
                }
                float kn[D];
                eval_core(stage, u, g, sc, isc, lvm, kn);
                B200UDE_SEIR_SETKL_ALL()
            }
            if (has) {
#pragma unroll
                for (int cc = 0; cc < D; ++cc) {
                    float a = 0.0f;
#pragma unroll
                    for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j][cc], a);
                    lam[cc] = fmaf(h, a, lam[cc]);
                }
                cur = ta;
                if (isave >= 0 && fabsf(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
    }
    if constexpr (GEMM == 1) {
        if (first_flush) lv32::tc::flush32(sum_row, macc, true);   // no accepted step at all: the sums are zero
    }
    }
#undef B200UDE_SEIR_SETKL_ALL
    if (p.grad_u0 && live) {
#pragma unroll
        for (int cc = 0; cc < D; ++cc) p.grad_u0[(size_t)cc * N + n] = lam[cc];
    }
    // ---- this group's partial gradient ----
    group_sync(c.bar_id);
    st->RED[tg] = loss * lv;
    if (tg >= 64) {   // upper half of the staged rows: hand the column sums to the lower-half owner of the same column
        float *x = st->B1 + jc * 8;
        x[0] = a_w3; x[1] = a_b2; x[2] = a_b3; x[3] = a_w10; x[4] = a_w11; x[5] = a_w12; x[6] = a_b1;
    }
    group_sync(c.bar_id);
    float *dst = p.partial + ((size_t)blockIdx.x * GROUPS + group) * (PS + 1);
    if constexpr (GEMM == 1) {
#pragma unroll
        for (int q = 0; q < 32; ++q) macc[q] = sum_row[q];
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int j = 16 * wg + fg, i = 8 * nt + 2 * tig;
            dst[OFF_W2 + i * HS + j] = macc[4 * nt + 0];
            dst[OFF_W2 + (i + 1) * HS + j] = macc[4 * nt + 1];
            dst[OFF_W2 + i * HS + j + 8] = macc[4 * nt + 2];
            dst[OFF_W2 + (i + 1) * HS + j + 8] = macc[4 * nt + 3];
        }
    } else {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            dst[OFF_W2 + (it * 4 + 0) * HS + (jt * 8 + jj)] = acc[2 * jj].x;
            dst[OFF_W2 + (it * 4 + 1) * HS + (jt * 8 + jj)] = acc[2 * jj].y;
            dst[OFF_W2 + (it * 4 + 2) * HS + (jt * 8 + jj)] = acc[2 * jj + 1].x;
            dst[OFF_W2 + (it * 4 + 3) * HS + (jt * 8 + jj)] = acc[2 * jj + 1].y;
        }
    }
    if (tg < 64) {
        const float *x = st->B1 + jc * 8;
        dst[OFF_W3 + jc] = a_w3 + x[0];
        dst[OFF_B2 + jc] = a_b2 + x[1];
        dst[OFF_W1 + jc] = a_w10 + x[3];
        dst[OFF_W1 + HS + jc] = a_w11 + x[4];
        dst[OFF_W1 + 2 * HS + jc] = a_w12 + x[5];
        dst[OFF_B1 + jc] = a_b1 + x[6];
        if (tg == 0) {
            dst[OFF_B3] = a_b3 + x[2];
            float ls = 0.0f;
            for (int t = 0; t < GROUP; ++t) ls += st->RED[t];   // fixed order
            dst[PS] = ls;
        }
    }
}

}  // namespace seir
}  // namespace b200ude
