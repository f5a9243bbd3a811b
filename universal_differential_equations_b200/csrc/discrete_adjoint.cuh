// discrete_adjoint.cuh -- discrete adjoint (sensealg = ForwardDiffSensitivity, B200UDE_DISCRETE_ADJOINT) of the runtime-shape
// explicit RK solves, written once over the real type and the tableau (Tsit5 or Vern7), fixed step or over the accepted steps of
// an adaptive Vern7 solve.
//
// The quantity is the exact derivative of the discrete scheme with the accepted step sequence held fixed, which is what
// ForwardDiffSensitivity computes (scenario_1.jl:84-87, scenario_2.jl:106-108, hudson_bay.jl:99-102): dual numbers through the
// stages, t and dt plain floats.  Per accepted step n, walking backwards from the last one:
//   1. load u_n (ustep) and h_n (dt, or hstep of the adaptive record);
//   2. recompute the stages g_i = u_n + h sum_{j<i} a_ij k_j, k_i = f(g_i) with the forward's own expression (bitwise the
//      forward's stages: no stage store, the record stays (steps + 1) x D x N);
//   3. kbar_i = h (b_i lambda_{n+1} + sum_{j>i} a_ji gbar_j),  gbar_i = J_u(g_i)^T kbar_i,  grad_theta += J_theta(g_i)^T kbar_i,
//      lambda_n = lambda_{n+1} + sum_i gbar_i.
// Only the stages that feed the update take part: Tsit5's k_7 (FSAL, b_7 = 0) and Vern7's 10th stage (error estimate only) do not
// enter the frozen-step scheme.  Where step n ends on a save point, the loss cotangent is added to lambda_{n+1} first: every
// save_every steps on a fixed grid; on an adaptive Vern7 grid at the steps clipped to a save time (save times are tstops).  With
// fused_l2 the cotangent is 2 w (u - data) of the recorded step-end state, which for Vern7 is bitwise the saved state.
//
// Geometry of the other runtime-shape adjoints: one trajectory per thread, grad_theta summed over the warp with a fixed shuffle
// tree into a per-warp shared vector, then one partial row per warp and the fixed-order reduce -- bitwise deterministic.  In
// adaptive mode the warp loops over its longest record; lanes with shorter records shadow step 0 with a zero cotangent, so the
// shuffles stay convergent and each trajectory's grad_u0 does not depend on its neighbours.
//
// `Ops` is the precision of the runtime-shape model layer (ude_generic.cuh): k_generic.cu instantiates it in fp32 (Ops32),
// k_f64.cu in fp64 (Ops64).  The stage VJPs go through generic::model_vjp with unit quadrature weight (h is inside kbar).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tsit5.cuh"
#include "ude_generic.cuh"
#include "vern7.cuh"

namespace b200ude {
namespace discrete {

// stages that feed the solution update, and their tableau
struct Tsit5Scheme {
    static constexpr int S = 6;
    __host__ __device__ static constexpr double a(int i, int j) { return Tsit5::a(i, j); }
    __host__ __device__ static constexpr double b(int j) { return Tsit5::b(j); }
};
struct Vern7Scheme {
    static constexpr int S = 9;
    __host__ __device__ static constexpr double a(int i, int j) { return Vern7::a(i, j); }
    __host__ __device__ static constexpr double b(int j) { return Vern7::b(j); }
};

template <typename R>
struct Params {
    const R *ustep;      // [steps+1][D][N]  u_n of every step (fixed: every step of the grid; adaptive: every accepted step)
    const R *cot;        // fused_l2 ? data : dL/dout, [n_save][D][N]
    R *grad_u0;          // [D][N] or nullptr
    R *partial;          // [gridDim.x * BLOCK/32][P+1], last entry = partial loss
    const R *tgrid;      // adaptive: [max_steps+1][N] step end times; nullptr = fixed step
    const R *hstep;      // adaptive: [max_steps][N] the step sizes the forward used
    const int *nacc;     // adaptive: [N] accepted steps
    int N, n_steps, save_every, n_save, fused_l2;
    R dt, t0, save_dt, margin;   // margin: a step end within `margin` of a save time is that save point (adaptive)
};

template <class Ops, class Tab, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(Params<typename Ops::real> p)
{
    using R = typename Ops::real;
    constexpr int S = Tab::S, MAXD = Ops::MAXD;
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
    const bool adaptive = p.tgrid != nullptr;
    const int nst = adaptive ? p.nacc[n] : p.n_steps;   // this trajectory's steps
    int nmax = live ? nst : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    R lam[MAXD], u[MAXD], gs[S][MAXD], k[S][MAXD], gb[S][MAXD], kb[MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    // loss cotangent of save point `is`, whose state is the step-end state in ustep row `row` (row < 0: a save point the solve
    // never reached -- its saved state is NaN, and so are the loss and the cotangent of the fused L2)
    auto jump = [&](int is, int row) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)is * D + c) * N + n;
            if (p.fused_l2) {
                const R us = row >= 0 ? p.ustep[((size_t)row * D + c) * N + n] : (R)NAN;
                const R r = us - p.cot[idx];
                const R wgt = Ops::lossw(c);
                loss = fma(wgt * r, r, loss);
                lam[c] = fma((R)2 * wgt, r, lam[c]);
            } else {
                lam[c] += p.cot[idx];
            }
        }
    };
    auto save_time = [&](int is) { return p.t0 + p.save_dt * (R)is; };
    int isave = p.n_save - 1;
    if (live && adaptive) {   // save points past the last accepted step (failed solve: non-finite state or max_steps)
        const R tend = p.tgrid[(size_t)nst * N + n];
        while (isave > 0 && tend < save_time(isave) - p.margin * fabs(save_time(isave))) { jump(isave, -1); --isave; }
    }
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act = live && s < nst;
        const int sr = act ? s : 0;   // inactive lanes shadow step 0 (finite data) with a zero cotangent
        bool at_save;
        if (adaptive) {
            // a step clipped to save time ts ends at ts; every other step ends more than twice the margin before the next save time
            const R te = p.tgrid[(size_t)(sr + 1) * N + n], ts = save_time(isave);
            at_save = isave > 0 && fabs(te - ts) <= p.margin * fabs(ts);
        } else {
            at_save = (s + 1) % p.save_every == 0;
        }
        if (act && at_save) { jump(isave, s + 1); --isave; }
        const R h = adaptive ? p.hstep[(size_t)sr * N + n] : p.dt;
        for (int c = 0; c < D; ++c) u[c] = p.ustep[((size_t)sr * D + c) * N + n];
        // stages, as the forward kernels evaluate them
        for (int c = 0; c < D; ++c) gs[0][c] = u[c];
        generic::model_rhs<Ops>(u, k[0]);
#pragma unroll
        for (int i = 1; i < S; ++i) {
            for (int c = 0; c < D; ++c) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tab::a(i, j) != 0.0) acc = fma((R)Tab::a(i, j), k[j][c], acc);
                gs[i][c] = fma(h, acc, u[c]);
            }
            generic::model_rhs<Ops>(gs[i], k[i]);
        }
        // reverse recurrence through the stages
        const R lv = act ? (R)1 : (R)0;
#pragma unroll
        for (int i = S - 1; i >= 0; --i) {
            for (int c = 0; c < D; ++c) {
                R acc = Tab::b(i) != 0.0 ? (R)Tab::b(i) * lam[c] : (R)0;
#pragma unroll
                for (int j = i + 1; j < S; ++j)
                    if (Tab::a(j, i) != 0.0) acc = fma((R)Tab::a(j, i), gb[j][c], acc);
                kb[c] = act ? h * acc : (R)0;
            }
            generic::model_vjp<Ops>(gs[i], kb, (R)1, lv, gb[i], gw, lane);
        }
        if (act)
            for (int c = 0; c < D; ++c) {
                R acc = lam[c];
#pragma unroll
                for (int i = 0; i < S; ++i) acc += gb[i][c];
                lam[c] = acc;
            }
    }
    if (live) jump(0, 0);
    if (p.grad_u0 && live)
        for (int c = 0; c < D; ++c) p.grad_u0[(size_t)c * N + n] = lam[c];
    loss *= live ? (R)1 : (R)0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (BLOCK / 32) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace discrete
}  // namespace b200ude
