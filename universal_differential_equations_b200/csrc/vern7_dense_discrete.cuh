// vern7_dense_discrete.cuh -- discrete adjoint (sensealg = ForwardDiffSensitivity, B200UDE_DISCRETE_ADJOINT) of the adaptive Vern7
// solve that saves through its lazy 7th-order interpolant (B200UDE_FLAG_DISCRETE_DENSE), written once over the real type.
//
// The forward is vern7_dense.cuh's: the steps stop only at the end of tspan, a save time inside an accepted step is
//     out_s = u_n + h sum_{i in W} b_i(theta_s) k_i,   theta_s = (t_s - t_n) / h,   W = {0, 3..8, 10..15},
// with the extra stages k_10..k_15 functions of u_n and k_0..k_8; a save time on a step end is u_{n+1}.  The quantity here is the
// exact derivative of that discrete computation with the accepted step sizes (and so every theta_s) held fixed, which is what
// ForwardDiffSensitivity computes when OrdinaryDiffEq fills saveat from the interpolant (scenario_1.jl:84-87, scenario_2.jl:106-108,
// hudson_bay.jl:99-102).  Per accepted step n, walking backwards from the last one:
//   1. the loss cotangents sbar_s of the step's save points: one on the step end is added to lambda_{n+1}; one inside adds
//      b_i(theta_s) sbar_s to the cotangent of k_i, i in W, and sbar_s to that of u_n.  A save point belongs to the step the forward
//      filled it in (same margins, from the recorded step end times);
//   2. k_0..k_8 recomputed from u_n and h_n with the forward's own expressions and, if any lane of the warp has a save inside its
//      step, the extra stages after them (stage 9 only feeds the error estimate and never enters);
//   3. the reverse recurrence in the order 15..10, 8..0,
//        kbar_i = h (b_i lambda_{n+1} [i <= 8] + sum_s b_i(theta_s) sbar_s + sum_{j>i} a_ji gbar_j),   gbar_i = J_u(g_i)^T kbar_i,
//        grad_theta += J_theta(g_i)^T kbar_i,   lambda_n = lambda_{n+1} + sum_s sbar_s + sum_i gbar_i,
//      with the stage point g_i = u_n + h sum_j a_ij k_j formed again from the k's instead of kept: 15 stages of MAXD states would
//      not fit beside k and gbar.  gbar_i's slot holds sum_s b_i(theta_s) sbar_s until stage i replaces it.
// With fused_l2 the cotangent is 2 w (out - data) of the saved state the forward returned; save points a failed solve never reached
// hold NaN there, and so do the loss and the gradient (as in discrete_adjoint.cuh).
//
// Geometry of discrete_adjoint.cuh: one trajectory per thread, grad_theta through the fixed shuffle tree into a per-warp shared
// vector, one partial row per warp, fixed-order reduce -- bitwise deterministic.  The warp loops over its longest record; lanes
// with shorter records shadow step 0 with zero weight, and a lane without a save inside its step runs the extra stages with a
// zero cotangent (exact zeros into the sums), so the shuffles stay convergent and a trajectory's grad_u0 does not depend on its
// neighbours.  The loop over a step's save points holds no collective and runs per lane.
//
// `Ops` is the precision of the runtime-shape model layer (ude_generic.cuh), as in discrete_adjoint.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "vern7_dense.cuh"

namespace b200ude {
namespace vern7_dense_discrete {

template <typename R>
struct Params {
    const R *ustep;     // [max_steps+1][D][N]  u_n of every accepted step
    const R *tgrid;     // [max_steps+1][N]     step end times (t0 first)
    const R *hstep;     // [max_steps][N]       the step sizes the forward used
    const int *nacc;    // [N]                  accepted steps
    const R *cot;       // fused_l2 ? data : dL/dout, [n_save][D][N]
    const R *saved;     // fused_l2: the saved states the forward returned, [n_save][D][N]
    R *grad_u0;         // [D][N] or nullptr
    R *partial;         // [gridDim.x * BLOCK/32][P+1], last entry = partial loss
    int N, n_save, fused_l2;
    R t0, save_dt;
};

// a_ji over the update and the extra stages
__host__ __device__ constexpr double a_all(int j, int i) { return j >= 10 ? Vern7Dense::a(j, i) : Vern7::a(j, i); }

// stage I of the reverse recurrence: gb[I] holds sum_s b_I(theta_s) sbar_s on entry and gbar_I on return
template <class Ops, int I>
__device__ __forceinline__ void back_stage(const typename Ops::real *u, typename Ops::real h, const typename Ops::real (*k)[Ops::MAXD],
                                           typename Ops::real (*gb)[Ops::MAXD], const typename Ops::real *lam, bool act,
                                           typename Ops::real *gw, int lane)
{
    using R = typename Ops::real;
    R g[Ops::MAXD], kb[Ops::MAXD];
    const int D = Ops::D();
    vern7_dense::stage_point<Ops, I>(u, h, k, g);
    for (int c = 0; c < D; ++c) {
        R acc = gb[I][c];
        if (I <= 8 && Vern7::b(I) != 0.0) acc = fma((R)Vern7::b(I), lam[c], acc);
#pragma unroll
        for (int j = I + 1; j < 16; ++j)
            if (j != 9 && a_all(j, I) != 0.0) acc = fma((R)a_all(j, I), gb[j][c], acc);
        kb[c] = act ? h * acc : (R)0;
    }
    generic::model_vjp<Ops>(g, kb, (R)1, act ? (R)1 : (R)0, gb[I], gw, lane);
}

template <class Ops, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(Params<typename Ops::real> p)
{
    using R = typename Ops::real;
    using PR = Prec<R>;
    constexpr int MAXD = Ops::MAXD;
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
    const int nst = p.nacc[n];   // this trajectory's steps
    int nmax = live ? nst : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    R lam[MAXD], u[MAXD], sb[MAXD], ssum[MAXD], g[MAXD], k[16][MAXD], gb[16][MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    // loss cotangent of save point `is` (fused L2: 2 w (out - data) of the state the forward saved there)
    auto cotangent = [&](int is) {
        for (int c = 0; c < D; ++c) {
            const size_t idx = ((size_t)is * D + c) * N + n;
            if (p.fused_l2) {
                const R r = p.saved[idx] - p.cot[idx];
                const R wgt = Ops::lossw(c);
                loss = fma(wgt * r, r, loss);
                sb[c] = (R)2 * wgt * r;
            } else {
                sb[c] = p.cot[idx];
            }
        }
    };
    auto save_time = [&](int is) { return p.t0 + p.save_dt * (R)is; };
    // the forward filled save point `is` >= 1 in step s or a later one iff its time lies beyond the margin of step s - 1's end
    auto from_step = [&](int is, int s) {
        if (s == 0) return true;
        const R ta = p.tgrid[(size_t)(s - 1) * N + n], tb = p.tgrid[(size_t)s * N + n];
        return save_time(is) > tb + PR::eta * (tb - ta);
    };
    int isave = p.n_save - 1;
    if (live)   // save points past the last accepted step (failed solve: non-finite state or max_steps)
        while (isave >= 1 && from_step(isave, nst)) {
            cotangent(isave);
            for (int c = 0; c < D; ++c) lam[c] += sb[c];
            --isave;
        }
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act = live && s < nst;
        const int sr = act ? s : 0;   // inactive lanes shadow step 0 (finite data) with zero weight
        const R h = p.hstep[(size_t)sr * N + n];
        const R tn = p.tgrid[(size_t)sr * N + n], tn1 = p.tgrid[(size_t)(sr + 1) * N + n];
        const R eps = PR::eta * (tn1 - tn);
        for (int c = 0; c < D; ++c) u[c] = p.ustep[((size_t)sr * D + c) * N + n];
#pragma unroll
        for (int i = 0; i < 16; ++i)
            for (int c = 0; c < D; ++c) gb[i][c] = (R)0;
        for (int c = 0; c < D; ++c) ssum[c] = (R)0;
        bool inner = false;
        if (act)
            while (isave >= 1 && from_step(isave, s)) {
                const R ts = save_time(isave);
                cotangent(isave);
                if (ts >= tn1 - eps) {   // on the step end
                    for (int c = 0; c < D; ++c) lam[c] += sb[c];
                } else {
                    R bw[16];
                    vern7_dense::interp_weights<R>((ts - tn) / h, bw);
                    for (int c = 0; c < D; ++c) ssum[c] += sb[c];
#pragma unroll
                    for (int i = 0; i < 16; ++i)
                        if (Vern7Dense::weighted(i))
                            for (int c = 0; c < D; ++c) gb[i][c] = fma(bw[i], sb[c], gb[i][c]);
                    inner = true;
                }
                --isave;
            }
        const bool extra = __any_sync(0xffffffffu, inner);
        // k_0..k_8 as the forward evaluated them, then the extra stages where a save point needs them
        generic::model_rhs<Ops>(u, k[0]);
        vern7_dense::stage<Ops, 1>(u, h, k, g);
        vern7_dense::stage<Ops, 2>(u, h, k, g);
        vern7_dense::stage<Ops, 3>(u, h, k, g);
        vern7_dense::stage<Ops, 4>(u, h, k, g);
        vern7_dense::stage<Ops, 5>(u, h, k, g);
        vern7_dense::stage<Ops, 6>(u, h, k, g);
        vern7_dense::stage<Ops, 7>(u, h, k, g);
        vern7_dense::stage<Ops, 8>(u, h, k, g);
        if (extra) {
            vern7_dense::extra_stages<Ops>(u, h, k, g);
            back_stage<Ops, 15>(u, h, k, gb, lam, act, gw, lane);
            back_stage<Ops, 14>(u, h, k, gb, lam, act, gw, lane);
            back_stage<Ops, 13>(u, h, k, gb, lam, act, gw, lane);
            back_stage<Ops, 12>(u, h, k, gb, lam, act, gw, lane);
            back_stage<Ops, 11>(u, h, k, gb, lam, act, gw, lane);
            back_stage<Ops, 10>(u, h, k, gb, lam, act, gw, lane);
        }
        back_stage<Ops, 8>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 7>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 6>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 5>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 4>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 3>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 2>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 1>(u, h, k, gb, lam, act, gw, lane);
        back_stage<Ops, 0>(u, h, k, gb, lam, act, gw, lane);
        if (act)
            for (int c = 0; c < D; ++c) {
                R acc = lam[c] + ssum[c];
#pragma unroll
                for (int i = 0; i < 16; ++i)
                    if (i != 9) acc += gb[i][c];
                lam[c] = acc;
            }
    }
    if (live) {   // t0
        cotangent(0);
        for (int c = 0; c < D; ++c) lam[c] += sb[c];
    }
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

}  // namespace vern7_dense_discrete
}  // namespace b200ude
