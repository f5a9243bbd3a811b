// fkpp_vern7_discrete.cuh -- adaptive Vern7 forward and discrete adjoint (sensealg = ForwardDiffSensitivity,
// B200UDE_DISCRETE_ADJOINT) of the Fisher-KPP UPDE, written once over the real type.
//
//   du_i = NN(u_i) + D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1}),  periodic, theta = [chain | w1 w2 w3 b | D0]
//   (LotkaVolterra/scenario_3.jl:121-126: solve(prob, Vern7(), saveat = T, sensealg = ForwardDiffSensitivity(convert_tspan = false))
//   at the default tolerances abstol 1e-6, reltol 1e-3).
//
// Geometry of fkpp_adaptive.cuh: one thread per grid point, `tpc` whole trajectories per CTA, neighbours through shared memory
// (fkpp_adapt::cta_geometry / exchange), every norm summed over the trajectory in point order (fkpp_adapt::traj_sum), so all
// threads of a trajectory hold the same bits and take the same decisions.  The attempt loop of the forward and the step loop of
// the adjoint run while any thread of the CTA still has work: every thread executes the same barrier sequence.
//
// Forward: the stepping of generic::vern7_adaptive_forward_kernel (ude_generic.cuh) -- 10 stages, error from btilde,
// PIControl<R, 7> (step_control.cuh), no FSAL (k_1 kept after a rejection), save times are tstops: a step is clipped to the
// next save time and out[isave] is the step-end state.  The record is the one the discrete adjoint needs and nothing more: ustep [nacc+1][N][Nx] (point-fastest),
// hstep [max_steps][N] (the h the step used: t_{n+1} - t_n is not bitwise h_n), tgrid [max_steps+1][N], nacc [N].
//
// Adjoint: the recurrence of discrete_adjoint.cuh per accepted step n, walking backwards --
//   recompute the 9 stages that feed the update from u_n and h_n (bitwise the forward's: the same right-hand side, rhs_point),
//   kbar_i = h (b_i lambda_{n+1} + sum_{j>i} a_ji gbar_j),  gbar_i = J_u(g_i)^T kbar_i,  grad_theta += J_theta(g_i)^T kbar_i,
//   lambda_n = lambda_{n+1} + sum_i gbar_i,
// with the loss cotangent added where step n ends on a save time.  J_u^T couples neighbours, so every kbar_i takes one exchange.
// The CTA loops over its longest record; a trajectory past its own record shadows step 0 with a zero cotangent (h = 0), so its
// grad_u0 does not depend on its neighbours.
//
// `Ops` is the precision of the runtime-shape model layer (ude_generic.cuh; k_generic.cu: Ops32, k_f64.cu: Ops64).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "discrete_adjoint.cuh"
#include "fkpp_adaptive.cuh"
#include "vern7.cuh"

namespace b200ude {
namespace fkpp_vern7 {

template <typename R>
struct Fwd {
    const R *u0;        // [Nx][N]
    R *out;             // [n_save][Nx][N]
    R *ustep;           // [max_steps+1][N][Nx]
    R *hstep;           // [max_steps][N]
    int32_t *status;    // [N] or nullptr
    R *tgrid;           // [max_steps+1][N]
    int *nacc;          // [N]
    int N, Nx, tpc, n_save, max_steps;
    R t0, save_dt, abstol, reltol;
};

template <typename R>
struct Adj {
    const R *ustep, *hstep, *tgrid;
    const int *nacc;
    const R *cot;       // fused_l2 ? data : dL/dout, [n_save][Nx][N]
    R *grad_u0;         // [Nx][N] or nullptr
    R *partial;         // [gridDim.x * nwarps][P+1], last entry = partial loss
    int N, Nx, tpc, n_save, fused_l2;
    R t0, save_dt, margin;   // margin: a step end within `margin` (relative) of a save time is that save point
};

// the right-hand side at one grid point from its state and its two neighbours: shared by the forward and the stage recompute
template <class Ops>
__device__ __forceinline__ typename Ops::real rhs_point(typename Ops::real g, typename Ops::real gm, typename Ops::real gp, typename Ops::real w1,
                                                        typename Ops::real w2, typename Ops::real w3, typename Ops::real D0)
{
    return fma(D0, fma(w1, gm, fma(w2, g, w3 * gp)), fkpp_adapt::point_chain<Ops>(g));
}

template <class Ops>
__global__ void __launch_bounds__(256) vern7_forward_kernel(Fwd<typename Ops::real> p)
{
    using R = typename Ops::real;
    extern __shared__ __align__(16) unsigned char s_raw[];
    const int Nx = p.Nx, slots = p.tpc * Nx;
    R *sU = reinterpret_cast<R *>(s_raw);   // [slots] neighbour exchange
    R *sE = sU + slots;                     // [slots] per-point terms of the trajectory norms
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * p.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const R t0 = p.t0, t1 = p.t0 + p.save_dt * (R)(p.n_save - 1);
    const R abstol = p.abstol, reltol = p.reltol;
    const R ttol = Prec<R>::clip;   // relative slack of the clip test (as in the one-thread kernels)
    const R big = Prec<R>::huge;
    const int sx = Ops::P() - 5;
    const R w1 = Ops::theta(sx), w2 = Ops::theta(sx + 1), w3 = Ops::theta(sx + 2), D0 = Ops::theta(sx + 4);
    auto rhs = [&](R g) {
        R gm, gp;
        fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
        return rhs_point<Ops>(g, gm, gp, w1, w2, w3, D0);
    };
    auto rms = [&](R v) { return Prec<R>::sq(fkpp_adapt::traj_sum(sE, slot, base, Nx, valid, v) / (R)Nx); };
    auto store_int = [&](R *b, int row, R v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
    auto store_abi = [&](R *b, int row, R v) { if (live) b[((size_t)row * Nx + i) * N + n] = v; };

    R u = p.u0[(size_t)i * N + n];
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    if (live && i == 0) p.tgrid[n] = t0;
    R k[10];
    k[0] = rhs(u);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq, order-7 exponent, norms over the trajectory
    PIControl<R, 7> pi;
    {
        const R sk = abstol + reltol * fabs(u);
        const R d0 = rms((u / sk) * (u / sk));
        const R d1 = rms((k[0] / sk) * (k[0] / sk));
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        const R f1 = rhs(fma(dt0, k[0], u));
        const R e = (f1 - k[0]) / sk;
        const R d2 = rms(e * e) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    bool done = !live || isave >= p.n_save;   // uniform over the trajectory's threads
    bool have_k1 = true;                      // not FSAL: k_1 = f(u) is re-evaluated after an accepted step
    while (__syncthreads_or(!done)) {
        const R tend = p.t0 + p.save_dt * (R)isave;
        R h = done ? (R)0 : pi.dt;
        bool clipped = false;
        if (!done && t + h >= tend - ttol * fabs(tend)) { h = tend - t; clipped = true; }
        // CTA-uniform condition: a trajectory that still holds k_1 re-evaluates it to the same bits (u has not changed); a finished
        // one steps with h = 0 and its stages are not used
        if (__syncthreads_or(!have_k1 && !done)) k[0] = rhs(u);
#pragma unroll
        for (int st = 1; st < 10; ++st) {
            R acc = (R)0;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Vern7::a(st, j) != 0.0) acc = fma((R)Vern7::a(st, j), k[j], acc);
            k[st] = rhs(fma(h, acc, u));
        }
        R acc = (R)0, e = (R)0;
#pragma unroll
        for (int j = 0; j < 10; ++j) {
            if (Vern7::b(j) != 0.0) acc = fma((R)Vern7::b(j), k[j], acc);
            if (Vern7::bt(j) != 0.0) e = fma((R)Vern7::bt(j), k[j], e);
        }
        const R un = fma(h, acc, u);
        e *= h;
        const R sc = abstol + reltol * fmax(fabs(u), fabs(un));
        const R EEst = rms((e / sc) * (e / sc));
        if (done) continue;
        if (!(EEst <= big)) { bad = 1; done = true; continue; }   // NaN / Inf
        if (pi.judge(EEst)) {
            if (nacc >= p.max_steps) { bad = 2; done = true; continue; }
            if (live && i == 0) p.hstep[(size_t)nacc * N + n] = h;
            ++nacc;
            if (clipped) {
                store_abi(p.out, isave, un);
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = clipped ? tend : t + h;
            if (live && i == 0) p.tgrid[(size_t)nacc * N + n] = t;
            store_int(p.ustep, nacc, un);
            u = un;
            have_k1 = false;
            if (isave >= p.n_save) done = true;
        } else {
            pi.reject(h);
            have_k1 = true;
        }
    }
    if (bad && live) {   // failed solve (non-finite error estimate / max_steps): the unreached save points are NaN
        const R nan = Prec<R>::nan();
        for (int is = isave; is < p.n_save; ++is) store_abi(p.out, is, nan);
    }
    if (live && i == 0) p.nacc[n] = nacc;
    if (p.status) {   // a trajectory is flagged when any of its points is non-finite
        const R nonfinite = fkpp_adapt::traj_sum(sE, slot, base, Nx, valid, fabs(u) <= big ? (R)0 : (R)1);
        if (live && i == 0) p.status[n] = bad == 2 ? 2 : ((bad || nonfinite > (R)0) ? 1 : 0);
    }
}

template <class Ops>
__global__ void __launch_bounds__(256) discrete_adjoint_kernel(Adj<typename Ops::real> p)
{
    using R = typename Ops::real;
    using Tab = discrete::Vern7Scheme;
    constexpr int S = Tab::S;
    extern __shared__ __align__(16) unsigned char s_raw[];
    __shared__ int s_nmax;
    const int Nx = p.Nx, slots = p.tpc * Nx, P = Ops::P();
    R *sU = reinterpret_cast<R *>(s_raw);       // [slots] neighbour exchange
    R *s_g = sU + ((slots + 3) / 4) * 4;        // [nwarps][P+1]
    const int slot = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    R *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = (R)0;
    __syncwarp();
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * p.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const int sx = P - 5;
    const R w1 = Ops::theta(sx), w2 = Ops::theta(sx + 1), w3 = Ops::theta(sx + 2), D0 = Ops::theta(sx + 4);
    const int nacc = live ? p.nacc[n] : 0;
    // steps of the CTA's longest trajectory (max: order-independent)
    if (threadIdx.x == 0) s_nmax = 0;
    __syncthreads();
    if (live && i == 0) atomicMax(&s_nmax, nacc);
    __syncthreads();
    const int nmax = s_nmax;
    R lam = (R)0, loss = (R)0;
    // loss cotangent of save point `is`, whose state is the step-end state in ustep row `row` (row < 0: a save point the solve
    // never reached -- its saved state is NaN, and so are the loss and the cotangent of the fused L2)
    auto jump = [&](int is, int row) {
        const size_t idx = ((size_t)is * Nx + i) * N + n;
        if (p.fused_l2) {
            const R nan = Prec<R>::nan();
            const R us = row >= 0 ? p.ustep[((size_t)row * N + n) * Nx + i] : nan;
            const R r = us - p.cot[idx];
            loss = fma(r, r, loss);
            lam = fma((R)2, r, lam);
        } else {
            lam += p.cot[idx];
        }
    };
    auto save_time = [&](int is) { return p.t0 + p.save_dt * (R)is; };
    int isave = p.n_save - 1;
    if (live) {   // save points past the last accepted step (failed solve: non-finite state or max_steps)
        const R tend = p.tgrid[(size_t)nacc * N + n];
        while (isave > 0 && tend < save_time(isave) - p.margin * fabs(save_time(isave))) { jump(isave, -1); --isave; }
    }
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act = live && s < nacc;
        const int sr = act ? s : 0;   // past its record: shadow step 0 (finite data) with h = 0 and a zero cotangent
        if (act) {
            // a step clipped to save time ts ends at ts; every other step ends more than twice the margin before the next save time
            const R te = p.tgrid[(size_t)(sr + 1) * N + n], ts = save_time(isave);
            if (isave > 0 && fabs(te - ts) <= p.margin * fabs(ts)) { jump(isave, s + 1); --isave; }
        }
        const R h = act ? p.hstep[(size_t)sr * N + n] : (R)0;
        const R u_n = p.ustep[((size_t)sr * N + n) * Nx + i];
        // stages, as the forward evaluates them; each stage state with its two neighbours
        R gs[S], gsm[S], gsp[S], k[S];
#pragma unroll
        for (int st = 0; st < S; ++st) {
            R acc = (R)0;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Tab::a(st, j) != 0.0) acc = fma((R)Tab::a(st, j), k[j], acc);
            gs[st] = st == 0 ? u_n : fma(h, acc, u_n);
            fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, gs[st], gsm[st], gsp[st]);
            k[st] = rhs_point<Ops>(gs[st], gsm[st], gsp[st], w1, w2, w3, D0);
        }
        // reverse recurrence through the stages
        const R lv = act ? (R)1 : (R)0;   // h is inside kbar: the VJP weight only switches the shadow steps off
        R gb[S];
#pragma unroll
        for (int st = S - 1; st >= 0; --st) {
            R acc = Tab::b(st) != 0.0 ? (R)Tab::b(st) * lam : (R)0;
#pragma unroll
            for (int j = st + 1; j < S; ++j)
                if (Tab::a(j, st) != 0.0) acc = fma((R)Tab::a(j, st), gb[j], acc);
            const R kb = act ? h * acc : (R)0;
            R kbm, kbp;
            fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, kb, kbm, kbp);
            const R dx = fkpp_adapt::point_chain_vjp<Ops>(gs[st], kb, lv, gw, lane);
            gb[st] = dx + D0 * fma(w2, kb, fma(w1, kbp, w3 * kbm));   // (J^T kb)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
            const R xm = gsm[st], x = gs[st], xp = gsp[st];
            generic::warp_acc(gw, sx + 0, D0 * xm * kb, lane);
            generic::warp_acc(gw, sx + 1, D0 * x * kb, lane);
            generic::warp_acc(gw, sx + 2, D0 * xp * kb, lane);
            generic::warp_acc(gw, sx + 4, fma(w1, xm, fma(w2, x, w3 * xp)) * kb, lane);
        }
        if (act) {
            R acc = lam;
#pragma unroll
            for (int st = 0; st < S; ++st) acc += gb[st];
            lam = acc;
        }
    }
    if (live) jump(0, 0);
    if (p.grad_u0 && live) p.grad_u0[(size_t)i * N + n] = lam;
    loss = live ? loss : (R)0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);   // fixed tree
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace fkpp_vern7
}  // namespace b200ude
