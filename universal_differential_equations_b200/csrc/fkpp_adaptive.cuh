// fkpp_adaptive.cuh -- adaptive Tsit5 forward and replay adjoint of the Fisher-KPP UPDE, written once over the real type.
//
//   du_i = NN(u_i) + D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1}),  periodic, theta = [chain | w1 w2 w3 b | D0]
//   (FisherKPP/Fisher-KPP-CNN.jl:111-126, :136 -- concrete_solve(prob_nn, Tsit5(), ...) with no dt: adaptive, default tolerances).
//
// Geometry of the fixed-step Fisher-KPP kernels (k_generic.cu): one thread per grid point, `tpc` whole trajectories per CTA,
// neighbours through shared memory; the step record (ustep, dense) is point-fastest [row][trajectory][point], the ABI arrays
// (u0, out, cot, grad_u0) trajectory-fastest [row][point][trajectory]; tgrid [max_steps+1][N] and nacc [N] as in the other
// adaptive kernels.
//
// The controller is PIControl<R, 5> (step_control.cuh: OrdinaryDiffEq's PI controller and Hairer initial step), the last step
// clipped to t1, saveat from the free interpolant.  The error norm -- and d0 / d1 / d2
// of the initial step -- is OrdinaryDiffEq's default norm over the whole trajectory, sqrt(sum_i (e_i / sc_i)^2 / Nx).  Every thread
// of a trajectory sums the same Nx shared-memory terms in point order, so all of them hold the same bits, take the same
// accept / reject decision and keep the same (t, dt, qold, nacc, isave); the result does not depend on which slot of the CTA the
// trajectory occupies or on its neighbours.  The attempt loop of the forward and the sub-interval loop of the adjoint run while
// any thread of the CTA still has work (__syncthreads_or), so every thread executes the same barrier sequence; a trajectory that
// has finished keeps stepping with h = 0 on its frozen state and records nothing.
//
// `Ops` is the precision of the runtime-shape model layer (ude_generic.cuh): k_generic.cu: fp32 over the constant bank (Ops32);
// k_f64.cu: fp64 over the handle's theta (Ops64).
//
// CKPT (B200UDE_FLAG_CHECKPOINT, InterpolatingAdjoint(checkpointing = true)): the forward keeps u_n only at n = 0, K, 2K, ...
// (`ustep` holds those checkpoints) and the step size h_n of every accepted step (`hstep`), no `dense` record.  The adjoint takes
// the segments of K accepted steps from the last to the first: it recomputes a segment's u_n and k_1..k_7 from its checkpoint and
// the recorded h_n into a per-trajectory scratch area, with the stage code of the forward (tsit5_stages), and replays the segment
// from there exactly as the full-record adjoint replays it from `ustep` / `dense`.  The recomputed record is bitwise the forward's,
// so the gradients are bitwise those of the full record.  K = max(1, round(sqrt(max_steps / 7))) (b200ude_create) makes the
// checkpoint rows (max_steps / K + 1) plus the scratch rows (7K + 2) smallest.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "tsit5.cuh"
#include "ude_generic.cuh"

namespace b200ude {
namespace fkpp_adapt {

// CTA shape of every Fisher-KPP kernel, fixed step (k_generic.cu) and adaptive (adj_rows_fkpp sizes the partial rows of all):
// tpc whole trajectories in about 128 threads, a warp multiple
static inline void cta_geometry(int Nx, int *tpc, int *threads)
{
    *tpc = Nx >= 128 ? 1 : 128 / Nx;
    *threads = ((*tpc * Nx + 31) / 32) * 32;
}
// dynamic shared memory of the forward / adjoint kernels, in bytes (real_bytes = sizeof(real))
static inline size_t fwd_smem(int Nx, int real_bytes)
{
    int tpc, th;
    cta_geometry(Nx, &tpc, &th);
    return (size_t)real_bytes * 2 * (size_t)tpc * Nx;
}
static inline size_t adj_smem(int Nx, int P, int real_bytes)
{
    int tpc, th;
    cta_geometry(Nx, &tpc, &th);
    return (size_t)real_bytes * ((((size_t)tpc * Nx + 3) / 4) * 4 + (size_t)(th / 32) * (P + 1));
}

template <typename R>
struct Fwd {
    const R *u0;        // [Nx][N]
    R *out;             // [n_save][Nx][N]
    R *ustep;           // [max_steps+1][N][Nx]
    R *dense;           // [max_steps*6+1][N][Nx]
    int32_t *status;    // [N] or nullptr
    R *tgrid;           // [max_steps+1][N]
    int *nacc;          // [N]
    int N, Nx, tpc, n_save, max_steps;
    R t0, save_dt, abstol, reltol;
    // CKPT only: ustep is then [ceil(max_steps/seg)+1][N][Nx], u_n at n = 0, seg, 2 seg, ...; dense is not written
    R *hstep;           // [max_steps][N] h_n of every accepted step
    int seg;            // K, accepted steps per checkpoint
};

template <typename R>
struct Adj {
    const R *ustep, *dense, *tgrid;
    const int *nacc;
    const R *cot;       // dL/dout [n_save][Nx][N]
    R *grad_u0;         // [Nx][N] or nullptr
    R *partial;         // [gridDim.x * nwarps][P+1]
    int N, Nx, tpc, n_save;
    R t0, save_dt;
    // CKPT only: ustep holds the forward's checkpoints, dense is not read
    const R *hstep;     // [max_steps][N]
    R *scratch;         // [6 seg + 1][N][Nx] stage derivatives, then [seg + 1][N][Nx] u_n, of the segment being replayed
    int seg;
};

// the chain at one grid point (one input, one output), and its VJP: returns dx, this warp's gradient vector += w (dchain/dtheta)^T dy
template <class Ops>
__device__ __forceinline__ typename Ops::real point_chain(typename Ops::real x)
{
    typename Ops::real y;
    generic::chain_fwd<Ops, false>(&x, &y, nullptr, nullptr);
    return y;
}
template <class Ops>
__device__ __forceinline__ typename Ops::real point_chain_vjp(typename Ops::real x, typename Ops::real dy, typename Ops::real w,
                                                              typename Ops::real *gw, int lane)
{
    typename Ops::real dx;
    generic::chain_vjp<Ops>(&x, &dy, w, &dx, gw, lane);
    return dx;
}

template <typename R>
__device__ __forceinline__ void exchange(R *sU, int slot, int base, int i, int Nx, bool valid, R v, R &vm, R &vp)
{
    if (valid) sU[slot] = v;
    __syncthreads();
    vm = sU[base + (i + Nx - 1) % Nx];
    vp = sU[base + (i + 1) % Nx];
    __syncthreads();
}

// the right-hand side at the trajectory's point i (two barriers: every thread of the CTA calls it)
template <class Ops>
struct PointRhs {
    using R = typename Ops::real;
    R *sU;
    int slot, base, i, Nx;
    bool valid;
    R w1, w2, w3, D0;
    __device__ __forceinline__ R operator()(R g) const
    {
        R gm, gp;
        exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
        const R y = point_chain<Ops>(g);
        return fma(D0, fma(w1, gm, fma(w2, g, w3 * gp)), y);
    }
};

// stages 2..7 of one Tsit5 step of size h from u, k[0] = f(u): fills k[1..6] and returns the step's end state (the 7th stage's
// argument).  The forward's attempts and the checkpointed adjoint's recomputation of the accepted steps both run this code, so the
// recomputed stages are bitwise the forward's.
template <class Ops>
__device__ __forceinline__ typename Ops::real tsit5_stages(const PointRhs<Ops> &rhs, typename Ops::real u, typename Ops::real h,
                                                           typename Ops::real (&k)[7])
{
    using R = typename Ops::real;
    R un = u;
#pragma unroll
    for (int st = 1; st < 7; ++st) {
        R acc = (R)0;
#pragma unroll
        for (int j = 0; j < st; ++j)
            if (Tsit5::a(st, j) != 0.0) acc = fma((R)Tsit5::a(st, j), k[j], acc);
        const R g = fma(h, acc, u);
        if (st == 6) un = g;
        k[st] = rhs(g);
    }
    return un;
}

// sum of v over the trajectory's Nx points, in point order; every thread of the trajectory returns the same value
template <typename R>
__device__ __forceinline__ R traj_sum(R *sE, int slot, int base, int Nx, bool valid, R v)
{
    if (valid) sE[slot] = v;
    __syncthreads();
    R acc = (R)0;
    for (int q = 0; q < Nx; ++q) acc += sE[base + q];
    __syncthreads();
    return acc;
}

template <class Ops, bool CKPT>
__global__ void __launch_bounds__(256) forward_kernel(Fwd<typename Ops::real> p)
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
    const R ttol = Prec<R>::clip;   // relative slack of the clip / save-time tests (as in the one-thread kernels)
    const R big = Prec<R>::huge;
    const int sx = Ops::P() - 5;
    const R w1 = Ops::theta(sx), w2 = Ops::theta(sx + 1), w3 = Ops::theta(sx + 2), D0 = Ops::theta(sx + 4);
    const PointRhs<Ops> rhs{sU, slot, base, i, Nx, valid, w1, w2, w3, D0};
    auto rms = [&](R v) { return Prec<R>::sq(traj_sum(sE, slot, base, Nx, valid, v) / (R)Nx); };
    auto store_int = [&](R *b, int row, R v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
    auto store_abi = [&](R *b, int row, R v) { if (live) b[((size_t)row * Nx + i) * N + n] = v; };

    R u = p.u0[(size_t)i * N + n];
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    if (live && i == 0) p.tgrid[n] = t0;
    R k[7];
    k[0] = rhs(u);
    if (!CKPT) store_int(p.dense, 0, k[0]);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq, norms over the trajectory
    PIControl<R, 5> pi;
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
    while (__syncthreads_or(!done)) {
        R h = done ? (R)0 : pi.dt;
        bool clipped = false;
        if (!done && t + h >= t1 - ttol * fabs(t1)) { h = t1 - t; clipped = true; }
        const R un = tsit5_stages(rhs, u, h, k);
        R e = (R)0;
#pragma unroll
        for (int j = 0; j < 7; ++j) e = fma((R)Tsit5::bt(j), k[j], e);
        e *= h;
        const R sc = abstol + reltol * fmax(fabs(u), fabs(un));
        const R EEst = rms((e / sc) * (e / sc));
        if (done) continue;
        if (!(EEst <= big)) { bad = 1; done = true; continue; }   // NaN / Inf
        if (pi.judge(EEst)) {
            if (nacc >= p.max_steps) { bad = 2; done = true; continue; }
            const R tn = clipped ? t1 : t + h;
            // dense record of this step: k_1..k_6 at rows nacc*6 + st, k_7 at (nacc+1)*6 (= k_1 of the next step); checkpointed:
            // the step size, from which the adjoint recomputes them (t_{n+1} - t_n is not h_n bitwise)
            if (CKPT) {
                if (live && i == 0) p.hstep[(size_t)nacc * N + n] = h;
            } else {
                for (int st = 1; st < 7; ++st) store_int(p.dense, nacc * 6 + st, k[st]);
            }
            while (isave < p.n_save) {
                const R ts = t0 + p.save_dt * (R)isave;
                if (ts > tn + ttol * fabs(tn)) break;
                R bw[7];
                Tsit5::weights(fmin((ts - t) / h, (R)1), bw);
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < 7; ++j) acc = fma(bw[j], k[j], acc);
                store_abi(p.out, isave, fma(h, acc, u));
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = tn;
            ++nacc;
            if (live && i == 0) p.tgrid[(size_t)nacc * N + n] = t;
            u = un;
            k[0] = k[6];
            if (!CKPT) store_int(p.ustep, nacc, u);
            else if (nacc % p.seg == 0) store_int(p.ustep, nacc / p.seg, u);
            if (isave >= p.n_save) done = true;
        } else {
            pi.reject(h);
        }
    }
    if (bad && live) {   // failed solve (non-finite error estimate / max_steps): the unreached save points are NaN
        const R nan = Prec<R>::nan();
        for (int is = isave; is < p.n_save; ++is) store_abi(p.out, is, nan);
    }
    if (live && i == 0) p.nacc[n] = nacc;
    if (p.status) {   // a trajectory is flagged when any of its points is non-finite
        const R nonfinite = traj_sum(sE, slot, base, Nx, valid, fabs(u) <= big ? (R)0 : (R)1);
        if (live && i == 0) p.status[n] = bad == 2 ? 2 : ((bad || nonfinite > (R)0) ? 1 : 0);
    }
}

template <class Ops, bool CKPT>
__global__ void __launch_bounds__(256) adjoint_kernel(Adj<typename Ops::real> p)
{
    using R = typename Ops::real;
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
    const R eps_rel = Prec<R>::eta;   // sub-interval end tests, relative to the step (as in the one-thread kernels)
    const int sx = P - 5;
    const R w1 = Ops::theta(sx), w2 = Ops::theta(sx + 1), w3 = Ops::theta(sx + 2), D0 = Ops::theta(sx + 4);
    const int nacc = live ? p.nacc[n] : 0;
    // steps of the CTA's longest trajectory (max: order-independent)
    if (threadIdx.x == 0) s_nmax = 0;
    __syncthreads();
    if (live && i == 0) atomicMax(&s_nmax, nacc);
    __syncthreads();
    const int nmax = s_nmax;
    auto cot = [&](int is) { return p.cot[((size_t)is * Nx + i) * N + n]; };
    R lam = (R)0, kl[6];
    int isave = p.n_save - 1;
    if (live) lam += cot(isave);
    --isave;
    // the replay of accepted step s, whose u_n and k_1..k_7 are rows r and 6r..6r+6 of ust / den
    auto replay = [&](int s, const R *ust, const R *den, int r) {
        // trajectories past their own record shadow step 0 (their initial state, row 0 of the record) with weight 0
        const bool act_s = live && s < nacc;
        const int sc_ = act_s ? s : 0, rc = act_s ? r : 0;
        const R tn = act_s ? p.tgrid[(size_t)sc_ * N + n] : (R)0;
        const R tn1 = act_s ? p.tgrid[(size_t)(sc_ + 1) * N + n] : (R)0;
        const R hn = tn1 - tn, eps = eps_rel * hn;
        const R u_n = (act_s ? ust : p.ustep)[((size_t)rc * N + n) * Nx + i];
        R cur = tn1;
        while (true) {
            const bool has = act_s && cur > tn + eps;   // uniform over the trajectory
            if (!__syncthreads_or(has)) break;
            R ta = tn;
            const R ts = p.t0 + p.save_dt * (R)isave;
            if (has && isave >= 0 && ts > tn + eps) ta = ts;
            const R h = has ? cur - ta : (R)0;
#pragma unroll
            for (int st = 0; st < 6; ++st) {
                R x = u_n;
                if (act_s) {
                    R bw[7];
                    Tsit5::weights(fmin(fmax((cur - (R)Tsit5::c(st) * h - tn) / hn, (R)0), (R)1), bw);
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], den[((size_t)(rc * 6 + j) * N + n) * Nx + i], acc);
                    x = fma(hn, acc, u_n);
                }
                R a2 = (R)0;
#pragma unroll
                for (int j = 0; j < st; ++j)
                    if (Tsit5::a(st, j) != 0.0) a2 = fma((R)Tsit5::a(st, j), kl[j], a2);
                const R g = fma(h, a2, lam);
                const R w = has ? h * (R)Tsit5::b(st) : (R)0;
                // neighbours of u (for the stencil-weight gradients) and of the stage cotangent (for the transposed stencil)
                R xm, xp, gm, gp;
                exchange(sU, slot, base, i, Nx, valid, x, xm, xp);
                exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
                const R dx = point_chain_vjp<Ops>(x, g, w, gw, lane);
                kl[st] = dx + D0 * fma(w2, g, fma(w1, gp, w3 * gm));   // (J^T g)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
                generic::warp_acc(gw, sx + 0, w * D0 * xm * g, lane);
                generic::warp_acc(gw, sx + 1, w * D0 * x * g, lane);
                generic::warp_acc(gw, sx + 2, w * D0 * xp * g, lane);
                generic::warp_acc(gw, sx + 4, w * fma(w1, xm, fma(w2, x, w3 * xp)) * g, lane);
            }
            if (has) {
                R acc = (R)0;
#pragma unroll
                for (int j = 0; j < 6; ++j) acc = fma((R)Tsit5::b(j), kl[j], acc);
                lam = fma(h, acc, lam);
                cur = ta;
                if (isave >= 0 && fabs(ts - ta) <= eps) { lam += cot(isave); --isave; }
            }
        }
    };
    if constexpr (!CKPT) {
        for (int s = nmax - 1; s >= 0; --s) replay(s, p.ustep, p.dense, s);
    } else {
        // segments [s0, s0 + len) of K accepted steps, last first; len is CTA-uniform (nmax), so is every barrier of the recomputation
        const int K = p.seg;
        const PointRhs<Ops> rhs{sU, slot, base, i, Nx, valid, w1, w2, w3, D0};
        R *sk = p.scratch, *su = p.scratch + (size_t)(6 * K + 1) * N * Nx;
        auto store = [&](R *b, int row, R v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
        for (int s0 = nmax > 0 ? (nmax - 1) / K * K : -1; s0 >= 0; s0 -= K) {
            const int len = min(K, nmax - s0);
            // 1. the segment's u_n and stages from its checkpoint and the recorded h_n; a trajectory past its own record steps
            // with h = 0 and stores nothing
            const bool act0 = live && s0 < nacc;
            R u = p.ustep[((size_t)(act0 ? s0 / K : 0) * N + n) * Nx + i];
            R k[7];
            k[0] = rhs(u);   // = the forward's k_7 of step s0 - 1 (FSAL)
            if (act0) { store(su, 0, u); store(sk, 0, k[0]); }
            for (int j = 0; j < len; ++j) {
                const bool act = live && s0 + j < nacc;
                const R h = act ? p.hstep[(size_t)(s0 + j) * N + n] : (R)0;
                const R un = tsit5_stages(rhs, u, h, k);
                if (act) {
                    for (int st = 1; st < 7; ++st) store(sk, j * 6 + st, k[st]);
                    store(su, j + 1, un);
                }
                u = un;
                k[0] = k[6];
            }
            // 2. its replay, read from the scratch area (each thread reads back only what it wrote)
            for (int s = s0 + len - 1; s >= s0; --s) replay(s, su, sk, s - s0);
        }
    }
    if (p.grad_u0 && live) p.grad_u0[(size_t)i * N + n] = lam;
    if (lane == 0) gw[P] = (R)0;   // the adaptive path takes a generic cotangent; the L2 loss is formed beside it
    __syncwarp();
    R *dst = p.partial + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

}  // namespace fkpp_adapt
}  // namespace b200ude
