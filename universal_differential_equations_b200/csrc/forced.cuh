// forced.cuh -- the forced neural ODE with a readout network (B200UDE_MODEL_FORCED), written once over the real type.
//
//     du/dt = f1([u; gamma(t)]),    y = f0([u; gamma(t)]),    gamma_n(t) = sum_j A_jn cos(w_jn t + phi_jn)
//
// (NonNewtonianFluids/FENEP.jl:41-62: dudt = f1([u; gd(t)]), sigma_out = f0([u; gd(t)]) inside the loss).  Every trajectory has
// its own forcing coefficients (the script's six strain rates are one ensemble); each thread loads its coefficients into
// registers once and evaluates gamma at the time of every stage.  The loss sees the states and the readout at every save:
// `out`, `data` and the cotangent have d + r rows per save, the readout rows after the state rows.
//
// The four kernels are those of the other runtime-shape forms (ude_generic.cuh): fixed-step Tsit5 forward with the dense
// record, the interpolating adjoint on the fixed grid, the PI-controlled forward with saves from the free interpolant, and the
// replay of an adaptive solve.  They differ in three places: each stage gets its time t_n + c_i h; the saves evaluate f0; and
// the adjoint's cotangent jump at a save passes the readout rows' cotangent through f0's VJP (its u-part joins lambda, its
// theta part goes into the same per-warp gradient vector, gamma gets none).  The fused L2 recomputes the readout from the saved
// state.  The model is its own `Ops` (a compile-time variant), so the existing kernels, which dispatch on Ops::model() at run
// time, are untouched.
//
// Shapes: d + 1 <= 8 chain inputs, r <= 8 readout outputs, widths <= 64, L0 + L1 <= 5 layers in all.  theta = [f0 layers;
// f1 layers], each vec(W) column-major then b (Flux.params(f0, f1), FENEP.jl:98).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ude_generic.cuh"

namespace b200ude {
namespace forced {

using generic::MAXD;
constexpr int MAXJ = 4;   // forcing harmonics

// the per-handle shape, read from one __constant__ struct per precision (k_forced.cu)
template <typename R>
struct Shape {
    uint64_t serial;
    int D, Rr, J, L0, L1, P;
    int widths[8];   // f0: widths[0 .. L0], f1: widths[L0 + 1 .. L0 + L1 + 1]
    int acts[8];     // f0's L0 activations, then f1's L1
    int woff[8];     // offset of layer l (f0's then f1's) in theta
    const R *theta;  // the handle's device copy
    R lossw[16];     // d + r loss weights
};

template <typename R>
struct Fwd {
    const R *u0;       // [d][N]
    R *out;            // [n_save][d + r][N]
    R *ustep, *dense;  // handle record, [..][d][N]
    R *usave;          // adaptive: the handle's copy of the saved states [n_save][d][N], which the replay adjoint reads
    int32_t *status;
    const R *forcing;  // [3J][fstride]: rows A_j, w_j, phi_j
    int N, n_steps, save_every, fstride;
    R t0, dt;
};

template <typename R>
struct Adj {
    const R *ustep, *dense;
    const R *cot;      // fused_l2 ? data : dL/dout, [n_save][d + r][N]
    const R *saved;    // adaptive: the saved (interpolated) states the forward recorded, [n_save][d][N]
    const R *forcing;
    R *grad_u0, *partial;
    int N, n_steps, save_every, fused_l2, fstride;
    R t0, dt;
};

template <typename R>
struct Adapt {
    R t0, save_dt, abstol, reltol;
    int n_save, max_steps;
    R *tgrid;
    int *nacc;
};

template <typename R>
__device__ __forceinline__ R cos_r(R a);
template <>
__device__ __forceinline__ float cos_r<float>(float a) { return cosf(a); }
template <>
__device__ __forceinline__ double cos_r<double>(double a) { return cos(a); }

// gamma(t) of one trajectory: the coefficients live in registers
template <typename R>
struct Forcing {
    R A[MAXJ], W[MAXJ], F[MAXJ];
    __device__ __forceinline__ void load(const R *coef, int J, int fstride, size_t n)
    {
#pragma unroll
        for (int j = 0; j < MAXJ; ++j) {
            const bool on = j < J;
            A[j] = on ? __ldg(coef + (size_t)(3 * j) * fstride + n) : (R)0;
            W[j] = on ? __ldg(coef + (size_t)(3 * j + 1) * fstride + n) : (R)0;
            F[j] = on ? __ldg(coef + (size_t)(3 * j + 2) * fstride + n) : (R)0;
        }
    }
    __device__ __forceinline__ R operator()(R t, int J) const
    {
        R g = (R)0;
#pragma unroll
        for (int j = 0; j < MAXJ; ++j)
            if (j < J) g = fma(A[j], cos_r<R>(fma(W[j], t, F[j])), g);
        return g;
    }
};

// one of the two chains as the `Ops` that generic::chain_fwd / chain_vjp read: C = 0 the readout f0, C = 1 the dynamics f1
template <class B, int C>
struct Chain {
    using real = typename B::real;
    static __device__ __forceinline__ int base() { return C == 0 ? 0 : B::s().L0; }
    static __device__ __forceinline__ int n_layers() { return C == 0 ? B::s().L0 : B::s().L1; }
    static __device__ __forceinline__ int width(int l) { return B::s().widths[C == 0 ? l : B::s().L0 + 1 + l]; }
    static __device__ __forceinline__ int woff(int l) { return B::s().woff[base() + l]; }
    static __device__ __forceinline__ int layer_act(int l) { return B::s().acts[base() + l]; }
    static __device__ __forceinline__ const real &theta(int i) { return B::s().theta[i]; }
    static __device__ __forceinline__ real act(int k, real a) { return B::act(k, a); }
};

template <class B>
__device__ __forceinline__ void inputs(const typename B::real *u, typename B::real gam, typename B::real *x)
{
    using R = typename B::real;
#pragma unroll
    for (int c = 0; c < MAXD; ++c) x[c] = c < B::s().D ? u[c] : (c == B::s().D ? gam : (R)0);
}

// du = f1([u; gamma])
template <class B>
__device__ __forceinline__ void rhs(const typename B::real *u, typename B::real gam, typename B::real *du)
{
    using R = typename B::real;
    R x[MAXD], y[MAXD];
    inputs<B>(u, gam, x);
    generic::chain_fwd<Chain<B, 1>, false>(x, y, nullptr, nullptr);
    for (int k = 0; k < B::s().D; ++k) du[k] = y[k];
}

// y = f0([u; gamma])
template <class B>
__device__ __forceinline__ void readout(const typename B::real *u, typename B::real gam, typename B::real *y)
{
    using R = typename B::real;
    R x[MAXD];
    inputs<B>(u, gam, x);
    generic::chain_fwd<Chain<B, 0>, false>(x, y, nullptr, nullptr);
}

// kl = (df1/du)^T g; gradient vector += w (df1/dtheta)^T g   (all lanes of the warp participate)
template <class B>
__device__ __forceinline__ void rhs_vjp(const typename B::real *u, typename B::real gam, const typename B::real *g, typename B::real w,
                                        typename B::real *kl, typename B::real *gw, int lane)
{
    using R = typename B::real;
    R x[MAXD], dy[MAXD], dx[MAXD];
    inputs<B>(u, gam, x);
#pragma unroll
    for (int c = 0; c < MAXD; ++c) dy[c] = c < B::s().D ? g[c] : (R)0;
    generic::chain_vjp<Chain<B, 1>>(x, dy, w, dx, gw, lane);
    for (int k = 0; k < B::s().D; ++k) kl[k] = dx[k];
}

// lam += (df0/du)^T dy; gradient vector += w (df0/dtheta)^T dy   (all lanes of the warp participate; gamma gets no cotangent)
template <class B>
__device__ __forceinline__ void readout_vjp(const typename B::real *u, typename B::real gam, const typename B::real *dy, typename B::real w,
                                            typename B::real *lam, typename B::real *gw, int lane)
{
    using R = typename B::real;
    R x[MAXD], dx[MAXD];
    inputs<B>(u, gam, x);
    generic::chain_vjp<Chain<B, 0>>(x, dy, w, dx, gw, lane);
    for (int k = 0; k < B::s().D; ++k) lam[k] += dx[k];
}

// states and readout of one save point into out[is][0 .. d + r)
template <class B>
__device__ __forceinline__ void write_save(typename B::real *out, int is, const typename B::real *u, typename B::real gam, size_t N, size_t n)
{
    using R = typename B::real;
    const int D = B::s().D, DR = D + B::s().Rr;
    for (int c = 0; c < D; ++c) out[((size_t)is * DR + c) * N + n] = u[c];
    R y[MAXD];
    readout<B>(u, gam, y);
    for (int k = 0; k < B::s().Rr; ++k) out[((size_t)is * DR + D + k) * N + n] = y[k];
}

// the cotangent of save point `is` at the state us: lam += the state rows' cotangent + f0's VJP of the readout rows'.
// on = false (a lane with no save here): nothing is added, the lane still takes part in the warp's VJP with a zero cotangent
template <class B>
__device__ __forceinline__ void save_jump(const typename B::real *cot, int fused, int is, bool on, const typename B::real *us,
                                          typename B::real gam, typename B::real lv, typename B::real *lam, typename B::real &loss,
                                          typename B::real *gw, int lane, size_t N, size_t n)
{
    using R = typename B::real;
    const int D = B::s().D, Rr = B::s().Rr, DR = D + Rr;
    R dy[MAXD];
    if (fused) {
        R y[MAXD];
        readout<B>(us, gam, y);   // recomputed from the saved state
        for (int c = 0; c < D; ++c) {
            const R r = us[c] - __ldg(cot + ((size_t)is * DR + c) * N + n), w = B::s().lossw[c];
            if (on) { loss = fma(w * r, r, loss); lam[c] = fma((R)2 * w, r, lam[c]); }
        }
        for (int k = 0; k < Rr; ++k) {
            const R r = y[k] - __ldg(cot + ((size_t)is * DR + D + k) * N + n), w = B::s().lossw[D + k];
            if (on) loss = fma(w * r, r, loss);
            dy[k] = on ? (R)2 * w * r : (R)0;
        }
    } else {
        for (int c = 0; c < D; ++c)
            if (on) lam[c] += __ldg(cot + ((size_t)is * DR + c) * N + n);
        for (int k = 0; k < Rr; ++k) dy[k] = on ? __ldg(cot + ((size_t)is * DR + D + k) * N + n) : (R)0;
    }
    readout_vjp<B>(us, gam, dy, on ? lv : (R)0, lam, gw, lane);
}

template <class B, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) forward_kernel(Fwd<typename B::real> p)
{
    using R = typename B::real;
    using PR = Prec<R>;
    const int D = B::s().D, J = B::s().J;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    const R dt = p.dt;
    Forcing<R> f;
    f.load(p.forcing, J, p.fstride, n);
    R u[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](R *base, int row, const R *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    write_save<B>(p.out, 0, u, f(p.t0, J), N, n);
    store(p.ustep, 0, u);
    rhs<B>(u, f(p.t0, J), k[0]);
    store(p.dense, 0, k[0]);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
        const R tn = fma((R)s, dt, p.t0);
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
            rhs<B>(g, f(fma((R)Tsit5::c(i), dt, tn), J), k[i]);
            store(p.dense, s * 6 + i, k[i]);
        }
        store(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { write_save<B>(p.out, isave, u, f(fma((R)(s + 1), dt, p.t0), J), N, n); ++isave; }
        for (int c = 0; c < D; ++c) k[0][c] = k[6][c];
    }
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = ok ? 0 : 1;
    }
}

template <class B, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adjoint_kernel(Adj<typename B::real> p)
{
    using R = typename B::real;
    extern __shared__ __align__(16) unsigned char s_raw[];
    R *s_g = reinterpret_cast<R *>(s_raw);   // [BLOCK/32][P+1]
    const int D = B::s().D, J = B::s().J, P = B::s().P;
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
    Forcing<R> f;
    f.load(p.forcing, J, p.fstride, n);
    R lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    auto jump = [&](int is) {
        const int row = is * p.save_every;
        R us[MAXD];
        for (int c = 0; c < D; ++c) us[c] = __ldg(p.ustep + ((size_t)row * D + c) * N + n);
        save_jump<B>(p.cot, p.fused_l2, is, true, us, f(fma((R)row, dt, p.t0), J), lv, lam, loss, gw, lane, N, n);
    };
    const int n_save = p.n_steps / p.save_every + 1;
    jump(n_save - 1);
    for (int s = p.n_steps - 1; s >= 0; --s) {
        const R tn1 = fma((R)(s + 1), dt, p.t0);
#pragma unroll
        for (int i = 0; i < 6; ++i) {
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
            rhs_vjp<B>(x, f(fma(-(R)Tsit5::c(i), dt, tn1), J), g, dt * (R)Tsit5::b(i) * lv, kl[i], gw, lane);
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

// PI-controlled Tsit5 as generic::adaptive_forward_kernel (PIControl, saves from the free interpolant), with the
// stage times and the readout rows
template <class B, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_forward_kernel(Fwd<typename B::real> p, Adapt<typename B::real> ap)
{
    using R = typename B::real;
    using PR = Prec<R>;
    const int D = B::s().D, J = B::s().J, DR = D + B::s().Rr;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    if (gid >= p.N) return;
    const size_t n = (size_t)gid;
    Forcing<R> f;
    f.load(p.forcing, J, p.fstride, n);
    const R t0 = ap.t0, t1 = ap.t0 + ap.save_dt * (R)(ap.n_save - 1);
    const R abstol = ap.abstol, reltol = ap.reltol;
    R u[MAXD], un[MAXD], g[MAXD], k[7][MAXD];
    for (int c = 0; c < D; ++c) u[c] = __ldg(p.u0 + (size_t)c * N + n);
    auto store = [&](R *base, int row, const R *v) {
        for (int c = 0; c < D; ++c) base[((size_t)row * D + c) * N + n] = v[c];
    };
    write_save<B>(p.out, 0, u, f(t0, J), N, n);
    store(p.usave, 0, u);
    store(p.ustep, 0, u);
    ap.tgrid[n] = t0;
    rhs<B>(u, f(t0, J), k[0]);
    store(p.dense, 0, k[0]);
    PIControl<R, 5> pi;
    {   // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq (f at t0 + dt0 for the second derivative estimate)
        R d0 = 0, d1 = 0, d2 = 0;
        for (int c = 0; c < D; ++c) {
            const R sk = abstol + reltol * fabs(u[c]);
            d0 += (u[c] / sk) * (u[c] / sk);
            d1 += (k[0][c] / sk) * (k[0][c] / sk);
        }
        d0 = PR::sq(d0 / D); d1 = PR::sq(d1 / D);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        for (int c = 0; c < D; ++c) g[c] = fma(dt0, k[0][c], u[c]);
        rhs<B>(g, f(t0 + dt0, J), un);
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
            rhs<B>(g, f(fma((R)Tsit5::c(i), h, t), J), k[i]);
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
            for (int i = 1; i < 7; ++i) store(p.dense, nacc * 6 + i, k[i]);
            while (isave < ap.n_save) {
                const R ts = t0 + ap.save_dt * (R)isave;
                if (ts > tn + PR::clip * fabs(tn)) break;
                R bw[7], us[MAXD];
                Tsit5::weights(fmin((ts - t) / h, (R)1), bw);
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) acc = fma(bw[j], k[j][c], acc);
                    us[c] = fma(h, acc, u[c]);
                }
                write_save<B>(p.out, isave, us, f(ts, J), N, n);
                store(p.usave, isave, us);
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
    if (bad) {   // failed solve: the unreached save points are NaN, states and readout
        for (int is = isave; is < ap.n_save; ++is) {
            for (int c = 0; c < DR; ++c) p.out[((size_t)is * DR + c) * N + n] = PR::nan();
            for (int c = 0; c < D; ++c) p.usave[((size_t)is * D + c) * N + n] = PR::nan();
        }
    }
    ap.nacc[n] = nacc;
    if (p.status) {
        bool ok = true;
        for (int c = 0; c < D; ++c) ok = ok && (fabs(u[c]) <= PR::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// replay adjoint of an adaptive solve (generic::adaptive_adjoint_kernel with stage times and the readout jumps).  The cotangent of
// a save is taken at the saved (interpolated) state the forward recorded (p.saved, the handle's copy: the caller's `out` may be
// gone by then, e.g. in an autograd backward); with fused_l2 the loss 2 w (out - data) is formed here,
// the readout rows recomputed from that state.  A warp loops to its longest record; the save jumps are warp-uniform calls in
// which lanes without a save carry a zero cotangent
template <class B, int BLOCK>
__global__ void __launch_bounds__(BLOCK, 1) adaptive_adjoint_kernel(Adj<typename B::real> p, Adapt<typename B::real> ap)
{
    using R = typename B::real;
    using PR = Prec<R>;
    extern __shared__ __align__(16) unsigned char s_raw[];
    R *s_g = reinterpret_cast<R *>(s_raw);   // [BLOCK/32][P+1]
    const int D = B::s().D, J = B::s().J, P = B::s().P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    R *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = (R)0;
    __syncwarp();
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const R lv = live ? (R)1 : (R)0;
    Forcing<R> f;
    f.load(p.forcing, J, p.fstride, n);
    const int nacc = ap.nacc[n];
    int nmax = live ? nacc : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nmax = max(nmax, __shfl_xor_sync(0xffffffffu, nmax, o));
    R lam[MAXD], x[MAXD], g[MAXD], kl[6][MAXD], un_[MAXD];
    R loss = (R)0;
    for (int c = 0; c < D; ++c) lam[c] = (R)0;
    auto jump = [&](int is, bool on) {
        const int isc = is < 0 ? 0 : is;
        R us[MAXD];
        for (int c = 0; c < D; ++c) us[c] = __ldg(p.saved + ((size_t)isc * D + c) * N + n);
        save_jump<B>(p.cot, p.fused_l2, isc, on, us, f(ap.t0 + ap.save_dt * (R)isc, J), lv, lam, loss, gw, lane, N, n);
    };
    int isave = ap.n_save - 1;
    jump(isave, live);
    --isave;
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act_s = live && s < nacc;
        const int sc_ = act_s ? s : 0;
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
                rhs_vjp<B>(x, f(cur - (R)Tsit5::c(i) * h, J), g, has ? h * (R)Tsit5::b(i) : (R)0, kl[i], gw, lane);
            }
            bool on = false;
            if (has) {
                for (int c = 0; c < D; ++c) {
                    R acc = (R)0;
#pragma unroll
                    for (int j = 0; j < 6; ++j) acc = fma((R)Tsit5::b(j), kl[j][c], acc);
                    lam[c] = fma(h, acc, lam[c]);
                }
                cur = ta;
                on = isave >= 0 && fabs(ts - ta) <= eps;
            }
            if (__any_sync(0xffffffffu, on)) jump(isave, on);
            if (on) --isave;
        }
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

}  // namespace forced
}  // namespace b200ude
