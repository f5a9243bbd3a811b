// operator.cuh -- wide-state operator UDEs (B200UDE_MODEL_OPERATOR), written once over the real type:
//
//     du/dt = D1 · NN(u) + D2 · u,     NN: d -> ... -> m,  D1 (d x m), D2 (d x d) fixed, column-major
//
// (Climate/NeuralPDE/npde.jl:75-78: dudt_(u, p, t) = ops.D1 * re(p)(u) + ops.D2 * u, a method-of-lines PDE with a learned
// closure).  d and every width go up to 64, so one thread per trajectory would hold u and the Tsit5 stages on its stack and
// run ~2 d^2 dependent FMAs per right-hand side.  Here a WARP integrates one trajectory:
//
//   - lane l holds state component l and l + 32 (the second slot only when d > 32); each layer's units follow the same rule.
//     Runge-Kutta state, stages and lambda are a few registers per lane.
//   - a matrix-vector product D·v: a lane computes its own output rows, the inputs v_k come from their owner lanes by
//     __shfl_sync in a fixed order of k.  D^T·g: a lane computes its own columns, g_i by shuffle in a fixed order of i.
//   - D1, D2 (the handle's padded copy, one 16-byte-multiple block, with the loss weights in front) are staged once per CTA by
//     one elected thread with cp.async.bulk completing on an mbarrier.  theta, which ADAM updates in place every iteration, is
//     staged by the CTA into the same padded layout.  Every leading dimension in shared memory is odd, so that the lanes'
//     column reads (D·v) and row reads (D^T·g) are both free of bank conflicts.  Nothing goes through the constant bank:
//     handles of this model run concurrently on one device.
//   - the parameter gradient: one P-vector per warp in shared memory; dW_ik belongs to the lane that owns unit i, each bias to
//     its owner lane, so there are no atomics and the summation order is fixed.  The CTA then sums its warps in a fixed order
//     into its partial row (launch_reduce / launch_reduce_f64 do the rest).
//   - adaptive stepping: the error norm is a shuffle-xor butterfly, so every lane holds the same bits and the accept / reject
//     decision is warp-uniform.  No CTA barrier sits inside any stepping loop: each warp runs its own step count, and each
//     trajectory's results are bitwise those of the trajectory solved alone.
//
// Handle records are component-fastest within a trajectory, [row][N][d]; the ABI arrays stay [..][d][N].
//   Tsit5: dense (6 steps + 1) d N (row s*6 + j = k_j of step s; k_0 of step s = k_6 of step s-1), ustep (steps + 1) d N.
//   RKC2:  ustep (steps + 1) d N and, in `dense`, f(u_n) (steps + 1) d N; adaptive RKC2 also the stage count of each
//          accepted step, sstep [max_steps][N].
// theta = per layer vec(W) column-major then b (Flux.destructure).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "ude_generic.cuh"

namespace b200ude {
namespace op {

constexpr int MAXL = 5;
constexpr int LW = 64;          // loss-weight slots at the front of the staged operator block
constexpr int RKC_MAX = 64;     // RKC2 stages
constexpr unsigned FULL = 0xffffffffu;
// RKC2 table layout (the handle's device copy, in the handle's dtype): mt1, then c, w, mu, nu, mt, ga with RKC_MAX + 1 entries each
constexpr int RKC_C = 1, RKC_W = RKC_C + RKC_MAX + 1, RKC_MU = RKC_W + RKC_MAX + 1, RKC_NU = RKC_MU + RKC_MAX + 1,
              RKC_MT = RKC_NU + RKC_MAX + 1, RKC_GA = RKC_MT + RKC_MAX + 1, RKC_LEN = RKC_GA + RKC_MAX + 1;

template <typename R>
struct Run {
    int D, M, L, P, has_d2;
    int widths[MAXL + 1], acts[MAXL];
    int woff[MAXL];   // layer l's vec(W) in theta (and in the gradient vector); b follows at woff + a b
    int soff[MAXL];   // layer l's W in the staged theta, leading dimension ldw[l] (odd); b follows at soff + a ldw
    int ldw[MAXL];
    int ld1, ld2;     // odd leading dimensions of the staged D1 / D2
    int ops_elems, theta_elems, gstride;   // staged block sizes (elements); gstride: one warp's gradient vector (>= P + 1)
    const R *ops;     // [LW loss weights | D1 (ld1 x M) | D2 (ld2 x D)], ops_elems elements
    const R *theta;   // the handle's theta [P]
    const R *rkc;     // RKC2 tables (RKC_LEN; adaptive RKC2: (S - 1) RKC_LEN, the block of s stages at (s - 2) RKC_LEN)
    int S;            // RKC2 stages
    const R *u0;      // [d][N]
    R *out;           // [n_save][d][N]
    R *ustep, *dense, *usave;   // records [row][N][d]
    int32_t *status;
    const R *cot;     // fused_l2 ? data : dL/dout, [n_save][d][N]
    R *grad_u0, *partial;
    int fused_l2;
    R *tgrid;         // adaptive: accepted step times [max_steps + 1][N]
    int *nacc;
    int N, n_steps, save_every, n_save, max_steps;
    R t0, dt, save_dt, abstol, reltol;
    // adaptive RKC2 (appended, so that the fields above keep their parameter offsets): `rkc` then holds one RKC_LEN block per
    // stage count 2..S, beta[s] is the real stability interval of s stages, sstep [max_steps][N] the stage count of each
    // accepted step, rho the caller's bound of the spectral radius of df/du (eigen_est)
    const R *beta;
    int *sstep;
    R rho;
};

template <typename R>
struct V {
    R a, b;   // components lane, lane + 32
};

template <typename R>
__device__ __forceinline__ R act(int k, R z);
template <>
__device__ __forceinline__ float act<float>(int k, float z) { return k == ACT_TANH ? tanhf(z) : (k == ACT_RBF ? expf(-z * z) : z); }
template <>
__device__ __forceinline__ double act<double>(int k, double z) { return k == ACT_TANH ? tanh(z) : (k == ACT_RBF ? exp(-z * z) : z); }

// v[c * stride] for the lane's components c < D (zero elsewhere)
template <typename R>
__device__ __forceinline__ V<R> ldv(const R *p, size_t stride, int D, int lane)
{
    return {lane < D ? p[(size_t)lane * stride] : (R)0, lane + 32 < D ? p[(size_t)(lane + 32) * stride] : (R)0};
}
template <typename R>
__device__ __forceinline__ void stv(R *p, size_t stride, V<R> v, int D, int lane)
{
    if (lane < D) p[(size_t)lane * stride] = v.a;
    if (lane + 32 < D) p[(size_t)(lane + 32) * stride] = v.b;
}

template <typename R>
__device__ __forceinline__ R wsum(R v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}

// y_i = sum_{k < cols} A[i + k ld] x_k for the lane's rows i < rows, zero elsewhere
template <typename R>
__device__ __forceinline__ V<R> matvec(const R *A, int ld, int rows, int cols, V<R> x, int lane)
{
    const int r0 = lane < rows ? lane : 0, r1 = lane + 32 < rows ? lane + 32 : 0;
    R y0 = (R)0, y1 = (R)0;
    if (rows > 32) {
        for (int k = 0; k < cols; ++k) {
            const R xk = __shfl_sync(FULL, k < 32 ? x.a : x.b, k & 31);
            y0 = fma(A[k * ld + r0], xk, y0);
            y1 = fma(A[k * ld + r1], xk, y1);
        }
    } else {
        for (int k = 0; k < cols; ++k) y0 = fma(A[k * ld + r0], __shfl_sync(FULL, k < 32 ? x.a : x.b, k & 31), y0);
    }
    return {lane < rows ? y0 : (R)0, lane + 32 < rows ? y1 : (R)0};
}

// y_k = sum_{i < rows} A[i + k ld] g_i for the lane's columns k < cols, zero elsewhere
template <typename R>
__device__ __forceinline__ V<R> matvec_t(const R *A, int ld, int rows, int cols, V<R> g, int lane)
{
    const int k0 = lane < cols ? lane : 0, k1 = lane + 32 < cols ? lane + 32 : 0;
    R y0 = (R)0, y1 = (R)0;
    if (cols > 32) {
        for (int i = 0; i < rows; ++i) {
            const R gi = __shfl_sync(FULL, i < 32 ? g.a : g.b, i & 31);
            y0 = fma(A[k0 * ld + i], gi, y0);
            y1 = fma(A[k1 * ld + i], gi, y1);
        }
    } else {
        for (int i = 0; i < rows; ++i) y0 = fma(A[k0 * ld + i], __shfl_sync(FULL, i < 32 ? g.a : g.b, i & 31), y0);
    }
    return {lane < cols ? y0 : (R)0, lane + 32 < cols ? y1 : (R)0};
}

// the chain NN(x); with KEEP, xs[l] = input of layer l (xs[L] = output) and zs[l] = its pre-activation
template <typename R, bool KEEP>
__device__ __forceinline__ V<R> chain(const Run<R> &p, const R *sth, V<R> x, V<R> *xs, V<R> *zs, int lane)
{
#pragma unroll
    for (int l = 0; l < MAXL; ++l) {
        if (l < p.L) {
            const int a = p.widths[l], b = p.widths[l + 1], ld = p.ldw[l];
            const R *W = sth + p.soff[l];
            if (KEEP) xs[l] = x;
            V<R> z = matvec(W, ld, b, a, x, lane);
            z.a += lane < b ? W[a * ld + lane] : (R)0;
            z.b += lane + 32 < b ? W[a * ld + lane + 32] : (R)0;
            if (KEEP) zs[l] = z;
            x.a = lane < b ? act<R>(p.acts[l], z.a) : (R)0;
            x.b = lane + 32 < b ? act<R>(p.acts[l], z.b) : (R)0;
        }
    }
    if (KEEP) {
#pragma unroll
        for (int l = 1; l <= MAXL; ++l)
            if (l == p.L) xs[l] = x;
    }
    return x;
}

// f(u) = D1 NN(u) + D2 u
template <typename R>
__device__ __forceinline__ V<R> rhs(const Run<R> &p, const R *sops, const R *sth, V<R> u, int lane)
{
    const V<R> y = chain<R, false>(p, sth, u, nullptr, nullptr, lane);
    V<R> f = matvec(sops + LW, p.ld1, p.D, p.M, y, lane);
    if (p.has_d2) {
        const V<R> e = matvec(sops + LW + p.ld1 * p.M, p.ld2, p.D, p.D, u, lane);
        f.a += e.a;
        f.b += e.b;
    }
    return f;
}

// (df/du)^T g; the warp's gradient vector gw += w (df/dtheta)^T g
template <typename R>
__device__ __forceinline__ V<R> rhs_vjp(const Run<R> &p, const R *sops, const R *sth, V<R> x, V<R> g, R w, R *gw, int lane)
{
    V<R> xs[MAXL + 1], zs[MAXL];
    chain<R, true>(p, sth, x, xs, zs, lane);
    V<R> v = matvec_t(sops + LW, p.ld1, p.D, p.M, g, lane);   // D1^T g
#pragma unroll
    for (int l = MAXL - 1; l >= 0; --l) {
        if (l < p.L) {
            const int a = p.widths[l], b = p.widths[l + 1];
            V<R> dl;
            dl.a = lane < b ? v.a * generic::actder_rt<R>(p.acts[l], zs[l].a, xs[l + 1].a) : (R)0;
            dl.b = lane + 32 < b ? v.b * generic::actder_rt<R>(p.acts[l], zs[l].b, xs[l + 1].b) : (R)0;
            R *gW = gw + p.woff[l];
            const R wa = w * dl.a, wb = w * dl.b;
            for (int k = 0; k < a; ++k) {
                const R xk = __shfl_sync(FULL, k < 32 ? xs[l].a : xs[l].b, k & 31);
                if (lane < b) gW[k * b + lane] = fma(wa, xk, gW[k * b + lane]);
                if (lane + 32 < b) gW[k * b + lane + 32] = fma(wb, xk, gW[k * b + lane + 32]);
            }
            if (lane < b) gW[a * b + lane] += wa;
            if (lane + 32 < b) gW[a * b + lane + 32] += wb;
            v = matvec_t(sth + p.soff[l], p.ldw[l], b, a, dl, lane);
        }
    }
    if (p.has_d2) {
        const V<R> e = matvec_t(sops + LW + p.ld1 * p.M, p.ld2, p.D, p.D, g, lane);
        v.a += e.a;
        v.b += e.b;
    }
    return v;
}

// Stage the operator block (bulk copy on an mbarrier) and theta (padded, by the CTA) into shared memory.  Ends with every
// thread past the mbarrier; the only CTA barrier of the kernel before its closing reduction.
template <typename R>
__device__ __forceinline__ void stage(const Run<R> &p, R *sops, R *sth)
{
    __shared__ __align__(8) uint64_t bar;
    const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(&bar), dst_a = (uint32_t)__cvta_generic_to_shared(sops);
    const uint32_t bytes = (uint32_t)(p.ops_elems * sizeof(R));
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a), "l"(p.ops),
                     "r"(bytes), "r"(bar_a)
                     : "memory");
    }
    for (int l = 0; l < p.L; ++l) {
        const int a = p.widths[l], b = p.widths[l + 1], ld = p.ldw[l];
        const R *src = p.theta + p.woff[l];
        R *dst = sth + p.soff[l];
        for (int e = threadIdx.x; e < a * b; e += blockDim.x) dst[(e / b) * ld + e % b] = __ldg(src + e);
        for (int e = threadIdx.x; e < b; e += blockDim.x) dst[a * ld + e] = __ldg(src + a * b + e);
    }
    __syncthreads();   // theta staged; the mbarrier is initialised and armed before anybody polls it
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar_a) : "memory");
}

template <typename R>
struct Smem {
    R *ops, *th, *g;
};
template <typename R>
__device__ __forceinline__ Smem<R> carve(const Run<R> &p)
{
    extern __shared__ __align__(128) unsigned char s_raw[];
    R *base = reinterpret_cast<R *>(s_raw);
    return {base, base + p.ops_elems, base + p.ops_elems + p.theta_elems};
}

// the CTA's warps' gradient vectors (and losses at index P) summed in warp order into the CTA's partial row
template <typename R>
__device__ __forceinline__ void cta_reduce(const Run<R> &p, const R *sg)
{
    __syncthreads();
    const int W = blockDim.x >> 5;
    R *dst = p.partial + (size_t)blockIdx.x * (p.P + 1);
    for (int e = threadIdx.x; e < p.P + 1; e += blockDim.x) {
        R tot = sg[e];
        for (int w = 1; w < W; ++w) tot += sg[(size_t)w * p.gstride + e];
        dst[e] = tot;
    }
}

template <typename R>
__device__ __forceinline__ bool warp_finite(V<R> u)
{
    return __all_sync(FULL, fabs(u.a) <= Prec<R>::huge && fabs(u.b) <= Prec<R>::huge);
}

// the cotangent of save `is` at state us: lam += cot, or (fused L2) loss += w r^2, lam += 2 w r with r = us - data
template <typename R>
__device__ __forceinline__ void save_jump(const Run<R> &p, const R *sops, int is, V<R> us, V<R> &lam, R &loss, size_t n, int lane)
{
    const size_t N = (size_t)p.N;
    const V<R> c = ldv(p.cot + (size_t)is * p.D * N + n, N, p.D, lane);
    if (p.fused_l2) {
        const R ra = us.a - c.a, rb = us.b - c.b;
        const R wa = lane < p.D ? sops[lane] : (R)0, wb = lane + 32 < p.D ? sops[lane + 32] : (R)0;
        loss = fma(wa * ra, ra, loss);
        loss = fma(wb * rb, rb, loss);
        lam.a = fma((R)2 * wa, ra, lam.a);
        lam.b = fma((R)2 * wb, rb, lam.b);
    } else {
        lam.a += c.a;
        lam.b += c.b;
    }
}

// ---- 1. fixed-step Tsit5 forward, with the dense record ----
template <typename R>
__global__ void __launch_bounds__(128) tsit5_forward_kernel(Run<R> p)
{
    const Smem<R> sm = carve(p);
    stage(p, sm.ops, sm.th);
    const int lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const int traj = blockIdx.x * W + (threadIdx.x >> 5);
    if (traj >= p.N) return;
    const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
    const R dt = p.dt;
    auto rec = [&](R *b, int row) { return b + ((size_t)row * N + n) * D; };
    V<R> u = ldv(p.u0 + n, N, p.D, lane), k[7];
    stv(p.out + n, N, u, p.D, lane);
    stv(rec(p.ustep, 0), 1, u, p.D, lane);
    k[0] = rhs(p, sm.ops, sm.th, u, lane);
    stv(rec(p.dense, 0), 1, k[0], p.D, lane);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            R aa = (R)0, ab = (R)0;
#pragma unroll
            for (int j = 0; j < i; ++j)
                if (Tsit5::a(i, j) != 0.0) { aa = fma((R)Tsit5::a(i, j), k[j].a, aa); ab = fma((R)Tsit5::a(i, j), k[j].b, ab); }
            const V<R> g{fma(dt, aa, u.a), fma(dt, ab, u.b)};
            if (i == 6) u = g;
            k[i] = rhs(p, sm.ops, sm.th, g, lane);
            stv(rec(p.dense, s * 6 + i), 1, k[i], p.D, lane);
        }
        stv(rec(p.ustep, s + 1), 1, u, p.D, lane);
        if ((s + 1) % p.save_every == 0) { stv(p.out + (size_t)isave * D * N + n, N, u, p.D, lane); ++isave; }
        k[0] = k[6];
    }
    const bool ok = warp_finite(u);
    if (p.status && lane == 0) p.status[n] = ok ? 0 : 1;
}

// ---- 2. interpolating adjoint on the fixed Tsit5 grid ----
template <typename R>
__global__ void __launch_bounds__(128) tsit5_adjoint_kernel(Run<R> p)
{
    const Smem<R> sm = carve(p);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    R *gw = sm.g + (size_t)warp * p.gstride;
    for (int q = lane; q < p.P + 1; q += 32) gw[q] = (R)0;
    stage(p, sm.ops, sm.th);
    const int traj = blockIdx.x * W + warp;
    if (traj < p.N) {
        const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
        const R dt = p.dt;
        auto rec = [&](const R *b, int row) { return b + ((size_t)row * N + n) * D; };
        V<R> lam{(R)0, (R)0}, kl[6];
        R loss = (R)0;
        auto jump = [&](int is) { save_jump(p, sm.ops, is, ldv(rec(p.ustep, is * p.save_every), 1, p.D, lane), lam, loss, n, lane); };
        jump(p.n_steps / p.save_every);
        for (int s = p.n_steps - 1; s >= 0; --s) {
            const V<R> us = ldv(rec(p.ustep, s), 1, p.D, lane);
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                R xa = (R)0, xb = (R)0, ga = (R)0, gb = (R)0;
#pragma unroll
                for (int j = 0; j < 7; ++j)
                    if (Tsit5::bw(i, j) != 0.0) {
                        const V<R> kj = ldv(rec(p.dense, s * 6 + j), 1, p.D, lane);
                        xa = fma((R)Tsit5::bw(i, j), kj.a, xa);
                        xb = fma((R)Tsit5::bw(i, j), kj.b, xb);
                    }
#pragma unroll
                for (int j = 0; j < i; ++j)
                    if (Tsit5::a(i, j) != 0.0) { ga = fma((R)Tsit5::a(i, j), kl[j].a, ga); gb = fma((R)Tsit5::a(i, j), kl[j].b, gb); }
                const V<R> x{fma(dt, xa, us.a), fma(dt, xb, us.b)}, g{fma(dt, ga, lam.a), fma(dt, gb, lam.b)};
                kl[i] = rhs_vjp(p, sm.ops, sm.th, x, g, dt * (R)Tsit5::b(i), gw, lane);
            }
            R aa = (R)0, ab = (R)0;
#pragma unroll
            for (int j = 0; j < 6; ++j) { aa = fma((R)Tsit5::b(j), kl[j].a, aa); ab = fma((R)Tsit5::b(j), kl[j].b, ab); }
            lam.a = fma(dt, aa, lam.a);
            lam.b = fma(dt, ab, lam.b);
            if (s % p.save_every == 0) jump(s / p.save_every);
        }
        if (p.grad_u0) stv(p.grad_u0 + n, N, lam, p.D, lane);
        loss = wsum(loss);
        if (lane == 0) gw[p.P] = loss;
    }
    cta_reduce(p, sm.g);
}

// ---- 3. adaptive Tsit5 forward: OrdinaryDiffEq's PI controller and initial step, saves from the free interpolant
// (PIControl on one warp).  The norms are butterflies, so every decision is warp-uniform ----
template <typename R>
__global__ void __launch_bounds__(128) tsit5_adaptive_forward_kernel(Run<R> p)
{
    using PR = Prec<R>;
    const Smem<R> sm = carve(p);
    stage(p, sm.ops, sm.th);
    const int lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const int traj = blockIdx.x * W + (threadIdx.x >> 5);
    if (traj >= p.N) return;
    const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
    const bool on_a = lane < p.D, on_b = lane + 32 < p.D;
    auto rec = [&](R *b, int row) { return b + ((size_t)row * N + n) * D; };
    const R t0 = p.t0, t1 = p.t0 + p.save_dt * (R)(p.n_save - 1);
    const R abstol = p.abstol, reltol = p.reltol, Dr = (R)p.D;
    V<R> u = ldv(p.u0 + n, N, p.D, lane), un, k[7];
    stv(p.out + n, N, u, p.D, lane);
    stv(rec(p.usave, 0), 1, u, p.D, lane);
    stv(rec(p.ustep, 0), 1, u, p.D, lane);
    if (lane == 0) p.tgrid[n] = t0;
    k[0] = rhs(p, sm.ops, sm.th, u, lane);
    stv(rec(p.dense, 0), 1, k[0], p.D, lane);
    // (x / (abstol + reltol |s|))^2 summed over the lane's components
    auto sq2 = [&](R xa, R xb, R sa, R sb) {
        const R ea = xa / (abstol + reltol * sa), eb = xb / (abstol + reltol * sb);
        return (on_a ? ea * ea : (R)0) + (on_b ? eb * eb : (R)0);
    };
    PIControl<R, 5> pi;
    {   // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
        const R d0 = PR::sq(wsum(sq2(u.a, u.b, fabs(u.a), fabs(u.b))) / Dr);
        const R d1 = PR::sq(wsum(sq2(k[0].a, k[0].b, fabs(u.a), fabs(u.b))) / Dr);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        const V<R> g{fma(dt0, k[0].a, u.a), fma(dt0, k[0].b, u.b)};
        un = rhs(p, sm.ops, sm.th, g, lane);
        const R d2 = PR::sq(wsum(sq2(un.a - k[0].a, un.b - k[0].b, fabs(u.a), fabs(u.b))) / Dr) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    while (isave < p.n_save) {
        R h = pi.dt;
        bool clipped = false;
        if (t + h >= t1 - PR::clip * fabs(t1)) { h = t1 - t; clipped = true; }
#pragma unroll
        for (int i = 1; i < 7; ++i) {
            R aa = (R)0, ab = (R)0;
#pragma unroll
            for (int j = 0; j < i; ++j)
                if (Tsit5::a(i, j) != 0.0) { aa = fma((R)Tsit5::a(i, j), k[j].a, aa); ab = fma((R)Tsit5::a(i, j), k[j].b, ab); }
            const V<R> g{fma(h, aa, u.a), fma(h, ab, u.b)};
            if (i == 6) un = g;
            k[i] = rhs(p, sm.ops, sm.th, g, lane);
        }
        R ea = (R)0, eb = (R)0;
#pragma unroll
        for (int j = 0; j < 7; ++j) { ea = fma((R)Tsit5::bt(j), k[j].a, ea); eb = fma((R)Tsit5::bt(j), k[j].b, eb); }
        const R EEst = PR::sq(wsum(sq2(h * ea, h * eb, fmax(fabs(u.a), fabs(un.a)), fmax(fabs(u.b), fabs(un.b)))) / Dr);
        if (!(EEst <= PR::huge)) { bad = 1; break; }   // NaN / Inf
        if (pi.judge(EEst)) {
            if (nacc >= p.max_steps) { bad = 2; break; }
            const R tn = clipped ? t1 : t + h;
            for (int i = 1; i < 7; ++i) stv(rec(p.dense, nacc * 6 + i), 1, k[i], p.D, lane);
            while (isave < p.n_save) {
                const R ts = t0 + p.save_dt * (R)isave;
                if (ts > tn + PR::clip * fabs(tn)) break;
                R bw[7];
                Tsit5::weights(fmin((ts - t) / h, (R)1), bw);
                R aa = (R)0, ab = (R)0;
#pragma unroll
                for (int j = 0; j < 7; ++j) { aa = fma(bw[j], k[j].a, aa); ab = fma(bw[j], k[j].b, ab); }
                const V<R> us{fma(h, aa, u.a), fma(h, ab, u.b)};
                stv(p.out + (size_t)isave * D * N + n, N, us, p.D, lane);
                stv(rec(p.usave, isave), 1, us, p.D, lane);
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = tn;
            ++nacc;
            if (lane == 0) p.tgrid[(size_t)nacc * N + n] = t;
            u = un;
            k[0] = k[6];
            stv(rec(p.ustep, nacc), 1, u, p.D, lane);
        } else {
            pi.reject(h);
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        const V<R> nan{PR::nan(), PR::nan()};
        for (int is = isave; is < p.n_save; ++is) {
            stv(p.out + (size_t)is * D * N + n, N, nan, p.D, lane);
            stv(rec(p.usave, is), 1, nan, p.D, lane);
        }
    }
    const bool ok = warp_finite(u);
    if (lane == 0) {
        p.nacc[n] = nacc;
        if (p.status) p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// ---- 4. replay adjoint of an adaptive solve: each accepted step split at the save times inside it, u(t) from the step's free
// interpolant; the save cotangents at the saved states the forward recorded (the handle's copy, not the caller's `out`) ----
template <typename R>
__global__ void __launch_bounds__(128) tsit5_adaptive_adjoint_kernel(Run<R> p)
{
    using PR = Prec<R>;
    const Smem<R> sm = carve(p);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    R *gw = sm.g + (size_t)warp * p.gstride;
    for (int q = lane; q < p.P + 1; q += 32) gw[q] = (R)0;
    stage(p, sm.ops, sm.th);
    const int traj = blockIdx.x * W + warp;
    if (traj < p.N) {
        const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
        auto rec = [&](const R *b, int row) { return b + ((size_t)row * N + n) * D; };
        const int nacc = p.nacc[n];
        V<R> lam{(R)0, (R)0}, kl[6];
        R loss = (R)0;
        auto jump = [&](int is) { save_jump(p, sm.ops, is, ldv(rec(p.usave, is), 1, p.D, lane), lam, loss, n, lane); };
        int isave = p.n_save - 1;
        jump(isave);
        --isave;
        for (int s = nacc - 1; s >= 0; --s) {
            const R tn = p.tgrid[(size_t)s * N + n], tn1 = p.tgrid[(size_t)(s + 1) * N + n], hn = tn1 - tn;
            const R eps = PR::eta * hn;
            const V<R> u_s = ldv(rec(p.ustep, s), 1, p.D, lane);
            R cur = tn1;
            while (cur > tn + eps) {
                const R ts = p.t0 + p.save_dt * (R)isave;
                const R ta = (isave >= 0 && ts > tn + eps) ? ts : tn;
                const R h = cur - ta;
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                    R bw[7];
                    Tsit5::weights(fmin(fmax((cur - (R)Tsit5::c(i) * h - tn) / hn, (R)0), (R)1), bw);
                    R xa = (R)0, xb = (R)0, ga = (R)0, gb = (R)0;
#pragma unroll
                    for (int j = 0; j < 7; ++j) {
                        const V<R> kj = ldv(rec(p.dense, s * 6 + j), 1, p.D, lane);
                        xa = fma(bw[j], kj.a, xa);
                        xb = fma(bw[j], kj.b, xb);
                    }
#pragma unroll
                    for (int j = 0; j < i; ++j)
                        if (Tsit5::a(i, j) != 0.0) { ga = fma((R)Tsit5::a(i, j), kl[j].a, ga); gb = fma((R)Tsit5::a(i, j), kl[j].b, gb); }
                    const V<R> x{fma(hn, xa, u_s.a), fma(hn, xb, u_s.b)}, g{fma(h, ga, lam.a), fma(h, gb, lam.b)};
                    kl[i] = rhs_vjp(p, sm.ops, sm.th, x, g, h * (R)Tsit5::b(i), gw, lane);
                }
                R aa = (R)0, ab = (R)0;
#pragma unroll
                for (int j = 0; j < 6; ++j) { aa = fma((R)Tsit5::b(j), kl[j].a, aa); ab = fma((R)Tsit5::b(j), kl[j].b, ab); }
                lam.a = fma(h, aa, lam.a);
                lam.b = fma(h, ab, lam.b);
                cur = ta;
                if (isave >= 0 && fabs(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
        if (p.grad_u0) stv(p.grad_u0 + n, N, lam, p.D, lane);
        loss = wsum(loss);
        if (lane == 0) gw[p.P] = loss;
    }
    cta_reduce(p, sm.g);
}

// ---- 5. RKC2 forward (the recurrence of fkpp_tuned.cuh::forward_rkc_kernel2); records u_n and f(u_n) ----
template <typename R>
__global__ void __launch_bounds__(128) rkc2_forward_kernel(Run<R> p)
{
    const Smem<R> sm = carve(p);
    stage(p, sm.ops, sm.th);
    const int lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const int traj = blockIdx.x * W + (threadIdx.x >> 5);
    if (traj >= p.N) return;
    const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
    const R dt = p.dt, mt1 = __ldg(p.rkc);
    auto rec = [&](R *b, int row) { return b + ((size_t)row * N + n) * D; };
    V<R> u = ldv(p.u0 + n, N, p.D, lane);
    stv(p.out + n, N, u, p.D, lane);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
        const V<R> F0 = rhs(p, sm.ops, sm.th, u, lane);
        stv(rec(p.ustep, s), 1, u, p.D, lane);
        stv(rec(p.dense, s), 1, F0, p.D, lane);
        // the stages as increments D_j = Y_j - u: they are O(h f), so their round-off is not the recurrence's amplification of
        // |u| (carried as Y_j, fp32 adaptive solves at 32..64 stages were 5.9e-5 off the fp64 reference; now 6.4e-7)
        V<R> D0{(R)0, (R)0}, D1{mt1 * dt * F0.a, mt1 * dt * F0.b};
        for (int j = 2; j <= p.S; ++j) {
            const V<R> F = rhs(p, sm.ops, sm.th, V<R>{u.a + D1.a, u.b + D1.b}, lane);
            const R mu = __ldg(p.rkc + RKC_MU + j), nu = __ldg(p.rkc + RKC_NU + j), mt = __ldg(p.rkc + RKC_MT + j), ga = __ldg(p.rkc + RKC_GA + j);
            const V<R> D2{fma(ga * dt, F0.a, fma(mt * dt, F.a, fma(nu, D0.a, mu * D1.a))),
                          fma(ga * dt, F0.b, fma(mt * dt, F.b, fma(nu, D0.b, mu * D1.b)))};
            D0 = D1;
            D1 = D2;
        }
        u = V<R>{u.a + D1.a, u.b + D1.b};
        if ((s + 1) % p.save_every == 0) { stv(p.out + (size_t)isave * D * N + n, N, u, p.D, lane); ++isave; }
    }
    stv(rec(p.ustep, p.n_steps), 1, u, p.D, lane);
    stv(rec(p.dense, p.n_steps), 1, rhs(p, sm.ops, sm.th, u, lane), p.D, lane);
    const bool ok = warp_finite(u);
    if (p.status && lane == 0) p.status[n] = ok ? 0 : 1;
}

// ---- 6. RKC2 adjoint (fkpp_tuned.cuh::adjoint_kernel2<.., true>, the oracle's ude_adjoint_rkc2_fixed): lambda stepped backwards
// with RKC2 itself, u(t) from the cubic Hermite interpolant on (u_n, f_n, u_{n+1}, f_{n+1}); stage j sits at t_{n+1} - c_j dt;
// the theta-gradient of a step is dt sum_j w_j (df/dtheta)^T(x_j) Y_j with the recurrence's quadrature weights ----
template <typename R>
__global__ void __launch_bounds__(128) rkc2_adjoint_kernel(Run<R> p)
{
    const Smem<R> sm = carve(p);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    R *gw = sm.g + (size_t)warp * p.gstride;
    for (int q = lane; q < p.P + 1; q += 32) gw[q] = (R)0;
    stage(p, sm.ops, sm.th);
    const int traj = blockIdx.x * W + warp;
    if (traj < p.N) {
        const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
        const R dt = p.dt, mt1 = __ldg(p.rkc);
        auto rec = [&](const R *b, int row) { return b + ((size_t)row * N + n) * D; };
        V<R> lam{(R)0, (R)0};
        R loss = (R)0;
        auto jump = [&](int is) { save_jump(p, sm.ops, is, ldv(rec(p.ustep, is * p.save_every), 1, p.D, lane), lam, loss, n, lane); };
        jump(p.n_steps / p.save_every);
        for (int s = p.n_steps - 1; s >= 0; --s) {
            const V<R> y0 = ldv(rec(p.ustep, s), 1, p.D, lane), y1 = ldv(rec(p.ustep, s + 1), 1, p.D, lane);
            const V<R> f0 = ldv(rec(p.dense, s), 1, p.D, lane), f1 = ldv(rec(p.dense, s + 1), 1, p.D, lane);
            V<R> D0{(R)0, (R)0}, D1{(R)0, (R)0}, F0{(R)0, (R)0};   // increments Y_j - lambda (kernel 5)
            for (int j = 0; j < p.S; ++j) {
                const R Th = (R)1 - __ldg(p.rkc + RKC_C + j);
                // x = (1 - Th) y0 + Th y1 + Th (Th - 1) ((1 - 2 Th) (y1 - y0) + (Th - 1) dt f0 + Th dt f1)
                auto herm = [&](R a0, R a1, R g0, R g1) {
                    return ((R)1 - Th) * a0 + Th * a1 + Th * (Th - (R)1) * (((R)1 - (R)2 * Th) * (a1 - a0) + (Th - (R)1) * dt * g0 + Th * dt * g1);
                };
                const V<R> x{herm(y0.a, y1.a, f0.a, f1.a), herm(y0.b, y1.b, f0.b, f1.b)};
                const V<R> F = rhs_vjp(p, sm.ops, sm.th, x, V<R>{lam.a + D1.a, lam.b + D1.b}, dt * __ldg(p.rkc + RKC_W + j), gw, lane);
                if (j == 0) {
                    F0 = F;
                    D1 = V<R>{mt1 * dt * F0.a, mt1 * dt * F0.b};
                } else {
                    const R mu = __ldg(p.rkc + RKC_MU + j + 1), nu = __ldg(p.rkc + RKC_NU + j + 1), mt = __ldg(p.rkc + RKC_MT + j + 1),
                            ga = __ldg(p.rkc + RKC_GA + j + 1);
                    const V<R> D2{fma(ga * dt, F0.a, fma(mt * dt, F.a, fma(nu, D0.a, mu * D1.a))),
                                  fma(ga * dt, F0.b, fma(mt * dt, F.b, fma(nu, D0.b, mu * D1.b)))};
                    D0 = D1;
                    D1 = D2;
                }
            }
            lam = V<R>{lam.a + D1.a, lam.b + D1.b};
            if (s % p.save_every == 0) jump(s / p.save_every);
        }
        if (p.grad_u0) stv(p.grad_u0 + n, N, lam, p.D, lane);
        loss = wsum(loss);
        if (lane == 0) gw[p.P] = loss;
    }
    cta_reduce(p, sm.g);
}

// The adaptive RKC2 kernels below repeat the stage recurrence of kernels 5 / 6 instead of calling shared helpers.

// the cubic Hermite interpolant on (a0, g0, a1, g1) over a step of length h at fraction Th (OrdinaryDiffEq's dense output of
// the ROCK methods; kernel 6 writes the same expression inline)
template <typename R>
__device__ __forceinline__ R herm3(R Th, R h, R a0, R a1, R g0, R g1)
{
    return ((R)1 - Th) * a0 + Th * a1 + Th * (Th - (R)1) * (((R)1 - (R)2 * Th) * (a1 - a0) + (Th - (R)1) * h * g0 + Th * h * g1);
}

// ---- 7. adaptive RKC2 forward (ROCK2(eigen_est = rho) without dt, npde.jl:80-84,120-123).  Per attempt the fewest stages
// s in 2..S with beta(s) >= 1.05 h rho (none: s = S and h = beta(S) / (1.05 rho)), the s-stage recurrence of kernel 5, the
// error estimate of Sommeijer, Shampine and Verwer est = 0.8 (u_n - u_{n+1}) + 0.4 h (f(u_n) + f(u_{n+1})), kernel 3's PI
// controller with the order-2 exponents (7/20, 1/5) and the initial step's exponent 1/3.  Saves from the cubic Hermite interpolant; f(u_{n+1}) is the next
// step's f(u_n), so an accepted step of s stages costs s right-hand sides.  Records u_n, f(u_n), t_n and s_n ----
template <typename R>
__global__ void __launch_bounds__(128) rkc2_adaptive_forward_kernel(Run<R> p)
{
    using PR = Prec<R>;
    const Smem<R> sm = carve(p);
    stage(p, sm.ops, sm.th);
    const int lane = threadIdx.x & 31, W = blockDim.x >> 5;
    const int traj = blockIdx.x * W + (threadIdx.x >> 5);
    if (traj >= p.N) return;
    const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
    const bool on_a = lane < p.D, on_b = lane + 32 < p.D;
    auto rec = [&](R *b, int row) { return b + ((size_t)row * N + n) * D; };
    const R t0 = p.t0, t1 = p.t0 + p.save_dt * (R)(p.n_save - 1);
    const R abstol = p.abstol, reltol = p.reltol, Dr = (R)p.D, rho = p.rho;
    V<R> u = ldv(p.u0 + n, N, p.D, lane), F0, un, F1;
    stv(p.out + n, N, u, p.D, lane);
    stv(rec(p.usave, 0), 1, u, p.D, lane);
    stv(rec(p.ustep, 0), 1, u, p.D, lane);
    if (lane == 0) p.tgrid[n] = t0;
    F0 = rhs(p, sm.ops, sm.th, u, lane);
    stv(rec(p.dense, 0), 1, F0, p.D, lane);
    auto sq2 = [&](R xa, R xb, R sa, R sb) {
        const R ea = xa / (abstol + reltol * sa), eb = xb / (abstol + reltol * sb);
        return (on_a ? ea * ea : (R)0) + (on_b ? eb * eb : (R)0);
    };
    PIControl<R, 2, 3> pi;   // order-2 gains, initial-step exponent 1/3 (the Python reference divides by 3 too)
    {   // initial step: kernel 3's heuristic
        const R d0 = PR::sq(wsum(sq2(u.a, u.b, fabs(u.a), fabs(u.b))) / Dr);
        const R d1 = PR::sq(wsum(sq2(F0.a, F0.b, fabs(u.a), fabs(u.b))) / Dr);
        const R dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        const V<R> g{fma(dt0, F0.a, u.a), fma(dt0, F0.b, u.b)};
        un = rhs(p, sm.ops, sm.th, g, lane);
        const R d2 = PR::sq(wsum(sq2(un.a - F0.a, un.b - F0.b, fabs(u.a), fabs(u.b))) / Dr) / dt0;
        pi.hnw(dt0, d1, d2, t1 - t0);
    }
    R t = t0;
    int nacc = 0, isave = 1, bad = 0;
    while (isave < p.n_save) {
        R h = pi.dt;
        bool clipped = false;
        if (t + h >= t1 - PR::clip * fabs(t1)) { h = t1 - t; clipped = true; }
        const R hr = (R)1.05 * h * rho;
        int s = 2;
        while (s < p.S && __ldg(p.beta + s) < hr) ++s;
        if (__ldg(p.beta + s) < hr) {   // even S stages are not stable at h: the step the cap allows
            h = __ldg(p.beta + s) / ((R)1.05 * rho);
            clipped = false;
        }
        const R *T = p.rkc + (size_t)(s - 2) * RKC_LEN;
        const R mt1 = __ldg(T);
        V<R> D0{(R)0, (R)0}, D1{mt1 * h * F0.a, mt1 * h * F0.b};   // increments Y_j - u (kernel 5)
        for (int j = 2; j <= s; ++j) {
            const V<R> F = rhs(p, sm.ops, sm.th, V<R>{u.a + D1.a, u.b + D1.b}, lane);
            const R mu = __ldg(T + RKC_MU + j), nu = __ldg(T + RKC_NU + j), mt = __ldg(T + RKC_MT + j), ga = __ldg(T + RKC_GA + j);
            const V<R> D2{fma(ga * h, F0.a, fma(mt * h, F.a, fma(nu, D0.a, mu * D1.a))),
                          fma(ga * h, F0.b, fma(mt * h, F.b, fma(nu, D0.b, mu * D1.b)))};
            D0 = D1;
            D1 = D2;
        }
        un = V<R>{u.a + D1.a, u.b + D1.b};
        F1 = rhs(p, sm.ops, sm.th, un, lane);
        // u_n - u_{n+1} = -D_s
        const R ea = fma((R)0.4 * h, F0.a + F1.a, (R)-0.8 * D1.a), eb = fma((R)0.4 * h, F0.b + F1.b, (R)-0.8 * D1.b);
        const R EEst = PR::sq(wsum(sq2(ea, eb, fmax(fabs(u.a), fabs(un.a)), fmax(fabs(u.b), fabs(un.b)))) / Dr);
        if (!(EEst <= PR::huge)) { bad = 1; break; }   // NaN / Inf
        if (pi.judge(EEst)) {
            if (nacc >= p.max_steps) { bad = 2; break; }
            const R tn = clipped ? t1 : t + h;
            while (isave < p.n_save) {
                const R ts = t0 + p.save_dt * (R)isave;
                if (ts > tn + PR::clip * fabs(tn)) break;
                const R Th = fmin((ts - t) / h, (R)1);
                const V<R> us{herm3(Th, h, u.a, un.a, F0.a, F1.a), herm3(Th, h, u.b, un.b, F0.b, F1.b)};
                stv(p.out + (size_t)isave * D * N + n, N, us, p.D, lane);
                stv(rec(p.usave, isave), 1, us, p.D, lane);
                ++isave;
            }
            pi.accept(EEst, h, clipped);
            t = tn;
            if (lane == 0) p.sstep[(size_t)nacc * N + n] = s;
            ++nacc;
            if (lane == 0) p.tgrid[(size_t)nacc * N + n] = t;
            u = un;
            F0 = F1;
            stv(rec(p.ustep, nacc), 1, u, p.D, lane);
            stv(rec(p.dense, nacc), 1, F0, p.D, lane);
        } else {
            pi.reject(h);
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        const V<R> nan{PR::nan(), PR::nan()};
        for (int is = isave; is < p.n_save; ++is) {
            stv(p.out + (size_t)is * D * N + n, N, nan, p.D, lane);
            stv(rec(p.usave, is), 1, nan, p.D, lane);
        }
    }
    const bool ok = warp_finite(u);
    if (lane == 0) {
        p.nacc[n] = nacc;
        if (p.status) p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// ---- 8. replay adjoint of an adaptive RKC2 solve: each accepted step split at the save times inside it (kernel 4); a piece
// of length h' <= h_n steps lambda back with RKC2 of the step's recorded s_n stages (stable: h' rho <= h_n rho), stage j at
// cur - c_j h' with u from the step's Hermite interpolant, the theta-gradient with the quadrature weights h' w_j (kernel 6 with
// dt -> h'); the save cotangents at the saved states the forward recorded ----
template <typename R>
__global__ void __launch_bounds__(128) rkc2_adaptive_adjoint_kernel(Run<R> p)
{
    using PR = Prec<R>;
    const Smem<R> sm = carve(p);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    R *gw = sm.g + (size_t)warp * p.gstride;
    for (int q = lane; q < p.P + 1; q += 32) gw[q] = (R)0;
    stage(p, sm.ops, sm.th);
    const int traj = blockIdx.x * W + warp;
    if (traj < p.N) {
        const size_t N = (size_t)p.N, n = (size_t)traj, D = (size_t)p.D;
        auto rec = [&](const R *b, int row) { return b + ((size_t)row * N + n) * D; };
        const int nacc = p.nacc[n];
        V<R> lam{(R)0, (R)0};
        R loss = (R)0;
        auto jump = [&](int is) { save_jump(p, sm.ops, is, ldv(rec(p.usave, is), 1, p.D, lane), lam, loss, n, lane); };
        int isave = p.n_save - 1;
        jump(isave);
        --isave;
        for (int st = nacc - 1; st >= 0; --st) {
            const R tn = p.tgrid[(size_t)st * N + n], tn1 = p.tgrid[(size_t)(st + 1) * N + n], hn = tn1 - tn;
            const R eps = PR::eta * hn;
            const V<R> y0 = ldv(rec(p.ustep, st), 1, p.D, lane), y1 = ldv(rec(p.ustep, st + 1), 1, p.D, lane);
            const V<R> f0 = ldv(rec(p.dense, st), 1, p.D, lane), f1 = ldv(rec(p.dense, st + 1), 1, p.D, lane);
            const int s = p.sstep[(size_t)st * N + n];
            const R *T = p.rkc + (size_t)(s - 2) * RKC_LEN;
            const R mt1 = __ldg(T);
            R cur = tn1;
            while (cur > tn + eps) {
                const R ts = p.t0 + p.save_dt * (R)isave;
                const R ta = (isave >= 0 && ts > tn + eps) ? ts : tn;
                const R h = cur - ta;
                V<R> D0{(R)0, (R)0}, D1{(R)0, (R)0}, F0{(R)0, (R)0};   // increments Y_j - lambda (kernel 5)
                for (int j = 0; j < s; ++j) {
                    const R Th = fmin(fmax((cur - __ldg(T + RKC_C + j) * h - tn) / hn, (R)0), (R)1);
                    const V<R> x{herm3(Th, hn, y0.a, y1.a, f0.a, f1.a), herm3(Th, hn, y0.b, y1.b, f0.b, f1.b)};
                    const V<R> F = rhs_vjp(p, sm.ops, sm.th, x, V<R>{lam.a + D1.a, lam.b + D1.b}, h * __ldg(T + RKC_W + j), gw, lane);
                    if (j == 0) {
                        F0 = F;
                        D1 = V<R>{mt1 * h * F0.a, mt1 * h * F0.b};
                    } else {
                        const R mu = __ldg(T + RKC_MU + j + 1), nu = __ldg(T + RKC_NU + j + 1), mt = __ldg(T + RKC_MT + j + 1),
                                ga = __ldg(T + RKC_GA + j + 1);
                        const V<R> D2{fma(ga * h, F0.a, fma(mt * h, F.a, fma(nu, D0.a, mu * D1.a))),
                                      fma(ga * h, F0.b, fma(mt * h, F.b, fma(nu, D0.b, mu * D1.b)))};
                        D0 = D1;
                        D1 = D2;
                    }
                }
                lam = V<R>{lam.a + D1.a, lam.b + D1.b};
                cur = ta;
                if (isave >= 0 && fabs(ts - ta) <= eps) { jump(isave); --isave; }
            }
        }
        if (p.grad_u0) stv(p.grad_u0 + n, N, lam, p.D, lane);
        loss = wsum(loss);
        if (lane == 0) gw[p.P] = loss;
    }
    cta_reduce(p, sm.g);
}

}  // namespace op
}  // namespace b200ude
