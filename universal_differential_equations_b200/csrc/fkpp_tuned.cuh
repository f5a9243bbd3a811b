// fkpp_tuned.cuh -- Fisher-KPP UPDE kernels for a compile-time reaction chain 1 -> H -> H -> 1 (tanh, tanh, identity):
// BASELINE config 4 (256-point grid, 1 -> 16 -> 16 -> 1).  Replaces, per Runge-Kutta stage and for every grid point of every
// ensemble member, the reference's `nn_ode` (FisherKPP/Fisher-KPP-CNN.jl:111-126; Lux twin scenario_3.jl:103-114):
//     du_i = rx_nn([u_i]) + D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1}),  periodic wrap,
// theta = [chain | w1, w2, w3, conv bias (unused), D0] (Fisher-KPP-CNN.jl:106-109), and its interpolating adjoint.
//
// One thread per grid point, a CTA holds whole trajectories (same geometry and handle-internal point-fastest stores as the
// runtime-shape kernels in ude_generic.cuh, which remain the path for every other chain shape).  What is tuned here:
//   * chain weights are compile-time-indexed 128-bit constant-bank loads (uniform registers), the RHS is one function;
//   * u and lambda neighbours travel through ONE double-buffered shared-memory exchange per stage (one barrier);
//   * the ensemble-summed gradient of the H x H layer is a per-warp FFMA outer-product GEMM over the warp's 32 points
//     (operands staged as conflict-free 128-bit rows, 2 x 4 register tile per lane), everything thin (first/last layer,
//     biases, stencil weights, D0) accumulates in per-lane registers and is reduced once, at the end of the kernel, with
//     a fixed shuffle tree and a fixed-order sum over the CTA's warps -> bitwise reproducible.
#pragma once
#include "lv32_packed.cuh"   // fma2 / bc / ldw4 / c_zero helpers
#include "ude_adjoint.cuh"

namespace b200ude {
namespace fkpp {

using lv32::add2;
using lv32::bc;
using lv32::fma2;
using lv32::ldw4;
using lv32::mul2;
using lv32::tanh2;

struct Geom {
    int Nx, tpc;   // grid points per trajectory, trajectories per CTA
};

template <int H>
struct Off {
    static constexpr int W1 = 0, B1 = H, W2 = 2 * H, B2 = 2 * H + H * H, W3 = 3 * H + H * H, B3 = 4 * H + H * H;
    static constexpr int CHAIN = 4 * H + H * H + 1;
    static constexpr int SX = CHAIN;          // w1, w2, w3, conv bias, D0
    static constexpr int P = CHAIN + 5;
};

// reaction chain, value only
template <int H, int TM>
__device__ __noinline__ float chain_value(float g, int zsel)
{
    using O = Off<H>;
    const int zb = lv32::c_zero[zsel & 7] << 2;
    float h1[H];
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 w = ldw4(zb + O::W1 + j4), b = ldw4(zb + O::B1 + j4);
        h1[j4 + 0] = tanh_dev<TM>(fmaf(w.x, g, b.x));
        h1[j4 + 1] = tanh_dev<TM>(fmaf(w.y, g, b.y));
        h1[j4 + 2] = tanh_dev<TM>(fmaf(w.z, g, b.z));
        h1[j4 + 3] = tanh_dev<TM>(fmaf(w.w, g, b.w));
    }
    float a2[H];
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 b = ldw4(zb + O::B2 + j4);
        a2[j4] = b.x; a2[j4 + 1] = b.y; a2[j4 + 2] = b.z; a2[j4 + 3] = b.w;
    }
#pragma unroll
    for (int i = 0; i < H; ++i) {
#pragma unroll
        for (int j4 = 0; j4 < H; j4 += 4) {
            const float4 w = ldw4(zb + O::W2 + i * H + j4);
            a2[j4 + 0] = fmaf(w.x, h1[i], a2[j4 + 0]);
            a2[j4 + 1] = fmaf(w.y, h1[i], a2[j4 + 1]);
            a2[j4 + 2] = fmaf(w.z, h1[i], a2[j4 + 2]);
            a2[j4 + 3] = fmaf(w.w, h1[i], a2[j4 + 3]);
        }
    }
    float y0 = c_theta[zb + O::B3], y1 = 0.0f;
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 w = ldw4(zb + O::W3 + j4);
        y0 = fmaf(w.x, tanh_dev<TM>(a2[j4 + 0]), y0);
        y1 = fmaf(w.y, tanh_dev<TM>(a2[j4 + 1]), y1);
        y0 = fmaf(w.z, tanh_dev<TM>(a2[j4 + 2]), y0);
        y1 = fmaf(w.w, tanh_dev<TM>(a2[j4 + 3]), y1);
    }
    return y0 + y1;
}

// ---- forward ----------------------------------------------------------------------------------------------------------
template <int H, int TM>
__global__ void __launch_bounds__(256) forward_kernel(FwdParams p, Geom geo)
{
    using O = Off<H>;
    extern __shared__ __align__(16) float s_dyn[];   // [2][slots] neighbour exchange, double buffered
    const int Nx = geo.Nx, slots = geo.tpc * Nx;
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int im = base + (i + Nx - 1) % Nx, ip = base + (i + 1) % Nx;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float dt = p.dt;
    const float w1 = c_theta[O::SX], w2 = c_theta[O::SX + 1], w3 = c_theta[O::SX + 2], D0 = c_theta[O::SX + 4];
    float u = __ldg(p.u0 + (size_t)i * N + n);
    int flip = 0;
    auto rhs = [&](float g, int zsel) {
        float *sU = s_dyn + flip * slots;
        flip ^= 1;
        if (valid) sU[slot] = g;
        __syncthreads();   // the buffer written two evaluations ago is free again: every thread passed this barrier since
        const float gm = sU[im], gp = sU[ip];
        const float y = chain_value<H, TM>(g, zsel);
        return fmaf(D0, fmaf(w1, gm, fmaf(w2, g, w3 * gp)), y);
    };
    auto store_int = [&](float *b, int row, float v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
    auto store_abi = [&](float *b, int row, float v) { if (live) b[((size_t)row * Nx + i) * N + n] = v; };
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    float k[7];
    k[0] = rhs(u, 0);
    store_int(p.dense, 0, k[0]);
#pragma unroll
    for (int j = 1; j < 7; ++j) k[j] = 0.0f;
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll 1
        for (int st = 1; st < 7; ++st) {
            float acc = 0.0f;
#define B200UDE_FKPP_COMB(I)                                                                                  \
    case I: {                                                                                                 \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) acc = fmaf((float)Tsit5::a(I, j), k[j], acc); \
    } break;
            switch (st) {
                B200UDE_FKPP_COMB(1)
                B200UDE_FKPP_COMB(2)
                B200UDE_FKPP_COMB(3)
                B200UDE_FKPP_COMB(4)
                B200UDE_FKPP_COMB(5)
            default:
                B200UDE_FKPP_COMB(6)
            }
#undef B200UDE_FKPP_COMB
            const float g = fmaf(dt, acc, u);
            if (st == 6) u = g;
            const float kk = rhs(g, st);
            switch (st) {
            case 1: k[1] = kk; break;
            case 2: k[2] = kk; break;
            case 3: k[3] = kk; break;
            case 4: k[4] = kk; break;
            case 5: k[5] = kk; break;
            default: k[6] = kk; break;
            }
            store_int(p.dense, s * 6 + st, kk);
        }
        store_int(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store_abi(p.out, isave, u); ++isave; }
        k[0] = k[6];
    }
    if (p.status) {   // a trajectory is flagged when any of its points is non-finite
        __syncthreads();
        float *sU = s_dyn;
        if (valid) sU[slot] = (fabsf(u) <= 3.0e38f) ? 0.0f : 1.0f;
        __syncthreads();
        if (live && i == 0) {
            float any = 0.0f;
            for (int q = 0; q < Nx; ++q) any += sU[base + q];
            p.status[n] = any > 0.0f ? 1 : 0;
        }
    }
}

// ---- adjoint ----------------------------------------------------------------------------------------------------------
template <int H>
struct __align__(16) WarpRows {
    static constexpr int LD = H + 4;   // 128-bit rows, conflict-free for the per-lane row stores and the tile loads
    float Q[32 * LD];                  // q2 rows of the warp's 32 points
    float A[32 * LD];                  // h1 rows
};

template <int H, int TM>
__global__ void __launch_bounds__(256) adjoint_kernel(AdjParams p, Geom geo)
{
    using O = Off<H>;
    static_assert(H == 16, "the 2 x 4 lane tile below covers a 16 x 16 layer with 32 lanes");
    constexpr int P = O::P;
    extern __shared__ __align__(16) float s_dyn[];
    const int Nx = geo.Nx, slots = geo.tpc * Nx;
    const int nwarp = blockDim.x >> 5;
    float2 *sX = reinterpret_cast<float2 *>(s_dyn);                       // [2][slots] (x, g) exchange, double buffered
    WarpRows<H> *rows = reinterpret_cast<WarpRows<H> *>(s_dyn + 4 * ((slots + 1) / 2) * 2);
    const int slot = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpRows<H> &wr = rows[warp];
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int im = base + (i + Nx - 1) % Nx, ip = base + (i + 1) % Nx;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt, inv_dt = 1.0f / dt;
    const float w1 = c_theta[O::SX], w2 = c_theta[O::SX + 1], w3 = c_theta[O::SX + 2], D0 = c_theta[O::SX + 4];
    const int jt = lane >> 2, it = lane & 3;   // dW2 tile: j = 2 jt + {0, 1}, i = 4 it + {0..3}

    float2 acc[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[q] = bc(0.0f);
    float a_w3[H], a_b2[H], a_w1[H], a_b1[H];
#pragma unroll
    for (int j = 0; j < H; ++j) { a_w3[j] = 0.f; a_b2[j] = 0.f; a_w1[j] = 0.f; a_b1[j] = 0.f; }
    float a_b3 = 0.f, a_s1 = 0.f, a_s2 = 0.f, a_s3 = 0.f, a_D0 = 0.f;

    float lam = 0.0f, loss = 0.0f;
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
    int flip = 0;
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        float kl[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) kl[j] = 0.0f;
#pragma unroll 1
        for (int st = 0; st < 6; ++st) {
            float xa = 0.0f, ga = 0.0f, sc, isc;
#define B200UDE_FKPP_PRE(I)                                                                                              \
    case I: {                                                                                                            \
        _Pragma("unroll") for (int j = 0; j < 7; ++j) if (Tsit5::bw(I, j) != 0.0)                                         \
            xa = fmaf((float)Tsit5::bw(I, j), __ldg(p.dense + ((size_t)(s * 6 + j) * N + n) * Nx + i), xa);               \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) ga = fmaf((float)Tsit5::a(I, j), kl[j], ga); \
        sc = dt * (float)Tsit5::b(I);                                                                                    \
        isc = inv_dt * (float)(1.0 / Tsit5::b(I));                                                                       \
    } break;
            switch (st) {
                B200UDE_FKPP_PRE(0)
                B200UDE_FKPP_PRE(1)
                B200UDE_FKPP_PRE(2)
                B200UDE_FKPP_PRE(3)
                B200UDE_FKPP_PRE(4)
            default:
                B200UDE_FKPP_PRE(5)
            }
#undef B200UDE_FKPP_PRE
            const float x = fmaf(dt, xa, __ldg(p.ustep + ((size_t)s * N + n) * Nx + i));
            const float g = fmaf(dt, ga, lam);
            const int zb = lv32::c_zero[st] << 2;
            // neighbours of u (stencil-weight gradients) and of lambda (transposed stencil): one exchange
            float2 *sx = sX + flip * slots;
            flip ^= 1;
            if (valid) sx[slot] = make_float2(x, g);
            __syncthreads();
            const float2 nm = sx[im], np = sx[ip];
            const float sg = lv * sc * g;
            // ---- chain forward, activations kept ----
            float h1[H], v[H];
#pragma unroll
            for (int j4 = 0; j4 < H; j4 += 4) {
                const float4 w = ldw4(zb + O::W1 + j4), b = ldw4(zb + O::B1 + j4);
                h1[j4 + 0] = tanh_dev<TM>(fmaf(w.x, x, b.x));
                h1[j4 + 1] = tanh_dev<TM>(fmaf(w.y, x, b.y));
                h1[j4 + 2] = tanh_dev<TM>(fmaf(w.z, x, b.z));
                h1[j4 + 3] = tanh_dev<TM>(fmaf(w.w, x, b.w));
                *reinterpret_cast<float4 *>(&wr.A[lane * WarpRows<H>::LD + j4]) = make_float4(h1[j4], h1[j4 + 1], h1[j4 + 2], h1[j4 + 3]);
            }
#pragma unroll
            for (int j4 = 0; j4 < H; j4 += 4) {
                const float4 b = ldw4(zb + O::B2 + j4);
                v[j4] = b.x; v[j4 + 1] = b.y; v[j4 + 2] = b.z; v[j4 + 3] = b.w;
            }
#pragma unroll
            for (int ii = 0; ii < H; ++ii) {
#pragma unroll
                for (int j4 = 0; j4 < H; j4 += 4) {
                    const float4 w = ldw4(zb + O::W2 + ii * H + j4);
                    v[j4 + 0] = fmaf(w.x, h1[ii], v[j4 + 0]);
                    v[j4 + 1] = fmaf(w.y, h1[ii], v[j4 + 1]);
                    v[j4 + 2] = fmaf(w.z, h1[ii], v[j4 + 2]);
                    v[j4 + 3] = fmaf(w.w, h1[ii], v[j4 + 3]);
                }
            }
            // h2 = tanh(v); output-layer gradients; q2 = W3 * sg * (1 - h2^2) -> v and the warp's Q rows
            a_b3 += sg;
#pragma unroll
            for (int j4 = 0; j4 < H; j4 += 4) {
                const float4 w = ldw4(zb + O::W3 + j4);
                const float w_[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float h2 = tanh_dev<TM>(v[j4 + k]);
                    a_w3[j4 + k] = fmaf(sg, h2, a_w3[j4 + k]);
                    v[j4 + k] = w_[k] * sg * fmaf(-h2, h2, 1.0f);
                    a_b2[j4 + k] += v[j4 + k];
                }
                *reinterpret_cast<float4 *>(&wr.Q[lane * WarpRows<H>::LD + j4]) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);
            }
            __syncwarp();
            // ---- dW2 += q2 (x) h1 over the warp's 32 points ----
#pragma unroll 8
            for (int t = 0; t < 32; ++t) {
                const float2 q = *reinterpret_cast<const float2 *>(&wr.Q[t * WarpRows<H>::LD + 2 * jt]);
                const float4 hh = *reinterpret_cast<const float4 *>(&wr.A[t * WarpRows<H>::LD + 4 * it]);
                const float2 h01 = make_float2(hh.x, hh.y), h23 = make_float2(hh.z, hh.w);
                acc[0] = fma2(bc(q.x), h01, acc[0]);
                acc[1] = fma2(bc(q.x), h23, acc[1]);
                acc[2] = fma2(bc(q.y), h01, acc[2]);
                acc[3] = fma2(bc(q.y), h23, acc[3]);
            }
            __syncwarp();
            // ---- q1 = (W2^T q2) * (1 - h1^2); first-layer gradients; dx ----
            float dx0 = 0.0f, dx1 = 0.0f;
#pragma unroll
            for (int ii = 0; ii < H; ++ii) {
                float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
                for (int j4 = 0; j4 < H; j4 += 4) {
                    const float4 w = ldw4(zb + O::W2 + ii * H + j4);
                    s0 = fmaf(w.x, v[j4 + 0], s0);
                    s1 = fmaf(w.y, v[j4 + 1], s1);
                    s0 = fmaf(w.z, v[j4 + 2], s0);
                    s1 = fmaf(w.w, v[j4 + 3], s1);
                }
                const float q1 = (s0 + s1) * fmaf(-h1[ii], h1[ii], 1.0f);
                a_b1[ii] += q1;
                a_w1[ii] = fmaf(q1, x, a_w1[ii]);
                const float wi = c_theta[zb + O::W1 + ii];
                if (ii & 1) dx1 = fmaf(wi, q1, dx1);
                else dx0 = fmaf(wi, q1, dx0);
            }
            const float dx = (dx0 + dx1) * isc;
            // (J^T g)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
            const float kn = dx + D0 * fmaf(w2, g, fmaf(w1, np.y, w3 * nm.y));
            switch (st) {
            case 0: kl[0] = kn; break;
            case 1: kl[1] = kn; break;
            case 2: kl[2] = kn; break;
            case 3: kl[3] = kn; break;
            case 4: kl[4] = kn; break;
            default: kl[5] = kn; break;
            }
            a_s1 = fmaf(sg * D0, nm.x, a_s1);
            a_s2 = fmaf(sg * D0, x, a_s2);
            a_s3 = fmaf(sg * D0, np.x, a_s3);
            a_D0 = fmaf(sg, fmaf(w1, nm.x, fmaf(w2, x, w3 * np.x)), a_D0);
        }
        float a = 0.0f;
#pragma unroll
        for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j], a);
        lam = fmaf(dt, a, lam);
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    if (p.grad_u0 && live) p.grad_u0[(size_t)i * N + n] = lam;

    // ---- reduction: lanes -> warp (fixed shuffle tree), warps -> CTA (fixed order) ----
    __syncthreads();
    float *gw = s_dyn + (size_t)warp * (P + 1);   // the staging area is free now: [nwarp][P+1]
    auto wsum = [&](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
    __syncthreads();
#pragma unroll
    for (int j = 0; j < H; ++j) {
        const float r0 = wsum(a_w1[j]), r1 = wsum(a_b1[j]), r2 = wsum(a_b2[j]), r3 = wsum(a_w3[j]);
        if (lane == 0) { gw[O::W1 + j] = r0; gw[O::B1 + j] = r1; gw[O::B2 + j] = r2; gw[O::W3 + j] = r3; }
    }
    {
        const float r0 = wsum(a_b3), r1 = wsum(a_s1), r2 = wsum(a_s2), r3 = wsum(a_s3), r4 = wsum(a_D0), r5 = wsum(loss * lv);
        if (lane == 0) {
            gw[O::B3] = r0; gw[O::SX] = r1; gw[O::SX + 1] = r2; gw[O::SX + 2] = r3; gw[O::SX + 3] = 0.0f; gw[O::SX + 4] = r4;
            gw[P] = r5;
        }
    }
    gw[O::W2 + (4 * it + 0) * H + 2 * jt] = acc[0].x;
    gw[O::W2 + (4 * it + 1) * H + 2 * jt] = acc[0].y;
    gw[O::W2 + (4 * it + 2) * H + 2 * jt] = acc[1].x;
    gw[O::W2 + (4 * it + 3) * H + 2 * jt] = acc[1].y;
    gw[O::W2 + (4 * it + 0) * H + 2 * jt + 1] = acc[2].x;
    gw[O::W2 + (4 * it + 1) * H + 2 * jt + 1] = acc[2].y;
    gw[O::W2 + (4 * it + 2) * H + 2 * jt + 1] = acc[3].x;
    gw[O::W2 + (4 * it + 3) * H + 2 * jt + 1] = acc[3].y;
    __syncthreads();
    float *dst = p.partial + (size_t)blockIdx.x * (P + 1);
    for (int q = threadIdx.x; q < P + 1; q += blockDim.x) {
        float tot = 0.0f;
        for (int w = 0; w < nwarp; ++w) tot += s_dyn[(size_t)w * (P + 1) + q];
        dst[q] = tot;
    }
}


// =====================================================================================================================
// Packed variant (even grids): a thread carries TWO adjacent grid points in the halves of 64-bit register pairs and does
// the chain arithmetic on float2 pairs (weights are scalar broadcast operands), which halves the constant-load instruction
// count of the one-point-per-thread kernels above (those were at 90 % issue-slot utilisation).  Same algorithm, same
// handle-internal layouts; a trajectory occupies Nx/2 consecutive threads.
// =====================================================================================================================
template <int H, int TM>
__device__ __noinline__ float2 chain_value2(float2 g, int zsel)
{
    using O = Off<H>;
    const int zb = lv32::c_zero[zsel & 7] << 2;
    float2 h1[H];
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 w = ldw4(zb + O::W1 + j4), b = ldw4(zb + O::B1 + j4);
        h1[j4 + 0] = tanh2<TM>(fma2(bc(w.x), g, bc(b.x)));
        h1[j4 + 1] = tanh2<TM>(fma2(bc(w.y), g, bc(b.y)));
        h1[j4 + 2] = tanh2<TM>(fma2(bc(w.z), g, bc(b.z)));
        h1[j4 + 3] = tanh2<TM>(fma2(bc(w.w), g, bc(b.w)));
    }
    float2 a2[H];
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 b = ldw4(zb + O::B2 + j4);
        a2[j4] = bc(b.x); a2[j4 + 1] = bc(b.y); a2[j4 + 2] = bc(b.z); a2[j4 + 3] = bc(b.w);
    }
#pragma unroll
    for (int i = 0; i < H; ++i) {
#pragma unroll
        for (int j4 = 0; j4 < H; j4 += 4) {
            const float4 w = ldw4(zb + O::W2 + i * H + j4);
            a2[j4 + 0] = fma2(bc(w.x), h1[i], a2[j4 + 0]);
            a2[j4 + 1] = fma2(bc(w.y), h1[i], a2[j4 + 1]);
            a2[j4 + 2] = fma2(bc(w.z), h1[i], a2[j4 + 2]);
            a2[j4 + 3] = fma2(bc(w.w), h1[i], a2[j4 + 3]);
        }
    }
    float2 y0 = bc(c_theta[zb + O::B3]), y1 = bc(0.0f);
#pragma unroll
    for (int j4 = 0; j4 < H; j4 += 4) {
        const float4 w = ldw4(zb + O::W3 + j4);
        // (the batched-inversion tanh of lv32_packed.cuh is not used here: these kernels are issue-bound and its overflow clamps
        // cost more issue slots than the saved reciprocals)
        y0 = fma2(bc(w.x), tanh2<TM>(a2[j4 + 0]), y0);
        y1 = fma2(bc(w.y), tanh2<TM>(a2[j4 + 1]), y1);
        y0 = fma2(bc(w.z), tanh2<TM>(a2[j4 + 2]), y0);
        y1 = fma2(bc(w.w), tanh2<TM>(a2[j4 + 3]), y1);
    }
    return add2(y0, y1);
}

template <int H, int TM>
__global__ void __launch_bounds__(256) forward_kernel2(FwdParams p, Geom geo)
{
    using O = Off<H>;
    extern __shared__ __align__(16) float s_dyn[];   // [2][slots] float2 neighbour exchange, double buffered
    float2 *sX = reinterpret_cast<float2 *>(s_dyn);
    const int Nx = geo.Nx, Nh = Nx >> 1, slots = geo.tpc * Nh;   // a slot = one thread = two grid points
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nh : 0, q = valid ? slot % Nh : 0;
    const int base = t_loc * Nh;
    const int im = base + (q + Nh - 1) % Nh, ip = base + (q + 1) % Nh;
    const int i0 = 2 * q;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float dt = p.dt;
    const float w1 = c_theta[O::SX], w2 = c_theta[O::SX + 1], w3 = c_theta[O::SX + 2], D0 = c_theta[O::SX + 4];
    float2 u = make_float2(__ldg(p.u0 + (size_t)i0 * N + n), __ldg(p.u0 + (size_t)(i0 + 1) * N + n));
    int flip = 0;
    auto rhs = [&](float2 g, int zsel) {
        float2 *sU = sX + flip * slots;
        flip ^= 1;
        if (valid) sU[slot] = g;
        __syncthreads();
        const float gl = sU[im].y, gr = sU[ip].x;
        const float2 y = chain_value2<H, TM>(g, zsel);
        return make_float2(fmaf(D0, fmaf(w1, gl, fmaf(w2, g.x, w3 * g.y)), y.x), fmaf(D0, fmaf(w1, g.x, fmaf(w2, g.y, w3 * gr)), y.y));
    };
    auto store_int = [&](float *b, int row, float2 v) { if (live) *reinterpret_cast<float2 *>(&b[((size_t)row * N + n) * Nx + i0]) = v; };
    auto store_abi = [&](float *b, int row, float2 v) {
        if (live) { b[((size_t)row * Nx + i0) * N + n] = v.x; b[((size_t)row * Nx + i0 + 1) * N + n] = v.y; }
    };
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    float2 k[7];
    k[0] = rhs(u, 0);
    store_int(p.dense, 0, k[0]);
#pragma unroll
    for (int j = 1; j < 7; ++j) k[j] = bc(0.0f);
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll 1
        for (int st = 1; st < 7; ++st) {
            float2 acc = bc(0.0f);
#define B200UDE_FKPP_COMB(I)                                                                                  \
    case I: {                                                                                                 \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) acc = fma2(bc((float)Tsit5::a(I, j)), k[j], acc); \
    } break;
            switch (st) {
                B200UDE_FKPP_COMB(1)
                B200UDE_FKPP_COMB(2)
                B200UDE_FKPP_COMB(3)
                B200UDE_FKPP_COMB(4)
                B200UDE_FKPP_COMB(5)
            default:
                B200UDE_FKPP_COMB(6)
            }
#undef B200UDE_FKPP_COMB
            const float2 g = fma2(bc(dt), acc, u);
            if (st == 6) u = g;
            const float2 kk = rhs(g, st);
            switch (st) {
            case 1: k[1] = kk; break;
            case 2: k[2] = kk; break;
            case 3: k[3] = kk; break;
            case 4: k[4] = kk; break;
            case 5: k[5] = kk; break;
            default: k[6] = kk; break;
            }
            store_int(p.dense, s * 6 + st, kk);
        }
        store_int(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store_abi(p.out, isave, u); ++isave; }
        k[0] = k[6];
    }
    if (p.status) {
        __syncthreads();
        float *sU = s_dyn;
        if (valid) sU[slot] = ((fabsf(u.x) <= 3.0e38f) && (fabsf(u.y) <= 3.0e38f)) ? 0.0f : 1.0f;
        __syncthreads();
        if (live && q == 0) {
            float any = 0.0f;
            for (int r = 0; r < Nh; ++r) any += sU[base + r];
            p.status[n] = any > 0.0f ? 1 : 0;
        }
    }
}

// ---- RKC2 (second-order Runge-Kutta-Chebyshev): the closed-form stabilised explicit method of the ROCK2 class the north star
// names for this stiff grid (Climate/NeuralPDE/npde.jl:61; ROCK2's own tables are not in the reference).  Recurrence per step:
//   Y0 = u, Y1 = u + mt1 h F0,  Yj = (1 - mu_j - nu_j) u + mu_j Y_{j-1} + nu_j Y_{j-2} + mt_j h F_{j-1} + ga_j h F0,  u_next = Y_s.
// The coefficient tables are computed on the host (b200ude.cu) for the handle's stage count.
struct RkcTables {
    int s;
    float mt1;
    float mu[65], nu[65], mt[65], ga[65], c[65], w[65];
};
static __constant__ RkcTables c_rkc;

template <int H, int TM>
__global__ void __launch_bounds__(256) forward_rkc_kernel2(FwdParams p, Geom geo)
{
    using O = Off<H>;
    extern __shared__ __align__(16) float s_dyn[];
    float2 *sX = reinterpret_cast<float2 *>(s_dyn);
    const int Nx = geo.Nx, Nh = Nx >> 1, slots = geo.tpc * Nh;
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nh : 0, q = valid ? slot % Nh : 0;
    const int base = t_loc * Nh;
    const int im = base + (q + Nh - 1) % Nh, ip = base + (q + 1) % Nh;
    const int i0 = 2 * q;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float dt = p.dt;
    const float w1 = c_theta[O::SX], w2 = c_theta[O::SX + 1], w3 = c_theta[O::SX + 2], D0 = c_theta[O::SX + 4];
    float2 u = make_float2(__ldg(p.u0 + (size_t)i0 * N + n), __ldg(p.u0 + (size_t)(i0 + 1) * N + n));
    int flip = 0;
    auto rhs = [&](float2 g, int zsel) {
        float2 *sU = sX + flip * slots;
        flip ^= 1;
        if (valid) sU[slot] = g;
        __syncthreads();
        const float gl = sU[im].y, gr = sU[ip].x;
        const float2 y = chain_value2<H, TM>(g, zsel);
        return make_float2(fmaf(D0, fmaf(w1, gl, fmaf(w2, g.x, w3 * g.y)), y.x), fmaf(D0, fmaf(w1, g.x, fmaf(w2, g.y, w3 * gr)), y.y));
    };
    auto store_int = [&](float *b, int row, float2 v) { if (live) *reinterpret_cast<float2 *>(&b[((size_t)row * N + n) * Nx + i0]) = v; };
    auto store_abi = [&](float *b, int row, float2 v) {
        if (live) { b[((size_t)row * Nx + i0) * N + n] = v.x; b[((size_t)row * Nx + i0 + 1) * N + n] = v.y; }
    };
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    const int S = c_rkc.s;
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
        const float2 F0 = rhs(u, 0);
        store_int(p.dense, s, F0);   // row s of the record = f(u_s): with u_s, u_{s+1}, f(u_{s+1}) the cubic-Hermite dense output
        float2 Y0 = u, Y1 = fma2(bc(c_rkc.mt1 * dt), F0, u);
#pragma unroll 1
        for (int j = 2; j <= S; ++j) {
            const float2 F = rhs(Y1, j);
            const float mu = c_rkc.mu[j], nu = c_rkc.nu[j], mt = c_rkc.mt[j], ga = c_rkc.ga[j];
            const float2 Y2 = fma2(bc(ga * dt), F0, fma2(bc(mt * dt), F, fma2(bc(nu), Y0, fma2(bc(mu), Y1, mul2(bc(1.0f - mu - nu), u)))));
            Y0 = Y1;
            Y1 = Y2;
        }
        u = Y1;
        store_int(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store_abi(p.out, isave, u); ++isave; }
    }
    store_int(p.dense, p.n_steps, rhs(u, 0));
    if (p.status) {
        __syncthreads();
        float *sU = s_dyn;
        if (valid) sU[slot] = ((fabsf(u.x) <= 3.0e38f) && (fabsf(u.y) <= 3.0e38f)) ? 0.0f : 1.0f;
        __syncthreads();
        if (live && q == 0) {
            float any = 0.0f;
            for (int r = 0; r < Nh; ++r) any += sU[base + r];
            p.status[n] = any > 0.0f ? 1 : 0;
        }
    }
}

template <int H>
struct __align__(16) WarpRows2 {
    static constexpr int LD = H + 4;
    float Q[64 * LD];   // q2 rows of the warp's 64 points (row = 2 * lane + point)
    float A[64 * LD];   // h1 rows
};

template <int H, int TM, bool RKC = false>
__global__ void __launch_bounds__(256) adjoint_kernel2(AdjParams p, Geom geo)
{
    using O = Off<H>;
    static_assert(H == 16, "the 2 x 4 lane tile below covers a 16 x 16 layer with 32 lanes");
    constexpr int P = O::P;
    constexpr int LD = WarpRows2<H>::LD;
    extern __shared__ __align__(16) float s_dyn[];
    const int Nx = geo.Nx, Nh = Nx >> 1, slots = geo.tpc * Nh;
    const int nwarp = blockDim.x >> 5;
    float4 *sX = reinterpret_cast<float4 *>(s_dyn);                        // [2][slots] (x0, x1, g0, g1), double buffered
    WarpRows2<H> *rows = reinterpret_cast<WarpRows2<H> *>(s_dyn + 8 * slots);
    const int slot = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpRows2<H> &wr = rows[warp];
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nh : 0, q = valid ? slot % Nh : 0;
    const int base = t_loc * Nh;
    const int im = base + (q + Nh - 1) % Nh, ip = base + (q + 1) % Nh;
    const int i0 = 2 * q;
    const int traj = blockIdx.x * geo.tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt, inv_dt = 1.0f / dt;
    const float w1 = c_theta[O::SX], w2 = c_theta[O::SX + 1], w3 = c_theta[O::SX + 2], D0 = c_theta[O::SX + 4];
    const int jt = lane >> 2, it = lane & 3;

    float2 acc[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) acc[r] = bc(0.0f);
    float a_w3[H], a_b2[H], a_w1[H], a_b1[H];
#pragma unroll
    for (int j = 0; j < H; ++j) { a_w3[j] = 0.f; a_b2[j] = 0.f; a_w1[j] = 0.f; a_b1[j] = 0.f; }
    float a_b3 = 0.f, a_s1 = 0.f, a_s2 = 0.f, a_s3 = 0.f, a_D0 = 0.f;

    float2 lam = bc(0.0f);
    float loss = 0.0f;
    auto ld2 = [&](const float *b, size_t row) { return __ldg(reinterpret_cast<const float2 *>(&b[(row * N + n) * Nx + i0])); };
    auto jump = [&](int isave) {
        const float c0 = __ldg(p.cot + ((size_t)isave * Nx + i0) * N + n), c1 = __ldg(p.cot + ((size_t)isave * Nx + i0 + 1) * N + n);   // ABI layout
        if (p.fused_l2) {
            const float2 us = ld2(p.ustep, (size_t)(isave * p.save_every));
            const float r0 = us.x - c0, r1 = us.y - c1;
            loss = fmaf(r0, r0, fmaf(r1, r1, loss));
            lam.x = fmaf(2.0f, r0, lam.x);
            lam.y = fmaf(2.0f, r1, lam.y);
        } else {
            lam.x += c0;
            lam.y += c1;
        }
    };
    const int n_save = p.n_steps / p.save_every + 1;
    jump(n_save - 1);
    int flip = 0;
    // One evaluation at state x (two adjacent grid points), cotangent g: returns kn = (df/du)^T g and accumulates the theta-gradient
    // terms with quadrature weight sc (isc = 1 / sc).
    auto eval_core = [&](float2 x, float2 g, float sc, float isc, int zsel) -> float2 {
        const int zb = lv32::c_zero[zsel & 7] << 2;
        float4 *sx = sX + flip * slots;
        flip ^= 1;
        if (valid) sx[slot] = make_float4(x.x, x.y, g.x, g.y);
        __syncthreads();
        const float4 nm = sx[im], np = sx[ip];   // left neighbour thread: its .y / .w border this thread's first point
        const float xl = nm.y, gl = nm.w, xr = np.x, gr = np.z;
        const float2 sg = mul2(bc(lv * sc), g);
        // ---- chain forward, activations kept ----
        float2 h1[H], v[H];
#pragma unroll
        for (int j4 = 0; j4 < H; j4 += 4) {
            const float4 w = ldw4(zb + O::W1 + j4), b = ldw4(zb + O::B1 + j4);
            h1[j4 + 0] = tanh2<TM>(fma2(bc(w.x), x, bc(b.x)));
            h1[j4 + 1] = tanh2<TM>(fma2(bc(w.y), x, bc(b.y)));
            h1[j4 + 2] = tanh2<TM>(fma2(bc(w.z), x, bc(b.z)));
            h1[j4 + 3] = tanh2<TM>(fma2(bc(w.w), x, bc(b.w)));
            *reinterpret_cast<float4 *>(&wr.A[(2 * lane) * LD + j4]) = make_float4(h1[j4].x, h1[j4 + 1].x, h1[j4 + 2].x, h1[j4 + 3].x);
            *reinterpret_cast<float4 *>(&wr.A[(2 * lane + 1) * LD + j4]) = make_float4(h1[j4].y, h1[j4 + 1].y, h1[j4 + 2].y, h1[j4 + 3].y);
        }
#pragma unroll
        for (int j4 = 0; j4 < H; j4 += 4) {
            const float4 b = ldw4(zb + O::B2 + j4);
            v[j4] = bc(b.x); v[j4 + 1] = bc(b.y); v[j4 + 2] = bc(b.z); v[j4 + 3] = bc(b.w);
        }
#pragma unroll
        for (int ii = 0; ii < H; ++ii) {
#pragma unroll
            for (int j4 = 0; j4 < H; j4 += 4) {
                const float4 w = ldw4(zb + O::W2 + ii * H + j4);
                v[j4 + 0] = fma2(bc(w.x), h1[ii], v[j4 + 0]);
                v[j4 + 1] = fma2(bc(w.y), h1[ii], v[j4 + 1]);
                v[j4 + 2] = fma2(bc(w.z), h1[ii], v[j4 + 2]);
                v[j4 + 3] = fma2(bc(w.w), h1[ii], v[j4 + 3]);
            }
        }
        a_b3 += sg.x + sg.y;
#pragma unroll
        for (int j4 = 0; j4 < H; j4 += 4) {
            const float4 w = ldw4(zb + O::W3 + j4);
            const float w_[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 h2 = tanh2<TM>(v[j4 + k]);
                a_w3[j4 + k] = fmaf(sg.x, h2.x, fmaf(sg.y, h2.y, a_w3[j4 + k]));
                v[j4 + k] = mul2(mul2(bc(w_[k]), sg), fma2(mul2(bc(-1.0f), h2), h2, bc(1.0f)));   // q2
                a_b2[j4 + k] += v[j4 + k].x + v[j4 + k].y;
            }
            *reinterpret_cast<float4 *>(&wr.Q[(2 * lane) * LD + j4]) = make_float4(v[j4].x, v[j4 + 1].x, v[j4 + 2].x, v[j4 + 3].x);
            *reinterpret_cast<float4 *>(&wr.Q[(2 * lane + 1) * LD + j4]) = make_float4(v[j4].y, v[j4 + 1].y, v[j4 + 2].y, v[j4 + 3].y);
        }
        __syncwarp();
        // ---- dW2 += q2 (x) h1 over the warp's 64 points ----
#pragma unroll 8
        for (int t = 0; t < 64; ++t) {
            const float2 qq = *reinterpret_cast<const float2 *>(&wr.Q[t * LD + 2 * jt]);
            const float4 hh = *reinterpret_cast<const float4 *>(&wr.A[t * LD + 4 * it]);
            const float2 h01 = make_float2(hh.x, hh.y), h23 = make_float2(hh.z, hh.w);
            acc[0] = fma2(bc(qq.x), h01, acc[0]);
            acc[1] = fma2(bc(qq.x), h23, acc[1]);
            acc[2] = fma2(bc(qq.y), h01, acc[2]);
            acc[3] = fma2(bc(qq.y), h23, acc[3]);
        }
        __syncwarp();
        // ---- q1 = (W2^T q2) * (1 - h1^2); first-layer gradients; dx ----
        float2 dxa = bc(0.0f), dxb = bc(0.0f);
#pragma unroll
        for (int ii = 0; ii < H; ++ii) {
            float2 s0 = bc(0.0f), s1 = bc(0.0f);
#pragma unroll
            for (int j4 = 0; j4 < H; j4 += 4) {
                const float4 w = ldw4(zb + O::W2 + ii * H + j4);
                s0 = fma2(bc(w.x), v[j4 + 0], s0);
                s1 = fma2(bc(w.y), v[j4 + 1], s1);
                s0 = fma2(bc(w.z), v[j4 + 2], s0);
                s1 = fma2(bc(w.w), v[j4 + 3], s1);
            }
            const float2 q1 = mul2(add2(s0, s1), fma2(mul2(bc(-1.0f), h1[ii]), h1[ii], bc(1.0f)));
            a_b1[ii] += q1.x + q1.y;
            a_w1[ii] = fmaf(q1.x, x.x, fmaf(q1.y, x.y, a_w1[ii]));
            const float wi = c_theta[zb + O::W1 + ii];
            if (ii & 1) dxb = fma2(bc(wi), q1, dxb);
            else dxa = fma2(bc(wi), q1, dxa);
        }
        const float2 dx = mul2(add2(dxa, dxb), bc(isc));
        // (J^T g)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
        const float2 kn = make_float2(dx.x + D0 * fmaf(w2, g.x, fmaf(w1, g.y, w3 * gl)), dx.y + D0 * fmaf(w2, g.y, fmaf(w1, gr, w3 * g.x)));
        // stencil-weight and D0 gradients: point 0 has neighbours (xl, x.y), point 1 has (x.x, xr)
        a_s1 = fmaf(sg.x * D0, xl, fmaf(sg.y * D0, x.x, a_s1));
        a_s2 = fmaf(sg.x * D0, x.x, fmaf(sg.y * D0, x.y, a_s2));
        a_s3 = fmaf(sg.x * D0, x.y, fmaf(sg.y * D0, xr, a_s3));
        a_D0 = fmaf(sg.x, fmaf(w1, xl, fmaf(w2, x.x, w3 * x.y)), fmaf(sg.y, fmaf(w1, x.x, fmaf(w2, x.y, w3 * xr)), a_D0));
        return kn;
    };

    if constexpr (!RKC) {
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        float2 kl[6];
#pragma unroll
        for (int j = 0; j < 6; ++j) kl[j] = bc(0.0f);
#pragma unroll 1
        for (int st = 0; st < 6; ++st) {
            float2 xa = bc(0.0f), ga = bc(0.0f);
            float sc, isc;
#define B200UDE_FKPP_PRE(I)                                                                                              \
    case I: {                                                                                                            \
        _Pragma("unroll") for (int j = 0; j < 7; ++j) if (Tsit5::bw(I, j) != 0.0)                                         \
            xa = fma2(bc((float)Tsit5::bw(I, j)), ld2(p.dense, (size_t)(s * 6 + j)), xa);                                 \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) ga = fma2(bc((float)Tsit5::a(I, j)), kl[j], ga); \
        sc = dt * (float)Tsit5::b(I);                                                                                    \
        isc = inv_dt * (float)(1.0 / Tsit5::b(I));                                                                       \
    } break;
            switch (st) {
                B200UDE_FKPP_PRE(0)
                B200UDE_FKPP_PRE(1)
                B200UDE_FKPP_PRE(2)
                B200UDE_FKPP_PRE(3)
                B200UDE_FKPP_PRE(4)
            default:
                B200UDE_FKPP_PRE(5)
            }
#undef B200UDE_FKPP_PRE
            const float2 x = fma2(bc(dt), xa, ld2(p.ustep, (size_t)s));
            const float2 g = fma2(bc(dt), ga, lam);
            const float2 kn = eval_core(x, g, sc, isc, st);
            switch (st) {
            case 0: kl[0] = kn; break;
            case 1: kl[1] = kn; break;
            case 2: kl[2] = kn; break;
            case 3: kl[3] = kn; break;
            case 4: kl[4] = kn; break;
            default: kl[5] = kn; break;
            }
        }
        float2 a = bc(0.0f);
#pragma unroll
        for (int j = 0; j < 6; ++j) a = fma2(bc((float)Tsit5::b(j)), kl[j], a);
        lam = fma2(bc(dt), a, lam);
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    } else {
    // ---- RKC2 forward solve: lambda is stepped backwards with RKC2 itself; u(t) = cubic Hermite on (u_n, f_n, u_{n+1}, f_{n+1})
    // (ustep rows n, n+1 and dense rows n, n+1 = f(u_n), f(u_{n+1})); stage k sits at t_{n+1} - c_k dt; the theta-gradient of the
    // step is dt sum_k w_k (df/dtheta)^T(x_k) Y_k (quadrature weights from the recurrence, see the oracle) ----
    const int S = c_rkc.s;
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        const float2 y0 = ld2(p.ustep, (size_t)s), y1 = ld2(p.ustep, (size_t)s + 1), f0 = ld2(p.dense, (size_t)s), f1 = ld2(p.dense, (size_t)s + 1);
        const float2 dy = add2(y1, mul2(bc(-1.0f), y0));
        float2 Y0 = lam, Y1 = lam, F0 = bc(0.0f);
#pragma unroll 1
        for (int j = 0; j < S; ++j) {
            const float Th = 1.0f - c_rkc.c[j];
            // x = (1 - Th) y0 + Th y1 + Th (Th - 1) ((1 - 2 Th) (y1 - y0) + (Th - 1) dt f0 + Th dt f1)
            const float2 inner = fma2(bc(1.0f - 2.0f * Th), dy, fma2(bc((Th - 1.0f) * dt), f0, mul2(bc(Th * dt), f1)));
            const float2 x = fma2(bc(Th * (Th - 1.0f)), inner, fma2(bc(Th), dy, y0));
            const float2 g = j == 0 ? lam : Y1;
            const float sc = dt * c_rkc.w[j], isc = 1.0f / sc;
            const float2 kn = eval_core(x, g, sc, isc, j);
            if (j == 0) {
                F0 = kn;
                Y0 = lam;
                Y1 = fma2(bc(c_rkc.mt1 * dt), F0, lam);
            } else {
                const float mu = c_rkc.mu[j + 1], nu = c_rkc.nu[j + 1], mt = c_rkc.mt[j + 1], ga = c_rkc.ga[j + 1];
                const float2 Y2 = fma2(bc(ga * dt), F0, fma2(bc(mt * dt), kn, fma2(bc(nu), Y0, fma2(bc(mu), Y1, mul2(bc(1.0f - mu - nu), lam)))));
                Y0 = Y1;
                Y1 = Y2;
            }
        }
        lam = Y1;
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    }
    if (p.grad_u0 && live) {
        p.grad_u0[(size_t)i0 * N + n] = lam.x;
        p.grad_u0[(size_t)(i0 + 1) * N + n] = lam.y;
    }

    // ---- reduction: lanes -> warp (fixed shuffle tree), warps -> CTA (fixed order) ----
    __syncthreads();
    float *gw = s_dyn + (size_t)warp * (P + 1);
    auto wsum = [&](float v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        return v;
    };
#pragma unroll
    for (int j = 0; j < H; ++j) {
        const float r0 = wsum(a_w1[j]), r1 = wsum(a_b1[j]), r2 = wsum(a_b2[j]), r3 = wsum(a_w3[j]);
        if (lane == 0) { gw[O::W1 + j] = r0; gw[O::B1 + j] = r1; gw[O::B2 + j] = r2; gw[O::W3 + j] = r3; }
    }
    {
        const float r0 = wsum(a_b3), r1 = wsum(a_s1), r2 = wsum(a_s2), r3 = wsum(a_s3), r4 = wsum(a_D0), r5 = wsum(loss * lv);
        if (lane == 0) {
            gw[O::B3] = r0; gw[O::SX] = r1; gw[O::SX + 1] = r2; gw[O::SX + 2] = r3; gw[O::SX + 3] = 0.0f; gw[O::SX + 4] = r4;
            gw[P] = r5;
        }
    }
    gw[O::W2 + (4 * it + 0) * H + 2 * jt] = acc[0].x;
    gw[O::W2 + (4 * it + 1) * H + 2 * jt] = acc[0].y;
    gw[O::W2 + (4 * it + 2) * H + 2 * jt] = acc[1].x;
    gw[O::W2 + (4 * it + 3) * H + 2 * jt] = acc[1].y;
    gw[O::W2 + (4 * it + 0) * H + 2 * jt + 1] = acc[2].x;
    gw[O::W2 + (4 * it + 1) * H + 2 * jt + 1] = acc[2].y;
    gw[O::W2 + (4 * it + 2) * H + 2 * jt + 1] = acc[3].x;
    gw[O::W2 + (4 * it + 3) * H + 2 * jt + 1] = acc[3].y;
    __syncthreads();
    float *dst = p.partial + (size_t)blockIdx.x * (P + 1);
    for (int e = threadIdx.x; e < P + 1; e += blockDim.x) {
        float tot = 0.0f;
        for (int w = 0; w < nwarp; ++w) tot += s_dyn[(size_t)w * (P + 1) + e];
        dst[e] = tot;
    }
}

}  // namespace fkpp
}  // namespace b200ude
