// lv32_tc.cuh -- tensor-core variant of the LV 2 -> 32 -> 32 -> 2 kernels (one trajectory per thread).
//
// The chain's 32 x 32 layer, evaluated for the 32 trajectories of a warp, is a [32 x 32] x [32 x 32] GEMM: 2 x 4 tiles of
// mma.sync.m16n8k8 (M = trajectories, N = output units, K = input units) per k-step.
// fp32 accuracy is kept with the 3xTF32 split  A_hi B_hi + A_lo B_hi + A_hi B_lo  (weights: hi = round-to-nearest
// TF32, lo = remainder, split once per launch; activations: the tensor core reads only the upper 19 bits of a tf32
// operand, so the value itself is the hi operand and lo = x - trunc(x)): 96 HMMA per warp and sweep instead of
// 1024 FFMAs per trajectory.
//   - every thread owns a trajectory and writes its 32-wide activation row into the warp's rows in shared memory; the
//     warp reads A fragments from those rows, B fragments from the staged weights (row stride 36 floats: conflict-free
//     fragment loads), and writes D back into the rows, from where each thread reads its own row again;
//   - a sweep is warp-collective (__syncwarp only): no CTA barrier inside the time loops of the fixed-step kernels.
// Kernels in this file: forward_kernel (fixed step), adaptive_forward_kernel (PI controller, saveat interpolation, step
// record), adjoint_kernel<GEMM, ADAPT, DISC> (interpolating adjoint on the fixed grid / replay of an adaptive solve /
// discrete adjoint; gradient GEMM on the FMA pipe or on mma.sync).
#pragma once
#include "lv32_packed.cuh"
#include "step_control.cuh"
#include "ude_adjoint.cuh"

namespace b200ude {
namespace lv32 {
namespace tc {

// round-to-nearest (ties away) to TF32's 10-bit mantissa == cvt.rna.tf32.f32, done with two integer ops on
// the ALU pipe (the cvt instruction issues on the XU pipe, which the tanh's MUFUs already load)
__device__ __forceinline__ float tf32_rna(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }

// defined with the gradient GEMM of the adjoint kernel below
__device__ __forceinline__ void mma_m16n8k8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]);
__device__ __forceinline__ void split_tf32(float x, uint32_t &hi, uint32_t &lo);

// D = A B for the 32 rows of the calling warp (3xTF32 mma.sync.m16n8k8; M = the warp's trajectories, N = NO output units,
// K = input units).  A: src[r * SA + k], r = 0..31.  B(k, n) = Bm[n * SB + k] (BT = false) or Bm[k * SB + n] (BT = true),
// given as the hi / lo split made at staging.  D goes to dst[r * SA + n]; dst may alias src (every A fragment is read
// before the first store).  Warp-collective; starts and ends with __syncwarp, so the rows may be written right before.
template <int K, int NO, int SA, int SB, bool BT>
__device__ __forceinline__ void warp_gemm(const float *src, float *dst, const float *Bhi, const float *Blo)
{
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    float d[2][NO / 8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NO / 8; ++nt)
#pragma unroll
            for (int q = 0; q < 4; ++q) d[mt][nt][q] = 0.0f;
    __syncwarp();
#pragma unroll
    for (int ks = 0; ks < K / 8; ++ks) {
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const float *r0 = src + (16 * mt + g) * SA + 8 * ks + t, *r1 = r0 + 8 * SA;
            split_tf32(r0[0], ah[mt][0], al[mt][0]);
            split_tf32(r1[0], ah[mt][1], al[mt][1]);
            split_tf32(r0[4], ah[mt][2], al[mt][2]);
            split_tf32(r1[4], ah[mt][3], al[mt][3]);
        }
#pragma unroll
        for (int nt = 0; nt < NO / 8; ++nt) {
            const int n = 8 * nt + g, k = 8 * ks + t;
            const int o0 = BT ? k * SB + n : n * SB + k, o1 = BT ? (k + 4) * SB + n : n * SB + k + 4;
            const uint32_t bh[2] = {__float_as_uint(Bhi[o0]), __float_as_uint(Bhi[o1])};
            const uint32_t bl[2] = {__float_as_uint(Blo[o0]), __float_as_uint(Blo[o1])};
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                mma_m16n8k8(d[mt][nt], al[mt], bh);
                mma_m16n8k8(d[mt][nt], ah[mt], bl);
                mma_m16n8k8(d[mt][nt], ah[mt], bh);
            }
        }
    }
    __syncwarp();
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NO / 8; ++nt) {
            float *o = dst + (16 * mt + g) * SA + 8 * nt + 2 * t;
            *reinterpret_cast<float2 *>(o) = make_float2(d[mt][nt][0], d[mt][nt][1]);
            *reinterpret_cast<float2 *>(o + 8 * SA) = make_float2(d[mt][nt][2], d[mt][nt][3]);
        }
    __syncwarp();
}

template <int NV>
__device__ __forceinline__ void store_row(float *row, const float (&v)[NV])
{
#pragma unroll
    for (int j = 0; j < NV; j += 4) *reinterpret_cast<float4 *>(row + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
}
template <int NV>
__device__ __forceinline__ void load_row(const float *row, float (&v)[NV])
{
#pragma unroll
    for (int j = 0; j < NV; j += 4) {
        const float4 q = *reinterpret_cast<const float4 *>(row + j);
        v[j] = q.x; v[j + 1] = q.y; v[j + 2] = q.z; v[j + 3] = q.w;
    }
}

constexpr int SW = 36;   // row stride (floats) of the staged W2 copies and of the activation rows: conflict-free fragment loads

// per-warp tensor-core context: the warp's 32 activation rows (row r belongs to lane r)
struct TcCtx {
    float *rows;
};
__device__ __forceinline__ TcCtx tc_ctx(float *cta_rows) { return TcCtx{cta_rows + (threadIdx.x >> 5) * 32 * SW}; }

// weights Wt[n][k] = B(k, n) at n * SW + k, hi / lo split.
// FWD orientation: n = output unit j, k = input unit i  ->  W2[j][i] = theta[OFF_W2 + i*32 + j]
// BWD orientation: n = input unit i,  k = output unit j ->  W2[j][i]   (for q1 = W2^T q2)
template <bool BWD>
__device__ __forceinline__ void stage_weights(const float *__restrict__ theta, float *sBhi, float *sBlo, int tid, int nthreads)
{
    for (int e = tid; e < 32 * 32; e += nthreads) {
        const int n = e >> 5, k = e & 31;
        const float x = BWD ? theta[OFF_W2 + n * 32 + k] : theta[OFF_W2 + k * 32 + n];
        const float hi = tf32_rna(x);
        sBhi[n * SW + k] = hi;
        sBlo[n * SW + k] = x - hi;
    }
}

// d = a W2^T (FWD weights) or a W2 (BWD weights) for this thread's row a, through the warp's rows
__device__ __forceinline__ void gemm_row32(const TcCtx &c, const float (&a)[32], const float *sBhi, const float *sBlo, float (&d)[32])
{
    float *row = c.rows + (threadIdx.x & 31) * SW;
    store_row(row, a);
    warp_gemm<32, 32, SW, SW, false>(c.rows, c.rows, sBhi, sBlo);
    load_row(row, d);
}

// ---- UDE right-hand side, one trajectory per thread, the 32x32 layer on the tensor core.  A real function
// (one copy in the instruction cache; the inlined 7-copy version was 106 KB and 32 % instruction-fetch stalled).
template <int TM>
__device__ __noinline__ float2 rhs_tc(TcCtx *cp, const float *sBhi, const float *sBlo, float x0, float x1, int zsel)
{
    const TcCtx c = *cp;
    const int zb = c_zero[zsel & 7] << 2;   // opaque zero: keeps the constant-bank loads inside the caller's loops
    float h[32], a2[32];
#pragma unroll
    for (int j4 = 0; j4 < 32; j4 += 4) {
        const float4 wb1 = ldw4(zb + OFF_B1 + j4), w10 = ldw4(zb + OFF_W1 + j4), w11 = ldw4(zb + OFF_W1 + H + j4);
        const float b_[4] = {wb1.x, wb1.y, wb1.z, wb1.w}, w0_[4] = {w10.x, w10.y, w10.z, w10.w}, w1_[4] = {w11.x, w11.y, w11.z, w11.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) h[j4 + k] = fmaf(w1_[k], x1, fmaf(w0_[k], x0, b_[k]));
        tanh_quad_s<TM>(h[j4], h[j4 + 1], h[j4 + 2], h[j4 + 3]);   // one reciprocal per four values (lv32_packed.cuh)
    }
    gemm_row32(c, h, sBhi, sBlo, a2);
    float y0 = c_theta[zb + OFF_B3], y1 = c_theta[zb + OFF_B3 + 1];
#pragma unroll
    for (int j4 = 0; j4 < 32; j4 += 4) {
        const float4 b2 = ldw4(zb + OFF_B2 + j4), w3a = ldw4(zb + OFF_W3 + 2 * j4), w3b = ldw4(zb + OFF_W3 + 2 * j4 + 4);
        const float b_[4] = {b2.x, b2.y, b2.z, b2.w};
        const float w3_[8] = {w3a.x, w3a.y, w3a.z, w3a.w, w3b.x, w3b.y, w3b.z, w3b.w};   // (w0j, w1j) pairs
#pragma unroll
        float v_[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) v_[k] = a2[j4 + k] + b_[k];
        tanh_quad_s<TM>(v_[0], v_[1], v_[2], v_[3]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            y0 = fmaf(w3_[2 * k], v_[k], y0);
            y1 = fmaf(w3_[2 * k + 1], v_[k], y1);
        }
    }
    // du1 = p1*u1 + NN1(u), du2 = -p4*u2 + NN2(u)   (scenario_1.jl:71-72)
    return make_float2(fmaf(c_consts[0], x0, y0), fmaf(-c_consts[1], x1, y1));
}

// ---- forward kernel: one trajectory per thread, 128 per CTA ------------------------------------------------
template <int TM, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) forward_kernel(FwdParams p)
{
    static_assert(BLOCK % 32 == 0, "whole warps: the 32 x 32 sweeps are warp-collective");
    __shared__ __align__(16) float sBhi[32 * SW], sBlo[32 * SW], sRows[BLOCK * SW];
    TcCtx c = tc_ctx(sRows);
    stage_weights<false>(p.theta, sBhi, sBlo, threadIdx.x, BLOCK);
    __syncthreads();

    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);   // padding threads shadow the last trajectory; stores masked
    const float dt = p.dt;
    float u0 = __ldg(p.u0 + n), u1 = __ldg(p.u0 + N + n);
    auto store2 = [&](float *base, int row, float v0, float v1) {
        if (live) {
            float *r0 = base + (size_t)row * 2 * N;
            r0[n] = v0;
            r0[N + n] = v1;
        }
    };
    store2(p.out, 0, u0, u1);
    store2(p.ustep, 0, u0, u1);
    float k0[7], k1[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) { k0[j] = 0.f; k1[j] = 0.f; }
    int isave = 1;
    // stage index runs 0..6 within a step; "stage 0" (k_1) is evaluated only for the very first step (FSAL afterwards)
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll 1
        for (int i = (s == 0 ? 0 : 1); i < 7; ++i) {
            float a0 = 0.0f, a1 = 0.0f;
#define B200UDE_FWD_COMB(I)                                                           \
    case I: {                                                                         \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) {    \
            a0 = fmaf((float)Tsit5::a(I, j), k0[j], a0);                              \
            a1 = fmaf((float)Tsit5::a(I, j), k1[j], a1);                              \
        }                                                                             \
    } break;
            switch (i) {
                B200UDE_FWD_COMB(1)
                B200UDE_FWD_COMB(2)
                B200UDE_FWD_COMB(3)
                B200UDE_FWD_COMB(4)
                B200UDE_FWD_COMB(5)
                B200UDE_FWD_COMB(6)
            default: break;
            }
#undef B200UDE_FWD_COMB
            const float g0 = fmaf(dt, a0, u0), g1 = fmaf(dt, a1, u1);
            if (i == 6) { u0 = g0; u1 = g1; }   // stage 7's argument is u_{n+1} (row 7 = b, FSAL)
            const float2 kk = rhs_tc<TM>(&c, sBhi, sBlo, g0, g1, i);
            switch (i) {
            case 0: k0[0] = kk.x; k1[0] = kk.y; break;
            case 1: k0[1] = kk.x; k1[1] = kk.y; break;
            case 2: k0[2] = kk.x; k1[2] = kk.y; break;
            case 3: k0[3] = kk.x; k1[3] = kk.y; break;
            case 4: k0[4] = kk.x; k1[4] = kk.y; break;
            case 5: k0[5] = kk.x; k1[5] = kk.y; break;
            default: k0[6] = kk.x; k1[6] = kk.y; break;
            }
            store2(p.dense, s * 6 + i, kk.x, kk.y);   // row (s+1)*6 for i = 6: k_7(s) = k_1(s+1)
        }
        store2(p.ustep, s + 1, u0, u1);
        if ((s + 1) % p.save_every == 0) {
            store2(p.out, isave, u0, u1);
            ++isave;
        }
        k0[0] = k0[6];
        k1[0] = k1[6];
    }
    if (p.status && live) p.status[n] = ((fabsf(u0) <= 3.0e38f) && (fabsf(u1) <= 3.0e38f)) ? 0 : 1;   // false for NaN/Inf
}

// ---- adaptive forward kernel (abstol / reltol; scenario_1.jl:84-85, seir_exposure.jl:138-139 style calls) --------------
// Tsit5 with OrdinaryDiffEq's PI controller and initial-step heuristic per trajectory (PIControl, step_control.cuh; the
// oracle's ude_solve_adaptive), saveat by the free interpolant, and the record of
// accepted steps (tgrid, ustep, the stage derivatives) that the replay adjoint reads.  The 32 x 32 sweeps are CTA-collective,
// so the attempt loop is CTA-uniform: a trajectory that has reached the end keeps evaluating (results discarded) until the
// slowest of the CTA's 128 trajectories is done.
template <int TM, int BLOCK, int MINB>
__global__ void __launch_bounds__(BLOCK, MINB) adaptive_forward_kernel(FwdParams p, AdaptiveGrid ag)
{
    static_assert(BLOCK % 32 == 0, "whole warps: the 32 x 32 sweeps are warp-collective");
    __shared__ __align__(16) float sBhi[32 * SW], sBlo[32 * SW], sRows[BLOCK * SW];
    TcCtx c = tc_ctx(sRows);
    stage_weights<false>(p.theta, sBhi, sBlo, threadIdx.x, BLOCK);
    __syncthreads();

    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);   // padding threads shadow the last trajectory; stores masked
    const float t0 = ag.t0, t1 = ag.t0 + ag.save_dt * (float)(ag.n_save - 1);
    const float abstol = ag.abstol, reltol = ag.reltol;
    float u0 = __ldg(p.u0 + n), u1 = __ldg(p.u0 + N + n);
    auto store2 = [&](float *base, int row, float v0, float v1) {
        if (live) {
            float *r0 = base + (size_t)row * 2 * N;
            r0[n] = v0;
            r0[N + n] = v1;
        }
    };
    store2(p.out, 0, u0, u1);
    store2(p.ustep, 0, u0, u1);
    if (live) ag.tgrid[n] = t0;
    float k0[7], k1[7];
#pragma unroll
    for (int j = 0; j < 7; ++j) { k0[j] = 0.f; k1[j] = 0.f; }
    PIControl<float, 5> pi;
    {
        const float2 kk = rhs_tc<TM>(&c, sBhi, sBlo, u0, u1, 0);
        k0[0] = kk.x; k1[0] = kk.y;
    }
    store2(p.dense, 0, k0[0], k1[0]);
    // initial step: Hairer-Norsett-Wanner as in OrdinaryDiffEq
    {
        const float s0 = abstol + reltol * fabsf(u0), s1 = abstol + reltol * fabsf(u1);
        float d0 = Prec<float>::sq(0.5f * ((u0 / s0) * (u0 / s0) + (u1 / s1) * (u1 / s1)));
        float d1 = Prec<float>::sq(0.5f * ((k0[0] / s0) * (k0[0] / s0) + (k1[0] / s1) * (k1[0] / s1)));
        const float dt0 = pi.hnw_dt0(d0, d1, t1 - t0);
        const float2 f1 = rhs_tc<TM>(&c, sBhi, sBlo, fmaf(dt0, k0[0], u0), fmaf(dt0, k1[0], u1), 1);
        const float e0 = (f1.x - k0[0]) / s0, e1 = (f1.y - k1[0]) / s1;
        const float d2 = Prec<float>::sq(0.5f * (e0 * e0 + e1 * e1)) / dt0;
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
        float un0 = u0, un1 = u1;
#pragma unroll 1
        for (int i = 1; i < 7; ++i) {
            float a0 = 0.0f, a1 = 0.0f;
#define B200UDE_FWD_COMB(I)                                                           \
    case I: {                                                                         \
        _Pragma("unroll") for (int j = 0; j < I; ++j) if (Tsit5::a(I, j) != 0.0) {    \
            a0 = fmaf((float)Tsit5::a(I, j), k0[j], a0);                              \
            a1 = fmaf((float)Tsit5::a(I, j), k1[j], a1);                              \
        }                                                                             \
    } break;
            switch (i) {
                B200UDE_FWD_COMB(1)
                B200UDE_FWD_COMB(2)
                B200UDE_FWD_COMB(3)
                B200UDE_FWD_COMB(4)
                B200UDE_FWD_COMB(5)
            default:
                B200UDE_FWD_COMB(6)
            }
#undef B200UDE_FWD_COMB
            const float g0 = fmaf(h, a0, u0), g1 = fmaf(h, a1, u1);
            if (i == 6) { un0 = g0; un1 = g1; }
            const float2 kk = rhs_tc<TM>(&c, sBhi, sBlo, g0, g1, i);
            switch (i) {
            case 1: k0[1] = kk.x; k1[1] = kk.y; break;
            case 2: k0[2] = kk.x; k1[2] = kk.y; break;
            case 3: k0[3] = kk.x; k1[3] = kk.y; break;
            case 4: k0[4] = kk.x; k1[4] = kk.y; break;
            case 5: k0[5] = kk.x; k1[5] = kk.y; break;
            default: k0[6] = kk.x; k1[6] = kk.y; break;
            }
        }
        if (active) {
            float e0 = 0.0f, e1 = 0.0f;
#pragma unroll
            for (int j = 0; j < 7; ++j) { e0 = fmaf((float)Tsit5::bt(j), k0[j], e0); e1 = fmaf((float)Tsit5::bt(j), k1[j], e1); }
            e0 *= h; e1 *= h;
            const float c0 = abstol + reltol * fmaxf(fabsf(u0), fabsf(un0)), c1 = abstol + reltol * fmaxf(fabsf(u1), fabsf(un1));
            const float EEst = Prec<float>::sq(0.5f * ((e0 / c0) * (e0 / c0) + (e1 / c1) * (e1 / c1)));
            if (!(EEst <= Prec<float>::huge)) {
                bad = 1;   // NaN / Inf
            } else {
                if (pi.judge(EEst)) {
                    if (nacc >= ag.max_steps) {
                        bad = 2;
                    } else {
                        const float tn = clipped ? t1 : t + h;
                        // dense record of this step: k_1..k_6 at rows nacc*6 + i (k_1 is already there), k_7 at (nacc+1)*6
#define B200UDE_ST(I) store2(p.dense, nacc * 6 + I, k0[I], k1[I]);
                        B200UDE_ST(1) B200UDE_ST(2) B200UDE_ST(3) B200UDE_ST(4) B200UDE_ST(5) B200UDE_ST(6)
#undef B200UDE_ST
                        while (isave < ag.n_save) {
                            const float ts = t0 + ag.save_dt * (float)isave;
                            if (ts > tn + Prec<float>::clip * fabsf(tn)) break;
                            float bw[7];
                            Tsit5::weights(fminf((ts - t) / h, 1.0f), bw);
                            float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
                            for (int j = 0; j < 7; ++j) { a0 = fmaf(bw[j], k0[j], a0); a1 = fmaf(bw[j], k1[j], a1); }
                            store2(p.out, isave, fmaf(h, a0, u0), fmaf(h, a1, u1));
                            ++isave;
                        }
                        pi.accept(EEst, h, clipped);
                        t = tn;
                        ++nacc;
                        if (live) ag.tgrid[(size_t)nacc * N + n] = t;
                        u0 = un0; u1 = un1;
                        k0[0] = k0[6]; k1[0] = k1[6];
                        store2(p.ustep, nacc, u0, u1);
                    }
                } else {
                    pi.reject(h);
                }
            }
        }
    }
    if (bad) {   // failed solve: the unreached save points are NaN
        for (int is = isave; is < ag.n_save; ++is) store2(p.out, is, Prec<float>::nan(), Prec<float>::nan());
    }
    if (live) ag.nacc[n] = nacc;
    if (p.status && live) {
        const bool ok = (fabsf(u0) <= Prec<float>::huge) && (fabsf(u1) <= Prec<float>::huge);
        p.status[n] = bad == 2 ? 2 : ((bad || !ok) ? 1 : 0);
    }
}

// ---- adjoint kernel: one trajectory per thread, 128 per CTA; the two 32x32 sweeps of every backward stage
// (chain forward and W2^T q2) run on the tensor core; the ensemble-summed parameter gradient is a per-warp GEMM over
// the warp's 32 trajectories (FFMA or mma.sync), run before the second sweep overwrites the staged q2 rows. ----
constexpr int SLD = 36;   // staged row stride (floats): 32 + 4 -> conflict-free 128-bit row stores and tile loads
struct __align__(16) WarpStageT {
    float B1[32 * SLD];   // h2 rows, then q2 rows, then q1 rows   [lane][j]
    float B2[32 * SLD];   // h1 rows                                [lane][i]
    float SG[32 * 2];     // scaled, masked chain-output cotangent  [lane][m]
    float U[32 * 2];      // chain input                            [lane][m]
};

// warp-level m16n8k8 TF32 MMA (legacy tensor-core path), D += A B
__device__ __forceinline__ void mma_m16n8k8(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2])
{
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// 3xTF32 operand split for mma.sync: the tensor core reads only the upper 19 bits of a .tf32 operand register (the low 13
// mantissa bits are ignored), so the fp32 value itself serves as the "hi" operand (= its truncation) and only the residual
// lo = x - trunc(x) has to be formed: one LOP + one FADD per element.  (B200UDE_TF32_RNA_SPLIT: explicit round-to-nearest hi.)
__device__ __forceinline__ void split_tf32(float x, uint32_t &hi, uint32_t &lo)
{
#ifdef B200UDE_TF32_RNA_SPLIT
    const float h = tf32_rna(x);
    hi = __float_as_uint(h);
    lo = __float_as_uint(x - h);
#else
    hi = __float_as_uint(x);
    lo = __float_as_uint(x - __uint_as_float(hi & 0xFFFFE000u));
#endif
}

// Running sums kept in a per-thread row of shared memory (stride 33 words: conflict-free): sum += m with ordinary
// round-to-nearest adds, m = 0.  The tensor core adds into its accumulator with truncation, so a long mma accumulation
// chain drifts (2.4e-5 relative on dW2 after the 2160 MMAs of a whole backward solve); short chains flushed through this
// keep the error at the FFMA level without spending 32 more registers.
__device__ __forceinline__ void flush32(float *sum, float (&m)[32], bool first)
{
#pragma unroll
    for (int q = 0; q < 32; ++q) {
        sum[q] = first ? m[q] : sum[q] + m[q];
        m[q] = 0.0f;
    }
}

// GEMM = 0: the per-warp gradient GEMM dW2 += q2 (x) h1 on the FMA pipe (FFMA, 8 x 4 register tile per lane);
// GEMM = 1: the same product as 3xTF32 warp-level mma.sync.m16n8k8 (M = j, N = i, K = the warp's 32 trajectories):
//           fragments are read straight from the staged rows; the contraction index inside a k-step is permuted
//           (k = tig -> t = 2 tig, k = tig + 4 -> t = 2 tig + 1) so that every fragment load is bank-conflict free.
// DISC: discrete adjoint (exact gradient of the fixed-step scheme, ude_adjoint.cuh) instead of the interpolating adjoint.
template <int TM, int BLOCK, int MINB, int GEMM, bool ADAPT = false, bool DISC = false>
__global__ void __launch_bounds__(BLOCK, MINB) adjoint_kernel(AdjParams p, AdaptiveGrid ag)
{
    static_assert(BLOCK == 128, "four warps: the partial-gradient rows are laid out as blockIdx.x * 4 + warp");
    __shared__ __align__(16) float sWf_hi[32 * SW], sWf_lo[32 * SW], sWb_hi[32 * SW], sWb_lo[32 * SW];
    __shared__ float s_sum[GEMM == 1 ? BLOCK * 33 : 1];   // running dW2 sums of the mma.sync gradient GEMM (flush32)
    extern __shared__ __align__(16) unsigned char s_raw[];
    stage_weights<false>(p.theta, sWf_hi, sWf_lo, threadIdx.x, BLOCK);
    stage_weights<true>(p.theta, sWb_hi, sWb_lo, threadIdx.x, BLOCK);
    __syncthreads();

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int jt = lane >> 3, it = lane & 7;
    WarpStageT *st = reinterpret_cast<WarpStageT *>(s_raw) + warp;
    float *const rowB1 = st->B1 + lane * SLD, *const rowB2 = st->B2 + lane * SLD;
    const size_t N = (size_t)p.N;
    const int gid = blockIdx.x * BLOCK + threadIdx.x;
    const bool live = gid < p.N;
    const size_t n = live ? (size_t)gid : (size_t)(p.N - 1);
    const float lv = live ? 1.0f : 0.0f;   // padding trajectories: zero mask on their cotangents
    const float dt = p.dt, inv_dt = 1.0f / dt;
    const float p1 = c_consts[0], p4 = c_consts[1];

    // gradient accumulators: dW2 tile (jt*8 + jj, it*4 + {0,1},{2,3}) packed along i; thin layers as lane-owned columns
    float2 acc[16];
#pragma unroll
    for (int q = 0; q < 16; ++q) acc[q] = bc(0.0f);
    float macc[32];   // GEMM = 1: C fragments of the 2 x 4 (j x i) tiles, tile (mt, nt) at 16 mt + 4 nt
#pragma unroll
    for (int q = 0; q < 32; ++q) macc[q] = 0.0f;
    const int fg = lane >> 2, tig = lane & 3;   // mma fragment coordinates (groupID, threadID_in_group)
    float g_w30 = 0.f, g_w31 = 0.f, g_b30 = 0.f, g_b31 = 0.f, g_b2 = 0.f, g_b1 = 0.f, g_w10 = 0.f, g_w11 = 0.f;

    float lam[2] = {0.0f, 0.0f};
    float loss = 0.0f;
    const int n_save = p.n_steps / p.save_every + 1;
    bool first_flush = true;
    float *const sum_row = s_sum + (GEMM == 1 ? threadIdx.x * 33 : 0);

    // One evaluation of (df/du)^T g and of the theta-gradient quadrature term at state x, stage argument g:
    // sc = quadrature weight (h b_i), isc = 1 / sc (0 for a masked lane), lvm = 0/1 mask.  Returns kn = (df/du)^T g.
    auto eval_core = [&](int stage, const float (&x)[2], const float (&g)[2], float sc, float isc, float lvm, float &kn0, float &kn1) {
        const int zb = c_zero[stage] << 2;
        const float sg0 = lvm * sc * g[0], sg1 = lvm * sc * g[1];
        *reinterpret_cast<float2 *>(&st->SG[lane * 2]) = make_float2(sg0, sg1);
        *reinterpret_cast<float2 *>(&st->U[lane * 2]) = make_float2(x[0], x[1]);

        // ---- chain forward: layer 1 on the FMA pipe, layer 2 on the tensor core ----
        float v[32];
#pragma unroll
        for (int j4 = 0; j4 < 32; j4 += 4) {
            const float4 wb1 = ldw4(zb + OFF_B1 + j4), w10 = ldw4(zb + OFF_W1 + j4), w11 = ldw4(zb + OFF_W1 + H + j4);
            const float b_[4] = {wb1.x, wb1.y, wb1.z, wb1.w}, w0_[4] = {w10.x, w10.y, w10.z, w10.w}, w1_[4] = {w11.x, w11.y, w11.z, w11.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) v[j4 + k] = fmaf(w1_[k], x[1], fmaf(w0_[k], x[0], b_[k]));
            tanh_quad_s<TM>(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);
            *reinterpret_cast<float4 *>(rowB2 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // h1 row
        }
        warp_gemm<32, 32, SLD, SW, false>(st->B2, st->B1, sWf_hi, sWf_lo);
        load_row(rowB1, v);  // v = W2 h1
        // h2 = tanh(. + b2) -> B1 row;  q2 = (W3^T sg) * (1 - h2^2) stays in v
#pragma unroll
        for (int j4 = 0; j4 < 32; j4 += 4) {
            const float4 b2 = ldw4(zb + OFF_B2 + j4), w3a = ldw4(zb + OFF_W3 + 2 * j4), w3b = ldw4(zb + OFF_W3 + 2 * j4 + 4);
            const float b_[4] = {b2.x, b2.y, b2.z, b2.w};
            const float w3_[8] = {w3a.x, w3a.y, w3a.z, w3a.w, w3b.x, w3b.y, w3b.z, w3b.w};
            float h2[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) h2[k] = v[j4 + k] + b_[k];
            tanh_quad_s<TM>(h2[0], h2[1], h2[2], h2[3]);
#pragma unroll
            for (int k = 0; k < 4; ++k) v[j4 + k] = fmaf(w3_[2 * k + 1], sg1, w3_[2 * k] * sg0) * fmaf(-h2[k], h2[k], 1.0f);
            *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(h2[0], h2[1], h2[2], h2[3]);
        }
        __syncwarp();
        // thin pass A: lane j owns output-layer column j: dW3[m][j] += sum_t SG[t][m] h2[t][j]; db3
#pragma unroll 8
        for (int t = 0; t < 32; ++t) {
            const float hh = st->B1[t * SLD + lane];
            const float2 s2 = *reinterpret_cast<const float2 *>(&st->SG[t * 2]);
            g_w30 = fmaf(s2.x, hh, g_w30);
            g_w31 = fmaf(s2.y, hh, g_w31);
            g_b30 += s2.x;
            g_b31 += s2.y;
        }
        __syncwarp();
#pragma unroll
        for (int j4 = 0; j4 < 32; j4 += 4) *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // q2 row
        // ---- gradient GEMM of this warp, then W2^T q2 on the tensor core (in place over the q2 rows) ----
        __syncwarp();
        if constexpr (GEMM == 1) {
#pragma unroll
            for (int ks = 0; ks < 4; ++ks) {
                const float *q0 = st->B1 + (8 * ks + 2 * tig) * SLD + fg, *q1 = q0 + SLD;
                const float *h0 = st->B2 + (8 * ks + 2 * tig) * SLD + fg, *h1r = h0 + SLD;
                uint32_t ah[2][4], al[2][4], bh[4][2], bl[4][2];
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) {
                    split_tf32(q0[16 * mt], ah[mt][0], al[mt][0]);
                    split_tf32(q0[16 * mt + 8], ah[mt][1], al[mt][1]);
                    split_tf32(q1[16 * mt], ah[mt][2], al[mt][2]);
                    split_tf32(q1[16 * mt + 8], ah[mt][3], al[mt][3]);
                }
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) {
                    split_tf32(h0[8 * nt], bh[nt][0], bl[nt][0]);
                    split_tf32(h1r[8 * nt], bh[nt][1], bl[nt][1]);
                }
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int nt = 0; nt < 4; ++nt) {
                        float (&cf)[4] = *reinterpret_cast<float (*)[4]>(&macc[16 * mt + 4 * nt]);
                        mma_m16n8k8(cf, al[mt], bh[nt]);
                        mma_m16n8k8(cf, ah[mt], bl[nt]);
                        mma_m16n8k8(cf, ah[mt], bh[nt]);
                    }
            }
#pragma unroll 8
            for (int t = 0; t < 32; ++t) g_b2 += st->B1[t * SLD + lane];
        } else {
            float4 G0[2], G1[2], Hh[2];
            float qc[2];
            auto load_row = [&](int t, int b) {
                const float *r1 = st->B1 + t * SLD, *r2 = st->B2 + t * SLD;
                G0[b] = *reinterpret_cast<const float4 *>(r1 + jt * 8);
                G1[b] = *reinterpret_cast<const float4 *>(r1 + jt * 8 + 4);
                Hh[b] = *reinterpret_cast<const float4 *>(r2 + it * 4);
                qc[b] = r1[lane];
            };
            auto use_row = [&](int b) {
                const float gj[8] = {G0[b].x, G0[b].y, G0[b].z, G0[b].w, G1[b].x, G1[b].y, G1[b].z, G1[b].w};
                const float2 h01 = make_float2(Hh[b].x, Hh[b].y), h23 = make_float2(Hh[b].z, Hh[b].w);
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                    acc[2 * jj] = fma2(bc(gj[jj]), h01, acc[2 * jj]);
                    acc[2 * jj + 1] = fma2(bc(gj[jj]), h23, acc[2 * jj + 1]);
                }
                g_b2 += qc[b];
            };
            load_row(0, 0);
#pragma unroll 1
            for (int t = 0; t < 32; t += 2) {
                load_row(t + 1, 1);
                use_row(0);
                if (t + 2 < 32) load_row(t + 2, 0);
                use_row(1);
            }
        }
        warp_gemm<32, 32, SLD, SW, false>(st->B1, st->B1, sWb_hi, sWb_lo);
        load_row(rowB1, v);  // v = W2^T q2
        // q1 = v * (1 - h1^2) (h1 re-read from this lane's own row), (df/du)^T g
        float dx0 = 0.0f, dx1 = 0.0f;
        __syncwarp();        // all lanes are done reading B2 rows in the GEMM pass before q1 overwrites B1
#pragma unroll
        for (int j4 = 0; j4 < 32; j4 += 4) {
            const float4 hh = *reinterpret_cast<const float4 *>(rowB2 + j4);
            const float4 wx0 = ldw4(zb + OFF_W1 + j4), wx1 = ldw4(zb + OFF_W1 + H + j4);
            const float h_[4] = {hh.x, hh.y, hh.z, hh.w}, wx0_[4] = {wx0.x, wx0.y, wx0.z, wx0.w}, wx1_[4] = {wx1.x, wx1.y, wx1.z, wx1.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                v[j4 + k] *= fmaf(-h_[k], h_[k], 1.0f);
                dx0 = fmaf(wx0_[k], v[j4 + k], dx0);
                dx1 = fmaf(wx1_[k], v[j4 + k], dx1);
            }
            *reinterpret_cast<float4 *>(rowB1 + j4) = make_float4(v[j4], v[j4 + 1], v[j4 + 2], v[j4 + 3]);   // q1 row
        }
        kn0 = fmaf(p1, g[0], dx0 * isc);
        kn1 = fmaf(-p4, g[1], dx1 * isc);   // LV physics: diag(p1, -p4)
        __syncwarp();
        // thin pass B: lane i owns input-layer row i: dW1[i][m] += sum_t q1[t][i] x[t][m]; db1
#pragma unroll 8
        for (int t = 0; t < 32; ++t) {
            const float qq = st->B1[t * SLD + lane];
            const float2 u2 = *reinterpret_cast<const float2 *>(&st->U[t * 2]);
            g_b1 += qq;
            g_w10 = fmaf(qq, u2.x, g_w10);
            g_w11 = fmaf(qq, u2.y, g_w11);
        }
        __syncwarp();
    };

    if constexpr (!ADAPT) {
    loss_jump<2>(p, n_save - 1, n, N, lam, loss);
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        float kl[6][2];
#pragma unroll
        for (int j = 0; j < 6; ++j) { kl[j][0] = 0.f; kl[j][1] = 0.f; }
#pragma unroll 1
        for (int it6 = 0; it6 < 6; ++it6) {
            const int stage = DISC ? 5 - it6 : it6;   // the discrete adjoint walks the forward stages backwards
            float x[2], g[2], sc, isc;
#define B200UDE_TC_STAGE_PRE(I)                                    \
    case I: {                                                      \
        if constexpr (DISC) {                                      \
            fwd_stage_state<2, I>(p, s, n, N, dt, x);              \
            disc_stage_cot<2, I>(lam, kl, dt, g);                  \
            sc = 1.0f;                                             \
            isc = 1.0f;                                            \
        } else {                                                   \
            interp_state<2, I>(p, s, n, N, dt, x);                 \
            stage_arg<2, I>(lam, kl, dt, g);                       \
            sc = dt * (float)Tsit5::b(I);                          \
            isc = inv_dt * (float)(1.0 / Tsit5::b(I));             \
        }                                                          \
    } break;
            switch (stage) {
                B200UDE_TC_STAGE_PRE(0)
                B200UDE_TC_STAGE_PRE(1)
                B200UDE_TC_STAGE_PRE(2)
                B200UDE_TC_STAGE_PRE(3)
                B200UDE_TC_STAGE_PRE(4)
            default:
                B200UDE_TC_STAGE_PRE(5)
            }
#undef B200UDE_TC_STAGE_PRE
            float kn0, kn1;
            eval_core(stage, x, g, sc, isc, lv, kn0, kn1);
            switch (stage) {
            case 0: kl[0][0] = kn0; kl[0][1] = kn1; break;
            case 1: kl[1][0] = kn0; kl[1][1] = kn1; break;
            case 2: kl[2][0] = kn0; kl[2][1] = kn1; break;
            case 3: kl[3][0] = kn0; kl[3][1] = kn1; break;
            case 4: kl[4][0] = kn0; kl[4][1] = kn1; break;
            default: kl[5][0] = kn0; kl[5][1] = kn1; break;
            }
        }
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
            if constexpr (DISC) {
                float a = lam[cc];
#pragma unroll
                for (int j = 0; j < 6; ++j) a += kl[j][cc];
                lam[cc] = a;
            } else {
                float a = 0.0f;
#pragma unroll
                for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j][cc], a);
                lam[cc] = fmaf(dt, a, lam[cc]);
            }
        }
        if (s % p.save_every == 0) loss_jump<2>(p, s / p.save_every, n, N, lam, loss);
        if constexpr (GEMM == 1) { flush32(sum_row, macc, first_flush); first_flush = false; }   // per step: 72-MMA chains
    }
    } else {
    // ---- adaptive: replay the accepted forward steps backwards, split at the save times where the loss cotangent jumps in
    // (same algorithm as generic::adaptive_adjoint_kernel; loops are CTA-uniform because the sweeps are CTA-collective) ----
    __shared__ int s_nmax;
    if (threadIdx.x == 0) s_nmax = 0;
    __syncthreads();
    const int nacc = ag.nacc[n];
    atomicMax(&s_nmax, live ? nacc : 0);
    __syncthreads();
    const int nmax = s_nmax;
    int isave = ag.n_save - 1;
    auto jump = [&](int is) {
        lam[0] += __ldg(p.cot + ((size_t)is * 2 + 0) * N + n);
        lam[1] += __ldg(p.cot + ((size_t)is * 2 + 1) * N + n);
    };
    if (live) jump(isave);
    --isave;
#pragma unroll 1
    for (int s = nmax - 1; s >= 0; --s) {
        const bool act_s = live && s < nacc;
        const int sc_ = act_s ? s : 0;   // inactive lanes shadow step 0 (finite data), weight 0
        const float tn = ag.tgrid[(size_t)sc_ * N + n], tn1 = ag.tgrid[(size_t)(sc_ + 1) * N + n], hn = tn1 - tn;
        const float eps = 1e-5f * hn, inv_hn = 1.0f / hn;
        const float un0 = __ldg(p.ustep + ((size_t)sc_ * 2 + 0) * N + n), un1 = __ldg(p.ustep + ((size_t)sc_ * 2 + 1) * N + n);
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
            float kl[6][2];
#pragma unroll
            for (int j = 0; j < 6; ++j) { kl[j][0] = 0.f; kl[j][1] = 0.f; }
#pragma unroll 1
            for (int stage = 0; stage < 6; ++stage) {
                float x[2], g[2], sc, isc, ci;
#define B200UDE_TC_STAGE_PRE(I)                                    \
    case I: {                                                      \
        stage_arg<2, I>(lam, kl, h, g);                            \
        sc = h * (float)Tsit5::b(I);                               \
        isc = inv_h * (float)(1.0 / Tsit5::b(I));                  \
        ci = (float)Tsit5::c(I);                                   \
    } break;
                switch (stage) {
                    B200UDE_TC_STAGE_PRE(0)
                    B200UDE_TC_STAGE_PRE(1)
                    B200UDE_TC_STAGE_PRE(2)
                    B200UDE_TC_STAGE_PRE(3)
                    B200UDE_TC_STAGE_PRE(4)
                default:
                    B200UDE_TC_STAGE_PRE(5)
                }
#undef B200UDE_TC_STAGE_PRE
                {   // u at time cur - c_i h from the dense output of forward step sc_ (free 4th-order interpolant)
                    const float Th = fminf(fmaxf((cur - ci * h - tn) * inv_hn, 0.0f), 1.0f);
                    float bw[7];
                    Tsit5::weights(Th, bw);
                    float a0 = 0.0f, a1 = 0.0f;
#pragma unroll
                    for (int j = 0; j < 7; ++j) {
                        a0 = fmaf(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * 2 + 0) * N + n), a0);
                        a1 = fmaf(bw[j], __ldg(p.dense + ((size_t)(sc_ * 6 + j) * 2 + 1) * N + n), a1);
                    }
                    x[0] = fmaf(hn, a0, un0);
                    x[1] = fmaf(hn, a1, un1);
                }
                float kn0, kn1;
                eval_core(stage, x, g, sc, isc, lvm, kn0, kn1);
                switch (stage) {
                case 0: kl[0][0] = kn0; kl[0][1] = kn1; break;
                case 1: kl[1][0] = kn0; kl[1][1] = kn1; break;
                case 2: kl[2][0] = kn0; kl[2][1] = kn1; break;
                case 3: kl[3][0] = kn0; kl[3][1] = kn1; break;
                case 4: kl[4][0] = kn0; kl[4][1] = kn1; break;
                default: kl[5][0] = kn0; kl[5][1] = kn1; break;
                }
            }
            if (has) {
#pragma unroll
                for (int cc = 0; cc < 2; ++cc) {
                    float a = 0.0f;
#pragma unroll
                    for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j][cc], a);
                    lam[cc] = fmaf(h, a, lam[cc]);
                }
                cur = ta;
                if (isave >= 0 && fabsf(ts - ta) <= eps) { jump(isave); --isave; }
            }
            if constexpr (GEMM == 1) { flush32(sum_row, macc, first_flush); first_flush = false; }
        }
    }
    if constexpr (GEMM == 1) {
        if (first_flush) flush32(sum_row, macc, true);   // no accepted step at all: the sums are zero
    }
    }
    if (p.grad_u0 && live) {
        p.grad_u0[n] = lam[0];
        p.grad_u0[N + n] = lam[1];
    }
    loss *= lv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    // this warp's partial gradient
    float *dst = p.partial + ((size_t)blockIdx.x * 4 + warp) * (P + 1);
    if constexpr (GEMM == 1) {
#pragma unroll
        for (int q = 0; q < 32; ++q) macc[q] = sum_row[q];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int j = 16 * mt + fg, i = 8 * nt + 2 * tig;
                dst[OFF_W2 + i * H + j] = macc[16 * mt + 4 * nt + 0];
                dst[OFF_W2 + (i + 1) * H + j] = macc[16 * mt + 4 * nt + 1];
                dst[OFF_W2 + i * H + j + 8] = macc[16 * mt + 4 * nt + 2];
                dst[OFF_W2 + (i + 1) * H + j + 8] = macc[16 * mt + 4 * nt + 3];
            }
    } else {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            dst[OFF_W2 + (it * 4 + 0) * H + (jt * 8 + jj)] = acc[2 * jj].x;
            dst[OFF_W2 + (it * 4 + 1) * H + (jt * 8 + jj)] = acc[2 * jj].y;
            dst[OFF_W2 + (it * 4 + 2) * H + (jt * 8 + jj)] = acc[2 * jj + 1].x;
            dst[OFF_W2 + (it * 4 + 3) * H + (jt * 8 + jj)] = acc[2 * jj + 1].y;
        }
    }
    dst[OFF_W3 + lane * 2 + 0] = g_w30;
    dst[OFF_W3 + lane * 2 + 1] = g_w31;
    dst[OFF_B2 + lane] = g_b2;
    dst[OFF_B1 + lane] = g_b1;
    dst[OFF_W1 + lane] = g_w10;
    dst[OFF_W1 + H + lane] = g_w11;
    if (lane == 0) {
        dst[OFF_B3 + 0] = g_b30;   // identical in every lane (sums over the staged rows)
        dst[OFF_B3 + 1] = g_b31;
        dst[P] = loss;
    }
}

}  // namespace tc
}  // namespace lv32
}  // namespace b200ude
