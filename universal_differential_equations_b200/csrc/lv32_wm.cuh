// lv32_wm.cuh -- warp-collective variant of the LV 2 -> 32 -> 32 -> 2 kernels ("one warp = 16 trajectories").
//
// The one-trajectory-per-thread family (lv32_tc.cuh) passes every 32 x 32 sweep through shared-memory rows; its latency
// per right-hand-side evaluation is what bounds a small ensemble.  Here a warp integrates 16 trajectories
// (G groups of 16) with the hidden units spread over its lanes, so that nothing is wider than a warp:
//   * lane (fg, tig) = (lane >> 2, lane & 3) holds, for the two trajectories r in {fg, fg + 8} of a group, the eight
//     hidden units f in {8 q + 2 tig, 8 q + 2 tig + 1 : q = 0..3} -- exactly the C/D fragment layout of mma.sync.m16n8k8
//     with M = trajectories, N = hidden units;
//   * the 32 x 32 layer is H2[16 x 32] = H1[16 x 32] W2^T as 3xTF32 mma.sync (48 HMMA per group and sweep); because the
//     contraction index may be permuted freely (k = tig <-> unit 2 tig, k = tig + 4 <-> unit 2 tig + 1 inside a k-step), a
//     D fragment IS the A fragment of the next product: the chain forward, W2^T q2 of the adjoint and all element-wise
//     work stay in registers with no layout change; W2 (hi/lo split once per CTA) is read from shared memory as B fragments;
//   * the thin layers are FFMA partial sums over the lane's 8 units + a 3-shuffle reduce-scatter over the 4 lanes of a quad,
//     which leaves every lane with the ONE (trajectory, component) pair it owns: the Runge-Kutta state, the stage
//     derivatives and the adjoint state are kept once per (trajectory, component), not once per lane;
//   * tanh = 1 - 2 / (1 + 2^(2 log2(e) x)) with ONE reciprocal per four values (Montgomery's batched inversion: the MUFU
//     pipe -- 16 lanes/clk/SM -- is the scarcest unit of this path): 1.25 MUFU per tanh instead of 2; the affine map to the
//     exponent is folded into the staged weights (tanh_quad_z);
//   * adjoint: the ensemble-summed dW2 += q2^T h1 (K = the group's 16 trajectories) is a third 2-way-split fp16 mma.sync
//     product whose operands are the hi/lo words of the two other products, transposed in registers (movmatrix) and scaled
//     by one power of two per group; thin-layer gradients are per-lane register sums reduced once at the end of the kernel.
// No CTA-wide barrier inside the time loops; theta is bulk-copied by the TMA from the handle's device copy
// into shared memory once per CTA (no constant bank: handles are independent, any number can be in flight on a device).
//
// Reference semantics replaced: RHS scenario_1.jl:69-76; Tsit5 perform_step! and InterpolatingAdjoint as in
// ude_common.cuh / ude_adjoint.cuh (same record layout: ustep / dense rows, so either family's adjoint follows either
// family's forward).
#pragma once
#include <cuda_fp16.h>

#include "lv32_packed.cuh"

namespace b200ude {
namespace lv32 {
namespace wm {

constexpr int WSH = 24;   // row stride (32-bit words) of the fp16 copy of W2: 16 words per output unit + 8 padding -> conflict-free LDS.64

// The chain forward computes the pre-activations as z = 2 log2(e) (W x + b) - 1, the argument of tanh_quad_z: layers 1 and 2
// are staged with that scale and shift folded in (w1a, w1b, b1, b2 and the fp16 copy of W2), which saves the multiply per
// tanh.  The VJP's weights (W1 in SmemT, W2^T, W3) are staged unscaled.
struct __align__(16) SmemT {                // adjoint only: operand of W2^T q2, fp16 pairs over the contraction index j
    uint32_t w2t_hi[32 * WSH], w2t_lo[32 * WSH];   // word (i, s, tig, b) = (W2[16 s + 8 b + 2 tig][i], W2[.. + 1][i])
    float w1a[32], w1b[32];               // W1[f][0], W1[f][1], unscaled
    float w3max;                          // max |W3|: bound of the cotangent rows (scaling of the fp16 product)
};
struct __align__(16) SmemW {
    uint32_t w2h_hi[32 * WSH], w2h_lo[32 * WSH];   // k W2[j][.] as fp16 pairs in B-fragment order of mma.m16n8k16 (gemm32h): hi + lo split
    float w1a[32], w1b[32], b1[32];       // k W1[f][0], k W1[f][1], k b1[f] - 1   (k = 2 log2(e))
    float b2[32], w3a[32], w3b[32];       // k b2[j] - 1, W3[0][j], W3[1][j]
    float b3[4];
};

constexpr int RAW_FLOATS = ((P + 3) / 4) * 4;   // the handle's device copy of theta is padded to 16 bytes (b200ude_create)

// Weights into shared memory.  One elected thread bulk-copies theta (4.9 KB) with the TMA (1-D cp.async.bulk, completion on an
// mbarrier's transaction count -- SASS UBLKCP); then all threads of the CTA cut it into the operand layouts: fp16 hi/lo pairs
// of W2 in B-fragment order (and of W2^T for the adjoint), the thin layers as contiguous rows.  `raw` is RAW_FLOATS floats of
// (dynamic) shared memory, free again after the call returns.  Ends with a CTA barrier.
__device__ __forceinline__ void stage_weights(const float *__restrict__ theta, float *raw, SmemW &w, SmemT *t, int tid, int nthreads)
{
    __shared__ __align__(8) uint64_t bar;
    const uint32_t bar_a = (uint32_t)__cvta_generic_to_shared(&bar), dst_a = (uint32_t)__cvta_generic_to_shared(raw);
    constexpr uint32_t bytes = RAW_FLOATS * 4;
    if (tid == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_a));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a), "l"(theta),
                     "r"(bytes), "r"(bar_a)
                     : "memory");
    }
    __syncthreads();   // the barrier is initialised (and armed) before anybody polls it
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar_a) : "memory");
    auto pack = [](float x0, float x1, uint32_t &hi, uint32_t &lo) {
        const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
        const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
        hi = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    };
    // theta[OFF_W2 + i*32 + j] = W2[j][i]
    for (int e = tid; e < 32 * 16; e += nthreads) {
        const int a = e >> 4, r = e & 15, s_ = r >> 3, tg = (r >> 1) & 3, b = r & 1;
        const int c0 = 16 * s_ + 8 * b + 2 * tg;
        // forward copy: word (j = a, s, tig, b) = k (W2[j][c0], W2[j][c0 + 1])
        pack(TANH_K * raw[OFF_W2 + c0 * 32 + a], TANH_K * raw[OFF_W2 + (c0 + 1) * 32 + a], w.w2h_hi[a * WSH + r], w.w2h_lo[a * WSH + r]);
        // transposed copy: word (i = a, s, tig, b) = (W2[c0][i], W2[c0 + 1][i])
        if (t) pack(raw[OFF_W2 + a * 32 + c0], raw[OFF_W2 + a * 32 + c0 + 1], t->w2t_hi[a * WSH + r], t->w2t_lo[a * WSH + r]);
    }
    for (int f = tid; f < 32; f += nthreads) {
        w.w1a[f] = TANH_K * raw[OFF_W1 + f];
        w.w1b[f] = TANH_K * raw[OFF_W1 + H + f];
        w.b1[f] = fmaf(TANH_K, raw[OFF_B1 + f], -1.0f);
        w.b2[f] = fmaf(TANH_K, raw[OFF_B2 + f], -1.0f);
        if (t) {
            t->w1a[f] = raw[OFF_W1 + f];
            t->w1b[f] = raw[OFF_W1 + H + f];
        }
        w.w3a[f] = raw[OFF_W3 + 2 * f];
        w.w3b[f] = raw[OFF_W3 + 2 * f + 1];
    }
    if (tid < 2) w.b3[tid] = raw[OFF_B3 + tid];
    if (t && tid < 32) {   // warp 0: max |W3| over the 64 entries
        float m = fmaxf(fabsf(raw[OFF_W3 + tid]), fabsf(raw[OFF_W3 + 32 + tid]));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        if (tid == 0) t->w3max = m;
    }
    __syncthreads();
}

__device__ __forceinline__ float2 lds2(const float *p) { return *reinterpret_cast<const float2 *>(p); }

// per-lane constants of a warp
struct Lane {
    int fg, tig, comp, rsel;   // rsel = tig >> 1: which of the group's two rows (fg / fg + 8) this lane owns; comp = tig & 1
    int quad;                  // lane & ~3
};
__device__ __forceinline__ Lane make_lane()
{
    Lane L;
    const int lane = threadIdx.x & 31;
    L.fg = lane >> 2; L.tig = lane & 3; L.comp = L.tig & 1; L.rsel = L.tig >> 1; L.quad = lane & ~3;
    return L;
}
// R = rows per lane: 2 -> a group is 16 trajectories (rows fg, fg + 8 of the MMA tile), every lane owns one (row, component);
//                    1 -> a group is 8 trajectories (rows 8..15 of the tile are zero): half the element-wise work per warp for
//                         the latency-bound small ensembles; lanes with tig >= 2 shadow the (row, component) of tig - 2.

// every lane contributes the value of the (row, component) it owns; returns x[r][c] for the rows of the group
template <int R>
__device__ __forceinline__ void gather4(const Lane &L, float own, float (&x)[R][2])
{
    x[0][0] = __shfl_sync(0xffffffffu, own, L.quad + 0);
    x[0][1] = __shfl_sync(0xffffffffu, own, L.quad + 1);
    if constexpr (R == 2) {
        x[1][0] = __shfl_sync(0xffffffffu, own, L.quad + 2);
        x[1][1] = __shfl_sync(0xffffffffu, own, L.quad + 3);
    }
}
// y[r][c] partial sums over the quad's 4 lanes -> the total for the (row, component) this lane owns
template <int R>
__device__ __forceinline__ float scatter_sum(const Lane &L, const float (&y)[R][2])
{
    const bool c1 = L.comp != 0;
    float ka = c1 ? y[0][1] : y[0][0];
    const float sa = c1 ? y[0][0] : y[0][1];
    ka += __shfl_xor_sync(0xffffffffu, sa, 1);
    if constexpr (R == 2) {
        const bool r1 = L.rsel != 0;
        float kb = c1 ? y[1][1] : y[1][0];
        const float sb = c1 ? y[1][0] : y[1][1];
        kb += __shfl_xor_sync(0xffffffffu, sb, 1);
        const float keep = r1 ? kb : ka, send = r1 ? ka : kb;
        return keep + __shfl_xor_sync(0xffffffffu, send, 2);
    } else {
        return ka + __shfl_xor_sync(0xffffffffu, ka, 2);
    }
}

// layer 1 of the chain for G groups: h[g][r][q] = tanh(W1 x + b1) at the lane's units (8q + 2 tig, +1)
template <int TM, int G, int R>
__device__ __forceinline__ void layer1(const SmemW &w, const Lane &L, const float (&x)[G][R][2], float2 (&h)[G][R][4])
{
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const float2 w0 = lds2(w.w1a + 8 * q + 2 * L.tig), w1 = lds2(w.w1b + 8 * q + 2 * L.tig), bb = lds2(w.b1 + 8 * q + 2 * L.tig);
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int r = 0; r < R; ++r) h[g][r][q] = fma2(w0, bc(x[g][r][0]), fma2(w1, bc(x[g][r][1]), bb));
    }
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int r = 0; r < R; ++r) {
            tanh_quad_z<TM>(h[g][r][0], h[g][r][1]);
            tanh_quad_z<TM>(h[g][r][2], h[g][r][3]);
        }
}

// D += A B, m16n8k16, fp16 inputs, fp32 accumulate
__device__ __forceinline__ void mma16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1)
{
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
// (hi, lo) fp16 pairs of a float2: hi = the value truncated to 10 mantissa bits (exact in fp16), lo = fp16(x - hi): 22 bits
__device__ __forceinline__ void split_h2(float2 v, uint32_t &hi, uint32_t &lo)
{
    const float hx = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u), hy = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(hy), "f"(hx));
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(v.y - hy), "f"(v.x - hx));
}
// d[g][nt] += A[g] B (B fragments from a staged fp16 copy of W2 or W2^T) as a 2-way-split fp16 product (hi hi + lo hi + hi lo:
// 22-bit operands, fp32 accumulate): half the tensor-pipe time of 3xTF32.  For operands bounded like the tanh outputs
// (|a| <= 1; the cotangent rows are scaled into that range by the caller) and weights below 65504 in the staged copy: the
// forward copy holds 2 log2(e) W2, so |W2| >= ~22 700 there, |W2| >= 65504 in the W2^T copy (beyond that the fp16 copy is
// inf, the product NaN, and the trajectory's status word reports the non-finite result).  A = a[g][r][q]: the D-fragment layout is
// the A-fragment layout under the k permutation (k = 2 tig, 2 tig + 1 <-> units 16 s + 2 tig, + 1; k + 8 <-> units + 8).
template <int G, int R>
__device__ __forceinline__ void gemm32h(const uint32_t *__restrict__ bhi, const uint32_t *__restrict__ blo, const Lane &L,
                                        const float2 (&a)[G][R][4], float (&d)[G][4][4])
{
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        uint32_t ah[G][4], al[G][4];
#pragma unroll
        for (int g = 0; g < G; ++g) {
            split_h2(a[g][0][2 * s], ah[g][0], al[g][0]);
            split_h2(a[g][0][2 * s + 1], ah[g][2], al[g][2]);
            if constexpr (R == 2) {
                split_h2(a[g][1][2 * s], ah[g][1], al[g][1]);
                split_h2(a[g][1][2 * s + 1], ah[g][3], al[g][3]);
            } else {
                ah[g][1] = ah[g][3] = al[g][1] = al[g][3] = 0u;
            }
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const uint2 bh = *reinterpret_cast<const uint2 *>(bhi + (8 * nt + L.fg) * WSH + 8 * s + 2 * L.tig);
            const uint2 bl = *reinterpret_cast<const uint2 *>(blo + (8 * nt + L.fg) * WSH + 8 * s + 2 * L.tig);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                mma16(d[g][nt], al[g], bh.x, bh.y);
                mma16(d[g][nt], ah[g], bl.x, bl.y);
                mma16(d[g][nt], ah[g], bh.x, bh.y);
            }
        }
    }
}

// The adjoint's operands split once and used twice: by gemm32h_w as rows, and transposed by the dW2 product.
// hi[r][q] / lo[r][q] = split_h2(a[r][q]): one f16x2 word per lane of the 8 x 8 block (rows fg + 8 r, units 8 q + 2 tig, + 1)
template <int R>
__device__ __forceinline__ void split_rows(const float2 (&a)[R][4], uint32_t (&hi)[R][4], uint32_t (&lo)[R][4])
{
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) split_h2(a[r][q], hi[r][q], lo[r][q]);
}
// gemm32h<1, R> on words made by split_rows: the same HMMA sequence, so the same result bit for bit
template <int R>
__device__ __forceinline__ void gemm32h_w(const uint32_t *__restrict__ bhi, const uint32_t *__restrict__ blo, const Lane &L,
                                          const uint32_t (&hi)[R][4], const uint32_t (&lo)[R][4], float (&d)[4][4])
{
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const uint32_t ah[4] = {hi[0][2 * s], R == 2 ? hi[R - 1][2 * s] : 0u, hi[0][2 * s + 1], R == 2 ? hi[R - 1][2 * s + 1] : 0u};
        const uint32_t al[4] = {lo[0][2 * s], R == 2 ? lo[R - 1][2 * s] : 0u, lo[0][2 * s + 1], R == 2 ? lo[R - 1][2 * s + 1] : 0u};
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const uint2 bh = *reinterpret_cast<const uint2 *>(bhi + (8 * nt + L.fg) * WSH + 8 * s + 2 * L.tig);
            const uint2 bl = *reinterpret_cast<const uint2 *>(blo + (8 * nt + L.fg) * WSH + 8 * s + 2 * L.tig);
            mma16(d[nt], al, bh.x, bh.y);
            mma16(d[nt], ah, bl.x, bl.y);
            mma16(d[nt], ah, bh.x, bh.y);
        }
    }
}
// D += A B, m16n8k8, fp16 inputs, fp32 accumulate
__device__ __forceinline__ void mma16k8(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t b0)
{
    asm("mma.sync.aligned.m16n8k8.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(b0));
}
// transpose of the 8 x 8 fp16 block held one f16x2 word per lane: lane (fg, tig) gets (M[2 tig][fg], M[2 tig + 1][fg])
__device__ __forceinline__ uint32_t movm_t(uint32_t x)
{
    uint32_t y;
    asm("movmatrix.sync.aligned.m8n8.trans.b16 %0, %1;" : "=r"(y) : "r"(x));
    return y;
}
__device__ __forceinline__ uint32_t hmul2(uint32_t a, uint32_t b)
{
    uint32_t y;
    asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(y) : "r"(a), "r"(b));   // no .ftz: fp16 subnormals are kept
    return y;
}
// 2^(e - 127) for a biased exponent e in [0, 255]: 0 for e = 0, inf for e = 255
__device__ __forceinline__ float exp2_biased(int e) { return __uint_as_float((uint32_t)e << 23); }

// UDE right-hand side for G groups; gv[g] = this lane's (row, component) of the stage argument, returns the same
// component of du/dt.  du1 = p1 u1 + NN1(u), du2 = -p4 u2 + NN2(u)  (scenario_1.jl:71-72): pc = p1 / -p4 by component.
template <int TM, int G, int R>
__device__ __forceinline__ void rhs_wm(const SmemW *wp, float pc, const float (&gv)[G], float (&kout)[G])
{
    const SmemW &w = *wp;
    const Lane L = make_lane();
    float x[G][R][2];
#pragma unroll
    for (int g = 0; g < G; ++g) gather4<R>(L, gv[g], x[g]);
    float2 h[G][R][4];
    layer1<TM, G, R>(w, L, x, h);
    float d[G][4][4];
#pragma unroll
    for (int nt = 0; nt < 4; ++nt) {
        const float2 bias = lds2(w.b2 + 8 * nt + 2 * L.tig);
#pragma unroll
        for (int g = 0; g < G; ++g) { d[g][nt][0] = bias.x; d[g][nt][1] = bias.y; d[g][nt][2] = bias.x; d[g][nt][3] = bias.y; }
    }
    gemm32h<G, R>(w.w2h_hi, w.w2h_lo, L, h, d);
    const float b3c = w.b3[L.comp];
#pragma unroll
    for (int g = 0; g < G; ++g) {
        float y[R][2];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float2 v[4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) v[nt] = make_float2(d[g][nt][2 * r], d[g][nt][2 * r + 1]);
            tanh_quad_z<TM>(v[0], v[1]);
            tanh_quad_z<TM>(v[2], v[3]);
            float2 s0 = bc(0.0f), s1 = bc(0.0f);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                s0 = fma2(lds2(w.w3a + 8 * nt + 2 * L.tig), v[nt], s0);
                s1 = fma2(lds2(w.w3b + 8 * nt + 2 * L.tig), v[nt], s1);
            }
            y[r][0] = s0.x + s0.y;
            y[r][1] = s1.x + s1.y;
        }
        kout[g] = fmaf(pc, gv[g], scatter_sum<R>(L, y) + b3c);
    }
}

// Tsit5 tables for the rolled stage loops (uniform constant-bank loads instead of a jump table per stage)
#define B200UDE_ROW7(F, I) {(float)F(I, 0), (float)F(I, 1), (float)F(I, 2), (float)F(I, 3), (float)F(I, 4), (float)F(I, 5), (float)F(I, 6), 0.0f}
static __constant__ float c_bw[6][8] = {B200UDE_ROW7(Tsit5::bw, 0), B200UDE_ROW7(Tsit5::bw, 1), B200UDE_ROW7(Tsit5::bw, 2),
                                        B200UDE_ROW7(Tsit5::bw, 3), B200UDE_ROW7(Tsit5::bw, 4), B200UDE_ROW7(Tsit5::bw, 5)};
static __constant__ float c_a[7][8] = {B200UDE_ROW7(Tsit5::a, 0), B200UDE_ROW7(Tsit5::a, 1), B200UDE_ROW7(Tsit5::a, 2), B200UDE_ROW7(Tsit5::a, 3),
                                       B200UDE_ROW7(Tsit5::a, 4), B200UDE_ROW7(Tsit5::a, 5), B200UDE_ROW7(Tsit5::a, 6)};
#undef B200UDE_ROW7
static __constant__ float c_binv[6] = {(float)(1.0 / Tsit5::b(0)), (float)(1.0 / Tsit5::b(1)), (float)(1.0 / Tsit5::b(2)),
                                       (float)(1.0 / Tsit5::b(3)), (float)(1.0 / Tsit5::b(4)), (float)(1.0 / Tsit5::b(5))};

struct Consts {
    float p1, p4;       // du1 = p1 u1 + ..., du2 = -p4 u2 + ...
    float lw0, lw1;     // L2 loss weights per component
};

// ---- forward: fixed-step Tsit5, WPC warps per CTA, G groups of 8 R trajectories per warp -------------------------------
template <int TM, int G, int R, int WPC>
__global__ void __launch_bounds__(32 * WPC, 32 / (WPC * G)) forward_kernel(FwdParams p, Consts cs)
{
    __shared__ SmemW w;
    extern __shared__ __align__(16) unsigned char s_raw[];
    stage_weights(p.theta, reinterpret_cast<float *>(s_raw), w, nullptr, threadIdx.x, 32 * WPC);
    const Lane L = make_lane();
    const size_t N = (size_t)p.N;
    const int wg = blockIdx.x * WPC + (threadIdx.x >> 5);
    const float pc = L.comp ? -cs.p4 : cs.p1;
    const float dt = p.dt;
    bool live[G];
    size_t idx[G];   // comp * N + n
    float u[G], k[G][6];
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const long n = (long)(wg * G + g) * (8 * R) + L.fg + (R == 2 ? 8 * L.rsel : 0);
        live[g] = n < (long)N && (R == 2 || L.rsel == 0);                     // R = 1: lanes tig >= 2 only shadow
        idx[g] = (size_t)L.comp * N + (size_t)(n < (long)N ? n : (long)N - 1);   // padding lanes shadow the last trajectory; stores masked
        u[g] = __ldg(p.u0 + idx[g]);
#pragma unroll
        for (int j = 0; j < 6; ++j) k[g][j] = 0.0f;
    }
    auto store = [&](float *base, int row, const float (&v)[G]) {
#pragma unroll
        for (int g = 0; g < G; ++g)
            if (live[g]) base[(size_t)row * 2 * N + idx[g]] = v[g];
    };
    store(p.out, 0, u);
    store(p.ustep, 0, u);
    int isave = 1;
#pragma unroll 1
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll 1
        for (int i = (s == 0 ? 0 : 1); i < 7; ++i) {
            // stage argument from the uniform row a[i][.] (zero beyond the stage's own coefficients: the same sum, in the
            // same order, as the unrolled stage), the new derivative into its slot by selects: no jump table per stage
            float gv[G];
#pragma unroll
            for (int g = 0; g < G; ++g) {
                float a = 0.0f;
#pragma unroll
                for (int j = 0; j < 6; ++j) a = fmaf(c_a[i][j], k[g][j], a);
                gv[g] = fmaf(dt, a, u[g]);
                u[g] = i == 6 ? gv[g] : u[g];   // stage 7's argument is u_{n+1} (row 7 = b, FSAL)
            }
            float kk[G];
            rhs_wm<TM, G, R>(&w, pc, gv, kk);
            const int slot = i == 6 ? 0 : i;   // k_7(s) = k_1(s+1) (FSAL)
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int j = 0; j < 6; ++j) k[g][j] = slot == j ? kk[g] : k[g][j];
            store(p.dense, s * 6 + i, kk);   // row (s+1)*6 for i = 6: k_7(s) = k_1(s+1)
        }
        store(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) {
            store(p.out, isave, u);
            ++isave;
        }
    }
    if (p.status) {
#pragma unroll
        for (int g = 0; g < G; ++g) {
            // a trajectory is bad if either of its components is non-finite: combine the two lanes that own them
            int bad = (fabsf(u[g]) <= 3.0e38f) ? 0 : 1;
            bad |= __shfl_xor_sync(0xffffffffu, bad, 1);
            if (live[g] && L.comp == 0) p.status[idx[g]] = bad;
        }
    }
}

// ---- adjoint: interpolating adjoint on the fixed grid, one group of 8 R trajectories per warp --------------------------
struct __align__(16) WarpTiles {
    float sum[32 * 32];     // running dW2 sums of this warp, element k*32 + lane <-> accumulator register k of that lane
};

// Backward stage i scales the cotangent by dt b_i, so the dW2 operand of stage i exceeds that of stage 0 by up to
// max |b_i| / |b_0| = 34.1 (times the change of lambda over the step): the smallest e with 2^e above that ratio (6) is the
// headroom the first stage of a step leaves in the accumulator's scale, so that the later stages seldom have to rescale it
constexpr int stage_headroom()
{
    double r = 0.0;
    for (int i = 0; i < 6; ++i) {
        const double q = Tsit5::b(i) / Tsit5::b(0);
        r = q > r ? q : (-q > r ? -q : r);
    }
    int e = 0;
    while ((double)(1 << e) <= r) ++e;
    return e;
}
constexpr int STAGE_HEADROOM = stage_headroom();
static_assert(STAGE_HEADROOM == 6, "Tsit5: max |b_i| / b_0 = 34.1");

// the lambda-free part of a backward stage at one state: what the cotangent products of that point read
template <int R>
struct ChainRows {
    float xo;                           // own component of the state (its rows are gathered where they are used)
    float2 om1[R][4];                   // 1 - h1^2
    uint32_t h1hi[R][4], h1lo[R][4];    // h1 split once: A operand of layer 2, (transposed) B operand of dW2
    float2 h2[R][4];                    // tanh of layer 2
};

template <int TM, int R, int WPC, int MINB>
__global__ void __launch_bounds__(32 * WPC, MINB) adjoint_kernel(AdjParams p, Consts cs)
{
    __shared__ SmemW w;
    __shared__ SmemT wt;
    extern __shared__ __align__(16) unsigned char s_raw[];   // [raw theta (staging only)] [WarpTiles x WPC]
    stage_weights(p.theta, reinterpret_cast<float *>(s_raw), w, &wt, threadIdx.x, 32 * WPC);
    const Lane L = make_lane();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpTiles &T = reinterpret_cast<WarpTiles *>(s_raw + RAW_FLOATS * 4)[warp];
#pragma unroll
    for (int q = 0; q < 32; ++q) T.sum[q * 32 + lane] = 0.0f;
    __syncwarp();

    const size_t N = (size_t)p.N;
    const int wg = blockIdx.x * WPC + warp;
    const long n_end = p.n_cnt ? (long)p.n0 + p.n_cnt : (long)N;
    const long n = (long)p.n0 + (long)wg * (8 * R) + L.fg + (R == 2 ? 8 * L.rsel : 0);
    const bool live = n < n_end && (R == 2 || L.rsel == 0);   // R = 1: lanes tig >= 2 shadow tig - 2 (weight 0, stores masked)
    const size_t idx = (size_t)L.comp * N + (size_t)(n < (long)N ? n : (long)N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float pc = L.comp ? -cs.p4 : cs.p1;
    const float lw = L.comp ? cs.lw1 : cs.lw0;
    const float dt = p.dt, inv_dt = 1.0f / dt;

    // C fragments of 2^(127 - e_acc) dW2 (+)= q2^T h1: tile (mt, nt): rows j = 16 mt + fg (+8), columns i = 8 nt + 2 tig (+1).
    // e_acc (warp-uniform) is the largest row exponent of the cotangent operand since the last flush
    float macc[2][4][4];
    int e_acc = 0;
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b)
#pragma unroll
            for (int c = 0; c < 4; ++c) macc[a][b][c] = 0.0f;
    // thin-layer gradients: sums over the lane's trajectories at its 8 units, reduced over fg at the end
    float2 gW3a[4], gW3b[4], gB2[4], gB1[4], gW1a[4], gW1b[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) { gW3a[q] = gW3b[q] = gB2[q] = gB1[q] = gW1a[q] = gW1b[q] = bc(0.0f); }
    float gb3 = 0.0f;   // own component's output-bias gradient
    float lam = 0.0f, loss = 0.0f;
    const int n_save = p.n_steps / p.save_every + 1;

    auto jump = [&](int isave) {
        const size_t id = (size_t)isave * 2 * N + idx;
        if (p.fused_l2) {
            const float r = __ldg(p.ustep + (size_t)(isave * p.save_every) * 2 * N + idx) - __ldg(p.cot + id);
            loss = fmaf(lw * r, r, loss);
            lam = fmaf(2.0f * lw, r, lam);
        } else {
            lam += __ldg(p.cot + id);
        }
    };

    // A backward stage is three parts: the chain forward at its state (lambda-free), the VJP of its lambda argument (the
    // cotangent rows sg = dt b_i lambda-argument give q2, W2^T q2, q1 and the stage's k) and the theta sums, linear in sg.
    // Where two stages share a state, the chain forward runs once and dW3 once, on the summed rows.

    // the chain forward at the state whose own component is xo
    auto chain = [&](float xo, ChainRows<R> &c) {
        float x[1][R][2];
        gather4<R>(L, xo, x[0]);
        c.xo = xo;
        float2 h1[1][R][4];
        layer1<TM, 1, R>(w, L, x, h1);
        split_rows<R>(h1[0], c.h1hi, c.h1lo);
        float d[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const float2 bias = lds2(w.b2 + 8 * nt + 2 * L.tig);
            d[nt][0] = bias.x; d[nt][1] = bias.y; d[nt][2] = bias.x; d[nt][3] = bias.y;
        }
        gemm32h_w<R>(w.w2h_hi, w.w2h_lo, L, c.h1hi, c.h1lo, d);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float2 v[4];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) v[nt] = make_float2(d[nt][2 * r], d[nt][2 * r + 1]);
            tanh_quad_z<TM>(v[0], v[1]);
            tanh_quad_z<TM>(v[2], v[3]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                c.h2[r][nt] = v[nt];
                const float2 hh = h1[0][r][nt];
                c.om1[r][nt] = fma2(make_float2(-hh.x, -hh.y), hh, bc(1.0f));
            }
        }
    };
    // Every cotangent row q2[t][.] is scaled by a power of two into fp16's range for the W2^T q2 product (|q2[t][j]| <=
    // max|W3| (|sg_t0| + |sg_t1|) =: B_t; scale 2^(127 - e_t), e_t = biased exponent of B_t, undone on the product -- both exact)
    auto row_exp = [&](const float (&sg)[R][2], uint32_t (&eb)[R]) {
#pragma unroll
        for (int r = 0; r < R; ++r) eb[r] = (__float_as_uint(wt.w3max * (fabsf(sg[r][0]) + fabsf(sg[r][1]))) >> 23) & 0xFFu;
    };
    // the scaled rows 2^(127 - e_t) q2 as fp16 hi/lo words: operand of W2^T q2 and (transposed) of dW2
    auto split_q2 = [&](const float2 (&q2)[R][4], const uint32_t (&eb)[R], uint32_t (&hi)[R][4], uint32_t (&lo)[R][4]) {
        float2 q2s[R][4];
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float2 sc2 = bc(__uint_as_float((254u - eb[r]) << 23));
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) q2s[r][nt] = mul2(q2[r][nt], sc2);
        }
        split_rows<R>(q2s, hi, lo);
    };
    // q2 = (W3^T sg) (1 - h2^2) of cotangent rows sg; db2 += q2
    auto q2_rows = [&](const ChainRows<R> &c, const float (&sg)[R][2], float2 (&q2)[R][4]) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float2 s0 = bc(sg[r][0]), s1 = bc(sg[r][1]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const float2 w3a = lds2(w.w3a + 8 * nt + 2 * L.tig), w3b = lds2(w.w3b + 8 * nt + 2 * L.tig);
                const float2 t = fma2(w3b, s1, mul2(w3a, s0));
                const float2 v = c.h2[r][nt];
                const float2 om = fma2(make_float2(-v.x, -v.y), v, bc(1.0f));
                q2[r][nt] = mul2(t, om);
                gB2[nt] = add2(gB2[nt], q2[r][nt]);
            }
        }
    };
    // the VJP of one lambda argument from its q2 words (split_q2): go = own component of the lambda argument,
    // isc = 1 / (dt b_i); returns the stage's own component of k.  dW1 += q1 (x) x and db1 += q1 are accumulated here,
    // once per stage: q1 is not summed over the two stages of a shared point
    auto vjp = [&](const ChainRows<R> &c, const uint32_t (&eb)[R], const uint32_t (&q2hi)[R][4], const uint32_t (&q2lo)[R][4],
                   float go, float isc) -> float {
        float2 unscale[R];
#pragma unroll
        for (int r = 0; r < R; ++r) unscale[r] = bc(__uint_as_float(eb[r] << 23));
        float e[4][4];
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int c4 = 0; c4 < 4; ++c4) e[nt][c4] = 0.0f;
        gemm32h_w<R>(wt.w2t_hi, wt.w2t_lo, L, q2hi, q2lo, e);
        // q1 = (W2^T q2) (1 - h1^2); (df/du)^T g; dW1 += q1 (x) x, db1 += q1
        float x[R][2], y[R][2];
        gather4<R>(L, c.xo, x);
#pragma unroll
        for (int r = 0; r < R; ++r) {
            float2 s0 = bc(0.0f), s1 = bc(0.0f);
            const float2 x0 = bc(x[r][0]), x1 = bc(x[r][1]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const float2 om = mul2(c.om1[r][nt], unscale[r]);
                const float2 q1 = mul2(make_float2(e[nt][2 * r], e[nt][2 * r + 1]), om);
                s0 = fma2(lds2(wt.w1a + 8 * nt + 2 * L.tig), q1, s0);
                s1 = fma2(lds2(wt.w1b + 8 * nt + 2 * L.tig), q1, s1);
                gB1[nt] = add2(gB1[nt], q1);
                gW1a[nt] = fma2(q1, x0, gW1a[nt]);
                gW1b[nt] = fma2(q1, x1, gW1b[nt]);
            }
            y[r][0] = s0.x + s0.y;
            y[r][1] = s1.x + s1.y;
        }
        const float dxo = scatter_sum<R>(L, y);
        return fmaf(pc, go, dxo * isc);   // LV physics: diag(p1, -p4)
    };
    // dW3 += sg (x) h2
    auto acc_w3 = [&](const ChainRows<R> &c, const float (&sg)[R][2]) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const float2 s0 = bc(sg[r][0]), s1 = bc(sg[r][1]);
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                gW3a[nt] = fma2(s0, c.h2[r][nt], gW3a[nt]);
                gW3b[nt] = fma2(s1, c.h2[r][nt], gW3b[nt]);
            }
        }
    };
    // one stage's dW2 += q2^T h1 from the words of its q2 (split_q2); first = the first stage since macc was flushed
    auto acc_w2 = [&](const ChainRows<R> &c, const uint32_t (&eb)[R], const uint32_t (&q2hi)[R][4], const uint32_t (&q2lo)[R][4], bool first) {
        // dW2 += q2^T h1 (below) sums over rows, so the rows' scales become one per group: the words of row t are
        // multiplied by 2^(e_t - e_acc) (exact down to fp16's subnormals; below them the error is at most 2^-24 B_max per
        // element), e_acc >= every e_t since the last flush.  All maxima are over the integer exponents, so an inf/NaN row
        // (255) poisons the sums as a non-finite q2 does.
        int e_max = (int)eb[0];
        if constexpr (R == 2) e_max = max(e_max, (int)eb[1]);
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) e_max = max(e_max, __shfl_xor_sync(0xffffffffu, e_max, o));   // over fg: warp-uniform
        if (first) {   // macc is zero; room for the larger b_i of the later stages, at most 2^127 for finite rows
            e_acc = e_max == 255 ? 255 : min(e_max + STAGE_HEADROOM, 254);
        } else if (e_max > e_acc) {   // above the step's scale so far: rare, lambda changes smoothly over a step
            const float rs = exp2_biased(max(e_acc - e_max + 127, 0));
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                    for (int c4 = 0; c4 < 4; ++c4) macc[mt][nt][c4] *= rs;
            e_acc = e_max;
        }
        // dW2 += q2^T h1: M = j (2 tiles), N = i (4 tiles), K = the group's 8 R trajectories (m16n8k16 for R = 2, m16n8k8 for
        // R = 1), 2-way split on the words of the two products, each 8 x 8 block transposed by one movmatrix
        uint32_t ah[2][2 * R], al[2][2 * R];   // A fragments of q2^T: (mt, 2 r + (nt & 1)) <- block (r, nt) of q2, nt >> 1 = mt
#pragma unroll
        for (int r = 0; r < R; ++r) {
            uint32_t m2;
            asm("cvt.rn.f16x2.f32 %0, %1, %1;" : "=r"(m2) : "f"(exp2_biased(max((int)eb[r] - e_acc + 127, 0))));
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                ah[nt >> 1][2 * r + (nt & 1)] = movm_t(hmul2(q2hi[r][nt], m2));
                al[nt >> 1][2 * r + (nt & 1)] = movm_t(hmul2(q2lo[r][nt], m2));
            }
        }
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            uint32_t bh[R], bl[R];   // B fragment of h1: k-step half r <- block (r, nt) of h1
#pragma unroll
            for (int r = 0; r < R; ++r) { bh[r] = movm_t(c.h1hi[r][nt]); bl[r] = movm_t(c.h1lo[r][nt]); }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                if constexpr (R == 2) {
                    mma16(macc[mt][nt], al[mt], bh[0], bh[1]);
                    mma16(macc[mt][nt], ah[mt], bl[0], bl[1]);
                    mma16(macc[mt][nt], ah[mt], bh[0], bh[1]);
                } else {
                    mma16k8(macc[mt][nt], al[mt][0], al[mt][1], bh[0]);
                    mma16k8(macc[mt][nt], ah[mt][0], ah[mt][1], bl[0]);
                    mma16k8(macc[mt][nt], ah[mt][0], ah[mt][1], bh[0]);
                }
            }
        }
    };
    // the tensor core adds into its accumulator with truncation: keep the chains at most one step long and add them into the
    // running sums with round-to-nearest, undoing the step's scale 2^(127 - e_acc) (exact: a power of two)
    auto flush = [&]() {
        const float us_acc = exp2_biased(e_acc);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int c4 = 0; c4 < 4; ++c4) {
                    float &slot = T.sum[((mt * 4 + nt) * 4 + c4) * 32 + lane];
                    slot = fmaf(macc[mt][nt][c4], us_acc, slot);
                    macc[mt][nt][c4] = 0.0f;
                }
    };

    jump(n_save - 1);
    // stage derivatives k_1..k_7 and the start state of the forward step being traversed: read once per step (the next
    // step's rows are requested while the last stage of the current one is evaluated), u(t) of every stage from registers
    float kd[7], us, kl[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) kl[j] = 0.0f;
    auto load_step = [&](int s) {
#pragma unroll
        for (int j = 0; j < 7; ++j) kd[j] = __ldg(p.dense + (size_t)(s * 6 + j) * 2 * N + idx);
        us = __ldg(p.ustep + (size_t)s * 2 * N + idx);
    };
    load_step(p.n_steps - 1);
    // lambda_s from the step's stage derivatives, then the data jump at a save point
    auto step_end = [&](int s) {
        float a = 0.0f;
#pragma unroll
        for (int j = 0; j < 6; ++j) a = fmaf((float)Tsit5::b(j), kl[j], a);
        lam = fmaf(dt, a, lam);
        if (s % p.save_every == 0) jump(s / p.save_every);
    };
    // backward stage i of step s evaluates at t_{s+1} - c_i dt.  Stage 5 (c = 1) of step s and stage 0 (c = 0) of step s - 1
    // share the state u(t_s) = ustep[s]: the interpolant's weights are zero at theta = 0, and at theta = 1 they are the
    // forward's b_j in fp32, so the same fma chain rebuilds ustep[s] bit for bit.  Both are evaluated at the end of step s.
#pragma unroll 1
    for (int s = p.n_steps - 1; s >= 0; --s) {
        // stage 0 of the last step and stage 5 of step 0 run alone; every other stage 0 runs with stage 5 of the step above
#pragma unroll 1
        for (int stage = s == p.n_steps - 1 ? 0 : 1; stage < (s == 0 ? 6 : 5); ++stage) {
            float xa = 0.0f, ga = 0.0f;
#pragma unroll
            for (int j = 0; j < 7; ++j) xa = fmaf(c_bw[stage][j], kd[j], xa);
#pragma unroll
            for (int j = 0; j < 5; ++j) ga = fmaf(c_a[stage][j], kl[j], ga);
            const float xo = fmaf(dt, xa, us);      // u(t_{s+1} - c_i dt), own component (Tsit5 free interpolant)
            const float go = fmaf(dt, ga, lam);     // lambda argument of backward stage i
            const float sgo = lv * (dt * c_a[6][stage]) * go;
            ChainRows<R> c;
            chain(xo, c);
            float sg[R][2];
            gather4<R>(L, sgo, sg);
            gb3 += sgo;
            uint32_t eb[R];
            row_exp(sg, eb);
            float2 q2[R][4];
            q2_rows(c, sg, q2);
            uint32_t q2hi[R][4], q2lo[R][4];
            split_q2(q2, eb, q2hi, q2lo);
            acc_w3(c, sg);   // before the VJP: h2 and the h1 words end here
            acc_w2(c, eb, q2hi, q2lo, stage == 0);
            const float kn = vjp(c, eb, q2hi, q2lo, go, inv_dt * c_binv[stage]);
#pragma unroll
            for (int j = 0; j < 6; ++j) kl[j] = (stage == j) ? kn : kl[j];
        }
        if (s == 0) {
            step_end(0);
            break;
        }
        // stage 5 of step s and stage 0 of step s - 1 at u(t_s): the chain forward once, each stage's VJP and its dW2 product
        // (on the words of its own q2, so that the sums are those of separate stages), dW3 once on the summed rows
        flush();   // stages 0..4 of the step: the accumulators hold no registers through the chain forward
        ChainRows<R> c;
        chain(us, c);
        float ga = 0.0f;
#pragma unroll
        for (int j = 0; j < 5; ++j) ga = fmaf(c_a[5][j], kl[j], ga);
        const float go = fmaf(dt, ga, lam);
        const float sgo = lv * (dt * c_a[6][5]) * go;
        float sg[R][2];
        gather4<R>(L, sgo, sg);
        gb3 += sgo;
        uint32_t eb[R];
        row_exp(sg, eb);
        float2 q2[R][4];
        q2_rows(c, sg, q2);
        uint32_t q2hi[R][4], q2lo[R][4];
        split_q2(q2, eb, q2hi, q2lo);
        acc_w2(c, eb, q2hi, q2lo, false);   // at the step's scale e_acc
        flush();   // ... and stage 5, before the two VJPs
        kl[5] = vjp(c, eb, q2hi, q2lo, go, inv_dt * c_binv[5]);
        step_end(s);
        // stage 0 of step s - 1: its lambda argument is lambda_s
        const float sgo0 = lv * (dt * c_a[6][0]) * lam;
        float sg0[R][2];
        gather4<R>(L, sgo0, sg0);
        gb3 += sgo0;
        row_exp(sg0, eb);
        q2_rows(c, sg0, q2);
        split_q2(q2, eb, q2hi, q2lo);
        const float k0 = vjp(c, eb, q2hi, q2lo, lam, inv_dt * c_binv[0]);
        load_step(s - 1);
#pragma unroll
        for (int j = 0; j < 6; ++j) kl[j] = j == 0 ? k0 : 0.0f;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            sg[r][0] += sg0[r][0];
            sg[r][1] += sg0[r][1];
        }
        acc_w3(c, sg);
        acc_w2(c, eb, q2hi, q2lo, true);
    }
    flush();
    if (p.grad_u0 && live) p.grad_u0[idx] = lam;
    loss *= lv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    // own-component sums of the output bias: add the lanes that own the same component
    gb3 += __shfl_xor_sync(0xffffffffu, gb3, 2);
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) gb3 += __shfl_xor_sync(0xffffffffu, gb3, o);
    // thin layers: sum over fg (lanes with equal tig own the same units)
    auto red_fg = [&](float2 &v) {
#pragma unroll
        for (int o = 4; o < 32; o <<= 1) {
            v.x += __shfl_xor_sync(0xffffffffu, v.x, o);
            v.y += __shfl_xor_sync(0xffffffffu, v.y, o);
        }
    };
#pragma unroll
    for (int q = 0; q < 4; ++q) { red_fg(gW3a[q]); red_fg(gW3b[q]); red_fg(gB2[q]); red_fg(gB1[q]); red_fg(gW1a[q]); red_fg(gW1b[q]); }
    float *dst = p.partial + (size_t)(p.row0 + wg) * (P + 1);
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            const int j = 16 * mt + L.fg, i = 8 * nt + 2 * L.tig;
            const float *sm = &T.sum[((mt * 4 + nt) * 4) * 32 + lane];
            dst[OFF_W2 + i * H + j] = sm[0];
            dst[OFF_W2 + (i + 1) * H + j] = sm[32];
            dst[OFF_W2 + i * H + j + 8] = sm[64];
            dst[OFF_W2 + (i + 1) * H + j + 8] = sm[96];
        }
    if (L.fg == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int f = 8 * q + 2 * L.tig;
            dst[OFF_W3 + 2 * f + 0] = gW3a[q].x; dst[OFF_W3 + 2 * (f + 1) + 0] = gW3a[q].y;
            dst[OFF_W3 + 2 * f + 1] = gW3b[q].x; dst[OFF_W3 + 2 * (f + 1) + 1] = gW3b[q].y;
            dst[OFF_B2 + f] = gB2[q].x; dst[OFF_B2 + f + 1] = gB2[q].y;
            dst[OFF_B1 + f] = gB1[q].x; dst[OFF_B1 + f + 1] = gB1[q].y;
            dst[OFF_W1 + f] = gW1a[q].x; dst[OFF_W1 + f + 1] = gW1a[q].y;
            dst[OFF_W1 + H + f] = gW1b[q].x; dst[OFF_W1 + H + f + 1] = gW1b[q].y;
        }
    }
    if (lane < 2) dst[OFF_B3 + lane] = gb3;   // lane 0 owns component 0, lane 1 component 1
    if (lane == 0) dst[P] = loss;
}

}  // namespace wm
}  // namespace lv32
}  // namespace b200ude
