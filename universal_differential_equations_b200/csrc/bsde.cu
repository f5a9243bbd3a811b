// bsde.cu -- deep-BSDE solve of a terminal PDE with batched SDE paths: the NNPDENS path of highdim_pde/lambaem.jl (SURVEY section 8 f4,
// BASELINE config 5).
//
// Reference call (highdim_pde/lambaem.jl:18-34):
//     prob = TerminalPDEProblem(g, f, mu, sigma, x0, tspan);  pdealg = NNPDENS(u0, sigmaT_grad_u, opt = ADAM(0.03))
//     solve(prob, pdealg; maxiters = 500, trajectories = m, alg = LambaEM(), ...)
// NNPDENS [EXT NeuralNetDiffEq 1.1.0] integrates  dX = mu dt + sigma dW,  du = -f(X, u, z, p, t) dt + z . dW,  z = sigmaT_grad_u([X; t]),
// u(0) = u0(x0), for `trajectories` paths and minimises mean (g(X_T) - u_T)^2 over both networks with ADAM; the answer is u0(x0).
// Here, for the script's family  mu = 0, sigma = s I, f = -lambda |z|^2, g(X) = log(a + b |X|^2)  (Hamilton-Jacobi-Bellman):
//   * all paths of an iteration advance together; the networks work on [width x paths] column-major activations (a path = a column), so
//     theta's vec(W) is already the operand of every layer product -- no repacking of the reference's parameter vector;
//   * fp64 (BASELINE's config 5), dim <= 110 and hidden <= 111 (the augmented rows [X; t; 1] and [h; 1] fit FT unit tiles): hand-written
//     DMMA kernels -- a fused forward sweep (all layers and all steps in one launch, two warps per 8-path tile, weights streamed through
//     a TMA slab ring, relu / Euler-Maruyama / residual on the fragments), a fused cotangent sweep and, when dim and hidden are both
//     even, a fused weight-gradient kernel (see "fused fp64 sweeps" below; odd widths take library GEMMs for [dW | db]); Brownian
//     increments from a counter-based generator (Philox4x32-10 + Box-Muller) in a separate parallel pass;
//   * fp32, and wider networks: one library GEMM per layer (cuBLAS) with hand-written kernels between them (fused Euler-Maruyama
//     with the increments regenerated in place, relu / masks, the loss and its cotangents);
//   * the backward sweep is the exact reverse-mode derivative of the discretised solve (what Tracker computes through the SDE
//     solver in the reference).  Nothing is recomputed: with 80 GB of HBM every step's activations and cotangents stay resident
//     ((4 d + 6 hls) x paths x n_steps elements, 1.5 GB for the benchmark's 10 000 fp64 paths);
//   * every activation matrix carries a constant row of ones below it, and theta stores a layer as vec(W) followed by b, i.e.
//     the column-major out x (in + 1) matrix [W | b]: the forward product over the augmented activations adds the bias for free,
//     and ONE product per layer over all steps at once (k = n_steps x paths) writes [dW | db] straight into the gradient in
//     theta's layout -- no bias kernels, no per-step weight-gradient products;
//   * relu'(0) = 1 as Flux 0.9 / Tracker differentiate max(zero(x), x): the sign bit of a zero activation records the side;
//   * fixed-step Euler-Maruyama (the script's LambaEM is EM with step-size control; for this family X is exact under EM and only
//     the u-quadrature depends on dt);
//   * the whole iteration -- forward, loss, backward, ADAM -- is replayed as one CUDA graph; the per-iteration seed lives in
//     device memory so the graph's arguments never change.
#include <cublas_v2.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <string>
#include <vector>

#include "../../include/b200ude.h"

namespace {

std::string g_bsde_create_error;

// ---- Philox4x32-10 -------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void philox4x32(uint32_t &c0, uint32_t &c1, uint32_t &c2, uint32_t &c3, uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
}
// four standard normals for (path, component block q, step): counter (path, q, step, 0), key = seed; Box-Muller on (x + 0.5) 2^-32
__device__ __forceinline__ void normals4(uint64_t seed, uint32_t path, uint32_t q, uint32_t step, double (&z)[4])
{
    uint32_t c0 = path, c1 = q, c2 = step, c3 = 0u;
    philox4x32(c0, c1, c2, c3, (uint32_t)seed, (uint32_t)(seed >> 32));
    const double s32 = 2.3283064365386963e-10;   // 2^-32
    const double u0 = ((double)c0 + 0.5) * s32, u1 = ((double)c1 + 0.5) * s32, u2 = ((double)c2 + 0.5) * s32, u3 = ((double)c3 + 0.5) * s32;
    const double ra = sqrt(-2.0 * log(u0)), rb = sqrt(-2.0 * log(u2));
    double sa, ca, sb, cb;
    sincos(6.283185307179586 * u1, &sa, &ca);
    sincos(6.283185307179586 * u3, &sb, &cb);
    z[0] = ra * ca; z[1] = ra * sa; z[2] = rb * cb; z[3] = rb * sb;
}

// Brownian increments of a whole iteration for the fused sweeps: dW[n][path][m] = sqrt(dt) * normal(path, m, n), one thread per
// (step, path, block of 4 components).  A separate, fully parallel pass: inside the forward sweep the fp64 log / sincos chains of the
// Box-Muller transform sit on every warp's critical path.
__global__ void k_dw_tape(double *__restrict__ dW, const uint64_t *seed, uint32_t path0, int M, int N, int d, double sq)
{
    const int nq = (d + 3) / 4;
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long)N * M * nq) return;
    const int q = (int)(i % nq), m = (int)((i / nq) % M), n = (int)(i / ((long)nq * M));
    double nz[4];
    normals4(*seed, path0 + (uint32_t)m, (uint32_t)q, (uint32_t)n, nz);
    double *o = dW + ((size_t)n * M + m) * d + 4 * q;
#pragma unroll
    for (int e = 0; e < 4; ++e)
        if (4 * q + e < d) o[e] = sq * nz[e];
}

// ---- element-wise kernels (R = float or double) ------------------------------------------------------------------------------
// constant rows of the augmented activations for all steps: IN[n] = [X_n (d rows); t_n; 1], H_k[n] = [h (hls rows); 1]
template <class R>
__global__ void k_init_aug(R *IN, R *H1, R *H2, R *H3, int d, int hls, int ldh, int M, int n_steps, double dt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (n_steps + 1) * M) return;
    const int n = i / M;
    IN[(size_t)i * (d + 2) + d] = (R)(n * dt);
    IN[(size_t)i * (d + 2) + d + 1] = (R)1;
    if (n < n_steps) {
        for (int k = hls; k < ldh; ++k) {   // the ones row, then zero padding up to the (even) leading dimension
            const R v = k == hls ? (R)1 : (R)0;
            H1[(size_t)i * ldh + k] = v; H2[(size_t)i * ldh + k] = v; H3[(size_t)i * ldh + k] = v;
        }
    }
}
template <class R>
__global__ void k_init_paths(R *IN0, R *u, const R *x0, const R *u0_val, int d, int M)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < d * M) IN0[(size_t)(i / d) * (d + 2) + i % d] = x0[i % d];
    if (i < M) u[i] = *u0_val;
}
// u0 net (one column): A[n] += b, relu on hidden layers
template <class R>
__global__ void k_bias_act(R *A, const R *b, int n, int M, int relu)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * M) return;
    const R a = A[i] + b[i % n];
    A[i] = relu ? (a >= (R)0 ? a : (R)(-0.0)) : a;
}
// relu in place on the first n rows of an [ld x M] matrix; the side of a zero is kept in its sign bit (+0: a >= 0, derivative 1;
// -0: a < 0, derivative 0)
template <class R>
__global__ void k_relu(R *A, int n, int ld, int M)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * M) return;
    const size_t j = (size_t)(i / n) * ld + i % n;
    const R a = A[j];
    if (!(a >= (R)0)) A[j] = (R)(-0.0);
}
// C [n x M] (ld n) *= relu'(H), H [ldh x M]
template <class R>
__global__ void k_relu_mask(R *C, const R *H, int n, int ldh, int M)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n * M && signbit(H[(size_t)(i / n) * ldh + i % n])) C[i] = (R)0;
}
// Euler-Maruyama step, one warp per path: u += lambda |z|^2 dt + z . dW, X_{n+1} = X_n + s dW  (X rows of IN[n] -> IN[n + 1])
template <class R>
__global__ void k_em_step(const R *Xn, R *Xn1, R *u, const R *Z, const uint64_t *seed, uint32_t path0, int step, int d, int M, double dt, double lam,
                          double s)
{
    const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (m >= M) return;
    const double sq = sqrt(dt);
    double zz = 0.0, zw = 0.0;
    for (int q = lane; 4 * q < d; q += 32) {
        double nz[4];
        normals4(*seed, path0 + (uint32_t)m, (uint32_t)q, (uint32_t)step, nz);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int c = 4 * q + e;
            if (c < d) {
                const double dw = sq * nz[e], z = (double)Z[(size_t)m * d + c];
                zz = fma(z, z, zz);
                zw = fma(z, dw, zw);
                Xn1[(size_t)m * (d + 2) + c] = (R)((double)Xn[(size_t)m * (d + 2) + c] + s * dw);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { zz += __shfl_xor_sync(0xffffffffu, zz, o); zw += __shfl_xor_sync(0xffffffffu, zw, o); }
    if (lane == 0) u[m] = (R)((double)u[m] + lam * zz * dt + zw);
}
// cotangent of z_n: ubar (2 lambda z dt + dW_n)   (dW regenerated from the counters)
template <class R>
__global__ void k_zbar(R *Zb, const R *Z, const R *ubar, const uint64_t *seed, uint32_t path0, int step, int d, int M, double dt, double lam)
{
    const int nq = (d + 3) / 4;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nq * M) return;
    const int q = i % nq, m = i / nq;
    double nz[4];
    normals4(*seed, path0 + (uint32_t)m, (uint32_t)q, (uint32_t)step, nz);
    const double sq = sqrt(dt), ub = (double)ubar[m];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int c = 4 * q + e;
        if (c < d) Zb[(size_t)m * d + c] = (R)(ub * (2.0 * lam * (double)Z[(size_t)m * d + c] * dt + sq * nz[e]));
    }
}
// r = g(X_T) - u_T per path (one warp per path), ubar = -2 r / M_total; X = the X rows of IN[n_steps]
template <class R>
__global__ void k_residual(const R *X, const R *u, R *r2, R *ubar, int d, int M, double ga, double gb, double inv_total)
{
    const int m = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (m >= M) return;
    double nn = 0.0;
    for (int c = lane; c < d; c += 32) { const double x = (double)X[(size_t)m * (d + 2) + c]; nn = fma(x, x, nn); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nn += __shfl_xor_sync(0xffffffffu, nn, o);
    if (lane == 0) {
        const double r = log(ga + gb * nn) - (double)u[m];
        r2[m] = (R)(r * r);
        ubar[m] = (R)(-2.0 * r * inv_total);
    }
}
// fixed-order sums: out[0] = scale0 * sum a, out[1] = sum b   (one CTA)
template <class R>
__global__ void k_sum2(const R *a, const R *b, int M, double scale0, R *out0, R *out1)
{
    __shared__ double sa[256], sb[256];
    double x = 0.0, y = 0.0;
    for (int i = threadIdx.x; i < M; i += 256) { x += (double)a[i]; y += (double)b[i]; }
    sa[threadIdx.x] = x; sb[threadIdx.x] = y;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) { sa[threadIdx.x] += sa[threadIdx.x + o]; sb[threadIdx.x] += sb[threadIdx.x + o]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { *out0 = (R)(scale0 * sa[0]); *out1 = (R)sb[0]; }
}
template <class R>
__global__ void k_fill(R *p, R v, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
// Flux.ADAM on theta; also records the pre-update loss / u0(x0) of this iteration and advances the seed
template <class R>
__global__ void k_adam(R *theta, R *m, R *v, const R *grad, int P, int *t_dev, uint64_t *seed, double eta, double b1, double b2, double eps,
                       const R *loss, const R *u0_val, R *loss_hist, R *u0_hist, int t_base)
{
    __shared__ int s_t;
    if (threadIdx.x == 0) s_t = *t_dev + 1;
    __syncthreads();
    const int t = s_t;
    const double c1 = 1.0 / (1.0 - pow(b1, (double)t)), c2 = 1.0 / (1.0 - pow(b2, (double)t));
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const double g = (double)grad[i];
        const double mm = b1 * (double)m[i] + (1.0 - b1) * g, vv = b2 * (double)v[i] + (1.0 - b2) * g * g;
        m[i] = (R)mm; v[i] = (R)vv;
        theta[i] = (R)((double)theta[i] - eta * (mm * c1) / (sqrt(vv * c2) + eps));
    }
    if (threadIdx.x == 0) {
        if (loss_hist) loss_hist[t - 1 - t_base] = *loss;
        if (u0_hist) u0_hist[t - 1 - t_base] = *u0_val;
        *t_dev = t;
        *seed += 1;
    }
}

// ---- fused fp64 sweeps (DMMA) ---------------------------------------------------------------------------------------------
// One warp owns 8 paths and carries them through the whole network in the fragment layout of mma.sync.m8n8k4.f64: M = the 8 paths,
// N = the units of a layer (<= FT tiles of 8), K = the layer's inputs + the bias row.  The D fragment of a layer (path lane >> 2, unit
// pair 2 (lane & 3)) is written as one 16-byte word into the warp's own shared-memory rows and read back as the A fragment of the next
// layer -- no other warp ever touches those rows.  The weights (0.4 MB in fp64: more than an SM's shared memory) stream through a
// two-slab ring in shared memory that all warps of the CTA share: a zero-padded operand copy of theta is cut into slabs of FSR
// contraction rows x FLD (unit-contiguous, already in the padded shared-memory layout), and ONE elected thread moves a whole slab
// with one TMA bulk copy (cp.async.bulk + mbarrier transaction count) two slabs ahead of the math; a slab is released by a CTA barrier.
// (Reading the B fragments straight from L2 instead made every warp stream all weights: 10 TFLOP/s, L2-bound.)  relu (with the side
// of a zero in its sign bit), the bias (K includes the ones row), the Euler-Maruyama update, the Brownian increments, the terminal
// residual (forward) and the cotangent of z, the relu' masks (backward) are applied to the fragments in registers; the tape
// (activations, cotangents) is written from the fragments for the batched weight-gradient GEMMs.
constexpr int FT = 14;        // unit tiles per layer: widths up to 112
constexpr int FW = 8 * FT;    // padded unit count
constexpr int FLD = 116;      // row stride in doubles of activations and slabs (= 4 mod 16: conflict-free 8-byte fragment reads per half warp)
constexpr int FSR = 16;       // contraction rows per slab
constexpr int FSLAB = FSR * FLD;                          // doubles per slab
constexpr uint32_t FSLAB_BYTES = FSLAB * sizeof(double);   // 14 848
constexpr int FWPC = 4;       // warps per CTA; three CTAs per SM run out of step with one another, so one's barrier / tape-latency /
                              // Euler-Maruyama phases are covered by the others' DMMA phases
constexpr int FWF = 4;        // forward sweep: warps per CTA (one per scheduler: the warps of a CTA then share their schedulers with equally
                              // many others and run at the same pace -- with 5 the ring made the faster ones wait for the slower)
constexpr int FMAXSLABS = 32;

struct FusedArgs {
    const double *slabs;   // forward slabs, then backward slabs
    int n_f, n_b;          // slab counts
    // per slab: layer, first contraction row, k-steps of 4 valid rows, last slab of its layer?
    unsigned char f_layer[FMAXSLABS], f_k0[FMAXSLABS], f_ks[FMAXSLABS], f_last[FMAXSLABS];
    unsigned char b_layer[FMAXSLABS], b_k0[FMAXSLABS], b_ks[FMAXSLABS], b_last[FMAXSLABS];
    double *IN, *H[3], *Z, *Zb, *C[3], *u, *r2, *ubar;   // Z holds G = 2 lambda z dt + dW here (zbar = ubar G)
    const double *dW;      // Brownian increments [n][path][d] of this iteration (k_dw_tape)
    uint32_t *mask;        // relu' bits of the hidden layers: word ((n * 3 + l) * M + path) * 4 + (lane & 3), bit 2 nt + e
    const double *x0, *u0;
    const uint64_t *seed;
    uint32_t path0;
    int M, N, d, hl, ldh;
    double dt, lam, s, ga, gb, inv_total;
};

__device__ __forceinline__ void dmma(double (&c)[2], double a, double b)
{
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t phase)
{
    uint32_t done = 0;
    while (!done)
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(bar), "r"(phase) : "memory");
}
// the slab ring: FRING buffers with one "full" mbarrier each; the stream of slabs (n_slabs per round, round after round) is
// consumed in order; (cb, cph) = buffer and barrier phase of the slab being consumed
constexpr int FRING = 3;
struct SlabShared {       // per-CTA bookkeeping in shared memory
    int done[FRING];      // warps that have finished with the slab in buffer b
};
struct SlabRing {
    double *base;         // FRING slabs
    uint32_t bar0;        // FRING "full" mbarriers, 8 bytes apart
    SlabShared *sh;
    const double *src;
    long total, idx;      // slabs of this CTA's stream; index of the slab being consumed
    int n_slabs, nwarps;  // slabs per round (the stream repeats round after round)
    int depth;            // buffers in use (<= FRING)
    int cb, cph;          // buffer and barrier phase of the slab being consumed
    __device__ __forceinline__ void issue(long i, int b) const   // one thread: slab i of the stream -> buffer b
    {
        if (i >= total) return;
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(base + (size_t)b * FSLAB), br = bar0 + 8u * b;
        const double *g = src + (size_t)(i % n_slabs) * FSLAB;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(br), "r"(FSLAB_BYTES) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(g), "r"(FSLAB_BYTES),
                     "r"(br)
                     : "memory");
    }
    __device__ __forceinline__ const double *cur() const { return base + (size_t)cb * FSLAB; }
    __device__ __forceinline__ void wait_cur() const { mbar_wait(bar0 + 8u * cb, (uint32_t)cph); }
    // This warp is done with the current slab.  No CTA barrier: the LAST warp to finish refills the buffer with the slab FRING ahead,
    // so the warps of a CTA drift freely within the ring's depth (a barrier per slab cost the forward sweep a sixth of its time).
    __device__ __forceinline__ void release(int lane)
    {
        __syncwarp();
        if (lane == 0) {   // release (this warp's reads of the slab, gathered by __syncwarp) ... acquire (everybody's) around the counter
            __threadfence_block();
            if (atomicAdd(&sh->done[cb], 1) == nwarps - 1) {
                __threadfence_block();
                sh->done[cb] = 0;
                issue(idx + depth, cb);
            }
        }
        cb = cb == depth - 1 ? 0 : cb + 1;
        if (cb == 0) cph ^= 1;
        ++idx;
    }
};
// One slab of a layer: acc[nt] += sum over its FSR rows of in[r][k0 + k] * slab[k][8 nt + r'].  Each B fragment register is reloaded
// for the next k-step right behind the DMMA that read it (the other warps of the scheduler cover the load latency); rows beyond a
// layer's inputs are zero in the slab and finite in `in`, so every slab runs all its k-steps.
__device__ __forceinline__ void slab_mma(const double *in, const SlabRing &ring, int k0, int r, int c, double (&acc)[FT][2])
{
    ring.wait_cur();
    const double *wp = ring.cur() + c * FLD + r;
    const double *ap = in + r * FLD + k0 + c;
    double bv[FT];
#pragma unroll
    for (int nt = 0; nt < FT; ++nt) bv[nt] = wp[8 * nt];
#pragma unroll
    for (int ks = 0; ks < FSR / 4; ++ks) {
        const double av = ap[4 * ks];
#pragma unroll
        for (int nt = 0; nt < FT; ++nt) {
            dmma(acc[nt], av, bv[nt]);
            if (ks < FSR / 4 - 1) bv[nt] = wp[(ks + 1) * 4 * FLD + 8 * nt];
        }
    }
}
// shared-memory carve-up: [FRING slabs][per warp: one activation buffer of 8 rows, updated in place][FRING mbarriers][SlabShared]
__device__ __forceinline__ void fused_setup(double *fsm, int nwarps, SlabRing &ring, const double *src, int n_slabs, long total, int depth = FRING,
                                            int act_rows = 0)
{
    ring.base = fsm;
    ring.depth = depth;
    uint64_t *bars = reinterpret_cast<uint64_t *>(fsm + depth * FSLAB + (size_t)(act_rows ? act_rows : nwarps * 8) * FLD);
    ring.bar0 = (uint32_t)__cvta_generic_to_shared(bars);
    ring.sh = reinterpret_cast<SlabShared *>(bars + FRING);
    ring.src = src; ring.n_slabs = n_slabs; ring.total = total; ring.idx = 0; ring.nwarps = nwarps;
    ring.cb = 0; ring.cph = 0;
    if (threadIdx.x == 0) {
#pragma unroll
        for (int i = 0; i < FRING; ++i) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(ring.bar0 + 8u * i));
            ring.sh->done[i] = 0;
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 0; i < depth; ++i) ring.issue(i, i);
    }
}

__global__ void __launch_bounds__(32 * FWF, 3) k_fused_forward(const FusedArgs a)
{
    extern __shared__ __align__(16) double fsm[];
    const int nwarps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, c = lane & 3;
    SlabRing ring;
    fused_setup(fsm, nwarps, ring, a.slabs, a.n_f, (long)a.n_f * a.N);
    double *buf = fsm + FRING * FSLAB + (size_t)warp * 8 * FLD;
    const int path = (blockIdx.x * nwarps + warp) * 8 + r;
    const bool live = path < a.M;
    const size_t pc = (size_t)(live ? path : a.M - 1);
    const int d = a.d, hl = a.hl;
    double u = *a.u0;
    const size_t s_in = (size_t)(d + 2) * a.M, s_h = (size_t)a.ldh * a.M, s_z = (size_t)d * a.M;
    const bool even_d = (d & 1) == 0;   // then (path * ld + m) is even for the lane's pairs: 16-byte tape accesses
    double X[FT][2];   // the warp's paths in the fragment layout
#pragma unroll
    for (int nt = 0; nt < FT; ++nt) {
        const int m = 8 * nt + 2 * c;
        X[nt][0] = m < d ? a.x0[m] : 0.0;
        X[nt][1] = m + 1 < d ? a.x0[m + 1] : 0.0;
    }
    for (int n = 0; n <= a.N; ++n) {
        // X_n -> the tape (rows d, d + 1 of IN hold t_n and 1 already) and the warp's input rows [X; t; 1; 0...]
        double *inx = a.IN + n * s_in + pc * (d + 2);
#pragma unroll
        for (int nt = 0; nt < FT; ++nt) {
            const int m = 8 * nt + 2 * c;
            if (live && even_d && m < d) *reinterpret_cast<double2 *>(inx + m) = make_double2(X[nt][0], X[nt][1]);
            else {
                if (live && m < d) inx[m] = X[nt][0];
                if (live && m + 1 < d) inx[m + 1] = X[nt][1];
            }
            *reinterpret_cast<double2 *>(buf + r * FLD + m) = make_double2(X[nt][0], X[nt][1]);
        }
        if (n == a.N) break;
        {   // the step's Brownian increments towards L2 while the layers run (8 rows of d doubles: lane i asks for lines i, i + 32)
            const int p0 = path - r, rows = p0 < a.M ? (a.M - p0 < 8 ? a.M - p0 : 8) : 0;
            const char *w0 = reinterpret_cast<const char *>(a.dW + n * s_z + (size_t)(rows ? p0 : 0) * d);
            const size_t bytes = (size_t)rows * d * sizeof(double);
            for (size_t o = (size_t)lane * 128; o < bytes; o += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(w0 + o));
        }
        __syncwarp();
        if (c == 0) { buf[r * FLD + d] = n * a.dt; buf[r * FLD + d + 1] = 1.0; }
        __syncwarp();
        double acc[FT][2];
#pragma unroll 1
        for (int i = 0; i < a.n_f; ++i) {
            const int l = a.f_layer[i];
            if (a.f_k0[i] == 0) {
#pragma unroll
                for (int nt = 0; nt < FT; ++nt) acc[nt][0] = acc[nt][1] = 0.0;
            }
            slab_mma(buf, ring, a.f_k0[i], r, c, acc);
            ring.release(lane);
            if (!a.f_last[i]) continue;
            if (l < 3) {   // the layer's output replaces its input in the warp's own rows
                double *hp = a.H[l] + n * s_h + pc * a.ldh;
                uint32_t bits = 0u;
#pragma unroll
                for (int nt = 0; nt < FT; ++nt) {
                    const int m = 8 * nt + 2 * c;
                    const bool neg0 = !(acc[nt][0] >= 0.0), neg1 = !(acc[nt][1] >= 0.0);
                    const double h0 = neg0 ? -0.0 : acc[nt][0], h1 = neg1 ? -0.0 : acc[nt][1];
                    bits |= (neg0 ? 1u : 0u) << (2 * nt) | (neg1 ? 1u : 0u) << (2 * nt + 1);
                    *reinterpret_cast<double2 *>(buf + r * FLD + m) = make_double2(h0, h1);
                    if (live && m + 1 < hl) *reinterpret_cast<double2 *>(hp + m) = make_double2(h0, h1);   // ldh is even
                    else if (live && m < hl) hp[m] = h0;
                }
                if (live) a.mask[((size_t)(n * 3 + l) * a.M + pc) * 4 + c] = bits;
                __syncwarp();
                if (c == 0) buf[r * FLD + hl] = 1.0;   // the ones row (the padded weights are zero beyond it)
                __syncwarp();
            }
        }
        // acc = z_n for the warp's paths: Euler-Maruyama update in the fragment layout
        double zz = 0.0, zw = 0.0;
        double *zp = a.Z + n * s_z + pc * d;
        const double *wn = a.dW + n * s_z + pc * d;
#pragma unroll
        for (int nt = 0; nt < FT; ++nt) {
            const int m = 8 * nt + 2 * c;
            if (even_d && m < d) {
                const double2 dw = *reinterpret_cast<const double2 *>(wn + m);
                const double z0 = acc[nt][0], z1 = acc[nt][1];
                zz = fma(z0, z0, fma(z1, z1, zz)); zw = fma(z0, dw.x, fma(z1, dw.y, zw));
                X[nt][0] += a.s * dw.x; X[nt][1] += a.s * dw.y;
                if (live) *reinterpret_cast<double2 *>(zp + m) = make_double2(2.0 * a.lam * z0 * a.dt + dw.x, 2.0 * a.lam * z1 * a.dt + dw.y);   // d(u_T)/d(z_n) / ubar
            } else if (m < d) {
                const double dw0 = wn[m], z0 = acc[nt][0];
                zz = fma(z0, z0, zz); zw = fma(z0, dw0, zw);
                X[nt][0] += a.s * dw0;
                if (live) zp[m] = 2.0 * a.lam * z0 * a.dt + dw0;
                if (m + 1 < d) {
                    const double dw1 = wn[m + 1], z1 = acc[nt][1];
                    zz = fma(z1, z1, zz); zw = fma(z1, dw1, zw);
                    X[nt][1] += a.s * dw1;
                    if (live) zp[m + 1] = 2.0 * a.lam * z1 * a.dt + dw1;
                }
            }
        }
        zz += __shfl_xor_sync(0xffffffffu, zz, 1); zw += __shfl_xor_sync(0xffffffffu, zw, 1);
        zz += __shfl_xor_sync(0xffffffffu, zz, 2); zw += __shfl_xor_sync(0xffffffffu, zw, 2);
        u += a.lam * zz * a.dt + zw;
        __syncwarp();
    }
    double nn = 0.0;
#pragma unroll
    for (int nt = 0; nt < FT; ++nt) nn = fma(X[nt][0], X[nt][0], fma(X[nt][1], X[nt][1], nn));
    nn += __shfl_xor_sync(0xffffffffu, nn, 1);
    nn += __shfl_xor_sync(0xffffffffu, nn, 2);
    if (live && c == 0) {
        const double res = log(a.ga + a.gb * nn) - u;
        a.u[path] = u;
        a.r2[path] = res * res;
        a.ubar[path] = -2.0 * res * a.inv_total;
    }
}

// The forward sweep with a path tile shared by TWO warps, each owning half of a layer's unit tiles: twice as many warps on the same
// DMMA work (1 250 tiles of 8 paths are only 2.1 warps per scheduler, too few to cover each warp's own non-DMMA phases), finer balance.
// The pair meets at a named barrier after every layer (activation rows, relu' bits) and after the Euler-Maruyama update (the two
// halves of |z|^2 and z . dW); the activation rows are double-buffered because one warp's output units are the other's inputs.
constexpr int FPW = 10;        // warps per CTA: five pairs, two CTAs per SM
constexpr int FHT = FT / 2;    // unit tiles per warp
constexpr int FP_DEPTH = 2;    // slab ring depth of this kernel (shared memory: 2 slabs + 5 pairs x 2 x 8 rows = 104 KB per CTA)
struct PairExch {
    double zz[2][8], zw[2][8], nn[2][8];
    uint32_t bits[2][2][32];   // [layer parity][half][lane]
};
__device__ __forceinline__ void pair_sync(int pair) { asm volatile("bar.sync %0, 64;" ::"r"(pair + 1) : "memory"); }

__device__ __forceinline__ void slab_mma_half(const double *in, const SlabRing &ring, int k0, int r, int c, int uoff, double (&acc)[FHT][2])
{
    ring.wait_cur();
    const double *wp = ring.cur() + c * FLD + r + uoff;
    const double *ap = in + r * FLD + k0 + c;
    double bv[FHT];
#pragma unroll
    for (int nt = 0; nt < FHT; ++nt) bv[nt] = wp[8 * nt];
#pragma unroll
    for (int ks = 0; ks < FSR / 4; ++ks) {
        const double av = ap[4 * ks];
#pragma unroll
        for (int nt = 0; nt < FHT; ++nt) {
            dmma(acc[nt], av, bv[nt]);
            if (ks < FSR / 4 - 1) bv[nt] = wp[(ks + 1) * 4 * FLD + 8 * nt];
        }
    }
}

__global__ void __launch_bounds__(32 * FPW, 2) k_fused_forward2(const FusedArgs a)
{
    extern __shared__ __align__(16) double fsm[];
    constexpr int NP = FPW / 2;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, c = lane & 3;
    const int pair = warp >> 1, half = warp & 1, uoff = 8 * FHT * half;
    SlabRing ring;
    fused_setup(fsm, FPW, ring, a.slabs, a.n_f, (long)a.n_f * a.N, FP_DEPTH, NP * 2 * 8);
    double *in = fsm + FP_DEPTH * FSLAB + (size_t)pair * 2 * 8 * FLD, *out = in + 8 * FLD;
    PairExch *ex = reinterpret_cast<PairExch *>(fsm + FP_DEPTH * FSLAB + (size_t)NP * 2 * 8 * FLD + FRING + (sizeof(SlabShared) + 7) / 8) + pair;
    const int path = (blockIdx.x * NP + pair) * 8 + r;
    const bool live = path < a.M;
    const size_t pc = (size_t)(live ? path : a.M - 1);
    const int d = a.d, hl = a.hl;
    double u = *a.u0;
    const size_t s_in = (size_t)(d + 2) * a.M, s_h = (size_t)a.ldh * a.M, s_z = (size_t)d * a.M;
    const bool even_d = (d & 1) == 0;
    const int ones_half = hl >= 8 * FHT ? 1 : 0;
    double X[FHT][2];   // this warp's components of the pair's paths
#pragma unroll
    for (int nt = 0; nt < FHT; ++nt) {
        const int m = uoff + 8 * nt + 2 * c;
        X[nt][0] = m < d ? a.x0[m] : 0.0;
        X[nt][1] = m + 1 < d ? a.x0[m + 1] : 0.0;
    }
    for (int n = 0; n <= a.N; ++n) {
        double *inx = a.IN + n * s_in + pc * (d + 2);
#pragma unroll
        for (int nt = 0; nt < FHT; ++nt) {
            const int m = uoff + 8 * nt + 2 * c;
            if (live && even_d && m < d) *reinterpret_cast<double2 *>(inx + m) = make_double2(X[nt][0], X[nt][1]);
            else {
                if (live && m < d) inx[m] = X[nt][0];
                if (live && m + 1 < d) inx[m + 1] = X[nt][1];
            }
            *reinterpret_cast<double2 *>(in + r * FLD + m) = make_double2(X[nt][0], X[nt][1]);
        }
        if (n == a.N) break;
        if (half == 0) {   // the step's Brownian increments towards L2 while the layers run
            const int p0 = path - r, rows = p0 < a.M ? (a.M - p0 < 8 ? a.M - p0 : 8) : 0;
            const char *w0 = reinterpret_cast<const char *>(a.dW + n * s_z + (size_t)(rows ? p0 : 0) * d);
            const size_t bytes = (size_t)rows * d * sizeof(double);
            for (size_t o = (size_t)lane * 128; o < bytes; o += 32 * 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(w0 + o));
        }
        pair_sync(pair);
        if (half == 0 && c == 0) { in[r * FLD + d] = n * a.dt; in[r * FLD + d + 1] = 1.0; }
        pair_sync(pair);
        double acc[FHT][2];
#pragma unroll 1
        for (int i = 0; i < a.n_f; ++i) {
            const int l = a.f_layer[i];
            if (a.f_k0[i] == 0) {
#pragma unroll
                for (int nt = 0; nt < FHT; ++nt) acc[nt][0] = acc[nt][1] = 0.0;
            }
            slab_mma_half(in, ring, a.f_k0[i], r, c, uoff, acc);
            ring.release(lane);
            if (!a.f_last[i] || l == 3) continue;
            double *hp = a.H[l] + n * s_h + pc * a.ldh;
            uint32_t bits = 0u;
#pragma unroll
            for (int nt = 0; nt < FHT; ++nt) {
                const int m = uoff + 8 * nt + 2 * c;
                const bool neg0 = !(acc[nt][0] >= 0.0), neg1 = !(acc[nt][1] >= 0.0);
                const double h0 = neg0 ? -0.0 : acc[nt][0], h1 = neg1 ? -0.0 : acc[nt][1];
                bits |= (neg0 ? 1u : 0u) << (2 * nt) | (neg1 ? 1u : 0u) << (2 * nt + 1);
                *reinterpret_cast<double2 *>(out + r * FLD + m) = make_double2(h0, h1);
                if (live && m + 1 < hl) *reinterpret_cast<double2 *>(hp + m) = make_double2(h0, h1);   // ldh is even
                else if (live && m < hl) hp[m] = h0;
            }
            ex->bits[l & 1][half][lane] = bits;
            if (half == ones_half) {
                __syncwarp();
                if (c == 0) out[r * FLD + hl] = 1.0;   // the ones row (the padded weights are zero beyond it)
            }
            pair_sync(pair);
            if (half == 0 && live) a.mask[((size_t)(n * 3 + l) * a.M + pc) * 4 + c] = bits | (ex->bits[l & 1][1][lane] << (2 * FHT));
            double *t = in; in = out; out = t;
        }
        // acc = this warp's components of z_n: Euler-Maruyama update; the pair adds its halves of |z|^2 and z . dW
        double zz = 0.0, zw = 0.0;
        double *zp = a.Z + n * s_z + pc * d;
        const double *wn = a.dW + n * s_z + pc * d;
#pragma unroll
        for (int nt = 0; nt < FHT; ++nt) {
            const int m = uoff + 8 * nt + 2 * c;
            if (even_d && m < d) {
                const double2 dw = *reinterpret_cast<const double2 *>(wn + m);
                const double z0 = acc[nt][0], z1 = acc[nt][1];
                zz = fma(z0, z0, fma(z1, z1, zz)); zw = fma(z0, dw.x, fma(z1, dw.y, zw));
                X[nt][0] += a.s * dw.x; X[nt][1] += a.s * dw.y;
                if (live) *reinterpret_cast<double2 *>(zp + m) = make_double2(2.0 * a.lam * z0 * a.dt + dw.x, 2.0 * a.lam * z1 * a.dt + dw.y);
            } else if (m < d) {
                const double dw0 = wn[m], z0 = acc[nt][0];
                zz = fma(z0, z0, zz); zw = fma(z0, dw0, zw);
                X[nt][0] += a.s * dw0;
                if (live) zp[m] = 2.0 * a.lam * z0 * a.dt + dw0;
                if (m + 1 < d) {
                    const double dw1 = wn[m + 1], z1 = acc[nt][1];
                    zz = fma(z1, z1, zz); zw = fma(z1, dw1, zw);
                    X[nt][1] += a.s * dw1;
                    if (live) zp[m + 1] = 2.0 * a.lam * z1 * a.dt + dw1;
                }
            }
        }
        zz += __shfl_xor_sync(0xffffffffu, zz, 1); zw += __shfl_xor_sync(0xffffffffu, zw, 1);
        zz += __shfl_xor_sync(0xffffffffu, zz, 2); zw += __shfl_xor_sync(0xffffffffu, zw, 2);
        if (c == 0) { ex->zz[half][r] = zz; ex->zw[half][r] = zw; }
        pair_sync(pair);
        u += a.lam * (ex->zz[0][r] + ex->zz[1][r]) * a.dt + (ex->zw[0][r] + ex->zw[1][r]);
        // (the next writes to ex->zz / zw come a whole step later, behind several pair barriers)
    }
    double nn = 0.0;
#pragma unroll
    for (int nt = 0; nt < FHT; ++nt) nn = fma(X[nt][0], X[nt][0], fma(X[nt][1], X[nt][1], nn));
    nn += __shfl_xor_sync(0xffffffffu, nn, 1);
    nn += __shfl_xor_sync(0xffffffffu, nn, 2);
    if (c == 0) ex->nn[half][r] = nn;
    pair_sync(pair);
    if (live && c == 0 && half == 0) {
        const double res = log(a.ga + a.gb * (ex->nn[0][r] + ex->nn[1][r])) - u;
        a.u[path] = u;
        a.r2[path] = res * res;
        a.ubar[path] = -2.0 * res * a.inv_total;
    }
}

// cotangents: a warp takes one (step, 8-path tile) at a time: zbar = ubar G -> hidden 3 -> hidden 2 -> hidden 1; persistent CTAs walk
// the task groups (the slab stream just keeps repeating)
__global__ void __launch_bounds__(32 * FWPC, 3) k_fused_backward(const FusedArgs a)
{
    extern __shared__ __align__(16) double fsm[];
    const int nwarps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, c = lane & 3;
    const int tiles = (a.M + 7) / 8;
    const long tasks = (long)tiles * a.N, groups = (tasks + nwarps - 1) / nwarps;
    const long my_groups = groups > blockIdx.x ? (groups - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    SlabRing ring;
    fused_setup(fsm, nwarps, ring, a.slabs + (size_t)a.n_f * FSLAB, a.n_b, (long)a.n_b * my_groups);
    double *buf = fsm + FRING * FSLAB + (size_t)warp * 8 * FLD;
    const int d = a.d, hl = a.hl;
    const size_t s_z = (size_t)d * a.M, s_c = (size_t)hl * a.M;
    const bool even_d = (d & 1) == 0, even_h = (hl & 1) == 0;
    for (long g = blockIdx.x; g < groups; g += gridDim.x) {
        const long task = g * nwarps + warp;
        const bool task_live = task < tasks;
        const int n = (int)((task_live ? task : tasks - 1) / tiles), p0 = (int)((task_live ? task : tasks - 1) % tiles) * 8;
        const int path = p0 + r;
        const bool live = task_live && path < a.M;
        const size_t pc = (size_t)(path < a.M ? path : a.M - 1);
        const double ub = a.ubar[pc];
        const double *gp = a.Z + n * s_z + pc * d;
        double *zb = a.Zb + n * s_z + pc * d;
        uint32_t bits[3];
#pragma unroll
        for (int l = 0; l < 3; ++l) bits[l] = a.mask[((size_t)(n * 3 + l) * a.M + pc) * 4 + c];
#pragma unroll
        for (int nt = 0; nt < FT; ++nt) {
            const int m = 8 * nt + 2 * c;
            double b0 = 0.0, b1 = 0.0;
            if (even_d && m < d) {   // (path * d + m) is even: 16-byte tape accesses
                const double2 gg = *reinterpret_cast<const double2 *>(gp + m);
                b0 = ub * gg.x; b1 = ub * gg.y;
                if (live) *reinterpret_cast<double2 *>(zb + m) = make_double2(b0, b1);
            } else if (m < d) {
                b0 = ub * gp[m];
                if (live) zb[m] = b0;
                if (m + 1 < d) {
                    b1 = ub * gp[m + 1];
                    if (live) zb[m + 1] = b1;
                }
            }
            *reinterpret_cast<double2 *>(buf + r * FLD + m) = make_double2(b0, b1);
        }
        __syncwarp();
        double acc[FT][2];
#pragma unroll 1
        for (int i = 0; i < a.n_b; ++i) {
            const int l = a.b_layer[i];
            if (a.b_k0[i] == 0) {
#pragma unroll
                for (int nt = 0; nt < FT; ++nt) acc[nt][0] = acc[nt][1] = 0.0;
            }
            slab_mma(buf, ring, a.b_k0[i], r, c, acc);
            ring.release(lane);
            if (!a.b_last[i]) continue;
            const uint32_t mb = l == 3 ? bits[2] : (l == 2 ? bits[1] : bits[0]);
            double *cp = a.C[l - 1] + n * s_c + pc * hl;
#pragma unroll
            for (int nt = 0; nt < FT; ++nt) {
                const int m = 8 * nt + 2 * c;
                const double c0 = (m < hl && !((mb >> (2 * nt)) & 1u)) ? acc[nt][0] : 0.0;
                const double c1 = (m + 1 < hl && !((mb >> (2 * nt + 1)) & 1u)) ? acc[nt][1] : 0.0;
                if (live && even_h && m + 1 < hl) *reinterpret_cast<double2 *>(cp + m) = make_double2(c0, c1);
                else {
                    if (live && m < hl) cp[m] = c0;
                    if (live && m + 1 < hl) cp[m + 1] = c1;
                }
                *reinterpret_cast<double2 *>(buf + r * FLD + m) = make_double2(c0, c1);
            }
            __syncwarp();
        }
    }
}

// zero-padded operand slabs of the sigmaT_grad_u network (blockIdx.y = slab, one thread per element).  Forward operand of layer l: row k
// holds [W_l | b_l][m][k] (k < in + 1, m < out); backward operand: row i holds W_l[i][j] (i < out, j < in).
struct PackArgs {
    size_t w_off[4];
    int nin[4], nout[4];
};
__global__ void k_pack_slabs(const double *__restrict__ theta, double *dst, const FusedArgs a, const PackArgs q)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x, sl = blockIdx.y;
    if (i >= FSLAB) return;
    const bool backward = sl >= a.n_f;
    const int l = backward ? a.b_layer[sl - a.n_f] : a.f_layer[sl], k0 = backward ? a.b_k0[sl - a.n_f] : a.f_k0[sl];
    const int k = k0 + i / FLD, m = i % FLD, nin = q.nin[l], nout = q.nout[l];
    double v = 0.0;
    if (!backward) { if (k < nin + 1 && m < nout) v = theta[q.w_off[l] + (size_t)k * nout + m]; }
    else           { if (k < nout && m < nin) v = theta[q.w_off[l] + (size_t)m * nout + k]; }
    dst[(size_t)sl * FSLAB + i] = v;
}

// ---- fused weight-gradient products (fp64) ---------------------------------------------------------------------------------------
// [dW | db] of layer l = sum over all (step, path) rows k of cot_l[k][j] * act_l[k][i] -- a 112 x 112 x (steps x paths) product whose long
// dimension is the tape.  One launch for the four layers: blockIdx.y = layer, blockIdx.x = a contiguous range of 16-row chunks of the
// tape; warp w of a CTA owns unit tile w of the layer's outputs (8 values of j) against all 14 input tiles (28 accumulator registers
// x 2), so a k-step is 1 + 14 fragment loads for 14 DMMAs.  Both tapes stream through a four-stage ring of shared memory, every stage
// filled by two TMA bulk copies (the tapes' rows are contiguous: a chunk is one block of memory) and released by its last reader.
// Rows of a tape beyond a layer's width are the next path's data: they only reach output elements that are never stored.  Partial
// sums per CTA, then a fixed-order reduction into the gradient in theta's layout.
constexpr int WGW = FT;          // warps per CTA
constexpr int WGR = 16;          // tape rows per chunk
constexpr int WGD = 4;           // ring depth
constexpr int WGLD = 120;        // row stride bound of a staged tape (>= the largest leading dimension in use: 116)
constexpr int WGSTAGE = 2 * (WGR * WGLD + 16);   // doubles per stage: cot chunk + act chunk (+ slack for the over-read of the last row)
struct WgradArgs {
    const double *cot[4], *act[4];
    int ldc[4], lda[4], nout[4], nact[4];
    long K;                // rows of the tapes (steps x paths)
    double *partial;       // [4][gridDim.x][FW * FW]
};
__global__ void __launch_bounds__(32 * WGW, 1) k_wgrad(const WgradArgs a)
{
    extern __shared__ __align__(16) double fsm[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, r = lane >> 2, c = lane & 3;
    const int l = blockIdx.y, ldc = a.ldc[l], lda = a.lda[l];
    const double *cot = a.cot[l], *act = a.act[l];
    uint64_t *bars = reinterpret_cast<uint64_t *>(fsm + (size_t)WGD * WGSTAGE);
    int *done = reinterpret_cast<int *>(bars + WGD);
    const uint32_t bar0 = (uint32_t)__cvta_generic_to_shared(bars);
    for (int i = threadIdx.x; i < WGD * WGSTAGE; i += blockDim.x) fsm[i] = 0.0;   // stale rows must be finite (they meet zero operands)
    const long chunks = (a.K + WGR - 1) / WGR;
    const long c_lo = chunks * blockIdx.x / gridDim.x, c_hi = chunks * (blockIdx.x + 1) / gridDim.x;
    auto issue = [&](long ch, int b) {   // one thread: chunk ch of both tapes -> stage b
        if (ch >= c_hi) return;
        const long k0 = ch * WGR;
        const int rows = (int)(a.K - k0 < WGR ? a.K - k0 : WGR);
        const uint32_t br = bar0 + 8u * b, bytes_c = (uint32_t)(rows * ldc * 8), bytes_a = (uint32_t)(rows * lda * 8);
        const uint32_t dc = (uint32_t)__cvta_generic_to_shared(fsm + (size_t)b * WGSTAGE), da = dc + (WGR * WGLD + 16) * 8;
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(br), "r"(bytes_c + bytes_a) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dc), "l"(cot + k0 * ldc), "r"(bytes_c), "r"(br) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(da), "l"(act + k0 * lda), "r"(bytes_a), "r"(br) : "memory");
    };
    if (threadIdx.x == 0) {
        for (int i = 0; i < WGD; ++i) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar0 + 8u * i)); done[i] = 0; }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();   // (also: the zero fill is complete before any copy lands)
    if (threadIdx.x == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the zero fill (generic proxy) before the bulk copies (async proxy)
        for (int i = 0; i < WGD; ++i) issue(c_lo + i, i);
    }
    double acc[FT][2];
#pragma unroll
    for (int nt = 0; nt < FT; ++nt) acc[nt][0] = acc[nt][1] = 0.0;
    const int nti = (a.nact[l] + 7) / 8;             // input tiles the layer really has
    const bool wactive = 8 * warp < a.nout[l];
    int b = 0, ph = 0;
    for (long ch = c_lo; ch < c_hi; ++ch) {
        mbar_wait(bar0 + 8u * b, (uint32_t)ph);
        const double *sc = fsm + (size_t)b * WGSTAGE, *sa = sc + WGR * WGLD + 16;
        const long k0 = ch * WGR;
        const int rows = (int)(a.K - k0 < WGR ? a.K - k0 : WGR);
        const double *ap = sc + c * ldc + 8 * warp + r, *bp = sa + c * lda + r;
        if (wactive) {   // (a warp whose unit tile lies beyond the layer's outputs only takes part in the ring protocol)
#pragma unroll
            for (int ks = 0; ks < WGR / 4; ++ks) {
                const double av = 4 * ks + c < rows ? ap[ks * 4 * ldc] : 0.0;   // rows past the tape's end contribute nothing
                double bv[FT];
#pragma unroll
                for (int nt = 0; nt < FT; ++nt)
                    if (nt < nti) bv[nt] = bp[ks * 4 * lda + 8 * nt];
#pragma unroll
                for (int nt = 0; nt < FT; ++nt)
                    if (nt < nti) dmma(acc[nt], av, bv[nt]);
            }
        }
        __syncwarp();
        if (lane == 0) {   // release ... acquire around the reader counter; the last reader refills the stage
            __threadfence_block();
            if (atomicAdd(&done[b], 1) == WGW - 1) {
                __threadfence_block();
                done[b] = 0;
                issue(ch + WGD, b);
            }
        }
        b = b == WGD - 1 ? 0 : b + 1;
        if (b == 0) ph ^= 1;
    }
    double *P = a.partial + ((size_t)l * gridDim.x + blockIdx.x) * (FW * FW);
#pragma unroll
    for (int nt = 0; nt < FT; ++nt) {
        const int j = 8 * warp + r, i = 8 * nt + 2 * c;
        P[(size_t)i * FW + j] = acc[nt][0];
        P[(size_t)(i + 1) * FW + j] = acc[nt][1];
    }
}
// grad[w_off_l + i * nout + j] = sum over the CTAs' partial sums, in a fixed order
__global__ void k_wgrad_reduce(const double *__restrict__ partial, int splits, double *grad, const PackArgs q)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x, l = blockIdx.y;
    if (e >= FW * FW) return;
    const int i = e / FW, j = e % FW;
    if (j >= q.nout[l] || i >= q.nin[l] + 1) return;
    const double *p = partial + (size_t)l * splits * (FW * FW) + e;
    double s = 0.0;
    for (int k = 0; k < splits; ++k) s += p[(size_t)k * (FW * FW)];
    grad[q.w_off[l] + (size_t)i * q.nout[l] + j] = s;
}

inline cublasStatus_t gemm(cublasHandle_t h, cublasOperation_t ta, cublasOperation_t tb, int m, int n, int k, const float *al, const float *A, int lda,
                           const float *B, int ldb, const float *be, float *C, int ldc)
{
    return cublasSgemm(h, ta, tb, m, n, k, al, A, lda, B, ldb, be, C, ldc);
}
inline cublasStatus_t gemm(cublasHandle_t h, cublasOperation_t ta, cublasOperation_t tb, int m, int n, int k, const double *al, const double *A, int lda,
                           const double *B, int ldb, const double *be, double *C, int ldc)
{
    return cublasDgemm(h, ta, tb, m, n, k, al, A, lda, B, ldb, be, C, ldc);
}
inline cublasStatus_t gemv(cublasHandle_t h, int m, int n, const float *al, const float *A, int lda, const float *x, const float *be, float *y)
{
    return cublasSgemv(h, CUBLAS_OP_N, m, n, al, A, lda, x, 1, be, y, 1);
}
inline cublasStatus_t gemv(cublasHandle_t h, int m, int n, const double *al, const double *A, int lda, const double *x, const double *be, double *y)
{
    return cublasDgemv(h, CUBLAS_OP_N, m, n, al, A, lda, x, 1, be, y, 1);
}

struct Net {
    int n_layers = 0;
    int widths[6] = {};
    size_t w_off[5] = {}, b_off[5] = {};   // offsets inside theta
    size_t P = 0;
};
Net make_net(const int *widths, int n_layers, size_t base)
{
    Net n;
    n.n_layers = n_layers;
    size_t o = base;
    for (int l = 0; l <= n_layers; ++l) n.widths[l] = widths[l];
    for (int l = 0; l < n_layers; ++l) {
        n.w_off[l] = o; o += (size_t)widths[l] * widths[l + 1];
        n.b_off[l] = o; o += (size_t)widths[l + 1];
    }
    n.P = o - base;
    return n;
}

}  // namespace

struct b200ude_bsde_handle {
    b200ude_bsde_desc desc;
    int d = 0, hls = 0, P = 0;
    int ldh = 0;   // leading dimension of the hidden-activation tapes: >= hls + 1 (the ones row), = 4 mod 16 (even: 16-byte columns in fp64;
                   // conflict-free 8-byte fragment reads when a tape chunk is staged in shared memory with this row stride)
    bool f64 = true;
    size_t cap = 0;
    Net nu, nz;
    cublasHandle_t blas = nullptr;
    cudaStream_t stream = nullptr;
    void *workspace = nullptr;
    // device buffers (element type = the handle's dtype)
    void *theta = nullptr, *grad = nullptr, *adam_m = nullptr, *adam_v = nullptr, *x0 = nullptr;
    // per-step storage, step n of an M-path evaluation at element offset n * ld * M:
    //   IN [n_steps + 1][d + 2][cap]  = [X_n; t_n; 1]      H[k] [n_steps][ldh][cap] = [hidden k; 1; 0 pad]      Z, Zb [n_steps][d][cap]
    //   C[k] [n_steps][hls][cap] = cotangents of hidden k
    void *IN = nullptr, *u = nullptr, *H[3] = {}, *Z = nullptr, *Zb = nullptr, *C[3] = {}, *r2 = nullptr, *ubar = nullptr, *ones = nullptr;
    int init_M = 0;   // the constant rows are laid out for this many paths
    bool fused = false;       // fp64, dim <= 110, hidden <= 111: the fused DMMA sweeps instead of per-layer library GEMMs
    void *packed = nullptr;   // zero-padded operand copies of the z network for the fused sweeps
    void *mask = nullptr;     // relu' bits of the hidden layers (fused sweeps)
    void *dW = nullptr;       // Brownian increments of the iteration (fused sweeps)
    FusedArgs fa;             // slab tables (the pointers are filled per call)
    int sm_count = 0;         // the device's SM count (set at create; sizes the persistent cotangent-sweep grid)
    bool fwd_pairs = true;    // forward sweep with two warps per path tile (k_fused_forward2)
    void *wg_partial = nullptr;   // per-CTA partial sums of the fused weight-gradient products (null: library GEMMs)
    int wg_splits = 0;
    void *hu[3] = {}, *cu_[3] = {};   // u0 net (single column): activations / cotangents
    void *scal = nullptr;             // [0] loss, [1] sum ubar, [2] u0(x0)
    int *t_dev = nullptr;
    uint64_t *seed_dev = nullptr;
    int adam_t = 0;
    bool have_theta = false;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_ms = 0.0f;
    cudaEvent_t kev[5] = {};   // around the sweeps of an eager b200ude_bsde_loss_gradient call: start, forward, loss sums, backward, weight gradients
    bool time_kernels = false;
    std::vector<double> x0_host;
    std::string err;
};

namespace {

int32_t bfail(b200ude_bsde_handle *h, int32_t code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (h) h->err = buf;
    else g_bsde_create_error = buf;
    return code;
}
#define BS_CUDA(h, expr)                                                                                                        \
    do {                                                                                                                        \
        cudaError_t e_ = (expr);                                                                                                \
        if (e_ != cudaSuccess) return bfail((h), (int32_t)e_, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)
#define BS_BLAS(h, expr)                                                                                                        \
    do {                                                                                                                        \
        cublasStatus_t s_ = (expr);                                                                                             \
        if (s_ != CUBLAS_STATUS_SUCCESS) return bfail((h), 1000 + (int32_t)s_, "%s failed: cuBLAS status %d (%s:%d)", #expr, (int)s_, __FILE__, __LINE__); \
    } while (0)

inline int blocks(size_t n, int per = 256) { return (int)((n + per - 1) / per); }

// chain forward on [width x M] activations: acts[0] = input, acts[l + 1] = layer l's output
template <class R>
int32_t net_forward(b200ude_bsde_handle *h, const Net &n, const R *in, R *const *outs, int M, cudaStream_t st)
{
    const R one = 1, zero = 0;
    const R *th = (const R *)h->theta;
    const R *cur = in;
    for (int l = 0; l < n.n_layers; ++l) {
        const int nin = n.widths[l], nout = n.widths[l + 1];
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_N, nout, M, nin, &one, th + n.w_off[l], nout, cur, nin, &zero, outs[l], nout));
        k_bias_act<R><<<blocks((size_t)nout * M), 256, 0, st>>>(outs[l], th + n.b_off[l], nout, M, l < n.n_layers - 1 ? 1 : 0);
        cur = outs[l];
    }
    return B200UDE_OK;
}
// chain backward: cot of the output in cots[L-1] (overwritten); weight / bias gradients ACCUMULATE into grad (theta layout)
template <class R>
int32_t net_backward(b200ude_bsde_handle *h, const Net &n, const R *in, R *const *outs, R *const *cots, int M, cudaStream_t st)
{
    const R one = 1, zero = 0;
    const R *th = (const R *)h->theta;
    R *g = (R *)h->grad;
    for (int l = n.n_layers - 1; l >= 0; --l) {
        const int nin = n.widths[l], nout = n.widths[l + 1];
        if (l < n.n_layers - 1) k_relu_mask<R><<<blocks((size_t)nout * M), 256, 0, st>>>(cots[l], outs[l], nout, nout, M);
        const R *a_in = l == 0 ? in : outs[l - 1];
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_T, nout, nin, M, &one, cots[l], nout, a_in, nin, &one, g + n.w_off[l], nout));
        BS_BLAS(h, gemv(h->blas, nout, M, &one, cots[l], nout, (const R *)h->ones, &one, g + n.b_off[l]));
        if (l > 0) BS_BLAS(h, gemm(h->blas, CUBLAS_OP_T, CUBLAS_OP_N, nin, M, nout, &one, th + n.w_off[l], nout, cots[l], nout, &zero, cots[l - 1], nin));
    }
    return B200UDE_OK;
}

inline size_t fused_smem(int warps) { return ((size_t)FRING * FSLAB + (size_t)warps * 8 * FLD) * sizeof(double) + 8 * FRING + sizeof(SlabShared); }

inline size_t fused_smem2() { return ((size_t)FP_DEPTH * FSLAB + (size_t)(FPW / 2) * 2 * 8 * FLD) * sizeof(double) + 8 * FRING + ((sizeof(SlabShared) + 7) / 8) * 8 + (FPW / 2) * sizeof(PairExch); }

inline size_t wgrad_smem() { return (size_t)WGD * WGSTAGE * sizeof(double) + 8 * WGD + 4 * WGD + 16; }

// the fused fp64 path of one iteration: operand slabs, forward sweep (+ residual), loss sums, cotangent sweep
int32_t fused_sweeps(b200ude_bsde_handle *h, int M, uint32_t path0, double inv_total, cudaStream_t st)
{
    const Net &nz = h->nz;
    double *pk = (double *)h->packed;
    FusedArgs a = h->fa;
    PackArgs q;
    for (int l = 0; l < 4; ++l) { q.w_off[l] = nz.w_off[l]; q.nin[l] = nz.widths[l]; q.nout[l] = nz.widths[l + 1]; }
    k_pack_slabs<<<dim3(blocks((size_t)FSLAB), a.n_f + a.n_b), 256, 0, st>>>((const double *)h->theta, pk, a, q);
    a.slabs = pk;
    a.IN = (double *)h->IN; a.Z = (double *)h->Z; a.Zb = (double *)h->Zb; a.u = (double *)h->u; a.r2 = (double *)h->r2; a.ubar = (double *)h->ubar;
    for (int k = 0; k < 3; ++k) { a.H[k] = (double *)h->H[k]; a.C[k] = (double *)h->C[k]; }
    a.x0 = (const double *)h->x0; a.u0 = (const double *)h->scal + 2; a.seed = h->seed_dev; a.path0 = path0;
    a.M = M; a.N = h->desc.n_steps; a.d = h->d; a.hl = h->hls; a.ldh = h->ldh;
    a.dt = h->desc.T / h->desc.n_steps; a.lam = h->desc.lambda; a.s = h->desc.sigma; a.ga = h->desc.g_a; a.gb = h->desc.g_b; a.inv_total = inv_total;
    a.mask = (uint32_t *)h->mask;
    a.dW = (const double *)h->dW;
    {
        const long total = (long)a.N * M * ((a.d + 3) / 4);
        k_dw_tape<<<(unsigned)((total + 255) / 256), 256, 0, st>>>((double *)h->dW, h->seed_dev, path0, M, a.N, a.d, sqrt(a.dt));
    }
    const int tiles = (M + 7) / 8;
    const size_t smem = fused_smem(FWPC);
    if (h->time_kernels) cudaEventRecord(h->kev[0], st);
    if (h->fwd_pairs) k_fused_forward2<<<(tiles + FPW / 2 - 1) / (FPW / 2), 32 * FPW, fused_smem2(), st>>>(a);
    else k_fused_forward<<<(tiles + FWF - 1) / FWF, 32 * FWF, fused_smem(FWF), st>>>(a);
    if (h->time_kernels) cudaEventRecord(h->kev[1], st);
    k_sum2<double><<<1, 256, 0, st>>>((const double *)h->r2, (const double *)h->ubar, M, inv_total, (double *)h->scal, (double *)h->scal + 1);
    if (h->time_kernels) cudaEventRecord(h->kev[2], st);
    const long groups = ((long)tiles * a.N + FWPC - 1) / FWPC;
    const long slots = 3L * h->sm_count;
    k_fused_backward<<<(unsigned)(groups < slots ? groups : slots), 32 * FWPC, smem, st>>>(a);
    if (h->time_kernels) cudaEventRecord(h->kev[3], st);
    BS_CUDA(h, cudaGetLastError());
    return B200UDE_OK;
}

// one NNPDENS iteration: loss -> scal[0], u0(x0) -> scal[2], gradient -> grad
template <class R>
int32_t loss_gradient(b200ude_bsde_handle *h, int M, uint32_t path0, double inv_total, cudaStream_t st)
{
    const int d = h->d, hl = h->hls, N = h->desc.n_steps;
    const double dt = h->desc.T / N, lam = h->desc.lambda, s = h->desc.sigma;
    const R one = 1, zero = 0;
    const R *th = (const R *)h->theta;
    const Net &nz = h->nz;
    R *u = (R *)h->u, *scal = (R *)h->scal, *IN = (R *)h->IN, *Z = (R *)h->Z, *Zb = (R *)h->Zb;
    R *H[3] = {(R *)h->H[0], (R *)h->H[1], (R *)h->H[2]}, *C[3] = {(R *)h->C[0], (R *)h->C[1], (R *)h->C[2]};
    const int ldh = h->ldh;
    const size_t s_in = (size_t)(d + 2) * M, s_h = (size_t)ldh * M, s_c = (size_t)hl * M, s_z = (size_t)d * M;
    R *outs_u[3] = {(R *)h->hu[0], (R *)h->hu[1], scal + 2};
    R *cots_u[3] = {(R *)h->cu_[0], (R *)h->cu_[1], scal + 1};
    BS_CUDA(h, cudaMemsetAsync(h->grad, 0, sizeof(R) * h->nu.P, st));   // the u0 net's gradients accumulate; the z net's are written
    int32_t rc = net_forward<R>(h, h->nu, (const R *)h->x0, outs_u, 1, st);   // u0(x0)
    if (rc) return rc;
    bool fused = false;
    if constexpr (sizeof(R) == 8) fused = h->fused;
    if (fused) {
        rc = fused_sweeps(h, M, path0, inv_total, st);
        if (rc) return rc;
    } else {
        k_init_paths<R><<<blocks((size_t)d * M), 256, 0, st>>>(IN, u, (const R *)h->x0, scal + 2, d, M);
        for (int n = 0; n < N; ++n) {
            // layer l: [W | b] (out x (in + 1), theta's own layout) times the ones-augmented activations
            const R *a = IN + n * s_in;
            int ka = d + 2, lda = d + 2;   // contraction length (inputs + ones row) and leading dimension of the input block
            for (int l = 0; l < 3; ++l) {
                R *o = H[l] + n * s_h;
                BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_N, hl, M, ka, &one, th + nz.w_off[l], hl, a, lda, &zero, o, ldh));
                k_relu<R><<<blocks((size_t)hl * M), 256, 0, st>>>(o, hl, ldh, M);
                a = o; ka = hl + 1; lda = ldh;
            }
            BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_N, d, M, ka, &one, th + nz.w_off[3], d, a, lda, &zero, Z + n * s_z, d));
            k_em_step<R><<<blocks((size_t)M * 32, 256), 256, 0, st>>>(IN + n * s_in, IN + (n + 1) * s_in, u, Z + n * s_z, h->seed_dev, path0, n, d, M, dt, lam, s);
        }
        k_residual<R><<<blocks((size_t)M * 32, 256), 256, 0, st>>>(IN + N * s_in, u, (R *)h->r2, (R *)h->ubar, d, M, h->desc.g_a, h->desc.g_b, inv_total);
        k_sum2<R><<<1, 256, 0, st>>>((const R *)h->r2, (const R *)h->ubar, M, inv_total, scal, scal + 1);
        // cotangents, step by step (the steps only couple through ubar, which is the same for all of them: any order works)
        for (int n = 0; n < N; ++n) {
            k_zbar<R><<<blocks((size_t)((d + 3) / 4) * M), 256, 0, st>>>(Zb + n * s_z, Z + n * s_z, (const R *)h->ubar, h->seed_dev, path0, n, d, M, dt, lam);
            const R *c = Zb + n * s_z;
            int nc = d;
            for (int l = 3; l >= 1; --l) {   // cot of hidden l = W_{l+1}^T cot_{l+1}, masked by relu'
                R *o = C[l - 1] + n * s_c;
                BS_BLAS(h, gemm(h->blas, CUBLAS_OP_T, CUBLAS_OP_N, hl, M, nc, &one, th + nz.w_off[l], nc, c, nc, &zero, o, hl));
                k_relu_mask<R><<<blocks((size_t)hl * M), 256, 0, st>>>(o, H[l - 1] + n * s_h, hl, ldh, M);
                c = o; nc = hl;
            }
        }
    }
    // [dW | db] of every layer over all steps at once: cot [out x (N M)] times augmented activation^T [(N M) x (in + 1)]
    R *g = (R *)h->grad;
    const int K = N * M;
    bool wg_fused = false;
    if constexpr (sizeof(R) == 8) wg_fused = fused && h->wg_partial != nullptr;
    if (wg_fused) {
        if constexpr (sizeof(R) == 8) {
            WgradArgs w;
            const double *cots[4] = {C[0], C[1], C[2], Zb}, *acts[4] = {IN, H[0], H[1], H[2]};
            for (int l = 0; l < 4; ++l) {
                w.cot[l] = cots[l]; w.act[l] = acts[l];
                w.ldc[l] = l < 3 ? hl : d; w.lda[l] = l == 0 ? d + 2 : ldh;
                w.nout[l] = nz.widths[l + 1]; w.nact[l] = nz.widths[l] + 1;
            }
            w.K = K; w.partial = (double *)h->wg_partial;
            PackArgs q;
            for (int l = 0; l < 4; ++l) { q.w_off[l] = nz.w_off[l]; q.nin[l] = nz.widths[l]; q.nout[l] = nz.widths[l + 1]; }
            k_wgrad<<<dim3(h->wg_splits, 4), 32 * WGW, wgrad_smem(), st>>>(w);
            k_wgrad_reduce<<<dim3(blocks((size_t)FW * FW), 4), 256, 0, st>>>((const double *)h->wg_partial, h->wg_splits, g, q);
        }
    } else {
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_T, hl, d + 2, K, &one, C[0], hl, IN, d + 2, &zero, g + nz.w_off[0], hl));
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_T, hl, hl + 1, K, &one, C[1], hl, H[0], ldh, &zero, g + nz.w_off[1], hl));
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_T, hl, hl + 1, K, &one, C[2], hl, H[1], ldh, &zero, g + nz.w_off[2], hl));
        BS_BLAS(h, gemm(h->blas, CUBLAS_OP_N, CUBLAS_OP_T, d, hl + 1, K, &one, Zb, d, H[2], ldh, &zero, g + nz.w_off[3], d));
    }
    if (h->time_kernels) cudaEventRecord(h->kev[4], st);
    rc = net_backward<R>(h, h->nu, (const R *)h->x0, outs_u, cots_u, 1, st);   // cotangent of u0(x0) = sum of ubar (already in scal[1])
    if (rc) return rc;
    BS_CUDA(h, cudaGetLastError());
    return B200UDE_OK;
}

// (re)write the constant rows when the number of paths of the evaluation changes (outside any graph capture)
template <class R>
int32_t prepare(b200ude_bsde_handle *h, int M)
{
    if (h->init_M == M) return B200UDE_OK;
    const int N = h->desc.n_steps;
    k_init_aug<R><<<blocks((size_t)(N + 1) * M), 256, 0, h->stream>>>((R *)h->IN, (R *)h->H[0], (R *)h->H[1], (R *)h->H[2], h->d, h->hls, h->ldh, M, N, h->desc.T / N);
    BS_CUDA(h, cudaGetLastError());
    h->init_M = M;
    return B200UDE_OK;
}

template <class R>
int32_t alloc_all(b200ude_bsde_handle *h)
{
    const size_t M = h->cap, d = h->d, hl = h->hls;
    auto A = [&](void **p, size_t n) { return cudaMalloc(p, sizeof(R) * n) == cudaSuccess; };
    const size_t N = h->desc.n_steps;
    bool ok = A(&h->theta, h->P) && A(&h->grad, h->P) && A(&h->adam_m, h->P) && A(&h->adam_v, h->P) && A(&h->x0, d) && A(&h->u, M) &&
              A(&h->IN, (N + 1) * (d + 2) * M) && A(&h->H[0], N * (size_t)h->ldh * M) && A(&h->H[1], N * (size_t)h->ldh * M) && A(&h->H[2], N * (size_t)h->ldh * M) &&
              A(&h->Z, N * d * M) && A(&h->Zb, N * d * M) && A(&h->C[0], N * hl * M) && A(&h->C[1], N * hl * M) && A(&h->C[2], N * hl * M) && A(&h->r2, M) &&
              A(&h->ubar, M) && A(&h->ones, M) && A(&h->hu[0], hl) &&
              A(&h->hu[1], hl) && A(&h->cu_[0], hl) && A(&h->cu_[1], hl) && A(&h->scal, 4);
    ok = ok && cudaMalloc((void **)&h->t_dev, sizeof(int)) == cudaSuccess && cudaMalloc((void **)&h->seed_dev, sizeof(uint64_t)) == cudaSuccess &&
         cudaMalloc(&h->workspace, 32u << 20) == cudaSuccess;
    if (!ok) return B200UDE_ENOMEM;
    k_fill<R><<<blocks(M), 256>>>((R *)h->ones, (R)1, (int)M);
    cudaMemset(h->adam_m, 0, sizeof(R) * h->P);
    cudaMemset(h->adam_v, 0, sizeof(R) * h->P);
    cudaMemset(h->t_dev, 0, sizeof(int));
    std::vector<R> x0(d);
    for (size_t i = 0; i < d; ++i) x0[i] = (R)h->x0_host[i];
    cudaMemcpy(h->x0, x0.data(), sizeof(R) * d, cudaMemcpyHostToDevice);
    return cudaDeviceSynchronize() == cudaSuccess ? B200UDE_OK : B200UDE_ENOMEM;
}

template <class R>
int32_t train(b200ude_bsde_handle *h, const b200ude_adam *o, int M, int iters, uint64_t seed0, uint32_t path0, R *loss_hist, R *u0_hist, bool update)
{
    cudaStream_t st = h->stream;
    BS_CUDA(h, cudaMemcpyAsync(h->seed_dev, &seed0, sizeof(seed0), cudaMemcpyHostToDevice, st));
    {
        const int32_t rp = prepare<R>(h, M);
        if (rp) return rp;
    }
    BS_CUDA(h, cudaStreamSynchronize(st));
    R *scal = (R *)h->scal;
    const int t_base = h->adam_t;
    auto one = [&]() -> int32_t {
        int32_t rc = loss_gradient<R>(h, M, path0, 1.0 / M, st);
        if (rc) return rc;
        if (update)
            k_adam<R><<<1, 1024, 0, st>>>((R *)h->theta, (R *)h->adam_m, (R *)h->adam_v, (const R *)h->grad, h->P, h->t_dev, h->seed_dev, o->eta, o->beta1,
                                          o->beta2, o->eps, scal, scal + 2, loss_hist, u0_hist, t_base);
        return B200UDE_OK;
    };
    BS_CUDA(h, cudaEventRecord(h->ev0, st));
    int32_t rc = one();   // eagerly once (cuBLAS initialisation), the rest as replays of one captured graph
    if (rc) return rc;
    if (iters > 1) {
        cudaGraph_t graph = nullptr;
        cudaGraphExec_t exec = nullptr;
        bool graphed = false;
        if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
            const int32_t r = one();
            const cudaError_t ce = cudaStreamEndCapture(st, &graph);
            if (r == B200UDE_OK && ce == cudaSuccess && graph && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) graphed = true;
            else cudaGetLastError();
        }
        for (int it = 1; it < iters; ++it) {
            if (graphed) BS_CUDA(h, cudaGraphLaunch(exec, st));
            else if ((rc = one()) != 0) break;
        }
        if (exec) cudaGraphExecDestroy(exec);
        if (graph) cudaGraphDestroy(graph);
        if (rc) return rc;
    }
    if (update) h->adam_t = t_base + iters;
    BS_CUDA(h, cudaEventRecord(h->ev1, st));
    BS_CUDA(h, cudaStreamSynchronize(st));
    BS_CUDA(h, cudaEventElapsedTime(&h->last_ms, h->ev0, h->ev1));
    return B200UDE_OK;
}

}  // namespace

extern "C" {

const char *b200ude_bsde_last_error(const b200ude_bsde_handle *h) { return h ? h->err.c_str() : g_bsde_create_error.c_str(); }

int32_t b200ude_bsde_create(const b200ude_bsde_desc *d, b200ude_bsde_handle **out)
{
    if (!d || !out) return bfail(nullptr, B200UDE_EINVAL, "bsde_create: null argument");
    *out = nullptr;
    if (d->struct_size != sizeof(b200ude_bsde_desc)) return bfail(nullptr, B200UDE_EINVAL, "bsde_create: struct_size mismatch (ABI)");
    if (d->dtype != B200UDE_F32 && d->dtype != B200UDE_F64) return bfail(nullptr, B200UDE_EINVAL, "bsde_create: unknown dtype");
    if (d->dim < 1 || d->dim > 1024 || d->hidden < 1 || d->hidden > 1024 || d->n_steps < 1 || !(d->T > 0) || d->max_paths < 1 || d->max_paths > (1u << 22) || !d->x0 ||
        (double)d->n_steps * (double)d->max_paths > 2.0e9)
        return bfail(nullptr, B200UDE_EINVAL, "bsde_create: need 1 <= dim, hidden <= 1024, n_steps >= 1, T > 0, 1 <= max_paths <= 2^22, n_steps * max_paths <= 2e9, x0 != NULL");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return bfail(nullptr, B200UDE_ENODEVICE, "bsde_create: no CUDA device");
    if (d->device < 0 || d->device >= ndev) return bfail(nullptr, B200UDE_EINVAL, "bsde_create: device %d of %d", d->device, ndev);
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, d->device) != cudaSuccess || prop.major != 9 || prop.minor != 0)
        return bfail(nullptr, B200UDE_ENODEVICE, "bsde_create: device %d is not an sm_90 part", d->device);
    if (cudaSetDevice(d->device) != cudaSuccess) return bfail(nullptr, B200UDE_ENODEVICE, "bsde_create: cudaSetDevice failed");
    b200ude_bsde_handle *h = new (std::nothrow) b200ude_bsde_handle();
    if (!h) return bfail(nullptr, B200UDE_ENOMEM, "bsde_create: out of host memory");
    h->desc = *d;
    h->d = d->dim; h->hls = d->hidden; h->ldh = ((d->hidden + 1 - 4 + 15) / 16) * 16 + 4; /* >= hidden + 1 (the ones row), = 4 mod 16 */ h->f64 = d->dtype == B200UDE_F64; h->cap = d->max_paths;
    const int wu[4] = {d->dim, d->hidden, d->hidden, 1}, wz[5] = {d->dim + 1, d->hidden, d->hidden, d->hidden, d->dim};
    h->nu = make_net(wu, 3, 0);
    h->nz = make_net(wz, 4, h->nu.P);
    h->P = (int)(h->nu.P + h->nz.P);
    h->x0_host.assign(d->x0, d->x0 + d->dim);
    h->desc.x0 = nullptr;   // the caller's array is not kept
    bool ok = cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) == cudaSuccess && cublasCreate(&h->blas) == CUBLAS_STATUS_SUCCESS &&
              cudaEventCreate(&h->ev0) == cudaSuccess && cudaEventCreate(&h->ev1) == cudaSuccess;
    for (int i = 0; ok && i < 5; ++i) ok = cudaEventCreate(&h->kev[i]) == cudaSuccess;
    int32_t rc = ok ? (h->f64 ? alloc_all<double>(h) : alloc_all<float>(h)) : B200UDE_ENOMEM;
    const char *fenv = getenv("B200UDE_BSDE_FUSED");
    if (rc == B200UDE_OK && h->f64 && d->dim <= FW - 2 && d->hidden <= FW - 1 && !(fenv && fenv[0] == '0')) {
        FusedArgs &fa = h->fa;
        memset(&fa, 0, sizeof(fa));
        for (int l = 0; l < 4; ++l)   // forward: contraction over in_l + 1 rows
            for (int k0 = 0; k0 < h->nz.widths[l] + 1; k0 += FSR) {
                const int rows = h->nz.widths[l] + 1 - k0 < FSR ? h->nz.widths[l] + 1 - k0 : FSR;
                const int i = fa.n_f++;
                fa.f_layer[i] = (unsigned char)l; fa.f_k0[i] = (unsigned char)k0; fa.f_ks[i] = (unsigned char)((rows + 3) / 4);
                fa.f_last[i] = (unsigned char)(k0 + FSR >= h->nz.widths[l] + 1);
            }
        for (int l = 3; l >= 1; --l)  // backward: contraction over out_l rows
            for (int k0 = 0; k0 < h->nz.widths[l + 1]; k0 += FSR) {
                const int rows = h->nz.widths[l + 1] - k0 < FSR ? h->nz.widths[l + 1] - k0 : FSR;
                const int i = fa.n_b++;
                fa.b_layer[i] = (unsigned char)l; fa.b_k0[i] = (unsigned char)k0; fa.b_ks[i] = (unsigned char)((rows + 3) / 4);
                fa.b_last[i] = (unsigned char)(k0 + FSR >= h->nz.widths[l + 1]);
            }
        h->sm_count = prop.multiProcessorCount;
        const char *penv = getenv("B200UDE_BSDE_PAIRS");
        h->fwd_pairs = !(penv && penv[0] == '0');
        const char *wenv = getenv("B200UDE_BSDE_WGRAD");
        if (!(wenv && wenv[0] == '0') && d->dim % 2 == 0 && d->hidden % 2 == 0) {   // TMA chunks of the tapes: even leading dimensions
            h->wg_splits = prop.multiProcessorCount / 4 > 0 ? prop.multiProcessorCount / 4 : 1;
            if (cudaMalloc(&h->wg_partial, (size_t)4 * h->wg_splits * FW * FW * sizeof(double)) != cudaSuccess ||
                cudaFuncSetAttribute(k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wgrad_smem()) != cudaSuccess) {
                cudaGetLastError();
                cudaFree(h->wg_partial);
                h->wg_partial = nullptr;
            }
        }
        const int smem = (int)fused_smem(FWF);
        if (cudaMalloc(&h->packed, (size_t)(fa.n_f + fa.n_b) * FSLAB * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&h->mask, (size_t)d->n_steps * 3 * d->max_paths * 4 * sizeof(uint32_t)) == cudaSuccess &&
            cudaMalloc(&h->dW, (size_t)d->n_steps * d->dim * d->max_paths * sizeof(double)) == cudaSuccess &&
            cudaFuncSetAttribute(k_fused_forward, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess &&
            cudaFuncSetAttribute(k_fused_forward2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fused_smem2()) == cudaSuccess &&
            cudaFuncSetAttribute(k_fused_backward, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) == cudaSuccess)
            h->fused = true;
        else
            rc = B200UDE_ENOMEM;
    }
    if (rc == B200UDE_OK) {
        ok = cublasSetStream(h->blas, h->stream) == CUBLAS_STATUS_SUCCESS && cublasSetWorkspace(h->blas, h->workspace, 32u << 20) == CUBLAS_STATUS_SUCCESS &&
             cublasSetPointerMode(h->blas, CUBLAS_POINTER_MODE_HOST) == CUBLAS_STATUS_SUCCESS &&
             cublasSetMathMode(h->blas, CUBLAS_DEFAULT_MATH) == CUBLAS_STATUS_SUCCESS;   // plain fp32 / fp64 arithmetic: no TF32 down-conversion
        if (!ok) rc = B200UDE_ENOMEM;
    }
    if (rc != B200UDE_OK) {
        char msg[256];
        const double per = (4.0 * d->dim + 6.0 * d->hidden + 8.0) * (double)d->n_steps * (double)d->max_paths * (d->dtype == B200UDE_F64 ? 8.0 : 4.0);
        snprintf(msg, sizeof(msg), "bsde_create: device allocation (%.2f GB of per-step storage for max_paths = %llu) or cuBLAS initialisation failed",
                 per * 1e-9, (unsigned long long)d->max_paths);
        g_bsde_create_error = msg;
        b200ude_bsde_destroy(h);
        return rc;
    }
    *out = h;
    return B200UDE_OK;
}

void b200ude_bsde_destroy(b200ude_bsde_handle *h)
{
    if (!h) return;
    void *bufs[] = {h->theta, h->grad, h->adam_m, h->adam_v, h->x0, h->IN, h->u, h->H[0], h->H[1], h->H[2], h->Z, h->Zb, h->C[0], h->C[1], h->C[2],
                    h->r2, h->ubar, h->ones, h->hu[0], h->hu[1], h->cu_[0], h->cu_[1], h->scal, h->t_dev, h->seed_dev, h->workspace, h->packed, h->mask, h->dW, h->wg_partial};
    for (void *b : bufs) cudaFree(b);
    for (cudaEvent_t e : h->kev)
        if (e) cudaEventDestroy(e);
    if (h->ev0) cudaEventDestroy(h->ev0);
    if (h->ev1) cudaEventDestroy(h->ev1);
    if (h->blas) cublasDestroy(h->blas);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

size_t b200ude_bsde_num_params(const b200ude_bsde_handle *h) { return h ? (size_t)h->P : 0; }
double b200ude_bsde_last_train_ms(const b200ude_bsde_handle *h) { return h ? (double)h->last_ms : 0.0; }
int32_t b200ude_bsde_last_sweep_ms(b200ude_bsde_handle *h, double *ms)
{
    if (!h || !ms) return B200UDE_EINVAL;
    if (!h->fused) return bfail(h, B200UDE_EUNSUPPORTED, "bsde_last_sweep_ms: the handle runs on library GEMMs (fp32, dim > 110, hidden > 111 or B200UDE_BSDE_FUSED=0)");
    const int pairs[3][2] = {{0, 1}, {2, 3}, {3, 4}};
    for (int i = 0; i < 3; ++i) {
        float t = 0.0f;
        if (cudaEventElapsedTime(&t, h->kev[pairs[i][0]], h->kev[pairs[i][1]]) != cudaSuccess) {
            cudaGetLastError();
            return bfail(h, B200UDE_ESTATE, "bsde_last_sweep_ms: no completed b200ude_bsde_loss_gradient call yet");
        }
        ms[i] = t;
    }
    return B200UDE_OK;
}

int32_t b200ude_bsde_set_params(b200ude_bsde_handle *h, const void *theta, size_t P, int32_t mem)
{
    if (!h) return B200UDE_EINVAL;
    if (!theta || P != (size_t)h->P) return bfail(h, B200UDE_EINVAL, "bsde_set_params: P=%zu, expected %d", P, h->P);
    BS_CUDA(h, cudaSetDevice(h->desc.device));
    const size_t es = h->f64 ? 8 : 4;
    BS_CUDA(h, cudaMemcpy(h->theta, theta, es * P, mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    BS_CUDA(h, cudaMemset(h->adam_m, 0, es * P));
    BS_CUDA(h, cudaMemset(h->adam_v, 0, es * P));
    BS_CUDA(h, cudaMemset(h->t_dev, 0, sizeof(int)));
    h->adam_t = 0;
    h->have_theta = true;
    return B200UDE_OK;
}

int32_t b200ude_bsde_get_params(b200ude_bsde_handle *h, void *theta, size_t P, int32_t mem)
{
    if (!h) return B200UDE_EINVAL;
    if (!theta || P != (size_t)h->P) return bfail(h, B200UDE_EINVAL, "bsde_get_params: P=%zu, expected %d", P, h->P);
    BS_CUDA(h, cudaSetDevice(h->desc.device));
    BS_CUDA(h, cudaMemcpy(theta, h->theta, (h->f64 ? 8 : 4) * P, mem == B200UDE_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost));
    return B200UDE_OK;
}

int32_t b200ude_bsde_loss_gradient(b200ude_bsde_handle *h, size_t n_paths, uint64_t seed, uint64_t path_offset, size_t total_paths, void *loss,
                                   void *grad, void *u0)
{
    if (!h) return B200UDE_EINVAL;
    if (!h->have_theta) return bfail(h, B200UDE_ESTATE, "bsde_loss_gradient: set_params has not been called");
    if (n_paths == 0 || n_paths > h->cap) return bfail(h, B200UDE_EINVAL, "bsde_loss_gradient: n_paths=%zu outside (0, %zu]", n_paths, h->cap);
    BS_CUDA(h, cudaSetDevice(h->desc.device));
    BS_CUDA(h, cudaMemcpyAsync(h->seed_dev, &seed, sizeof(seed), cudaMemcpyHostToDevice, h->stream));
    const double inv_total = 1.0 / (double)(total_paths ? total_paths : n_paths);
    int32_t rc = h->f64 ? prepare<double>(h, (int)n_paths) : prepare<float>(h, (int)n_paths);
    if (rc) return rc;
    h->time_kernels = h->fused;
    rc = h->f64 ? loss_gradient<double>(h, (int)n_paths, (uint32_t)path_offset, inv_total, h->stream)
                        : loss_gradient<float>(h, (int)n_paths, (uint32_t)path_offset, inv_total, h->stream);
    if (rc) return rc;
    const size_t es = h->f64 ? 8 : 4;
    h->time_kernels = false;
    if (loss) BS_CUDA(h, cudaMemcpyAsync(loss, h->scal, es, cudaMemcpyDefault, h->stream));
    if (u0) BS_CUDA(h, cudaMemcpyAsync(u0, (char *)h->scal + 2 * es, es, cudaMemcpyDefault, h->stream));
    if (grad) BS_CUDA(h, cudaMemcpyAsync(grad, h->grad, es * (size_t)h->P, cudaMemcpyDefault, h->stream));
    BS_CUDA(h, cudaStreamSynchronize(h->stream));
    return B200UDE_OK;
}

int32_t b200ude_bsde_train_adam(b200ude_bsde_handle *h, const b200ude_adam *opt, size_t n_paths, int32_t iters, uint64_t seed0, void *loss_history,
                                void *u0_history)
{
    if (!h) return B200UDE_EINVAL;
    if (!opt || opt->struct_size != sizeof(b200ude_adam) || !(opt->eta > 0)) return bfail(h, B200UDE_EINVAL, "bsde_train_adam: bad options struct");
    if (!h->have_theta) return bfail(h, B200UDE_ESTATE, "bsde_train_adam: set_params has not been called");
    if (n_paths == 0 || n_paths > h->cap || iters < 1) return bfail(h, B200UDE_EINVAL, "bsde_train_adam: n_paths=%zu outside (0, %zu] or iters < 1", n_paths, h->cap);
    BS_CUDA(h, cudaSetDevice(h->desc.device));
    return h->f64 ? train<double>(h, opt, (int)n_paths, iters, seed0, 0u, (double *)loss_history, (double *)u0_history, true)
                  : train<float>(h, opt, (int)n_paths, iters, seed0, 0u, (float *)loss_history, (float *)u0_history, true);
}

int32_t b200ude_bsde_adam_step(b200ude_bsde_handle *h, const b200ude_adam *opt, const void *grad)
{
    if (!h) return B200UDE_EINVAL;
    if (!opt || opt->struct_size != sizeof(b200ude_adam) || !(opt->eta > 0) || !grad) return bfail(h, B200UDE_EINVAL, "bsde_adam_step: bad arguments");
    if (!h->have_theta) return bfail(h, B200UDE_ESTATE, "bsde_adam_step: set_params has not been called");
    BS_CUDA(h, cudaSetDevice(h->desc.device));
    if (h->f64)
        k_adam<double><<<1, 1024, 0, h->stream>>>((double *)h->theta, (double *)h->adam_m, (double *)h->adam_v, (const double *)grad, h->P, h->t_dev, h->seed_dev,
                                                  opt->eta, opt->beta1, opt->beta2, opt->eps, nullptr, nullptr, nullptr, nullptr, 0);
    else
        k_adam<float><<<1, 1024, 0, h->stream>>>((float *)h->theta, (float *)h->adam_m, (float *)h->adam_v, (const float *)grad, h->P, h->t_dev, h->seed_dev,
                                                 opt->eta, opt->beta1, opt->beta2, opt->eps, nullptr, nullptr, nullptr, nullptr, 0);
    BS_CUDA(h, cudaGetLastError());
    BS_CUDA(h, cudaStreamSynchronize(h->stream));
    h->adam_t += 1;
    return B200UDE_OK;
}

}  // extern "C"
