// k_forced.cu -- the forced neural ODE with a readout network (forced.cuh) in fp32 and fp64.  A translation unit of its own:
// the model's shape lives in its own __constant__ structs, and the runtime-shape kernels of k_generic.cu / k_f64.cu are not
// recompiled with it.
#include "forced.cuh"

#include "params.h"

namespace b200ude {

namespace forced {
static __constant__ Shape<float> c_f32;
static __constant__ Shape<double> c_f64;

// fp32: theta read from the handle's device copy (L1-resident; every lane reads the same address), tanhf / expf
struct Ops32 {
    using real = float;
    static __device__ __forceinline__ const Shape<float> &s() { return c_f32; }
    static __device__ __forceinline__ float act(int k, float a) { return k == ACT_TANH ? tanhf(a) : (k == ACT_RBF ? expf(-a * a) : a); }
};
struct Ops64 {
    using real = double;
    static __device__ __forceinline__ const Shape<double> &s() { return c_f64; }
    static __device__ __forceinline__ double act(int k, double a) { return k == ACT_TANH ? tanh(a) : (k == ACT_RBF ? exp(-a * a) : a); }
};
}  // namespace forced

constexpr int FORCED_BLOCK32 = 128;
constexpr int FORCED_BLOCK64 = 64;   // two warps per CTA: the per-warp gradient vector (P + 1 doubles) lives in shared memory

int adj_rows_forced(int N, int dtype)
{
    const int b = dtype == 1 ? FORCED_BLOCK64 : FORCED_BLOCK32;
    return ((N + b - 1) / b) * (b / 32);
}

template <typename R>
static void fill(const ForcedHost &h, forced::Shape<R> &d)
{
    d.serial = h.serial; d.D = h.D; d.Rr = h.R; d.J = h.J; d.L0 = h.L0; d.L1 = h.L1; d.P = h.P;
    for (int i = 0; i < 8; ++i) { d.widths[i] = h.widths[i]; d.acts[i] = h.acts[i]; }
    // layer l of the combined list: f0's layers l < L0 read widths[l] -> widths[l + 1], f1's read one entry further on
    int off = 0;
    for (int l = 0; l < 8; ++l) {
        d.woff[l] = off;
        if (l < h.L0 + h.L1) {
            const int a = l < h.L0 ? l : l + 1;
            off += h.widths[a] * h.widths[a + 1] + h.widths[a + 1];
        }
    }
    d.theta = (const R *)h.theta;
    for (int i = 0; i < 16; ++i) d.lossw[i] = (R)h.lossw[i];
}

template <typename R>
static cudaError_t upload_shape(const ForcedHost &h, cudaStream_t st)
{
    static SerialCache cache;
    if (cache.hit(h.serial)) return cudaSuccess;
    forced::Shape<R> d;
    fill(h, d);
    cudaError_t e = sizeof(R) == 8 ? cudaMemcpyToSymbolAsync(forced::c_f64, &d, sizeof(d), 0, cudaMemcpyHostToDevice, st)
                                   : cudaMemcpyToSymbolAsync(forced::c_f32, &d, sizeof(d), 0, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(st);   // `d` is a stack object
        if (e == cudaSuccess) cache.set(h.serial);
    }
    return e;
}

template <class B, int BLOCK>
static cudaError_t fwd(const ForcedHost &h, const ForcedRun &r, cudaStream_t st)
{
    using R = typename B::real;
    cudaError_t e = upload_shape<R>(h, st);
    if (e != cudaSuccess) return e;
    forced::Fwd<R> p;
    p.u0 = (const R *)r.u0; p.out = (R *)r.out; p.ustep = (R *)r.ustep; p.dense = (R *)r.dense; p.usave = (R *)r.usave; p.status = r.status;
    p.forcing = (const R *)r.forcing; p.N = r.N; p.n_steps = r.n_steps; p.save_every = r.save_every; p.fstride = r.fstride;
    p.t0 = (R)r.t0; p.dt = (R)r.dt;
    const int grid = (r.N + BLOCK - 1) / BLOCK;
    if (r.adaptive) {
        forced::Adapt<R> a{(R)r.t0, (R)r.save_dt, (R)r.abstol, (R)r.reltol, r.n_save, r.max_steps, (R *)r.tgrid, r.nacc};
        forced::adaptive_forward_kernel<B, BLOCK><<<grid, BLOCK, 0, st>>>(p, a);
    } else {
        forced::forward_kernel<B, BLOCK><<<grid, BLOCK, 0, st>>>(p);
    }
    return cudaGetLastError();
}

template <class B, int BLOCK>
static cudaError_t adj(const ForcedHost &h, const ForcedRun &r, cudaStream_t st, int *rows_out)
{
    using R = typename B::real;
    cudaError_t e = upload_shape<R>(h, st);
    if (e != cudaSuccess) return e;
    forced::Adj<R> p;
    p.ustep = (const R *)r.ustep; p.dense = (const R *)r.dense; p.cot = (const R *)r.cot; p.saved = (const R *)r.saved;
    p.forcing = (const R *)r.forcing; p.grad_u0 = (R *)r.grad_u0; p.partial = (R *)r.partial;
    p.N = r.N; p.n_steps = r.n_steps; p.save_every = r.save_every; p.fused_l2 = r.fused_l2; p.fstride = r.fstride;
    p.t0 = (R)r.t0; p.dt = (R)r.dt;
    const size_t smem = sizeof(R) * (size_t)(BLOCK / 32) * (h.P + 1);
    const int grid = (r.N + BLOCK - 1) / BLOCK;
    *rows_out = grid * (BLOCK / 32);
    if (r.adaptive) {
        auto kern = forced::adaptive_adjoint_kernel<B, BLOCK>;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        forced::Adapt<R> a{(R)r.t0, (R)r.save_dt, (R)r.abstol, (R)r.reltol, r.n_save, r.max_steps, (R *)r.tgrid, r.nacc};
        kern<<<grid, BLOCK, smem, st>>>(p, a);
    } else {
        auto kern = forced::adjoint_kernel<B, BLOCK>;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, BLOCK, smem, st>>>(p);
    }
    return cudaGetLastError();
}

// the forcing on the kernels' time axis s = t - t0: cos(w t + phi) = cos(w s + (phi + w t0)).  The sum is taken in double without
// contraction (as  phi + w * t0  evaluates on the host) and reduced to [-pi, pi] exactly, then rounded once to R.
template <typename R>
__global__ void fold_forcing_kernel(R *coef, int J, int fstride, int N, double t0)
{
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    for (int j = 0; j < J; ++j) {
        const double w = coef[(size_t)(3 * j + 1) * fstride + n];
        R &phi = coef[(size_t)(3 * j + 2) * fstride + n];
        phi = (R)remainder(__dadd_rn((double)phi, __dmul_rn(w, t0)), 6.283185307179586476925);
    }
}

cudaError_t launch_fold_forcing(int dtype, void *forcing, int J, int fstride, int N, double t0, cudaStream_t st)
{
    const int grid = (N + 127) / 128;
    if (dtype == 1) fold_forcing_kernel<double><<<grid, 128, 0, st>>>((double *)forcing, J, fstride, N, t0);
    else fold_forcing_kernel<float><<<grid, 128, 0, st>>>((float *)forcing, J, fstride, N, t0);
    return cudaGetLastError();
}

cudaError_t launch_fwd_forced(const ForcedHost &h, const ForcedRun &r, cudaStream_t st)
{
    return h.dtype == 1 ? fwd<forced::Ops64, FORCED_BLOCK64>(h, r, st) : fwd<forced::Ops32, FORCED_BLOCK32>(h, r, st);
}

cudaError_t launch_adj_forced(const ForcedHost &h, const ForcedRun &r, cudaStream_t st, int *rows_out)
{
    return h.dtype == 1 ? adj<forced::Ops64, FORCED_BLOCK64>(h, r, st, rows_out) : adj<forced::Ops32, FORCED_BLOCK32>(h, r, st, rows_out);
}

}  // namespace b200ude
