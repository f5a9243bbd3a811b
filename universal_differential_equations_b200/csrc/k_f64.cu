// k_f64.cu -- double-precision kernels (dtype = B200UDE_F64): the runtime-shape kernels (ude_generic.cuh and the headers written
// over its Ops) in fp64 + the fp64 reduction / L2 helpers.
#include "ude_generic.cuh"
#include "fkpp_adaptive.cuh"
#include "discrete_adjoint.cuh"
#include "fkpp_vern7_discrete.cuh"
#include "vern7_dense.cuh"
#include "vern7_dense_discrete.cuh"

#include "params.h"

namespace b200ude {

namespace f64 {
struct Shape64 {
    uint64_t serial;
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[6];
    int acts[5];
    int woff[5];          // offset of layer l's W in theta (column-major, out x in), its bias follows at woff + in*out
    const double *theta;  // the handle's device copy
    double consts[16], lossw[16];
};
static __constant__ Shape64 c_gen;
}  // namespace f64

// the fp64 precision of the runtime-shape model layer: shape, constants and loss weights from one small __constant__ struct,
// theta from the handle's device copy (global memory, L1-resident)
struct Ops64 {
    using real = double;
    using Fwd = Fwd64Host;
    using Adj = Adj64Host;
    using Adapt = Adapt64Host;
    static constexpr int MAXD = generic::MAXD;
    static __device__ __forceinline__ int model() { return f64::c_gen.model; }
    static __device__ __forceinline__ int D() { return f64::c_gen.D; }
    static __device__ __forceinline__ int din() { return f64::c_gen.din; }
    static __device__ __forceinline__ int dout() { return f64::c_gen.dout; }
    static __device__ __forceinline__ int n_layers() { return f64::c_gen.n_layers; }
    static __device__ __forceinline__ int n_prefix() { return f64::c_gen.n_prefix; }
    static __device__ __forceinline__ int P() { return f64::c_gen.P; }
    static __device__ __forceinline__ int width(int l) { return f64::c_gen.widths[l]; }
    static __device__ __forceinline__ int woff(int l) { return f64::c_gen.woff[l]; }
    static __device__ __forceinline__ int layer_act(int l) { return f64::c_gen.acts[l]; }
    static __device__ __forceinline__ const double &theta(int i) { return f64::c_gen.theta[i]; }
    static __device__ __forceinline__ const double &consts(int i) { return f64::c_gen.consts[i]; }
    static __device__ __forceinline__ const double &lossw(int c) { return f64::c_gen.lossw[c]; }
    static __device__ __forceinline__ double act(int k, double a) { return k == ACT_TANH ? tanh(a) : (k == ACT_RBF ? exp(-a * a) : a); }
};

constexpr int F64_BLOCK = 64;   // two warps per CTA: the per-warp gradient vector (P + 1 doubles) lives in shared memory

int adj_rows_f64(int N) { return ((N + F64_BLOCK - 1) / F64_BLOCK) * (F64_BLOCK / 32); }

static cudaError_t upload_shape(const Shape64Host &h, cudaStream_t st)
{
    // theta's address and the constants are per handle; the struct is small (0.4 KB): re-sent when the handle changes
    static SerialCache cache;
    if (cache.hit(h.serial)) return cudaSuccess;
    f64::Shape64 d;
    d.serial = h.serial; d.model = h.model; d.D = h.D; d.din = h.din; d.dout = h.dout; d.n_layers = h.n_layers; d.n_prefix = h.n_prefix; d.P = h.P;
    int off = h.n_prefix;
    for (int l = 0; l < 6; ++l) d.widths[l] = l <= h.n_layers ? h.widths[l] : 0;
    for (int l = 0; l < 5; ++l) {
        d.acts[l] = l < h.n_layers ? h.acts[l] : 0;
        d.woff[l] = off;
        if (l < h.n_layers) off += h.widths[l] * h.widths[l + 1] + h.widths[l + 1];
    }
    d.theta = h.theta;
    for (int i = 0; i < 16; ++i) { d.consts[i] = h.consts[i]; d.lossw[i] = h.lossw[i]; }
    cudaError_t e = cudaMemcpyToSymbolAsync(f64::c_gen, &d, sizeof(d), 0, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(st);   // `d` is a stack object
        cache.set(h.serial);
    }
    return e;
}

cudaError_t launch_fwd_f64(const Shape64Host &s, const Fwd64Host &p, int solver, const Adapt64Host *ad, cudaStream_t st)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + F64_BLOCK - 1) / F64_BLOCK;
    if (solver == 1) {   // Vern7: the step record only for the discrete adjoint (p.ustep set)
        if (ad) generic::vern7_adaptive_forward_kernel<Ops64, F64_BLOCK><<<grid, F64_BLOCK, 0, st>>>(p, *ad);
        else generic::vern7_forward_kernel<Ops64, F64_BLOCK><<<grid, F64_BLOCK, 0, st>>>(p);
    } else {
        if (ad) generic::adaptive_forward_kernel<Ops64, F64_BLOCK><<<grid, F64_BLOCK, 0, st>>>(p, *ad);
        else generic::forward_kernel<Ops64, F64_BLOCK><<<grid, F64_BLOCK, 0, st>>>(p);
    }
    return cudaGetLastError();
}

cudaError_t launch_adj_f64(const Shape64Host &s, const Adj64Host &p, const Adapt64Host *ad, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    const size_t smem = sizeof(double) * (size_t)(F64_BLOCK / 32) * (s.P + 1);
    const int grid = (p.N + F64_BLOCK - 1) / F64_BLOCK;
    *rows_out = grid * (F64_BLOCK / 32);
    if (ad) {
        auto kern = generic::adaptive_adjoint_kernel<Ops64, F64_BLOCK>;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, F64_BLOCK, smem, st>>>(p, *ad);
    } else {
        auto kern = generic::adjoint_kernel<Ops64, F64_BLOCK>;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        kern<<<grid, F64_BLOCK, smem, st>>>(p);
    }
    return cudaGetLastError();
}

// ---- discrete adjoint (discrete_adjoint.cuh in fp64) ----

cudaError_t launch_adj_discrete_f64(const Shape64Host &s, const Adj64Host &p, int solver, const Adapt64Host *ad, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    discrete::Params<double> q;
    q.ustep = p.ustep; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.tgrid = ad ? ad->tgrid : nullptr; q.hstep = ad ? ad->hstep : nullptr; q.nacc = ad ? ad->nacc : nullptr;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ad ? ad->t0 : 0.0; q.save_dt = ad ? ad->save_dt : 0.0;
    q.margin = 5e-13;   // half the clipping margin of vern7_adaptive_forward_kernel
    auto kern = solver == 1 ? discrete::adjoint_kernel<Ops64, discrete::Vern7Scheme, F64_BLOCK>
                            : discrete::adjoint_kernel<Ops64, discrete::Tsit5Scheme, F64_BLOCK>;
    const size_t smem = sizeof(double) * (size_t)(F64_BLOCK / 32) * (s.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + F64_BLOCK - 1) / F64_BLOCK;
    *rows_out = grid * (F64_BLOCK / 32);
    kern<<<grid, F64_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- Vern7 with its lazy dense output (vern7_dense.cuh in fp64) ----

cudaError_t launch_fwd_vern7_dense_f64(const Shape64Host &s, const Fwd64Host &p, const Adapt64Host &a, cudaStream_t st)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Fwd<double> q;
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.tgrid = a.tgrid; q.hstep = a.hstep; q.nacc = a.nacc; q.status = p.status;
    q.N = p.N; q.n_save = a.n_save; q.max_steps = a.max_steps;
    q.t0 = a.t0; q.save_dt = a.save_dt; q.abstol = a.abstol; q.reltol = a.reltol;
    vern7_dense::forward_kernel<Ops64, F64_BLOCK><<<(p.N + F64_BLOCK - 1) / F64_BLOCK, F64_BLOCK, 0, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_vern7_dense_f64(const Shape64Host &s, const Adj64Host &p, const Adapt64Host *ad, const double *saved, cudaStream_t st,
                                       int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Adj<double> q;
    q.ustep = p.ustep; q.tgrid = ad ? ad->tgrid : nullptr; q.hstep = ad ? ad->hstep : nullptr; q.nacc = ad ? ad->nacc : nullptr;
    q.cot = p.cot; q.saved = saved; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ad ? ad->t0 : 0.0; q.save_dt = ad ? ad->save_dt : 0.0;
    auto kern = vern7_dense::adjoint_kernel<Ops64, F64_BLOCK>;
    const size_t smem = sizeof(double) * (size_t)(F64_BLOCK / 32) * (s.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + F64_BLOCK - 1) / F64_BLOCK;
    *rows_out = grid * (F64_BLOCK / 32);
    kern<<<grid, F64_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- discrete adjoint through the interpolated saves of the dense-output forward (vern7_dense_discrete.cuh in fp64) ----
cudaError_t launch_adj_vern7_dense_discrete_f64(const Shape64Host &s, const Adj64Host &p, const Adapt64Host &a, const double *saved,
                                                cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    vern7_dense_discrete::Params<double> q;
    q.ustep = p.ustep; q.tgrid = a.tgrid; q.hstep = a.hstep; q.nacc = a.nacc; q.cot = p.cot; q.saved = saved;
    q.grad_u0 = p.grad_u0; q.partial = p.partial; q.N = p.N; q.n_save = a.n_save; q.fused_l2 = p.fused_l2;
    q.t0 = a.t0; q.save_dt = a.save_dt;
    auto kern = vern7_dense_discrete::adjoint_kernel<Ops64, F64_BLOCK>;
    const size_t smem = sizeof(double) * (size_t)(F64_BLOCK / 32) * (s.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + F64_BLOCK - 1) / F64_BLOCK;
    *rows_out = grid * (F64_BLOCK / 32);
    kern<<<grid, F64_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- Fisher-KPP, adaptive Tsit5 (fkpp_adaptive.cuh in fp64) ----
cudaError_t launch_fwd_fkpp_f64(const Shape64Host &s, const Fwd64Host &p, const Adapt64Host &a, cudaStream_t st)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Fwd<double> q;
    int th;
    fkpp_adapt::cta_geometry(s.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.dense = p.dense; q.status = p.status; q.tgrid = a.tgrid; q.nacc = a.nacc;
    q.N = p.N; q.Nx = s.D; q.n_save = a.n_save; q.max_steps = a.max_steps;
    q.t0 = a.t0; q.save_dt = a.save_dt; q.abstol = a.abstol; q.reltol = a.reltol;
    auto kern = fkpp_adapt::forward_kernel<Ops64>;
    const size_t smem = fkpp_adapt::fwd_smem(s.D, sizeof(double));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<(p.N + q.tpc - 1) / q.tpc, th, smem, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp_f64(const Shape64Host &s, const Adj64Host &p, const Adapt64Host &a, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Adj<double> q;
    int th;
    fkpp_adapt::cta_geometry(s.D, &q.tpc, &th);
    q.ustep = p.ustep; q.dense = p.dense; q.tgrid = a.tgrid; q.nacc = a.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = s.D; q.n_save = a.n_save; q.t0 = a.t0; q.save_dt = a.save_dt;
    auto kern = fkpp_adapt::adjoint_kernel<Ops64>;
    const size_t smem = fkpp_adapt::adj_smem(s.D, s.P, sizeof(double));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + q.tpc - 1) / q.tpc;
    *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- Fisher-KPP, adaptive Vern7 with the discrete adjoint (fkpp_vern7_discrete.cuh in fp64) ----
cudaError_t launch_fwd_fkpp_vern7_f64(const Shape64Host &s, const Fwd64Host &p, const Adapt64Host &a, cudaStream_t st)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Fwd<double> q;
    int th;
    fkpp_adapt::cta_geometry(s.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.hstep = a.hstep; q.status = p.status; q.tgrid = a.tgrid; q.nacc = a.nacc;
    q.N = p.N; q.Nx = s.D; q.n_save = a.n_save; q.max_steps = a.max_steps;
    q.t0 = a.t0; q.save_dt = a.save_dt; q.abstol = a.abstol; q.reltol = a.reltol;
    auto kern = fkpp_vern7::vern7_forward_kernel<Ops64>;
    const size_t smem = fkpp_adapt::fwd_smem(s.D, sizeof(double));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<(p.N + q.tpc - 1) / q.tpc, th, smem, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp_vern7_f64(const Shape64Host &s, const Adj64Host &p, const Adapt64Host &a, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_shape(s, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Adj<double> q;
    int th;
    fkpp_adapt::cta_geometry(s.D, &q.tpc, &th);
    q.ustep = p.ustep; q.hstep = a.hstep; q.tgrid = a.tgrid; q.nacc = a.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = s.D; q.n_save = a.n_save; q.fused_l2 = p.fused_l2; q.t0 = a.t0; q.save_dt = a.save_dt;
    q.margin = 5e-13;   // half the clipping margin of the forward
    auto kern = fkpp_vern7::discrete_adjoint_kernel<Ops64>;
    const size_t smem = fkpp_adapt::adj_smem(s.D, s.P, sizeof(double));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + q.tpc - 1) / q.tpc;
    *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(q);
    return cudaGetLastError();
}

// fixed-order sum of the per-warp partial rows (one warp per entry; lane l sums rows l, l + 32, ... then a fixed butterfly)
static __global__ void reduce64_kernel(const double *__restrict__ partial, int nrows, int P1, double *__restrict__ grad, double *__restrict__ loss)
{
    const int lane = threadIdx.x & 31;
    const int q = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (q >= P1) return;
    double acc = 0.0;
    for (int b = lane; b < nrows; b += 32) acc += partial[(size_t)b * P1 + q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
        if (q == P1 - 1) {
            if (loss) *loss = acc;
        } else {
            grad[q] = acc;
        }
    }
}
cudaError_t launch_reduce_f64(const double *partial, int nrows, int P1, double *grad, double *loss, cudaStream_t st)
{
    reduce64_kernel<<<(P1 + 7) / 8, 256, 0, st>>>(partial, nrows, P1, grad, loss);
    return cudaGetLastError();
}

// L2 cotangent 2 w (out - data) and loss for the adaptive path (generic cotangent); one CTA, fixed order
struct LossW64 { double w[16]; };
static __global__ void l2_cot64_kernel(const double *__restrict__ out, const double *__restrict__ data, double *__restrict__ cot,
                                       double *__restrict__ loss, LossW64 lw, int D, size_t N, size_t total)
{
    __shared__ double red[1024];
    double acc = 0.0;
    for (size_t e = threadIdx.x; e < total; e += blockDim.x) {
        const int c = (int)((e / N) % (size_t)D);
        const double wgt = D <= 16 ? lw.w[c] : 1.0;
        const double r = out[e] - data[e];
        cot[e] = 2.0 * wgt * r;
        acc = fma(wgt * r, r, acc);
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0 && loss) *loss = red[0];
}
cudaError_t launch_l2_cot_f64(const Shape64Host &s, const double *out, const double *data, double *cot, double *loss, size_t N, int n_save, cudaStream_t st)
{
    LossW64 lw;
    for (int i = 0; i < 16; ++i) lw.w[i] = s.lossw[i];
    l2_cot64_kernel<<<1, 1024, 0, st>>>(out, data, cot, loss, lw, s.D, N, (size_t)n_save * s.D * N);
    return cudaGetLastError();
}

}  // namespace b200ude
