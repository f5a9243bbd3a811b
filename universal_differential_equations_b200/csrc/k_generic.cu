// k_generic.cu -- shape-generic UDE kernels (runtime chain widths / activations; LV, SEIR, NODE forms).
#include "ude_generic.cuh"
#include "fkpp_adaptive.cuh"
#include "discrete_adjoint.cuh"
#include "fkpp_vern7_discrete.cuh"
#include "vern7_dense.cuh"
#include "vern7_dense_discrete.cuh"

#include <algorithm>

namespace b200ude {

constexpr int GEN_BLOCK = 128;

int adj_rows_generic(int N) { return ((N + GEN_BLOCK - 1) / GEN_BLOCK) * (GEN_BLOCK / 32); }

static cudaError_t upload_gen(const GenericShape &g, cudaStream_t st)
{
    static SerialCache cache;
    if (cache.hit(g.serial)) return cudaSuccess;
    generic::GenDesc d;
    d.model = g.model; d.D = g.D; d.din = g.din; d.dout = g.dout; d.n_layers = g.n_layers; d.n_prefix = g.n_prefix; d.P = g.P;
    int off = g.n_prefix;
    for (int l = 0; l <= generic::MAXL; ++l) d.widths[l] = l <= g.n_layers ? g.widths[l] : 0;
    for (int l = 0; l < generic::MAXL; ++l) {
        d.acts[l] = l < g.n_layers ? g.acts[l] : 0;
        d.woff[l] = off;
        if (l < g.n_layers) off += g.widths[l] * g.widths[l + 1] + g.widths[l + 1];
    }
    cudaError_t e = cudaMemcpyToSymbolAsync(generic::c_gen, &d, sizeof(d), 0, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) cache.set(g.serial);
    return e;
}

cudaError_t launch_fwd_generic(const GenericShape &g, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    generic::forward_kernel<GEN_BLOCK><<<(p.N + GEN_BLOCK - 1) / GEN_BLOCK, GEN_BLOCK, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_adj_generic(const GenericShape &g, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    auto kern = generic::adjoint_kernel<GEN_BLOCK>;
    const size_t smem = sizeof(float) * (size_t)(GEN_BLOCK / 32) * (g.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + GEN_BLOCK - 1) / GEN_BLOCK;
    *rows_out = grid * (GEN_BLOCK / 32);
    kern<<<grid, GEN_BLOCK, smem, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fwd_vern7(const GenericShape &g, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    generic::vern7_forward_kernel<GEN_BLOCK><<<(p.N + GEN_BLOCK - 1) / GEN_BLOCK, GEN_BLOCK, 0, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fwd_vern7_adaptive(const GenericShape &g, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    // the step record only for the discrete adjoint (p.ustep set); the interpolating adjoint re-solves with Tsit5
    const bool rec = p.ustep != nullptr;
    generic::AdaptParams ap{ag.t0, ag.save_dt, ag.abstol, ag.reltol, ag.n_save, ag.max_steps, rec ? ag.tgrid : nullptr, rec ? ag.nacc : nullptr,
                            rec ? ag.hstep : nullptr};
    generic::vern7_adaptive_forward_kernel<GEN_BLOCK><<<(p.N + GEN_BLOCK - 1) / GEN_BLOCK, GEN_BLOCK, 0, st>>>(p, ap);
    return cudaGetLastError();
}

// ---- discrete adjoint (discrete_adjoint.cuh in fp32: theta from the constant bank, runtime chain shape) ----
struct DiscreteOps32 {
    using real = float;
    static constexpr int MAXD = generic::MAXD;
    static __device__ __forceinline__ int D() { return generic::c_gen.D; }
    static __device__ __forceinline__ int P() { return generic::c_gen.P; }
    static __device__ __forceinline__ float lossw(int c) { return c_lossw[c]; }
    static __device__ __forceinline__ void rhs(const float *u, float *du) { generic::model_rhs(u, du); }
    static __device__ __forceinline__ void vjp(const float *u, const float *g, float lv, float *kl, float *gw, int lane)
    {
        generic::model_vjp(u, g, 1.0f, lv, kl, gw, lane);
    }
};

cudaError_t launch_adj_discrete(const GenericShape &g, const ConstTables &t, const AdjParams &p, int solver, const AdaptiveGrid *ag,
                                cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    discrete::Params<float> q;
    q.ustep = p.ustep; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.tgrid = ag ? ag->tgrid : nullptr; q.hstep = ag ? ag->hstep : nullptr; q.nacc = ag ? ag->nacc : nullptr;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ag ? ag->t0 : 0.0f; q.save_dt = ag ? ag->save_dt : 0.0f;
    q.margin = 5e-7f;   // half the clipping margin of vern7_adaptive_forward_kernel
    auto kern = solver == 1 ? discrete::adjoint_kernel<DiscreteOps32, discrete::Vern7Scheme, GEN_BLOCK>
                            : discrete::adjoint_kernel<DiscreteOps32, discrete::Tsit5Scheme, GEN_BLOCK>;
    const size_t smem = sizeof(float) * (size_t)(GEN_BLOCK / 32) * (g.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + GEN_BLOCK - 1) / GEN_BLOCK;
    *rows_out = grid * (GEN_BLOCK / 32);
    kern<<<grid, GEN_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- Vern7 with its lazy dense output (vern7_dense.cuh in fp32) ----
struct DenseOps32 : DiscreteOps32 {
    static __device__ __forceinline__ void vjp(const float *u, const float *g, float sc, float lv, float *kl, float *gw, int lane)
    {
        generic::model_vjp(u, g, sc, lv, kl, gw, lane);
    }
};

cudaError_t launch_fwd_vern7_dense(const GenericShape &g, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Fwd<float> q;
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.tgrid = ag.tgrid; q.hstep = ag.hstep; q.nacc = ag.nacc; q.status = p.status;
    q.N = p.N; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    vern7_dense::forward_kernel<DenseOps32, GEN_BLOCK><<<(p.N + GEN_BLOCK - 1) / GEN_BLOCK, GEN_BLOCK, 0, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_vern7_dense(const GenericShape &g, const ConstTables &t, const AdjParams &p, const AdaptiveGrid *ag, const float *saved,
                                   cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    vern7_dense::Adj<float> q;
    q.ustep = p.ustep; q.tgrid = ag ? ag->tgrid : nullptr; q.hstep = ag ? ag->hstep : nullptr; q.nacc = ag ? ag->nacc : nullptr;
    q.cot = p.cot; q.saved = saved; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.n_steps = p.n_steps; q.save_every = p.save_every; q.n_save = p.n_steps / p.save_every + 1; q.fused_l2 = p.fused_l2;
    q.dt = p.dt; q.t0 = ag ? ag->t0 : 0.0f; q.save_dt = ag ? ag->save_dt : 0.0f;
    auto kern = vern7_dense::adjoint_kernel<DenseOps32, GEN_BLOCK>;
    const size_t smem = sizeof(float) * (size_t)(GEN_BLOCK / 32) * (g.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + GEN_BLOCK - 1) / GEN_BLOCK;
    *rows_out = grid * (GEN_BLOCK / 32);
    kern<<<grid, GEN_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- discrete adjoint through the interpolated saves of the dense-output forward (vern7_dense_discrete.cuh in fp32) ----
cudaError_t launch_adj_vern7_dense_discrete(const GenericShape &g, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag,
                                            const float *saved, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    vern7_dense_discrete::Params<float> q;
    q.ustep = p.ustep; q.tgrid = ag.tgrid; q.hstep = ag.hstep; q.nacc = ag.nacc; q.cot = p.cot; q.saved = saved;
    q.grad_u0 = p.grad_u0; q.partial = p.partial; q.N = p.N; q.n_save = ag.n_save; q.fused_l2 = p.fused_l2;
    q.t0 = ag.t0; q.save_dt = ag.save_dt;
    auto kern = vern7_dense_discrete::adjoint_kernel<DiscreteOps32, GEN_BLOCK>;
    const size_t smem = sizeof(float) * (size_t)(GEN_BLOCK / 32) * (g.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + GEN_BLOCK - 1) / GEN_BLOCK;
    *rows_out = grid * (GEN_BLOCK / 32);
    kern<<<grid, GEN_BLOCK, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- adaptive stepping ----
cudaError_t launch_fwd_adaptive(const GenericShape &g, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    generic::AdaptParams ap{ag.t0, ag.save_dt, ag.abstol, ag.reltol, ag.n_save, ag.max_steps, ag.tgrid, ag.nacc};
    generic::adaptive_forward_kernel<GEN_BLOCK><<<(p.N + GEN_BLOCK - 1) / GEN_BLOCK, GEN_BLOCK, 0, st>>>(p, ap);
    return cudaGetLastError();
}

cudaError_t launch_adj_adaptive(const GenericShape &g, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(g, st);
    if (e != cudaSuccess) return e;
    generic::AdaptParams ap{ag.t0, ag.save_dt, ag.abstol, ag.reltol, ag.n_save, ag.max_steps, ag.tgrid, ag.nacc};
    auto kern = generic::adaptive_adjoint_kernel<GEN_BLOCK>;
    const size_t smem = sizeof(float) * (size_t)(GEN_BLOCK / 32) * (g.P + 1);
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + GEN_BLOCK - 1) / GEN_BLOCK;
    *rows_out = grid * (GEN_BLOCK / 32);
    kern<<<grid, GEN_BLOCK, smem, st>>>(p, ap);
    return cudaGetLastError();
}

// L2 cotangent 2 w (out - data) and loss for paths that take a generic cotangent (adaptive solves)
struct LossW { float w[16]; };
static __global__ void l2_cot_kernel(const float *__restrict__ out, const float *__restrict__ data, float *__restrict__ cot,
                                     float *__restrict__ block_loss, LossW lw, int D, size_t N, size_t total)
{
    __shared__ float red[256];
    float acc = 0.0f;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
        const int c = (int)((e / N) % (size_t)D);
        const float wgt = D <= 16 ? lw.w[c] : 1.0f;
        const float r = out[e] - data[e];
        cot[e] = 2.0f * wgt * r;
        acc = fmaf(wgt * r, r, acc);
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
        __syncthreads();
    }
    if (threadIdx.x == 0) block_loss[blockIdx.x] = red[0];
}
static __global__ void l2_finish_kernel(const float *__restrict__ block_loss, int nb, float *__restrict__ loss)
{
    float acc = 0.0f;
    for (int b = 0; b < nb; ++b) acc += block_loss[b];   // fixed order
    *loss = acc;
}
cudaError_t launch_l2_cot(const ConstTables &t, const float *out, const float *data, float *cot, float *block_loss, int D, size_t N, int n_save, cudaStream_t st)
{
    LossW lw;
    for (int i = 0; i < 16; ++i) lw.w[i] = t.lossw[i];
    l2_cot_kernel<<<L2_BLOCKS, 256, 0, st>>>(out, data, cot, block_loss, lw, D, N, (size_t)n_save * D * N);
    return cudaGetLastError();
}
cudaError_t launch_l2_finish(const float *block_loss, float *loss, cudaStream_t st)
{
    l2_finish_kernel<<<1, 1, 0, st>>>(block_loss, L2_BLOCKS, loss);
    return cudaGetLastError();
}

// ---- Fisher-KPP ----
static void fkpp_geom(int Nx, generic::FkppGeom *g, int *threads)
{
    g->Nx = Nx;
    g->tpc = Nx >= 128 ? 1 : 128 / Nx;
    *threads = ((g->tpc * Nx + 31) / 32) * 32;
}

int adj_rows_fkpp(int N, int Nx)
{
    generic::FkppGeom g; int th;
    fkpp_geom(Nx, &g, &th);
    return ((N + g.tpc - 1) / g.tpc) * (th / 32);
}

cudaError_t launch_fwd_fkpp(const GenericShape &gs, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    generic::FkppGeom g; int th;
    fkpp_geom(gs.D, &g, &th);
    const int grid = (p.N + g.tpc - 1) / g.tpc;
    generic::fkpp_forward_kernel<0><<<grid, th, sizeof(float) * g.tpc * g.Nx, st>>>(p, g);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp(const GenericShape &gs, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    generic::FkppGeom g; int th;
    fkpp_geom(gs.D, &g, &th);
    const int grid = (p.N + g.tpc - 1) / g.tpc;
    const size_t smem = sizeof(float) * (((g.tpc * g.Nx + 3) / 4) * 4 + (size_t)(th / 32) * (gs.P + 1));
    auto kern = generic::fkpp_adjoint_kernel<0>;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(p, g);
    return cudaGetLastError();
}

// ---- Fisher-KPP, adaptive Tsit5 (fkpp_adaptive.cuh in fp32: theta from the constant bank, runtime chain shape) ----
struct FkppOps32 {
    using real = float;
    static __device__ __forceinline__ float theta(int i) { return c_theta[i]; }
    static __device__ __forceinline__ int P() { return generic::c_gen.P; }
    static __device__ __forceinline__ float chain(float x)
    {
        float y;
        generic::chain_fwd<false>(&x, &y, nullptr, nullptr);
        return y;
    }
    static __device__ __forceinline__ float chain_vjp(float x, float dy, float w, float *gw, int lane)
    {
        float dx;
        generic::chain_vjp(&x, &dy, w, &dx, gw, lane);
        return dx;
    }
    static __device__ __forceinline__ void warp_acc(float *gw, int idx, float v, int lane) { generic::warp_acc(gw, idx, v, lane); }
    static __device__ __forceinline__ void interp(float Th, float *bw) { generic::tsit5_bw_rt(Th, bw); }
    static __device__ __forceinline__ float btilde(int j) { return generic::tsit5_btilde(j); }
};

size_t fkpp_adaptive_smem(int Nx, int P, int real_bytes)
{
    return std::max(fkpp_adapt::fwd_smem(Nx, real_bytes), fkpp_adapt::adj_smem(Nx, P, real_bytes));
}

cudaError_t launch_fwd_fkpp_adaptive(const GenericShape &gs, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Fwd<float> q;
    int th;
    fkpp_adapt::cta_geometry(gs.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.dense = p.dense; q.status = p.status; q.tgrid = ag.tgrid; q.nacc = ag.nacc;
    q.N = p.N; q.Nx = gs.D; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    auto kern = fkpp_adapt::forward_kernel<FkppOps32>;
    const size_t smem = fkpp_adapt::fwd_smem(gs.D, sizeof(float));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<(p.N + q.tpc - 1) / q.tpc, th, smem, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp_adaptive(const GenericShape &gs, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    fkpp_adapt::Adj<float> q;
    int th;
    fkpp_adapt::cta_geometry(gs.D, &q.tpc, &th);
    q.ustep = p.ustep; q.dense = p.dense; q.tgrid = ag.tgrid; q.nacc = ag.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = gs.D; q.n_save = ag.n_save; q.t0 = ag.t0; q.save_dt = ag.save_dt;
    auto kern = fkpp_adapt::adjoint_kernel<FkppOps32>;
    const size_t smem = fkpp_adapt::adj_smem(gs.D, gs.P, sizeof(float));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + q.tpc - 1) / q.tpc;
    *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(q);
    return cudaGetLastError();
}

// ---- Fisher-KPP, adaptive Vern7 with the discrete adjoint (fkpp_vern7_discrete.cuh in fp32) ----
cudaError_t launch_fwd_fkpp_vern7(const GenericShape &gs, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Fwd<float> q;
    int th;
    fkpp_adapt::cta_geometry(gs.D, &q.tpc, &th);
    q.u0 = p.u0; q.out = p.out; q.ustep = p.ustep; q.hstep = ag.hstep; q.status = p.status; q.tgrid = ag.tgrid; q.nacc = ag.nacc;
    q.N = p.N; q.Nx = gs.D; q.n_save = ag.n_save; q.max_steps = ag.max_steps;
    q.t0 = ag.t0; q.save_dt = ag.save_dt; q.abstol = ag.abstol; q.reltol = ag.reltol;
    auto kern = fkpp_vern7::vern7_forward_kernel<FkppOps32>;
    const size_t smem = fkpp_adapt::fwd_smem(gs.D, sizeof(float));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    kern<<<(p.N + q.tpc - 1) / q.tpc, th, smem, st>>>(q);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp_vern7(const GenericShape &gs, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_gen(gs, st);
    if (e != cudaSuccess) return e;
    fkpp_vern7::Adj<float> q;
    int th;
    fkpp_adapt::cta_geometry(gs.D, &q.tpc, &th);
    q.ustep = p.ustep; q.hstep = ag.hstep; q.tgrid = ag.tgrid; q.nacc = ag.nacc; q.cot = p.cot; q.grad_u0 = p.grad_u0; q.partial = p.partial;
    q.N = p.N; q.Nx = gs.D; q.n_save = ag.n_save; q.fused_l2 = p.fused_l2; q.t0 = ag.t0; q.save_dt = ag.save_dt;
    q.margin = 5e-7f;   // half the clipping margin of the forward
    auto kern = fkpp_vern7::discrete_adjoint_kernel<FkppOps32>;
    const size_t smem = fkpp_adapt::adj_smem(gs.D, gs.P, sizeof(float));
    e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + q.tpc - 1) / q.tpc;
    *rows_out = grid * (th / 32);
    kern<<<grid, th, smem, st>>>(q);
    return cudaGetLastError();
}

}  // namespace b200ude
