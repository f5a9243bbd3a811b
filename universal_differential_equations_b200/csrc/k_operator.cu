// k_operator.cu -- the wide-state operator UDE (operator.cuh) in fp32 and fp64.  A translation unit of its own: no existing
// kernel is recompiled with it, and the model keeps no __constant__ state (the shape travels in the kernel parameters).
#include "operator.cuh"

#include "params.h"

namespace b200ude {

namespace {
int odd(int x) { return x | 1; }
}  // namespace

void operator_layout(OperatorHost &h)
{
    const int es = h.dtype == 1 ? 8 : 4, q = 16 / es;   // the bulk copy moves a 16-byte multiple
    h.ld1 = odd(h.D);
    h.ld2 = odd(h.D);
    h.ops_elems = (op::LW + h.ld1 * h.M + h.ld2 * h.D + q - 1) / q * q;
    int off = 0, soff = 0;
    for (int l = 0; l < op::MAXL; ++l) {
        h.woff[l] = off;
        h.soff[l] = soff;
        h.ldw[l] = 0;
        if (l < h.L) {
            const int a = h.widths[l], b = h.widths[l + 1];
            h.ldw[l] = odd(b);
            off += a * b + b;
            soff += a * h.ldw[l] + b;
        }
    }
    h.P = off;
    h.theta_elems = soff;
    h.gstride = h.P + 1;
}

size_t operator_smem(const OperatorHost &h, int warps)
{
    const size_t es = h.dtype == 1 ? sizeof(double) : sizeof(float);
    return es * ((size_t)h.ops_elems + (size_t)h.theta_elems + (size_t)warps * h.gstride);
}

template <typename R>
static op::Run<R> make_run(const OperatorHost &h, const OperatorRun &r)
{
    op::Run<R> p;
    p.D = h.D; p.M = h.M; p.L = h.L; p.P = h.P; p.has_d2 = h.has_d2;
    for (int l = 0; l <= op::MAXL; ++l) p.widths[l] = h.widths[l];
    for (int l = 0; l < op::MAXL; ++l) { p.acts[l] = h.acts[l]; p.woff[l] = h.woff[l]; p.soff[l] = h.soff[l]; p.ldw[l] = h.ldw[l]; }
    p.ld1 = h.ld1; p.ld2 = h.ld2; p.ops_elems = h.ops_elems; p.theta_elems = h.theta_elems; p.gstride = h.gstride;
    p.ops = (const R *)h.ops; p.theta = (const R *)h.theta; p.rkc = (const R *)h.rkc; p.S = h.S;
    p.u0 = (const R *)r.u0; p.out = (R *)r.out; p.ustep = (R *)r.ustep; p.dense = (R *)r.dense; p.usave = (R *)r.usave;
    p.status = r.status; p.cot = (const R *)r.cot; p.grad_u0 = (R *)r.grad_u0; p.partial = (R *)r.partial; p.fused_l2 = r.fused_l2;
    p.tgrid = (R *)r.tgrid; p.nacc = r.nacc;
    p.beta = (const R *)h.beta; p.sstep = r.sstep; p.rho = (R)h.rho;
    p.N = r.N; p.n_steps = r.n_steps; p.save_every = r.save_every; p.n_save = r.n_save; p.max_steps = r.max_steps;
    p.t0 = (R)r.t0; p.dt = (R)r.dt; p.save_dt = (R)r.save_dt; p.abstol = (R)r.abstol; p.reltol = (R)r.reltol;
    return p;
}

// The dynamic shared-memory cap is set to the same device-wide value (dyn_cap) by every handle, so that host threads driving
// handles of different shapes on one device cannot lower it between another thread's set and launch.
template <typename R>
static cudaError_t launch(void (*kern)(op::Run<R>), const op::Run<R> &p, int warps, size_t smem, int dyn_cap, cudaStream_t st)
{
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dyn_cap);
    if (e != cudaSuccess) return e;
    const int grid = (p.N + warps - 1) / warps;
    kern<<<grid, warps * 32, smem, st>>>(p);
    return cudaGetLastError();
}

template <typename R>
static cudaError_t fwd(const OperatorHost &h, const OperatorRun &r, cudaStream_t st)
{
    const op::Run<R> p = make_run<R>(h, r);
    const size_t smem = operator_smem(h, 0);
    if (h.rkc2 && r.adaptive) return launch<R>(op::rkc2_adaptive_forward_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    if (h.rkc2) return launch<R>(op::rkc2_forward_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    if (r.adaptive) return launch<R>(op::tsit5_adaptive_forward_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    return launch<R>(op::tsit5_forward_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
}

template <typename R>
static cudaError_t adj(const OperatorHost &h, const OperatorRun &r, cudaStream_t st)
{
    const op::Run<R> p = make_run<R>(h, r);
    const size_t smem = operator_smem(h, h.warps);
    if (h.rkc2 && r.adaptive) return launch<R>(op::rkc2_adaptive_adjoint_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    if (h.rkc2) return launch<R>(op::rkc2_adjoint_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    if (r.adaptive) return launch<R>(op::tsit5_adaptive_adjoint_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
    return launch<R>(op::tsit5_adjoint_kernel<R>, p, h.warps, smem, h.dyn_cap, st);
}

int adj_rows_operator(int N, int warps) { return (N + warps - 1) / warps; }

template <typename R>
static cudaError_t static_smem(size_t *bytes)
{
    void (*kerns[8])(op::Run<R>) = {op::tsit5_forward_kernel<R>,         op::tsit5_adjoint_kernel<R>,
                                    op::tsit5_adaptive_forward_kernel<R>, op::tsit5_adaptive_adjoint_kernel<R>,
                                    op::rkc2_forward_kernel<R>,          op::rkc2_adjoint_kernel<R>,
                                    op::rkc2_adaptive_forward_kernel<R>, op::rkc2_adaptive_adjoint_kernel<R>};
    *bytes = 0;
    for (auto k : kerns) {
        cudaFuncAttributes a;
        const cudaError_t e = cudaFuncGetAttributes(&a, k);
        if (e != cudaSuccess) return e;
        *bytes = a.sharedSizeBytes > *bytes ? a.sharedSizeBytes : *bytes;
    }
    return cudaSuccess;
}

cudaError_t operator_static_smem(int dtype, size_t *bytes) { return dtype == 1 ? static_smem<double>(bytes) : static_smem<float>(bytes); }

cudaError_t launch_fwd_operator(const OperatorHost &h, const OperatorRun &r, cudaStream_t st)
{
    return h.dtype == 1 ? fwd<double>(h, r, st) : fwd<float>(h, r, st);
}

cudaError_t launch_adj_operator(const OperatorHost &h, const OperatorRun &r, cudaStream_t st, int *rows_out)
{
    *rows_out = adj_rows_operator(r.N, h.warps);
    return h.dtype == 1 ? adj<double>(h, r, st) : adj<float>(h, r, st);
}

}  // namespace b200ude
