// k_fkpp.cu -- tuned Fisher-KPP UPDE kernels, reaction chain 1 -> 16 -> 16 -> 1 tanh (BASELINE config 4;
// FisherKPP/Fisher-KPP-CNN.jl:111-126 with the chain widths of the config).
#include "fkpp_tuned.cuh"

namespace b200ude {

#include <cstdlib>
// packed kernels (two adjacent grid points per thread) for even grids; B200UDE_FKPP_PACKED=0 selects the scalar ones
static bool use_packed(int Nx)
{
    const char *e = getenv("B200UDE_FKPP_PACKED");
    return (Nx % 2 == 0) && !(e && *e == '0');
}

static void geom16(int Nx, fkpp::Geom *g, int *threads)
{
    const int per_traj = use_packed(Nx) ? Nx / 2 : Nx;   // threads per trajectory
    g->Nx = Nx;
    g->tpc = per_traj >= 128 ? 1 : 128 / per_traj;
    *threads = ((g->tpc * per_traj + 31) / 32) * 32;
}

int adj_rows_fkpp16(int N, int Nx)
{
    fkpp::Geom g; int th;
    geom16(Nx, &g, &th);
    return (N + g.tpc - 1) / g.tpc;   // one partial row per CTA
}

template <int TM>
static cudaError_t fwd(const FwdParams &p, int Nx, cudaStream_t st)
{
    fkpp::Geom g; int th;
    geom16(Nx, &g, &th);
    const int grid = (p.N + g.tpc - 1) / g.tpc;
    if (use_packed(Nx)) fkpp::forward_kernel2<16, TM><<<grid, th, sizeof(float) * 2 * g.tpc * g.Nx, st>>>(p, g);   // [2][tpc * Nx/2] float2
    else fkpp::forward_kernel<16, TM><<<grid, th, sizeof(float) * 2 * g.tpc * g.Nx, st>>>(p, g);
    return cudaGetLastError();
}

template <int TM>
static cudaError_t adj(const AdjParams &p, int Nx, cudaStream_t st, int *rows_out)
{
    fkpp::Geom g; int th;
    geom16(Nx, &g, &th);
    const int grid = (p.N + g.tpc - 1) / g.tpc, nwarp = th / 32;
    const size_t red = sizeof(float) * (size_t)nwarp * (fkpp::Off<16>::P + 1);
    *rows_out = grid;
    if (use_packed(Nx)) {
        const int slots = g.tpc * (g.Nx / 2);
        size_t smem = sizeof(float) * 8 * (size_t)slots + (size_t)nwarp * sizeof(fkpp::WarpRows2<16>);
        if (red > smem) smem = red;
        auto kern = fkpp::adjoint_kernel2<16, TM>;
        static PerDeviceOnce once;
        bool &done = once.flag();
        if (!done) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
            if (e != cudaSuccess) return e;
            done = true;
        }
        kern<<<grid, th, smem, st>>>(p, g);
        return cudaGetLastError();
    }
    const int slots = g.tpc * g.Nx;
    size_t smem = sizeof(float) * 4 * (size_t)(((slots + 1) / 2) * 2) + (size_t)nwarp * sizeof(fkpp::WarpRows<16>);
    if (red > smem) smem = red;
    fkpp::adjoint_kernel<16, TM><<<grid, th, smem, st>>>(p, g);
    return cudaGetLastError();
}

// RKC2 forward / adjoint (packed kernels, even grids only)
static cudaError_t upload_rkc(const RkcHost &r, uint64_t serial, cudaStream_t st)
{
    static SerialCache cache;
    if (cache.hit(serial)) return cudaSuccess;
    fkpp::RkcTables t;
    t.s = r.s; t.mt1 = r.mt1;
    for (int j = 0; j < 65; ++j) { t.mu[j] = r.mu[j]; t.nu[j] = r.nu[j]; t.mt[j] = r.mt[j]; t.ga[j] = r.ga[j]; t.c[j] = r.c[j]; t.w[j] = r.w[j]; }
    cudaError_t e = cudaMemcpyToSymbolAsync(fkpp::c_rkc, &t, sizeof(t), 0, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess) {
        e = cudaStreamSynchronize(st);   // `t` is a stack object: the copy must have left it before we return
        cache.set(serial);
    }
    return e;
}

cudaError_t launch_fwd_fkpp16_rkc(const Variant &v, const ConstTables &t, const RkcHost &r, const FwdParams &p, int Nx, cudaStream_t st)
{
    if (Nx % 2) return cudaErrorInvalidValue;
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_rkc(r, t.serial, st);
    if (e != cudaSuccess) return e;
    fkpp::Geom g;
    g.Nx = Nx;
    g.tpc = Nx / 2 >= 128 ? 1 : 128 / (Nx / 2);
    const int th = ((g.tpc * (Nx / 2) + 31) / 32) * 32, grid = (p.N + g.tpc - 1) / g.tpc;
    const size_t smem = sizeof(float) * 2 * g.tpc * g.Nx;
    if (v.approx_tanh) fkpp::forward_rkc_kernel2<16, 1><<<grid, th, smem, st>>>(p, g);
    else fkpp::forward_rkc_kernel2<16, 0><<<grid, th, smem, st>>>(p, g);
    return cudaGetLastError();
}

template <int TM>
static cudaError_t adj_rkc(const AdjParams &p, int Nx, cudaStream_t st, int *rows_out)
{
    fkpp::Geom g;
    g.Nx = Nx;
    g.tpc = Nx / 2 >= 128 ? 1 : 128 / (Nx / 2);
    const int th = ((g.tpc * (Nx / 2) + 31) / 32) * 32, grid = (p.N + g.tpc - 1) / g.tpc, nwarp = th / 32, slots = g.tpc * (Nx / 2);
    size_t smem = sizeof(float) * 8 * (size_t)slots + (size_t)nwarp * sizeof(fkpp::WarpRows2<16>);
    const size_t red = sizeof(float) * (size_t)nwarp * (fkpp::Off<16>::P + 1);
    if (red > smem) smem = red;
    *rows_out = grid;
    auto kern = fkpp::adjoint_kernel2<16, TM, true>;
    static PerDeviceOnce once;
    bool &done = once.flag();
    if (!done) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
        if (e != cudaSuccess) return e;
        done = true;
    }
    kern<<<grid, th, smem, st>>>(p, g);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp16_rkc(const Variant &v, const ConstTables &t, const RkcHost &r, const AdjParams &p, int Nx, cudaStream_t st, int *rows_out)
{
    if (Nx % 2) return cudaErrorInvalidValue;
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    e = upload_rkc(r, t.serial, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? adj_rkc<1>(p, Nx, st, rows_out) : adj_rkc<0>(p, Nx, st, rows_out);
}

cudaError_t launch_fwd_fkpp16(const Variant &v, const ConstTables &t, const FwdParams &p, int Nx, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? fwd<1>(p, Nx, st) : fwd<0>(p, Nx, st);
}

cudaError_t launch_adj_fkpp16(const Variant &v, const ConstTables &t, const AdjParams &p, int Nx, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? adj<1>(p, Nx, st, rows_out) : adj<0>(p, Nx, st, rows_out);
}

}  // namespace b200ude
