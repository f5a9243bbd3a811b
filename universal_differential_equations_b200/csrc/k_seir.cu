// k_seir.cu -- tensor-core kernels of the SEIR exposure UDE 3 -> 64 -> 64 -> 1 tanh (BASELINE config 3,
// SEIR_exposure/seir_exposure.jl:114-147).
#include "lv32_packed.cuh"
#include "ude_adjoint.cuh"
#include "seir_tc.cuh"

namespace b200ude {

int adj_rows_seir(int N) { return ((N + seir::BLOCK - 1) / seir::BLOCK) * seir::GROUPS; }

template <class K>
static cudaError_t set_smem(K kern, size_t smem, bool *done)
{
    if (*done) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    *done = true;
    return cudaSuccess;
}

template <int TM>
static cudaError_t launch_fwd(const FwdParams &p, cudaStream_t st)
{
    auto kern = seir::forward_kernel<TM>;
    constexpr size_t smem = (2 * seir::HS * seir::SWS + seir::BLOCK * seir::SLD64) * sizeof(float);
    static PerDeviceOnce once;
    cudaError_t e = set_smem(kern, smem, &once.flag());
    if (e != cudaSuccess) return e;
    kern<<<(p.N + seir::BLOCK - 1) / seir::BLOCK, seir::BLOCK, smem, st>>>(p);
    return cudaGetLastError();
}

template <int TM>
static cudaError_t launch_fwd_adaptive_t(const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    auto kern = seir::adaptive_forward_kernel<TM>;
    constexpr size_t smem = (2 * seir::HS * seir::SWS + seir::BLOCK * seir::SLD64) * sizeof(float);
    static PerDeviceOnce once;
    cudaError_t e = set_smem(kern, smem, &once.flag());
    if (e != cudaSuccess) return e;
    kern<<<(p.N + seir::BLOCK - 1) / seir::BLOCK, seir::BLOCK, smem, st>>>(p, ag);
    return cudaGetLastError();
}

template <int TM, int GEMM>
static cudaError_t launch_adj(const AdjParams &p, cudaStream_t st)
{
    auto kern = seir::adjoint_kernel<TM, GEMM>;
    constexpr size_t smem = 2 * seir::HS * seir::SWS * sizeof(float) + seir::GROUPS * sizeof(seir::GroupStage) + seir::BLOCK * 33 * sizeof(float);
    static PerDeviceOnce once;
    cudaError_t e = set_smem(kern, smem, &once.flag());
    if (e != cudaSuccess) return e;
    kern<<<(p.N + seir::BLOCK - 1) / seir::BLOCK, seir::BLOCK, smem, st>>>(p, AdaptiveGrid{});
    return cudaGetLastError();
}

template <int TM>
static cudaError_t launch_adj_adaptive_t(const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    auto kern = seir::adjoint_kernel<TM, 1, true>;
    constexpr size_t smem = 2 * seir::HS * seir::SWS * sizeof(float) + seir::GROUPS * sizeof(seir::GroupStage) + seir::BLOCK * 33 * sizeof(float);
    static PerDeviceOnce once;
    cudaError_t e = set_smem(kern, smem, &once.flag());
    if (e != cudaSuccess) return e;
    kern<<<(p.N + seir::BLOCK - 1) / seir::BLOCK, seir::BLOCK, smem, st>>>(p, ag);
    return cudaGetLastError();
}

cudaError_t launch_fwd_seir(const Variant &v, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? launch_fwd<1>(p, st) : launch_fwd<0>(p, st);
}

template <int TM>
static cudaError_t launch_fwd_vern7_t(const FwdParams &p, cudaStream_t st)
{
    auto kern = seir::vern7_forward_kernel<TM>;
    constexpr size_t smem = (2 * seir::HS * seir::SWS + seir::BLOCK * seir::SLD64) * sizeof(float);
    static PerDeviceOnce once;
    cudaError_t e = set_smem(kern, smem, &once.flag());
    if (e != cudaSuccess) return e;
    kern<<<(p.N + seir::BLOCK - 1) / seir::BLOCK, seir::BLOCK, smem, st>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_fwd_seir_vern7(const Variant &v, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? launch_fwd_vern7_t<1>(p, st) : launch_fwd_vern7_t<0>(p, st);
}

cudaError_t launch_adj_seir(const Variant &v, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    *rows_out = adj_rows_seir(p.N);
    if (v.adj_tc == 1) return v.approx_tanh ? launch_adj<1, 0>(p, st) : launch_adj<0, 0>(p, st);   // B200UDE_ADJ_TC=1: FFMA gradient GEMM
    return v.approx_tanh ? launch_adj<1, 1>(p, st) : launch_adj<0, 1>(p, st);
}

cudaError_t launch_fwd_seir_adaptive(const Variant &v, const ConstTables &t, const FwdParams &p, const AdaptiveGrid &ag, cudaStream_t st)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? launch_fwd_adaptive_t<1>(p, ag, st) : launch_fwd_adaptive_t<0>(p, ag, st);
}

cudaError_t launch_adj_seir_adaptive(const Variant &v, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    *rows_out = adj_rows_seir(p.N);
    return v.approx_tanh ? launch_adj_adaptive_t<1>(p, ag, st) : launch_adj_adaptive_t<0>(p, ag, st);
}

}  // namespace b200ude
