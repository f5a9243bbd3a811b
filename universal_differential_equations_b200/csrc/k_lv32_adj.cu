// k_lv32_adj.cu -- interpolating-adjoint kernels of the LV 2 -> 32 -> 32 -> 2 tanh UDE (BASELINE config 2).
#include "lv32_packed.cuh"
#include "ude_adjoint.cuh"
#include "lv32_tc.cuh"

namespace b200ude {

// rows of the per-warp partial-gradient buffer: enough for either variant (packed: one row per 64 trajectories,
// tensor-core: one row per 32)
int adj_grid_lv32(int N) { return ((N + 127) / 128) * 4; }

template <int TM, class W>
static cudaError_t launch_one(const AdjParams &p, int grid, cudaStream_t st)
{
    auto kern = lv32::adjoint_kernel<TM, W, ADJ_BLOCK_GEMM, 1>;
    constexpr size_t smem = sizeof(lv32::WarpStage3);
    static PerDeviceOnce once;
    bool &attr_set = once.flag();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    kern<<<grid, ADJ_BLOCK_GEMM, smem, st>>>(p);
    return cudaGetLastError();
}

template <int TM, int GEMM, bool DISC = false>
static cudaError_t launch_tc(const AdjParams &p, int *rows_out, cudaStream_t st)
{
    auto kern = lv32::tc::adjoint_kernel<TM, 128, 3, GEMM, false, DISC>;
    constexpr size_t smem = sizeof(lv32::tc::WarpStageT) * 4;
    static PerDeviceOnce once;
    bool &attr_set = once.flag();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    const int grid = (p.N + 127) / 128;
    *rows_out = grid * 4;
    kern<<<grid, 128, smem, st>>>(p, AdaptiveGrid{});
    return cudaGetLastError();
}

// adaptive (abstol / reltol) replay adjoint on the tensor-core kernels
template <int TM>
static cudaError_t launch_tc_adaptive(const AdjParams &p, const AdaptiveGrid &ag, int *rows_out, cudaStream_t st)
{
    auto kern = lv32::tc::adjoint_kernel<TM, 128, 3, 1, true>;
    constexpr size_t smem = sizeof(lv32::tc::WarpStageT) * 4;
    static PerDeviceOnce once;
    bool &attr_set = once.flag();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    const int grid = (p.N + 127) / 128;
    *rows_out = grid * 4;
    kern<<<grid, 128, smem, st>>>(p, ag);
    return cudaGetLastError();
}

cudaError_t launch_adj_lv32_adaptive(const Variant &v, const ConstTables &t, const AdjParams &p, const AdaptiveGrid &ag, cudaStream_t st, int *rows_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    return v.approx_tanh ? launch_tc_adaptive<1>(p, ag, rows_out, st) : launch_tc_adaptive<0>(p, ag, rows_out, st);
}

cudaError_t launch_adj_lv32(const Variant &v, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *grid_out)
{
    cudaError_t e = upload_tables(t, st);
    if (e != cudaSuccess) return e;
    if (v.discrete) return v.approx_tanh ? launch_tc<1, 1, true>(p, grid_out, st) : launch_tc<0, 1, true>(p, grid_out, st);
    if (v.adj_tc == 2) return v.approx_tanh ? launch_tc<1, 1>(p, grid_out, st) : launch_tc<0, 1>(p, grid_out, st);
    if (v.adj_tc) return v.approx_tanh ? launch_tc<1, 0>(p, grid_out, st) : launch_tc<0, 0>(p, grid_out, st);
    const int grid = ((p.N + 1) / 2 + ADJ_BLOCK_GEMM - 1) / ADJ_BLOCK_GEMM;
    *grid_out = grid;
    if (v.approx_tanh) return launch_one<1, WConst>(p, grid, st);
    return launch_one<0, WConst>(p, grid, st);
}

cudaError_t launch_reduce(const float *partial, int nblocks, int P1, float *grad, float *loss, cudaStream_t st)
{
    ude_reduce_kernel<<<(P1 + 7) / 8, 256, 0, st>>>(partial, nblocks, P1, grad, loss);
    return cudaGetLastError();
}

cudaError_t launch_reduce_exchange(const float *partial, int nblocks, int P1, const PeerLinks &pl, float *grad, float *loss, cudaStream_t st)
{
    PeerCtx c;
    for (int r = 0; r < 16; ++r) {
        c.flags[r] = r < pl.world ? reinterpret_cast<unsigned *>(pl.base[r]) : nullptr;
        c.slots[r] = r < pl.world ? reinterpret_cast<float *>(reinterpret_cast<char *>(pl.base[r]) + PEER_HEADER_BYTES) : nullptr;
    }
    c.ticket = reinterpret_cast<unsigned *>(pl.base[pl.rank]) + 16;
    c.rank = pl.rank; c.world = pl.world; c.P1pad = pl.P1pad;
    ude_reduce_exchange_kernel<<<(P1 + 7) / 8, 256, 0, st>>>(partial, nblocks, P1, c, grad, loss);
    return cudaGetLastError();
}

}  // namespace b200ude
