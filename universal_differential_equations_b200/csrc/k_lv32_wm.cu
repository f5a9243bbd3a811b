// k_lv32_wm.cu -- warp-collective (mma.sync, 16 trajectories per warp) kernels of the LV 2 -> 32 -> 32 -> 2 tanh UDE:
// the low-latency family for small and medium ensembles (lv32_wm.cuh).
#include "lv32_wm.cuh"

namespace b200ude {

int adj_rows_lv32_wm(int N) { return (N + 7) / 8; }   // rows of the partial-gradient buffer: one per warp, R = 1 is the finest

static lv32::wm::Consts make_consts(const ConstTables &t)
{
    lv32::wm::Consts c;
    c.p1 = t.consts[0]; c.p4 = t.consts[1]; c.lw0 = t.lossw[0]; c.lw1 = t.lossw[1];
    return c;
}

// rows per lane: small ensembles are latency-bound -> 8 trajectories per warp (twice the warps, half the element-wise work
// per warp); larger ones are throughput-bound -> 16 per warp
static int pick_rows(const Variant &v, int N) { return v.wm_rows == 1 || v.wm_rows == 2 ? v.wm_rows : (N <= v.wm_r1_max ? 1 : 2); }

template <int TM, int G, int R>
static cudaError_t launch_fwd(const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    constexpr int WPC = 2;   // two warps share one staged copy of the weights (11.8 KB of shared memory per CTA)
    const int warps = (p.N + 8 * R * G - 1) / (8 * R * G);
    lv32::wm::forward_kernel<TM, G, R, WPC><<<(warps + WPC - 1) / WPC, 32 * WPC, lv32::wm::RAW_FLOATS * 4, st>>>(p, make_consts(t));
    return cudaGetLastError();
}

template <int TM>
static cudaError_t launch_fwd_tm(const Variant &v, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    if (pick_rows(v, p.N) == 1) return launch_fwd<TM, 1, 1>(t, p, st);
    // two groups per warp: fewer instructions per trajectory (shared weight loads and loop overhead) at 4 instead of 8 warps per
    // scheduler; pays once the ensemble still gives every scheduler two such warps (on an H100 at N = 65 536: forward 0.57 ms
    // instead of 0.63 ms)
    const int groups = v.wm_groups == 1 || v.wm_groups == 2 ? v.wm_groups : (p.N >= v.wm_g2_min ? 2 : 1);
    return groups == 2 ? launch_fwd<TM, 2, 2>(t, p, st) : launch_fwd<TM, 1, 2>(t, p, st);
}

cudaError_t launch_fwd_lv32_wm(const Variant &v, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    return v.approx_tanh ? launch_fwd_tm<1>(v, t, p, st) : launch_fwd_tm<0>(v, t, p, st);
}

template <int TM, int R>
static cudaError_t launch_adj(const ConstTables &t, const AdjParams &p, int *rows_out, cudaStream_t st)
{
    // single-warp CTAs, no register cap: a 168-register cap (3 warps per scheduler instead of 2) puts spill code in the stage loop
    constexpr int WPC = 1;
    auto kern = lv32::wm::adjoint_kernel<TM, R, WPC, 1>;
    constexpr size_t smem = lv32::wm::RAW_FLOATS * 4 + sizeof(lv32::wm::WarpTiles) * WPC;
    static PerDeviceOnce once;
    bool &attr_set = once.flag();
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    const int warps = ((p.n_cnt ? p.n_cnt : p.N) + 8 * R - 1) / (8 * R);
    *rows_out = warps;
    kern<<<(warps + WPC - 1) / WPC, 32 * WPC, smem, st>>>(p, make_consts(t));
    return cudaGetLastError();
}

cudaError_t launch_adj_lv32_wm(const Variant &v, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *rows_out)
{
    const int R = pick_rows(v, p.N);   // by the whole ensemble, also for a sub-range launch (both halves use the same rows per warp)
    if (v.approx_tanh) return R == 1 ? launch_adj<1, 1>(t, p, rows_out, st) : launch_adj<1, 2>(t, p, rows_out, st);
    return R == 1 ? launch_adj<0, 1>(t, p, rows_out, st) : launch_adj<0, 2>(t, p, rows_out, st);
}

static __global__ void tanh_selftest_kernel(const float *__restrict__ x, float *__restrict__ y, size_t n)
{
    const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    if (i >= n) return;
    float v[4];
    for (int k = 0; k < 4; ++k) v[k] = i + k < n ? x[i + k] : 0.0f;
    // the kernels' tanh on the argument z = 2 log2(e) x - 1 that their staged weights and biases produce
    float2 a = make_float2(v[0], v[1]), b = make_float2(v[2], v[3]);
    a = lv32::fma2(a, lv32::bc(lv32::TANH_K), lv32::bc(-1.0f));
    b = lv32::fma2(b, lv32::bc(lv32::TANH_K), lv32::bc(-1.0f));
    lv32::tanh_quad_z<0>(a, b);
    const float r[4] = {a.x, a.y, b.x, b.y};
    for (int k = 0; k < 4; ++k)
        if (i + k < n) y[i + k] = r[k];
}

cudaError_t launch_tanh_selftest(const float *x, float *y, size_t n, cudaStream_t st)
{
    const size_t quads = (n + 3) / 4;
    tanh_selftest_kernel<<<(unsigned)((quads + 255) / 256), 256, 0, st>>>(x, y, n);
    return cudaGetLastError();
}

}  // namespace b200ude
