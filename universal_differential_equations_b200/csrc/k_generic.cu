// k_generic.cu -- shape-generic UDE kernels (runtime chain widths / activations; LV, SEIR, NODE forms) in fp32: their constant-bank
// symbols and launchers (ude_launch.cuh), the two-stage L2 cotangent, and the fixed-step Fisher-KPP kernels.
#include "ude_adjoint.cuh"
#include "ude_launch.cuh"

#include <algorithm>

namespace b200ude {

namespace generic {
struct GenDesc {
    int model, D, din, dout, n_layers, n_prefix, P;
    int widths[MAXL + 1];
    int acts[MAXL];
    int woff[MAXL];   // offset of layer l's W in theta (column-major, out x in), its bias follows at woff + in*out
};
static __constant__ GenDesc c_gen;
}  // namespace generic

// the fp32 precision of the runtime-shape model layer: theta, constants and loss weights from the constant bank, the MUFU
// activations of the specialised kernels
struct Ops32 {
    using real = float;
    using Fwd = FwdParams;
    using Adj = AdjParams;
    using Adapt = AdaptiveGrid;
    static constexpr int MAXD = generic::MAXD;
    static __device__ __forceinline__ int model() { return generic::c_gen.model; }
    static __device__ __forceinline__ int D() { return generic::c_gen.D; }
    static __device__ __forceinline__ int din() { return generic::c_gen.din; }
    static __device__ __forceinline__ int dout() { return generic::c_gen.dout; }
    static __device__ __forceinline__ int n_layers() { return generic::c_gen.n_layers; }
    static __device__ __forceinline__ int n_prefix() { return generic::c_gen.n_prefix; }
    static __device__ __forceinline__ int P() { return generic::c_gen.P; }
    static __device__ __forceinline__ int width(int l) { return generic::c_gen.widths[l]; }
    static __device__ __forceinline__ int woff(int l) { return generic::c_gen.woff[l]; }
    static __device__ __forceinline__ int layer_act(int l) { return generic::c_gen.acts[l]; }
    static __device__ __forceinline__ const float &theta(int i) { return c_theta[i]; }
    static __device__ __forceinline__ const float &consts(int i) { return c_consts[i]; }
    static __device__ __forceinline__ const float &lossw(int c) { return c_lossw[c]; }
    static __device__ __forceinline__ float act(int k, float a) { return k == ACT_TANH ? tanh_dev<0>(a) : (k == ACT_RBF ? rbf_dev(a) : a); }
};

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

template <>
struct ShapeUnit<float> {
    using Ops = Ops32;
    static constexpr int BLOCK = 128;
    static cudaError_t upload(const GenericShape &g, const ConstTables &t, cudaStream_t st)
    {
        cudaError_t e = upload_tables(t, st);
        return e != cudaSuccess ? e : upload_gen(g, st);
    }
};
template struct RuntimeShape<float>;

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

// =====================================================================================================
// Fisher-KPP UPDE, fixed step (FisherKPP/Fisher-KPP-CNN.jl:111-126, LotkaVolterra/scenario_3.jl:103-114), fp32:
//   du_i = NN(u_i) + D0 * (w1 u_{i-1} + w2 u_i + w3 u_{i+1}),  periodic, theta = [chain | w1 w2 w3 b | D0].
// One thread per grid point; a CTA holds `tpc` whole trajectories (tpc * Nx threads, rounded up to a warp
// multiple: fkpp_adapt::cta_geometry); neighbours are exchanged through shared memory.  The handle's internal stores (ustep,
// dense) are point-fastest ([row][trajectory][point]) so that every warp access is contiguous; the ABI arrays
// (u0, out, data, grad_u0) keep the documented trajectory-fastest layout.
// =====================================================================================================
static __global__ void fkpp_forward_kernel(FwdParams p, int Nx, int tpc)
{
    extern __shared__ __align__(16) float s_dyn[];
    float *sU = s_dyn;
    const int slots = tpc * Nx;
    const int slot = threadIdx.x;
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float dt = p.dt;
    const int sx = Ops32::P() - 5;
    const float w1 = Ops32::theta(sx), w2 = Ops32::theta(sx + 1), w3 = Ops32::theta(sx + 2), D0 = Ops32::theta(sx + 4);
    float u = __ldg(p.u0 + (size_t)i * N + n);
    auto rhs = [&](float g) {
        float gm, gp;
        fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
        const float y = fkpp_adapt::point_chain<Ops32>(g);
        return fmaf(D0, fmaf(w1, gm, fmaf(w2, g, w3 * gp)), y);
    };
    auto store_int = [&](float *b, int row, float v) { if (live) b[((size_t)row * N + n) * Nx + i] = v; };
    auto store_abi = [&](float *b, int row, float v) { if (live) b[((size_t)row * Nx + i) * N + n] = v; };
    store_abi(p.out, 0, u);
    store_int(p.ustep, 0, u);
    float k[7];
    k[0] = rhs(u);
    store_int(p.dense, 0, k[0]);
    int isave = 1;
    for (int s = 0; s < p.n_steps; ++s) {
#pragma unroll
        for (int st = 1; st < 7; ++st) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Tsit5::a(st, j) != 0.0) acc = fmaf((float)Tsit5::a(st, j), k[j], acc);
            const float g = fmaf(dt, acc, u);
            if (st == 6) u = g;
            k[st] = rhs(g);
            store_int(p.dense, s * 6 + st, k[st]);
        }
        store_int(p.ustep, s + 1, u);
        if ((s + 1) % p.save_every == 0) { store_abi(p.out, isave, u); ++isave; }
        k[0] = k[6];
    }
    if (p.status) {
        // a trajectory is flagged when any of its points is non-finite
        const float big = Prec<float>::huge;
        const int bad = __syncthreads_or((live && !(fabsf(u) <= big)) ? 1 : 0);   // CTA-wide; refined per trajectory below
        if (bad) {
            if (valid) sU[slot] = (fabsf(u) <= big) ? 0.0f : 1.0f;
            __syncthreads();
            if (live && i == 0) {
                float any = 0.0f;
                for (int q = 0; q < Nx; ++q) any += sU[base + q];
                p.status[n] = any > 0.0f ? 1 : 0;
            }
        } else if (live && i == 0) {
            p.status[n] = 0;
        }
    }
}

static __global__ void fkpp_adjoint_kernel(AdjParams p, int Nx, int tpc)
{
    extern __shared__ __align__(16) float s_dyn[];
    const int slots = tpc * Nx, P = Ops32::P();
    float *sU = s_dyn;                                   // [slots] neighbour exchange
    float *s_g = s_dyn + ((slots + 3) / 4) * 4;          // [nwarps][P+1]
    const int slot = threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float *gw = s_g + (size_t)warp * (P + 1);
    for (int q = lane; q < P + 1; q += 32) gw[q] = 0.0f;
    __syncwarp();
    const bool valid = slot < slots;
    const int t_loc = valid ? slot / Nx : 0, i = valid ? slot % Nx : 0;
    const int base = t_loc * Nx;
    const int traj = blockIdx.x * tpc + t_loc;
    const bool live = valid && traj < p.N;
    const size_t N = (size_t)p.N, n = (size_t)(live ? traj : p.N - 1);
    const float lv = live ? 1.0f : 0.0f;
    const float dt = p.dt;
    const int sx = P - 5;
    const float w1 = Ops32::theta(sx), w2 = Ops32::theta(sx + 1), w3 = Ops32::theta(sx + 2), D0 = Ops32::theta(sx + 4);
    float lam = 0.0f, loss = 0.0f, kl[6];
    auto jump = [&](int isave) {
        const size_t idx = ((size_t)isave * Nx + i) * N + n;   // ABI layout
        if (p.fused_l2) {
            const float r = __ldg(p.ustep + ((size_t)(isave * p.save_every) * N + n) * Nx + i) - __ldg(p.cot + idx);
            loss = fmaf(r, r, loss);
            lam = fmaf(2.0f, r, lam);
        } else {
            lam += __ldg(p.cot + idx);
        }
    };
    const int n_save = p.n_steps / p.save_every + 1;
    jump(n_save - 1);
    for (int s = p.n_steps - 1; s >= 0; --s) {
#pragma unroll
        for (int st = 0; st < 6; ++st) {
            float acc = 0.0f;
#pragma unroll
            for (int j = 0; j < 7; ++j)
                if (Tsit5::bw(st, j) != 0.0)
                    acc = fmaf((float)Tsit5::bw(st, j), __ldg(p.dense + ((size_t)(s * 6 + j) * N + n) * Nx + i), acc);
            const float x = fmaf(dt, acc, __ldg(p.ustep + ((size_t)s * N + n) * Nx + i));
            float a2 = 0.0f;
#pragma unroll
            for (int j = 0; j < st; ++j)
                if (Tsit5::a(st, j) != 0.0) a2 = fmaf((float)Tsit5::a(st, j), kl[j], a2);
            const float g = fmaf(dt, a2, lam);
            const float w = dt * (float)Tsit5::b(st) * lv;
            // neighbours of u (for the stencil-weight gradients) and of lambda (for the transposed stencil)
            float xm, xp, gm, gp;
            fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, x, xm, xp);
            fkpp_adapt::exchange(sU, slot, base, i, Nx, valid, g, gm, gp);
            const float dx = fkpp_adapt::point_chain_vjp<Ops32>(x, g, w, gw, lane);
            kl[st] = dx + D0 * fmaf(w2, g, fmaf(w1, gp, w3 * gm));   // (J^T g)_i: w1 couples i+1 -> i, w3 couples i-1 -> i
            generic::warp_acc(gw, sx + 0, w * D0 * xm * g, lane);
            generic::warp_acc(gw, sx + 1, w * D0 * x * g, lane);
            generic::warp_acc(gw, sx + 2, w * D0 * xp * g, lane);
            generic::warp_acc(gw, sx + 4, w * fmaf(w1, xm, fmaf(w2, x, w3 * xp)) * g, lane);
        }
        float acc = 0.0f;
#pragma unroll
        for (int j = 0; j < 6; ++j) acc = fmaf((float)Tsit5::b(j), kl[j], acc);
        lam = fmaf(dt, acc, lam);
        if (s % p.save_every == 0) jump(s / p.save_every);
    }
    if (p.grad_u0 && live) p.grad_u0[(size_t)i * N + n] = lam;
    loss *= lv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) gw[P] = loss;
    __syncwarp();
    float *dst = p.partial + ((size_t)blockIdx.x * (blockDim.x >> 5) + warp) * (P + 1);
    for (int q = lane; q < P + 1; q += 32) dst[q] = gw[q];
}

int adj_rows_fkpp(int N, int Nx)
{
    int tpc, th;
    fkpp_adapt::cta_geometry(Nx, &tpc, &th);
    return ((N + tpc - 1) / tpc) * (th / 32);
}

cudaError_t launch_fwd_fkpp(const GenericShape &gs, const ConstTables &t, const FwdParams &p, cudaStream_t st)
{
    cudaError_t e = ShapeUnit<float>::upload(gs, t, st);
    if (e != cudaSuccess) return e;
    int tpc, th;
    fkpp_adapt::cta_geometry(gs.D, &tpc, &th);
    const int grid = (p.N + tpc - 1) / tpc;
    fkpp_forward_kernel<<<grid, th, sizeof(float) * tpc * gs.D, st>>>(p, gs.D, tpc);
    return cudaGetLastError();
}

cudaError_t launch_adj_fkpp(const GenericShape &gs, const ConstTables &t, const AdjParams &p, cudaStream_t st, int *rows_out)
{
    cudaError_t e = ShapeUnit<float>::upload(gs, t, st);
    if (e != cudaSuccess) return e;
    int tpc, th;
    fkpp_adapt::cta_geometry(gs.D, &tpc, &th);
    const int grid = (p.N + tpc - 1) / tpc;
    const size_t smem = fkpp_adapt::adj_smem(gs.D, gs.P, sizeof(float));
    e = cudaFuncSetAttribute(fkpp_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    *rows_out = grid * (th / 32);
    fkpp_adjoint_kernel<<<grid, th, smem, st>>>(p, gs.D, tpc);
    return cudaGetLastError();
}

// ---- Fisher-KPP, adaptive (fkpp_adaptive.cuh): the shared-memory check of b200ude_create, both precisions ----
size_t fkpp_adaptive_smem(int Nx, int P, int real_bytes)
{
    return std::max(fkpp_adapt::fwd_smem(Nx, real_bytes), fkpp_adapt::adj_smem(Nx, P, real_bytes));
}

}  // namespace b200ude
